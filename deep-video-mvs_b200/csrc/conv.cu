// Convolution-stack kernels, fp32 CUDA-core path (exact fp32 arithmetic; also the on-device cross-check of
// the wgmma implicit-GEMM path).  Channel-last activations.  sm_90a.
//
// Replaces (reference root relative): dvmvs/layers.py:39-65 conv_layer / depth_layer_3x3,
// dvmvs/fusionnet/model.py:15-119 building blocks (torch.cat / F.interpolate fused into the input loader),
// torchvision MnasNet _InvertedResidual depthwise convs and FeaturePyramidNetwork's top-down add.
#include <cuda_fp16.h>

#include "common.cuh"

namespace dvmvs {

// =====================================================================================================
// Generic direct convolution
// =====================================================================================================
constexpr int TH = 8, TW = 16;    // output-pixel tile
constexpr int TN = 32;            // output-channel tile
constexpr int CK = 8;             // input-channel chunk
constexpr int kConvThreads = 128; // 8 channel groups (x4) x 16 pixel groups (x8 pixels along x)

struct ConvParams {
  dvmvs_conv_desc d;
  int Hout, Wout, Cin, tiles_x, tiles_y, ksplit, chunks_total;
  size_t out_elems;
  int src_cin_offset[3];
};

__host__ __device__ constexpr int patch_h(int ks, int s) { return (TH - 1) * s + ks; }
__host__ __device__ constexpr int patch_w(int ks, int s) { return (TW - 1) * s + ks; }
__host__ __device__ constexpr int plane_stride(int ks, int s) {
  // >= PH*PW and == 4 (mod 32): the transposing smem fill (lane -> (ck, pixel)) is then bank-conflict free
  return ((patch_h(ks, s) * patch_w(ks, s) - 4 + 31) / 32) * 32 + 4;
}

// value of source `s` at input-resolution pixel (iy, ix), channel c (fuses F.interpolate x2 bilinear,
// align_corners=True: ATen upsample_bilinear2d arithmetic)
__device__ __forceinline__ float fetch_src(const dvmvs_conv_desc& d, int s, int b, int iy, int ix, int c) {
  const int Cs = d.src_channels[s];
  const float* src = d.src[s];
  if (d.src_mode[s] == DVMVS_SRC_DIRECT) return __ldg(src + (((size_t)b * d.Hin + iy) * d.Win + ix) * Cs + c);
  const int Hs = d.Hin >> 1, Ws = d.Win >> 1;
  const float sh = (d.Hin > 1) ? (float)(Hs - 1) / (float)(d.Hin - 1) : 0.f;
  const float sw = (d.Win > 1) ? (float)(Ws - 1) / (float)(d.Win - 1) : 0.f;
  const float fy = sh * iy, fx = sw * ix;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < Hs - 1), x1 = x0 + (x0 < Ws - 1);
  const float ly1 = fy - y0, lx1 = fx - x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
  const float* base = src + (size_t)b * Hs * Ws * Cs + c;
  const float v00 = __ldg(base + ((size_t)y0 * Ws + x0) * Cs), v01 = __ldg(base + ((size_t)y0 * Ws + x1) * Cs);
  const float v10 = __ldg(base + ((size_t)y1 * Ws + x0) * Cs), v11 = __ldg(base + ((size_t)y1 * Ws + x1) * Cs);
  return bilerp(ly0, ly1, lx0, lx1, v00, v01, v10, v11);
}

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == DVMVS_ACT_RELU) return fmaxf(v, 0.f);
  if (act == DVMVS_ACT_SIGMOID) return 1.f / (1.f + expf(-v));
  return v;
}

__device__ __forceinline__ float residual_at(const dvmvs_conv_desc& d, int Hout, int Wout, int b, int oy, int ox, int c) {
  if (d.residual_mode == DVMVS_RES_SAME) return __ldg(d.residual + (((size_t)b * Hout + oy) * Wout + ox) * d.Cout + c);
  const int ry = (int)(((long long)oy * d.Hr) / Hout), rx = (int)(((long long)ox * d.Wr) / Wout);   // nearest (FPN top-down)
  return __ldg(d.residual + (((size_t)b * d.Hr + ry) * d.Wr + rx) * d.Cout + c);
}

template <int KS, int STRIDE>
__global__ void __launch_bounds__(kConvThreads) conv2d_direct_kernel(ConvParams p) {
  constexpr int PH = patch_h(KS, STRIDE), PW = patch_w(KS, STRIDE), PLANE = plane_stride(KS, STRIDE);
  constexpr int PAD = (KS - 1) / 2;
  constexpr int NIV = 7 * STRIDE + KS;
  extern __shared__ __align__(16) float smem[];
  float* s_in = smem;                    // [CK][PLANE]
  float* s_w = smem + CK * PLANE;        // [KS*KS][CK][TN]

  pdl_launch_dependents();
  pdl_wait();
  const dvmvs_conv_desc& d = p.d;
  const int tid = threadIdx.x;
  const int tx = tid & 7, ty = tid >> 3;
  const int r = ty >> 1, x0 = (ty & 1) * 8;
  const int tile = blockIdx.x;
  const int ty_t = tile / p.tiles_x, tx_t = tile - ty_t * p.tiles_x;
  const int oy0 = ty_t * TH, ox0 = tx_t * TW;
  const int n0 = blockIdx.y * TN;
  const int b = blockIdx.z / p.ksplit, split = blockIdx.z - b * p.ksplit;

  float acc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int n = 0; n < 4; ++n) acc[j][n] = 0.f;

  // chunk range of this split
  const int per = (p.chunks_total + p.ksplit - 1) / p.ksplit;
  const int chunk_begin = split * per, chunk_end = min(p.chunks_total, chunk_begin + per);

  int chunk = 0;
  for (int s = 0; s < d.n_src; ++s) {
    const int Cs = d.src_channels[s];
    for (int c0 = 0; c0 < Cs; c0 += CK, ++chunk) {
      if (chunk < chunk_begin || chunk >= chunk_end) continue;
      const int nvalid = min(CK, Cs - c0);
      __syncthreads();   // previous chunk's compute done before overwrite
      // ---- input patch (transposed to [ck][pixel])
      for (int idx = tid; idx < PH * PW * CK; idx += kConvThreads) {
        const int ck = idx & (CK - 1);
        const int pp = idx >> 3;
        const int py = pp / PW, px = pp - py * PW;
        const int iy = oy0 * STRIDE - PAD + py, ix = ox0 * STRIDE - PAD + px;
        float v = 0.f;
        if (ck < nvalid && iy >= 0 && iy < d.Hin && ix >= 0 && ix < d.Win) v = fetch_src(d, s, b, iy, ix, c0 + ck);
        s_in[ck * PLANE + pp] = v;
      }
      // ---- weights [tap][ck][TN]
      const int cin0 = p.src_cin_offset[s] + c0;
      if ((d.Cout & 3) == 0) {
        for (int idx = tid; idx < KS * KS * CK * (TN / 4); idx += kConvThreads) {
          const int n4 = idx & (TN / 4 - 1);
          const int ck = (idx >> 3) & (CK - 1);
          const int tap = idx >> 6;
          float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ck < nvalid && n0 + n4 * 4 < d.Cout)
            wv = __ldg(reinterpret_cast<const float4*>(d.weight + ((size_t)tap * p.Cin + cin0 + ck) * d.Cout + n0 + n4 * 4));
          *reinterpret_cast<float4*>(s_w + (tap * CK + ck) * TN + n4 * 4) = wv;
        }
      } else {
        for (int idx = tid; idx < KS * KS * CK * TN; idx += kConvThreads) {
          const int n = idx & (TN - 1);
          const int ck = (idx >> 5) & (CK - 1);
          const int tap = idx >> 8;
          float wv = 0.f;
          if (ck < nvalid && n0 + n < d.Cout) wv = __ldg(d.weight + ((size_t)tap * p.Cin + cin0 + ck) * d.Cout + n0 + n);
          s_w[(tap * CK + ck) * TN + n] = wv;
        }
      }
      __syncthreads();
      // ---- compute
#pragma unroll 1
      for (int ky = 0; ky < KS; ++ky) {
#pragma unroll 2
        for (int ck = 0; ck < CK; ++ck) {
          const float* inrow = s_in + ck * PLANE + (r * STRIDE + ky) * PW + x0 * STRIDE;
          float iv[NIV];
#pragma unroll
          for (int i = 0; i < NIV; ++i) iv[i] = inrow[i];
#pragma unroll
          for (int kx = 0; kx < KS; ++kx) {
            const float4 wv = *reinterpret_cast<const float4*>(s_w + ((ky * KS + kx) * CK + ck) * TN + tx * 4);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float a = iv[j * STRIDE + kx];
              acc[j][0] = fmaf(a, wv.x, acc[j][0]);
              acc[j][1] = fmaf(a, wv.y, acc[j][1]);
              acc[j][2] = fmaf(a, wv.z, acc[j][2]);
              acc[j][3] = fmaf(a, wv.w, acc[j][3]);
            }
          }
        }
      }
    }
  }

  // ---- epilogue
  const int oy = oy0 + r;
  if (oy >= p.Hout) return;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ox = ox0 + x0 + j;
    if (ox >= p.Wout) continue;
    const size_t o = (((size_t)b * p.Hout + oy) * p.Wout + ox) * d.Cout;
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      const int c = n0 + tx * 4 + n;
      if (c >= d.Cout) continue;
      if (p.ksplit > 1) {
        d.workspace[(size_t)split * p.out_elems + o + c] = acc[j][n];      // partial sum; reduced in fixed order later
      } else {
        float v = acc[j][n];
        if (d.bias) v += __ldg(d.bias + c);
        if (d.residual_mode != DVMVS_RES_NONE) v += residual_at(d, p.Hout, p.Wout, b, oy, ox, c);
        v = apply_act(v, d.act);
        d.out[o + c] = v;
        if (d.aux_out) d.aux_out[o + c] = 1.f / (d.aux_mult * v + d.aux_base);
      }
    }
  }
}

// bias / residual / activation pass for split-K launches (in place on the accumulated sums)
__global__ void conv_epilogue_kernel(ConvParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const dvmvs_conv_desc& d = p.d;
  const size_t total = (size_t)d.B * p.Hout * p.Wout * d.Cout;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = (int)(idx % d.Cout);
  const size_t pix = idx / d.Cout;
  const int ox = (int)(pix % p.Wout);
  const int oy = (int)((pix / p.Wout) % p.Hout);
  const int b = (int)(pix / ((size_t)p.Wout * p.Hout));
  float v = 0.f;
  for (int sp = 0; sp < p.ksplit; ++sp) v += d.workspace[(size_t)sp * p.out_elems + idx];   // deterministic order
  if (d.bias) v += __ldg(d.bias + c);
  if (d.residual_mode != DVMVS_RES_NONE) v += residual_at(d, p.Hout, p.Wout, b, oy, ox, c);
  v = apply_act(v, d.act);
  d.out[idx] = v;
  if (d.aux_out) d.aux_out[idx] = 1.f / (d.aux_mult * v + d.aux_base);
}

// Single-output-channel 3x3 head (depth_layer_3x3): LPP lanes per output pixel (a quarter warp on large maps, a whole
// warp on the small ones, where the grid would otherwise be a handful of CTAs on the decoder's critical path), 16-byte
// channel reads, the nine taps' loads issued back to back with three independent accumulators.
template <int LPP>
__global__ void __launch_bounds__(256) conv_head_kernel(ConvParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const dvmvs_conv_desc& d = p.d;
  constexpr int PPW = 32 / LPP;                 // pixels per warp
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPP, quad = lane / LPP;
  const size_t npix = (size_t)d.B * p.Hout * p.Wout;
  const size_t pix = ((size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * PPW + quad;
  const bool active = pix < npix;
  const size_t pc = active ? pix : 0;
  const int ox = (int)(pc % p.Wout);
  const int oy = (int)((pc / p.Wout) % p.Hout);
  const int b = (int)(pc / ((size_t)p.Wout * p.Hout));
  const int C = p.Cin;
  float acc[3] = {0.f, 0.f, 0.f};
  if (active) {
    unsigned mask = 0;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int iy = oy + t / 3 - 1, ix = ox + t % 3 - 1;
      if (iy >= 0 && iy < d.Hin && ix >= 0 && ix < d.Win) mask |= 1u << t;
    }
    const float* x0 = d.src[0] + (((size_t)b * d.Hin + oy) * d.Win + ox) * C;
    for (int c = sub * 4; c < C; c += LPP * 4) {
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        if (mask & (1u << t)) {
          const float4 xv = __ldg(reinterpret_cast<const float4*>(x0 + ((long long)(t / 3 - 1) * d.Win + (t % 3 - 1)) * C + c));
          const float4 wv = __ldg(reinterpret_cast<const float4*>(d.weight + (size_t)t * C + c));
          acc[t % 3] = fmaf(xv.x, wv.x, fmaf(xv.y, wv.y, fmaf(xv.z, wv.z, fmaf(xv.w, wv.w, acc[t % 3]))));
        }
      }
    }
  }
  float a = acc[0] + acc[1] + acc[2];
#pragma unroll
  for (int o = 1; o < LPP; o <<= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (active && sub == 0) {
    float v = a + (d.bias ? __ldg(d.bias) : 0.f);
    v = apply_act(v, d.act);
    d.out[pix] = v;
    if (d.aux_out) d.aux_out[pix] = 1.f / (d.aux_mult * v + d.aux_base);
  }
}

template <int KS, int STRIDE>
static int launch_conv(const ConvParams& p, cudaStream_t s) {
  const size_t smem = (size_t)(CK * plane_stride(KS, STRIDE) + KS * KS * CK * TN) * sizeof(float);
  static PerDeviceOnce attr_set;
  if (attr_set.first()) {
    cudaFuncSetAttribute(conv2d_direct_kernel<KS, STRIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  dim3 grid(p.tiles_x * p.tiles_y, (p.d.Cout + TN - 1) / TN, p.d.B * p.ksplit);
  launch_k(conv2d_direct_kernel<KS, STRIDE>, grid, dim3(kConvThreads), smem, s, p);
  return check_launch("conv2d_direct_kernel");
}

// =====================================================================================================
// MnasNet stem: 3x3 stride-2 convolution of the (B,3,H,W) NCHW image straight to channel-last (B,H/2,W/2,32) with
// folded BN + ReLU.  One thread per output pixel and 8 output channels (4 threads share a pixel); reads the image in
// its native layout (no NCHW->NHWC pass), weights [3][3][3][32] broadcast from shared memory.
// =====================================================================================================
__global__ void __launch_bounds__(256) stem_conv_kernel(const float* __restrict__ img, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ y, int B, int H, int W,
                                                        int Cout) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_w[27 * 32];
  __shared__ float s_b[32];
  for (int i = threadIdx.x; i < 27 * Cout; i += blockDim.x) s_w[i] = w[i];
  if (threadIdx.x < Cout) s_b[threadIdx.x] = bias ? bias[threadIdx.x] : 0.f;
  __syncthreads();
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;      // k=3, pad=1, stride=2
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int cg = (int)(idx & 3);
  const size_t pix = idx >> 2;
  if (pix >= (size_t)B * Ho * Wo) return;
  const int ox = (int)(pix % Wo);
  const int oy = (int)((pix / Wo) % Ho);
  const int b = (int)(pix / ((size_t)Wo * Ho));
  float acc[8];
#pragma unroll
  for (int n = 0; n < 8; ++n) acc[n] = s_b[cg * 8 + n];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = oy * 2 - 1 + ky;
    if (iy < 0 || iy >= H) continue;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int ix = ox * 2 - 1 + kx;
      if (ix < 0 || ix >= W) continue;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = __ldg(img + (((size_t)b * 3 + c) * H + iy) * W + ix);
        const float* wp = s_w + ((ky * 3 + kx) * 3 + c) * Cout + cg * 8;
#pragma unroll
        for (int n = 0; n < 8; ++n) acc[n] = fmaf(v, wp[n], acc[n]);
      }
    }
  }
  float* o = y + pix * Cout + cg * 8;
  *reinterpret_cast<float4*>(o) = make_float4(fmaxf(acc[0], 0.f), fmaxf(acc[1], 0.f), fmaxf(acc[2], 0.f), fmaxf(acc[3], 0.f));
  *reinterpret_cast<float4*>(o + 4) = make_float4(fmaxf(acc[4], 0.f), fmaxf(acc[5], 0.f), fmaxf(acc[6], 0.f), fmaxf(acc[7], 0.f));
}

// =====================================================================================================
// Depthwise convolution
// =====================================================================================================
// KS is a template parameter so that the tap loops unroll completely: all k*k (predicated) 16-byte loads of a thread are
// in flight together instead of one load -> FMA round trip per tap (these launches are latency-bound, not bandwidth-bound).
template <int KS>
__global__ void __launch_bounds__(128) dwconv_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                     float* __restrict__ y, __half* __restrict__ planes, int B, int H, int W, int C, int Hout,
                                                     int Wout, int stride, int act) {
  constexpr int ks = KS;
  pdl_launch_dependents();
  pdl_wait();
  const int c4n = C >> 2;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)B * Hout * Wout * c4n;
  if (idx >= total) return;
  const int cg = (int)(idx % c4n);
  const size_t pix = idx / c4n;
  const int ox = (int)(pix % Wout);
  const int oy = (int)((pix / Wout) % Hout);
  const int b = (int)(pix / ((size_t)Wout * Hout));
  const int pad = ks >> 1;
  float4 acc = bias ? __ldg(reinterpret_cast<const float4*>(bias) + cg) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int ky = 0; ky < ks; ++ky) {
    const int iy = oy * stride - pad + ky;
    const bool yok = iy >= 0 && iy < H;
#pragma unroll
    for (int kx = 0; kx < ks; ++kx) {
      const int ix = ox * stride - pad + kx;
      if (!(yok && ix >= 0 && ix < W)) continue;      // predicated after unrolling; skipped taps contribute exactly 0
      const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (((size_t)b * H + iy) * W + ix) * C) + cg);
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w + (size_t)(ky * ks + kx) * C) + cg);
      acc.x = fmaf(xv.x, wv.x, acc.x);
      acc.y = fmaf(xv.y, wv.y, acc.y);
      acc.z = fmaf(xv.z, wv.z, acc.z);
      acc.w = fmaf(xv.w, wv.w, acc.w);
    }
  }
  if (act == DVMVS_ACT_RELU) {
    acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f);
  }
  if (y) reinterpret_cast<float4*>(y + pix * C)[cg] = acc;
  if (planes) {   // fp16 (hi, lo) pair for the tensor-core consumer (the pointwise projection)
    const float v[4] = {acc.x, acc.y, acc.z, acc.w};
    __align__(8) __half hi[4];
    __align__(8) __half lo[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      hi[e] = __float2half_rn(v[e]);
      lo[e] = __float2half_rn(v[e] - __half2float(hi[e]));
    }
    *reinterpret_cast<uint2*>(planes + pix * C + cg * 4) = *reinterpret_cast<const uint2*>(hi);
    *reinterpret_cast<uint2*>(planes + total * 4 + pix * C + cg * 4) = *reinterpret_cast<const uint2*>(lo);
  }
}

// =====================================================================================================
// x2 bilinear upsampling (align_corners=True)
// =====================================================================================================
__global__ void upsample2x_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
  pdl_launch_dependents();
  pdl_wait();
  const int Ho = 2 * H, Wo = 2 * W;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)B * Ho * Wo * C;
  if (idx >= total) return;
  const int c = (int)(idx % C);
  const size_t pix = idx / C;
  const int ox = (int)(pix % Wo);
  const int oy = (int)((pix / Wo) % Ho);
  const int b = (int)(pix / ((size_t)Wo * Ho));
  const float sh = (Ho > 1) ? (float)(H - 1) / (float)(Ho - 1) : 0.f;
  const float sw = (Wo > 1) ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
  const float fy = sh * oy, fx = sw * ox;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < H - 1), x1 = x0 + (x0 < W - 1);
  const float ly1 = fy - y0, lx1 = fx - x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
  const float* base = x + (size_t)b * H * W * C + c;
  const float v00 = __ldg(base + ((size_t)y0 * W + x0) * C), v01 = __ldg(base + ((size_t)y0 * W + x1) * C);
  const float v10 = __ldg(base + ((size_t)y1 * W + x0) * C), v11 = __ldg(base + ((size_t)y1 * W + x1) * C);
  y[idx] = bilerp(ly0, ly1, lx0, lx1, v00, v01, v10, v11);
}

// =====================================================================================================
// Layout: per batch, transpose the [R][Cc] matrix to [Cc][R] through a 32x33 shared tile
// =====================================================================================================
__global__ void transpose_kernel(const float* __restrict__ x, float* __restrict__ y, int R, int Cc) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float tile[32][33];
  const size_t boff = (size_t)blockIdx.z * R * Cc;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    if (r < R && c < Cc) tile[i][threadIdx.x] = x[boff + (size_t)r * Cc + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < R && c < Cc) y[boff + (size_t)c * R + r] = tile[threadIdx.x][i];
  }
}

// =====================================================================================================
// ConvLSTM gate epilogue (convlstm.py:45-59).  Block = 32 channels (lanes) x NW warps striding over pixels.
// =====================================================================================================
__device__ __forceinline__ float celu1(float x) { return x > 0.f ? x : expm1f(x); }
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

constexpr int kLstmWarps = 8;

// A block owns CPB channels of one clip over all h*w positions (LayerNorm reduces over the positions): a warp covers CPB
// channels x (32 / CPB) positions, so every load instruction reads (32 / CPB) contiguous 4*CPB-byte spans.  CPB = 32 is the wide
// form (C/32 blocks per clip); CPB = 8 quadruples the number of blocks -- the kernel sits on the loop-carried critical path of
// the pipeline and at batch 1 reads ~5 MB of split-K partial sums with C/32 = 16 blocks otherwise.
// PPW = positions per thread, a template parameter so that each thread's gate / cell values are loaded ONCE, all loads in
// flight together, and stay in registers across the four reduction passes.
template <int PPW, int CPB>
__global__ void __launch_bounds__(32 * kLstmWarps) lstm_gates_kernel(const float* __restrict__ gates, int n_parts, size_t part_stride,
                                                                     const float* __restrict__ addend, const float* __restrict__ c_in,
                                                                     float* __restrict__ h_out, float* __restrict__ c_out, int hw, int C) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int kSub = 32 / CPB;                     // positions per warp pass
  constexpr int kStride = kLstmWarps * kSub;         // positions per block pass
  __shared__ float s_red[kLstmWarps * CPB];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cl = lane % CPB, sub = lane / CPB;
  const int c = blockIdx.x * CPB + cl;
  const int b = blockIdx.y;
  const int p0 = warp * kSub + sub;                  // this thread's positions: p0 + j * kStride
  const float* g = gates + (size_t)b * hw * 4 * C;
  const float* ad = addend ? addend + (size_t)b * hw * 4 * C : nullptr;
  const float inv_n = 1.f / (float)hw;
  // gate pre-activations = sum of the n_parts split-K partial sums of the gate convolution, in split order (what
  // conv_tc_finish_kernel computes), + the state-independent half `addend`: the finishing pass of the GEMM is this epilogue
  auto pre = [&](size_t off) -> float {
    float x = 0.f;
    for (int sp = 0; sp < n_parts; ++sp) x += g[(size_t)sp * part_stride + off];
    if (ad) x += __ldg(ad + off);
    return x;
  };

  auto block_sum = [&](float v) -> float {           // sum over all positions for this thread's channel
#pragma unroll
    for (int o = CPB; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (sub == 0) s_red[warp * CPB + cl] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < kLstmWarps; ++i) t += s_red[i * CPB + cl];
    return t;
  };

  float vi[PPW], vf[PPW], vo[PPW], vg[PPW], vc[PPW];
#pragma unroll
  for (int j = 0; j < PPW; ++j) {
    const int p = p0 + j * kStride;
    const bool ok = p < hw;
    const size_t gp = (size_t)(ok ? p : 0) * 4 * C;
    vi[j] = ok ? pre(gp + c) : 0.f;
    vf[j] = ok ? pre(gp + C + c) : 0.f;
    vo[j] = ok ? pre(gp + 2 * C + c) : 0.f;
    vg[j] = ok ? pre(gp + 3 * C + c) : 0.f;
    vc[j] = ok ? c_in[((size_t)b * hw + (ok ? p : 0)) * C + c] : 0.f;
  }
  // LayerNorm statistics of cc_g over the spatial positions (two-pass: mean, then centred variance)
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < PPW; ++j) s += vg[j];                  // absent positions hold 0
  const float mean_g = block_sum(s) * inv_n;
  s = 0.f;
#pragma unroll
  for (int j = 0; j < PPW; ++j) {
    const float dlt = vg[j] - mean_g;
    if (p0 + j * kStride < hw) s += dlt * dlt;
  }
  const float rstd_g = rsqrtf(block_sum(s) * inv_n + 1e-5f);
  // c_next (pre-LN) = f*c + i*celu(LN(cc_g))
  s = 0.f;
#pragma unroll
  for (int j = 0; j < PPW; ++j) {
    const float ig = sigmoidf_(vi[j]), fg = sigmoidf_(vf[j]);
    const float gg = celu1((vg[j] - mean_g) * rstd_g);
    vg[j] = (p0 + j * kStride < hw) ? fg * vc[j] + ig * gg : 0.f;      // vg now holds c_next (pre-LN)
    s += vg[j];
  }
  const float mean_c = block_sum(s) * inv_n;
  s = 0.f;
#pragma unroll
  for (int j = 0; j < PPW; ++j) {
    const float dlt = vg[j] - mean_c;
    if (p0 + j * kStride < hw) s += dlt * dlt;
  }
  const float rstd_c = rsqrtf(block_sum(s) * inv_n + 1e-5f);
#pragma unroll
  for (int j = 0; j < PPW; ++j) {
    const int p = p0 + j * kStride;
    if (p < hw) {
      const float cn = (vg[j] - mean_c) * rstd_c;
      c_out[((size_t)b * hw + p) * C + c] = cn;
      h_out[((size_t)b * hw + p) * C + c] = sigmoidf_(vo[j]) * celu1(cn);
    }
  }
}

}  // namespace dvmvs

using namespace dvmvs;

extern "C" int dvmvs_conv2d(const dvmvs_conv_desc* desc, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(desc != nullptr, "conv2d: null descriptor");
  ConvParams p;
  p.d = *desc;
  const dvmvs_conv_desc& d = p.d;
  DVMVS_REQUIRE(d.n_src >= 1 && d.n_src <= 3, "conv2d: n_src=%d", d.n_src);
  DVMVS_REQUIRE(d.ksize == 1 || d.ksize == 3 || d.ksize == 5, "conv2d: ksize=%d", d.ksize);
  DVMVS_REQUIRE(d.stride == 1 || d.stride == 2, "conv2d: stride=%d", d.stride);
  DVMVS_REQUIRE(d.B > 0 && d.Hin > 0 && d.Win > 0 && d.Cout > 0 && d.weight && d.out, "conv2d: bad shape / null pointer");
  DVMVS_REQUIRE(d.act >= 0 && d.act <= 2, "conv2d: act=%d", d.act);
  p.Cin = 0;
  p.chunks_total = 0;
  for (int s = 0; s < d.n_src; ++s) {
    DVMVS_REQUIRE(d.src[s] && d.src_channels[s] > 0, "conv2d: source %d null/empty", s);
    DVMVS_REQUIRE(d.src_mode[s] == DVMVS_SRC_DIRECT || (d.src_mode[s] == DVMVS_SRC_UPSAMPLE2X && d.Hin % 2 == 0 && d.Win % 2 == 0),
                  "conv2d: source %d bad mode", s);
    p.src_cin_offset[s] = p.Cin;
    p.Cin += d.src_channels[s];
    p.chunks_total += (d.src_channels[s] + CK - 1) / CK;
  }
  const int pad = (d.ksize - 1) / 2;
  p.Hout = (d.Hin + 2 * pad - d.ksize) / d.stride + 1;
  p.Wout = (d.Win + 2 * pad - d.ksize) / d.stride + 1;
  DVMVS_REQUIRE(d.residual_mode == DVMVS_RES_NONE || d.residual, "conv2d: residual pointer missing");
  DVMVS_REQUIRE(d.residual_mode != DVMVS_RES_NEAREST_UP || (d.Hr > 0 && d.Wr > 0), "conv2d: residual size missing");
  cudaStream_t s = (cudaStream_t)stream;

  // single-channel 3x3 head
  if (d.Cout == 1 && d.n_src == 1 && d.src_mode[0] == DVMVS_SRC_DIRECT && d.ksize == 3 && d.stride == 1 && p.Cin % 32 == 0 &&
      d.residual_mode == DVMVS_RES_NONE && ((uintptr_t)d.src[0] % 16 == 0) && ((uintptr_t)d.weight % 16 == 0)) {
    p.ksplit = 1;
    const size_t npix = (size_t)d.B * p.Hout * p.Wout;
    if (npix <= 4096 && p.Cin >= 128) {                      // small map, many channels: a warp per pixel
      launch_k(conv_head_kernel<32>, dim3((unsigned)((npix + 7) / 8)), dim3(256), 0, s, p);
    } else {                                                 // 8 warps x 4 pixels
      launch_k(conv_head_kernel<8>, dim3((unsigned)((npix + 31) / 32)), dim3(256), 0, s, p);
    }
    return check_launch("conv_head_kernel");
  }

  DVMVS_REQUIRE((d.Cout % 4 != 0) || ((uintptr_t)d.weight % 16 == 0), "conv2d: weight must be 16-byte aligned");
  p.tiles_x = (p.Wout + TW - 1) / TW;
  p.tiles_y = (p.Hout + TH - 1) / TH;
  const int ctas = p.tiles_x * p.tiles_y * ((d.Cout + TN - 1) / TN) * d.B;
  p.ksplit = 1;
  p.out_elems = (size_t)d.B * p.Hout * p.Wout * d.Cout;
  if (ctas < 96 && p.chunks_total >= 8 && d.workspace) {   // under-filled grid: split the reduction over input-channel chunks
    int want = (296 + ctas - 1) / ctas;
    int maxsplit = p.chunks_total / 4;
    long long fit = d.workspace_bytes / (long long)(p.out_elems * sizeof(float));
    p.ksplit = (int)max(1LL, min((long long)min(want, maxsplit), fit));
  }
  int rc;
  if (d.ksize == 1 && d.stride == 1) rc = launch_conv<1, 1>(p, s);
  else if (d.ksize == 1 && d.stride == 2) rc = launch_conv<1, 2>(p, s);
  else if (d.ksize == 3 && d.stride == 1) rc = launch_conv<3, 1>(p, s);
  else if (d.ksize == 3 && d.stride == 2) rc = launch_conv<3, 2>(p, s);
  else if (d.ksize == 5 && d.stride == 1) rc = launch_conv<5, 1>(p, s);
  else rc = launch_conv<5, 2>(p, s);
  if (rc != DVMVS_OK) return rc;
  if (p.ksplit > 1) {
    const size_t total = (size_t)d.B * p.Hout * p.Wout * d.Cout;
    launch_k(conv_epilogue_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, p);
    return check_launch("conv_epilogue_kernel");
  }
  return DVMVS_OK;
}

extern "C" int dvmvs_stem_conv(const float* image_nchw, const float* weight, const float* bias, float* y, int B, int H, int W,
                               dvmvs_stream_t stream) {
  DVMVS_REQUIRE(image_nchw && weight && y && B > 0 && H > 1 && W > 1, "stem_conv: bad argument");
  DVMVS_REQUIRE((uintptr_t)y % 16 == 0, "stem_conv: output must be 16-byte aligned");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const size_t threads = (size_t)B * Ho * Wo * 4;
  launch_k(stem_conv_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, image_nchw, weight, bias, y, B,
           H, W, 32);
  return check_launch("stem_conv_kernel");
}

extern "C" int dvmvs_dwconv2d(const float* x, const float* weight, const float* bias, float* y, void* y_planes, int B, int H, int W,
                              int C, int ksize, int stride, int act, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(x && weight && (y || y_planes), "dwconv2d: null pointer");
  DVMVS_REQUIRE(!y_planes || C % 8 == 0, "dwconv2d: fp16-pair output needs C %% 8 == 0");
  DVMVS_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "dwconv2d: bad shape (C must be a multiple of 4)");
  DVMVS_REQUIRE((ksize == 3 || ksize == 5) && (stride == 1 || stride == 2), "dwconv2d: ksize/stride");
  DVMVS_REQUIRE(act == DVMVS_ACT_NONE || act == DVMVS_ACT_RELU, "dwconv2d: act");
  DVMVS_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)weight % 16 == 0 && (uintptr_t)y % 16 == 0 && (!bias || (uintptr_t)bias % 16 == 0) &&
                    (uintptr_t)y_planes % 16 == 0,
                "dwconv2d: pointers must be 16-byte aligned");
  const int pad = ksize / 2;
  const int Hout = (H + 2 * pad - ksize) / stride + 1, Wout = (W + 2 * pad - ksize) / stride + 1;
  const size_t total = (size_t)B * Hout * Wout * (C / 4);
  if (ksize == 3)
    launch_k(dwconv_kernel<3>, dim3((unsigned)((total + 127) / 128)), dim3(128), 0, (cudaStream_t)stream, x, weight, bias, y, (__half*)y_planes,
             B, H, W, C, Hout, Wout, stride, act);
  else
    launch_k(dwconv_kernel<5>, dim3((unsigned)((total + 127) / 128)), dim3(128), 0, (cudaStream_t)stream, x, weight, bias, y, (__half*)y_planes,
             B, H, W, C, Hout, Wout, stride, act);
  return check_launch("dwconv_kernel");
}

extern "C" int dvmvs_lstm_gates_parts(const float* gate_parts, int n_parts, long long part_stride, const float* addend, const float* c_in,
                                      float* h_out, float* c_out, int B, int h, int w, int C, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(gate_parts && c_in && h_out && c_out, "lstm_gates: null pointer");
  DVMVS_REQUIRE(B > 0 && h > 0 && w > 0 && C > 0 && C % 32 == 0, "lstm_gates: bad shape (C must be a multiple of 32)");
  DVMVS_REQUIRE(n_parts >= 1 && (n_parts == 1 || part_stride >= (long long)B * h * w * 4 * C), "lstm_gates: bad partial-sum layout");
  const int hw = h * w;
  cudaStream_t st = (cudaStream_t)stream;
  // few (clip, 32-channel) blocks: narrow blocks of 8 channels put four times as many CTAs on the reduction of the partial sums
  const bool narrow = (B * (C / 32) < 74) && hw <= 8 * 4 * 16;
  if (narrow) {
    const int ppw = (hw + kLstmWarps * 4 - 1) / (kLstmWarps * 4);
    dim3 grid(C / 8, B);
    if (ppw <= 2) launch_k(lstm_gates_kernel<2, 8>, grid, dim3(32 * kLstmWarps), 0, st, gate_parts, n_parts, (size_t)part_stride, addend, c_in, h_out, c_out, hw, C);
    else if (ppw <= 4) launch_k(lstm_gates_kernel<4, 8>, grid, dim3(32 * kLstmWarps), 0, st, gate_parts, n_parts, (size_t)part_stride, addend, c_in, h_out, c_out, hw, C);
    else launch_k(lstm_gates_kernel<16, 8>, grid, dim3(32 * kLstmWarps), 0, st, gate_parts, n_parts, (size_t)part_stride, addend, c_in, h_out, c_out, hw, C);
    return check_launch("lstm_gates_kernel");
  }
  const int ppw = (hw + kLstmWarps - 1) / kLstmWarps;
  DVMVS_REQUIRE(ppw <= 64, "lstm_gates: h*w=%d too large (bottleneck maps up to 512 positions)", hw);
  dim3 grid(C / 32, B);
  const size_t ps = (size_t)part_stride;
  if (ppw <= 2) launch_k(lstm_gates_kernel<2, 32>, grid, dim3(32 * kLstmWarps), 0, st, gate_parts, n_parts, ps, addend, c_in, h_out, c_out, hw, C);
  else if (ppw <= 8) launch_k(lstm_gates_kernel<8, 32>, grid, dim3(32 * kLstmWarps), 0, st, gate_parts, n_parts, ps, addend, c_in, h_out, c_out, hw, C);
  else if (ppw <= 16) launch_k(lstm_gates_kernel<16, 32>, grid, dim3(32 * kLstmWarps), 0, st, gate_parts, n_parts, ps, addend, c_in, h_out, c_out, hw, C);
  else launch_k(lstm_gates_kernel<64, 32>, grid, dim3(32 * kLstmWarps), 0, st, gate_parts, n_parts, ps, addend, c_in, h_out, c_out, hw, C);
  return check_launch("lstm_gates_kernel");
}

extern "C" int dvmvs_lstm_gates(const float* gates, const float* c_in, float* h_out, float* c_out, int B, int h, int w, int C,
                                dvmvs_stream_t stream) {
  return dvmvs_lstm_gates_parts(gates, 1, 0, nullptr, c_in, h_out, c_out, B, h, w, C, stream);
}

extern "C" int dvmvs_upsample2x(const float* x, float* y, int B, int H, int W, int C, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(x && y && B > 0 && H > 0 && W > 0 && C > 0, "upsample2x: bad argument");
  const size_t total = (size_t)B * 4 * H * W * C;
  launch_k(upsample2x_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, x, y, B, H, W, C);
  return check_launch("upsample2x_kernel");
}

static int launch_transpose(const float* x, float* y, int B, int R, int Cc, cudaStream_t s) {
  dim3 grid((Cc + 31) / 32, (R + 31) / 32, B), block(32, 8);
  launch_k(transpose_kernel, grid, block, 0, s, x, y, R, Cc);
  return check_launch("transpose_kernel");
}

extern "C" int dvmvs_nchw_to_nhwc(const float* x, float* y, int B, int C, int H, int W, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(x && y && B > 0 && C > 0 && H > 0 && W > 0, "nchw_to_nhwc: bad argument");
  return launch_transpose(x, y, B, C, H * W, (cudaStream_t)stream);
}

extern "C" int dvmvs_nhwc_to_nchw(const float* x, float* y, int B, int C, int H, int W, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(x && y && B > 0 && C > 0 && H > 0 && W > 0, "nhwc_to_nchw: bad argument");
  return launch_transpose(x, y, B, H * W, C, (cudaStream_t)stream);
}
