// Implicit-GEMM convolution on the Hopper tensor cores (wgmma.mma_async, register accumulators, TMA-fed tiles).
// sm_90a only.
//
//   D[128 output pixels x BLOCK_N output channels] (fp32, registers) += A[128 x K] . W[BLOCK_N x K]^T
//
// * A is never materialised: for every filter tap (ky,kx) and every 32/64-channel chunk of every concatenated
//   source, ONE 4-D TMA box {channels, TW, TH, 1} of the channel-last fp16 activation tensor is loaded at the
//   tap-shifted coordinates; out-of-image pixels and channels beyond the tensor are zero-filled by the TMA unit
//   (= zero padding and channel padding for free).  The box lands in shared memory as 128 rows of 64/128 bytes in
//   the canonical K-major SWIZZLE_64B/128B layout that the wgmma shared-memory descriptor expects.
// * torch.cat of the reference (model.py:112,115,208,...; convlstm.py:43) is a K-split over up to three sources.
// * Precision: activations and weights are carried as fp16 (hi, lo) pairs, x = hi + lo to ~22 bits.  A k-block
//   issues hi*hi + lo*hi + hi*lo (3 MMAs per K=16 step, fp32 accumulate), which reproduces fp32 convolution to
//   ~1e-6 -- the parity budget (1e-3 on inverse depth) does not admit plain bf16/fp16/tf32 (SURVEY.md section 0).
//   `terms` = 1 runs plain fp16 (hi*hi) for layers that tolerate it.
// * Warp roles (160 threads): warps 0-3 = one warpgroup that issues the MMAs (two m64 halves of the 128-row tile) and runs
//   the epilogue (accumulators -> shared-memory staging tile -> bias/residual/activation -> fp32 and/or fp16-pair stores),
//   warp 4 = TMA producer.  smem ring of kStages stages with full/empty mbarriers; one MMA batch stays in flight while the
//   previous stage is released.
// * Small-M layers (8x8 .. 16x16 maps) split K (filter taps) over blockIdx.z: every split publishes fp32 partial sums,
//   a finishing kernel reduces them in split order (deterministic) and applies the epilogue.
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <unordered_map>

#include "tc_ptx.cuh"

namespace dvmvs {

// ----------------------------------------------------------------------------------------------- parameters
constexpr int kTcThreads = 160;     // warps 0-3: MMA warpgroup + epilogue, warp 4: TMA producer
constexpr int kTileM = 128;


struct TcParams {
  CUtensorMap a_map[3][2];    // [source][hi/lo]
  CUtensorMap w_map[2][2];    // [chunk kind: 0 = 32-wide (SW64), 1 = 64-wide (SW128)][hi/lo]
  int src_chunks[3];          // number of K chunks per tap for each source
  int src_kchunk[3];          // 32 or 64
  int n_src, terms;           // terms: 1 = hi*hi, 3 = hi*hi + lo*hi + hi*lo
  int ksize, pad, stride;
  int B, Hout, Wout, Cout, tile_w, tile_h, tiles_x, tiles_y;
  int ksplit, k_per_tap;      // k_per_tap: packed-weight columns consumed per tap
  const float* bias;
  const float* residual;
  int residual_mode, Hr, Wr;
  float* out_f32;             // [B][Hout][Wout][Cout] or null
  __half* out_planes;         // [2][B][Hout][Wout][Cout] or null
  __half* out_blk;            // blocked planes [2][B][Cout/8][Hout][Wout][8] or null (operand layout of conv_halo_kernel)
  float* aux_out;
  float aux_mult, aux_base;
  int act;
  float* workspace;           // split-K partial sums [ksplit][out elements]
  int hi_only;                // fp16 outputs: write the hi plane only (every consumer runs 1-term products)
  int num_stages, stage_bytes, a_bytes, w_bytes;   // smem ring geometry (runtime: sized by the widest K chunk in use)
  int ring_bytes;             // ring, or the epilogue's accumulator staging tile that reuses it, whichever is larger
};

constexpr int kMaxStages = 8;
constexpr int kBarrierBytes = 256;   // full[8] + empty[8]
constexpr int kMaxSmemBytes = 227 * 1024;

// fp32 accumulator staging tile [128][BLOCK_N + 4]: the pitch keeps the epilogue's 16-byte row reads conflict-free
template <int BLOCK_N>
constexpr int tc_staging_bytes() { return kTileM * (BLOCK_N + 4) * 4; }

// bias / residual / activation and all requested output formats for 8 consecutive output channels of one pixel
__device__ __forceinline__ void tc_emit8(const TcParams& p, float (&v)[8], int b, int oy, int ox, int cbase) {
  const size_t pix = ((size_t)b * p.Hout + oy) * p.Wout + ox;
  const size_t plane_stride = (size_t)p.B * p.Hout * p.Wout * p.Cout;
  if (p.bias) {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + cbase)), b1 = __ldg(reinterpret_cast<const float4*>(p.bias + cbase + 4));
    v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w; v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
  }
  const float* res_row = nullptr;
  if (p.residual_mode == DVMVS_RES_SAME) {
    res_row = p.residual + pix * p.Cout;
  } else if (p.residual_mode == DVMVS_RES_NEAREST_UP) {
    const int ry = (int)(((long long)oy * p.Hr) / p.Hout), rx = (int)(((long long)ox * p.Wr) / p.Wout);
    res_row = p.residual + (((size_t)b * p.Hr + ry) * p.Wr + rx) * p.Cout;
  }
  if (res_row) {
    const float4 r0 = __ldg(reinterpret_cast<const float4*>(res_row + cbase)), r1 = __ldg(reinterpret_cast<const float4*>(res_row + cbase + 4));
    v[0] += r0.x; v[1] += r0.y; v[2] += r0.z; v[3] += r0.w; v[4] += r1.x; v[5] += r1.y; v[6] += r1.z; v[7] += r1.w;
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = tc_act(v[e], p.act);
  if (p.out_f32) {
    float* o = p.out_f32 + pix * p.Cout + cbase;
    *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
  if (p.aux_out) {
    float* o = p.aux_out + pix * p.Cout + cbase;
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = 1.f / (p.aux_mult * v[e] + p.aux_base);
  }
  if (p.out_planes) {
    __align__(16) __half hi[8];
    __align__(16) __half lo[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      hi[e] = __float2half_rn(v[e]);
      lo[e] = __float2half_rn(v[e] - __half2float(hi[e]));
    }
    __half* oh = p.out_planes + pix * p.Cout + cbase;
    *reinterpret_cast<uint4*>(oh) = *reinterpret_cast<const uint4*>(hi);
    if (!p.hi_only) *reinterpret_cast<uint4*>(oh + plane_stride) = *reinterpret_cast<const uint4*>(lo);
    if (p.out_blk) {
      __half* ob = p.out_blk + ((((size_t)b * (p.Cout >> 3) + (cbase >> 3)) * p.Hout + oy) * p.Wout + ox) * 8;
      *reinterpret_cast<uint4*>(ob) = *reinterpret_cast<const uint4*>(hi);
      if (!p.hi_only) *reinterpret_cast<uint4*>(ob + plane_stride) = *reinterpret_cast<const uint4*>(lo);
    }
  }
}

// the MMAs of one ring stage, issued by the whole warpgroup and committed as one group: KSTEPS = K chunk / 16 (2: 32-channel
// chunks in SWIZZLE_64B rows, 4: 64-channel chunks in SWIZZLE_128B rows), TERMS = hi*hi (+ lo*hi + hi*lo)
template <int BLOCK_N, int KSTEPS, int TERMS>
__device__ __forceinline__ void tc_mma_chunk(float (&acc)[2][BLOCK_N / 2], uint32_t sb, uint32_t off_a_lo, uint32_t off_w_hi, uint32_t off_w_lo) {
  constexpr uint32_t layout = (KSTEPS == 4) ? kGmmaSw128 : kGmmaSw64;
  constexpr uint32_t sbo = KSTEPS * 256u;                 // 8 rows x row bytes
  constexpr uint32_t half_rows = 64u * KSTEPS * 32u;      // byte offset of A rows [64, 128)
  wgmma_fence_regs(acc[0]);
  wgmma_fence_regs(acc[1]);
  wgmma_fence();
#pragma unroll
  for (int term = 0; term < TERMS; ++term) {
    const uint32_t a_s = sb + ((term == 1) ? off_a_lo : 0u);
    const uint32_t w_s = sb + ((term == 2) ? off_w_lo : off_w_hi);
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k) {          // a K step of 16 fp16 = 32 bytes along the swizzled rows
      const uint64_t bd = gmma_desc(w_s + 32u * k, 16u, sbo, layout);
      wgmma_f16<BLOCK_N>(acc[0], gmma_desc(a_s + 32u * k, 16u, sbo, layout), bd);
      wgmma_f16<BLOCK_N>(acc[1], gmma_desc(a_s + half_rows + 32u * k, 16u, sbo, layout), bd);
    }
  }
  wgmma_commit();
}

template <int BLOCK_N>
__global__ void __launch_bounds__(kTcThreads) conv_tc_kernel(const __grid_constant__ TcParams p) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;          // SWIZZLE_128B tiles need 1024-byte alignment
  uint8_t* base_ptr = smem_raw + (base - raw_addr);
  const int n_stages = p.num_stages;
  const uint32_t bars = base + p.ring_bytes;
  // barrier layout (8 bytes each): full[8], empty[8]
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (kMaxStages + s); };
  const uint32_t off_a_lo = p.a_bytes, off_w_hi = (p.terms > 1 ? 2u : 1u) * p.a_bytes, off_w_lo = off_w_hi + p.w_bytes;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int b = blockIdx.x / tiles_per_img;
  const int t_in = blockIdx.x - b * tiles_per_img;
  const int oy0 = (t_in / p.tiles_x) * p.tile_h, ox0 = (t_in % p.tiles_x) * p.tile_w;
  const int n0 = blockIdx.y * BLOCK_N;
  const int n_taps = p.ksize * p.ksize;
  const int taps_per_split = (n_taps + p.ksplit - 1) / p.ksplit;
  const int tap_begin = blockIdx.z * taps_per_split, tap_end = min(n_taps, tap_begin + taps_per_split);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.n_src; ++s) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&p.a_map[s][0]) : "memory");
      if (p.terms > 1) asm volatile("prefetch.tensormap [%0];" ::"l"(&p.a_map[s][1]) : "memory");
    }
    for (int s = 0; s < n_stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4);        // one arrival per MMA warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();      // everything above touched only this CTA's smem; global reads (TMA) and writes start below

  if (warp == 4) {
    // ============================== TMA producer ==============================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tap = tap_begin; tap < tap_end; ++tap) {
        const int ky = tap / p.ksize, kx = tap - ky * p.ksize;
        const int iy = oy0 * p.stride - p.pad + ky, ix = ox0 * p.stride - p.pad + kx;
        int wk = tap * p.k_per_tap;
        for (int s = 0; s < p.n_src; ++s) {
          const int kc = p.src_kchunk[s];
          const int kind = (kc == 64) ? 1 : 0;
          for (int ch = 0; ch < p.src_chunks[s]; ++ch, wk += kc) {
            mbar_wait(empty_bar(stage), phase ^ 1u);
            const uint32_t sb = base + stage * p.stage_bytes;
            const uint32_t a_bytes = kTileM * kc * 2, w_bytes = BLOCK_N * kc * 2;
            mbar_expect_tx(full_bar(stage), (p.terms > 1 ? 2u : 1u) * (a_bytes + w_bytes));
            tma_load_4d(sb, &p.a_map[s][0], full_bar(stage), ch * kc, ix, iy, b);
            tma_load_2d(sb + off_w_hi, &p.w_map[kind][0], full_bar(stage), wk, n0);
            if (p.terms > 1) {
              tma_load_4d(sb + off_a_lo, &p.a_map[s][1], full_bar(stage), ch * kc, ix, iy, b);
              tma_load_2d(sb + off_w_lo, &p.w_map[kind][1], full_bar(stage), wk, n0);
            }
            if (++stage == n_stages) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
  } else {
    // ============================== MMA warpgroup (warps 0-3) ==============================
    float acc[2][BLOCK_N / 2];         // rows [0, 64) and [64, 128) of the tile
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[h][i] = 0.f;
    {
      int stage = 0, prev_stage = -1;
      uint32_t phase = 0;
      for (int tap = tap_begin; tap < tap_end; ++tap) {
        for (int s = 0; s < p.n_src; ++s) {
          const int kc = p.src_kchunk[s];
          for (int ch = 0; ch < p.src_chunks[s]; ++ch) {
            mbar_wait(full_bar(stage), phase);
            const uint32_t sb = base + stage * p.stage_bytes;
            if (kc == 64) {
              if (p.terms == 3) tc_mma_chunk<BLOCK_N, 4, 3>(acc, sb, off_a_lo, off_w_hi, off_w_lo);
              else tc_mma_chunk<BLOCK_N, 4, 1>(acc, sb, off_a_lo, off_w_hi, off_w_lo);
            } else {
              if (p.terms == 3) tc_mma_chunk<BLOCK_N, 2, 3>(acc, sb, off_a_lo, off_w_hi, off_w_lo);
              else tc_mma_chunk<BLOCK_N, 2, 1>(acc, sb, off_a_lo, off_w_hi, off_w_lo);
            }
            wgmma_wait<1>();                 // the previous stage's MMAs are complete: release it
            wgmma_fence_regs(acc[0]);
            wgmma_fence_regs(acc[1]);
            if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));
            prev_stage = stage;
            if (++stage == n_stages) { stage = 0; phase ^= 1u; }
          }
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
    }
    // ============================== epilogue ==============================
    // every TMA of this CTA has landed and every MMA has completed: the ring becomes the fp32 staging tile [128][BLOCK_N + 4]
    constexpr int kPitch = BLOCK_N + 4;
    float* stg = reinterpret_cast<float*>(base_ptr);
    asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = h * 64 + warp * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int c = 8 * j + 2 * (lane & 3);
        *reinterpret_cast<float2*>(stg + r * kPitch + c) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
        *reinterpret_cast<float2*>(stg + (r + 8) * kPitch + c) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
      }
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const size_t plane_stride = (size_t)p.B * p.Hout * p.Wout * p.Cout;
    const bool split = p.ksplit > 1;
    const bool vec8 = (p.Cout & 7) == 0;
    // compact, rolled epilogue (8 accumulator columns per iteration): keeps the kernel's code footprint small -- these
    // kernels are short, an unrolled 32-column epilogue costs more in instruction fetch than it saves in issue slots.
    // One thread per (pixel, 8-channel chunk), chunks fastest: consecutive threads store consecutive 32-byte (fp32) /
    // 16-byte (fp16) pieces of one channel-last pixel row, i.e. a warp writes whole contiguous runs of the output instead
    // of one 16-byte piece per pixel (a stride of Cout elements between lanes).  The staging reads are conflict-free for
    // BLOCK_N = 32 (the pitch of BLOCK_N + 4 floats puts the next pixel's chunks four banks further), two-way for wider tiles.
    constexpr int kChunks = BLOCK_N / 8;
#pragma unroll 1
    for (int item = threadIdx.x; item < kTileM * kChunks; item += 128) {
      const int row = item / kChunks, c0 = 8 * (item - row * kChunks);
      const int ty = row / p.tile_w, tx = row - ty * p.tile_w;
      const int oy = oy0 + ty, ox = ox0 + tx;
      const int cbase = n0 + c0;
      if (oy >= p.Hout || ox >= p.Wout || cbase >= p.Cout) continue;
      const size_t pix = ((size_t)b * p.Hout + oy) * p.Wout + ox;
      float v[8];
      *reinterpret_cast<float4*>(v) = *reinterpret_cast<const float4*>(stg + row * kPitch + c0);
      *reinterpret_cast<float4*>(v + 4) = *reinterpret_cast<const float4*>(stg + row * kPitch + c0 + 4);
      float* wsp_row = split ? p.workspace + (size_t)blockIdx.z * plane_stride + pix * p.Cout : nullptr;
      if (vec8) {
        if (split) {
          // partial sums of this tap range; conv_tc_finish_kernel reduces the splits in fixed order
          *reinterpret_cast<float4*>(wsp_row + cbase) = make_float4(v[0], v[1], v[2], v[3]);
          *reinterpret_cast<float4*>(wsp_row + cbase + 4) = make_float4(v[4], v[5], v[6], v[7]);
          continue;
        }
        tc_emit8(p, v, b, oy, ox, cbase);
      } else {        // generic tail (Cout not a multiple of 8): scalar, rolled
        const float* res_row = nullptr;
        if (p.residual_mode == DVMVS_RES_SAME) {
          res_row = p.residual + pix * p.Cout;
        } else if (p.residual_mode == DVMVS_RES_NEAREST_UP) {
          const int ry = (int)(((long long)oy * p.Hr) / p.Hout), rx = (int)(((long long)ox * p.Wr) / p.Wout);
          res_row = p.residual + (((size_t)b * p.Hr + ry) * p.Wr + rx) * p.Cout;
        }
#pragma unroll 1
        for (int e = 0; e < 8; ++e) {
          const int c = cbase + e;
          if (c >= p.Cout) break;
          float x = v[e];
          if (split) { wsp_row[c] = x; continue; }
          if (p.bias) x += __ldg(p.bias + c);
          if (res_row) x += __ldg(res_row + c);
          x = tc_act(x, p.act);
          if (p.out_f32) p.out_f32[pix * p.Cout + c] = x;
          if (p.aux_out) p.aux_out[pix * p.Cout + c] = 1.f / (p.aux_mult * x + p.aux_base);
          if (p.out_planes) {
            const __half h = __float2half_rn(x);
            p.out_planes[pix * p.Cout + c] = h;
            if (!p.hi_only) p.out_planes[plane_stride + pix * p.Cout + c] = __float2half_rn(x - __half2float(h));
          }
        }
      }
    }
  }
}

// finishing pass for split-K launches: sum the per-split partials in split order, bias / residual / activation,
// fp32 and / or fp16-pair stores
__global__ void conv_tc_finish_kernel(TcParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t total = (size_t)p.B * p.Hout * p.Wout * p.Cout;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = (int)(idx % p.Cout);
  const size_t pix = idx / p.Cout;
  const int ox = (int)(pix % p.Wout);
  const int oy = (int)((pix / p.Wout) % p.Hout);
  const int b = (int)(pix / ((size_t)p.Wout * p.Hout));
  float x = 0.f;
  for (int sp = 0; sp < p.ksplit; ++sp) x += p.workspace[(size_t)sp * total + idx];
  if (p.bias) x += __ldg(p.bias + c);
  if (p.residual_mode == DVMVS_RES_SAME) {
    x += __ldg(p.residual + idx);
  } else if (p.residual_mode == DVMVS_RES_NEAREST_UP) {
    const int ry = (int)(((long long)oy * p.Hr) / p.Hout), rx = (int)(((long long)ox * p.Wr) / p.Wout);
    x += __ldg(p.residual + (((size_t)b * p.Hr + ry) * p.Wr + rx) * p.Cout + c);
  }
  x = tc_act(x, p.act);
  if (p.out_f32) p.out_f32[idx] = x;
  if (p.aux_out) p.aux_out[idx] = 1.f / (p.aux_mult * x + p.aux_base);
  if (p.out_planes) {
    const __half h = __float2half_rn(x);
    const __half l = __float2half_rn(x - __half2float(h));
    p.out_planes[idx] = h;
    if (!p.hi_only) p.out_planes[total + idx] = l;
    if (p.out_blk) {
      const size_t o = ((((size_t)b * (p.Cout >> 3) + (c >> 3)) * p.Hout + oy) * p.Wout + ox) * 8 + (c & 7);
      p.out_blk[o] = h;
      if (!p.hi_only) p.out_blk[total + o] = l;
    }
  }
}

// fp32 channel-last -> fp16 (hi, lo) planes with the channel count padded to Cs (zeros); optional x2 bilinear
// (align_corners) upsampling on the way (materialises F.interpolate for the TMA-fed consumer).
__global__ void split_planes_kernel(const float* __restrict__ x, __half* __restrict__ planes, int B, int H, int W, int C, int Cs,
                                    int upsample, int c_offset, int c_cover) {
  pdl_launch_dependents();
  pdl_wait();
  // writes channels [c_offset, c_offset + c_cover) of the Cs-channel plane tensor: x for the first C of them, zeros after
  const int Ho = upsample ? 2 * H : H, Wo = upsample ? 2 * W : W;
  const size_t total = (size_t)B * Ho * Wo * Cs;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)B * Ho * Wo * c_cover) return;
  const int c = (int)(idx % c_cover);
  const size_t pix = idx / c_cover;
  float v = 0.f;
  if (c < C) {
    if (!upsample) {
      v = x[pix * C + c];
    } else {
      const int ox = (int)(pix % Wo);
      const int oy = (int)((pix / Wo) % Ho);
      const int b = (int)(pix / ((size_t)Wo * Ho));
      const float sh = (Ho > 1) ? (float)(H - 1) / (float)(Ho - 1) : 0.f;
      const float sw = (Wo > 1) ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
      const float fy = sh * oy, fx = sw * ox;
      const int y0 = (int)fy, x0 = (int)fx;
      const int y1 = y0 + (y0 < H - 1), x1 = x0 + (x0 < W - 1);
      const float ly1 = fy - y0, lx1 = fx - x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
      const float* bp = x + (size_t)b * H * W * C + c;
      v = bilerp(ly0, ly1, lx0, lx1, bp[((size_t)y0 * W + x0) * C], bp[((size_t)y0 * W + x1) * C], bp[((size_t)y1 * W + x0) * C],
                 bp[((size_t)y1 * W + x1) * C]);
    }
  }
  const __half h = __float2half_rn(v);
  const size_t o = pix * Cs + c_offset + c;
  planes[o] = h;
  planes[total + o] = __float2half_rn(v - __half2float(h));
}

// same for channel counts / windows that are multiples of 8: one thread per (pixel, 8 channels), 16-byte loads and stores
__global__ void split_planes8_kernel(const float* __restrict__ x, __half* __restrict__ planes, int B, int H, int W, int C, int Cs,
                                     int upsample, int c_offset, int c_cover) {
  pdl_launch_dependents();
  pdl_wait();
  const int Ho = upsample ? 2 * H : H, Wo = upsample ? 2 * W : W;
  const size_t total = (size_t)B * Ho * Wo * Cs;
  const int nblk = c_cover >> 3;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)B * Ho * Wo * nblk) return;
  const int c = (int)(idx % nblk) * 8;
  const size_t pix = idx / nblk;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.f;
  if (c < C) {
    if (!upsample) {
      const float* src = x + pix * C + c;
      *reinterpret_cast<float4*>(v) = __ldg(reinterpret_cast<const float4*>(src));
      *reinterpret_cast<float4*>(v + 4) = __ldg(reinterpret_cast<const float4*>(src + 4));
    } else {
      const int ox = (int)(pix % Wo);
      const int oy = (int)((pix / Wo) % Ho);
      const int b = (int)(pix / ((size_t)Wo * Ho));
      const float sh = (Ho > 1) ? (float)(H - 1) / (float)(Ho - 1) : 0.f;
      const float sw = (Wo > 1) ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
      const float fy = sh * oy, fx = sw * ox;
      const int y0 = (int)fy, x0 = (int)fx;
      const int y1 = y0 + (y0 < H - 1), x1 = x0 + (x0 < W - 1);
      const float ly1 = fy - y0, lx1 = fx - x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
      const float* bp = x + (size_t)b * H * W * C + c;
      float t00[8], t01[8], t10[8], t11[8];
      const float* q;
      q = bp + ((size_t)y0 * W + x0) * C;
      *reinterpret_cast<float4*>(t00) = __ldg(reinterpret_cast<const float4*>(q)); *reinterpret_cast<float4*>(t00 + 4) = __ldg(reinterpret_cast<const float4*>(q + 4));
      q = bp + ((size_t)y0 * W + x1) * C;
      *reinterpret_cast<float4*>(t01) = __ldg(reinterpret_cast<const float4*>(q)); *reinterpret_cast<float4*>(t01 + 4) = __ldg(reinterpret_cast<const float4*>(q + 4));
      q = bp + ((size_t)y1 * W + x0) * C;
      *reinterpret_cast<float4*>(t10) = __ldg(reinterpret_cast<const float4*>(q)); *reinterpret_cast<float4*>(t10 + 4) = __ldg(reinterpret_cast<const float4*>(q + 4));
      q = bp + ((size_t)y1 * W + x1) * C;
      *reinterpret_cast<float4*>(t11) = __ldg(reinterpret_cast<const float4*>(q)); *reinterpret_cast<float4*>(t11 + 4) = __ldg(reinterpret_cast<const float4*>(q + 4));
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = bilerp(ly0, ly1, lx0, lx1, t00[e], t01[e], t10[e], t11[e]);
    }
  }
  __align__(16) __half hi[8];
  __align__(16) __half lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    hi[e] = __float2half_rn(v[e]);
    lo[e] = __float2half_rn(v[e] - __half2float(hi[e]));
  }
  const size_t o = pix * Cs + c_offset + c;
  *reinterpret_cast<uint4*>(planes + o) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(planes + total + o) = *reinterpret_cast<const uint4*>(lo);
}

// ----------------------------------------------------------------------------------------------- host side
EncodeTiledFn tensor_map_encoder() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)ptr;
  }
  return fn;
}

namespace {
struct MapKeyAll {
  unsigned long long w[16];
  bool operator==(const MapKeyAll& o) const { return memcmp(w, o.w, sizeof(w)) == 0; }
};
struct MapKeyAllHash {
  size_t operator()(const MapKeyAll& k) const {
    unsigned long long h = 0xcbf29ce484222325ull;
    for (int i = 0; i < 16; ++i) { h ^= k.w[i]; h *= 0x100000001b3ull; h ^= h >> 29; }
    return (size_t)h;
  }
};
std::mutex g_tm_mutex;
std::unordered_map<MapKeyAll, CUtensorMap, MapKeyAllHash> g_tm_cache;
}  // namespace

CUresult cached_tensor_map(CUtensorMap* out, CUtensorMapDataType dtype, int rank, const void* ptr, const cuuint64_t* dims,
                           const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapSwizzle swizzle,
                           CUtensorMapL2promotion promo) {
  MapKeyAll key;
  memset(&key, 0, sizeof(key));
  int dev = 0;
  cudaGetDevice(&dev);
  key.w[0] = (unsigned long long)(uintptr_t)ptr;
  key.w[1] = ((unsigned long long)dtype << 48) | ((unsigned long long)rank << 40) | ((unsigned long long)swizzle << 32) | ((unsigned long long)promo << 24) |
             (unsigned long long)(dev & 0xff);
  for (int i = 0; i < rank && i < 5; ++i) {
    key.w[2 + i] = dims[i];
    key.w[7 + i] = (i + 1 < rank) ? strides[i] : 0;
    key.w[12 + (i >> 1)] |= ((unsigned long long)box[i] | ((unsigned long long)estr[i] << 24)) << (32 * (i & 1));
  }
  std::lock_guard<std::mutex> lock(g_tm_mutex);
  auto it = g_tm_cache.find(key);
  if (it != g_tm_cache.end()) { *out = it->second; return CUDA_SUCCESS; }
  CUresult r = tensor_map_encoder()(out, dtype, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                    swizzle, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) {
    if (g_tm_cache.size() > 16384) g_tm_cache.clear();
    g_tm_cache.emplace(key, *out);
  }
  return r;
}

static int make_act_map(CUtensorMap* map, const void* ptr, int B, int H, int W, int Cs, int kchunk, int tile_w, int tile_h,
                        int stride) {
  cuuint64_t dims[4] = {(cuuint64_t)Cs, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)Cs * 2, (cuuint64_t)W * Cs * 2, (cuuint64_t)H * W * Cs * 2};
  cuuint32_t box[4] = {(cuuint32_t)kchunk, (cuuint32_t)((tile_w - 1) * stride + 1), (cuuint32_t)((tile_h - 1) * stride + 1), 1};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = cached_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, ptr, dims, strides, box, estr,
                                 kchunk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(activation B=%d H=%d W=%d C=%d chunk=%d) failed: %d", B, H, W, Cs, kchunk, (int)r);
    return DVMVS_EINVAL;
  }
  return DVMVS_OK;
}

static int make_w_map(CUtensorMap* map, const void* ptr, int rows, int ktot, int kchunk, int block_n) {
  cuuint64_t dims[2] = {(cuuint64_t)ktot, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ktot * 2};
  cuuint32_t box[2] = {(cuuint32_t)kchunk, (cuuint32_t)block_n};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = cached_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, ptr, dims, strides, box, estr,
                                 kchunk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(weights rows=%d K=%d chunk=%d) failed: %d", rows, ktot, kchunk, (int)r);
    return DVMVS_EINVAL;
  }
  return DVMVS_OK;
}

template <int BLOCK_N>
static int launch_tc(TcParams& p, dim3 grid, int kc_max, cudaStream_t s) {
  static PerDeviceOnce attr_set;
  if (attr_set.first()) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BLOCK_N>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemBytes);
    if (e != cudaSuccess) { set_error("conv_tc smem attribute: %s", cudaGetErrorString(e)); return DVMVS_ELAUNCH; }
  }
  // smem ring sized by the widest K chunk actually used; small stages => several CTAs co-reside per SM, which is what
  // hides the prologue / epilogue / TMA latency of these short tiles
  p.a_bytes = kTileM * kc_max * 2;
  p.w_bytes = BLOCK_N * kc_max * 2;
  p.stage_bytes = (p.terms > 1 ? 2 : 1) * (p.a_bytes + p.w_bytes);
  const int overhead = 1024 + kBarrierBytes;
  int stages = 0;
  const int budgets[3] = {74 * 1024, 112 * 1024, kMaxSmemBytes};
  for (int i = 0; i < 3 && stages < 3; ++i) stages = (budgets[i] - overhead) / p.stage_bytes;
  stages = max(2, min(kMaxStages, stages));
  // ... but never more stages than this CTA has K chunks to load: a 1x1 layer over 32 channels has ONE.  The shared memory a
  // CTA does not claim is what lets CTAs of OTHER streams' kernels (the software pipeline runs five) share the SM with it.
  int chunks_per_tap = 0;
  for (int i = 0; i < p.n_src; ++i) chunks_per_tap += p.src_chunks[i];
  const int n_taps = p.ksize * p.ksize;
  const int cta_chunks = ((n_taps + p.ksplit - 1) / p.ksplit) * chunks_per_tap;
  static const bool tight_env = []() { const char* e = getenv("DVMVS_TC_TIGHT_SMEM"); return !(e && e[0] == '0'); }();
  if (tight_env) stages = max(1, min(stages, cta_chunks));
  p.num_stages = stages;
  p.ring_bytes = max(stages * p.stage_bytes, tc_staging_bytes<BLOCK_N>());
  const int smem = p.ring_bytes + overhead;
  launch_k(conv_tc_kernel<BLOCK_N>, grid, dim3(kTcThreads), (size_t)smem, s, p);
  return check_launch("conv_tc_kernel");
}

}  // namespace dvmvs

using namespace dvmvs;

extern "C" int dvmvs_conv2d_tc(const dvmvs_conv_tc_desc* d, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(d != nullptr, "conv2d_tc: null descriptor");
  DVMVS_REQUIRE(tensor_map_encoder() != nullptr, "conv2d_tc: cuTensorMapEncodeTiled entry point not available");
  DVMVS_REQUIRE(d->n_src >= 1 && d->n_src <= 3, "conv2d_tc: n_src=%d", d->n_src);
  DVMVS_REQUIRE(d->ksize == 1 || d->ksize == 3 || d->ksize == 5, "conv2d_tc: ksize=%d", d->ksize);
  DVMVS_REQUIRE(d->stride == 1 || d->stride == 2, "conv2d_tc: stride=%d", d->stride);
  DVMVS_REQUIRE(d->terms == 1 || d->terms == 3, "conv2d_tc: terms=%d", d->terms);
  DVMVS_REQUIRE(d->B > 0 && d->Hin > 0 && d->Win > 0 && d->Cout > 0 && d->w_hi && (d->terms == 1 || d->w_lo),
                "conv2d_tc: bad shape / null weights");
  DVMVS_REQUIRE(d->out_f32 || d->out_planes || d->defer_finish, "conv2d_tc: no output");
  DVMVS_REQUIRE(d->block_n == 32 || d->block_n == 64 || d->block_n == 128, "conv2d_tc: block_n=%d", d->block_n);
  DVMVS_REQUIRE(d->w_rows % d->block_n == 0 && d->w_rows >= d->Cout, "conv2d_tc: weight rows %d not a multiple of block_n", d->w_rows);
  DVMVS_REQUIRE(d->out_planes == nullptr || d->Cout % 8 == 0, "conv2d_tc: fp16-pair output needs Cout %% 8 == 0");
  TcParams p;
  memset(&p, 0, sizeof(p));
  const int pad = (d->ksize - 1) / 2;
  p.ksize = d->ksize; p.pad = pad; p.stride = d->stride;
  p.Hout = (d->Hin + 2 * pad - d->ksize) / d->stride + 1;
  p.Wout = (d->Win + 2 * pad - d->ksize) / d->stride + 1;
  p.B = d->B; p.Cout = d->Cout;
  // output-pixel tile: 16 wide x 8 high, or 8 x 16 for narrow maps
  p.tile_w = (p.Wout <= 8 && p.Hout > 8) ? 8 : 16;
  p.tile_h = kTileM / p.tile_w;
  p.tiles_x = (p.Wout + p.tile_w - 1) / p.tile_w;
  p.tiles_y = (p.Hout + p.tile_h - 1) / p.tile_h;
  p.n_src = d->n_src; p.terms = d->terms;
  int k_per_tap = 0, kc_max = 32;
  for (int s = 0; s < d->n_src; ++s) {
    const int Cs = d->src_channels[s];
    DVMVS_REQUIRE(d->src_planes[s] && Cs > 0 && Cs % 8 == 0, "conv2d_tc: source %d needs a channel count that is a multiple of 8", s);
    DVMVS_REQUIRE((uintptr_t)d->src_planes[s] % 16 == 0, "conv2d_tc: source %d not 16-byte aligned", s);
    p.src_kchunk[s] = (Cs % 64 == 0) ? 64 : 32;
    p.src_chunks[s] = (Cs + p.src_kchunk[s] - 1) / p.src_kchunk[s];
    kc_max = max(kc_max, p.src_kchunk[s]);
    k_per_tap += p.src_chunks[s] * p.src_kchunk[s];
    const size_t plane = (size_t)d->B * d->Hin * d->Win * Cs;
    int rc = make_act_map(&p.a_map[s][0], d->src_planes[s], d->B, d->Hin, d->Win, Cs, p.src_kchunk[s], p.tile_w, p.tile_h, d->stride);
    if (rc != DVMVS_OK) return rc;
    if (d->terms > 1) {
      rc = make_act_map(&p.a_map[s][1], (const __half*)d->src_planes[s] + plane, d->B, d->Hin, d->Win, Cs, p.src_kchunk[s], p.tile_w,
                        p.tile_h, d->stride);
      if (rc != DVMVS_OK) return rc;
    }
  }
  p.k_per_tap = k_per_tap;
  DVMVS_REQUIRE(d->ktot == k_per_tap * d->ksize * d->ksize, "conv2d_tc: packed weight K=%d, expected %d", d->ktot,
                k_per_tap * d->ksize * d->ksize);
  for (int kind = 0; kind < 2; ++kind) {
    const int kc = kind ? 64 : 32;
    int rc = make_w_map(&p.w_map[kind][0], d->w_hi, d->w_rows, d->ktot, kc, d->block_n);
    if (rc != DVMVS_OK) return rc;
    if (d->terms > 1) {
      rc = make_w_map(&p.w_map[kind][1], d->w_lo, d->w_rows, d->ktot, kc, d->block_n);
      if (rc != DVMVS_OK) return rc;
    }
  }
  p.bias = d->bias; p.residual = d->residual; p.residual_mode = d->residual_mode; p.Hr = d->Hr; p.Wr = d->Wr;
  DVMVS_REQUIRE(d->residual_mode == DVMVS_RES_NONE || d->residual, "conv2d_tc: residual pointer missing");
  p.out_f32 = d->out_f32; p.out_planes = (__half*)d->out_planes; p.aux_out = d->aux_out;
  p.out_blk = (__half*)d->out_blk;
  DVMVS_REQUIRE(!d->out_blk || (d->out_planes && d->Cout % 8 == 0), "conv2d_tc: out_blk needs out_planes and Cout %% 8 == 0");
  // Cout % 8 == 0: the epilogue (tc_emit8) loads bias / residual and stores every output but aux_out as 16-byte vectors, and the
  // split-K partial sums go to the workspace as float4
  DVMVS_REQUIRE(d->Cout % 8 != 0 || ((uintptr_t)d->bias % 16 == 0 && (uintptr_t)d->residual % 16 == 0 && (uintptr_t)d->out_f32 % 16 == 0 &&
                                     (uintptr_t)d->out_planes % 16 == 0 && (uintptr_t)d->out_blk % 16 == 0 && (uintptr_t)d->workspace % 16 == 0),
                "conv2d_tc: bias, residual, outputs and workspace must be 16-byte aligned");
  p.aux_mult = d->aux_mult; p.aux_base = d->aux_base; p.act = d->act;
  p.hi_only = d->out_hi_only ? 1 : 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int n_tiles = (d->Cout + d->block_n - 1) / d->block_n;
  const int ctas = p.tiles_x * p.tiles_y * d->B * n_tiles;
  p.ksplit = 1;
  const int n_taps = d->ksize * d->ksize;
  // the first 16 KiB of the workspace are reserved (historical: arrival counters); the partial sums follow
  const long long counter_bytes = 16384;
  p.workspace = d->workspace ? reinterpret_cast<float*>(reinterpret_cast<char*>(d->workspace) + counter_bytes) : nullptr;
  const size_t out_elems = (size_t)d->B * p.Hout * p.Wout * d->Cout;
  const int n_sms = device_sm_count();
  if (d->allow_split && d->workspace && d->workspace_bytes > counter_bytes && ctas < n_sms / 2 && n_taps > 1) {
    long long fit = (d->workspace_bytes - counter_bytes) / (long long)(out_elems * sizeof(float));
    p.ksplit = (int)max(1LL, min((long long)min(n_taps, (n_sms + ctas - 1) / ctas), fit));
    const int per = (n_taps + p.ksplit - 1) / p.ksplit;
    p.ksplit = (n_taps + per - 1) / per;              // no empty splits
  }
  dim3 grid(p.tiles_x * p.tiles_y * d->B, n_tiles, p.ksplit);
  // Measured and removed on the previous architecture: reducing the splits inside a thread-block cluster through distributed
  // shared memory (clusters of 5 / 9 one-CTA-per-SM blocks schedule worse than the short finishing launches they save) and a
  // fused finish by the last-arriving CTA (one CTA walks ksplit x BLOCK_N/8 dependent L2 round trips where the finishing
  // kernel spreads them over the GPU under the next prologue).
  int rc;
  if (d->block_n == 32) rc = launch_tc<32>(p, grid, kc_max, s);
  else if (d->block_n == 64) rc = launch_tc<64>(p, grid, kc_max, s);
  else rc = launch_tc<128>(p, grid, kc_max, s);
  if (rc != DVMVS_OK) return rc;
  if (d->defer_finish) {
    // the caller's own epilogue kernel sums the split-K partial sums (dvmvs_lstm_gates_parts): only legal when this launch split
    DVMVS_REQUIRE(p.ksplit > 1, "conv2d_tc: defer_finish without a split-K launch (ask dvmvs_conv2d_tc_ksplit first)");
    return DVMVS_OK;
  }
  if (p.ksplit > 1) {
    launch_k(conv_tc_finish_kernel, dim3((unsigned)((out_elems + 255) / 256)), dim3(256), 0, s, p);
    return check_launch("conv_tc_finish_kernel");
  }
  return DVMVS_OK;
}

// Split count dvmvs_conv2d_tc will use for this descriptor (1 = no split): lets a caller that fuses the finishing pass into its own
// epilogue (defer_finish) size its reads.  Mirrors the decision above.
extern "C" int dvmvs_conv2d_tc_ksplit(const dvmvs_conv_tc_desc* d) {
  if (!d || !(d->ksize == 1 || d->ksize == 3 || d->ksize == 5) || d->B <= 0) return 1;
  const int pad = (d->ksize - 1) / 2;
  const int Hout = (d->Hin + 2 * pad - d->ksize) / d->stride + 1, Wout = (d->Win + 2 * pad - d->ksize) / d->stride + 1;
  const int tile_w = (Wout <= 8 && Hout > 8) ? 8 : 16, tile_h = kTileM / tile_w;
  const int tiles = ((Wout + tile_w - 1) / tile_w) * ((Hout + tile_h - 1) / tile_h);
  const int n_tiles = (d->Cout + d->block_n - 1) / d->block_n;
  const int ctas = tiles * d->B * n_tiles;
  const int n_taps = d->ksize * d->ksize;
  const long long counter_bytes = 16384;
  const size_t out_elems = (size_t)d->B * Hout * Wout * d->Cout;
  int ksplit = 1;
  const int n_sms = device_sm_count();
  if (d->allow_split && d->workspace && d->workspace_bytes > counter_bytes && ctas < n_sms / 2 && n_taps > 1) {
    long long fit = (d->workspace_bytes - counter_bytes) / (long long)(out_elems * sizeof(float));
    ksplit = (int)max(1LL, min((long long)min(n_taps, (n_sms + ctas - 1) / ctas), fit));
    const int per = (n_taps + ksplit - 1) / ksplit;
    ksplit = (n_taps + per - 1) / per;
  }
  return ksplit;
}

extern "C" int dvmvs_split_planes(const float* x, void* planes, int B, int H, int W, int C, int Cs, int upsample2x, int c_offset,
                                  int c_cover, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(x && planes && B > 0 && H > 0 && W > 0 && C > 0 && Cs % 8 == 0, "split_planes: bad argument");
  DVMVS_REQUIRE(c_offset >= 0 && c_cover >= C && c_offset + c_cover <= Cs, "split_planes: channel window [%d,+%d) outside %d", c_offset,
                c_cover, Cs);
  if (C % 8 == 0 && c_offset % 8 == 0 && c_cover % 8 == 0 && (uintptr_t)x % 16 == 0 && (uintptr_t)planes % 16 == 0) {
    const size_t n8 = (size_t)B * H * W * (c_cover / 8) * (upsample2x ? 4 : 1);
    launch_k(split_planes8_kernel, dim3((unsigned)((n8 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, x, (__half*)planes, B, H, W, C, Cs,
             upsample2x, c_offset, c_cover);
    return check_launch("split_planes8_kernel");
  }
  const size_t total = (size_t)B * H * W * c_cover * (upsample2x ? 4 : 1);
  launch_k(split_planes_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, x, (__half*)planes, B, H, W, C, Cs,
           upsample2x, c_offset, c_cover);
  return check_launch("split_planes_kernel");
}
