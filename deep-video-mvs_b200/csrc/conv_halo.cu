// Stride-1 k x k convolution on the Hopper tensor cores (wgmma) WITHOUT im2col amplification: "halo" implicit GEMM.  sm_90a.
//
// conv_tc_kernel (conv_tc.cu) re-loads the activation tile once per filter tap (25x for 5x5), one TMA row per pixel;
// on the big 32-channel layers (refine, decoder block 4, aggregator0, FPN outputs) it is bound by the TMA request rate.
// Here the activations are stored in a channel-BLOCKED fp16 layout  [plane][B][C/8][H][W][8]  ("NC8HW8"), so that
//   * one TMA box {(8+k-1) pixels x 8 ch = one contiguous row, 16+k-1 rows, KC/8 channel blocks} brings the whole halo
//     of an 8-wide x 16-high output tile into shared memory ONCE per KC-channel group, in rows of (8+k-1)*16 bytes;
//   * in shared memory [channel block][halo y][halo x][8 ch] IS the canonical no-swizzle K-major wgmma layout: a core
//     matrix = 8 x-consecutive pixels x 16 bytes, the next 8 GEMM rows (= next tile row) lie one halo row further
//     (SBO), the next 8 channels one channel block further (LBO);
//   * a filter tap (ky,kx) is just a different START ADDRESS of the same halo tile: (ky*halo_w + kx)*16 bytes.
// So per KC channels the tile issues k*k*(KC/16) MMAs per term from one resident halo, and only the (tiny) per-tap
// weight blocks stream through a ring (one bulk copy per filter row: all kx taps are contiguous in the packed weights).
// Weights are pre-packed in exactly their shared-memory image [n-tile][k-group][ky][kx][KC/8][BLOCK_N][8].
// The epilogue writes fp32 channel-last and/or the blocked fp16 pair planes (16 bytes per pixel and channel block,
// coalesced over the 8 pixels of a tile row).
//
// Warp roles as in conv_tc_kernel: warps 0-3 = MMA warpgroup (two m64 halves of the 128-pixel tile, register accumulators)
// and epilogue, warp 4 = TMA / bulk-copy producer.  fp16 (hi, lo) pairs, 3 terms (hi*hi + lo*hi + hi*lo) or 1 term.
#include <string.h>

#include "tc_ptx.cuh"

namespace dvmvs {

constexpr int kHaloThreads = 160;
constexpr int kHaloTileW = 8, kHaloTileH = 16;
constexpr int kHaloWStages = 4;

struct HaloParams {
  CUtensorMap a_map[3][2];     // [source][hi/lo]: 4-D {W*8, H, C8, B} over the blocked planes
  const __half* w_hi;          // packed weights, see header comment
  const __half* w_lo;
  int src_groups[3];           // KC-channel groups per source
  int n_src, terms, ksize, pad, kc;           // kc: channels per group (16 or 32)
  int B, Hout, Wout, Cout, c8_out, tiles_x, tiles_y, n_groups;
  const float* bias;
  const float* residual;       // fp32 channel-last, same size (DVMVS_RES_SAME) or null
  float* out_f32;              // [B][H][W][Cout] or null
  __half* out_blk;             // [2][B][Cout/8][H][W][8] or null
  __half* out_nhwc;            // [2][B][H][W][Cout] or null
  int hi_only;                 // fp16 outputs: hi plane only
  int act;
  uint32_t a_bytes, w_bytes;   // per plane: halo tile bytes of one group, weight bytes of one (group, ky) stage
  uint32_t ring_bytes;         // A buffers + weight ring, or the epilogue's accumulator staging tile that reuses them
  unsigned long long* dbg;     // optional timeline dump: [cta][8] globaltimer ns at phase boundaries (profiling aid)
};

__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#define HALO_MARK(i) do { if (p.dbg) p.dbg[(size_t)(blockIdx.y * gridDim.x + blockIdx.x) * 8 + (i)] = gtimer(); } while (0)

// the MMAs of one filter row ky of one channel group: KSIZE taps x KC/16 K steps x TERMS products x two m64 halves, committed
// as one group.  Descriptor addresses in bytes: a0 / a1 = hi / lo halo tile at filter row ky, w0 / w1 = hi / lo weights of the row.
template <int BLOCK_N, int KSIZE, int KC, int TERMS>
__device__ __forceinline__ void halo_mma_row(float (&acc)[2][BLOCK_N / 2], uint32_t a0, uint32_t a1, uint32_t w0, uint32_t w1, uint32_t halo_w,
                                             uint32_t a_chunk_bytes) {
  constexpr uint32_t w_chunk_bytes = BLOCK_N * 16;               // one 8-channel block of a weight tap: [BLOCK_N][8]
  constexpr uint32_t w_tap_bytes = (KC / 8) * w_chunk_bytes;     // one tap: [KC/8][BLOCK_N][8]
  const uint32_t a_half = 8u * halo_w * 16u;                     // GEMM rows [64, 128) = tile rows 8..15
  wgmma_fence_regs(acc[0]);
  wgmma_fence_regs(acc[1]);
  wgmma_fence();
#pragma unroll
  for (int kx = 0; kx < KSIZE; ++kx) {
#pragma unroll
    for (int term = 0; term < TERMS; ++term) {
#pragma unroll
      for (int k2 = 0; k2 < KC / 16; ++k2) {
        // SBO = next tile row (next 8 GEMM rows) / next 8 output channels; LBO = next 8 input channels
        const uint32_t a = ((term == 1) ? a1 : a0) + kx * 16u + 2u * k2 * a_chunk_bytes;
        const uint32_t w = ((term == 2) ? w1 : w0) + kx * w_tap_bytes + 2u * k2 * w_chunk_bytes;
        const uint64_t bd = gmma_desc(w, w_chunk_bytes, 128u, kGmmaNoSwizzle);
        wgmma_f16<BLOCK_N>(acc[0], gmma_desc(a, a_chunk_bytes, halo_w * 16u, kGmmaNoSwizzle), bd);
        wgmma_f16<BLOCK_N>(acc[1], gmma_desc(a + a_half, a_chunk_bytes, halo_w * 16u, kGmmaNoSwizzle), bd);
      }
    }
  }
  wgmma_commit();
}

template <int BLOCK_N, int KSIZE, int KC, int TERMS>
__global__ void __launch_bounds__(kHaloThreads) conv_halo_kernel(const __grid_constant__ HaloParams p) {
  pdl_launch_dependents();
  if (threadIdx.x == 0) HALO_MARK(0);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 127u) & ~127u;
  uint8_t* base_ptr = smem_raw + (base - raw_addr);
  const int planes = p.terms > 1 ? 2 : 1;
  // layout: A[2 buffers][planes][a_bytes] | W[kHaloWStages][planes][w_bytes] | barriers
  const uint32_t a_buf_bytes = planes * p.a_bytes, w_stage_bytes = planes * p.w_bytes;
  const uint32_t a_base = base, w_base = base + 2 * a_buf_bytes;
  const uint32_t bars = base + p.ring_bytes;
  auto a_full = [&](int i) { return bars + 8u * i; };
  auto a_empty = [&](int i) { return bars + 8u * (2 + i); };
  auto w_full = [&](int i) { return bars + 8u * (4 + i); };
  auto w_empty = [&](int i) { return bars + 8u * (4 + kHaloWStages + i); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int b = blockIdx.x / tiles_per_img;
  const int t_in = blockIdx.x - b * tiles_per_img;
  const int oy0 = (t_in / p.tiles_x) * kHaloTileH, ox0 = (t_in % p.tiles_x) * kHaloTileW;
  const int nt = blockIdx.y, n0 = nt * BLOCK_N;
  const int halo_w = kHaloTileW + p.ksize - 1, halo_h = kHaloTileH + p.ksize - 1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.n_src; ++s) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&p.a_map[s][0]) : "memory");
      if (p.terms > 1) asm volatile("prefetch.tensormap [%0];" ::"l"(&p.a_map[s][1]) : "memory");
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(a_full(i), 1);
      mbar_init(a_empty(i), 4);          // one arrival per MMA warp
    }
    for (int i = 0; i < kHaloWStages; ++i) {
      mbar_init(w_full(i), 1);
      mbar_init(w_empty(i), 4);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) HALO_MARK(1);
  pdl_wait();
  if (threadIdx.x == 0) HALO_MARK(2);

  if (warp == 4) {
    // ============================== producer ==============================
    if (lane == 0) {
      int g = 0, wst = 0;
      uint32_t wphase = 0;
      for (int s = 0; s < p.n_src; ++s) {
        for (int cg = 0; cg < p.src_groups[s]; ++cg, ++g) {
          const int ab = g & 1;
          mbar_wait(a_empty(ab), ((g >> 1) & 1) ^ 1u);
          mbar_expect_tx(a_full(ab), planes * p.a_bytes);
          const uint32_t adst = a_base + ab * a_buf_bytes;
          // box {halo_w*8 elements, halo_h rows, kc/8 channel blocks, 1}; out-of-image rows / columns are zero-filled
          tma_load_4d(adst, &p.a_map[s][0], a_full(ab), (ox0 - p.pad) * 8, oy0 - p.pad, cg * (p.kc / 8), b);
          if (p.terms > 1) tma_load_4d(adst + p.a_bytes, &p.a_map[s][1], a_full(ab), (ox0 - p.pad) * 8, oy0 - p.pad, cg * (p.kc / 8), b);
          for (int ky = 0; ky < p.ksize; ++ky) {
            mbar_wait(w_empty(wst), wphase ^ 1u);
            mbar_expect_tx(w_full(wst), planes * p.w_bytes);
            const size_t woff = ((((size_t)nt * p.n_groups + g) * p.ksize + ky) * (size_t)p.w_bytes) / sizeof(__half);
            const uint32_t wdst = w_base + wst * w_stage_bytes;
            bulk_load(wdst, p.w_hi + woff, p.w_bytes, w_full(wst));
            if (p.terms > 1) bulk_load(wdst + p.w_bytes, p.w_lo + woff, p.w_bytes, w_full(wst));
            if (++wst == kHaloWStages) { wst = 0; wphase ^= 1u; }
          }
        }
      }
    }
  } else {
    // ============================== MMA warpgroup (warps 0-3) ==============================
    float acc[2][BLOCK_N / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[h][i] = 0.f;
    {
      const uint32_t a_chunk_bytes = (uint32_t)halo_h * halo_w * 16u;       // one 8-channel block of the halo tile
      int g = 0, wst = 0, prev_w = -1, prev_a = -1;
      uint32_t wphase = 0;
      for (int s = 0; s < p.n_src; ++s) {
        for (int cg = 0; cg < p.src_groups[s]; ++cg, ++g) {
          const int ab = g & 1;
          mbar_wait(a_full(ab), (g >> 1) & 1);
          if (g == 0 && threadIdx.x == 0) HALO_MARK(3);
          const uint32_t a_plane0 = a_base + ab * a_buf_bytes, a_plane1 = a_plane0 + p.a_bytes;
#pragma unroll 1
          for (int ky = 0; ky < KSIZE; ++ky) {
            mbar_wait(w_full(wst), wphase);
            const uint32_t w_plane0 = w_base + wst * w_stage_bytes, w_plane1 = w_plane0 + p.w_bytes;
            const uint32_t a_row = (uint32_t)ky * halo_w * 16u;
            halo_mma_row<BLOCK_N, KSIZE, KC, TERMS>(acc, a_plane0 + a_row, a_plane1 + a_row, w_plane0, w_plane1, (uint32_t)halo_w, a_chunk_bytes);
            wgmma_wait<1>();               // everything before this row's MMAs has completed: release those stages
            wgmma_fence_regs(acc[0]);
            wgmma_fence_regs(acc[1]);
            if (lane == 0) {
              if (prev_w >= 0) mbar_arrive(w_empty(prev_w));
              if (prev_a >= 0) mbar_arrive(a_empty(prev_a));
            }
            prev_a = -1;
            prev_w = wst;
            if (++wst == kHaloWStages) { wst = 0; wphase ^= 1u; }
          }
          prev_a = ab;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
      if (threadIdx.x == 0) HALO_MARK(4);
    }
    // ============================== epilogue ==============================
    // all loads have landed and all MMAs completed: the A buffers + weight ring become the fp32 staging tile [128][BLOCK_N + 4]
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
    if (threadIdx.x == 0) HALO_MARK(5);
    const size_t hw = (size_t)p.Hout * p.Wout;
    const size_t plane_elems = (size_t)p.B * p.c8_out * hw * 8;
    const size_t nhwc_plane = (size_t)p.B * hw * p.Cout;
    // One thread per (pixel, 8-channel chunk).  A channel-last output (fp32 or fp16 planes) is written chunks fastest:
    // consecutive threads store consecutive pieces of one pixel row of the tile, so a warp's stores are contiguous runs.
    // The blocked output alone is written pixels fastest: 8 consecutive pixels of one channel block are 128 contiguous bytes.
    constexpr int kChunks = BLOCK_N / 8;
    const bool chunks_fastest = p.out_f32 || p.out_nhwc;
#pragma unroll 1
    for (int item = threadIdx.x; item < 128 * kChunks; item += 128) {
      const int row = chunks_fastest ? item / kChunks : item % 128;
      const int c0 = 8 * (chunks_fastest ? item % kChunks : item / 128);
      const int oy = oy0 + (row >> 3), ox = ox0 + (row & 7);
      const int cbase = n0 + c0;
      if (oy >= p.Hout || ox >= p.Wout || cbase >= p.Cout) continue;
      const size_t pix = ((size_t)b * p.Hout + oy) * p.Wout + ox;
      float v[8];
      *reinterpret_cast<float4*>(v) = *reinterpret_cast<const float4*>(stg + row * kPitch + c0);
      *reinterpret_cast<float4*>(v + 4) = *reinterpret_cast<const float4*>(stg + row * kPitch + c0 + 4);
      if (p.bias) {
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + cbase)), b1 = __ldg(reinterpret_cast<const float4*>(p.bias + cbase + 4));
        v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w; v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
      }
      if (p.residual) {
        const float* rr = p.residual + pix * p.Cout + cbase;
        const float4 r0 = __ldg(reinterpret_cast<const float4*>(rr)), r1 = __ldg(reinterpret_cast<const float4*>(rr + 4));
        v[0] += r0.x; v[1] += r0.y; v[2] += r0.z; v[3] += r0.w; v[4] += r1.x; v[5] += r1.y; v[6] += r1.z; v[7] += r1.w;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = tc_act(v[e], p.act);
      if (p.out_f32) {
        float* o = p.out_f32 + pix * p.Cout + cbase;
        *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
      }
      if (p.out_blk || p.out_nhwc) {
        __align__(16) __half hi[8];
        __align__(16) __half lo[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          hi[e] = __float2half_rn(v[e]);
          lo[e] = __float2half_rn(v[e] - __half2float(hi[e]));
        }
        if (p.out_blk) {
          __half* o = p.out_blk + (((size_t)b * p.c8_out + (cbase >> 3)) * hw + (size_t)oy * p.Wout + ox) * 8;
          *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(hi);
          if (!p.hi_only) *reinterpret_cast<uint4*>(o + plane_elems) = *reinterpret_cast<const uint4*>(lo);
        }
        if (p.out_nhwc) {
          __half* o = p.out_nhwc + pix * p.Cout + cbase;
          *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(hi);
          if (!p.hi_only) *reinterpret_cast<uint4*>(o + nhwc_plane) = *reinterpret_cast<const uint4*>(lo);
        }
      }
    }
    if (threadIdx.x == 0) HALO_MARK(6);
    if (threadIdx.x == 0) HALO_MARK(7);
  }
}

// fp32 channel-last -> channel blocks [c_offset/8, (c_offset + c_cover)/8) of the blocked fp16 pair planes
// [2][B][C8][H'][W'][8] (the C values of x, then zeros); optional x2 bilinear (align_corners) upsampling on the way.
// hi_only: the lo plane is left unwritten (1-term operands never read it), which halves the bytes stored.
// One thread per (pixel, 8-channel block): 32-byte reads, one 16-byte store per plane, consecutive threads = consecutive
// pixels of one channel block (coalesced 512-byte stores per warp).  c_offset must be a multiple of 8.  x_aligned: x is 16-byte
// aligned, so with C % 4 == 0 every 8-channel block starts on a 16-byte boundary (the host checks; views need not be).
__global__ void split_blocked_kernel(const float* __restrict__ x, __half* __restrict__ planes, int B, int H, int W, int C, int C8,
                                     int upsample, int hi_only, int c_offset, int c_cover, int x_aligned) {
  pdl_launch_dependents();
  pdl_wait();
  const int Ho = upsample ? 2 * H : H, Wo = upsample ? 2 * W : W;
  const size_t hw = (size_t)Ho * Wo;
  const size_t total = (size_t)B * C8 * hw * 8;
  const int nblk = (c_cover + 7) >> 3;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)B * nblk * hw) return;
  const size_t p_in = idx % hw;
  const int cb = (int)((idx / hw) % nblk);
  const int b = (int)(idx / (hw * nblk));
  const int ox = (int)(p_in % Wo), oy = (int)(p_in / Wo);
  const int c0 = cb * 8;                       // first source channel of this block
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.f;
  const bool vec = x_aligned && ((C & 3) == 0) && (c0 + 8 <= C);
  if (!upsample) {
    const float* src = x + ((size_t)b * hw + p_in) * C + c0;
    if (vec) {
      const float4 a0 = __ldg(reinterpret_cast<const float4*>(src)), a1 = __ldg(reinterpret_cast<const float4*>(src + 4));
      v[0] = a0.x; v[1] = a0.y; v[2] = a0.z; v[3] = a0.w; v[4] = a1.x; v[5] = a1.y; v[6] = a1.z; v[7] = a1.w;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (c0 + e < C) v[e] = __ldg(src + e);
    }
  } else {
    const float sh = (Ho > 1) ? (float)(H - 1) / (float)(Ho - 1) : 0.f;
    const float sw = (Wo > 1) ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
    const float fy = sh * oy, fx = sw * ox;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < H - 1), x1 = x0 + (x0 < W - 1);
    const float ly1 = fy - y0, lx1 = fx - x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
    const float* bp = x + (size_t)b * H * W * C + c0;
    const float* p00 = bp + ((size_t)y0 * W + x0) * C;
    const float* p01 = bp + ((size_t)y0 * W + x1) * C;
    const float* p10 = bp + ((size_t)y1 * W + x0) * C;
    const float* p11 = bp + ((size_t)y1 * W + x1) * C;
    if (vec) {       // 8 x 16-byte loads instead of 32 scalar ones (this kernel is LSU-issue bound, not bandwidth bound)
      float t00[8], t01[8], t10[8], t11[8];
      *reinterpret_cast<float4*>(t00) = __ldg(reinterpret_cast<const float4*>(p00));
      *reinterpret_cast<float4*>(t00 + 4) = __ldg(reinterpret_cast<const float4*>(p00 + 4));
      *reinterpret_cast<float4*>(t01) = __ldg(reinterpret_cast<const float4*>(p01));
      *reinterpret_cast<float4*>(t01 + 4) = __ldg(reinterpret_cast<const float4*>(p01 + 4));
      *reinterpret_cast<float4*>(t10) = __ldg(reinterpret_cast<const float4*>(p10));
      *reinterpret_cast<float4*>(t10 + 4) = __ldg(reinterpret_cast<const float4*>(p10 + 4));
      *reinterpret_cast<float4*>(t11) = __ldg(reinterpret_cast<const float4*>(p11));
      *reinterpret_cast<float4*>(t11 + 4) = __ldg(reinterpret_cast<const float4*>(p11 + 4));
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = bilerp(ly0, ly1, lx0, lx1, t00[e], t01[e], t10[e], t11[e]);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (c0 + e < C) v[e] = bilerp(ly0, ly1, lx0, lx1, __ldg(p00 + e), __ldg(p01 + e), __ldg(p10 + e), __ldg(p11 + e));
    }
  }
  __align__(16) __half hi[8];
  __align__(16) __half lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    hi[e] = __float2half_rn(v[e]);
    lo[e] = __float2half_rn(v[e] - __half2float(hi[e]));
  }
  const size_t o = (((size_t)b * C8 + (c_offset >> 3) + cb) * hw + p_in) * 8;
  *reinterpret_cast<uint4*>(planes + o) = *reinterpret_cast<const uint4*>(hi);
  if (!hi_only) *reinterpret_cast<uint4*>(planes + total + o) = *reinterpret_cast<const uint4*>(lo);
}

static int make_halo_map(CUtensorMap* map, const void* ptr, int B, int H, int W, int C8, int halo_w, int halo_h, int kc8) {
  cuuint64_t dims[4] = {(cuuint64_t)W * 8, (cuuint64_t)H, (cuuint64_t)C8, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)W * 16, (cuuint64_t)H * W * 16, (cuuint64_t)C8 * H * W * 16};
  cuuint32_t box[4] = {(cuuint32_t)halo_w * 8, (cuuint32_t)halo_h, (cuuint32_t)kc8, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = cached_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, ptr, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(blocked activation B=%d H=%d W=%d C8=%d halo %dx%d) failed: %d", B, H, W, C8, halo_w, halo_h, (int)r);
    return DVMVS_EINVAL;
  }
  return DVMVS_OK;
}

template <int BLOCK_N, int KSIZE, int KC, int TERMS>
static int launch_halo(const HaloParams& p, dim3 grid, size_t smem, cudaStream_t s) {
  static PerDeviceOnce attr_set;
  if (attr_set.first()) {
    cudaError_t e = cudaFuncSetAttribute(conv_halo_kernel<BLOCK_N, KSIZE, KC, TERMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) { set_error("conv_halo smem attribute: %s", cudaGetErrorString(e)); return DVMVS_ELAUNCH; }
  }
  launch_k(conv_halo_kernel<BLOCK_N, KSIZE, KC, TERMS>, grid, dim3(kHaloThreads), smem, s, p);
  return check_launch("conv_halo_kernel");
}

template <int BLOCK_N, int KSIZE>
static int launch_halo_kt(const HaloParams& p, dim3 grid, size_t smem, cudaStream_t s) {
  if (p.kc == 16) return p.terms == 3 ? launch_halo<BLOCK_N, KSIZE, 16, 3>(p, grid, smem, s) : launch_halo<BLOCK_N, KSIZE, 16, 1>(p, grid, smem, s);
  return p.terms == 3 ? launch_halo<BLOCK_N, KSIZE, 32, 3>(p, grid, smem, s) : launch_halo<BLOCK_N, KSIZE, 32, 1>(p, grid, smem, s);
}

static void* g_halo_dbg = nullptr;

}  // namespace dvmvs

using namespace dvmvs;

// profiling aid: device buffer of (#CTAs x 8) uint64 receiving %globaltimer at the phase boundaries of conv_halo_kernel
// (0 start, 1 setup done, 2 dependencies resolved, 3 first halo landed, 4 last MMA completed, 5 accumulators staged,
// 6 epilogue stores issued, 7 exit); NULL switches it off.
extern "C" int dvmvs_debug_set_halo_timeline(void* device_buffer) {
  g_halo_dbg = device_buffer;
  return DVMVS_OK;
}

extern "C" int dvmvs_conv2d_halo(const dvmvs_conv_halo_desc* d, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(d != nullptr, "conv2d_halo: null descriptor");
  DVMVS_REQUIRE(tensor_map_encoder() != nullptr, "conv2d_halo: cuTensorMapEncodeTiled entry point not available");
  DVMVS_REQUIRE(d->n_src >= 1 && d->n_src <= 3, "conv2d_halo: n_src=%d", d->n_src);
  DVMVS_REQUIRE(d->ksize == 3 || d->ksize == 5, "conv2d_halo: ksize=%d (3 or 5)", d->ksize);
  DVMVS_REQUIRE(d->terms == 1 || d->terms == 3, "conv2d_halo: terms=%d", d->terms);
  DVMVS_REQUIRE(d->kc == 16 || d->kc == 32, "conv2d_halo: kc=%d", d->kc);
  DVMVS_REQUIRE(d->block_n == 32 || d->block_n == 64, "conv2d_halo: block_n=%d", d->block_n);
  DVMVS_REQUIRE(d->B > 0 && d->H > 0 && d->W > 0 && d->Cout > 0 && d->Cout % 8 == 0 && d->w_hi && (d->terms == 1 || d->w_lo),
                "conv2d_halo: bad shape / null weights (Cout must be a multiple of 8)");
  DVMVS_REQUIRE(d->out_f32 || d->out_blk || d->out_nhwc, "conv2d_halo: no output");
  DVMVS_REQUIRE((uintptr_t)d->bias % 16 == 0 && (uintptr_t)d->residual % 16 == 0 && (uintptr_t)d->out_f32 % 16 == 0 &&
                    (uintptr_t)d->out_blk % 16 == 0 && (uintptr_t)d->out_nhwc % 16 == 0,
                "conv2d_halo: bias, residual and outputs must be 16-byte aligned (the epilogue moves 8 channels as 16-byte vectors)");
  HaloParams p;
  memset(&p, 0, sizeof(p));
  p.ksize = d->ksize; p.pad = (d->ksize - 1) / 2; p.terms = d->terms; p.kc = d->kc; p.n_src = d->n_src;
  p.B = d->B; p.Hout = d->H; p.Wout = d->W; p.Cout = d->Cout; p.c8_out = d->Cout / 8;
  p.tiles_x = (d->W + kHaloTileW - 1) / kHaloTileW;
  p.tiles_y = (d->H + kHaloTileH - 1) / kHaloTileH;
  const int halo_w = kHaloTileW + d->ksize - 1, halo_h = kHaloTileH + d->ksize - 1;
  int n_groups = 0;
  for (int s = 0; s < d->n_src; ++s) {
    const int C8 = d->src_c8[s];
    DVMVS_REQUIRE(d->src_blk[s] && C8 > 0, "conv2d_halo: source %d null / empty", s);
    DVMVS_REQUIRE((uintptr_t)d->src_blk[s] % 16 == 0, "conv2d_halo: source %d not 16-byte aligned", s);
    p.src_groups[s] = (C8 * 8 + d->kc - 1) / d->kc;
    n_groups += p.src_groups[s];
    const size_t plane = (size_t)d->B * C8 * d->H * d->W * 8;
    int rc = make_halo_map(&p.a_map[s][0], d->src_blk[s], d->B, d->H, d->W, C8, halo_w, halo_h, d->kc / 8);
    if (rc != DVMVS_OK) return rc;
    if (d->terms > 1) {
      rc = make_halo_map(&p.a_map[s][1], (const __half*)d->src_blk[s] + plane, d->B, d->H, d->W, C8, halo_w, halo_h, d->kc / 8);
      if (rc != DVMVS_OK) return rc;
    }
  }
  p.n_groups = n_groups;
  DVMVS_REQUIRE(d->n_groups == n_groups, "conv2d_halo: weights packed for %d channel groups, sources give %d", d->n_groups, n_groups);
  p.a_bytes = (uint32_t)(d->kc / 8) * halo_h * halo_w * 16;
  p.w_bytes = (uint32_t)d->ksize * (d->kc / 8) * d->block_n * 16;
  p.w_hi = (const __half*)d->w_hi; p.w_lo = (const __half*)d->w_lo;
  p.bias = d->bias; p.residual = d->residual; p.act = d->act;
  p.out_f32 = d->out_f32; p.out_blk = (__half*)d->out_blk; p.out_nhwc = (__half*)d->out_nhwc;
  p.hi_only = d->out_hi_only ? 1 : 0;
  p.dbg = (unsigned long long*)g_halo_dbg;
  const int planes = d->terms > 1 ? 2 : 1;
  const size_t staging = (size_t)128 * (d->block_n + 4) * 4;
  const size_t ring = 2 * (size_t)planes * p.a_bytes + kHaloWStages * (size_t)planes * p.w_bytes;
  p.ring_bytes = (uint32_t)(ring > staging ? ring : staging);
  const size_t smem = p.ring_bytes + 256 + 128;
  DVMVS_REQUIRE(smem <= 227 * 1024, "conv2d_halo: shared memory %zu too large", smem);
  const int n_tiles = (d->Cout + d->block_n - 1) / d->block_n;
  dim3 grid(p.tiles_x * p.tiles_y * d->B, n_tiles, 1);
  cudaStream_t st = (cudaStream_t)stream;
  if (d->block_n == 32) return d->ksize == 3 ? launch_halo_kt<32, 3>(p, grid, smem, st) : launch_halo_kt<32, 5>(p, grid, smem, st);
  return d->ksize == 3 ? launch_halo_kt<64, 3>(p, grid, smem, st) : launch_halo_kt<64, 5>(p, grid, smem, st);
}

extern "C" int dvmvs_split_blocked(const float* x, void* planes, int B, int H, int W, int C, int C8, int flags, int c_offset,
                                   int c_cover, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(x && planes && B > 0 && H > 0 && W > 0 && C > 0 && C8 > 0, "split_blocked: bad argument");
  DVMVS_REQUIRE((flags & ~(DVMVS_SPLIT_UPSAMPLE2X | DVMVS_SPLIT_HI_ONLY)) == 0, "split_blocked: unknown flags 0x%x", flags);
  const int upsample2x = (flags & DVMVS_SPLIT_UPSAMPLE2X) ? 1 : 0;
  DVMVS_REQUIRE(c_offset >= 0 && c_cover >= C && c_offset + c_cover <= C8 * 8, "split_blocked: channel window [%d,+%d) outside %d",
                c_offset, c_cover, C8 * 8);
  DVMVS_REQUIRE(c_offset % 8 == 0, "split_blocked: c_offset must be a multiple of 8 (got %d)", c_offset);
  DVMVS_REQUIRE((uintptr_t)planes % 16 == 0, "split_blocked: planes must be 16-byte aligned");
  const size_t total = (size_t)B * H * W * ((c_cover + 7) / 8) * (upsample2x ? 4 : 1);
  launch_k(split_blocked_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, x, (__half*)planes, B, H, W, C,
           C8, upsample2x, (flags & DVMVS_SPLIT_HI_ONLY) ? 1 : 0, c_offset, c_cover, ((uintptr_t)x % 16 == 0) ? 1 : 0);
  return check_launch("split_blocked_kernel");
}
