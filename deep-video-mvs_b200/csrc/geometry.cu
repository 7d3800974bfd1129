// Geometric kernels of the plane-sweep depth path: fused plane-sweep warp+correlate, pose-aware hidden-state
// warp, forward depth re-projection.  sm_90a.
//
// Reference behaviour reproduced (paths relative to the reference root):
//   dvmvs/utils.py:45-107   calculate_cost_volume_by_warping / cost_volume_fusion
//   dvmvs/utils.py:205-258  warp_frame_depth            dvmvs/convlstm.py:30-41 (transformation, mask)
//   dvmvs/utils.py:110-154  get_non_differentiable_rectangle_depth_estimation
#include <stdarg.h>
#include <stdlib.h>

#include <atomic>

#include <cuda_fp16.h>

#include "common.cuh"

namespace dvmvs {

static thread_local char g_err[512] = "";
static std::atomic<int> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n); }
static std::atomic<int> g_pdl_override{-1};      // -1: environment default, 0 / 1: forced by dvmvs_set_programmatic_launch
bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("DVMVS_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  const int o = g_pdl_override.load();
  return o < 0 ? v == 1 : o == 1;
}

// =====================================================================================================
// Plane sweep
// =====================================================================================================
constexpr int kMaxMeas = 8;
constexpr int kMaxPlanes = 256;

struct SweepParams {
  const float* ref;
  const float* meas[kMaxMeas];
  const float* pose2[kMaxMeas];
  const float* pose1;
  const float* K;
  float* out;
  int B, C, h, w, D, M;
  double inv_base, inv_step;   // python doubles in the reference (utils.py:59-60)
  int mode;
  int prefetch;                // forward fast path: phase A prefetches the tap lines of the NEXT step into L1
};

// Per (b, m): G = K R K^-1 (9 floats), Kt = K t (3 floats)    (utils.py:51-56)
__host__ __device__ __forceinline__ void sweep_matrices(const float* pose1, const float* pose2, const float* K, float* G, float* Kt) {
  float inv2[16], E[16];
  mat4_rigid_free_inverse(pose2, inv2);
  mat4_mul(inv2, pose1, E);
  float R[9] = {E[0], E[1], E[2], E[4], E[5], E[6], E[8], E[9], E[10]};
  float t[3] = {E[3], E[7], E[11]};
  float Kinv[9], KR[9];
  mat3_inverse(K, Kinv);
  mat3_mul(K, R, KR);
  mat3_mul(KR, Kinv, G);
#pragma unroll
  for (int i = 0; i < 3; ++i) Kt[i] = fmaf(K[i * 3 + 2], t[2], fmaf(K[i * 3 + 1], t[1], K[i * 3 + 0] * t[0]));
}

// Sampling position of reference pixel (u,v) on plane with Kt/depth = kd (utils.py:68-73 + the align_corners
// un-normalisation of grid_sample: ((g + 1) / 2) * (size - 1)).
__host__ __device__ __forceinline__ void sweep_sample_pos(const float* base, const float* kd, float wn, float hn, float wm1, float hm1,
                                                 float& xs, float& ys) {
  float q0 = base[0] + kd[0], q1 = base[1] + kd[1], q2 = base[2] + kd[2];
  float den = q2 + 1e-8f;
  float x = q0 / den, y = q1 / den;
  float gx = (x - wn) / wn, gy = (y - hn) / hn;
  xs = ((gx + 1.f) * 0.5f) * wm1;
  ys = ((gy + 1.f) * 0.5f) * hm1;
}

// ---- fast path: C == 32, channel-last.
// The CTA owns kPix consecutive reference pixels of one image row; their 128-byte feature vectors are one contiguous
// span staged in shared memory by a single TMA bulk copy (cp.async.bulk -> UBLKCP).  Work proceeds in steps of
// (kGroup planes x one measurement frame):
//   phase A  one THREAD per (pixel, plane): homography, perspective divide, bilinear weights (zeroed for taps outside
//            the image) and the four clamped tap offsets -> 32 bytes in shared memory.  No redundancy across lanes.
//   phase B  a quarter warp (8 lanes x float4 = 32 channels) per pixel walks the kGroup planes: two broadcast LDS.128
//            for the parameters, four 128-byte-line gathers (one line per tap -- a warp instruction touches 4 lines),
//            16 FMAs to blend + 4 for the dot product; the 8 per-plane partial sums are reduced across the 8 lanes with
//            a transposing butterfly (7 shuffles for 8 planes) so lane j ends up owning plane j.
// Phase A of step i+1 is issued before phase B of step i (double-buffered parameters, one __syncthreads per step).
// Coordinate math: 3 adds, one reciprocal, 4 multiplies (x*(w-1)/w folded into one scale: <= 3 ulp from the
// reference's op sequence, ~1e-5 px).
constexpr int kPix = 32;
constexpr int kGroup = 8;
constexpr int kSweepThreads = 256;

struct __align__(16) SweepTapParams {
  unsigned off[4];   // BYTE offsets of the 4 taps from the start of the measurement feature tensor (clip offset included)
  float w[4];     // bilinear weights, 0 for taps outside the image
};
// The two 16-byte halves of entry e are stored at chunk slots 2e + (c ^ ((e >> 2) & 1)): eight consecutive threads
// then hit eight different 4-bank groups (conflict-free STS.128); readers apply the same swizzle.
__device__ __forceinline__ int sweep_chunk(int e, int c) { return 2 * e + (c ^ ((e >> 2) & 1)); }

__device__ __forceinline__ void sweep_phase_a(const SweepParams& p, const float* s_G, const float* s_kd, SweepTapParams* buf, int m,
                                              int d0, int u0, int v, int npix, float sx, float sy, unsigned clip_off) {
  const int pix = threadIdx.x & (kPix - 1), pl = threadIdx.x >> 5;
  const int d = min(d0 + pl, p.D - 1);
  const float uf = (float)(u0 + min(pix, npix - 1)), vf = (float)v;
  const float* G = s_G + m * 12;
  const float* kd = s_kd + (m * p.D + d) * 4;
  const float q0 = fmaf(G[0], uf, fmaf(G[1], vf, G[2])) + kd[0];
  const float q1 = fmaf(G[3], uf, fmaf(G[4], vf, G[5])) + kd[1];
  const float q2 = fmaf(G[6], uf, fmaf(G[7], vf, G[8])) + kd[2];
  const float r = __frcp_rn(q2 + 1e-8f);
  const float xs = q0 * r * sx, ys = q1 * r * sy;
  SweepTapParams t;
  t.off[0] = t.off[1] = t.off[2] = t.off[3] = clip_off;
  t.w[0] = t.w[1] = t.w[2] = t.w[3] = 0.f;
  // some tap inside the image  <=>  -1 < xs < w  and  -1 < ys < h   (false for NaN / Inf)
  if (xs > -1.f && xs < (float)p.w && ys > -1.f && ys < (float)p.h) {
    const float x0f = floorf(xs), y0f = floorf(ys);
    const float fx = xs - x0f, fy = ys - y0f;
    const float gx = (x0f + 1.f) - xs, gy = (y0f + 1.f) - ys;       // the reference's (x0 + 1 - x) weights
    const int x0 = (int)x0f, y0 = (int)y0f;
    const bool vx0 = x0 >= 0, vx1 = x0 + 1 < p.w, vy0 = y0 >= 0, vy1 = y0 + 1 < p.h;
    const int xa = max(x0, 0), xb = min(x0 + 1, p.w - 1), ya = max(y0, 0), yb = min(y0 + 1, p.h - 1);
    t.off[0] = clip_off + (unsigned)(ya * p.w + xa) * 128u;
    t.off[1] = clip_off + (unsigned)(ya * p.w + xb) * 128u;
    t.off[2] = clip_off + (unsigned)(yb * p.w + xa) * 128u;
    t.off[3] = clip_off + (unsigned)(yb * p.w + xb) * 128u;
    t.w[0] = (vy0 && vx0) ? gx * gy : 0.f;
    t.w[1] = (vy0 && vx1) ? fx * gy : 0.f;
    t.w[2] = (vy1 && vx0) ? gx * fy : 0.f;
    t.w[3] = (vy1 && vx1) ? fx * fy : 0.f;
    if (p.prefetch) {
      // experiment (off by default, slower when measured): phase B of this (plane group, frame) runs one step later;
      // start the 128-byte tap lines towards L1 now so that its gathers hit.
      const char* mb = reinterpret_cast<const char*>(p.meas[m]);
      asm volatile("prefetch.global.L1 [%0];" ::"l"(mb + t.off[0]));
      asm volatile("prefetch.global.L1 [%0];" ::"l"(mb + t.off[1]));
      asm volatile("prefetch.global.L1 [%0];" ::"l"(mb + t.off[2]));
      asm volatile("prefetch.global.L1 [%0];" ::"l"(mb + t.off[3]));
    }
  }
  int4* chunks = reinterpret_cast<int4*>(buf);
  const int e = pl * kPix + pix;
  chunks[sweep_chunk(e, 0)] = *reinterpret_cast<const int4*>(t.off);
  chunks[sweep_chunk(e, 1)] = *reinterpret_cast<const int4*>(t.w);
}

// MINB = CTAs per SM the register allocation is capped for (4: 64 registers, 32 resident warps; 3: 85 registers, 24 warps
// with more gathers in flight per warp -- DVMVS_SWEEP_MINB selects, default 4)
template <int MODE, int MINB = 4>
__global__ void __launch_bounds__(kSweepThreads, MINB) plane_sweep_c32_kernel(SweepParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_ref = reinterpret_cast<float*>(smem_raw);                                     // [kPix][32]
  SweepTapParams* s_par = reinterpret_cast<SweepTapParams*>(s_ref + kPix * 32);          // [2][kGroup][kPix]
  float* s_kd = reinterpret_cast<float*>(s_par + 2 * kGroup * kPix);                     // [M][D][4]  Kt / depth_i
  float* s_G = s_kd + p.M * p.D * 4;                                                     // [M][12]
  float* s_out = s_G + kMaxMeas * 12;                                                    // [kPix][D]
  __shared__ __align__(8) unsigned long long s_bar;

  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const int tiles_per_row = (p.w + kPix - 1) / kPix;
  const int tile = blockIdx.x;
  const int b = tile / (p.h * tiles_per_row);
  const int rem = tile - b * (p.h * tiles_per_row);
  const int v = rem / tiles_per_row;
  const int u0 = (rem - v * tiles_per_row) * kPix;
  const int npix = min(kPix, p.w - u0);

  // --- TMA bulk copy of the reference-feature span into shared memory
  const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&s_bar);
  const uint32_t dst = (uint32_t)__cvta_generic_to_shared(s_ref);
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  if (tid == 0) {
    const uint32_t bytes = (uint32_t)npix * 32u * 4u;
    const float* src = p.ref + (((size_t)b * p.h + v) * p.w + u0) * 32;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
  }
  // --- geometry prologue (overlaps the copy): one thread per measurement frame
  if (tid < p.M) {
    float G[9], Kt[3];
    sweep_matrices(p.pose1 + b * 16, p.pose2[tid] + b * 16, p.K + b * 9, G, Kt);
#pragma unroll
    for (int i = 0; i < 9; ++i) s_G[tid * 12 + i] = G[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) s_G[tid * 12 + 9 + i] = Kt[i];
  }
  __syncthreads();
  for (int i = tid; i < p.M * p.D; i += kSweepThreads) {
    const int m = i / p.D, d = i - m * p.D;
    const float this_depth = (float)(1.0 / (p.inv_base + d * p.inv_step));   // utils.py:66 (double, then fp32 divide)
#pragma unroll
    for (int k = 0; k < 3; ++k) s_kd[i * 4 + k] = s_G[m * 12 + 9 + k] / this_depth;   // utils.py:68
  }
  __syncthreads();

  const float sx = (float)(p.w - 1) / (float)p.w, sy = (float)(p.h - 1) / (float)p.h;   // the align_corners "shrink" (App. A.1)
  const int n_groups = (p.D + kGroup - 1) / kGroup;
  const int n_steps = n_groups * p.M;                     // step = (plane group, measurement frame), frame fastest
  const unsigned clip_off = (unsigned)b * (unsigned)(p.h * p.w) * 128u;     // host guarantees B*h*w*128 < 2^32
  sweep_phase_a(p, s_G, s_kd, s_par, 0, 0, u0, v, npix, sx, sy, clip_off);
  {  // wait for the TMA bytes
    uint32_t done = 0;
    while (!done) {
      asm volatile(
          "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
          : "=r"(done)
          : "r"(bar), "r"(0u)
          : "memory");
    }
  }
  __syncthreads();

  const int lane = tid & 31, warp = tid >> 5;
  const int sub = lane & 7;                 // channel group: channels sub*4 .. sub*4+3
  const int pix = warp * 4 + (lane >> 3);
  const bool active = pix < npix;
  const float4 f1 = *reinterpret_cast<const float4*>(s_ref + (active ? pix : 0) * 32 + sub * 4);
  const float scale = (MODE == DVMVS_SWEEP_DOT) ? (1.f / 32.f) : 1.f;       // utils.py:82 (/C) vs :84

  float acc[kGroup];
#pragma unroll
  for (int k = 0; k < kGroup; ++k) acc[k] = 0.f;

  const int e0 = active ? pix : 0;
  int g = 0, m = 0;                                       // step = g * M + m, kept as counters (no division in the loop)
  for (int step = 0; step < n_steps; ++step) {
    if (step + 1 < n_steps) {
      const int m1 = (m + 1 == p.M) ? 0 : m + 1, g1 = (m + 1 == p.M) ? g + 1 : g;
      sweep_phase_a(p, s_G, s_kd, s_par + ((step + 1) & 1) * kGroup * kPix, m1, g1 * kGroup, u0, v, npix, sx, sy, clip_off);
    }
    const int4* par = reinterpret_cast<const int4*>(s_par + (step & 1) * kGroup * kPix);
    // per-lane 64-bit base (frame m, this lane's 4 channels) + 32-bit byte offsets from phase A: one wide add per tap
    const char* img = reinterpret_cast<const char*>(p.meas[m]) + sub * 16;
#pragma unroll
    for (int k = 0; k < kGroup; ++k) {
      const int e = k * kPix + e0;
      const uint4 off = *reinterpret_cast<const uint4*>(&par[sweep_chunk(e, 0)]);
      const float4 wt = *reinterpret_cast<const float4*>(&par[sweep_chunk(e, 1)]);
      // taps outside the image carry weight 0 (phase A) and are not fetched at all: predicated-off lanes generate no L1
      // wavefronts, and on a forward-moving camera a quarter of all (pixel, plane) samples fall off the image at the
      // near planes.  grid_sample's zero padding contributes exactly 0 there, as does a skipped tap.
      const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
      float4 t00 = zero4, t01 = zero4, t10 = zero4, t11 = zero4;
      if (wt.x != 0.f) t00 = __ldg(reinterpret_cast<const float4*>(img + off.x));
      if (wt.y != 0.f) t01 = __ldg(reinterpret_cast<const float4*>(img + off.y));
      if (wt.z != 0.f) t10 = __ldg(reinterpret_cast<const float4*>(img + off.z));
      if (wt.w != 0.f) t11 = __ldg(reinterpret_cast<const float4*>(img + off.w));
      float4 ws;
      ws.x = fmaf(t11.x, wt.w, fmaf(t10.x, wt.z, fmaf(t01.x, wt.y, t00.x * wt.x)));
      ws.y = fmaf(t11.y, wt.w, fmaf(t10.y, wt.z, fmaf(t01.y, wt.y, t00.y * wt.x)));
      ws.z = fmaf(t11.z, wt.w, fmaf(t10.z, wt.z, fmaf(t01.z, wt.y, t00.z * wt.x)));
      ws.w = fmaf(t11.w, wt.w, fmaf(t10.w, wt.z, fmaf(t01.w, wt.y, t00.w * wt.x)));
      float part;
      if (MODE == DVMVS_SWEEP_DOT)
        part = fmaf(f1.w, ws.w, fmaf(f1.z, ws.z, fmaf(f1.y, ws.y, f1.x * ws.x)));
      else
        part = fabsf(f1.x - ws.x) + fabsf(f1.y - ws.y) + fabsf(f1.z - ws.z) + fabsf(f1.w - ws.w);
      acc[k] = fmaf(part, scale, acc[k]);
    }
    if (m == p.M - 1) {
      // transposing butterfly over the 8 lanes of the quarter warp: lane `sub` ends up with the sum for plane `sub`
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float send = (sub & 4) ? acc[k] : acc[k + 4];
        const float keep = (sub & 4) ? acc[k + 4] : acc[k];
        acc[k] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const float send = (sub & 2) ? acc[k] : acc[k + 2];
        const float keep = (sub & 2) ? acc[k + 2] : acc[k];
        acc[k] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
      }
      {
        const float send = (sub & 1) ? acc[0] : acc[1];
        const float keep = (sub & 1) ? acc[1] : acc[0];
        acc[0] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
      }
      const int d = g * kGroup + sub;
      if (active && d < p.D) s_out[pix * p.D + d] = acc[0] / (float)p.M;     // utils.py:105-106
#pragma unroll
      for (int k = 0; k < kGroup; ++k) acc[k] = 0.f;
    }
    __syncthreads();
    if (++m == p.M) { m = 0; ++g; }
  }
  // coalesced write-out: [npix][D] is contiguous in the channel-last cost volume
  float* o = p.out + (((size_t)b * p.h + v) * p.w + u0) * p.D;
  const int n_items = npix * p.D;
  for (int i = tid; i < n_items; i += kSweepThreads) o[i] = s_out[i];
}

// =====================================================================================================
// Backward of the plane sweep (SURVEY section 8 row f3; training entry point fusionnet/run-training.py:231)
// =====================================================================================================
// cost[b,d,v,u] = 1/(M*32) * sum_m sum_c f1[c] * sum_t w_t f2_m[q_t][c]      (dot-product mode, utils.py:45-107)
//   d cost / d f1[c]        = 1/(M*32) * sum_{m,d} g[d] * warped_{m,d}[c]     -> gather, same access pattern as the forward
//   d cost / d f2_m[q_t][c] = 1/(M*32) * g[d] * w_t * f1[c]                   -> scatter-add (vector red.global.add.v4.f32)
// Same tiling as the forward kernel: CTA = kPix pixels of a row, phase A (one thread per (pixel, plane): tap offsets and
// weights) / phase B (a quarter warp per pixel, 4 channels per lane).  The gradient w.r.t. the reference features is
// accumulated in registers and written once (deterministic); the measurement-feature gradient is accumulated with
// floating-point atomics into buffers the host zeroes, so its summation order is not reproducible bit-for-bit (as in
// PyTorch's grid_sampler backward).  Poses and intrinsics receive no gradient (the reference trains with fixed poses).
struct SweepBwdParams {
  SweepParams f;
  const float* gcost;              // (B, h, w, D)
  float* gref;                     // (B, h, w, 32)
  float* gmeas[kMaxMeas];          // (B, h, w, 32) each, zero-initialised
};

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

__global__ void __launch_bounds__(kSweepThreads, 2) plane_sweep_backward_c32_kernel(SweepBwdParams q) {
  const SweepParams& p = q.f;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_ref = reinterpret_cast<float*>(smem_raw);                                     // [kPix][32]
  SweepTapParams* s_par = reinterpret_cast<SweepTapParams*>(s_ref + kPix * 32);          // [kGroup][kPix]
  float* s_kd = reinterpret_cast<float*>(s_par + kGroup * kPix);                         // [M][D][4]
  float* s_G = s_kd + p.M * p.D * 4;                                                     // [M][12]
  float* s_g = s_G + kMaxMeas * 12;                                                      // [kPix][D] upstream gradient

  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const int tiles_per_row = (p.w + kPix - 1) / kPix;
  const int tile = blockIdx.x;
  const int b = tile / (p.h * tiles_per_row);
  const int rem = tile - b * (p.h * tiles_per_row);
  const int v = rem / tiles_per_row;
  const int u0 = (rem - v * tiles_per_row) * kPix;
  const int npix = min(kPix, p.w - u0);
  pdl_wait();

  const size_t pix0 = ((size_t)b * p.h + v) * p.w + u0;
  if (tid < npix * 8) reinterpret_cast<float4*>(s_ref)[tid] = __ldg(reinterpret_cast<const float4*>(p.ref + pix0 * 32) + tid);
  const float gscale = 1.f / (32.f * (float)p.M);
  for (int i = tid; i < npix * p.D; i += kSweepThreads) s_g[i] = q.gcost[pix0 * p.D + i] * gscale;
  if (tid < p.M) {
    float G[9], Kt[3];
    sweep_matrices(p.pose1 + b * 16, p.pose2[tid] + b * 16, p.K + b * 9, G, Kt);
#pragma unroll
    for (int i = 0; i < 9; ++i) s_G[tid * 12 + i] = G[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) s_G[tid * 12 + 9 + i] = Kt[i];
  }
  __syncthreads();
  for (int i = tid; i < p.M * p.D; i += kSweepThreads) {
    const int m = i / p.D, d = i - m * p.D;
    const float this_depth = (float)(1.0 / (p.inv_base + d * p.inv_step));
#pragma unroll
    for (int k = 0; k < 3; ++k) s_kd[i * 4 + k] = s_G[m * 12 + 9 + k] / this_depth;
  }
  __syncthreads();

  const float sx = (float)(p.w - 1) / (float)p.w, sy = (float)(p.h - 1) / (float)p.h;
  const unsigned clip_off = (unsigned)b * (unsigned)(p.h * p.w) * 128u;
  const int lane = tid & 31, warp = tid >> 5;
  const int sub = lane & 7;
  const int pix = warp * 4 + (lane >> 3);
  const bool active = pix < npix;
  const int e0 = active ? pix : 0;
  const float4 f1 = *reinterpret_cast<const float4*>(s_ref + e0 * 32 + sub * 4);
  float4 gacc = make_float4(0.f, 0.f, 0.f, 0.f);
  const int n_groups = (p.D + kGroup - 1) / kGroup;
  for (int g = 0; g < n_groups; ++g) {
    for (int m = 0; m < p.M; ++m) {
      sweep_phase_a(p, s_G, s_kd, s_par, m, g * kGroup, u0, v, npix, sx, sy, clip_off);
      __syncthreads();
      if (active) {
        const int4* par = reinterpret_cast<const int4*>(s_par);
        const char* img = reinterpret_cast<const char*>(p.meas[m]) + sub * 16;
        char* gimg = reinterpret_cast<char*>(q.gmeas[m]) + sub * 16;
#pragma unroll 2
        for (int k = 0; k < kGroup; ++k) {
          const int d = g * kGroup + k;
          if (d >= p.D) break;
          const float gd = s_g[e0 * p.D + d];
          if (gd == 0.f) continue;
          const int e = k * kPix + e0;
          const uint4 off = *reinterpret_cast<const uint4*>(&par[sweep_chunk(e, 0)]);
          const float4 wt = *reinterpret_cast<const float4*>(&par[sweep_chunk(e, 1)]);
          const float4 t00 = __ldg(reinterpret_cast<const float4*>(img + off.x));
          const float4 t01 = __ldg(reinterpret_cast<const float4*>(img + off.y));
          const float4 t10 = __ldg(reinterpret_cast<const float4*>(img + off.z));
          const float4 t11 = __ldg(reinterpret_cast<const float4*>(img + off.w));
          gacc.x = fmaf(gd, fmaf(t11.x, wt.w, fmaf(t10.x, wt.z, fmaf(t01.x, wt.y, t00.x * wt.x))), gacc.x);
          gacc.y = fmaf(gd, fmaf(t11.y, wt.w, fmaf(t10.y, wt.z, fmaf(t01.y, wt.y, t00.y * wt.x))), gacc.y);
          gacc.z = fmaf(gd, fmaf(t11.z, wt.w, fmaf(t10.z, wt.z, fmaf(t01.z, wt.y, t00.z * wt.x))), gacc.z);
          gacc.w = fmaf(gd, fmaf(t11.w, wt.w, fmaf(t10.w, wt.z, fmaf(t01.w, wt.y, t00.w * wt.x))), gacc.w);
          const float c0 = gd * wt.x, c1 = gd * wt.y, c2 = gd * wt.z, c3 = gd * wt.w;     // zero weight <=> tap outside the image
          if (c0 != 0.f) red_add_v4(reinterpret_cast<float*>(gimg + off.x), c0 * f1.x, c0 * f1.y, c0 * f1.z, c0 * f1.w);
          if (c1 != 0.f) red_add_v4(reinterpret_cast<float*>(gimg + off.y), c1 * f1.x, c1 * f1.y, c1 * f1.z, c1 * f1.w);
          if (c2 != 0.f) red_add_v4(reinterpret_cast<float*>(gimg + off.z), c2 * f1.x, c2 * f1.y, c2 * f1.z, c2 * f1.w);
          if (c3 != 0.f) red_add_v4(reinterpret_cast<float*>(gimg + off.w), c3 * f1.x, c3 * f1.y, c3 * f1.z, c3 * f1.w);
        }
      }
      __syncthreads();
    }
  }
  if (active) *reinterpret_cast<float4*>(q.gref + (pix0 + pix) * 32 + sub * 4) = gacc;
}

// =====================================================================================================
// Plane sweep over 16-bit measurement features -- EXPERIMENTAL, opt-in (DVMVS_SWEEP_FP16=1 in the Python binding), not yet
// measured on hardware.  Motivation (DESIGN.md section 9): the fp32 kernel sits on the L1 gather path; a CPU probe with the
// oracle (tools/feature_fp16_probe.py) shows that rounding the sweep's feature inputs to fp16 moves the final inverse depth
// by <= 1.3e-6 (budget 1e-3), and the FPN's output convolution already emits the fp16 "hi" plane of its result.
//   * a measurement pixel is 64 bytes, so the two taps of one bilinear ROW (x, x+1) are one contiguous 128-byte span:
//     a quarter warp fetches it with ONE 16-byte load per lane (lanes 0-3: left pixel, 4-7: right pixel) -- two load
//     instructions and <= 4 cache lines per sample instead of four and four;
//   * no blended vector is formed: cost = sum_taps w_t * (f1 . tap_t) is linear, each lane dots its 8 channels of its side
//     with the matching 8 reference channels and scales by its side's weight; the butterfly over the 8 lanes then adds
//     channels and sides at once.  fp32 accumulation; dot-product mode only.
// Phase A (one thread per (pixel, plane)) stores per row the byte offset of the in-image pixel pair (xa, xa+1),
// xa = clamp(x0, 0, w-2), and the weights of its left / right member (0 where the tap falls outside the image).
struct __align__(16) SweepPairParams {
  unsigned off[2];     // byte offsets of the pixel pairs of the two rows (clip offset included)
  unsigned pad[2];
  float w[4];          // row0-left, row0-right, row1-left, row1-right
};

__device__ __forceinline__ void sweep_phase_a_h16(const SweepParams& p, const float* s_G, const float* s_kd, SweepPairParams* buf, int m,
                                                  int d0, int u0, int v, int npix, float sx, float sy, unsigned clip_off) {
  const int pix = threadIdx.x & (kPix - 1), pl = threadIdx.x >> 5;
  const int d = min(d0 + pl, p.D - 1);
  const float uf = (float)(u0 + min(pix, npix - 1)), vf = (float)v;
  const float* G = s_G + m * 12;
  const float* kd = s_kd + (m * p.D + d) * 4;
  const float q0 = fmaf(G[0], uf, fmaf(G[1], vf, G[2])) + kd[0];
  const float q1 = fmaf(G[3], uf, fmaf(G[4], vf, G[5])) + kd[1];
  const float q2 = fmaf(G[6], uf, fmaf(G[7], vf, G[8])) + kd[2];
  const float r = __frcp_rn(q2 + 1e-8f);
  const float xs = q0 * r * sx, ys = q1 * r * sy;
  SweepPairParams t;
  t.off[0] = t.off[1] = clip_off;
  t.pad[0] = t.pad[1] = 0u;
  t.w[0] = t.w[1] = t.w[2] = t.w[3] = 0.f;
  if (xs > -1.f && xs < (float)p.w && ys > -1.f && ys < (float)p.h) {
    const float x0f = floorf(xs), y0f = floorf(ys);
    const float fx = xs - x0f, fy = ys - y0f;
    const float gx = (x0f + 1.f) - xs, gy = (y0f + 1.f) - ys;
    const int x0 = (int)x0f, y0 = (int)y0f;
    // pair (xa, xa+1) inside the image; the weights follow the taps: x0 -> gx, x0+1 -> fx
    const int xa = min(max(x0, 0), p.w - 2);
    const float wl = (x0 == xa) ? gx : ((x0 + 1 == xa) ? fx : 0.f);          // tap that lands on pixel xa
    const float wr = (x0 + 1 == xa + 1) ? fx : ((x0 == xa + 1) ? gx : 0.f);  // tap that lands on pixel xa + 1
    const bool vy0 = y0 >= 0, vy1 = y0 + 1 < p.h;
    const int ya = max(y0, 0), yb = min(y0 + 1, p.h - 1);
    t.off[0] = clip_off + (unsigned)(ya * p.w + xa) * 64u;
    t.off[1] = clip_off + (unsigned)(yb * p.w + xa) * 64u;
    t.w[0] = vy0 ? wl * gy : 0.f;
    t.w[1] = vy0 ? wr * gy : 0.f;
    t.w[2] = vy1 ? wl * fy : 0.f;
    t.w[3] = vy1 ? wr * fy : 0.f;
  }
  int4* chunks = reinterpret_cast<int4*>(buf);
  const int e = pl * kPix + pix;
  chunks[sweep_chunk(e, 0)] = *reinterpret_cast<const int4*>(t.off);
  chunks[sweep_chunk(e, 1)] = *reinterpret_cast<const int4*>(t.w);
}

__device__ __forceinline__ float dot8_h(const uint4 raw, const float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&raw);
  const float2 a = __half22float2(h[0]), b = __half22float2(h[1]), c = __half22float2(h[2]), d = __half22float2(h[3]);
  return fmaf(f[7], d.y, fmaf(f[6], d.x, fmaf(f[5], c.y, fmaf(f[4], c.x, fmaf(f[3], b.y, fmaf(f[2], b.x, fmaf(f[1], a.y, f[0] * a.x)))))));
}

__global__ void __launch_bounds__(kSweepThreads, 4) plane_sweep_c32_h16_kernel(SweepParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_ref = reinterpret_cast<float*>(smem_raw);                                     // [kPix][32] fp32
  SweepPairParams* s_par = reinterpret_cast<SweepPairParams*>(s_ref + kPix * 32);        // [2][kGroup][kPix]
  float* s_kd = reinterpret_cast<float*>(s_par + 2 * kGroup * kPix);                     // [M][D][4]
  float* s_G = s_kd + p.M * p.D * 4;                                                     // [M][12]
  float* s_out = s_G + kMaxMeas * 12;                                                    // [kPix][D]

  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const int tiles_per_row = (p.w + kPix - 1) / kPix;
  const int tile = blockIdx.x;
  const int b = tile / (p.h * tiles_per_row);
  const int rem = tile - b * (p.h * tiles_per_row);
  const int v = rem / tiles_per_row;
  const int u0 = (rem - v * tiles_per_row) * kPix;
  const int npix = min(kPix, p.w - u0);
  pdl_wait();
  const size_t pix0 = ((size_t)b * p.h + v) * p.w + u0;
  if (tid < npix * 8) reinterpret_cast<float4*>(s_ref)[tid] = __ldg(reinterpret_cast<const float4*>(p.ref + pix0 * 32) + tid);
  if (tid < p.M) {
    float G[9], Kt[3];
    sweep_matrices(p.pose1 + b * 16, p.pose2[tid] + b * 16, p.K + b * 9, G, Kt);
#pragma unroll
    for (int i = 0; i < 9; ++i) s_G[tid * 12 + i] = G[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) s_G[tid * 12 + 9 + i] = Kt[i];
  }
  __syncthreads();
  for (int i = tid; i < p.M * p.D; i += kSweepThreads) {
    const int m = i / p.D, d = i - m * p.D;
    const float this_depth = (float)(1.0 / (p.inv_base + d * p.inv_step));
#pragma unroll
    for (int k = 0; k < 3; ++k) s_kd[i * 4 + k] = s_G[m * 12 + 9 + k] / this_depth;
  }
  __syncthreads();

  const float sx = (float)(p.w - 1) / (float)p.w, sy = (float)(p.h - 1) / (float)p.h;
  const unsigned clip_off = (unsigned)b * (unsigned)(p.h * p.w) * 64u;
  const int n_groups = (p.D + kGroup - 1) / kGroup;
  const int n_steps = n_groups * p.M;
  sweep_phase_a_h16(p, s_G, s_kd, s_par, 0, 0, u0, v, npix, sx, sy, clip_off);
  __syncthreads();

  const int lane = tid & 31, warp = tid >> 5;
  const int sub = lane & 7;                 // lanes 0-3: left pixel of the pair, 4-7: right pixel; channels (sub & 3) * 8 .. + 7
  const int side = sub >> 2;
  const int pix = warp * 4 + (lane >> 3);
  const bool active = pix < npix;
  const int e0 = active ? pix : 0;
  float f1[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) f1[c] = s_ref[e0 * 32 + (sub & 3) * 8 + c];

  float acc[kGroup];
#pragma unroll
  for (int k = 0; k < kGroup; ++k) acc[k] = 0.f;
  int g = 0, m = 0;
  for (int step = 0; step < n_steps; ++step) {
    if (step + 1 < n_steps) {
      const int m1 = (m + 1 == p.M) ? 0 : m + 1, g1 = (m + 1 == p.M) ? g + 1 : g;
      sweep_phase_a_h16(p, s_G, s_kd, s_par + ((step + 1) & 1) * kGroup * kPix, m1, g1 * kGroup, u0, v, npix, sx, sy, clip_off);
    }
    const int4* par = reinterpret_cast<const int4*>(s_par + (step & 1) * kGroup * kPix);
    const char* img = reinterpret_cast<const char*>(p.meas[m]) + sub * 16;      // 16 bytes = 8 halfs of this lane's pixel of the pair
#pragma unroll
    for (int k = 0; k < kGroup; ++k) {
      const int e = k * kPix + e0;
      const uint4 off = *reinterpret_cast<const uint4*>(&par[sweep_chunk(e, 0)]);
      const float4 wt = *reinterpret_cast<const float4*>(&par[sweep_chunk(e, 1)]);
      const float w0 = side ? wt.y : wt.x, w1 = side ? wt.w : wt.z;           // this lane's side, rows 0 / 1
      float part = 0.f;
      if (w0 != 0.f) part = w0 * dot8_h(__ldg(reinterpret_cast<const uint4*>(img + off.x)), f1);
      if (w1 != 0.f) part = fmaf(w1, dot8_h(__ldg(reinterpret_cast<const uint4*>(img + off.y)), f1), part);
      acc[k] = fmaf(part, 1.f / 32.f, acc[k]);
    }
    if (m == p.M - 1) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float send = (sub & 4) ? acc[k] : acc[k + 4];
        const float keep = (sub & 4) ? acc[k + 4] : acc[k];
        acc[k] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const float send = (sub & 2) ? acc[k] : acc[k + 2];
        const float keep = (sub & 2) ? acc[k + 2] : acc[k];
        acc[k] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
      }
      {
        const float send = (sub & 1) ? acc[0] : acc[1];
        const float keep = (sub & 1) ? acc[1] : acc[0];
        acc[0] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
      }
      const int d = g * kGroup + sub;
      if (active && d < p.D) s_out[pix * p.D + d] = acc[0] / (float)p.M;
#pragma unroll
      for (int k = 0; k < kGroup; ++k) acc[k] = 0.f;
    }
    __syncthreads();
    if (++m == p.M) { m = 0; ++g; }
  }
  float* o = p.out + pix0 * p.D;
  const int n_items = npix * p.D;
  for (int i = tid; i < n_items; i += kSweepThreads) o[i] = s_out[i];
}

// ---- generic path: any C, one thread per (pixel, plane); also the on-device cross-check of the fast path.
__global__ void plane_sweep_generic_kernel(SweepParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)p.B * p.h * p.w * p.D;
  if (idx >= total) return;
  const int d = (int)(idx % p.D);
  size_t pixi = idx / p.D;
  const int u = (int)(pixi % p.w);
  const int v = (int)((pixi / p.w) % p.h);
  const int b = (int)(pixi / ((size_t)p.w * p.h));
  const float wn = p.w * 0.5f, hn = p.h * 0.5f, wm1 = (float)(p.w - 1), hm1 = (float)(p.h - 1);
  const float* f1 = p.ref + pixi * p.C;
  const float this_depth = (float)(1.0 / (p.inv_base + d * p.inv_step));
  float acc = 0.f;
  for (int m = 0; m < p.M; ++m) {
    float G[9], Kt[3];
    sweep_matrices(p.pose1 + b * 16, p.pose2[m] + b * 16, p.K + b * 9, G, Kt);
    float base[3], kd[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      base[k] = fmaf(G[k * 3 + 0], (float)u, fmaf(G[k * 3 + 1], (float)v, G[k * 3 + 2]));
      kd[k] = Kt[k] / this_depth;
    }
    float xs, ys;
    sweep_sample_pos(base, kd, wn, hn, wm1, hm1, xs, ys);
    const float x0f = floorf(xs), y0f = floorf(ys);
    const float wx[2] = {(x0f + 1.f) - xs, xs - x0f}, wy[2] = {(y0f + 1.f) - ys, ys - y0f};
    const float* img = p.meas[m] + (size_t)b * p.h * p.w * p.C;
    float part = 0.f;
    for (int c = 0; c < p.C; ++c) {
      float warped = 0.f;
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const float xf = x0f + dx, yf = y0f + dy;
          if (xf >= 0.f && xf <= wm1 && yf >= 0.f && yf <= hm1)
            warped = fmaf(img[((size_t)(int)yf * p.w + (int)xf) * p.C + c], wx[dx] * wy[dy], warped);
        }
      part += (p.mode == DVMVS_SWEEP_DOT) ? f1[c] * warped : fabsf(f1[c] - warped);
    }
    acc += (p.mode == DVMVS_SWEEP_DOT) ? part / (float)p.C : part;
  }
  p.out[idx] = acc / (float)p.M;
}

// =====================================================================================================
// Hidden-state warp (+ invalid-depth mask)
// =====================================================================================================
__global__ void hidden_warp_kernel(const float* __restrict__ h_in, const float* __restrict__ depth,
                                   const float* __restrict__ prev_pose, const float* __restrict__ cur_pose,
                                   const float* __restrict__ K, float* __restrict__ h_out, int B, int C, int h, int w,
                                   float invalid_thresh) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_T[16];
  const int b = blockIdx.y;
  if (threadIdx.x == 0) {
    if (prev_pose != nullptr) {
      float inv[16], T[16];
      mat4_rigid_free_inverse(prev_pose + b * 16, inv);                  // convlstm.py:30
      mat4_mul(inv, cur_pose + b * 16, T);
      for (int i = 0; i < 16; ++i) s_T[i] = T[i];
    } else {
      for (int i = 0; i < 16; ++i) s_T[i] = cur_pose[b * 16 + i];
    }
  }
  __syncthreads();
  const int c4 = C >> 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= h * w * c4) return;
  const int cg = idx % c4;
  const int pix = idx / c4;
  const int u = pix % w, v = pix / w;
  const float* Kb = K + b * 9;
  const float fx = Kb[0], fy = Kb[4], cx = Kb[2], cy = Kb[5];
  const float d = depth[(size_t)b * h * w + pix];
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!(d <= invalid_thresh)) {                                          // convlstm.py:32,40-41
    // kornia depth_to_3d / transform_points / relu(z) / project_points (guarded divide)   utils.py:241-252
    const float X = ((float)u - cx) / fx * d, Y = ((float)v - cy) / fy * d, Z = d;
    const float x = fmaf(s_T[0], X, fmaf(s_T[1], Y, s_T[2] * Z)) + s_T[3];
    const float y = fmaf(s_T[4], X, fmaf(s_T[5], Y, s_T[6] * Z)) + s_T[7];
    float z = fmaf(s_T[8], X, fmaf(s_T[9], Y, s_T[10] * Z)) + s_T[11];
    z = fmaxf(z, 0.f);
    const float scale = (fabsf(z) > 1e-8f) ? 1.f / z : 1.f;
    const float us = x * scale * fx + cx, vs = y * scale * fy + cy;
    // normalize_pixel_coordinates + align_corners=True == sample at (us, vs)
    const float gx = us * (2.f / (float)(w - 1)) - 1.f, gy = vs * (2.f / (float)(h - 1)) - 1.f;
    const float xs = ((gx + 1.f) * 0.5f) * (float)(w - 1), ys = ((gy + 1.f) * 0.5f) * (float)(h - 1);
    const float x0f = floorf(xs), y0f = floorf(ys);
    const float wx[2] = {(x0f + 1.f) - xs, xs - x0f}, wy[2] = {(y0f + 1.f) - ys, ys - y0f};
    const float* img = h_in + (size_t)b * h * w * C + cg * 4;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const float xf = x0f + dx, yf = y0f + dy;
        if (xf >= 0.f && xf <= (float)(w - 1) && yf >= 0.f && yf <= (float)(h - 1)) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(img + ((size_t)(int)yf * w + (int)xf) * C));
          const float wt = wx[dx] * wy[dy];
          o.x = fmaf(t.x, wt, o.x);
          o.y = fmaf(t.y, wt, o.y);
          o.z = fmaf(t.z, wt, o.z);
          o.w = fmaf(t.w, wt, o.w);
        }
      }
  }
  *reinterpret_cast<float4*>(h_out + ((size_t)b * h * w + pix) * C + cg * 4) = o;
}

// Backward of the hidden-state warp w.r.t. the warped tensor (row f3; BPTT through convlstm.py:33-41): the forward's
// bilinear weights scattered back, gh_in[q_t] += w_t * g[p] for valid depths (masked positions pass no gradient).
// The depth comes from the ground truth in training (run-training.py:245-258) and gets no gradient.  gh_in is zeroed by
// the host.
__global__ void hidden_warp_backward_kernel(const float* __restrict__ g_out, const float* __restrict__ depth,
                                            const float* __restrict__ prev_pose, const float* __restrict__ cur_pose,
                                            const float* __restrict__ K, float* __restrict__ gh_in, int B, int C, int h, int w,
                                            float invalid_thresh) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_T[16];
  const int b = blockIdx.y;
  if (threadIdx.x == 0) {
    if (prev_pose != nullptr) {
      float inv[16], T[16];
      mat4_rigid_free_inverse(prev_pose + b * 16, inv);
      mat4_mul(inv, cur_pose + b * 16, T);
      for (int i = 0; i < 16; ++i) s_T[i] = T[i];
    } else {
      for (int i = 0; i < 16; ++i) s_T[i] = cur_pose[b * 16 + i];
    }
  }
  __syncthreads();
  const int c4 = C >> 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= h * w * c4) return;
  const int cg = idx % c4;
  const int pix = idx / c4;
  const int u = pix % w, v = pix / w;
  const float* Kb = K + b * 9;
  const float fx = Kb[0], fy = Kb[4], cx = Kb[2], cy = Kb[5];
  const float d = depth[(size_t)b * h * w + pix];
  if (d <= invalid_thresh) return;
  const float X = ((float)u - cx) / fx * d, Y = ((float)v - cy) / fy * d, Z = d;
  const float x = fmaf(s_T[0], X, fmaf(s_T[1], Y, s_T[2] * Z)) + s_T[3];
  const float y = fmaf(s_T[4], X, fmaf(s_T[5], Y, s_T[6] * Z)) + s_T[7];
  float z = fmaf(s_T[8], X, fmaf(s_T[9], Y, s_T[10] * Z)) + s_T[11];
  z = fmaxf(z, 0.f);
  const float scale = (fabsf(z) > 1e-8f) ? 1.f / z : 1.f;
  const float us = x * scale * fx + cx, vs = y * scale * fy + cy;
  const float gx = us * (2.f / (float)(w - 1)) - 1.f, gy = vs * (2.f / (float)(h - 1)) - 1.f;
  const float xs = ((gx + 1.f) * 0.5f) * (float)(w - 1), ys = ((gy + 1.f) * 0.5f) * (float)(h - 1);
  const float x0f = floorf(xs), y0f = floorf(ys);
  const float wx[2] = {(x0f + 1.f) - xs, xs - x0f}, wy[2] = {(y0f + 1.f) - ys, ys - y0f};
  const float4 g = __ldg(reinterpret_cast<const float4*>(g_out + ((size_t)b * h * w + pix) * C + cg * 4));
  float* gimg = gh_in + (size_t)b * h * w * C + cg * 4;
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const float xf = x0f + dx, yf = y0f + dy;
      if (xf >= 0.f && xf <= (float)(w - 1) && yf >= 0.f && yf <= (float)(h - 1)) {
        const float wt = wx[dx] * wy[dy];
        red_add_v4(gimg + ((size_t)(int)yf * w + (int)xf) * C, wt * g.x, wt * g.y, wt * g.z, wt * g.w);
      }
    }
}

// =====================================================================================================
// Depth re-projection: z-as-uint atomicMax scatter (z >= 0 so the float order equals the uint order)
// =====================================================================================================
__global__ void depth_reproject_kernel(const float* __restrict__ cur_pose, const float* __restrict__ prev_pose,
                                       const float* __restrict__ prev_depth, const float* __restrict__ full_K,
                                       const float* __restrict__ half_K, unsigned int* __restrict__ out, int B, int H, int W) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_T[16];
  const int b = blockIdx.y;
  if (threadIdx.x == 0) {
    float inv[16], T[16];
    mat4_rigid_free_inverse(cur_pose + b * 16, inv);                     // utils.py:121
    mat4_mul(inv, prev_pose + b * 16, T);
    for (int i = 0; i < 16; ++i) s_T[i] = T[i];
  }
  __syncthreads();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= H * W) return;
  const int u = pix % W, v = pix / W;
  const float* Kf = full_K + b * 9;
  const float* Kh = half_K + b * 9;
  const float d = prev_depth[(size_t)b * H * W + pix];
  const float X = ((float)u - Kf[2]) / Kf[0] * d, Y = ((float)v - Kf[5]) / Kf[4] * d, Z = d;      // utils.py:122
  const float x = fmaf(s_T[0], X, fmaf(s_T[1], Y, s_T[2] * Z)) + s_T[3];
  const float y = fmaf(s_T[4], X, fmaf(s_T[5], Y, s_T[6] * Z)) + s_T[7];
  const float z = fmaf(s_T[8], X, fmaf(s_T[9], Y, s_T[10] * Z)) + s_T[11];
  const float zr = fmaxf(z, 0.f);                                        // utils.py:129
  const float scale = (fabsf(z) > 1e-8f) ? 1.f / z : 1.f;                // project_points on the un-relu'd point
  const float pu = rintf(x * scale * Kh[0] + Kh[2]);                     // torch.round = half-to-even
  const float pv = rintf(y * scale * Kh[4] + Kh[5]);
  const int hw = W / 2, hh = H / 2;
  if (pu >= 0.f && pv >= 0.f && pu < (float)hw && pv < (float)hh) {      // utils.py:137-139
    atomicMax(out + (size_t)b * hh * hw + (size_t)(int)pv * hw + (int)pu, __float_as_uint(zr));
  }
}

}  // namespace dvmvs

using namespace dvmvs;

extern "C" int dvmvs_abi_version(void) { return 6; }

// Programmatic dependent launch for the launches that follow (process-wide): 1 on, 0 off, -1 back to the default
// (on unless DVMVS_PDL=0).  What a launch was enqueued / captured with stays with it.
extern "C" int dvmvs_set_programmatic_launch(int mode) {
  DVMVS_REQUIRE(mode >= -1 && mode <= 1, "set_programmatic_launch: mode %d", mode);
  g_pdl_override.store(mode);
  return DVMVS_OK;
}

// Host-side evaluation of the geometry prologue (same code the kernels run); lets the CPU test-suite check the
// pose algebra without a GPU.  All pointers are HOST pointers here.
extern "C" int dvmvs_host_sweep_geometry(const float* pose1_host, const float* pose2_host, const float* K_host, float u, float v,
                                         int h, int w, int d, int D, float min_depth, float max_depth, float* G_Kt_host,
                                         float* xy_host) {
  DVMVS_REQUIRE(pose1_host && pose2_host && K_host && G_Kt_host && xy_host && D >= 2, "host_sweep_geometry: bad argument");
  float G[9], Kt[3];
  sweep_matrices(pose1_host, pose2_host, K_host, G, Kt);
  for (int i = 0; i < 9; ++i) G_Kt_host[i] = G[i];
  for (int i = 0; i < 3; ++i) G_Kt_host[9 + i] = Kt[i];
  const double inv_base = 1.0 / (double)max_depth, inv_step = (1.0 / (double)min_depth - 1.0 / (double)max_depth) / (double)(D - 1);
  const float this_depth = (float)(1.0 / (inv_base + d * inv_step));
  float base[3], kd[3];
  for (int k = 0; k < 3; ++k) {
    base[k] = fmaf(G[k * 3 + 0], u, fmaf(G[k * 3 + 1], v, G[k * 3 + 2]));
    kd[k] = Kt[k] / this_depth;
  }
  sweep_sample_pos(base, kd, w * 0.5f, h * 0.5f, (float)(w - 1), (float)(h - 1), xy_host[0], xy_host[1]);
  return DVMVS_OK;
}
extern "C" const char* dvmvs_last_error_string(void) { return g_err; }
extern "C" int dvmvs_kernel_launch_count(void) { return g_launches.load(); }

extern "C" int dvmvs_plane_sweep_fused(const float* ref, const float* const* meas_host, const float* pose1,
                                       const float* const* pose2_host, const float* K, float* cost_out, int B, int C,
                                       int h, int w, int D, int M, float min_depth, float max_depth, int mode,
                                       dvmvs_stream_t stream) {
  DVMVS_REQUIRE(ref && meas_host && pose1 && pose2_host && K && cost_out, "plane_sweep: null pointer");
  DVMVS_REQUIRE(B > 0 && C > 0 && h > 1 && w > 1, "plane_sweep: bad shape B=%d C=%d h=%d w=%d", B, C, h, w);
  DVMVS_REQUIRE(D >= 2 && D <= kMaxPlanes, "plane_sweep: D=%d outside [2,%d]", D, kMaxPlanes);
  DVMVS_REQUIRE(M >= 1 && M <= kMaxMeas, "plane_sweep: M=%d outside [1,%d]", M, kMaxMeas);
  DVMVS_REQUIRE(mode == DVMVS_SWEEP_DOT || mode == DVMVS_SWEEP_SAD, "plane_sweep: bad mode %d", mode);
  DVMVS_REQUIRE(min_depth > 0.f && max_depth > min_depth, "plane_sweep: bad depth range");
  SweepParams p;
  p.ref = ref;
  for (int m = 0; m < M; ++m) {
    DVMVS_REQUIRE(meas_host[m] && pose2_host[m], "plane_sweep: null measurement pointer %d", m);
    p.meas[m] = meas_host[m];
    p.pose2[m] = pose2_host[m];
  }
  p.pose1 = pose1;
  p.K = K;
  p.out = cost_out;
  p.B = B; p.C = C; p.h = h; p.w = w; p.D = D; p.M = M;
  p.inv_base = 1.0 / (double)max_depth;                                   // utils.py:59-60
  p.inv_step = (1.0 / (double)min_depth - 1.0 / (double)max_depth) / (double)(D - 1);
  p.mode = mode;
  // off by default: the extra LSU traffic of phase A was measured to cost more than the hits save; kept behind
  // DVMVS_SWEEP_PREFETCH=1 as an experiment switch
  static const int prefetch_env = []() { const char* e = getenv("DVMVS_SWEEP_PREFETCH"); return e ? atoi(e) : 0; }();
  p.prefetch = prefetch_env;
  cudaStream_t s = (cudaStream_t)stream;
  const bool aligned = ((uintptr_t)ref % 16 == 0);
  bool fast = (C == 32) && aligned && ((size_t)B * h * w * 128 < ((size_t)1 << 32));   // 32-bit tap byte offsets
  for (int m = 0; m < M && fast; ++m) fast = ((uintptr_t)meas_host[m] % 16 == 0);
  if (fast) {
    const int tiles = B * h * ((w + kPix - 1) / kPix);
    const size_t smem = (size_t)(kPix * 32 + M * D * 4 + kMaxMeas * 12 + kPix * D) * sizeof(float) + 2 * kGroup * kPix * sizeof(SweepTapParams);
    static PerDeviceOnce attr_set;
    if (attr_set.first()) {
      cudaFuncSetAttribute(plane_sweep_c32_kernel<DVMVS_SWEEP_DOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
      cudaFuncSetAttribute(plane_sweep_c32_kernel<DVMVS_SWEEP_SAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    }
    DVMVS_REQUIRE(smem <= 96 * 1024, "plane_sweep: shared memory %zu too large", smem);
    // DVMVS_SWEEP_CTAS_PER_SM=n (1..3) pads the dynamic shared memory so that at most n CTAs of this kernel share an SM
    // (default: 4, the register limit) -- leaves room for other streams' kernels in pipelined engines (experiment switch)
    static const int occ_limit = []() { const char* e = getenv("DVMVS_SWEEP_CTAS_PER_SM"); return e ? atoi(e) : 0; }();
    size_t smem_launch = smem;
    if (occ_limit >= 1 && occ_limit <= 3) {
      const size_t want = (size_t)(227 * 1024) / (occ_limit + 1) + 1024;      // occ_limit + 1 CTAs no longer fit
      if (want > smem_launch && want <= 96 * 1024) smem_launch = want;
      else if (want > 96 * 1024) smem_launch = 96 * 1024;
    }
    static const int minb = []() { const char* e = getenv("DVMVS_SWEEP_MINB"); return e ? atoi(e) : 4; }();
    if (mode == DVMVS_SWEEP_DOT && (minb == 2 || minb == 3)) {
      static PerDeviceOnce attr2;
      if (attr2.first()) {
        cudaFuncSetAttribute(plane_sweep_c32_kernel<DVMVS_SWEEP_DOT, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
        cudaFuncSetAttribute(plane_sweep_c32_kernel<DVMVS_SWEEP_DOT, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
      }
      if (minb == 2) launch_k(plane_sweep_c32_kernel<DVMVS_SWEEP_DOT, 2>, dim3(tiles), dim3(kSweepThreads), smem_launch, s, p);
      else launch_k(plane_sweep_c32_kernel<DVMVS_SWEEP_DOT, 3>, dim3(tiles), dim3(kSweepThreads), smem_launch, s, p);
    } else if (mode == DVMVS_SWEEP_DOT)
      launch_k(plane_sweep_c32_kernel<DVMVS_SWEEP_DOT>, dim3(tiles), dim3(kSweepThreads), smem_launch, s, p);
    else
      launch_k(plane_sweep_c32_kernel<DVMVS_SWEEP_SAD>, dim3(tiles), dim3(kSweepThreads), smem_launch, s, p);
    return check_launch("plane_sweep_c32_kernel");
  }
  const size_t total = (size_t)B * h * w * D;
  launch_k(plane_sweep_generic_kernel, dim3((unsigned)((total + 127) / 128)), dim3(128), 0, s, p);
  return check_launch("plane_sweep_generic_kernel");
}

// EXPERIMENTAL (see plane_sweep_c32_h16_kernel): reference features fp32 [B][h][w][32], measurement features FP16 [B][h][w][32]
// (the "hi" plane a tensor-core convolution emits), dot-product cost only.
extern "C" int dvmvs_plane_sweep_fused_h16(const float* ref, const void* const* meas_h16_host, const float* pose1,
                                           const float* const* pose2_host, const float* K, float* cost_out, int B, int C, int h, int w,
                                           int D, int M, float min_depth, float max_depth, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(ref && meas_h16_host && pose1 && pose2_host && K && cost_out, "plane_sweep_h16: null pointer");
  DVMVS_REQUIRE(B > 0 && C == 32 && h > 1 && w > 1, "plane_sweep_h16: bad shape B=%d C=%d h=%d w=%d (C must be 32)", B, C, h, w);
  DVMVS_REQUIRE(D >= 2 && D <= kMaxPlanes, "plane_sweep_h16: D=%d outside [2,%d]", D, kMaxPlanes);
  DVMVS_REQUIRE(M >= 1 && M <= kMaxMeas, "plane_sweep_h16: M=%d outside [1,%d]", M, kMaxMeas);
  DVMVS_REQUIRE(min_depth > 0.f && max_depth > min_depth, "plane_sweep_h16: bad depth range");
  DVMVS_REQUIRE((size_t)B * h * w * 64 < ((size_t)1 << 32), "plane_sweep_h16: feature tensor too large for 32-bit offsets");
  DVMVS_REQUIRE((uintptr_t)ref % 16 == 0, "plane_sweep_h16: pointers must be 16-byte aligned");
  SweepParams p;
  p.ref = ref;
  for (int m = 0; m < M; ++m) {
    DVMVS_REQUIRE(meas_h16_host[m] && pose2_host[m] && (uintptr_t)meas_h16_host[m] % 16 == 0, "plane_sweep_h16: bad measurement pointer %d", m);
    p.meas[m] = reinterpret_cast<const float*>(meas_h16_host[m]);
    p.pose2[m] = pose2_host[m];
  }
  p.pose1 = pose1; p.K = K; p.out = cost_out;
  p.B = B; p.C = C; p.h = h; p.w = w; p.D = D; p.M = M;
  p.inv_base = 1.0 / (double)max_depth;
  p.inv_step = (1.0 / (double)min_depth - 1.0 / (double)max_depth) / (double)(D - 1);
  p.mode = DVMVS_SWEEP_DOT;
  p.prefetch = 0;
  const int tiles = B * h * ((w + kPix - 1) / kPix);
  const size_t smem = (size_t)(kPix * 32 + M * D * 4 + kMaxMeas * 12 + kPix * D) * sizeof(float) + 2 * kGroup * kPix * sizeof(SweepPairParams);
  static PerDeviceOnce attr_set;
  if (attr_set.first()) {
    cudaFuncSetAttribute(plane_sweep_c32_h16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
  }
  DVMVS_REQUIRE(smem <= 96 * 1024, "plane_sweep_h16: shared memory %zu too large", smem);
  launch_k(plane_sweep_c32_h16_kernel, dim3(tiles), dim3(kSweepThreads), smem, (cudaStream_t)stream, p);
  return check_launch("plane_sweep_c32_h16_kernel");
}

// ---- backward entry points (row f3) -------------------------------------------------------------------------------
extern "C" int dvmvs_plane_sweep_backward(const float* ref, const float* const* meas_host, const float* pose1,
                                          const float* const* pose2_host, const float* K, const float* grad_cost, float* grad_ref,
                                          float* const* grad_meas_host, int B, int C, int h, int w, int D, int M, float min_depth,
                                          float max_depth, int mode, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(ref && meas_host && pose1 && pose2_host && K && grad_cost && grad_ref && grad_meas_host, "plane_sweep_backward: null pointer");
  DVMVS_REQUIRE(B > 0 && h > 1 && w > 1, "plane_sweep_backward: bad shape B=%d h=%d w=%d", B, h, w);
  DVMVS_REQUIRE(C == 32, "plane_sweep_backward: C=%d (the training path sweeps the 32-channel half-resolution features)", C);
  DVMVS_REQUIRE(mode == DVMVS_SWEEP_DOT, "plane_sweep_backward: only the dot-product cost is differentiable here (mode %d)", mode);
  DVMVS_REQUIRE(D >= 2 && D <= kMaxPlanes, "plane_sweep_backward: D=%d outside [2,%d]", D, kMaxPlanes);
  DVMVS_REQUIRE(M >= 1 && M <= kMaxMeas, "plane_sweep_backward: M=%d outside [1,%d]", M, kMaxMeas);
  DVMVS_REQUIRE(min_depth > 0.f && max_depth > min_depth, "plane_sweep_backward: bad depth range");
  DVMVS_REQUIRE((size_t)B * h * w * 128 < ((size_t)1 << 32), "plane_sweep_backward: feature tensor too large for 32-bit tap offsets");
  SweepBwdParams q;
  SweepParams& p = q.f;
  p.ref = ref;
  DVMVS_REQUIRE((uintptr_t)ref % 16 == 0 && (uintptr_t)grad_ref % 16 == 0, "plane_sweep_backward: pointers must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  for (int m = 0; m < M; ++m) {
    DVMVS_REQUIRE(meas_host[m] && pose2_host[m] && grad_meas_host[m], "plane_sweep_backward: null measurement pointer %d", m);
    DVMVS_REQUIRE((uintptr_t)meas_host[m] % 16 == 0 && (uintptr_t)grad_meas_host[m] % 16 == 0, "plane_sweep_backward: pointers must be 16-byte aligned");
    p.meas[m] = meas_host[m];
    p.pose2[m] = pose2_host[m];
    q.gmeas[m] = grad_meas_host[m];
  }
  p.pose1 = pose1;
  p.K = K;
  p.out = nullptr;
  p.B = B; p.C = C; p.h = h; p.w = w; p.D = D; p.M = M;
  p.inv_base = 1.0 / (double)max_depth;
  p.inv_step = (1.0 / (double)min_depth - 1.0 / (double)max_depth) / (double)(D - 1);
  p.mode = mode;
  p.prefetch = 0;
  q.gcost = grad_cost;
  q.gref = grad_ref;
  // the same measurement tensor may appear more than once in grad_meas_host (aliased gradients accumulate); zero each once
  for (int m = 0; m < M; ++m) {
    bool seen = false;
    for (int j = 0; j < m; ++j) seen = seen || grad_meas_host[j] == grad_meas_host[m];
    if (!seen && cudaMemsetAsync(grad_meas_host[m], 0, (size_t)B * h * w * 32 * sizeof(float), s) != cudaSuccess) {
      set_error("plane_sweep_backward: memset failed");
      return DVMVS_ELAUNCH;
    }
  }
  const int tiles = B * h * ((w + kPix - 1) / kPix);
  const size_t smem = (size_t)(kPix * 32 + M * D * 4 + kMaxMeas * 12 + kPix * D) * sizeof(float) + kGroup * kPix * sizeof(SweepTapParams);
  static PerDeviceOnce attr_set;
  if (attr_set.first()) {
    cudaFuncSetAttribute(plane_sweep_backward_c32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
  }
  DVMVS_REQUIRE(smem <= 96 * 1024, "plane_sweep_backward: shared memory %zu too large", smem);
  launch_k(plane_sweep_backward_c32_kernel, dim3(tiles), dim3(kSweepThreads), smem, s, q);
  return check_launch("plane_sweep_backward_c32_kernel");
}

extern "C" int dvmvs_hidden_warp_backward(const float* grad_out, const float* depth, const float* prev_pose, const float* cur_pose,
                                          const float* K, float* grad_h_in, int B, int C, int h, int w, float invalid_thresh,
                                          dvmvs_stream_t stream) {
  DVMVS_REQUIRE(grad_out && depth && cur_pose && K && grad_h_in, "hidden_warp_backward: null pointer");
  DVMVS_REQUIRE(B > 0 && C > 0 && C % 4 == 0 && h > 1 && w > 1, "hidden_warp_backward: bad shape (C must be a multiple of 4)");
  // float4 loads of grad_out, red.global.add.v4.f32 into grad_h_in
  DVMVS_REQUIRE((uintptr_t)grad_out % 16 == 0 && (uintptr_t)grad_h_in % 16 == 0, "hidden_warp_backward: grad_out and grad_h_in must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemsetAsync(grad_h_in, 0, (size_t)B * h * w * C * sizeof(float), s) != cudaSuccess) {
    set_error("hidden_warp_backward: memset failed");
    return DVMVS_ELAUNCH;
  }
  const int total = h * w * (C / 4);
  launch_k(hidden_warp_backward_kernel, dim3((total + 127) / 128, B), dim3(128), 0, s, grad_out, depth, prev_pose, cur_pose, K, grad_h_in, B, C,
           h, w, invalid_thresh);
  return check_launch("hidden_warp_backward_kernel");
}

// test hook: force the generic path (used by tests to cross-check the fast path on the device)
extern "C" int dvmvs_plane_sweep_generic(const float* ref, const float* const* meas_host, const float* pose1,
                                         const float* const* pose2_host, const float* K, float* cost_out, int B, int C,
                                         int h, int w, int D, int M, float min_depth, float max_depth, int mode,
                                         dvmvs_stream_t stream) {
  DVMVS_REQUIRE(ref && meas_host && pose1 && pose2_host && K && cost_out, "plane_sweep: null pointer");
  DVMVS_REQUIRE(M >= 1 && M <= kMaxMeas && D >= 2, "plane_sweep: bad M/D");
  SweepParams p;
  p.ref = ref;
  for (int m = 0; m < M; ++m) { p.meas[m] = meas_host[m]; p.pose2[m] = pose2_host[m]; }
  p.pose1 = pose1; p.K = K; p.out = cost_out;
  p.B = B; p.C = C; p.h = h; p.w = w; p.D = D; p.M = M;
  p.inv_base = 1.0 / (double)max_depth;
  p.inv_step = (1.0 / (double)min_depth - 1.0 / (double)max_depth) / (double)(D - 1);
  p.mode = mode;
  p.prefetch = 0;
  const size_t total = (size_t)B * h * w * D;
  launch_k(plane_sweep_generic_kernel, dim3((unsigned)((total + 127) / 128)), dim3(128), 0, (cudaStream_t)stream, p);
  return check_launch("plane_sweep_generic_kernel");
}

extern "C" int dvmvs_hidden_warp(const float* h_in, const float* depth, const float* prev_pose, const float* cur_pose,
                                 const float* K, float* h_out, int B, int C, int h, int w, float invalid_thresh,
                                 dvmvs_stream_t stream) {
  DVMVS_REQUIRE(h_in && depth && cur_pose && K && h_out, "hidden_warp: null pointer");
  DVMVS_REQUIRE(B > 0 && C > 0 && C % 4 == 0 && h > 1 && w > 1, "hidden_warp: bad shape B=%d C=%d h=%d w=%d", B, C, h, w);
  DVMVS_REQUIRE((uintptr_t)h_in % 16 == 0 && (uintptr_t)h_out % 16 == 0, "hidden_warp: pointers must be 16-byte aligned");
  const int n = h * w * (C / 4);
  dim3 grid((n + 127) / 128, B);
  launch_k(hidden_warp_kernel, grid, dim3(128), 0, (cudaStream_t)stream, h_in, depth, prev_pose, cur_pose, K, h_out, B, C, h, w, invalid_thresh);
  return check_launch("hidden_warp_kernel");
}

extern "C" int dvmvs_depth_reproject(const float* cur_pose, const float* prev_pose, const float* prev_depth,
                                     const float* full_K, const float* half_K, float* out, int B, int H, int W,
                                     dvmvs_stream_t stream) {
  DVMVS_REQUIRE(cur_pose && prev_pose && prev_depth && full_K && half_K && out, "depth_reproject: null pointer");
  DVMVS_REQUIRE(B > 0 && H >= 2 && W >= 2, "depth_reproject: bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(out, 0, (size_t)B * (H / 2) * (W / 2) * sizeof(float), s);
  if (e != cudaSuccess) { set_error("depth_reproject memset: %s", cudaGetErrorString(e)); return DVMVS_ELAUNCH; }
  dim3 grid((H * W + 255) / 256, B);
  launch_k(depth_reproject_kernel, grid, dim3(256), 0, s, cur_pose, prev_pose, prev_depth, full_K, half_K, (unsigned int*)out, B, H, W);
  return check_launch("depth_reproject_kernel");
}
