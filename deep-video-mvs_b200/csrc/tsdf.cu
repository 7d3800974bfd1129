// TSDF integration of one posed RGB-D frame into a voxel volume -- SURVEY.md section 8 row f4, the consumer of the depth
// maps this library predicts: `TSDFVolume.integrate` of the reference's sample-data/run-tsdf-reconstruction.py:220-323.
// The reference has two implementations, an inline pycuda kernel in float32 (:80-152) and a numba / numpy CPU path in mixed
// float32 / float64 (:181-218, :283-323) that it falls back to wherever pycuda is absent (the case in this image).  This
// kernel follows the CPU path operation by operation, in the precision each operation has there, so its volumes equal the
// reference's bit for bit (tests/test_tsdf.py against goldens of the unmodified script):
//   world  = f32( f64(origin) + voxel_size * f64(coord) )                                     vox2world
//   cam    = inv(cam_pose) * [world 1] in f64; per row an FMA chain in k order starting from the rounded first product --
//            what the 4 x N double GEMM of np.dot evaluates                                   rigid_transform
//   pixel  = rint( X * f64(fx) / Z + f64(cx) ) (half-even), valid iff inside the image and Z > 0    cam2pix
//   tsdf   = f32( ( f64( f32(w_old * tsdf_old) ) + obs * dist ) / f64(w_new) ),  w_new = f32( f64(w_old) + obs )
//   colour : float32 throughout, rintf, min(255, .) with NaN propagation as np.minimum
// No multiply-add contraction anywhere a rounding would be skipped (explicit _rn intrinsics).
//
// Culling: 98 % of a room-sized volume is outside the frustum or the truncation band of any one frame.  A thread owns a run of
// 8 consecutive z voxels and first projects the run's two END POINTS in float32 (9 FMAs each): the run is dropped when it is
// PROVABLY behind the camera or more than a pixel outside one image border -- the tests use error bounds of the float32
// evaluation computed on the host from the volume extent (eps), so a voxel the float64 path would update is never dropped
// (tests compare whole volumes with the reference bit for bit).  Voxels of surviving runs take the exact path.
// The per-voxel variant (one thread per voxel with a per-voxel pre-test) was instruction-issue bound.  What remains is the
// exact float64 projection (two double divisions) of the ~20 % of voxels inside the frustum, nine tenths of which then fail
// the truncation test; a conservative depth pre-test against a coarse max-depth image is the next step.
//
// Memory: volumes are the reference's C-order [x][y][z]; a thread's run is 32 contiguous bytes of each volume (one sector), a
// warp's runs are contiguous.  Voxels outside the frustum or the truncation band touch no volume memory at all.  Algorithmic
// bytes: 24 B per UPDATED voxel (tsdf, weight, colour: read + write fp32) + the frame (4 B depth + 3..12 B colour per pixel, L2
// resident).  The inverse pose, float32 intrinsics and trunc margin arrive by value in the launch parameters.
#include <math.h>
#include <stdlib.h>

#include "color_fold.cuh"
#include "common.cuh"

namespace dvmvs {

struct TsdfParams {
  float* tsdf;
  float* weight;
  float* color;
  const void* color_im;   // [h][w][3] RGB, uint8 or float32
  const void* depth_im;   // [h][w] float32 or float64
  int dim_x, dim_y, dim_z, im_h, im_w;
  float origin[3];
  double voxel_size, trunc, obs;
  double T[12];           // rows 0..2 of inv(cam_pose)
  double fx, fy, cx, cy;  // float32 intrinsics widened
  unsigned long long* updated;   // optional counter of updated voxels (nullptr = none)
  float Tf[12];           // float32 copy of T for the conservative pre-test
  float eps[3];           // bound on |float32 camera coordinate - float64 camera coordinate| per axis over the volume
  float fxf, fyf, lo_x, hi_x, lo_y, hi_y;   // lo = cx + 1.5, hi = im_w + 1.5 - cx (one pixel of margin on each side)
  int cull;
};

__device__ __forceinline__ float np_minimum(float a, float b) { return (a != a) ? a : ((b != b) ? b : (a < b ? a : b)); }
__device__ __forceinline__ double np_minimum(double a, double b) { return (a != a) ? a : ((b != b) ? b : (a < b ? a : b)); }

constexpr int kTsdfRun = 8;      // consecutive z voxels per thread: one frustum test covers the whole run

// float32 camera-space quantities of one world point for the conservative pre-test
struct CullEval {
  float Z, ux, uy, sx, sy;
};
__device__ __forceinline__ CullEval cull_eval(const TsdfParams& p, float wx, float wy, float wz) {
  CullEval e;
  const float X = fmaf(p.Tf[0], wx, fmaf(p.Tf[1], wy, fmaf(p.Tf[2], wz, p.Tf[3])));
  const float Y = fmaf(p.Tf[4], wx, fmaf(p.Tf[5], wy, fmaf(p.Tf[6], wz, p.Tf[7])));
  e.Z = fmaf(p.Tf[8], wx, fmaf(p.Tf[9], wy, fmaf(p.Tf[10], wz, p.Tf[11])));
  e.ux = X * p.fxf;
  e.uy = Y * p.fyf;
  const float bx = fabsf(p.lo_x) + fabsf(p.hi_x), by = fabsf(p.lo_y) + fabsf(p.hi_y);
  e.sx = p.fxf * p.eps[0] + bx * p.eps[2] + 1e-6f * (fabsf(e.ux) + bx * fabsf(e.Z));
  e.sy = p.fyf * p.eps[1] + by * p.eps[2] + 1e-6f * (fabsf(e.uy) + by * fabsf(e.Z));
  return e;
}

// the exact path for one voxel (mixed float32 / float64 as the reference's CPU path); returns whether the voxel was updated
template <typename ColorT, typename DepthT>
__device__ __forceinline__ bool tsdf_update_voxel(const TsdfParams& p, size_t idx, double wx, double wy, double wz) {
  const double cxp = __fma_rn(p.T[3], 1.0, __fma_rn(p.T[2], wz, __fma_rn(p.T[1], wy, __dmul_rn(p.T[0], wx))));
  const double cyp = __fma_rn(p.T[7], 1.0, __fma_rn(p.T[6], wz, __fma_rn(p.T[5], wy, __dmul_rn(p.T[4], wx))));
  const double czp = __fma_rn(p.T[11], 1.0, __fma_rn(p.T[10], wz, __fma_rn(p.T[9], wy, __dmul_rn(p.T[8], wx))));
  if (!(czp > 0.0)) return false;
  const double px = rint(__dadd_rn(__ddiv_rn(__dmul_rn(cxp, p.fx), czp), p.cx));
  const double py = rint(__dadd_rn(__ddiv_rn(__dmul_rn(cyp, p.fy), czp), p.cy));
  if (!(px >= 0.0 && px < (double)p.im_w && py >= 0.0 && py < (double)p.im_h)) return false;
  const size_t pix = (size_t)py * p.im_w + (size_t)px;
  const double depth = (double)((const DepthT*)p.depth_im)[pix];
  const double diff = __dsub_rn(depth, czp);
  if (!(depth > 0.0 && diff >= -p.trunc)) return false;
  const double dist = np_minimum(1.0, __ddiv_rn(diff, p.trunc));
  const float w_old = p.weight[idx], t_old = p.tsdf[idx], c_old = p.color[idx];
  const float w_new = __double2float_rn(__dadd_rn((double)w_old, p.obs));
  const double num = __dadd_rn((double)__fmul_rn(w_old, t_old), __dmul_rn(p.obs, dist));
  p.weight[idx] = w_new;
  p.tsdf[idx] = __double2float_rn(__ddiv_rn(num, (double)w_new));
  const ColorT* c = (const ColorT*)p.color_im + pix * 3;
  const float folded = floorf(__fadd_rn(__fadd_rn(__fmul_rn((float)c[2], 65536.f), __fmul_rn((float)c[1], 256.f)), (float)c[0]));
  float ob, og, orr, nb, ng, nr;
  unfold(c_old, ob, og, orr);
  unfold(folded, nb, ng, nr);
  const float ow = (float)p.obs;
  nb = np_minimum(255.f, rintf(__fdiv_rn(__fadd_rn(__fmul_rn(w_old, ob), __fmul_rn(ow, nb)), w_new)));
  ng = np_minimum(255.f, rintf(__fdiv_rn(__fadd_rn(__fmul_rn(w_old, og), __fmul_rn(ow, ng)), w_new)));
  nr = np_minimum(255.f, rintf(__fdiv_rn(__fadd_rn(__fmul_rn(w_old, orr), __fmul_rn(ow, nr)), w_new)));
  p.color[idx] = __fadd_rn(__fadd_rn(__fmul_rn(nb, 65536.f), __fmul_rn(ng, 256.f)), nr);
  return true;
}

// One thread per run of kTsdfRun consecutive z voxels of one (x, y) column.  Camera coordinates are affine along the run, so
// each frustum half-space test ("behind the camera", "left of the image by more than a pixel", ...) holds for the whole run
// iff it holds at both end points (slack = the larger of the end points' slacks: it is convex along the run).  The float32
// rounding of the in-between voxels' world coordinates (<= half an ulp off the segment) sits inside eps' 16x headroom.
template <typename ColorT, typename DepthT>
__global__ void __launch_bounds__(256) tsdf_integrate_kernel(TsdfParams p) {
  pdl_launch_dependents();
  const int runs_z = (p.dim_z + kTsdfRun - 1) / kTsdfRun;
  const long long total = (long long)p.dim_x * p.dim_y * runs_z;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int hits = 0;
  if (t < total) {
    long long col;
    int zr;
    if (total <= 0xffffffffLL) {       // 32-bit index arithmetic (64-bit division is emulated)
      const unsigned c32 = (unsigned)t / (unsigned)runs_z;
      zr = (int)((unsigned)t - c32 * (unsigned)runs_z);
      col = c32;
    } else {
      col = t / runs_z;
      zr = (int)(t - col * runs_z);
    }
    const int x = (int)(col / p.dim_y), y = (int)(col - (long long)x * p.dim_y);
    const int z0 = zr * kTsdfRun, z1 = min(z0 + kTsdfRun, p.dim_z) - 1;
    const float wxf = __double2float_rn(__dadd_rn((double)p.origin[0], __dmul_rn(p.voxel_size, (double)x)));
    const float wyf = __double2float_rn(__dadd_rn((double)p.origin[1], __dmul_rn(p.voxel_size, (double)y)));
    bool skip = false;
    if (p.cull) {
      const float wz0 = __double2float_rn(__dadd_rn((double)p.origin[2], __dmul_rn(p.voxel_size, (double)z0)));
      const float wz1 = __double2float_rn(__dadd_rn((double)p.origin[2], __dmul_rn(p.voxel_size, (double)z1)));
      const CullEval a = cull_eval(p, wxf, wyf, wz0), b = cull_eval(p, wxf, wyf, wz1);
      if (fmaxf(a.Z, b.Z) + p.eps[2] <= 0.f) {
        skip = true;                                                // the whole run is certainly behind the camera
      } else if (fminf(a.Z, b.Z) - p.eps[2] > 0.f) {                // certainly in front: image borders, with slack and a pixel to spare
        const float sx = fmaxf(a.sx, b.sx), sy = fmaxf(a.sy, b.sy);
        // pixel < -1.5  <=>  X fx + (cx + 1.5) Z < 0 ;   pixel > w + 0.5  <=>  X fx - (w + 1.5 - cx) Z > 0
        skip = fmaxf(a.ux + p.lo_x * a.Z, b.ux + p.lo_x * b.Z) < -sx || fminf(a.ux - p.hi_x * a.Z, b.ux - p.hi_x * b.Z) > sx ||
               fmaxf(a.uy + p.lo_y * a.Z, b.uy + p.lo_y * b.Z) < -sy || fminf(a.uy - p.hi_y * a.Z, b.uy - p.hi_y * b.Z) > sy;
      }
    }
    if (!skip) {
      pdl_wait();
      const double wx = (double)wxf, wy = (double)wyf;
      const size_t base = (size_t)col * p.dim_z;
      for (int z = z0; z <= z1; ++z) {
        const double wz = (double)__double2float_rn(__dadd_rn((double)p.origin[2], __dmul_rn(p.voxel_size, (double)z)));
        hits += tsdf_update_voxel<ColorT, DepthT>(p, base + z, wx, wy, wz) ? 1 : 0;
      }
    }
  }
  if (p.updated) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, o);
    if ((threadIdx.x & 31) == 0 && hits) atomicAdd(p.updated, (unsigned long long)hits);
  }
}

}  // namespace dvmvs

using namespace dvmvs;

extern "C" int dvmvs_tsdf_integrate(float* tsdf_vol, float* weight_vol, float* color_vol, int dim_x, int dim_y, int dim_z,
                                    const float* vol_origin3, double voxel_size, double trunc_margin, const void* color_im,
                                    int color_is_u8, const void* depth_im, int depth_is_f64, int im_h, int im_w,
                                    const float* intr4, const double* world_to_cam16, double obs_weight,
                                    unsigned long long* updated_count, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(tsdf_vol && weight_vol && color_vol && vol_origin3 && color_im && depth_im && intr4 && world_to_cam16, "tsdf_integrate: null argument");
  DVMVS_REQUIRE(dim_x > 0 && dim_y > 0 && dim_z > 0 && im_h > 0 && im_w > 0, "tsdf_integrate: bad extent %d x %d x %d, image %d x %d", dim_x, dim_y, dim_z, im_h, im_w);
  const long long n = (long long)dim_x * dim_y * dim_z;
  DVMVS_REQUIRE((n + 255) / 256 <= 0x7fffffffLL, "tsdf_integrate: volume of %lld voxels exceeds one launch", n);
  TsdfParams p;
  p.tsdf = tsdf_vol; p.weight = weight_vol; p.color = color_vol;
  p.color_im = color_im; p.depth_im = depth_im;
  p.dim_x = dim_x; p.dim_y = dim_y; p.dim_z = dim_z; p.im_h = im_h; p.im_w = im_w;
  for (int i = 0; i < 3; ++i) p.origin[i] = vol_origin3[i];
  p.voxel_size = voxel_size; p.trunc = trunc_margin; p.obs = obs_weight;
  for (int i = 0; i < 12; ++i) p.T[i] = world_to_cam16[i];
  p.fx = (double)intr4[0]; p.fy = (double)intr4[1]; p.cx = (double)intr4[2]; p.cy = (double)intr4[3];
  p.updated = updated_count;
  // conservative float32 pre-test: per camera axis r, |fl32 evaluation - exact| <= 2^-20 * (sum_k |T[r][k]| max|w_k| + |T[r][3]|)
  // (four roundings of 2^-24 each on the products / sums, plus 2^-24 relative on each float32 copy of T: 16x headroom)
  double maxabs[3];
  const int dims[3] = {dim_x, dim_y, dim_z};
  for (int k = 0; k < 3; ++k) {
    const double a = fabs((double)vol_origin3[k]), b = fabs((double)vol_origin3[k] + voxel_size * (double)dims[k]);
    maxabs[k] = a > b ? a : b;
  }
  bool finite = true;
  for (int r = 0; r < 3; ++r) {
    double sum = fabs(p.T[4 * r + 3]);
    for (int k = 0; k < 3; ++k) sum += fabs(p.T[4 * r + k]) * maxabs[k];
    p.eps[r] = (float)(sum * 9.5367431640625e-07) + 1e-30f;
    for (int k = 0; k < 4; ++k) {
      p.Tf[4 * r + k] = (float)p.T[4 * r + k];
      finite = finite && isfinite(p.Tf[4 * r + k]);
    }
    finite = finite && isfinite(p.eps[r]);
  }
  p.fxf = fabsf(intr4[0]); p.fyf = fabsf(intr4[1]);
  p.lo_x = intr4[2] + 1.5f; p.hi_x = (float)im_w + 1.5f - intr4[2];
  p.lo_y = intr4[3] + 1.5f; p.hi_y = (float)im_h + 1.5f - intr4[3];
  // the border inequalities assume positive focal lengths; anything unusual (negative / non-finite) takes the exact path only
  static const bool cull_env = []() { const char* e = getenv("DVMVS_TSDF_CULL"); return !(e && e[0] == '0'); }();
  p.cull = (cull_env && finite && intr4[0] > 0.f && intr4[1] > 0.f && isfinite(intr4[2]) && isfinite(intr4[3])) ? 1 : 0;
  const long long n_threads = (long long)dim_x * dim_y * ((dim_z + kTsdfRun - 1) / kTsdfRun);
  const dim3 grid((unsigned)((n_threads + 255) / 256)), block(256);
  cudaStream_t s = (cudaStream_t)stream;
  if (color_is_u8) {
    if (depth_is_f64) launch_k(tsdf_integrate_kernel<unsigned char, double>, grid, block, 0, s, p);
    else launch_k(tsdf_integrate_kernel<unsigned char, float>, grid, block, 0, s, p);
  } else {
    if (depth_is_f64) launch_k(tsdf_integrate_kernel<float, double>, grid, block, 0, s, p);
    else launch_k(tsdf_integrate_kernel<float, float>, grid, block, 0, s, p);
  }
  return check_launch("tsdf_integrate_kernel");
}
