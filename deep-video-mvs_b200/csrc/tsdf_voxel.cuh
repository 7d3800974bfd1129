// The per-voxel arithmetic of TSDF integration, shared by the dense volume (tsdf.cu) and the voxel-block volume
// (tsdf_sparse.cu): both update a voxel through tsdf_update_voxel, so both follow the reference's CPU path bit for bit
// (tsdf.cu's header states the operation order).
#pragma once
#include <math.h>

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

}  // namespace dvmvs
