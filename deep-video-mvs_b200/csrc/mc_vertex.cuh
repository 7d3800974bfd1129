// The per-edge arithmetic of marching cubes (contract in mesh.cu's header), shared by the dense mesh (mesh.cu) and the mesh of
// the voxel-block volume (tsdf_sparse_view.cu).  Parameterised on how a voxel is fetched, so both produce the same bits for the
// same voxel values: t, the index-space vertex, the world point, the np.gradient normal and the colour.
#pragma once

#include "color_fold.cuh"
#include "common.cuh"

namespace dvmvs {

__device__ __forceinline__ bool mc_inside(float v) { return v < 0.f; }   // NaN is never inside

// np.gradient of the volume at voxel q (box-relative), float32: (f[i+1] - f[i-1]) / 2 inside, f[1] - f[0] and
// f[n-1] - f[n-2] at the box border (every dimension is >= 2 here).  at(a, s) = tsdf of q's neighbour s in {-1, 0, 1} along a.
template <typename At>
__device__ __forceinline__ void mc_np_gradient(const int* q, const int* dim, At at, float* gr) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (q[a] == 0) gr[a] = __fsub_rn(at(a, 1), at(a, 0));
    else if (q[a] == dim[a] - 1) gr[a] = __fsub_rn(at(a, 0), at(a, -1));
    else gr[a] = __fdiv_rn(__fsub_rn(at(a, 1), at(a, -1)), 2.f);
  }
}

// The vertex on the +axis grid edge of voxel q (box-relative): a, b = tsdf at the edge's endpoints, grad(i, j, k, g) =
// np.gradient at box index (i, j, k), color_at(i, j, k) = the colour voxel there.  Returns the world point, the unit normal and
// uint8 RGB.
struct McVertex {
  float vert[3], norm[3];
  unsigned char rgb[3];
};

template <typename Grad, typename ColorAt>
__device__ __forceinline__ McVertex mc_vertex(float a, float b, const int* q, int axis, Grad grad, ColorAt color_at, const float* origin,
                                              float voxel) {
  const float t = __fdiv_rn(-a, __fsub_rn(b, a));
  float vi[3] = {(float)q[0], (float)q[1], (float)q[2]};
  vi[axis] = __fadd_rn(vi[axis], t);
  float ga[3], gb[3], nrm[3];
  grad(q[0], q[1], q[2], ga);
  grad(q[0] + (axis == 0), q[1] + (axis == 1), q[2] + (axis == 2), gb);
#pragma unroll
  for (int c = 0; c < 3; ++c) nrm[c] = __fadd_rn(ga[c], __fmul_rn(t, __fsub_rn(gb[c], ga[c])));
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nrm[0], nrm[0]), __fmul_rn(nrm[1], nrm[1])), __fmul_rn(nrm[2], nrm[2])));
  const int ix = (int)rintf(vi[0]), iy = (int)rintf(vi[1]), iz = (int)rintf(vi[2]);
  float cb, cg, cr;
  unfold(color_at(ix, iy, iz), cb, cg, cr);
  const float col[3] = {cr, cg, cb};
  McVertex m;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    m.vert[c] = __fadd_rn(__fmul_rn(vi[c], voxel), origin[c]);
    m.norm[c] = len > 0.f ? __fdiv_rn(nrm[c], len) : 0.f;
    m.rgb[c] = (unsigned char)__float2int_rz(floorf(col[c]));           // numpy's float -> uint8 cast (truncation)
  }
  return m;
}

}  // namespace dvmvs
