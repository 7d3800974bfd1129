// The ray-march arithmetic of TSDF ray casting (contract in raycast.cu's header), shared by the dense volume (raycast.cu) and
// the voxel-block volume (tsdf_sparse_view.cu).  Parameterised on how the 8 corners of a cell are fetched, so both march the
// same lattice, take the same skips and produce the same bits for the same voxel values.
#pragma once

#include "color_fold.cuh"
#include "common.cuh"

namespace dvmvs {

constexpr float kRayMaxSamples = 1073741824.f;     // 2^30: lattices longer than this (only degenerate poses) give no hits

// the skip length in lattice samples: trunc - (sqrt(3) / 2) voxel is the least distance to the surface of any point in a cell
// whose corners are all truncated
inline int rc_n_skip(double trunc_margin, double voxel_size) {
  const double n_skip = floor((trunc_margin / voxel_size - 0.8660254037844386) / 0.5);
  return (int)fmin(fmax(n_skip, 1.0), (double)(1 << 24));
}

__device__ __forceinline__ float rc_lerp(float a, float b, float f) { return __fadd_rn(a, __fmul_rn(f, __fsub_rn(b, a))); }

struct RayCell {
  float c[8];                      // corner (i, j, k) at c[i + 2 j + 4 k]
  float f[3];
};

// one ray in grid index space: origin o, direction d, the lattice z_k = z_near + f32(k) * dz for k = 0 .. n; ok = false: no hit
struct Ray {
  float o[3], d[3];
  float dz, z_near;
  int n;
  bool ok;
};

// the ray of pixel (u, v) of a view (fx fy cx cy, R row-major camera -> world, t) through the box [0, dim - 1]^3
__device__ __forceinline__ Ray rc_ray(const float* vw, int u, int v, const int* dim, const float* origin, float voxel) {
  Ray r;
  const float dcx = __fdiv_rn(__fsub_rn((float)u, vw[2]), vw[0]);
  const float dcy = __fdiv_rn(__fsub_rn((float)v, vw[3]), vw[1]);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float w = __fadd_rn(__fadd_rn(__fmul_rn(vw[4 + 3 * a], dcx), __fmul_rn(vw[5 + 3 * a], dcy)), vw[6 + 3 * a]);
    r.d[a] = __fdiv_rn(w, voxel);
    r.o[a] = __fdiv_rn(__fsub_rn(vw[13 + a], origin[a]), voxel);
  }
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(r.d[0], r.d[0]), __fmul_rn(r.d[1], r.d[1])), __fmul_rn(r.d[2], r.d[2])));
  r.dz = __fdiv_rn(0.5f, len);
  bool inside_box = dim[0] >= 2 && dim[1] >= 2 && dim[2] >= 2;
  float z_near = 0.f, z_far = INFINITY;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float hi = (float)(dim[a] - 1);
    if (r.d[a] == 0.f) {
      inside_box = inside_box && r.o[a] >= 0.f && r.o[a] <= hi;
    } else {
      const float t0 = __fdiv_rn(-r.o[a], r.d[a]), t1 = __fdiv_rn(__fsub_rn(hi, r.o[a]), r.d[a]);
      z_near = fmaxf(z_near, fminf(t0, t1));
      z_far = fminf(z_far, fmaxf(t0, t1));
    }
  }
  const float n_f = floorf(__fdiv_rn(__fsub_rn(z_far, z_near), r.dz));
  r.z_near = z_near;
  r.ok = inside_box && z_near <= z_far && n_f < kRayMaxSamples;     // false for NaN (a degenerate pose)
  r.n = r.ok ? (int)n_f : 0;
  return r;
}

// the cell and fractions of the point o + z d (clamped into the box); corners(ci, c) fetches the tsdf at the cell's corners
template <typename Corners>
__device__ __forceinline__ void rc_cell(const int* dim, const float* o, const float* d, float z, Corners corners, RayCell& cell) {
  int ci[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float g = fminf(fmaxf(__fadd_rn(o[a], __fmul_rn(z, d[a])), 0.f), (float)(dim[a] - 1));
    ci[a] = min((int)floorf(g), dim[a] - 2);
    cell.f[a] = __fsub_rn(g, (float)ci[a]);
  }
  corners(ci, cell.c);
}

__device__ __forceinline__ float rc_trilinear(const RayCell& s) {
  const float x00 = rc_lerp(s.c[0], s.c[1], s.f[0]), x10 = rc_lerp(s.c[2], s.c[3], s.f[0]);
  const float x01 = rc_lerp(s.c[4], s.c[5], s.f[0]), x11 = rc_lerp(s.c[6], s.c[7], s.f[0]);
  return rc_lerp(rc_lerp(x00, x10, s.f[1]), rc_lerp(x01, x11, s.f[1]), s.f[2]);
}

__device__ __forceinline__ bool rc_all_ones(const RayCell& s) {
  bool ones = true;
#pragma unroll
  for (int c = 0; c < 8; ++c) ones = ones && s.c[c] == 1.f;
  return ones;
}

// F at lattice sample k; *ones = the sample's cell is fully truncated
template <typename Corners>
__device__ __forceinline__ float rc_sample(const int* dim, const Ray& r, int k, Corners corners, bool* ones) {
  RayCell s;
  rc_cell(dim, r.o, r.d, __fadd_rn(r.z_near, __fmul_rn((float)k, r.dz)), corners, s);
  *ones = rc_all_ones(s);
  return rc_trilinear(s);
}

// the march: the first + -> - crossing with the n_skip rule; returns whether it hit and its depth in *z_hit
template <typename Corners>
__device__ __forceinline__ bool rc_march(const int* dim, const Ray& r, int n_skip, Corners corners, float* z_hit) {
  if (!r.ok) return false;
  const int n = r.n;
  bool ones;
  float f_prev = rc_sample(dim, r, 0, corners, &ones);
  int k = 0;
  while (k < n) {
    if (ones && k + n_skip <= n) {
      bool ones_j;
      const float f_j = rc_sample(dim, r, k + n_skip, corners, &ones_j);
      if (!(f_j < 0.f)) {
        k += n_skip;
        f_prev = f_j;
        ones = ones_j;
        continue;
      }
    }
    const float f_cur = rc_sample(dim, r, k + 1, corners, &ones);
    if (f_prev >= 0.f && f_cur < 0.f) {
      const float z_prev = __fadd_rn(r.z_near, __fmul_rn((float)k, r.dz));
      *z_hit = __fadd_rn(z_prev, __fdiv_rn(__fmul_rn(r.dz, f_prev), __fsub_rn(f_prev, f_cur)));
      return true;
    }
    f_prev = f_cur;
    ++k;
  }
  return false;
}

// the unit normal at the hit: the analytic gradient of the trilinear interpolant in the hit's cell
__device__ __forceinline__ void rc_normal(const RayCell& s, float* nrm) {
  const float* c = s.c;
  const float* f = s.f;
  // x differences over (y, z), y differences over (x, z), z differences over (x, y)
  const float gx = rc_lerp(rc_lerp(__fsub_rn(c[1], c[0]), __fsub_rn(c[3], c[2]), f[1]), rc_lerp(__fsub_rn(c[5], c[4]), __fsub_rn(c[7], c[6]), f[1]), f[2]);
  const float gy = rc_lerp(rc_lerp(__fsub_rn(c[2], c[0]), __fsub_rn(c[3], c[1]), f[0]), rc_lerp(__fsub_rn(c[6], c[4]), __fsub_rn(c[7], c[5]), f[0]), f[2]);
  const float gz = rc_lerp(rc_lerp(__fsub_rn(c[4], c[0]), __fsub_rn(c[5], c[1]), f[0]), rc_lerp(__fsub_rn(c[6], c[2]), __fsub_rn(c[7], c[3]), f[0]), f[1]);
  const float glen = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz)));
  if (glen > 0.f) {
    nrm[0] = __fdiv_rn(gx, glen);
    nrm[1] = __fdiv_rn(gy, glen);
    nrm[2] = __fdiv_rn(gz, glen);
  }
}

// the box index of the colour voxel at the hit: rint(g(z*)) (half-even)
__device__ __forceinline__ void rc_color_voxel(const int* dim, const Ray& r, float z_hit, int* vi) {
#pragma unroll
  for (int a = 0; a < 3; ++a) vi[a] = (int)rintf(fminf(fmaxf(__fadd_rn(r.o[a], __fmul_rn(z_hit, r.d[a])), 0.f), (float)(dim[a] - 1)));
}

// the reference's unfold of a colour voxel, as uint8 RGB (numpy's float -> uint8 cast: truncation)
__device__ __forceinline__ void rc_rgb(float folded, unsigned char* rgb) {
  float cb, cg, cr;
  unfold(folded, cb, cg, cr);
  rgb[0] = (unsigned char)__float2int_rz(floorf(cr));
  rgb[1] = (unsigned char)__float2int_rz(floorf(cg));
  rgb[2] = (unsigned char)__float2int_rz(floorf(cb));
}

}  // namespace dvmvs
