// Ray casting of the TSDF volume: depth, normal and colour maps of the fused model at given camera poses (TSDFVolume.render).
// No reference counterpart: the reference's volume has only the mesh as a way out.  oracle/raycast_oracle.py restates this file
// in numpy and tests/test_raycast.py compares with array_equal.  Everything that rounds is an explicit float32 _rn intrinsic (no
// multiply-add contraction).  Per view: fx fy cx cy, R (row-major, camera -> world, as TSDFVolume.integrate's pose), t.  Per
// pixel (u, v) of a view, in this order:
//   dc      = ((u - cx) / fx, (v - cy) / fy, 1)
//   w_a     = (R[a][0] * dc_x + R[a][1] * dc_y) + R[a][2]                       (R . dc, world frame)
//   d_a     = w_a / voxel;   o_a = (t_a - origin_a) / voxel                     (grid index space: voxel i sits at i)
//   |d|     = sqrt((d_x d_x + d_y d_y) + d_z d_z);   dz = 0.5 / |d|              (half a voxel of world length, in camera depth)
//   range   slabs of [0, dim - 1]^3: an axis with d_a = 0 admits the whole ray iff 0 <= o_a <= dim_a - 1, else
//           n_a = -o_a / d_a, f_a = (dim_a - 1 - o_a) / d_a, near_a = fminf(n_a, f_a), far_a = fmaxf(n_a, f_a);
//           z_near = fmaxf(fmaxf(fmaxf(0, near_x), near_y), near_z), z_far = fminf(fminf(far_x, far_y), far_z)
//           (axes without a slab skipped); no hit unless z_near <= z_far.  A volume with a dimension < 2 gives no hits.
//   lattice n = floor((z_far - z_near) / dz), no hit unless n < 2^30;   z_k = z_near + f32(k) * dz,  k = 0 .. n
//   sample  g_a = min(max(o_a + z_k * d_a, 0), dim_a - 1);  cell_a = min(floor(g_a), dim_a - 2);  f_a = g_a - cell_a
//           F = trilinear of the raw tsdf at the cell's 8 corners: lerps along x, then y, then z, lerp(a, b, f) = a + f (b - a)
//   hit     the first k >= 1 with F_{k-1} >= 0 and F_k < 0 (a NaN is never inside); z* = z_{k-1} + (dz F_{k-1}) / (F_{k-1} - F_k).
//           Back faces (- -> +) are marched through.
//   skip    at sample k whose cell's 8 corners are all exactly 1.0, the march moves to k + n_skip instead of k + 1 when
//           k + n_skip <= n and F_{k + n_skip} is not < 0.  n_skip = max(1, floor((trunc / voxel - sqrt(3) / 2) / 0.5)) on the
//           host (8 at trunc = 5 voxel).  A jump never lands inside, so every crossing stays between adjacent lattice samples;
//           for a Euclidean truncated SDF the skipped span holds no inside sample, and the result equals the march without it.
//   outputs depth z* (0 = no hit).  Normal: the analytic gradient of the trilinear interpolant in the cell of g(z*) (the
//           x / y / z differences of the cell, each interpolated over the other two axes in x, y, z order), divided by
//           sqrt((x x + y y) + z z); (0, 0, 0) where that length is not positive.  Points toward increasing tsdf.  Colour: the
//           reference's unfold (color_fold.cuh; mesh_oracle.colors_at) of the colour voxel at rint(g(z*)) (half-even), uint8 RGB.
//           Normals and colours are 0 where there is no hit.
//
// Launch: blockIdx.y = view, a CTA = 16 x 8 pixels, each warp an 8 x 4 block (neighbouring rays read neighbouring voxels).  Reads
// the tsdf volume (8 corners per sample, through L1 / L2) and one colour voxel per hit; never the weight volume (the raw tsdf is
// rendered, as get_mesh meshes it).  Bound: load latency of the dependent march, one sample per step.
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "raycast_march.cuh"

namespace dvmvs {

constexpr int kRayTileW = 16, kRayTileH = 8;       // pixels per CTA; 4 warps of 8 x 4
constexpr int kRayMaxViewsPerLaunch = 65535;       // gridDim.y

struct RaycastParams {
  const float* tsdf;
  const float* color;
  const float* views;              // [n_views][16]
  float* depth;                    // [n_views][H][W]
  float* normals;                  // [n_views][H][W][3]
  unsigned char* colors;           // [n_views][H][W][3]
  int dim[3];
  int im_h, im_w, n_skip;
  float origin[3];
  float voxel;
};

__global__ void __launch_bounds__(kRayTileW * kRayTileH) raycast_kernel(RaycastParams p) {
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_w = (p.im_w + kRayTileW - 1) / kRayTileW;
  const int u = (blockIdx.x % tiles_w) * kRayTileW + (warp & 1) * 8 + (lane & 7);
  const int v = (blockIdx.x / tiles_w) * kRayTileH + (warp >> 1) * 4 + (lane >> 3);
  if (u >= p.im_w || v >= p.im_h) return;
  pdl_wait();
  const float* view = p.views + (size_t)blockIdx.y * 16;
  float vw[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) vw[i] = __ldg(view + i);
  const Ray r = rc_ray(vw, u, v, p.dim, p.origin, p.voxel);
  const size_t sx = (size_t)p.dim[1] * p.dim[2], sy = (size_t)p.dim[2];
  const auto corners = [&](const int* ci, float* c) {
    const float* b = p.tsdf + (size_t)ci[0] * sx + (size_t)ci[1] * sy + ci[2];
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) c[i + 2 * j + 4 * k] = __ldg(b + i * sx + j * sy + k);
  };
  float z_hit = 0.f;
  const bool hit = rc_march(p.dim, r, p.n_skip, corners, &z_hit);
  const size_t pix = ((size_t)blockIdx.y * p.im_h + v) * p.im_w + u;
  float nrm[3] = {0.f, 0.f, 0.f};
  unsigned char rgb[3] = {0, 0, 0};
  if (hit) {
    RayCell s;
    rc_cell(p.dim, r.o, r.d, z_hit, corners, s);
    rc_normal(s, nrm);
    int vi[3];
    rc_color_voxel(p.dim, r, z_hit, vi);
    rc_rgb(p.color[((size_t)vi[0] * p.dim[1] + vi[1]) * p.dim[2] + vi[2]], rgb);
  }
  p.depth[pix] = z_hit;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    p.normals[pix * 3 + c] = nrm[c];
    p.colors[pix * 3 + c] = rgb[c];
  }
}

}  // namespace dvmvs

using namespace dvmvs;

extern "C" int dvmvs_tsdf_raycast(const float* tsdf_vol, const float* color_vol, int dim_x, int dim_y, int dim_z,
                                  const float* vol_origin3, double voxel_size, double trunc_margin, const float* views, int n_views,
                                  int im_h, int im_w, float* depth, float* normals, unsigned char* colors, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(tsdf_vol && color_vol && vol_origin3 && views && depth && normals && colors, "tsdf_raycast: null argument");
  DVMVS_REQUIRE(dim_x > 0 && dim_y > 0 && dim_z > 0 && im_h > 0 && im_w > 0 && n_views > 0,
                "tsdf_raycast: bad extent: volume %d x %d x %d, %d views of %d x %d", dim_x, dim_y, dim_z, n_views, im_h, im_w);
  DVMVS_REQUIRE((long long)n_views * im_h * im_w <= (long long)INT_MAX, "tsdf_raycast: %d views of %d x %d pixels exceed int32",
                n_views, im_h, im_w);
  DVMVS_REQUIRE(voxel_size > 0.0 && isfinite(voxel_size) && (float)voxel_size > 0.f, "tsdf_raycast: bad voxel size %g", voxel_size);
  RaycastParams p;
  p.tsdf = tsdf_vol;
  p.color = color_vol;
  p.dim[0] = dim_x;
  p.dim[1] = dim_y;
  p.dim[2] = dim_z;
  p.im_h = im_h;
  p.im_w = im_w;
  p.n_skip = rc_n_skip(trunc_margin, voxel_size);
  for (int a = 0; a < 3; ++a) p.origin[a] = vol_origin3[a];
  p.voxel = (float)voxel_size;
  const int tiles = ((im_w + kRayTileW - 1) / kRayTileW) * ((im_h + kRayTileH - 1) / kRayTileH);
  cudaStream_t s = (cudaStream_t)stream;
  for (int v0 = 0; v0 < n_views; v0 += kRayMaxViewsPerLaunch) {
    const int nv = min(n_views - v0, kRayMaxViewsPerLaunch);
    const size_t px = (size_t)v0 * im_h * im_w;
    p.views = views + (size_t)v0 * 16;
    p.depth = depth + px;
    p.normals = normals + px * 3;
    p.colors = colors + px * 3;
    launch_k(raycast_kernel, dim3((unsigned)tiles, (unsigned)nv), dim3(kRayTileW * kRayTileH), 0, s, p);
    const int err = check_launch("raycast_kernel");
    if (err) return err;
  }
  return DVMVS_OK;
}
