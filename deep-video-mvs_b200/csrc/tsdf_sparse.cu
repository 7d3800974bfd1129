// Voxel-block TSDF volume (include/dvmvs_tsdf_sparse.h): TSDF integration without bounds.  The volume is a pool of 8 x 8 x 8-voxel
// blocks found through an open-addressing hash table on the device; a frame allocates the blocks it can update and integrates
// only those.  Per voxel the arithmetic is tsdf_update_voxel (tsdf_voxel.cuh), the dense kernel's, at the dense kernel's world
// point f32(f64(origin) + voxel_size * f64(global index)), so the volume equals a dense volume with the same origin voxel for
// voxel.
//
// Per frame, four launches and no host read:
//   sparse_tile_max_kernel   largest valid depth (> 0; NaN never counts) of every 16 x 16-pixel tile
//   sparse_box_kernel        the frame's largest depth D and the world box of its view frustum up to D + trunc: the candidate
//                            blocks (blocks of that box; margin: one float32 spacing at the box's largest coordinate, which
//                            bounds how far a voxel's rounded world point strays from origin + voxel_size * index, plus two
//                            voxels)
//   sparse_alloc_kernel      one thread per candidate block: a conservative test (below), then insertion into the hash table
//                            (atomicCAS on the key, the pool slot from an atomic counter) and the block's slot appended to the
//                            frame's list of visible blocks
//   sparse_integrate_kernel  one thread per voxel of the listed blocks, a CTA half a block
// Halt mode (include/dvmvs_tsdf_sparse_grow.h, counters[3]): sparse_box_kernel, the frame's first reader of the counters after
// the previous frame's launches, decides once whether the frame starts with a pool- or table-full flag; if so its box is empty,
// so sparse_alloc_kernel inserts nothing.  sparse_integrate_kernel reads the flags after the frame's own allocation, so the
// frame that sets one is not integrated either.  sparse_rehash_kernel rebuilds the table of a grown pool.
// Conservative test of a candidate block.  Its voxels' world points lie in the box spanned by its corner voxels' points (the
// float32 rounding of origin + voxel_size * index is monotonic in the index), so their exact camera coordinates lie in the
// parallelepiped of the 8 corners' camera coordinates.  Those are evaluated in float64 with a slack eps of 2^-40 times the
// magnitude bound of the affine map (the voxel path's FMA chain and this evaluation are each within ~2^-51 of it).  The block is
// dropped iff, with the slack, (a) every corner is behind the camera, or (b) the block is in front and its projected pixel
// rectangle (corner projections, slack propagated through the division) misses the image, or (c) no tile the rectangle
// touches has a depth d with d + trunc >= z_min - eps.  Anything else (a block crossing the camera plane tests against every
// tile) is allocated, so a voxel the reference updates is never missed; over-allocation costs memory, never a result.
#include <limits.h>
#include <math.h>

#include "../../include/dvmvs_tsdf_sparse.h"
#include "../../include/dvmvs_tsdf_sparse_grow.h"
#include "tsdf_block_hash.cuh"
#include "tsdf_voxel.cuh"

namespace dvmvs {

constexpr int kTile = 16;                            // pixels per tile edge of the max-depth image
constexpr long long kMaxCandidates = 1ll << 31;
constexpr int kBoxBytes = 64;                        // scratch head: SparseBox
constexpr int kCapacityFlags = DVMVS_SPARSE_POOL_FULL | DVMVS_SPARSE_TABLE_FULL;

// halt mode is on and a frame found no room: later frames (and the rest of this one's launches) leave the volume alone
__device__ __forceinline__ bool sparse_halted(const int* counters) {
  return (counters[3] & DVMVS_SPARSE_HALT_ON_FULL) && (counters[1] & kCapacityFlags);
}

struct SparseBox {
  int lo[3], n[3];
  long long count;
};

struct SparseFrame {
  double T[12];            // rows 0..2 of inv(cam_pose)
  double fx, fy, cx, cy;   // float32 intrinsics widened
  double voxel_size, trunc;
  float origin[3];
  int im_h, im_w, tiles_x, tiles_y;
  double C[3];             // camera centre, world frame
  double dir[4][3];        // world-frame rays through the image's corners (1.5 pixels outside it) at camera depth 1
};

struct SparseTable {
  unsigned long long* keys;
  int* slots;
  int* coords;
  int* counters;
  int* visible;
  int mask, capacity;
};

// the pool slot of the block (inserted if new), or -1 (pool or table full: flagged).  Within one launch every key is looked up
// by one thread only, so a key found in the table was inserted by an earlier launch and its slot is published.
__device__ int sparse_insert(const SparseTable& t, int bx, int by, int bz) {
  const unsigned long long key = block_key(bx, by, bz);
  unsigned h = block_hash(key, t.mask);
  for (int probe = 0; probe <= t.mask; ++probe, h = (h + 1) & (unsigned)t.mask) {
    unsigned long long k = t.keys[h];                // a stale read can only be kEmpty: the CAS below then sees the truth
    if (k == kEmpty) k = atomicCAS(&t.keys[h], kEmpty, key);
    if (k == key) return t.slots[h];
    if (k != kEmpty) continue;
    int s = atomicAdd(&t.counters[0], 1);            // this thread inserted the key
    if (s < t.capacity) {
      t.coords[3 * s] = bx; t.coords[3 * s + 1] = by; t.coords[3 * s + 2] = bz;
    } else {
      s = -1;
      atomicOr(&t.counters[1], DVMVS_SPARSE_POOL_FULL);
    }
    t.slots[h] = s;
    return s;
  }
  atomicOr(&t.counters[1], DVMVS_SPARSE_TABLE_FULL);
  return -1;
}

// one thread per pool slot of a grown pool: its key into the fresh table with its own slot.  The keys are distinct and the
// table has >= 2 n_blocks entries, so every probe sequence reaches an empty entry.  Thread 0 resets the counters.
__global__ void __launch_bounds__(256) sparse_rehash_kernel(unsigned long long* keys, int* slots, int mask, const int* __restrict__ coords,
                                                            int n_blocks, int* counters) {
  pdl_launch_dependents();
  pdl_wait();
  const int stride = gridDim.x * blockDim.x;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n_blocks; s += stride) {
    const unsigned long long key = block_key(coords[3 * s], coords[3 * s + 1], coords[3 * s + 2]);
    unsigned h = block_hash(key, mask);
    while (atomicCAS(&keys[h], kEmpty, key) != kEmpty) h = (h + 1) & (unsigned)mask;
    slots[h] = s;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    counters[0] = n_blocks;
    counters[1] &= ~kCapacityFlags;
  }
}

__device__ __forceinline__ double voxel_world(const SparseFrame& f, int axis, long long g) {
  return (double)__double2float_rn(__dadd_rn((double)f.origin[axis], __dmul_rn(f.voxel_size, (double)g)));
}

template <typename DepthT>
__global__ void __launch_bounds__(256) sparse_tile_max_kernel(const DepthT* __restrict__ depth, int im_h, int im_w, int tiles_x,
                                                              double* __restrict__ tile_max) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * kTile + (threadIdx.x & (kTile - 1)), y = blockIdx.y * kTile + (threadIdx.x >> 4);
  double d = -1.0;
  if (x < im_w && y < im_h) {
    const double v = (double)depth[(size_t)y * im_w + x];
    if (v > 0.0) d = v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d = fmax(d, __shfl_xor_sync(0xffffffffu, d, o));
  __shared__ double warp_max[8];
  if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) d = fmax(d, warp_max[i]);
    tile_max[blockIdx.y * tiles_x + blockIdx.x] = d;
  }
}

// one CTA: the frame's largest depth, then its candidate box (empty when halted); resets the frame's visible-block count
__global__ void __launch_bounds__(256) sparse_box_kernel(SparseFrame f, const double* __restrict__ tile_max, SparseBox* box,
                                                         int* counters) {
  pdl_launch_dependents();
  pdl_wait();
  double d = -1.0;
  for (int i = threadIdx.x; i < f.tiles_x * f.tiles_y; i += blockDim.x) d = fmax(d, tile_max[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d = fmax(d, __shfl_xor_sync(0xffffffffu, d, o));
  __shared__ double warp_max[8];
  if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = d;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int i = 1; i < 8; ++i) d = fmax(d, warp_max[i]);
  counters[2] = 0;
  SparseBox b = {{0, 0, 0}, {0, 0, 0}, 0};
  if (d > 0.0 && !sparse_halted(counters)) {
    const double zfar = (d + f.trunc) * (1.0 + 1e-9) + 1e-9;
    bool ok = isfinite(zfar);
    long long count = 1;
    for (int a = 0; a < 3 && ok; ++a) {
      double lo = f.C[a], hi = f.C[a];
      for (int c = 0; c < 4; ++c) {
        const double p = f.C[a] + zfar * f.dir[c][a];
        lo = fmin(lo, p);
        hi = fmax(hi, p);
      }
      // A voxel the frame updates has its world point voxel_world(g) in [lo, hi], but the float32 rounding moves that point up
      // to half a float32 spacing away from origin + voxel_size * g -- many voxels far from the origin (0.5 m at 4.2e6 m).  So
      // the index range is widened by one float32 spacing at the box's largest magnitude, then by two voxels for the float64
      // evaluation of the frustum and of these quotients, then taken to blocks.
      const double m = fmax(fabs(lo), fabs(hi)) + 2.0 * f.voxel_size;
      const double spacing = ldexp(1.0, ilogb(m) - 23);
      const double vlo = floor((lo - spacing - (double)f.origin[a]) / f.voxel_size) - 2.0,
                   vhi = floor((hi + spacing - (double)f.origin[a]) / f.voxel_size) + 2.0;
      const double blo = floor(vlo / kBlock), bhi = floor(vhi / kBlock);
      if (!(blo >= -(double)kKeyBias && bhi < (double)kKeyBias)) {
        ok = false;
        break;
      }
      b.lo[a] = (int)blo;
      b.n[a] = (int)bhi - (int)blo + 1;
      count *= b.n[a];
      if (count > kMaxCandidates) ok = false;
    }
    if (ok) {
      b.count = count;
    } else {
      b = SparseBox{{0, 0, 0}, {0, 0, 0}, 0};
      atomicOr(&counters[1], DVMVS_SPARSE_FRUSTUM);
    }
  }
  *box = b;
}

// whether a frame may update a voxel of block (bx, by, bz): false only when provably not (file header)
__device__ bool sparse_block_seen(const SparseFrame& f, const double* __restrict__ tile_max, int bx, int by, int bz) {
  double w[3][2], mag[3];
  const int b[3] = {bx, by, bz};
  for (int a = 0; a < 3; ++a) {
    w[a][0] = voxel_world(f, a, (long long)b[a] * kBlock);
    w[a][1] = voxel_world(f, a, (long long)b[a] * kBlock + kBlock - 1);
    mag[a] = fmax(fabs(w[a][0]), fabs(w[a][1]));
  }
  double eps[3];
  for (int r = 0; r < 3; ++r)
    eps[r] = 0x1p-40 * (fabs(f.T[4 * r]) * mag[0] + fabs(f.T[4 * r + 1]) * mag[1] + fabs(f.T[4 * r + 2]) * mag[2] + fabs(f.T[4 * r + 3]));
  double X[8], Y[8], Z[8], zmin = INFINITY, zmax = -INFINITY;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const double x = w[0][c & 1], y = w[1][(c >> 1) & 1], z = w[2][c >> 2];
    X[c] = f.T[0] * x + f.T[1] * y + f.T[2] * z + f.T[3];
    Y[c] = f.T[4] * x + f.T[5] * y + f.T[6] * z + f.T[7];
    Z[c] = f.T[8] * x + f.T[9] * y + f.T[10] * z + f.T[11];
    zmin = fmin(zmin, Z[c]);
    zmax = fmax(zmax, Z[c]);
  }
  if (zmax + eps[2] <= 0.0) return false;                                  // (a) behind the camera
  int px0 = 0, px1 = f.im_w - 1, py0 = 0, py1 = f.im_h - 1;
  if (zmin > 2.0 * eps[2]) {                                               // (b) in front: the projected rectangle
    double u0 = INFINITY, u1 = -INFINITY, v0 = INFINITY, v1 = -INFINITY;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const double zl = Z[c] - eps[2];                                     // >= Z / 2 > 0
      const double u = X[c] * f.fx / Z[c] + f.cx, v = Y[c] * f.fy / Z[c] + f.cy;
      const double su = f.fx * (eps[0] + fabs(X[c]) * eps[2] / zl) / zl + 1e-9 * (fabs(u) + fabs(f.cx) + 1.0);
      const double sv = f.fy * (eps[1] + fabs(Y[c]) * eps[2] / zl) / zl + 1e-9 * (fabs(v) + fabs(f.cy) + 1.0);
      u0 = fmin(u0, u - su); u1 = fmax(u1, u + su);
      v0 = fmin(v0, v - sv); v1 = fmax(v1, v + sv);
    }
    // a voxel's pixel is rint(u) of a u in [u0, u1]: within [floor(u0), ceil(u1)]
    u0 = floor(u0); u1 = ceil(u1); v0 = floor(v0); v1 = ceil(v1);
    if (u1 < 0.0 || v1 < 0.0 || u0 > (double)(f.im_w - 1) || v0 > (double)(f.im_h - 1)) return false;
    px0 = (int)fmax(u0, 0.0); px1 = (int)fmin(u1, (double)(f.im_w - 1));
    py0 = (int)fmax(v0, 0.0); py1 = (int)fmin(v1, (double)(f.im_h - 1));
  }
  double d = -1.0;                                                         // (c) the tiles' largest valid depth
  for (int ty = py0 / kTile; ty <= py1 / kTile; ++ty)
    for (int tx = px0 / kTile; tx <= px1 / kTile; ++tx) d = fmax(d, tile_max[ty * f.tiles_x + tx]);
  if (!(d > 0.0)) return false;
  return d + f.trunc + 1e-9 * (d + fabs(zmin) + f.trunc) >= zmin - eps[2];
}

__global__ void __launch_bounds__(256) sparse_alloc_kernel(SparseFrame f, const double* __restrict__ tile_max,
                                                           const SparseBox* __restrict__ box, SparseTable t) {
  pdl_launch_dependents();
  pdl_wait();
  const SparseBox b = *box;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < b.count; i += stride) {
    const long long col = i / b.n[2];
    const int bz = b.lo[2] + (int)(i - col * b.n[2]);
    const int bx = b.lo[0] + (int)(col / b.n[1]), by = b.lo[1] + (int)(col % b.n[1]);
    if (!sparse_block_seen(f, tile_max, bx, by, bz)) continue;
    const int s = sparse_insert(t, bx, by, bz);
    if (s >= 0) {
      const int v = atomicAdd(&t.counters[2], 1);                          // < capacity: a slot is listed once per frame
      if (v < t.capacity) t.visible[v] = s;
    }
  }
}

// one thread per voxel, a CTA half a block ([x][y][z] within it: a warp reads and writes 128 contiguous bytes of each array)
template <typename ColorT, typename DepthT>
__global__ void __launch_bounds__(256) sparse_integrate_kernel(TsdfParams p, const int* __restrict__ coords, const int* __restrict__ counters,
                                                               const int* __restrict__ visible, int capacity) {
  pdl_launch_dependents();
  pdl_wait();
  if (sparse_halted(counters)) return;
  const int n_jobs = 2 * min(counters[2], capacity);
  const int lx = threadIdx.x >> 6, ly = (threadIdx.x >> 3) & 7, lz = threadIdx.x & 7;
  int hits = 0;
  for (int j = blockIdx.x; j < n_jobs; j += gridDim.x) {
    const int s = visible[j >> 1];
    const int x = 4 * (j & 1) + lx;
    const long long gx = (long long)coords[3 * s] * kBlock + x, gy = (long long)coords[3 * s + 1] * kBlock + ly,
                    gz = (long long)coords[3 * s + 2] * kBlock + lz;
    const double wx = (double)__double2float_rn(__dadd_rn((double)p.origin[0], __dmul_rn(p.voxel_size, (double)gx)));
    const double wy = (double)__double2float_rn(__dadd_rn((double)p.origin[1], __dmul_rn(p.voxel_size, (double)gy)));
    const double wz = (double)__double2float_rn(__dadd_rn((double)p.origin[2], __dmul_rn(p.voxel_size, (double)gz)));
    const size_t idx = (size_t)s * kBlockVoxels + (size_t)((x * kBlock + ly) * kBlock + lz);
    hits += tsdf_update_voxel<ColorT, DepthT>(p, idx, wx, wy, wz) ? 1 : 0;
  }
  if (p.updated) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, o);
    if ((threadIdx.x & 31) == 0 && hits) atomicAdd(p.updated, (unsigned long long)hits);
  }
}

__global__ void __launch_bounds__(256) sparse_export_kernel(const float* __restrict__ tsdf, const float* __restrict__ weight,
                                                            const float* __restrict__ color, const int* __restrict__ coords,
                                                            const int* __restrict__ counters, int capacity, long long gx0, long long gy0,
                                                            long long gz0, int dim_x, int dim_y, int dim_z, float* __restrict__ tsdf_vol,
                                                            float* __restrict__ weight_vol, float* __restrict__ color_vol) {
  pdl_launch_dependents();
  pdl_wait();
  const int n_jobs = 2 * min(counters[0], capacity);
  const int lx = threadIdx.x >> 6, ly = (threadIdx.x >> 3) & 7, lz = threadIdx.x & 7;
  for (int j = blockIdx.x; j < n_jobs; j += gridDim.x) {
    const int s = j >> 1, x = 4 * (j & 1) + lx;
    const long long i = (long long)coords[3 * s] * kBlock + x - gx0, k = (long long)coords[3 * s + 1] * kBlock + ly - gy0,
                    l = (long long)coords[3 * s + 2] * kBlock + lz - gz0;
    if (i < 0 || i >= dim_x || k < 0 || k >= dim_y || l < 0 || l >= dim_z) continue;
    const size_t src = (size_t)s * kBlockVoxels + (size_t)((x * kBlock + ly) * kBlock + lz);
    const size_t dst = ((size_t)i * dim_y + (size_t)k) * dim_z + (size_t)l;
    tsdf_vol[dst] = tsdf[src];
    weight_vol[dst] = weight[src];
    color_vol[dst] = color[src];
  }
}

__global__ void __launch_bounds__(1024) sparse_bounds_kernel(const int* __restrict__ coords, const int* __restrict__ counters, int capacity,
                                                             int* bounds6) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ int red[6];
  if (threadIdx.x < 6) red[threadIdx.x] = threadIdx.x < 3 ? INT_MAX : INT_MIN;
  __syncthreads();
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  const int n = min(counters[0], capacity);
  for (int s = threadIdx.x; s < n; s += blockDim.x)
    for (int a = 0; a < 3; ++a) {
      lo[a] = min(lo[a], coords[3 * s + a]);
      hi[a] = max(hi[a], coords[3 * s + a]);
    }
  for (int a = 0; a < 3; ++a) {
    atomicMin(&red[a], lo[a]);
    atomicMax(&red[3 + a], hi[a]);
  }
  __syncthreads();
  if (threadIdx.x < 6) bounds6[threadIdx.x] = red[threadIdx.x];
}

// host: the frame's parameters from the dvmvs_tsdf_integrate-style arguments; false when the pose's rotation part is singular
bool sparse_frame(SparseFrame& f, const float* vol_origin3, double voxel_size, double trunc, int im_h, int im_w, const float* intr4,
                  const double* T) {
  for (int i = 0; i < 12; ++i) f.T[i] = T[i];
  f.fx = intr4[0]; f.fy = intr4[1]; f.cx = intr4[2]; f.cy = intr4[3];
  f.voxel_size = voxel_size; f.trunc = trunc;
  for (int a = 0; a < 3; ++a) f.origin[a] = vol_origin3[a];
  f.im_h = im_h; f.im_w = im_w;
  f.tiles_x = (im_w + kTile - 1) / kTile; f.tiles_y = (im_h + kTile - 1) / kTile;
  // camera -> world: inv(A) (cofactors) and C = -inv(A) t of world -> camera [A t]
  const double a = T[0], b = T[1], c = T[2], d = T[4], e = T[5], g = T[6], h = T[8], k = T[9], l = T[10];
  const double det = a * (e * l - g * k) - b * (d * l - g * h) + c * (d * k - e * h);
  if (!(fabs(det) > 0.0) || !isfinite(det)) return false;
  const double R[9] = {(e * l - g * k) / det, (c * k - b * l) / det, (b * g - c * e) / det,
                       (g * h - d * l) / det, (a * l - c * h) / det, (c * d - a * g) / det,
                       (d * k - e * h) / det, (b * h - a * k) / det, (a * e - b * d) / det};
  for (int r = 0; r < 3; ++r) f.C[r] = -(R[3 * r] * T[3] + R[3 * r + 1] * T[7] + R[3 * r + 2] * T[11]);
  const double us[2] = {-1.5, im_w + 0.5}, vs[2] = {-1.5, im_h + 0.5};
  for (int q = 0; q < 4; ++q) {
    const double cam[3] = {(us[q & 1] - f.cx) / f.fx, (vs[q >> 1] - f.cy) / f.fy, 1.0};
    for (int r = 0; r < 3; ++r) f.dir[q][r] = R[3 * r] * cam[0] + R[3 * r + 1] * cam[1] + R[3 * r + 2] * cam[2];
  }
  bool finite = true;
  for (int r = 0; r < 3; ++r) {
    finite = finite && isfinite(f.C[r]);
    for (int q = 0; q < 4; ++q) finite = finite && isfinite(f.dir[q][r]);
  }
  return finite;
}

inline int sparse_grid() { return device_sm_count() * 8; }

}  // namespace dvmvs

using namespace dvmvs;

static bool sparse_geometry_ok(const float* vol_origin3, double voxel_size, double trunc_margin, const float* intr4) {
  return isfinite(vol_origin3[0]) && isfinite(vol_origin3[1]) && isfinite(vol_origin3[2]) && voxel_size > 0.0 && isfinite(voxel_size) &&
         trunc_margin > 0.0 && isfinite(trunc_margin) && intr4[0] > 0.f && intr4[1] > 0.f && isfinite(intr4[0]) && isfinite(intr4[1]) &&
         isfinite(intr4[2]) && isfinite(intr4[3]);
}

extern "C" int dvmvs_tsdf_sparse_scratch_bytes(int im_h, int im_w, long long* bytes_host) {
  DVMVS_REQUIRE(bytes_host, "tsdf_sparse_scratch_bytes: null argument");
  DVMVS_REQUIRE(im_h > 0 && im_w > 0, "tsdf_sparse_scratch_bytes: bad image %d x %d", im_h, im_w);
  *bytes_host = kBoxBytes + 8ll * ((im_h + kTile - 1) / kTile) * ((im_w + kTile - 1) / kTile);
  return DVMVS_OK;
}

extern "C" int dvmvs_tsdf_sparse_allocate(unsigned long long* keys, int* slots, int table_size, int* block_coords, int capacity, int* counters,
                                          int* visible, void* scratch, long long scratch_bytes, const float* vol_origin3, double voxel_size,
                                          double trunc_margin, const void* depth_im, int depth_is_f64, int im_h, int im_w, const float* intr4,
                                          const double* world_to_cam16, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(keys && slots && block_coords && counters && visible && scratch && vol_origin3 && depth_im && intr4 && world_to_cam16,
                "tsdf_sparse_allocate: null argument");
  DVMVS_REQUIRE(capacity > 0 && table_size >= capacity && table_size <= (1 << 30) && (table_size & (table_size - 1)) == 0,
                "tsdf_sparse_allocate: capacity %d, table size %d (a power of two >= capacity, <= 2^30)", capacity, table_size);
  DVMVS_REQUIRE(im_h > 0 && im_w > 0, "tsdf_sparse_allocate: bad image %d x %d", im_h, im_w);
  long long need = 0;
  dvmvs_tsdf_sparse_scratch_bytes(im_h, im_w, &need);
  DVMVS_REQUIRE(scratch_bytes >= need && (uintptr_t)scratch % 16 == 0, "tsdf_sparse_allocate: scratch of %lld bytes at %p, %lld 16-byte aligned needed",
                scratch_bytes, scratch, need);
  DVMVS_REQUIRE(sparse_geometry_ok(vol_origin3, voxel_size, trunc_margin, intr4),
                "tsdf_sparse_allocate: origin, voxel size, truncation and intrinsics must be finite, fx, fy, voxel size and truncation > 0");
  SparseFrame f;
  DVMVS_REQUIRE(sparse_frame(f, vol_origin3, voxel_size, trunc_margin, im_h, im_w, intr4, world_to_cam16),
                "tsdf_sparse_allocate: world_to_cam16 is not an invertible finite transform");
  SparseBox* box = (SparseBox*)scratch;
  double* tile_max = (double*)((char*)scratch + kBoxBytes);
  SparseTable t = {keys, slots, block_coords, counters, visible, table_size - 1, capacity};
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 tiles(f.tiles_x, f.tiles_y);
  if (depth_is_f64) launch_k(sparse_tile_max_kernel<double>, tiles, dim3(256), 0, s, (const double*)depth_im, im_h, im_w, f.tiles_x, tile_max);
  else launch_k(sparse_tile_max_kernel<float>, tiles, dim3(256), 0, s, (const float*)depth_im, im_h, im_w, f.tiles_x, tile_max);
  int rc = check_launch("sparse_tile_max_kernel");
  if (rc) return rc;
  launch_k(sparse_box_kernel, dim3(1), dim3(256), 0, s, f, (const double*)tile_max, box, counters);
  if ((rc = check_launch("sparse_box_kernel"))) return rc;
  launch_k(sparse_alloc_kernel, dim3(sparse_grid()), dim3(256), 0, s, f, (const double*)tile_max, (const SparseBox*)box, t);
  return check_launch("sparse_alloc_kernel");
}

extern "C" int dvmvs_tsdf_sparse_integrate(float* tsdf, float* weight, float* color, const int* block_coords, int capacity, const int* counters,
                                           const int* visible, const float* vol_origin3, double voxel_size, double trunc_margin,
                                           const void* color_im, int color_is_u8, const void* depth_im, int depth_is_f64, int im_h, int im_w,
                                           const float* intr4, const double* world_to_cam16, double obs_weight, unsigned long long* updated_count,
                                           dvmvs_stream_t stream) {
  DVMVS_REQUIRE(tsdf && weight && color && block_coords && counters && visible && vol_origin3 && color_im && depth_im && intr4 && world_to_cam16,
                "tsdf_sparse_integrate: null argument");
  DVMVS_REQUIRE(capacity > 0 && im_h > 0 && im_w > 0, "tsdf_sparse_integrate: capacity %d, image %d x %d", capacity, im_h, im_w);
  DVMVS_REQUIRE(sparse_geometry_ok(vol_origin3, voxel_size, trunc_margin, intr4),
                "tsdf_sparse_integrate: origin, voxel size, truncation and intrinsics must be finite, fx, fy, voxel size and truncation > 0");
  TsdfParams p = {};
  p.tsdf = tsdf; p.weight = weight; p.color = color;
  p.color_im = color_im; p.depth_im = depth_im;
  p.im_h = im_h; p.im_w = im_w;
  for (int i = 0; i < 3; ++i) p.origin[i] = vol_origin3[i];
  p.voxel_size = voxel_size; p.trunc = trunc_margin; p.obs = obs_weight;
  for (int i = 0; i < 12; ++i) p.T[i] = world_to_cam16[i];
  p.fx = (double)intr4[0]; p.fy = (double)intr4[1]; p.cx = (double)intr4[2]; p.cy = (double)intr4[3];
  p.updated = updated_count;
  const dim3 grid(sparse_grid()), block(256);
  cudaStream_t s = (cudaStream_t)stream;
  if (color_is_u8) {
    if (depth_is_f64) launch_k(sparse_integrate_kernel<unsigned char, double>, grid, block, 0, s, p, block_coords, counters, visible, capacity);
    else launch_k(sparse_integrate_kernel<unsigned char, float>, grid, block, 0, s, p, block_coords, counters, visible, capacity);
  } else {
    if (depth_is_f64) launch_k(sparse_integrate_kernel<float, double>, grid, block, 0, s, p, block_coords, counters, visible, capacity);
    else launch_k(sparse_integrate_kernel<float, float>, grid, block, 0, s, p, block_coords, counters, visible, capacity);
  }
  return check_launch("sparse_integrate_kernel");
}

extern "C" int dvmvs_tsdf_sparse_export(const float* tsdf, const float* weight, const float* color, const int* block_coords, int capacity,
                                        const int* counters, const int* box_lo_host, int dim_x, int dim_y, int dim_z, float* tsdf_vol,
                                        float* weight_vol, float* color_vol, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(tsdf && weight && color && block_coords && counters && box_lo_host && tsdf_vol && weight_vol && color_vol,
                "tsdf_sparse_export: null argument");
  DVMVS_REQUIRE(capacity > 0 && dim_x > 0 && dim_y > 0 && dim_z > 0, "tsdf_sparse_export: capacity %d, box %d x %d x %d", capacity, dim_x, dim_y, dim_z);
  launch_k(sparse_export_kernel, dim3(sparse_grid()), dim3(256), 0, (cudaStream_t)stream, tsdf, weight, color, block_coords, counters, capacity,
           (long long)box_lo_host[0], (long long)box_lo_host[1], (long long)box_lo_host[2], dim_x, dim_y, dim_z, tsdf_vol, weight_vol, color_vol);
  return check_launch("sparse_export_kernel");
}

extern "C" int dvmvs_tsdf_sparse_block_bounds(const int* block_coords, int capacity, const int* counters, int* bounds6, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(block_coords && counters && bounds6, "tsdf_sparse_block_bounds: null argument");
  DVMVS_REQUIRE(capacity > 0, "tsdf_sparse_block_bounds: capacity %d", capacity);
  launch_k(sparse_bounds_kernel, dim3(1), dim3(1024), 0, (cudaStream_t)stream, block_coords, counters, capacity, bounds6);
  return check_launch("sparse_bounds_kernel");
}

extern "C" int dvmvs_tsdf_sparse_rehash(unsigned long long* keys, int* slots, int table_size, const int* block_coords, int n_blocks, int* counters,
                                        dvmvs_stream_t stream) {
  DVMVS_REQUIRE(keys && slots && block_coords && counters, "tsdf_sparse_rehash: null argument");
  DVMVS_REQUIRE(table_size > 0 && table_size <= (1 << 30) && (table_size & (table_size - 1)) == 0 && n_blocks >= 0 &&
                    2ll * n_blocks <= table_size,
                "tsdf_sparse_rehash: table size %d, %d blocks (a power of two <= 2^30, >= 2 x the blocks)", table_size, n_blocks);
  int grid = (n_blocks + 255) / 256;
  grid = grid < 1 ? 1 : (grid > sparse_grid() ? sparse_grid() : grid);
  launch_k(sparse_rehash_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, keys, slots, table_size - 1, block_coords, n_blocks,
           counters);
  return check_launch("sparse_rehash_kernel");
}
