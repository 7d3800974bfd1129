// Mesh and ray casting of the voxel-block TSDF volume on its blocks (include/dvmvs_tsdf_sparse_view.h): over any lattice-aligned
// box, the results equal bit for bit those of the dense kernels (mesh.cu, raycast.cu) on the box dvmvs_tsdf_sparse_export
// fills, without materialising it.  A voxel of a block that is not allocated reads as the export writes it: tsdf 1.0, colour 0.
// The per-edge and per-sample arithmetic is the dense kernels' own (mc_vertex.cuh, raycast_march.cuh); only the voxel fetch
// differs: box index -> global voxel -> block -> pool slot through the hash table (tsdf_block_hash.cuh).
//
// Mesh: count -> scan -> (host reads the totals) -> emit -> resolve, as mesh.cu.
//   work list  the allocated blocks, plus every missing block whose +x, +y, +z or diagonal neighbour is allocated: a cube or
//              grid edge whose lowest corner is the voxel at local index 7 of such a block reaches into the allocated one and
//              can cross the surface (a missing voxel is never inside).  A missing block is listed once, by its allocated
//              neighbour of least offset index.  Blocks that do not meet the box are left out.
//   order      the dense mesh orders vertices by key 3 * (box linear index) + axis and faces by cube.  Within a block, the 8
//              voxels of a z-run (fixed local x, y) are consecutive in that order, so the work blocks are sorted by (x, y, z)
//              (CUB radix sort: deterministic) and each z-run gets its dense rank from its block's slab (same block x) and column
//              (same block x, y) in the sorted list:  rank = 64 s0 + 8 (c0 - s0) + (j - c0) + lx 8 S + ly C  (s0, S: the slab's
//              first position and size; c0, C: the column's; j the block's position).  Counts are kept per rank and scanned in
//              rank order (CUB scan), so emit writes every vertex and face at its dense position; faces resolve their 64-bit
//              edge keys to vertex ids by binary search, as mesh_resolve_kernel.  Nothing sized by the box's voxel count.
// Ray casting: raycast.cu's march over the box (rc_march), the 8 corners of a cell fetched through the hash with the slots of
// the last cell's 2 x 2 x 2 block neighbourhood cached per ray (probed lazily), so a sample probes the table only when the ray
// enters a new block.
#include <limits.h>
#include <math.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/dvmvs_tsdf_sparse_view.h"
#include "common.cuh"
#include "mc_tables.cuh"
#include "mc_vertex.cuh"
#include "raycast_march.cuh"
#include "tsdf_block_hash.cuh"

namespace dvmvs {

constexpr long long kMaxViewBlocks = 1ll << 22;     // mesh: below this, 8 x 64 z-runs per block + 1 stay below 2^31 scan items
constexpr long long kMaxBoxVoxels = 1ll << 61;      // 3 * box voxels + 2 fits the int64 vertex keys
constexpr int kViewThreads = 256;
constexpr int kRayTileW = 16, kRayTileH = 8;
constexpr int kRayMaxViewsPerLaunch = 65535;

// the volume, read-only, and the box: box index (i, j, k) is global voxel k0 + (i, j, k)
struct SparseView {
  const unsigned long long* keys;
  const int* slots;
  const int* coords;
  const int* counters;
  const float* tsdf;
  const float* color;
  int mask, capacity;
  long long k0[3];
  int dim[3];
};

// a value of the pool at global voxel g, or `missing` when its block is not allocated
__device__ __forceinline__ float sv_voxel(const SparseView& v, const float* pool, const long long* g, float missing) {
  const int s = sparse_find(v.keys, v.slots, v.mask, g[0] >> 3, g[1] >> 3, g[2] >> 3);
  if (s < 0) return missing;
  return __ldg(pool + (size_t)s * kBlockVoxels + (size_t)((((int)g[0] & 7) * kBlock + ((int)g[1] & 7)) * kBlock + ((int)g[2] & 7)));
}

// tsdf at box index (x, y, z) + s e_a
__device__ __forceinline__ float sv_tsdf_box(const SparseView& v, int x, int y, int z) {
  const long long g[3] = {v.k0[0] + x, v.k0[1] + y, v.k0[2] + z};
  return sv_voxel(v, v.tsdf, g, 1.f);
}

__device__ __forceinline__ long long sv_lin(const SparseView& v, long long x, long long y, long long z) {
  return (x * v.dim[1] + y) * v.dim[2] + z;
}

// ---- mesh -----------------------------------------------------------------------------------------------------------------
struct WorkBlock {
  int b[3];
  int slot;                        // -1: a missing block
};

struct ZBlock {                    // a work block at its sorted position
  int b[3];
  int nb[8];                       // pool slots of b + (i, j, k), i, j, k in {0, 1}, at nb[i + 2 j + 4 k] (-1: missing)
  int slab, column;                // S and C of the rank formula
  long long base;                  // rank of z-run (0, 0)
};

struct MeshScratch {               // device layout, in the order of the scratch
  long long* totals;               // [2] vertices, faces (the one host read)
  int* work_count;
  WorkBlock* work;                 // [W]
  unsigned long long* sort_keys;   // [2][W]
  int* sort_vals;                  // [2][W]
  ZBlock* blocks;                  // [W] sorted
  longlong2* counts;               // [64 W + 1] per rank: (vertices, faces), then their exclusive scan
  void* cub_temp;
  size_t cub_bytes;
  long long bytes;
};

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct AddPair {
  __device__ __forceinline__ longlong2 operator()(const longlong2& a, const longlong2& b) const { return make_longlong2(a.x + b.x, a.y + b.y); }
};

// the scratch layout for n_blocks allocated blocks (W = 8 n_blocks work blocks at most); base == nullptr: sizes only
static int mesh_scratch(long long n_blocks, void* base, MeshScratch& m) {
  const long long W = 8 * n_blocks;
  char* p = (char*)base;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* q = p ? p + off : nullptr; off += align256(bytes); return (void*)q; };
  m.totals = (long long*)take(64);
  m.work_count = (int*)(m.totals ? (char*)m.totals + 16 : nullptr);
  m.work = (WorkBlock*)take(sizeof(WorkBlock) * W);
  m.sort_keys = (unsigned long long*)take(sizeof(unsigned long long) * 2 * W);
  m.sort_vals = (int*)take(sizeof(int) * 2 * W);
  m.blocks = (ZBlock*)take(sizeof(ZBlock) * W);
  m.counts = (longlong2*)take(sizeof(longlong2) * (64 * W + 1));
  size_t sort_bytes = 0, scan_bytes = 0;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                                  (int*)nullptr, (int*)nullptr, (int)W);
  if (e == cudaSuccess)
    e = cub::DeviceScan::ExclusiveScan(nullptr, scan_bytes, (longlong2*)nullptr, (longlong2*)nullptr, AddPair(), make_longlong2(0, 0),
                                       (int)(64 * W + 1));
  if (e != cudaSuccess) {
    set_error("tsdf_sparse_mesh: CUB temp-storage query: %s", cudaGetErrorString(e));
    return DVMVS_ELAUNCH;
  }
  m.cub_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
  m.cub_temp = take(m.cub_bytes);
  m.bytes = (long long)off;
  return DVMVS_OK;
}

// one thread per (allocated block, offset index 0..7): the block itself (0) or its missing neighbour block - offset
__global__ void __launch_bounds__(kViewThreads) mesh_work_kernel(SparseView v, int n_blocks, WorkBlock* __restrict__ work, int* work_count) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = min(min(v.counters[0], v.capacity), n_blocks);
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < 8ll * n; i += stride) {
    const int s = (int)(i >> 3), d = (int)(i & 7);
    const int b[3] = {v.coords[3 * s], v.coords[3 * s + 1], v.coords[3 * s + 2]};
    const long long m[3] = {(long long)b[0] - (d & 1), (long long)b[1] - ((d >> 1) & 1), (long long)b[2] - (d >> 2)};
    bool keep = true;
    for (int a = 0; a < 3; ++a) keep = keep && 8 * m[a] + 7 >= v.k0[a] && 8 * m[a] < v.k0[a] + v.dim[a];
    if (!keep) continue;
    int slot = s;
    if (d != 0) {
      if (sparse_find(v.keys, v.slots, v.mask, m[0], m[1], m[2]) >= 0) continue;       // allocated: listed by itself
      for (int e = 1; e < d && keep; ++e)     // listed by the allocated neighbour of least offset index
        keep = sparse_find(v.keys, v.slots, v.mask, m[0] + (e & 1), m[1] + ((e >> 1) & 1), m[2] + (e >> 2)) < 0;
      if (!keep) continue;
      slot = -1;
    }
    const int w = atomicAdd(work_count, 1);
    work[w] = WorkBlock{{(int)m[0], (int)m[1], (int)m[2]}, slot};
  }
}

// sort keys: the box linear index of the block's first voxel in the box (monotone in (x, y, z) over blocks meeting the box);
// padding past the work count sorts last
__global__ void __launch_bounds__(kViewThreads) mesh_key_kernel(SparseView v, int W, const WorkBlock* __restrict__ work, const int* work_count,
                                                                unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = *work_count;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < W; i += gridDim.x * blockDim.x) {
    unsigned long long key = ~0ull;
    if (i < n) {
      long long q[3];
      for (int a = 0; a < 3; ++a) q[a] = max(8ll * work[i].b[a], v.k0[a]) - v.k0[a];
      key = (unsigned long long)sv_lin(v, q[0], q[1], q[2]);
    }
    keys[i] = key;
    vals[i] = i;
  }
}

// first sorted position in [0, n) whose block is not below `b` in its first `depth` coordinates
__device__ __forceinline__ int zb_lower(const WorkBlock* work, const int* order, int n, const int* b, int depth, bool upper) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const int* c = work[order[mid]].b;
    int cmp = c[0] != b[0] ? (c[0] < b[0] ? -1 : 1) : 0;
    if (depth == 2 && cmp == 0) cmp = c[1] != b[1] ? (c[1] < b[1] ? -1 : 1) : 0;
    if (cmp < 0 || (upper && cmp == 0)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kViewThreads) mesh_block_kernel(SparseView v, const WorkBlock* __restrict__ work, const int* work_count,
                                                                  const int* __restrict__ order, ZBlock* __restrict__ blocks) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = *work_count;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const WorkBlock w = work[order[j]];
    ZBlock z;
    for (int a = 0; a < 3; ++a) z.b[a] = w.b[a];
    z.nb[0] = w.slot;
    for (int d = 1; d < 8; ++d)
      z.nb[d] = sparse_find(v.keys, v.slots, v.mask, (long long)w.b[0] + (d & 1), (long long)w.b[1] + ((d >> 1) & 1), (long long)w.b[2] + (d >> 2));
    const int s0 = zb_lower(work, order, n, w.b, 1, false), s1 = zb_lower(work, order, n, w.b, 1, true);
    const int c0 = zb_lower(work, order, n, w.b, 2, false), c1 = zb_lower(work, order, n, w.b, 2, true);
    z.slab = s1 - s0;
    z.column = c1 - c0;
    z.base = 64ll * s0 + 8ll * (c0 - s0) + (j - c0);
    blocks[j] = z;
  }
}

// the classification of mesh.cu's mc_classify at one voxel of a work block; false where the voxel is outside the box
struct SparseClass {
  int q[3];                        // box index
  int cube_case;
  unsigned edges;
  float f0, fe[3];
};

// z in global memory: its slots are indexed by voxel, and a local copy would live on the stack
__device__ __forceinline__ float zb_corner(const SparseView& v, const ZBlock* z, int lx, int ly, int lz) {
  const int s = __ldg(&z->nb[(lx >> 3) + 2 * (ly >> 3) + 4 * (lz >> 3)]);
  if (s < 0) return 1.f;
  return __ldg(v.tsdf + (size_t)s * kBlockVoxels + (size_t)(((lx & 7) * kBlock + (ly & 7)) * kBlock + (lz & 7)));
}

__device__ __forceinline__ bool sparse_classify(const SparseView& v, const ZBlock* z, int lx, int ly, int lz, SparseClass& c) {
  const int l[3] = {lx, ly, lz};
  bool has[3];
  for (int a = 0; a < 3; ++a) {
    const long long q = 8ll * __ldg(&z->b[a]) + l[a] - v.k0[a];
    if (q < 0 || q >= v.dim[a]) return false;
    c.q[a] = (int)q;
    has[a] = q + 1 < v.dim[a];
  }
  c.f0 = zb_corner(v, z, lx, ly, lz);
  c.edges = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    c.fe[a] = has[a] ? zb_corner(v, z, lx + (a == 0), ly + (a == 1), lz + (a == 2)) : 1.f;
    if (has[a] && mc_inside(c.f0) != mc_inside(c.fe[a])) c.edges |= 1u << a;
  }
  c.cube_case = 0;
  if (has[0] && has[1] && has[2]) {
    int cs = (mc_inside(c.f0) ? 1 : 0) | (mc_inside(c.fe[0]) ? 2 : 0) | (mc_inside(c.fe[1]) ? 4 : 0) | (mc_inside(c.fe[2]) ? 16 : 0);
    const int rest[4] = {3, 5, 6, 7};
#pragma unroll
    for (int k = 0; k < 4; ++k)
      cs |= mc_inside(zb_corner(v, z, lx + (rest[k] & 1), ly + ((rest[k] >> 1) & 1), lz + (rest[k] >> 2))) ? (1 << rest[k]) : 0;
    c.cube_case = cs;
  }
  return true;
}

// one thread per voxel of the (padded) work list, 8 consecutive threads a z-run: per-rank (vertices, faces)
__global__ void __launch_bounds__(kViewThreads) mesh_sparse_count_kernel(SparseView v, int W, const int* work_count, const ZBlock* __restrict__ blocks,
                                                                         longlong2* __restrict__ counts) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = *work_count;
  if (blockIdx.x == 0 && threadIdx.x == 0) counts[64ll * W] = make_longlong2(0, 0);
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < 512ll * W; i += stride) {
    const int j = (int)(i >> 9), lx = (int)(i >> 6) & 7, ly = (int)(i >> 3) & 7, lz = (int)i & 7;
    unsigned packed = 0u;
    long long rank = 64ll * j + 8 * lx + ly;          // padding: the ranks past the work list
    if (j < n) {
      const ZBlock* z = blocks + j;
      SparseClass c;
      if (sparse_classify(v, z, lx, ly, lz, c)) packed = (unsigned)__popc(c.edges) | ((unsigned)kMcNumTris[c.cube_case] << 16);
      rank = z->base + 8ll * lx * z->slab + (long long)ly * z->column;
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) packed += __shfl_xor_sync(0xffffffffu, packed, o);
    if (lz == 0) counts[rank] = make_longlong2(packed & 0xffffu, packed >> 16);
  }
}

struct SparseEmit {
  SparseView v;
  const ZBlock* blocks;
  const int* work_count;
  const longlong2* offsets;        // scanned counts per rank
  float origin[3];
  float voxel;
  long long* vertex_keys;          // [V]
  long long* face_keys;            // [3 F]
  float* verts;
  float* norms;
  unsigned char* colors;
};

__global__ void __launch_bounds__(kViewThreads) mesh_sparse_emit_kernel(SparseEmit p, int W) {
  pdl_launch_dependents();
  pdl_wait();
  const SparseView& v = p.v;
  const int n = *p.work_count;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < 512ll * W; i += stride) {
    const int j = (int)(i >> 9), lx = (int)(i >> 6) & 7, ly = (int)(i >> 3) & 7, lz = (int)i & 7;
    if (j >= n) break;                                 // uniform per warp (512-thread groups)
    const ZBlock* z = p.blocks + j;
    SparseClass c;
    unsigned packed = 0u;
    if (sparse_classify(v, z, lx, ly, lz, c)) packed = (unsigned)__popc(c.edges) | ((unsigned)kMcNumTris[c.cube_case] << 16);
    unsigned incl = packed;
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      const unsigned u = __shfl_up_sync(0xffffffffu, incl, o, 8);
      if (lz >= o) incl += u;
    }
    if (packed == 0u) continue;
    const unsigned excl = incl - packed;
    const longlong2 base = p.offsets[z->base + 8ll * lx * z->slab + (long long)ly * z->column];
    long long slot = base.x + (excl & 0xffffu);
    const long long lin = sv_lin(v, c.q[0], c.q[1], c.q[2]);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!(c.edges & (1u << a))) continue;
      const McVertex m = mc_vertex(
          c.f0, c.fe[a], c.q, a,
          [&](int x, int y, int zz, float* gr) {
            // the (up to) 7 voxels np.gradient reads, fetched before its arithmetic
            const int q[3] = {x, y, zz};
            float f[3][3];
            f[0][1] = f[1][1] = f[2][1] = sv_tsdf_box(v, x, y, zz);
#pragma unroll
            for (int ax = 0; ax < 3; ++ax) {
              f[ax][0] = q[ax] > 0 ? sv_tsdf_box(v, x - (ax == 0), y - (ax == 1), zz - (ax == 2)) : 0.f;
              f[ax][2] = q[ax] < v.dim[ax] - 1 ? sv_tsdf_box(v, x + (ax == 0), y + (ax == 1), zz + (ax == 2)) : 0.f;
            }
            mc_np_gradient(q, v.dim, [&](int ax, int s) { return f[ax][s + 1]; }, gr);
          },
          [&](int ix, int iy, int iz) {
            const long long g[3] = {v.k0[0] + ix, v.k0[1] + iy, v.k0[2] + iz};
            return sv_voxel(v, v.color, g, 0.f);
          },
          p.origin, p.voxel);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        p.verts[3 * slot + k] = m.vert[k];
        p.norms[3 * slot + k] = m.norm[k];
        p.colors[3 * slot + k] = m.rgb[k];
      }
      p.vertex_keys[slot] = 3 * lin + a;
      ++slot;
    }
    const int n_tris = kMcNumTris[c.cube_case];
    long long* face = p.face_keys + 3 * (base.y + (excl >> 16));
    for (int k = 0; k < n_tris * 3; ++k) {
      const int e = kMcTris[c.cube_case][k], corner = kMcEdgeCorner[e][0];
      face[k] = 3 * sv_lin(v, c.q[0] + (corner & 1), c.q[1] + ((corner >> 1) & 1), c.q[2] + (corner >> 2)) + (e >> 2);
    }
  }
}

// edge key -> vertex id: lower bound in the sorted key array (every face key is present by construction)
__global__ void __launch_bounds__(256) mesh_sparse_resolve_kernel(const long long* __restrict__ face_keys, long long n, const long long* __restrict__ keys,
                                                                  int n_keys, int* __restrict__ faces) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const long long key = face_keys[i];
  int lo = 0, hi = n_keys;
  while (lo < hi) {
    const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
    if (__ldg(keys + mid) < key) lo = mid + 1;
    else hi = mid;
  }
  faces[i] = lo;
}

// ---- ray casting ----------------------------------------------------------------------------------------------------------
struct SparseRaycast {
  SparseView v;
  const float* views;
  float* depth;
  float* normals;
  unsigned char* colors;
  int im_h, im_w, n_skip;
  float origin[3];
  float voxel;
};

// the slots of the 2 x 2 x 2 blocks from `b` up, probed when first needed (-2: not probed yet)
struct BlockCache {
  long long b[3];
  int s[8];
};

__global__ void __launch_bounds__(kRayTileW * kRayTileH) sparse_raycast_kernel(SparseRaycast p) {
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_w = (p.im_w + kRayTileW - 1) / kRayTileW;
  const int u = (blockIdx.x % tiles_w) * kRayTileW + (warp & 1) * 8 + (lane & 7);
  const int v = (blockIdx.x / tiles_w) * kRayTileH + (warp >> 1) * 4 + (lane >> 3);
  if (u >= p.im_w || v >= p.im_h) return;
  pdl_wait();
  const SparseView& sv = p.v;
  const float* view = p.views + (size_t)blockIdx.y * 16;
  float vw[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) vw[i] = __ldg(view + i);
  const Ray r = rc_ray(vw, u, v, sv.dim, p.origin, p.voxel);
  BlockCache cache = {{LLONG_MIN, 0, 0}, {-2, -2, -2, -2, -2, -2, -2, -2}};
  const auto corners = [&](const int* ci, float* c) {
    const long long g[3] = {sv.k0[0] + ci[0], sv.k0[1] + ci[1], sv.k0[2] + ci[2]};
    const long long b[3] = {g[0] >> 3, g[1] >> 3, g[2] >> 3};
    if (b[0] != cache.b[0] || b[1] != cache.b[1] || b[2] != cache.b[2]) {
      for (int a = 0; a < 3; ++a) cache.b[a] = b[a];
#pragma unroll
      for (int d = 0; d < 8; ++d) cache.s[d] = -2;
    }
    const int l[3] = {(int)(g[0] & 7), (int)(g[1] & 7), (int)(g[2] & 7)};
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int x = l[0] + i, y = l[1] + j, z = l[2] + k;
          const int d = (x >> 3) + 2 * (y >> 3) + 4 * (z >> 3);
          int s = cache.s[d];
          if (s == -2) s = cache.s[d] = sparse_find(sv.keys, sv.slots, sv.mask, b[0] + (x >> 3), b[1] + (y >> 3), b[2] + (z >> 3));
          c[i + 2 * j + 4 * k] = s < 0 ? 1.f : __ldg(sv.tsdf + (size_t)s * kBlockVoxels + (size_t)(((x & 7) * kBlock + (y & 7)) * kBlock + (z & 7)));
        }
  };
  float z_hit = 0.f;
  const bool hit = rc_march(sv.dim, r, p.n_skip, corners, &z_hit);
  const size_t pix = ((size_t)blockIdx.y * p.im_h + v) * p.im_w + u;
  float nrm[3] = {0.f, 0.f, 0.f};
  unsigned char rgb[3] = {0, 0, 0};
  if (hit) {
    RayCell s;
    rc_cell(sv.dim, r.o, r.d, z_hit, corners, s);
    rc_normal(s, nrm);
    int vi[3];
    rc_color_voxel(sv.dim, r, z_hit, vi);
    const long long g[3] = {sv.k0[0] + vi[0], sv.k0[1] + vi[1], sv.k0[2] + vi[2]};
    rc_rgb(sv_voxel(sv, sv.color, g, 0.f), rgb);
  }
  p.depth[pix] = z_hit;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    p.normals[pix * 3 + c] = nrm[c];
    p.colors[pix * 3 + c] = rgb[c];
  }
}

static int view_check(const unsigned long long* keys, const int* slots, int table_size, const int* block_coords, int capacity,
                      const int* counters, const long long* box_lo_host, int dim_x, int dim_y, int dim_z, const char* what) {
  DVMVS_REQUIRE(keys && slots && block_coords && counters && box_lo_host, "%s: null argument", what);
  DVMVS_REQUIRE(capacity > 0 && table_size >= capacity && table_size <= (1 << 30) && (table_size & (table_size - 1)) == 0,
                "%s: capacity %d, table size %d (a power of two >= capacity, <= 2^30)", what, capacity, table_size);
  DVMVS_REQUIRE(dim_x >= 0 && dim_y >= 0 && dim_z >= 0, "%s: bad box %d x %d x %d", what, dim_x, dim_y, dim_z);
  DVMVS_REQUIRE((double)dim_x * dim_y * dim_z < (double)kMaxBoxVoxels, "%s: box of %d x %d x %d voxels exceeds 2^61", what, dim_x, dim_y, dim_z);
  for (int a = 0; a < 3; ++a)
    DVMVS_REQUIRE(box_lo_host[a] > -(1ll << 40) && box_lo_host[a] < (1ll << 40), "%s: box corner %lld out of range", what, box_lo_host[a]);
  return DVMVS_OK;
}

static SparseView make_view(const unsigned long long* keys, const int* slots, int table_size, const int* block_coords, int capacity,
                            const int* counters, const float* tsdf, const float* color, const long long* box_lo_host, int dim_x, int dim_y,
                            int dim_z) {
  SparseView v;
  v.keys = keys; v.slots = slots; v.coords = block_coords; v.counters = counters; v.tsdf = tsdf; v.color = color;
  v.mask = table_size - 1; v.capacity = capacity;
  for (int a = 0; a < 3; ++a) v.k0[a] = box_lo_host[a];
  v.dim[0] = dim_x; v.dim[1] = dim_y; v.dim[2] = dim_z;
  return v;
}

inline int view_grid() { return device_sm_count() * 8; }

static int cuda_rc(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return DVMVS_OK;
  set_error("%s: %s", what, cudaGetErrorString(e));
  return DVMVS_ELAUNCH;
}

}  // namespace dvmvs

using namespace dvmvs;

extern "C" int dvmvs_tsdf_sparse_mesh_scratch_bytes(int n_blocks, long long* bytes_host) {
  DVMVS_REQUIRE(bytes_host, "tsdf_sparse_mesh_scratch_bytes: null argument");
  DVMVS_REQUIRE(n_blocks >= 0 && n_blocks < kMaxViewBlocks, "tsdf_sparse_mesh_scratch_bytes: %d blocks (0 .. 2^22 - 1)", n_blocks);
  MeshScratch m;
  const int rc = mesh_scratch(n_blocks, nullptr, m);
  if (rc) return rc;
  *bytes_host = m.bytes;
  return DVMVS_OK;
}

extern "C" int dvmvs_tsdf_sparse_mesh_count(const unsigned long long* keys, const int* slots, int table_size, const int* block_coords, int capacity,
                                            const int* counters, const float* tsdf, int n_blocks, const long long* box_lo_host, int dim_x,
                                            int dim_y, int dim_z, void* scratch, long long scratch_bytes, dvmvs_stream_t stream) {
  int rc = view_check(keys, slots, table_size, block_coords, capacity, counters, box_lo_host, dim_x, dim_y, dim_z, "tsdf_sparse_mesh_count");
  if (rc) return rc;
  DVMVS_REQUIRE(tsdf && scratch, "tsdf_sparse_mesh_count: null argument");
  DVMVS_REQUIRE(n_blocks >= 0 && n_blocks < kMaxViewBlocks, "tsdf_sparse_mesh_count: %d blocks (0 .. 2^22 - 1)", n_blocks);
  MeshScratch m;
  if ((rc = mesh_scratch(n_blocks, scratch, m))) return rc;
  DVMVS_REQUIRE(scratch_bytes >= m.bytes && (uintptr_t)scratch % 256 == 0, "tsdf_sparse_mesh_count: scratch of %lld bytes at %p, %lld 256-byte aligned needed",
                scratch_bytes, scratch, m.bytes);
  cudaStream_t s = (cudaStream_t)stream;
  if ((rc = cuda_rc(cudaMemsetAsync(m.totals, 0, 64, s), "tsdf_sparse_mesh_count"))) return rc;
  if (n_blocks == 0 || dim_x < 2 || dim_y < 2 || dim_z < 2) return DVMVS_OK;    // no cube: an empty mesh, as mesh.cu
  const SparseView v = make_view(keys, slots, table_size, block_coords, capacity, counters, tsdf, nullptr, box_lo_host, dim_x, dim_y, dim_z);
  const int W = 8 * n_blocks, grid = view_grid();
  launch_k(mesh_work_kernel, dim3(grid), dim3(kViewThreads), 0, s, v, n_blocks, m.work, m.work_count);
  if ((rc = check_launch("mesh_work_kernel"))) return rc;
  launch_k(mesh_key_kernel, dim3(grid), dim3(kViewThreads), 0, s, v, W, (const WorkBlock*)m.work, (const int*)m.work_count, m.sort_keys, m.sort_vals);
  if ((rc = check_launch("mesh_key_kernel"))) return rc;
  size_t cub_bytes = m.cub_bytes;
  if ((rc = cuda_rc(cub::DeviceRadixSort::SortPairs(m.cub_temp, cub_bytes, m.sort_keys, m.sort_keys + W, m.sort_vals, m.sort_vals + W, W, 0, 64, s),
                    "tsdf_sparse_mesh_count: sort")))
    return rc;
  launch_k(mesh_block_kernel, dim3(grid), dim3(kViewThreads), 0, s, v, (const WorkBlock*)m.work, (const int*)m.work_count,
           (const int*)(m.sort_vals + W), m.blocks);
  if ((rc = check_launch("mesh_block_kernel"))) return rc;
  launch_k(mesh_sparse_count_kernel, dim3(grid), dim3(kViewThreads), 0, s, v, W, (const int*)m.work_count, (const ZBlock*)m.blocks, m.counts);
  if ((rc = check_launch("mesh_sparse_count_kernel"))) return rc;
  cub_bytes = m.cub_bytes;
  if ((rc = cuda_rc(cub::DeviceScan::ExclusiveScan(m.cub_temp, cub_bytes, m.counts, m.counts, AddPair(), make_longlong2(0, 0), 64 * W + 1, s),
                    "tsdf_sparse_mesh_count: scan")))
    return rc;
  return cuda_rc(cudaMemcpyAsync(m.totals, m.counts + 64ll * W, sizeof(longlong2), cudaMemcpyDeviceToDevice, s), "tsdf_sparse_mesh_count");
}

extern "C" int dvmvs_tsdf_sparse_mesh_extract(const unsigned long long* keys, const int* slots, int table_size, const int* block_coords,
                                              int capacity, const int* counters, const float* tsdf, const float* color, int n_blocks,
                                              const long long* box_lo_host, int dim_x, int dim_y, int dim_z, const float* vol_origin_host,
                                              float voxel_size, const void* scratch, long long scratch_bytes, int n_verts, int n_faces,
                                              long long* edge_keys, float* verts, int* faces, float* norms, unsigned char* colors,
                                              dvmvs_stream_t stream) {
  int rc = view_check(keys, slots, table_size, block_coords, capacity, counters, box_lo_host, dim_x, dim_y, dim_z, "tsdf_sparse_mesh_extract");
  if (rc) return rc;
  DVMVS_REQUIRE(tsdf && color && vol_origin_host && scratch, "tsdf_sparse_mesh_extract: null argument");
  DVMVS_REQUIRE(n_blocks >= 0 && n_blocks < kMaxViewBlocks, "tsdf_sparse_mesh_extract: %d blocks (0 .. 2^22 - 1)", n_blocks);
  MeshScratch m;
  if ((rc = mesh_scratch(n_blocks, (void*)scratch, m))) return rc;
  DVMVS_REQUIRE(scratch_bytes >= m.bytes && (uintptr_t)scratch % 256 == 0, "tsdf_sparse_mesh_extract: scratch of %lld bytes at %p, %lld 256-byte aligned needed",
                scratch_bytes, scratch, m.bytes);
  DVMVS_REQUIRE(n_verts >= 0 && n_faces >= 0 && 3ll * n_faces <= INT_MAX, "tsdf_sparse_mesh_extract: mesh of %d vertices, %d faces", n_verts, n_faces);
  if (n_verts == 0 && n_faces == 0) return DVMVS_OK;
  DVMVS_REQUIRE(n_blocks > 0 && dim_x >= 2 && dim_y >= 2 && dim_z >= 2, "tsdf_sparse_mesh_extract: a box with a dimension < 2 or no block has an empty mesh");
  DVMVS_REQUIRE(edge_keys && verts && norms && colors && (faces || n_faces == 0), "tsdf_sparse_mesh_extract: null output");
  SparseEmit p;
  p.v = make_view(keys, slots, table_size, block_coords, capacity, counters, tsdf, color, box_lo_host, dim_x, dim_y, dim_z);
  p.blocks = m.blocks;
  p.work_count = m.work_count;
  p.offsets = m.counts;
  for (int c = 0; c < 3; ++c) p.origin[c] = vol_origin_host[c];
  p.voxel = voxel_size;
  p.vertex_keys = edge_keys;
  p.face_keys = edge_keys + n_verts;
  p.verts = verts;
  p.norms = norms;
  p.colors = colors;
  cudaStream_t s = (cudaStream_t)stream;
  launch_k(mesh_sparse_emit_kernel, dim3(view_grid()), dim3(kViewThreads), 0, s, p, 8 * n_blocks);
  if ((rc = check_launch("mesh_sparse_emit_kernel")) || n_faces == 0) return rc;
  const long long n_idx = 3ll * n_faces;
  launch_k(mesh_sparse_resolve_kernel, dim3((unsigned)((n_idx + 255) / 256)), dim3(256), 0, s, (const long long*)p.face_keys, n_idx,
           (const long long*)edge_keys, n_verts, faces);
  return check_launch("mesh_sparse_resolve_kernel");
}

extern "C" int dvmvs_tsdf_sparse_raycast(const unsigned long long* keys, const int* slots, int table_size, const int* block_coords, int capacity,
                                         const int* counters, const float* tsdf, const float* color, const long long* box_lo_host, int dim_x,
                                         int dim_y, int dim_z, const float* vol_origin3, double voxel_size, double trunc_margin,
                                         const float* views, int n_views, int im_h, int im_w, float* depth, float* normals,
                                         unsigned char* colors, dvmvs_stream_t stream) {
  int rc = view_check(keys, slots, table_size, block_coords, capacity, counters, box_lo_host, dim_x, dim_y, dim_z, "tsdf_sparse_raycast");
  if (rc) return rc;
  DVMVS_REQUIRE(tsdf && color && vol_origin3 && views && depth && normals && colors, "tsdf_sparse_raycast: null argument");
  DVMVS_REQUIRE(dim_x > 0 && dim_y > 0 && dim_z > 0 && im_h > 0 && im_w > 0 && n_views > 0,
                "tsdf_sparse_raycast: bad extent: box %d x %d x %d, %d views of %d x %d", dim_x, dim_y, dim_z, n_views, im_h, im_w);
  DVMVS_REQUIRE((long long)n_views * im_h * im_w <= (long long)INT_MAX, "tsdf_sparse_raycast: %d views of %d x %d pixels exceed int32",
                n_views, im_h, im_w);
  DVMVS_REQUIRE(voxel_size > 0.0 && isfinite(voxel_size) && (float)voxel_size > 0.f, "tsdf_sparse_raycast: bad voxel size %g", voxel_size);
  SparseRaycast p;
  p.v = make_view(keys, slots, table_size, block_coords, capacity, counters, tsdf, color, box_lo_host, dim_x, dim_y, dim_z);
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
    launch_k(sparse_raycast_kernel, dim3((unsigned)tiles, (unsigned)nv), dim3(kRayTileW * kRayTileH), 0, s, p);
    if ((rc = check_launch("sparse_raycast_kernel"))) return rc;
  }
  return DVMVS_OK;
}
