// Marching cubes on the TSDF volume -- the mesh / point-cloud step of the reference's sample-data/run-tsdf-reconstruction.py
// (`get_mesh` :344-358, `get_point_cloud` :329-342), which hands the volume to scikit-image there.  The triangulation contract
// (inside = tsdf < 0, sign-only face resolution, one vertex per crossing grid edge, generated tables) is stated in
// tools/gen_mc_tables.py; oracle/mesh_oracle.py restates this file in numpy and tests/test_mesh.py compares with array_equal.
// Everything that rounds is an explicit _rn intrinsic (no multiply-add contraction), as in csrc/tsdf.cu:
//   t      = -a / (b - a)                      a = tsdf at the edge's lower-index endpoint
//   vertex = f32(i) + t along the edge's axis  (index space; output axes are the volume's axes)
//   world  = f32( f32(vertex * voxel_size) + origin )
//   normal = np.gradient (central inside, one-sided at the border) at both endpoints, g_a + t (g_b - g_a), divided by
//            sqrt((x x + y y) + z z); (0, 0, 0) where that length is not positive.  Points toward increasing tsdf.
//   colour = the reference's unfold of the colour voxel at rint(vertex) (half-even, as np.round)
//
// Three passes, deterministic by construction (no atomics decide a position):
//   count   a CTA owns kMcThreads consecutive voxels in C order (one per thread): it classifies the cube whose lowest corner
//           is the voxel and the voxel's +x / +y / +z grid edges, and reduces (vertices, faces) to one pair per CTA.  Reads
//           only the tsdf volume; the 8 corner loads of a warp are 4 pairs of contiguous runs, all but the first L2 hits.
//   scan    exclusive scan of the per-CTA pairs, kScanBlock per CTA, recursing on the block sums (any number of CTAs).
//   emit    recomputes the classification, scans the CTA's voxels once more in shared memory for their global slots and
//           writes vertices (world, normal, colour, edge key) in key order and faces as edge keys; resolve then turns each
//           face key into its vertex id by binary search in the sorted key array (vertices owned by other CTAs; no scratch
//           of volume size).
// Vertices come out sorted by key 3 * (linear index of the lower voxel) + axis, faces by cube, then table order.
// Bound: HBM on the classification read (4 B per voxel, twice: count and emit), then the mesh written.
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "mc_tables.cuh"
#include "mc_vertex.cuh"

namespace dvmvs {

constexpr int kMcThreads = 256;    // voxels per CTA of the count and emit passes
constexpr int kScanBlock = 256;    // per-CTA pairs per CTA of the scan

struct MeshGrid {
  int dx, dy, dz, n, sx;           // sx = dy * dz (stride of axis 0); axis 1 stride is dz
};

struct VoxelClass {
  int lin, x, y, z;
  int cube_case;                   // 0 where the voxel is not the lowest corner of a cube
  unsigned edges;                  // bit a: the voxel's +a grid edge crosses
  float f0, fe[3];                 // tsdf at the voxel and at its +x / +y / +z neighbours
};

__device__ __forceinline__ int mc_corner_offset(const MeshGrid& g, int c) {
  return (c & 1) * g.sx + ((c >> 1) & 1) * g.dz + ((c >> 2) & 1);
}

__device__ __forceinline__ VoxelClass mc_classify(const float* __restrict__ tsdf, const MeshGrid& g, int lin) {
  VoxelClass v;
  v.lin = lin;
  v.x = (int)((unsigned)lin / (unsigned)g.sx);
  const int rem = lin - v.x * g.sx;
  v.y = (int)((unsigned)rem / (unsigned)g.dz);
  v.z = rem - v.y * g.dz;
  const bool has[3] = {v.x + 1 < g.dx, v.y + 1 < g.dy, v.z + 1 < g.dz};
  const int step[3] = {g.sx, g.dz, 1};
  v.f0 = tsdf[lin];
  v.edges = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    v.fe[a] = has[a] ? tsdf[lin + step[a]] : 1.f;
    if (has[a] && mc_inside(v.f0) != mc_inside(v.fe[a])) v.edges |= 1u << a;
  }
  v.cube_case = 0;
  if (has[0] && has[1] && has[2]) {
    int cs = (mc_inside(v.f0) ? 1 : 0) | (mc_inside(v.fe[0]) ? 2 : 0) | (mc_inside(v.fe[1]) ? 4 : 0) | (mc_inside(v.fe[2]) ? 16 : 0);
    const int rest[4] = {3, 5, 6, 7};
#pragma unroll
    for (int k = 0; k < 4; ++k) cs |= mc_inside(tsdf[lin + mc_corner_offset(g, rest[k])]) ? (1 << rest[k]) : 0;
    v.cube_case = cs;
  }
  return v;
}

// (vertices | faces << 16) of one voxel; a CTA's sums stay below 2^16 vertices (3 per voxel) and 2^16 faces
__device__ __forceinline__ unsigned mc_packed_counts(const VoxelClass& v) {
  return (unsigned)__popc(v.edges) | ((unsigned)kMcNumTris[v.cube_case] << 16);
}

// inclusive scan over the CTA (blockDim.x a multiple of 32, at most 1024); `warp_sums` holds 32 elements
template <typename T>
__device__ __forceinline__ T block_inclusive_scan(T v, T* warp_sums) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) warp_sums[warp] = v;
  __syncthreads();
  if (warp == 0) {
    T w = lane < n_warps ? warp_sums[lane] : T(0);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T u = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += u;
    }
    if (lane < n_warps) warp_sums[lane] = w;
  }
  __syncthreads();
  return warp > 0 ? v + warp_sums[warp - 1] : v;
}

__global__ void __launch_bounds__(kMcThreads) mesh_count_kernel(const float* __restrict__ tsdf, MeshGrid g, int2* __restrict__ counts) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned warp_sums[32];
  const int lin = blockIdx.x * kMcThreads + threadIdx.x;
  const unsigned packed = lin < g.n ? mc_packed_counts(mc_classify(tsdf, g, lin)) : 0u;
  const unsigned total = block_inclusive_scan(packed, warp_sums);
  if (threadIdx.x == kMcThreads - 1) counts[blockIdx.x] = make_int2((int)(total & 0xffffu), (int)(total >> 16));
}

// exclusive scan of data[0, n) in place, CTA by CTA; each CTA's total goes to sums[blockIdx.x].  The two counts travel as
// one 64-bit integer (vertices low, faces high): every total is below 2^31, so the low half never carries.
__global__ void __launch_bounds__(kScanBlock) mesh_scan_kernel(int2* __restrict__ data, int n, int2* __restrict__ sums) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned long long warp_sums[32];
  const int i = blockIdx.x * kScanBlock + threadIdx.x;
  const int2 d = i < n ? data[i] : make_int2(0, 0);
  const unsigned long long v = (unsigned long long)(unsigned)d.x | ((unsigned long long)(unsigned)d.y << 32);
  const unsigned long long incl = block_inclusive_scan(v, warp_sums);
  const unsigned long long excl = incl - v;
  if (i < n) data[i] = make_int2((int)(unsigned)(excl & 0xffffffffull), (int)(unsigned)(excl >> 32));
  if (threadIdx.x == kScanBlock - 1) sums[blockIdx.x] = make_int2((int)(unsigned)(incl & 0xffffffffull), (int)(unsigned)(incl >> 32));
}

__global__ void __launch_bounds__(kScanBlock) mesh_scan_add_kernel(int2* __restrict__ data, int n, const int2* __restrict__ offsets) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * kScanBlock + threadIdx.x;
  if (i < n) {
    const int2 o = offsets[blockIdx.x];
    const int2 d = data[i];
    data[i] = make_int2(d.x + o.x, d.y + o.y);
  }
}

struct MeshEmitParams {
  const float* tsdf;
  const float* color;
  const int2* offsets;             // per-CTA exclusive (vertex, face) offsets: the scanned counts
  MeshGrid g;
  float origin[3];
  float voxel;
  int* keys;                       // [V] edge key of each vertex
  float* verts;                    // [V][3]
  float* norms;                    // [V][3]
  unsigned char* colors;           // [V][3]
  int* faces;                      // [F][3], edge keys until mesh_resolve_kernel
};

__device__ __forceinline__ void mc_gradient(const MeshEmitParams& p, int x, int y, int z, float* gr) {
  const int q[3] = {x, y, z}, dim[3] = {p.g.dx, p.g.dy, p.g.dz}, step[3] = {p.g.sx, p.g.dz, 1};
  const int lin = x * p.g.sx + y * p.g.dz + z;
  mc_np_gradient(q, dim, [&](int a, int s) { return p.tsdf[lin + s * step[a]]; }, gr);
}

__device__ __forceinline__ void mc_emit_vertex(const MeshEmitParams& p, const VoxelClass& v, int axis, int slot) {
  const int q[3] = {v.x, v.y, v.z};
  const McVertex m = mc_vertex(v.f0, v.fe[axis], q, axis, [&](int x, int y, int z, float* gr) { mc_gradient(p, x, y, z, gr); },
                               [&](int ix, int iy, int iz) { return p.color[(size_t)ix * p.g.sx + (size_t)iy * p.g.dz + iz]; }, p.origin,
                               p.voxel);
  const size_t o = (size_t)slot * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    p.verts[o + c] = m.vert[c];
    p.norms[o + c] = m.norm[c];
    p.colors[o + c] = m.rgb[c];
  }
  p.keys[slot] = 3 * v.lin + axis;
}

__global__ void __launch_bounds__(kMcThreads) mesh_emit_kernel(MeshEmitParams p) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned warp_sums[32];
  const int lin = blockIdx.x * kMcThreads + threadIdx.x;
  VoxelClass v;
  unsigned packed = 0u;
  if (lin < p.g.n) {
    v = mc_classify(p.tsdf, p.g, lin);
    packed = mc_packed_counts(v);
  }
  const unsigned excl = block_inclusive_scan(packed, warp_sums) - packed;
  if (packed == 0u) return;
  const int2 base = p.offsets[blockIdx.x];
  int slot = base.x + (int)(excl & 0xffffu);
#pragma unroll
  for (int a = 0; a < 3; ++a)
    if (v.edges & (1u << a)) mc_emit_vertex(p, v, a, slot++);
  const int n_tris = kMcNumTris[v.cube_case];
  int* face = p.faces + (size_t)(base.y + (int)(excl >> 16)) * 3;
  for (int k = 0; k < n_tris * 3; ++k) {
    const int e = kMcTris[v.cube_case][k];
    face[k] = 3 * (lin + mc_corner_offset(p.g, kMcEdgeCorner[e][0])) + (e >> 2);
  }
}

// edge key -> vertex id: lower bound in the sorted key array (every face key is present by construction)
__global__ void __launch_bounds__(256) mesh_resolve_kernel(int* __restrict__ faces, long long n, const int* __restrict__ keys, int n_keys) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const int key = faces[i];
  int lo = 0, hi = n_keys;
  while (lo < hi) {
    const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
    if (__ldg(keys + mid) < key) lo = mid + 1;
    else hi = mid;
  }
  faces[i] = lo;
}

// scan levels: level 0 holds the per-CTA counts of the count pass, level k + 1 the block sums of level k, up to the first
// level that fits one scan CTA.  Scratch = the (vertices, faces) totals, then every level.
struct MeshLayout {
  int n_levels;
  long long size[8];
  long long offset[8];             // in int2 elements from the start of the scratch (element 0 = totals)
  long long total_elems;
};

static MeshLayout mesh_layout(long long n_voxels) {
  MeshLayout L = {};
  long long n = (n_voxels + kMcThreads - 1) / kMcThreads, off = 1;
  for (;;) {
    L.size[L.n_levels] = n;
    L.offset[L.n_levels] = off;
    off += n;
    ++L.n_levels;
    if (n <= kScanBlock) break;
    n = (n + kScanBlock - 1) / kScanBlock;
  }
  L.total_elems = off;
  return L;
}

static int mesh_check_dims(int dim_x, int dim_y, int dim_z, const char* what) {
  DVMVS_REQUIRE(dim_x >= 0 && dim_y >= 0 && dim_z >= 0, "%s: bad extent %d x %d x %d", what, dim_x, dim_y, dim_z);
  const long long n = (long long)dim_x * dim_y * dim_z;
  // faces per cube <= kMcMaxTris and vertex keys < 3 n: both fit the int32 counts, keys and face ids
  DVMVS_REQUIRE(n * kMcMaxTris <= (long long)INT_MAX, "%s: volume of %lld voxels exceeds the int32 mesh indices (at most %lld voxels)",
                what, n, (long long)INT_MAX / kMcMaxTris);
  return DVMVS_OK;
}

static bool mesh_is_empty(int dim_x, int dim_y, int dim_z) { return dim_x < 2 || dim_y < 2 || dim_z < 2; }

}  // namespace dvmvs

using namespace dvmvs;

extern "C" int dvmvs_mesh_scratch_bytes(int dim_x, int dim_y, int dim_z, long long* bytes_host) {
  DVMVS_REQUIRE(bytes_host, "mesh_scratch_bytes: null argument");
  const int rc = mesh_check_dims(dim_x, dim_y, dim_z, "mesh_scratch_bytes");
  if (rc != DVMVS_OK) return rc;
  *bytes_host = mesh_layout((long long)dim_x * dim_y * dim_z).total_elems * (long long)sizeof(int2);
  return DVMVS_OK;
}

extern "C" int dvmvs_mesh_count(const float* tsdf_vol, int dim_x, int dim_y, int dim_z, void* scratch, long long scratch_bytes,
                                dvmvs_stream_t stream) {
  DVMVS_REQUIRE(tsdf_vol && scratch, "mesh_count: null argument");
  const int rc = mesh_check_dims(dim_x, dim_y, dim_z, "mesh_count");
  if (rc != DVMVS_OK) return rc;
  const MeshLayout L = mesh_layout((long long)dim_x * dim_y * dim_z);
  DVMVS_REQUIRE(scratch_bytes >= L.total_elems * (long long)sizeof(int2), "mesh_count: scratch of %lld bytes, needs %lld", scratch_bytes,
                L.total_elems * (long long)sizeof(int2));
  cudaStream_t s = (cudaStream_t)stream;
  int2* base = (int2*)scratch;
  if (mesh_is_empty(dim_x, dim_y, dim_z)) {              // no cube: an empty mesh (grid edges without faces are not emitted)
    const cudaError_t e = cudaMemsetAsync(base, 0, sizeof(int2), s);
    if (e != cudaSuccess) {
      set_error("mesh_count: %s", cudaGetErrorString(e));
      return DVMVS_ELAUNCH;
    }
    return DVMVS_OK;
  }
  const MeshGrid g = {dim_x, dim_y, dim_z, dim_x * dim_y * dim_z, dim_y * dim_z};
  launch_k(mesh_count_kernel, dim3((unsigned)L.size[0]), dim3(kMcThreads), 0, s, tsdf_vol, g, base + L.offset[0]);
  int err = check_launch("mesh_count_kernel");
  if (err) return err;
  for (int k = 0; k < L.n_levels; ++k) {                 // the last level is one CTA; its total is the mesh size
    int2* sums = k + 1 < L.n_levels ? base + L.offset[k + 1] : base;
    launch_k(mesh_scan_kernel, dim3((unsigned)((L.size[k] + kScanBlock - 1) / kScanBlock)), dim3(kScanBlock), 0, s, base + L.offset[k],
             (int)L.size[k], sums);
    if ((err = check_launch("mesh_scan_kernel"))) return err;
  }
  for (int k = L.n_levels - 2; k >= 0; --k) {
    launch_k(mesh_scan_add_kernel, dim3((unsigned)((L.size[k] + kScanBlock - 1) / kScanBlock)), dim3(kScanBlock), 0, s, base + L.offset[k],
             (int)L.size[k], (const int2*)(base + L.offset[k + 1]));
    if ((err = check_launch("mesh_scan_add_kernel"))) return err;
  }
  return DVMVS_OK;
}

extern "C" int dvmvs_mesh_extract(const float* tsdf_vol, const float* color_vol, int dim_x, int dim_y, int dim_z,
                                  const float* vol_origin_host, float voxel_size, const void* scratch, long long scratch_bytes,
                                  int n_verts, int n_faces, int* vertex_keys, float* verts, int* faces, float* norms,
                                  unsigned char* colors, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(tsdf_vol && color_vol && vol_origin_host && scratch, "mesh_extract: null argument");
  const int rc = mesh_check_dims(dim_x, dim_y, dim_z, "mesh_extract");
  if (rc != DVMVS_OK) return rc;
  const MeshLayout L = mesh_layout((long long)dim_x * dim_y * dim_z);
  DVMVS_REQUIRE(scratch_bytes >= L.total_elems * (long long)sizeof(int2), "mesh_extract: scratch of %lld bytes, needs %lld", scratch_bytes,
                L.total_elems * (long long)sizeof(int2));
  DVMVS_REQUIRE(n_verts >= 0 && n_faces >= 0, "mesh_extract: negative mesh size");
  if (n_verts == 0 && n_faces == 0) return DVMVS_OK;
  DVMVS_REQUIRE(!mesh_is_empty(dim_x, dim_y, dim_z), "mesh_extract: a volume with a dimension < 2 has an empty mesh");
  DVMVS_REQUIRE(vertex_keys && verts && norms && colors && (faces || n_faces == 0), "mesh_extract: null output");
  MeshEmitParams p;
  p.tsdf = tsdf_vol;
  p.color = color_vol;
  p.offsets = (const int2*)scratch + L.offset[0];
  p.g = {dim_x, dim_y, dim_z, dim_x * dim_y * dim_z, dim_y * dim_z};
  for (int c = 0; c < 3; ++c) p.origin[c] = vol_origin_host[c];
  p.voxel = voxel_size;
  p.keys = vertex_keys;
  p.verts = verts;
  p.norms = norms;
  p.colors = colors;
  p.faces = faces;
  cudaStream_t s = (cudaStream_t)stream;
  launch_k(mesh_emit_kernel, dim3((unsigned)L.size[0]), dim3(kMcThreads), 0, s, p);
  int err = check_launch("mesh_emit_kernel");
  if (err || n_faces == 0) return err;
  const long long n_idx = 3LL * n_faces;
  launch_k(mesh_resolve_kernel, dim3((unsigned)((n_idx + 255) / 256)), dim3(256), 0, s, faces, n_idx, (const int*)vertex_keys, n_verts);
  return check_launch("mesh_resolve_kernel");
}
