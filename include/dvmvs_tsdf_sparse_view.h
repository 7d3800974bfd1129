/*
 * dvmvs_tsdf_sparse_view.h -- C ABI of the mesh and the ray casting of the voxel-block TSDF volume, on its blocks, in
 * libdvmvs_sm90.so (csrc/tsdf_sparse_view.cu; Python mirror dvmvs.tsdf.SparseTSDFVolume.get_mesh_tensors / render_tensors).
 * Conventions, types and DVMVS_E* codes are those of dvmvs_b200.h: device pointers unless the name ends in _host, 0 or a
 * negative DVMVS_E* code, no device allocation, no synchronisation, work enqueued on `stream`.
 *
 * The volume's state is that of include/dvmvs_tsdf_sparse.h (keys, slots, table_size, block_coords, capacity, counters, tsdf,
 * color), read only, after every dvmvs_tsdf_sparse_allocate that fills it has been enqueued before.  The box: box voxel
 * (i, j, k) is global voxel box_lo_host + (i, j, k), 0 <= i < dim_x etc.  Over any box, each entry point computes bit for bit
 * what its dense counterpart (dvmvs_mesh_count / dvmvs_mesh_extract, dvmvs_tsdf_raycast) computes on the dense box
 * dvmvs_tsdf_sparse_export fills (voxels of blocks that are not allocated: tsdf 1, colour 0), without materialising it: the
 * scratch scales with the allocated blocks, never with the box's voxel count (at most 2^61 voxels).
 */
#ifndef DVMVS_TSDF_SPARSE_VIEW_H
#define DVMVS_TSDF_SPARSE_VIEW_H

#include "dvmvs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* HOST query: bytes of scratch the mesh of a volume with n_blocks allocated blocks (counters[0], 0 <= n_blocks < 2^22) needs.
 * Queries CUB's temporary-storage sizes: needs the CUDA runtime and a device. */
int dvmvs_tsdf_sparse_mesh_scratch_bytes(int n_blocks, long long* bytes_host);

/* Marching cubes, pass 1 (dvmvs_mesh_count on the exported box): lists the allocated blocks meeting the box and their missing
 * -x / -y / -z / diagonal neighbours, sorts them and counts the vertices and faces of every 8-voxel z-run in the dense mesh's
 * order, then scans the counts.  The first 16 bytes of scratch receive (int64 vertices, int64 faces) of the mesh, for the host
 * to read before dvmvs_tsdf_sparse_mesh_extract.  scratch: 256-byte aligned, dvmvs_tsdf_sparse_mesh_scratch_bytes(n_blocks). */
int dvmvs_tsdf_sparse_mesh_count(const unsigned long long* keys, const int* slots, int table_size, const int* block_coords, int capacity,
                                 const int* counters, const float* tsdf, int n_blocks, const long long* box_lo_host, int dim_x, int dim_y,
                                 int dim_z, void* scratch, long long scratch_bytes, dvmvs_stream_t stream);

/* Marching cubes, pass 2 (dvmvs_mesh_extract on the exported box; vol_origin_host and voxel_size as there): vertices, faces,
 * normals and colours in the dense mesh's order.  scratch as left by dvmvs_tsdf_sparse_mesh_count with the same volume, box and
 * n_blocks; n_verts, n_faces its totals (n_verts < 2^31, 3 n_faces < 2^31).  edge_keys: [n_verts + 3 n_faces] int64, scratch
 * of this call (the vertices' grid-edge keys, then the faces'). */
int dvmvs_tsdf_sparse_mesh_extract(const unsigned long long* keys, const int* slots, int table_size, const int* block_coords, int capacity,
                                   const int* counters, const float* tsdf, const float* color, int n_blocks, const long long* box_lo_host,
                                   int dim_x, int dim_y, int dim_z, const float* vol_origin_host, float voxel_size, const void* scratch,
                                   long long scratch_bytes, int n_verts, int n_faces, long long* edge_keys, float* verts, int* faces,
                                   float* norms, unsigned char* colors, dvmvs_stream_t stream);

/* Ray casting (dvmvs_tsdf_raycast on the exported box; vol_origin3 = the box's origin, every other argument as there): the
 * march's cell corners are fetched through the hash table.  No scratch. */
int dvmvs_tsdf_sparse_raycast(const unsigned long long* keys, const int* slots, int table_size, const int* block_coords, int capacity,
                              const int* counters, const float* tsdf, const float* color, const long long* box_lo_host, int dim_x, int dim_y,
                              int dim_z, const float* vol_origin3, double voxel_size, double trunc_margin, const float* views, int n_views,
                              int im_h, int im_w, float* depth, float* normals, unsigned char* colors, dvmvs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DVMVS_TSDF_SPARSE_VIEW_H */
