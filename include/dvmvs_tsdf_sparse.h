/*
 * dvmvs_tsdf_sparse.h -- C ABI of the voxel-block TSDF volume in libdvmvs_sm90.so (csrc/tsdf_sparse.cu; Python mirror
 * dvmvs.tsdf.SparseTSDFVolume).  Conventions, types and DVMVS_E* codes are those of dvmvs_b200.h: device pointers unless the
 * name ends in _host, 0 or a negative DVMVS_E* code, no device allocation, no synchronisation, work enqueued on `stream`.
 *
 * Extends TSDFVolume.integrate of the reference's sample-data/run-tsdf-reconstruction.py:220-323 (dvmvs_tsdf_integrate) to a
 * volume without bounds: 8 x 8 x 8-voxel blocks are allocated on the device the first time a frame can update one of their
 * voxels, found through a hash table, and only the blocks a frame sees are integrated.  Every voxel is updated by the same
 * arithmetic as dvmvs_tsdf_integrate, at world point f32(f64(origin) + voxel_size * f64(global index)) with signed global
 * indices, so the volume holds, voxel for voxel, what a dense volume with the same origin holds after the same frames.
 *
 * State of one volume (allocated by the caller; initial contents in brackets):
 *   keys        [table_size] uint64 block keys [all bits set = empty]; table_size a power of two >= capacity
 *   slots       [table_size] int32, pool slot of the key in the same entry (-1: the pool was full) [any]
 *   block_coords[capacity][3] int32 block coordinates of each pool slot (block = floor(global voxel index / 8)) [any]
 *   tsdf, weight, color [capacity][8][8][8] fp32 voxels of each pool slot, x-major as the dense volume [1 / 0 / 0]
 *   counters    [4] int32: keys inserted (= pool slots the frames so far need), error flags (DVMVS_SPARSE_*), blocks the last
 *               allocated frame sees, halt mode (include/dvmvs_tsdf_sparse_grow.h; 0 = off) [0 0 0 0]
 *   visible     [capacity] int32 pool slots the last allocated frame sees (its first counters[2] entries) [any]
 * A flag never clears (only dvmvs_tsdf_sparse_rehash of include/dvmvs_tsdf_sparse_grow.h clears the pool- and table-full flags
 * of a grown volume); a block the pool or the table had no room for is not integrated, and the flag says so.
 */
#ifndef DVMVS_TSDF_SPARSE_H
#define DVMVS_TSDF_SPARSE_H

#include "dvmvs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

enum {
  DVMVS_SPARSE_POOL_FULL = 1,     /* a block got no pool slot: capacity < counters[0] */
  DVMVS_SPARSE_TABLE_FULL = 2,    /* a block found no free hash entry */
  DVMVS_SPARSE_FRUSTUM = 4        /* a frame's view frustum, to its farthest depth, leaves the key range (+-2^20 blocks per
                                     axis) or spans more than 2^31 blocks: that frame allocated and integrated nothing */
};

/* HOST query: bytes of per-frame scratch dvmvs_tsdf_sparse_allocate needs for an im_h x im_w depth map (the frame's candidate
 * block box and its max-depth image of 16 x 16-pixel tiles). */
int dvmvs_tsdf_sparse_scratch_bytes(int im_h, int im_w, long long* bytes_host);

/* Allocation for one frame (extends run-tsdf-reconstruction.py:220-323 to a volume without bounds): every block holding a voxel
 * that projects into the image onto a pixel of depth > 0 with depth - z >= -trunc_margin (a voxel dvmvs_tsdf_integrate would
 * update) is inserted if new and listed in visible.  Candidates
 * are the blocks of the frame's view frustum up to its largest depth; each is kept unless float64 bounds on its voxels'
 * camera coordinates prove it behind the camera, outside the image, or farther than trunc_margin behind the largest depth of
 * the 16 x 16-pixel tiles it projects into.  Allocation is conservative: a voxel the reference updates is never missed.
 *   depth_im, im_h, im_w, depth_is_f64, intr4, world_to_cam16, vol_origin3, voxel_size, trunc_margin: as dvmvs_tsdf_integrate
 *   (intr4 fx, fy > 0 and finite; world_to_cam16's rotation part invertible)
 *   scratch     scratch_bytes bytes of device memory (dvmvs_tsdf_sparse_scratch_bytes), overwritten */
int dvmvs_tsdf_sparse_allocate(unsigned long long* keys, int* slots, int table_size, int* block_coords, int capacity, int* counters,
                               int* visible, void* scratch, long long scratch_bytes, const float* vol_origin3, double voxel_size,
                               double trunc_margin, const void* depth_im, int depth_is_f64, int im_h, int im_w, const float* intr4,
                               const double* world_to_cam16, dvmvs_stream_t stream);

/* Integration of one frame (run-tsdf-reconstruction.py:220-323) into the blocks the preceding dvmvs_tsdf_sparse_allocate of the
 * same frame listed: tsdf_update_voxel of dvmvs_tsdf_integrate on every voxel of those blocks.  Arguments as dvmvs_tsdf_integrate; updated_count optional. */
int dvmvs_tsdf_sparse_integrate(float* tsdf, float* weight, float* color, const int* block_coords, int capacity, const int* counters,
                                const int* visible, const float* vol_origin3, double voxel_size, double trunc_margin,
                                const void* color_im, int color_is_u8, const void* depth_im, int depth_is_f64, int im_h, int im_w,
                                const float* intr4, const double* world_to_cam16, double obs_weight, unsigned long long* updated_count,
                                dvmvs_stream_t stream);

/* Export into a dense box: the voxels of every allocated block inside the box are copied into tsdf_vol / weight_vol / color_vol
 * ([dim_x][dim_y][dim_z] fp32, C order, as dvmvs_tsdf_integrate's); the caller initialises the box to 1 / 0 / 0 (the reference's
 * initial state, :57-61), which unallocated voxels keep.  Dense voxel (i, j, k) is global voxel (i, j, k) + box_lo_host. */
int dvmvs_tsdf_sparse_export(const float* tsdf, const float* weight, const float* color, const int* block_coords, int capacity,
                             const int* counters, const int* box_lo_host, int dim_x, int dim_y, int dim_z, float* tsdf_vol,
                             float* weight_vol, float* color_vol, dvmvs_stream_t stream);

/* Bounds of the allocated blocks: bounds6 = min block x, y, z, then max block x, y, z (INT32_MAX x 3, INT32_MIN x 3 when none). */
int dvmvs_tsdf_sparse_block_bounds(const int* block_coords, int capacity, const int* counters, int* bounds6,
                                   dvmvs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DVMVS_TSDF_SPARSE_H */
