/*
 * dvmvs_tsdf_sparse_grow.h -- C ABI for growing the voxel-block TSDF volume of include/dvmvs_tsdf_sparse.h when its frames need
 * more blocks than its pool or hash table holds, in libdvmvs_sm90.so (csrc/tsdf_sparse.cu; Python mirror
 * dvmvs.tsdf.SparseTSDFVolume(max_capacity_blocks=...)).  Conventions, types and DVMVS_E* codes are those of dvmvs_b200.h:
 * device pointers unless the name ends in _host, 0 or a negative DVMVS_E* code, no device allocation, no synchronisation, work
 * enqueued on `stream`.
 *
 * Growth takes two pieces, both on the device:
 *   Halt mode.  With DVMVS_SPARSE_HALT_ON_FULL set in counters[3] and DVMVS_SPARSE_POOL_FULL or DVMVS_SPARSE_TABLE_FULL set in
 *     counters[1] when a frame starts, dvmvs_tsdf_sparse_allocate inserts nothing (it still sets counters[2] to 0) and
 *     dvmvs_tsdf_sparse_integrate touches no voxel and adds nothing to updated_count.  The frame that sets the flag
 *     finishes its own insertions, so counters[0] then counts every key the frames through it need, and its integration is
 *     skipped, so no voxel holds part of a frame.  With counters[3] = 0 (the volume's zero fill) both entry points behave as
 *     without this header.  DVMVS_SPARSE_FRUSTUM does not halt: that frame integrated nothing, and the next one runs.
 *   Rehash.  The caller allocates a larger pool, copies the old pool's slots 0 ... n_blocks-1 (block_coords and voxels) to the
 *     same slots of the new one, fills a new table with empty keys and calls dvmvs_tsdf_sparse_rehash; the frames from the
 *     one that set the flag are then allocated and integrated again, in order.  Keys the overflowing frame left with slot -1
 *     are not carried over: that frame's replay inserts them.
 */
#ifndef DVMVS_TSDF_SPARSE_GROW_H
#define DVMVS_TSDF_SPARSE_GROW_H

#include "dvmvs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

enum {
  DVMVS_SPARSE_HALT_ON_FULL = 1   /* counters[3] bit: a frame starting with a pool- or table-full flag allocates and integrates nothing */
};

/* Rebuilds the hash table of a volume from its pool: the key of every pool slot s in 0 ... n_blocks-1 (block_coords[s]) is
 * inserted into keys / slots (table_size entries, every key empty on entry) with slot s, by the block key and probe sequence
 * of dvmvs_tsdf_sparse_allocate.  Then counters[0] = n_blocks, DVMVS_SPARSE_POOL_FULL and DVMVS_SPARSE_TABLE_FULL are cleared
 * in counters[1] (DVMVS_SPARSE_FRUSTUM is kept) and counters[3] is left as it is.  table_size a power of two <= 2^30,
 * 0 <= n_blocks, 2 n_blocks <= table_size; the n_blocks blocks distinct. */
int dvmvs_tsdf_sparse_rehash(unsigned long long* keys, int* slots, int table_size, const int* block_coords, int n_blocks, int* counters,
                             dvmvs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DVMVS_TSDF_SPARSE_GROW_H */
