// Block keys and the hash table of the voxel-block TSDF volume (include/dvmvs_tsdf_sparse.h), shared by the allocation
// (tsdf_sparse.cu) and the mesh and ray-cast kernels that read the blocks (tsdf_sparse_view.cu): the key format and the probe
// sequence live here only.  The table is open addressing with linear probing from a multiplicative hash; an entry's key is
// kEmpty until inserted and never removed, so a probe sequence that reaches kEmpty proves the key absent.
#pragma once

namespace dvmvs {

constexpr int kBlock = 8;                            // voxels per block edge
constexpr int kBlockVoxels = kBlock * kBlock * kBlock;
constexpr int kKeyBits = 21;                         // per axis: block coordinates in [-2^20, 2^20)
constexpr int kKeyBias = 1 << (kKeyBits - 1);
constexpr unsigned long long kEmpty = ~0ull;         // bit 63 is never set in a key

__device__ __forceinline__ unsigned long long block_key(int bx, int by, int bz) {
  const unsigned long long m = (1ull << kKeyBits) - 1;
  return (((unsigned long long)(bx + kKeyBias) & m) << (2 * kKeyBits)) | (((unsigned long long)(by + kKeyBias) & m) << kKeyBits) |
         ((unsigned long long)(bz + kKeyBias) & m);
}

// first table entry of the key's probe sequence; the sequence continues h + 1, h + 2, ... modulo the table size
__device__ __forceinline__ unsigned block_hash(unsigned long long key, int mask) {
  return (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 32) & (unsigned)mask;
}

__device__ __forceinline__ bool block_in_key_range(long long bx, long long by, long long bz) {
  return bx >= -kKeyBias && bx < kKeyBias && by >= -kKeyBias && by < kKeyBias && bz >= -kKeyBias && bz < kKeyBias;
}

// read-only lookup: the pool slot of block (bx, by, bz), or -1 when it is not allocated (or got no slot: the pool was full).
// Only after every allocation launch that could insert it has completed.
__device__ __forceinline__ int sparse_find(const unsigned long long* __restrict__ keys, const int* __restrict__ slots, int mask, long long bx,
                                           long long by, long long bz) {
  if (!block_in_key_range(bx, by, bz)) return -1;
  const unsigned long long key = block_key((int)bx, (int)by, (int)bz);
  unsigned h = block_hash(key, mask);
  for (int probe = 0; probe <= mask; ++probe, h = (h + 1) & (unsigned)mask) {
    const unsigned long long k = __ldg(keys + h);
    if (k == key) return __ldg(slots + h);
    if (k == kEmpty) return -1;
  }
  return -1;
}

}  // namespace dvmvs
