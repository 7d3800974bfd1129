// Shared helpers for libdvmvs_sm90.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/dvmvs_b200.h"

namespace dvmvs {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

// Checks the launch that was just enqueued (no synchronisation).
inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return DVMVS_ELAUNCH;
  }
  count_launch();
  return DVMVS_OK;
}

// ---- programmatic dependent launch (PDL): every kernel of the library is launched with the programmatic-stream-
// serialization attribute, calls pdl_launch_dependents() first thing (the next kernel's CTAs may be scheduled as soon
// as all of ours are resident) and pdl_wait() before its first access to global memory (blocks until the preceding
// grid has completed and flushed).  Launch latency and per-kernel prologues (barrier init, tensor-map
// prefetch) thereby overlap the predecessor's tail; also inside captured CUDA graphs.  DVMVS_PDL=0 disables it.
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// same, with the grid's z dimension grouped into thread-block clusters of `cluster_z` CTAs (distributed shared memory)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, unsigned cluster_z,
                                    Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = cluster_z;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// One-time per-DEVICE initialisation guard (function attributes such as the >48 KB dynamic shared-memory opt-in are per
// device): returns true exactly once per (call site, current device); thread-safe.
struct PerDeviceOnce {
  std::atomic<unsigned long long> done{0};          // bit i: device i initialised (devices >= 64 re-run the init every time)
  bool first() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
    const unsigned long long bit = 1ull << dev;
    return (done.fetch_or(bit) & bit) == 0;
  }
};

// SM count of the current device, cached per device (grid sizing of persistent kernels and of split-K decisions)
inline int device_sm_count() {
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  int n = cache[dev].load();
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev].store(n);
  }
  return n;
}

#ifdef __CUDACC__
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

#define DVMVS_REQUIRE(cond, ...)        \
  do {                                  \
    if (!(cond)) {                      \
      ::dvmvs::set_error(__VA_ARGS__);  \
      return DVMVS_EINVAL;              \
    }                                   \
  } while (0)

#ifdef __CUDACC__
// x2 bilinear blend (align_corners upsampling) of the four taps with weights ly0/ly1 (rows) and lx0/lx1 (columns).  Every copy of
// the interpolation (upsample2x_kernel, the fused upsampled conv source, the split / staging kernels) calls this one function, with
// the roundings spelled out, so that all of them produce the same fp32 value bit for bit whatever the compiler would contract.
__device__ __forceinline__ float bilerp(float ly0, float ly1, float lx0, float lx1, float v00, float v01, float v10, float v11) {
  const float top = __fmaf_rn(lx1, v01, __fmul_rn(lx0, v00));
  const float bot = __fmaf_rn(lx0, v10, __fmul_rn(lx1, v11));
  return __fmaf_rn(ly0, top, __fmul_rn(ly1, bot));
}
#endif

// ---- tiny fp32 linear algebra used by the geometry prologues (device) ---------------------------------
// Row-major.  The reference does this algebra with torch.inverse / bmm in fp32 on the device
// (dvmvs/utils.py:51-57,121; dvmvs/convlstm.py:30); any fp32 method agrees to ~1e-7 for rigid poses.
__host__ __device__ __forceinline__ void mat4_rigid_free_inverse(const float* m, float* inv) {
  // general 4x4 inverse by cofactors, evaluated in double to stay at least as accurate as LU in fp32
  double a[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) a[i] = (double)m[i];
  double c[16];
  c[0] = a[5] * a[10] * a[15] - a[5] * a[11] * a[14] - a[9] * a[6] * a[15] + a[9] * a[7] * a[14] + a[13] * a[6] * a[11] - a[13] * a[7] * a[10];
  c[4] = -a[4] * a[10] * a[15] + a[4] * a[11] * a[14] + a[8] * a[6] * a[15] - a[8] * a[7] * a[14] - a[12] * a[6] * a[11] + a[12] * a[7] * a[10];
  c[8] = a[4] * a[9] * a[15] - a[4] * a[11] * a[13] - a[8] * a[5] * a[15] + a[8] * a[7] * a[13] + a[12] * a[5] * a[11] - a[12] * a[7] * a[9];
  c[12] = -a[4] * a[9] * a[14] + a[4] * a[10] * a[13] + a[8] * a[5] * a[14] - a[8] * a[6] * a[13] - a[12] * a[5] * a[10] + a[12] * a[6] * a[9];
  c[1] = -a[1] * a[10] * a[15] + a[1] * a[11] * a[14] + a[9] * a[2] * a[15] - a[9] * a[3] * a[14] - a[13] * a[2] * a[11] + a[13] * a[3] * a[10];
  c[5] = a[0] * a[10] * a[15] - a[0] * a[11] * a[14] - a[8] * a[2] * a[15] + a[8] * a[3] * a[14] + a[12] * a[2] * a[11] - a[12] * a[3] * a[10];
  c[9] = -a[0] * a[9] * a[15] + a[0] * a[11] * a[13] + a[8] * a[1] * a[15] - a[8] * a[3] * a[13] - a[12] * a[1] * a[11] + a[12] * a[3] * a[9];
  c[13] = a[0] * a[9] * a[14] - a[0] * a[10] * a[13] - a[8] * a[1] * a[14] + a[8] * a[2] * a[13] + a[12] * a[1] * a[10] - a[12] * a[2] * a[9];
  c[2] = a[1] * a[6] * a[15] - a[1] * a[7] * a[14] - a[5] * a[2] * a[15] + a[5] * a[3] * a[14] + a[13] * a[2] * a[7] - a[13] * a[3] * a[6];
  c[6] = -a[0] * a[6] * a[15] + a[0] * a[7] * a[14] + a[4] * a[2] * a[15] - a[4] * a[3] * a[14] - a[12] * a[2] * a[7] + a[12] * a[3] * a[6];
  c[10] = a[0] * a[5] * a[15] - a[0] * a[7] * a[13] - a[4] * a[1] * a[15] + a[4] * a[3] * a[13] + a[12] * a[1] * a[7] - a[12] * a[3] * a[5];
  c[14] = -a[0] * a[5] * a[14] + a[0] * a[6] * a[13] + a[4] * a[1] * a[14] - a[4] * a[2] * a[13] - a[12] * a[1] * a[6] + a[12] * a[2] * a[5];
  c[3] = -a[1] * a[6] * a[11] + a[1] * a[7] * a[10] + a[5] * a[2] * a[11] - a[5] * a[3] * a[10] - a[9] * a[2] * a[7] + a[9] * a[3] * a[6];
  c[7] = a[0] * a[6] * a[11] - a[0] * a[7] * a[10] - a[4] * a[2] * a[11] + a[4] * a[3] * a[10] + a[8] * a[2] * a[7] - a[8] * a[3] * a[6];
  c[11] = -a[0] * a[5] * a[11] + a[0] * a[7] * a[9] + a[4] * a[1] * a[11] - a[4] * a[3] * a[9] - a[8] * a[1] * a[7] + a[8] * a[3] * a[5];
  c[15] = a[0] * a[5] * a[10] - a[0] * a[6] * a[9] - a[4] * a[1] * a[10] + a[4] * a[2] * a[9] + a[8] * a[1] * a[6] - a[8] * a[2] * a[5];
  double det = a[0] * c[0] + a[1] * c[4] + a[2] * c[8] + a[3] * c[12];
  double r = 1.0 / det;
#pragma unroll
  for (int i = 0; i < 16; ++i) inv[i] = (float)(c[i] * r);
}

__host__ __device__ __forceinline__ void mat4_mul(const float* a, const float* b, float* o) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) s = fmaf(a[i * 4 + k], b[k * 4 + j], s);
      o[i * 4 + j] = s;
    }
}

__host__ __device__ __forceinline__ void mat3_inverse(const float* m, float* inv) {
  double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
  double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
  double r = 1.0 / (a * A + b * B + c * C);
  inv[0] = (float)(A * r);
  inv[1] = (float)(-(b * i - c * h) * r);
  inv[2] = (float)((b * f - c * e) * r);
  inv[3] = (float)(B * r);
  inv[4] = (float)((a * i - c * g) * r);
  inv[5] = (float)(-(a * f - c * d) * r);
  inv[6] = (float)(C * r);
  inv[7] = (float)(-(a * h - b * g) * r);
  inv[8] = (float)((a * e - b * d) * r);
}

__host__ __device__ __forceinline__ void mat3_mul(const float* a, const float* b, float* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < 3; ++k) s = fmaf(a[i * 3 + k], b[k * 3 + j], s);
      o[i * 3 + j] = s;
    }
}

}  // namespace dvmvs
