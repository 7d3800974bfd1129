// The reference's folded colour volume (run-tsdf-reconstruction.py:235-236, :311-323, :352-357): one float32 per voxel holding
// b * 65536 + g * 256 + r.  Shared by TSDF integration (csrc/tsdf.cu) and mesh extraction (csrc/mesh.cu).
#pragma once
#include <math.h>

namespace dvmvs {

// float32 unfold, as the reference's  b = floor(c / 65536); g = floor((c - b * 65536) / 256); r = c - b * 65536 - g * 256
__device__ __forceinline__ void unfold(float c, float& b, float& g, float& r) {
  b = floorf(__fdiv_rn(c, 65536.f));
  const float rest = __fsub_rn(c, __fmul_rn(b, 65536.f));
  g = floorf(__fdiv_rn(rest, 256.f));
  r = __fsub_rn(rest, __fmul_rn(g, 256.f));
}

}  // namespace dvmvs
