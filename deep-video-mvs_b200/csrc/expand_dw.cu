// MnasNet inverted-residual front half in one launch: 1x1 expansion on the tensor cores (wgmma) + BN bias + ReLU, then the
// k x k depthwise convolution + BN bias + ReLU, with the expanded activation kept in shared memory.  sm_90a only.
//
// The expanded tensor (3x or 6x the block's input channels) is the widest tensor of the trunk and is read exactly once, by
// the depthwise convolution.  Run as conv_tc_kernel + dwconv_kernel it goes to HBM as fp32 and comes back; here it never
// leaves the SM.  The depthwise filter is per channel, so the expanded channels split across CTAs without any reduction.
//
// One CTA = one output tile (tile_h x tile_w pixels of the depthwise output) x one slice of BLOCK_N expanded channels:
// * ONE TMA box per 32/64-channel K chunk loads the input halo ((tile_h - 1) * s + k) x ((tile_w - 1) * s + k) of the block
//   input's channel-last fp16 planes (the operand conv_tc_kernel reads); out-of-image pixels are zero-filled.  The box
//   lands as halo-pixel rows in the canonical K-major swizzled layout, so every 64 halo pixels are one wgmma m64 block.
//   The weight slice is BLOCK_N rows of the PackedConvTC matrix.
// * Two warpgroups take alternate m64 blocks.  Per block the MMAs run in conv_tc_kernel's order (K chunk, then term
//   hi*hi / lo*hi / hi*lo, then k16 step), so every expanded value is bit-identical to conv_tc_kernel's.  The epilogue adds
//   the bias and applies the activation in tc_emit8's order and stores fp32 [halo pixel][BLOCK_N + 4] in shared memory.
// * The depthwise pass reads that tile: accumulator = bias, fmaf over the in-image taps in (ky, kx) order, ReLU -- the
//   arithmetic of dwconv_kernel.  Out-of-image halo pixels hold ReLU(bias), not the reference's zero padding of the
//   expanded tensor, so their taps are skipped exactly as dwconv_kernel skips them.  Output: fp16 hi plane (and the lo plane
//   when the projection runs 3-term products) channel-last [2][B][Ho][Wo][mid], the projection's operand.
#include <string.h>

#include "tc_ptx.cuh"

namespace dvmvs {

constexpr int kEdThreads = 256;      // two MMA warpgroups; all eight warps run the depthwise pass
constexpr int kEdSmemBudget = 113 * 1024;   // two CTAs per SM

struct ExpandDwParams {
  CUtensorMap a_map[2];      // block input planes [hi/lo], box {kc, halo_w, halo_h, 1}
  CUtensorMap w_map[2];      // expansion weights [hi/lo], box {kc, BLOCK_N}
  int kc, n_chunks, terms, write_lo;
  int B, H, W, mid, Ho, Wo, stride, pad;
  int tile_h, tile_w, tiles_x, tiles_y, halo_h, halo_w, n_halo, m_blocks;
  const float* e_bias;
  int e_act;
  const float* dw_w;         // [k][k][mid]
  const float* dw_b;         // [mid]
  int dw_act;
  __half* out;               // [2][B][Ho][Wo][mid]
  int a_chunk_bytes, w_chunk_bytes, a_bytes, w_bytes, tile_off;   // smem layout: A [plane][chunk], W [plane][chunk], fp32 tile
};

// the MMAs of one m64 block over the whole K (chunks, then terms, then k16 steps -- conv_tc_kernel's order)
template <int BLOCK_N, int KSTEPS>
__device__ __forceinline__ void ed_mma_block(float (&acc)[BLOCK_N / 2], const ExpandDwParams& p, uint32_t a_base, uint32_t w_base, int mb) {
  constexpr uint32_t layout = (KSTEPS == 4) ? kGmmaSw128 : kGmmaSw64;
  constexpr uint32_t row_bytes = KSTEPS * 32u;
  constexpr uint32_t sbo = 8u * row_bytes;
  wgmma_fence_regs(acc);
  wgmma_fence();
  for (int ch = 0; ch < p.n_chunks; ++ch) {
    for (int term = 0; term < p.terms; ++term) {
      const uint32_t a_s = a_base + ((term == 1) ? p.a_bytes : 0u) + ch * p.a_chunk_bytes + mb * 64u * row_bytes;
      const uint32_t w_s = w_base + ((term == 2) ? p.w_bytes : 0u) + ch * p.w_chunk_bytes;
#pragma unroll
      for (int k = 0; k < KSTEPS; ++k)
        wgmma_f16<BLOCK_N>(acc, gmma_desc(a_s + 32u * k, 16u, sbo, layout), gmma_desc(w_s + 32u * k, 16u, sbo, layout));
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
}

template <int BLOCK_N, int KS>
__global__ void __launch_bounds__(kEdThreads, 2) expand_dw_kernel(const __grid_constant__ ExpandDwParams p) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;          // SWIZZLE_128B tiles need 1024-byte alignment
  uint8_t* base_ptr = smem_raw + (base - raw_addr);
  const uint32_t planes = p.terms > 1 ? 2u : 1u;
  const uint32_t a_base = base, w_base = base + planes * p.a_bytes;
  float* tile = reinterpret_cast<float*>(base_ptr + p.tile_off);
  const uint32_t bar = base + p.tile_off + ((p.n_halo * (BLOCK_N + 4) * 4 + 7) & ~7);
  constexpr int kPitch = BLOCK_N + 4;

  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int b = blockIdx.x / tiles_per_img;
  const int t_in = blockIdx.x - b * tiles_per_img;
  const int oy0 = (t_in / p.tiles_x) * p.tile_h, ox0 = (t_in % p.tiles_x) * p.tile_w;
  const int c0 = blockIdx.y * BLOCK_N;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&p.a_map[0]) : "memory");
    if (p.terms > 1) asm volatile("prefetch.tensormap [%0];" ::"l"(&p.a_map[1]) : "memory");
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();      // everything above touched only this CTA's smem; global reads (TMA) and writes start below

  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, planes * p.n_chunks * (p.n_halo * p.kc * 2 + BLOCK_N * p.kc * 2));
    const int iy = oy0 * p.stride - p.pad, ix = ox0 * p.stride - p.pad;
    for (uint32_t pl = 0; pl < planes; ++pl)
      for (int ch = 0; ch < p.n_chunks; ++ch) {
        tma_load_4d(a_base + pl * p.a_bytes + ch * p.a_chunk_bytes, &p.a_map[pl], bar, ch * p.kc, ix, iy, b);
        tma_load_2d(w_base + pl * p.w_bytes + ch * p.w_chunk_bytes, &p.w_map[pl], bar, ch * p.kc, c0);
      }
  }
  mbar_wait(bar, 0);

  // ---- expansion: warpgroup wg takes m64 blocks wg, wg + 2, ...; bias + activation into the fp32 halo tile
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  for (int mb = wg; mb < p.m_blocks; mb += 2) {
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    if (p.kc == 64) ed_mma_block<BLOCK_N, 4>(acc, p, a_base, w_base, mb);
    else ed_mma_block<BLOCK_N, 2>(acc, p, a_base, w_base, mb);
    const int r0 = mb * 64 + warp * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      const float b0 = (c0 + c < p.mid) ? __ldg(p.e_bias + c0 + c) : 0.f;
      const float b1 = (c0 + c + 1 < p.mid) ? __ldg(p.e_bias + c0 + c + 1) : 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        if (r < p.n_halo)
          *reinterpret_cast<float2*>(tile + r * kPitch + c) =
              make_float2(tc_act(acc[4 * j + 2 * h] + b0, p.e_act), tc_act(acc[4 * j + 2 * h + 1] + b1, p.e_act));
      }
    }
  }
  __syncthreads();

  // ---- depthwise from shared memory: one thread per (output pixel, 8 channels), channels fastest
  const int groups = (min(BLOCK_N, p.mid - c0)) >> 3;
  const size_t plane_stride = (size_t)p.B * p.Ho * p.Wo * p.mid;
#pragma unroll 1
  for (int item = threadIdx.x; item < p.tile_h * p.tile_w * groups; item += kEdThreads) {
    const int pix = item / groups, g = item - pix * groups;
    const int ty = pix / p.tile_w, tx = pix - ty * p.tile_w;
    const int oy = oy0 + ty, ox = ox0 + tx;
    if (oy >= p.Ho || ox >= p.Wo) continue;
    const int c = c0 + 8 * g;
    float acc[8];
    *reinterpret_cast<float4*>(acc) = __ldg(reinterpret_cast<const float4*>(p.dw_b + c));
    *reinterpret_cast<float4*>(acc + 4) = __ldg(reinterpret_cast<const float4*>(p.dw_b + c + 4));
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
      const int iy = oy * p.stride - p.pad + ky;
      const bool yok = iy >= 0 && iy < p.H;
#pragma unroll
      for (int kx = 0; kx < KS; ++kx) {
        const int ix = ox * p.stride - p.pad + kx;
        if (!(yok && ix >= 0 && ix < p.W)) continue;      // skipped taps contribute exactly 0 (the reference's zero padding)
        const float* xp = tile + ((ty * p.stride + ky) * p.halo_w + tx * p.stride + kx) * kPitch + 8 * g;
        float xv[8], wv[8];
        *reinterpret_cast<float4*>(xv) = *reinterpret_cast<const float4*>(xp);
        *reinterpret_cast<float4*>(xv + 4) = *reinterpret_cast<const float4*>(xp + 4);
        const float* wp = p.dw_w + (size_t)(ky * KS + kx) * p.mid + c;
        *reinterpret_cast<float4*>(wv) = __ldg(reinterpret_cast<const float4*>(wp));
        *reinterpret_cast<float4*>(wv + 4) = __ldg(reinterpret_cast<const float4*>(wp + 4));
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = fmaf(xv[e], wv[e], acc[e]);
      }
    }
    __align__(16) __half hi[8];
    __align__(16) __half lo[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float v = (p.dw_act == DVMVS_ACT_RELU) ? fmaxf(acc[e], 0.f) : acc[e];
      hi[e] = __float2half_rn(v);
      lo[e] = __float2half_rn(v - __half2float(hi[e]));
    }
    __half* o = p.out + (((size_t)b * p.Ho + oy) * p.Wo + ox) * p.mid + c;
    *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(hi);
    if (p.write_lo) *reinterpret_cast<uint4*>(o + plane_stride) = *reinterpret_cast<const uint4*>(lo);
  }
}

// shared memory of one CTA for an output tile of th x tw pixels (1024 bytes of alignment slack, the mbarrier at the end)
static int ed_smem_bytes(int th, int tw, int k, int s, int kc, int n_chunks, int terms, int block_n, int* n_halo, int* m_blocks) {
  const int hh = (th - 1) * s + k, hw = (tw - 1) * s + k;
  *n_halo = hh * hw;
  *m_blocks = (*n_halo + 63) / 64;
  const int planes = terms > 1 ? 2 : 1;
  const int a = planes * n_chunks * (*m_blocks * 64 * kc * 2), w = planes * n_chunks * block_n * kc * 2;
  return 1024 + a + w + ((*n_halo * (block_n + 4) * 4 + 7) & ~7) + 8;
}

template <int BLOCK_N, int KS>
static int launch_ed(const ExpandDwParams& p, dim3 grid, int smem, cudaStream_t s) {
  static PerDeviceOnce attr_set;
  if (attr_set.first()) {
    cudaError_t e = cudaFuncSetAttribute(expand_dw_kernel<BLOCK_N, KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) { set_error("expand_dw smem attribute: %s", cudaGetErrorString(e)); return DVMVS_ELAUNCH; }
  }
  launch_k(expand_dw_kernel<BLOCK_N, KS>, grid, dim3(kEdThreads), (size_t)smem, s, p);
  return check_launch("expand_dw_kernel");
}

}  // namespace dvmvs

using namespace dvmvs;

extern "C" int dvmvs_expand_dwconv(const void* x_planes, int B, int H, int W, int Cs, const void* w_hi, const void* w_lo, int w_rows, int ktot,
                                   const float* expand_bias, int expand_act, const float* dw_weight, const float* dw_bias, int ksize,
                                   int stride, int dw_act, int mid, int terms, int write_lo, void* y_planes, dvmvs_stream_t stream) {
  DVMVS_REQUIRE(tensor_map_encoder() != nullptr, "expand_dwconv: cuTensorMapEncodeTiled entry point not available");
  DVMVS_REQUIRE(x_planes && w_hi && (terms == 1 || w_lo) && expand_bias && dw_weight && dw_bias && y_planes, "expand_dwconv: null pointer");
  DVMVS_REQUIRE(B > 0 && H > 0 && W > 0 && Cs > 0 && Cs % 8 == 0 && mid > 0 && mid % 8 == 0,
                "expand_dwconv: bad shape (B=%d H=%d W=%d Cs=%d mid=%d; Cs and mid must be multiples of 8)", B, H, W, Cs, mid);
  DVMVS_REQUIRE((ksize == 3 || ksize == 5) && (stride == 1 || stride == 2), "expand_dwconv: ksize=%d stride=%d", ksize, stride);
  DVMVS_REQUIRE(terms == 1 || terms == 3, "expand_dwconv: terms=%d", terms);
  DVMVS_REQUIRE(expand_act == DVMVS_ACT_NONE || expand_act == DVMVS_ACT_RELU, "expand_dwconv: expand act %d", expand_act);
  DVMVS_REQUIRE(dw_act == DVMVS_ACT_NONE || dw_act == DVMVS_ACT_RELU, "expand_dwconv: depthwise act %d", dw_act);
  DVMVS_REQUIRE((uintptr_t)x_planes % 16 == 0 && (uintptr_t)w_hi % 16 == 0 && (uintptr_t)w_lo % 16 == 0 && (uintptr_t)dw_weight % 16 == 0 &&
                    (uintptr_t)dw_bias % 16 == 0 && (uintptr_t)y_planes % 16 == 0,
                "expand_dwconv: pointers must be 16-byte aligned");
  ExpandDwParams p;
  memset(&p, 0, sizeof(p));
  p.kc = (Cs % 64 == 0) ? 64 : 32;
  p.n_chunks = (Cs + p.kc - 1) / p.kc;
  DVMVS_REQUIRE(ktot == p.n_chunks * p.kc, "expand_dwconv: packed weight K=%d, expected %d", ktot, p.n_chunks * p.kc);
  // channel slice: 32 or 64 expanded channels, whichever pads mid less (ties: 64, one A tile load serves more channels)
  const int block_n = ((mid + 31) / 32 * 32 < (mid + 63) / 64 * 64) ? 32 : 64;
  const int n_slices = (mid + block_n - 1) / block_n;
  DVMVS_REQUIRE(w_rows % block_n == 0 && w_rows >= n_slices * block_n, "expand_dwconv: weight rows %d do not cover %d channels", w_rows, mid);
  p.terms = terms; p.write_lo = write_lo ? 1 : 0;
  p.B = B; p.H = H; p.W = W; p.mid = mid; p.stride = stride; p.pad = ksize / 2;
  p.Ho = (H + 2 * p.pad - ksize) / stride + 1;
  p.Wo = (W + 2 * p.pad - ksize) / stride + 1;
  // output tile: the largest that fits two CTAs per SM and still gives two CTAs per SM over the grid; else the smallest that fits
  static const int cands[4][2] = {{8, 16}, {8, 8}, {4, 8}, {4, 4}};
  const int n_sms = device_sm_count();
  int smem = 0;
  bool chosen = false;
  for (int i = 0; i < 4; ++i) {
    const int th = min(cands[i][0], p.Ho), tw = min(cands[i][1], p.Wo);
    int n_halo, m_blocks;
    const int bytes = ed_smem_bytes(th, tw, ksize, stride, p.kc, p.n_chunks, terms, block_n, &n_halo, &m_blocks);
    if (bytes > kEdSmemBudget && i < 3) continue;
    const int tiles = ((p.Ho + th - 1) / th) * ((p.Wo + tw - 1) / tw);
    p.tile_h = th; p.tile_w = tw; p.tiles_y = (p.Ho + th - 1) / th; p.tiles_x = (p.Wo + tw - 1) / tw;
    p.halo_h = (th - 1) * stride + ksize; p.halo_w = (tw - 1) * stride + ksize;
    p.n_halo = n_halo; p.m_blocks = m_blocks;
    smem = bytes;
    chosen = true;
    if ((long long)B * tiles * n_slices >= 2LL * n_sms) break;
  }
  DVMVS_REQUIRE(chosen && smem <= 227 * 1024, "expand_dwconv: no tile fits shared memory (Cs=%d mid=%d k=%d)", Cs, mid, ksize);
  const int planes = terms > 1 ? 2 : 1;
  p.a_chunk_bytes = p.m_blocks * 64 * p.kc * 2;
  p.w_chunk_bytes = block_n * p.kc * 2;
  p.a_bytes = p.n_chunks * p.a_chunk_bytes;
  p.w_bytes = p.n_chunks * p.w_chunk_bytes;
  p.tile_off = planes * (p.a_bytes + p.w_bytes);
  p.e_bias = expand_bias; p.e_act = expand_act;
  p.dw_w = dw_weight; p.dw_b = dw_bias; p.dw_act = dw_act;
  p.out = (__half*)y_planes;
  const size_t plane = (size_t)B * H * W * Cs;
  for (int pl = 0; pl < planes; ++pl) {
    const void* xp = (const __half*)x_planes + pl * plane;
    cuuint64_t dims[4] = {(cuuint64_t)Cs, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)Cs * 2, (cuuint64_t)W * Cs * 2, (cuuint64_t)H * W * Cs * 2};
    cuuint32_t box[4] = {(cuuint32_t)p.kc, (cuuint32_t)p.halo_w, (cuuint32_t)p.halo_h, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    const CUtensorMapSwizzle sw = p.kc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    CUresult r = cached_tensor_map(&p.a_map[pl], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, xp, dims, strides, box, estr, sw,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
    DVMVS_REQUIRE(r == CUDA_SUCCESS, "expand_dwconv: cuTensorMapEncodeTiled(activation) failed: %d", (int)r);
    cuuint64_t wdims[2] = {(cuuint64_t)ktot, (cuuint64_t)w_rows};
    cuuint64_t wstrides[1] = {(cuuint64_t)ktot * 2};
    cuuint32_t wbox[2] = {(cuuint32_t)p.kc, (cuuint32_t)block_n};
    cuuint32_t westr[2] = {1, 1};
    r = cached_tensor_map(&p.w_map[pl], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, pl ? w_lo : w_hi, wdims, wstrides, wbox, westr, sw,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    DVMVS_REQUIRE(r == CUDA_SUCCESS, "expand_dwconv: cuTensorMapEncodeTiled(weights) failed: %d", (int)r);
  }
  const dim3 grid(p.tiles_x * p.tiles_y * B, n_slices);
  cudaStream_t s = (cudaStream_t)stream;
  if (block_n == 32) return ksize == 3 ? launch_ed<32, 3>(p, grid, smem, s) : launch_ed<32, 5>(p, grid, smem, s);
  return ksize == 3 ? launch_ed<64, 3>(p, grid, smem, s) : launch_ed<64, 5>(p, grid, smem, s);
}
