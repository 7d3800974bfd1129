/*
 * dvmvs_b200.h -- C ABI of libdvmvs_sm90.so: the H100 (sm_90a) kernels behind the DeepVideoMVS
 * plane-sweep depth-inference path.
 *
 * The reference (ardaduz/deep-video-mvs) is pure Python/PyTorch and has no FFI; the "interface each entry
 * point replaces" is therefore the Python function / nn.Module.forward it stands behind (paths relative to
 * the reference root).  The host-side mirror of those names lives in deep-video-mvs_b200/dvmvs/ and binds
 * this library with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch types.
 *   - every pointer is a DEVICE pointer unless the name ends in _host.
 *   - every function returns 0 on success or a negative DVMVS_E* code; it never throws, never allocates
 *     device memory, never synchronises the device; work is enqueued on `stream`.
 *   - activations are channel-last fp32: [B][H][W][C] ("NHWC").  Cost volumes are [B][h][w][D].
 *   - poses are row-major 4x4 camera-to-world matrices, intrinsics row-major 3x3, fp32, on the device
 *     (the reference keeps them on the device too; no D2H copies anywhere on the path).
 */
#ifndef DVMVS_B200_H
#define DVMVS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* dvmvs_stream_t; /* cudaStream_t */

enum {
  DVMVS_OK = 0,
  DVMVS_EINVAL = -1,   /* bad argument (shape, alignment, null pointer) */
  DVMVS_ELAUNCH = -2,  /* CUDA launch error; see dvmvs_last_error_string() */
  DVMVS_EUNSUPPORTED = -3
};

enum { DVMVS_ACT_NONE = 0, DVMVS_ACT_RELU = 1, DVMVS_ACT_SIGMOID = 2 };
enum { DVMVS_SRC_DIRECT = 0, DVMVS_SRC_UPSAMPLE2X = 1 };     /* conv input source modes */
enum { DVMVS_SPLIT_UPSAMPLE2X = 1, DVMVS_SPLIT_HI_ONLY = 2 };   /* dvmvs_split_blocked flags */
enum { DVMVS_RES_NONE = 0, DVMVS_RES_SAME = 1, DVMVS_RES_NEAREST_UP = 2 };
enum { DVMVS_SWEEP_DOT = 0, DVMVS_SWEEP_SAD = 1 };
enum { DVMVS_LOSS_L1 = 0, DVMVS_LOSS_L1_INV = 1, DVMVS_LOSS_L1_REL = 2, DVMVS_LOSS_HUBER = 3 };   /* losses.py:33-40 loss_type */

/* Library identification / diagnostics. */
int dvmvs_abi_version(void);                 /* bumps when a signature changes */
/* Programmatic dependent launch (griddepcontrol) for the launches that follow, process-wide: 1 on, 0 off, -1 default
 * (on unless the environment says DVMVS_PDL=0).  Launches already enqueued or captured keep what they were made with. */
int dvmvs_set_programmatic_launch(int mode);
const char* dvmvs_last_error_string(void);   /* thread-local, static storage */
int dvmvs_kernel_launch_count(void);         /* kernels launched by this library since load (process-wide) */

/* ------------------------------------------------------------------------------------------------------
 * Plane-sweep warp + correlate, all planes and all measurement frames fused in ONE launch.
 * Replaces dvmvs/utils.py:89-107 cost_volume_fusion and :45-86 calculate_cost_volume_by_warping (M = 1).
 *   ref        [B][h][w][C]  reference-frame features (image1)
 *   meas_host  host array of M device pointers, each [B][h][w][C] (image2s)
 *   pose1      [B][4][4]     reference cam-to-world
 *   pose2_host host array of M device pointers, each [B][4][4] (pose2s)
 *   K          [B][3][3]     half-resolution intrinsics
 *   cost_out   [B][h][w][D]  fused cost volume; mean over M of  sum_c f1*warp / C  (DOT)  or
 *                            sum_c |f1 - warp|  (SAD)
 * Plane i has inverse depth 1/max_depth + i*(1/min_depth - 1/max_depth)/(D-1).  M <= 8, D <= 256.
 * C == 32 takes the fast path (quarter-warp per sample, 128-byte gathers); any other C a generic path. */
int dvmvs_plane_sweep_fused(const float* ref, const float* const* meas_host, const float* pose1,
                            const float* const* pose2_host, const float* K, float* cost_out,
                            int B, int C, int h, int w, int D, int M, float min_depth, float max_depth,
                            int mode, dvmvs_stream_t stream);

/* EXPERIMENTAL, opt-in (Python: DVMVS_SWEEP_FP16=1), not yet measured on hardware: the same fused plane sweep (DOT mode,
 * C = 32) gathering 16-bit measurement features -- meas_h16_host: host array of M device pointers to FP16 [B][h][w][32]
 * tensors (the "hi" plane a tensor-core convolution emits); ref stays fp32.  Replaces dvmvs/utils.py:89-107 like
 * dvmvs_plane_sweep_fused; rounding the sweep's feature inputs to fp16 moves the final inverse depth by <= 1.3e-6 in the
 * CPU oracle (tools/feature_fp16_probe.py). */
int dvmvs_plane_sweep_fused_h16(const float* ref, const void* const* meas_h16_host, const float* pose1,
                                const float* const* pose2_host, const float* K, float* cost_out, int B, int C, int h, int w,
                                int D, int M, float min_depth, float max_depth, dvmvs_stream_t stream);

/* The fused plane sweep (DOT mode, C = 32, D <= 128) in its tensor-core form: correlate-then-interpolate.  Replaces
 * dvmvs/utils.py:89-107 like dvmvs_plane_sweep_fused.  The cost is linear in the four bilinear taps, so the kernel forms the
 * 32-channel dot products of a 16x4 tile of reference pixels with the band of measurement pixels around the tile's
 * epipolar segment with wgmma (band rows fetched by TMA with zero fill = grid_sample's zero padding; register accumulators),
 * parks them in shared memory and blends four SCALARS per (pixel, plane) sample.  Degenerate homographies and bands that
 * do not fit take a direct gather path inside the same kernel.
 *   ref_hi / ref_lo            fp16 [B][h][w][32]: x = hi + lo (lo unused / may be NULL when terms == 1)
 *   meas_hi_host / meas_lo_host  host arrays of M device pointers, same layout
 *   terms                      3: hi*hi + lo*hi + hi*lo (fp32-equivalent dot products); 1: plain fp16 features
 *   other arguments as dvmvs_plane_sweep_fused. */
int dvmvs_plane_sweep_tc(const void* ref_hi, const void* ref_lo, const void* const* meas_hi_host, const void* const* meas_lo_host,
                         const float* pose1, const float* const* pose2_host, const float* K, float* cost_out, int B, int h, int w,
                         int D, int M, float min_depth, float max_depth, int terms, dvmvs_stream_t stream);

/* Development aid (tools/sweep_timeline.py): a device buffer of 8 x 64 int64 that subsequent dvmvs_plane_sweep_tc launches fill
 * with clock64 stamps of the phases of their first eight CTAs; NULL switches it off. */
int dvmvs_plane_sweep_tc_set_timeline(void* device_buffer);

/* Pose-aware hidden-state warp with the invalid-depth mask fused.
 * Replaces dvmvs/utils.py:205-258 warp_frame_depth plus dvmvs/convlstm.py:30-41 (transformation =
 * inverse(previous_pose) @ current_pose; h[depth <= invalid_thresh] = 0).
 *   h_in [B][h][w][C], depth [B][h][w], prev_pose/cur_pose [B][4][4], K [B][3][3], h_out [B][h][w][C].
 * If prev_pose is NULL, `cur_pose` is taken to be the ready-made src_trans_dst (plain warp_frame_depth)
 * and no mask is applied when invalid_thresh < 0. */
int dvmvs_hidden_warp(const float* h_in, const float* depth, const float* prev_pose, const float* cur_pose,
                      const float* K, float* h_out, int B, int C, int h, int w, float invalid_thresh,
                      dvmvs_stream_t stream);

/* Forward re-projection of the previous depth map into the current view at half resolution,
 * farthest point per pixel wins, unfilled pixels 0; no host round trip.
 * Replaces dvmvs/utils.py:110-154 get_non_differentiable_rectangle_depth_estimation.
 *   cur_pose ("reference_pose_torch"), prev_pose ("measurement_pose_torch") [B][4][4];
 *   prev_depth [B][H][W]; full_K, half_K [B][3][3]; out [B][H/2][W/2] (zeroed by the call). */
int dvmvs_depth_reproject(const float* cur_pose, const float* prev_pose, const float* prev_depth,
                          const float* full_K, const float* half_K, float* out, int B, int H, int W,
                          dvmvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Dense 2-D convolution (k in {1,3,5}, stride in {1,2}, pad (k-1)/2) with fused channel-concat of up to
 * three sources, optional on-the-fly x2 bilinear (align_corners) upsampling per source, folded-BN bias,
 * residual add (same size, or nearest-upsampled from a coarser map = FPN top-down) and activation.
 * Replaces torch.nn.Conv2d + BatchNorm2d(eval) + ReLU / Sigmoid as composed by dvmvs/layers.py:39-65,
 * torch.cat at dvmvs/fusionnet/model.py:112,115,208,212,216,220,295 and dvmvs/convlstm.py:43,
 * F.interpolate at model.py:59,114,293-294 and torchvision FeaturePyramidNetwork's top-down add. */
typedef struct {
  const float* src[3];   /* [B][Hs][Ws][C_i]; Hs = Hin (DIRECT) or Hin/2 (UPSAMPLE2X) */
  int src_channels[3];
  int src_mode[3];
  int n_src;
  const float* weight;   /* [k][k][Cin][Cout], Cin = sum(src_channels), BN folded */
  const float* bias;     /* [Cout] or NULL */
  const float* residual; /* NULL, [B][Hout][Wout][Cout] (SAME) or [B][Hr][Wr][Cout] (NEAREST_UP) */
  int residual_mode, Hr, Wr;
  float* out;            /* [B][Hout][Wout][Cout] */
  float* aux_out;        /* optional [B][Hout][Wout][Cout]: 1/(aux_mult*act(y) + aux_base) (depth heads) */
  float aux_mult, aux_base;
  int B, Hin, Win, Cout, ksize, stride, act;
  float* workspace;      /* optional scratch for deterministic split-K on small maps (partial sums, reduced in a */
  long long workspace_bytes; /* fixed order by a finishing kernel); NULL / too small => no split */
} dvmvs_conv_desc;

int dvmvs_conv2d(const dvmvs_conv_desc* desc_host, dvmvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * The same convolution on the Hopper tensor cores: implicit GEMM, wgmma.mma_async with register accumulators,
 * operand tiles fed by TMA (one 4-D box per filter tap and channel chunk; zero padding = TMA out-of-bounds fill).
 * Activations and weights are fp16 (hi, lo) pairs, x = hi + lo; terms = 3 issues hi*hi + lo*hi + hi*lo with fp32
 * accumulation (fp32-equivalent results), terms = 1 plain fp16.
 *   src_planes[i]  fp16 [2][B][Hin][Win][C_i]: plane 0 = hi, plane 1 = lo (plane 1 unused when terms == 1);
 *                  C_i a multiple of 8 (dvmvs_split_planes pads with zero channels)
 *   w_hi / w_lo    fp16 [w_rows][ktot], row n = output channel n (rows >= Cout are zero), BN folded; the K axis is
 *                  ordered tap-major, then source, then 32- or 64-channel chunks (64 when C_i % 64 == 0, else 32),
 *                  each chunk zero-padded to its full width -- see dvmvs/_ops.py pack_tc_weights
 *   out_f32 / out_planes   either or both; same epilogue options as dvmvs_conv2d. */
typedef struct {
  const void* src_planes[3];
  int src_channels[3];
  int n_src;
  const void* w_hi;
  const void* w_lo;
  int w_rows, ktot, block_n, terms, allow_split;
  const float* bias;
  const float* residual;
  int residual_mode, Hr, Wr;
  float* out_f32;
  void* out_planes;
  float* aux_out;
  float aux_mult, aux_base;
  int B, Hin, Win, Cout, ksize, stride, act;
  float* workspace;      /* as in dvmvs_conv_desc (split over filter taps) */
  long long workspace_bytes;
  void* out_blk;         /* optional: the same output also in the blocked layout [2][B][Cout/8][Hout][Wout][8] that
                            dvmvs_conv2d_halo consumes (needs out_planes) */
  int out_hi_only;       /* fp16 outputs: write plane 0 (hi) only -- every consumer of this tensor runs 1-term products */
  int defer_finish;      /* split-K launches only (dvmvs_conv2d_tc_ksplit > 1): leave the partial sums in the workspace
                            ([ksplit][B][Hout][Wout][Cout] fp32 at workspace + 16384 bytes) and skip the finishing kernel --
                            the caller's epilogue reduces them (dvmvs_lstm_gates_parts); no outputs are written */
} dvmvs_conv_tc_desc;

int dvmvs_conv2d_tc(const dvmvs_conv_tc_desc* desc_host, dvmvs_stream_t stream);
int dvmvs_conv2d_tc_ksplit(const dvmvs_conv_tc_desc* desc_host);   /* the split count that call will use (1 = none) */

/* ------------------------------------------------------------------------------------------------------
 * Stride-1 k x k convolution on the tensor cores (wgmma) without im2col amplification ("halo" implicit GEMM, csrc/conv_halo.cu): the
 * activations live in the channel-BLOCKED fp16 pair layout [2][B][C/8][H][W][8]; one TMA box loads the halo of an
 * 8 x 16 output tile once per kc-channel group and every filter tap is a start-address offset into it.
 *   src_blk[i]  blocked planes of source i (C8_i = channel blocks; padded channels are zero); sources concatenate
 *   w_hi/w_lo   fp16 weights in their shared-memory image: [n-tile][group][ky][kx][kc/8][block_n][8], BN folded; groups
 *               enumerate the kc-channel groups of source 0, then source 1, ... (zero rows for padded channels)
 *   w_cat       unused, kept for ABI compatibility (pass NULL)
 *   outputs     any of: out_f32 [B][H][W][Cout], out_blk [2][B][Cout/8][H][W][8], out_nhwc [2][B][H][W][Cout]
 *   residual    optional fp32 [B][H][W][Cout] added before the activation. */
typedef struct {
  const void* src_blk[3];
  int src_c8[3];
  int n_src;
  const void* w_hi;
  const void* w_lo;
  int n_groups, kc, block_n, terms;
  const float* bias;
  const float* residual;
  float* out_f32;
  void* out_blk;
  void* out_nhwc;
  int B, H, W, Cout, ksize, act;
  const void* w_cat;
  int out_hi_only;       /* fp16 outputs: hi plane only */
} dvmvs_conv_halo_desc;

int dvmvs_conv2d_halo(const dvmvs_conv_halo_desc* desc_host, dvmvs_stream_t stream);

/* fp32 channel-last [B][H][W][C] -> channels [c_offset, c_offset + c_cover) of the BLOCKED fp16 pair planes
 * [2][B][C8][H'][W'][8] (x, then zeros).  flags: DVMVS_SPLIT_UPSAMPLE2X applies x2 bilinear (align_corners) upsampling
 * (H' = 2H; the value 1 keeps its earlier meaning), DVMVS_SPLIT_HI_ONLY leaves the lo plane unwritten (for operands only
 * 1-term products read). */
int dvmvs_split_blocked(const float* x, void* planes, int B, int H, int W, int C, int C8, int flags, int c_offset,
                        int c_cover, dvmvs_stream_t stream);

/* fp32 channel-last [B][H][W][C] -> channels [c_offset, c_offset + c_cover) of fp16 (hi, lo) planes
 * [2][B][H'][W'][Cs] (Cs a multiple of 8): the C values of x, then zeros up to c_cover.  Several calls with different
 * offsets stage a channel concatenation (torch.cat) into one operand tensor.  upsample2x != 0 applies the x2 bilinear
 * (align_corners) interpolation on the way (H' = 2H). */
int dvmvs_split_planes(const float* x, void* planes, int B, int H, int W, int C, int Cs, int upsample2x, int c_offset,
                       int c_cover, dvmvs_stream_t stream);

/* MnasNet stem (torchvision mnasnet1_0 layers[0:3], fusionnet/model.py:125-127): 3x3 stride-2 pad-1 convolution 3 -> 32
 * + folded BN + ReLU, reading the NCHW image [B][3][H][W] directly and writing channel-last [B][H/2][W/2][32].
 * weight [3][3][3][32] (k, k, Cin, Cout), bias [32]. */
int dvmvs_stem_conv(const float* image_nchw, const float* weight, const float* bias, float* y, int B, int H, int W,
                    dvmvs_stream_t stream);

/* Depthwise k x k convolution (MnasNet), folded-BN bias + optional ReLU.
 * x [B][H][W][C], weight [k][k][C], bias [C]; outputs (either or both): y fp32 [B][Hout][Wout][C],
 * y_planes fp16 (hi, lo) [2][B][Hout][Wout][C] for a tensor-core consumer. */
int dvmvs_dwconv2d(const float* x, const float* weight, const float* bias, float* y, void* y_planes, int B, int H, int W,
                   int C, int ksize, int stride, int act, dvmvs_stream_t stream);

/* MnasNet inverted-residual front half in one launch (csrc/expand_dw.cu): the 1x1 expansion Cs -> mid on the tensor cores
 * (+ bias, expand_act) followed by the depthwise k x k convolution (+ bias, dw_act); the expanded tensor stays in shared
 * memory.  Results are bit-identical to dvmvs_conv2d_tc (1x1, out_f32) followed by dvmvs_dwconv2d (y_planes).
 *   x_planes      fp16 (hi, lo) planes [2][B][H][W][Cs] of the block input, Cs a multiple of 8 (plane 1 unused when terms == 1)
 *   w_hi / w_lo   the expansion's dvmvs_conv2d_tc weights [w_rows][ktot] (ksize 1, one source of Cs channels)
 *   dw_weight     [k][k][mid], dw_bias [mid]; ksize 3 or 5, stride 1 or 2, mid a multiple of 8
 *   y_planes      fp16 (hi, lo) [2][B][Hout][Wout][mid]; plane 1 is written only when write_lo != 0. */
int dvmvs_expand_dwconv(const void* x_planes, int B, int H, int W, int Cs, const void* w_hi, const void* w_lo, int w_rows, int ktot,
                        const float* expand_bias, int expand_act, const float* dw_weight, const float* dw_bias, int ksize, int stride,
                        int dw_act, int mid, int terms, int write_lo, void* y_planes, dvmvs_stream_t stream);

/* ConvLSTM gate epilogue: replaces dvmvs/convlstm.py:45-59.  gates [B][h][w][4*C] in the order i,f,o,g;
 * c_in [B][h][w][C]; writes h_out, c_out [B][h][w][C].  LayerNorm over (h,w) per (b,channel), biased
 * variance, eps 1e-5, no affine; CELU alpha = 1. */
int dvmvs_lstm_gates(const float* gates, const float* c_in, float* h_out, float* c_out, int B, int h, int w, int C,
                     dvmvs_stream_t stream);

/* The same epilogue as the FINISHING PASS of the gate convolution (convlstm.py:43-59 in one step after the GEMM): the gate
 * pre-activations are read as the sum, in split order, of the n_parts split-K partial sums a dvmvs_conv2d_tc launch with
 * defer_finish left in its workspace (part i at gate_parts + i * part_stride elements, each [B][h][w][4*C]) plus `addend`
 * ([B][h][w][4*C] or NULL: the state-independent half conv(W[:, :Cin], x)), then sigmoid / LayerNorm over (h,w) / CELU / state
 * update.  n_parts = 1, addend = NULL is dvmvs_lstm_gates. */
int dvmvs_lstm_gates_parts(const float* gate_parts, int n_parts, long long part_stride, const float* addend, const float* c_in,
                           float* h_out, float* c_out, int B, int h, int w, int C, dvmvs_stream_t stream);

/* x2 bilinear upsampling, align_corners=True (F.interpolate at dvmvs/fusionnet/model.py:59,114,293-294). */
int dvmvs_upsample2x(const float* x, float* y, int B, int H, int W, int C, dvmvs_stream_t stream);

/* Image pre-processing on the device: replaces the per-image host work of the test drivers -- load_image's float
 * conversion + BGR->RGB (dvmvs/dataset_loader.py:260-263), PreprocessImage.apply_rgb's crop + cv2.INTER_LINEAR
 * resize + /scale + (x-mean)/std (dvmvs/dataset_loader.py:322-334) and the HWC->CHW transpose + upload of
 * fusionnet/run-testing.py:127 (SURVEY.md section 8, row f2).
 * image: DEVICE pointer, [in_h][in_w][3] interleaved, uint8 (is_u8 = 1, what cv2.imread returns) or fp32;
 * swap_rb = 1 when the input is BGR.  crop_x / crop_y are removed on both sides before resizing to out_h x out_w.
 * out: DEVICE fp32 [3][out_h][out_w] (RGB planes).  mean3 / std3: HOST arrays of 3 floats (copied into the launch). */
int dvmvs_preprocess_rgb(const void* image, int is_u8, int swap_rb, int in_h, int in_w, int crop_x, int crop_y, float* out,
                         int out_h, int out_w, int normalize, float scale, const float* mean3, const float* std3,
                         dvmvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Training step, backward kernels (SURVEY.md section 8 row f3).  The reference differentiates these ops with
 * autograd (fusionnet/run-training.py:227-278 forward_pass; train.py:33-40 loss.backward()); here each has a
 * hand-written derivative.  Gradient buffers with scatter-adds are zeroed by the entry point (cudaMemsetAsync on
 * `stream`); their accumulation uses fp32 atomics, so sums are reproducible to round-off, not bit-for-bit.
 * ------------------------------------------------------------------------------------------------------ */

/* Backward of dvmvs_plane_sweep_fused in DOT mode, C = 32 (dvmvs/utils.py:45-107 under autograd).
 *   grad_cost      [B][h][w][D]   d loss / d cost volume
 *   grad_ref       [B][h][w][32]  out: d loss / d image1 (written, deterministic)
 *   grad_meas_host host array of M device pointers [B][h][w][32]: out, d loss / d image2s[m] (zeroed here, then
 *                  accumulated; the same pointer may appear for several m -- their gradients add up).
 * Poses, intrinsics and depth range get no gradient (the reference trains with given poses). */
int dvmvs_plane_sweep_backward(const float* ref, const float* const* meas_host, const float* pose1,
                               const float* const* pose2_host, const float* K, const float* grad_cost, float* grad_ref,
                               float* const* grad_meas_host, int B, int C, int h, int w, int D, int M, float min_depth,
                               float max_depth, int mode, dvmvs_stream_t stream);

/* Backward of dvmvs_hidden_warp w.r.t. h_in (BPTT through dvmvs/convlstm.py:33-41): grad_h_in [B][h][w][C] (zeroed
 * here) += bilinear weights * grad_out at positions with depth > invalid_thresh.  The depth (ground truth in training,
 * run-training.py:245-258) gets no gradient.  NOTE: the reference applies its mask with `h_cur.data[non_valid] = 0.0`
 * (convlstm.py:41), which autograd does not see -- its gradient is that of the UNMASKED warp; the Python binding
 * therefore passes invalid_thresh = -inf here (dvmvs/training.py). */
int dvmvs_hidden_warp_backward(const float* grad_out, const float* depth, const float* prev_pose, const float* cur_pose,
                               const float* K, float* grad_h_in, int B, int C, int h, int w, float invalid_thresh,
                               dvmvs_stream_t stream);

/* Backward of dvmvs_lstm_gates (dvmvs/convlstm.py:45-59): from the saved pre-activations `gates` and `c_in` and the
 * incoming grad_h / grad_c [B][h][w][C] (grad_c may be NULL) writes grad_gates [B][h][w][4*C] (i,f,o,g order) and
 * grad_c_in [B][h][w][C].  Forward values are recomputed inside the kernel. */
int dvmvs_lstm_gates_backward(const float* gates, const float* c_in, const float* grad_h, const float* grad_c, float* grad_gates,
                              float* grad_c_in, int B, int h, int w, int C, dvmvs_stream_t stream);

/* Multi-scale depth loss, dvmvs/losses.py:43-82 calculate_loss for every prediction scale in ONE launch.
 *   preds_host   host array of n_scales device pointers, prediction j is [B][hs_host[j]][ws_host[j]]
 *   groundtruth  [B][H][W]; scale j compares against its nearest-neighbour down-sampling (F.interpolate 'nearest'),
 *                pixels with ground truth 0 are invalid
 *   sums         out [n_scales][5]: sum |g-p|, sum smooth_l1(p,g), sum |1/g-1/p|, sum |g-p|/g, valid count */
int dvmvs_depth_loss_forward(const float* const* preds_host, const int* hs_host, const int* ws_host, int n_scales,
                             const float* groundtruth, float* sums, int B, int H, int W, dvmvs_stream_t stream);

/* d/d prediction of  sum_j weights_host[j] * sums[j][loss_type] / sums[j][count]  (losses.py:33-40), times the scalar
 * upstream gradient read from DEVICE memory; written to grads_host[j] (same shapes as the predictions). */
int dvmvs_depth_loss_backward(const float* const* preds_host, float* const* grads_host, const int* hs_host, const int* ws_host,
                              const float* weights_host, int n_scales, const float* groundtruth, const float* sums,
                              const float* upstream, int loss_type, int B, int H, int W, dvmvs_stream_t stream);

/* Layout helpers: NCHW <-> NHWC fp32 copies. */
int dvmvs_nchw_to_nhwc(const float* x, float* y, int B, int C, int H, int W, dvmvs_stream_t stream);
int dvmvs_nhwc_to_nchw(const float* x, float* y, int B, int C, int H, int W, dvmvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * TSDF fusion of the predicted depth maps (SURVEY.md section 8 row f4): replaces TSDFVolume.integrate of the
 * reference's sample-data/run-tsdf-reconstruction.py:220-323 -- both its inline pycuda kernel (:80-152) and the
 * numba / numpy CPU path (:181-218, :283-323) it runs when pycuda is absent.  Arithmetic follows the CPU path
 * (mixed float32 / float64) so that volumes are bit-identical to it.
 *   tsdf_vol, weight_vol, color_vol : DEVICE fp32 [dim_x][dim_y][dim_z] (C order), updated in place; initial state
 *                                     1 / 0 / 0 (:57-61).  color is folded b*65536 + g*256 + r.
 *   vol_origin3   : HOST, 3 floats (:50)            voxel_size, trunc_margin (= 5 * voxel_size, :46) : doubles
 *   color_im      : DEVICE [im_h][im_w][3] RGB, uint8 (color_is_u8 = 1) or fp32
 *   depth_im      : DEVICE [im_h][im_w], fp32 or fp64 (depth_is_f64 = 1); 0 = invalid
 *   intr4         : HOST fx, fy, cx, cy as the float32 values of cam_intr.astype(float32) (:197-199)
 *   world_to_cam16: HOST, row-major float64 inv(cam_pose) (:285; the 4x4 inverse stays host logic as in the reference)
 *   updated_count : optional DEVICE counter incremented by the number of voxels updated (NULL = none)          */
int dvmvs_tsdf_integrate(float* tsdf_vol, float* weight_vol, float* color_vol, int dim_x, int dim_y, int dim_z,
                         const float* vol_origin3, double voxel_size, double trunc_margin, const void* color_im,
                         int color_is_u8, const void* depth_im, int depth_is_f64, int im_h, int im_w, const float* intr4,
                         const double* world_to_cam16, double obs_weight, unsigned long long* updated_count,
                         dvmvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Marching cubes on the TSDF volume: replaces the reference's scikit-image call in TSDFVolume.get_mesh
 * (run-tsdf-reconstruction.py:344-358, and get_point_cloud :329-342 through it).  Contract (inside = tsdf < 0, sign-only
 * face resolution, vertex / normal / colour arithmetic, output order) in csrc/mesh.cu and tools/gen_mc_tables.py.
 * Two calls with one device-to-host read between them, which the caller makes to size the outputs:
 *   dvmvs_mesh_scratch_bytes  HOST query: bytes of scratch for a volume (proportional to the voxel count / 65536)
 *   dvmvs_mesh_count          classifies every cube and grid edge and scans the per-CTA counts; the first two ints of
 *                             scratch are then (n_verts, n_faces)
 *   dvmvs_mesh_extract        with the same volume and scratch: verts [n_verts][3] fp32 world coordinates, norms
 *                             [n_verts][3] fp32 unit normals (toward increasing tsdf), colors [n_verts][3] uint8 RGB, faces
 *                             [n_faces][3] int32 vertex ids (counter-clockwise seen from the normal side); vertex_keys
 *                             [n_verts] int32 is scratch for the face ids.
 *   tsdf_vol, color_vol : DEVICE fp32 [dim_x][dim_y][dim_z] (C order), colour folded b*65536 + g*256 + r
 *   vol_origin_host     : HOST, 3 floats (:52)            voxel_size : the float32 voxel size (:351)
 * A volume with a dimension < 2 (0 included) has an empty mesh.  DVMVS_EINVAL when dim_x * dim_y * dim_z * 5 exceeds INT32_MAX (the
 * int32 counts, keys and face ids). */
int dvmvs_mesh_scratch_bytes(int dim_x, int dim_y, int dim_z, long long* bytes_host);
int dvmvs_mesh_count(const float* tsdf_vol, int dim_x, int dim_y, int dim_z, void* scratch, long long scratch_bytes,
                     dvmvs_stream_t stream);
int dvmvs_mesh_extract(const float* tsdf_vol, const float* color_vol, int dim_x, int dim_y, int dim_z,
                       const float* vol_origin_host, float voxel_size, const void* scratch, long long scratch_bytes, int n_verts,
                       int n_faces, int* vertex_keys, float* verts, int* faces, float* norms, unsigned char* colors,
                       dvmvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------
 * Ray casting of the TSDF volume (TSDFVolume.render): what a camera sees of the fused model.  New: the reference has no
 * counterpart (its volume's only way out is the mesh).  One launch for all views, one thread per pixel ray; the ray through
 * integer pixel (u, v) is marched on a lattice of half-voxel steps clipped to the volume box, with an empty-space skip over
 * fully truncated cells, and stops at the first + -> - crossing of the trilinear tsdf.  Contract (operation order, skip rule)
 * in csrc/raycast.cu.
 *   tsdf_vol, color_vol : DEVICE fp32 [dim_x][dim_y][dim_z] (C order), colour folded b*65536 + g*256 + r; the weight volume is
 *                         not read (the raw tsdf is rendered, as get_mesh meshes it)
 *   vol_origin3         : HOST, 3 floats            voxel_size, trunc_margin : doubles (trunc_margin sets the skip length)
 *   views               : DEVICE fp32 [n_views][16]: fx fy cx cy (pixels of the rendered image), R (3x3 row-major,
 *                         camera -> world, as integrate's cam_pose), t
 *   depth               : DEVICE fp32 [n_views][im_h][im_w], camera depth of the hit, 0 = no hit
 *   normals             : DEVICE fp32 [n_views][im_h][im_w][3], world-frame unit normal toward increasing tsdf, 0 = no hit
 *   colors              : DEVICE uint8 [n_views][im_h][im_w][3] RGB, 0 = no hit
 * A volume with a dimension < 2 gives no hits.  DVMVS_EINVAL on null pointers, non-positive extents or view counts, and
 * n_views * im_h * im_w beyond INT32_MAX.  Allocates nothing, does not synchronise. */
int dvmvs_tsdf_raycast(const float* tsdf_vol, const float* color_vol, int dim_x, int dim_y, int dim_z, const float* vol_origin3,
                       double voxel_size, double trunc_margin, const float* views, int n_views, int im_h, int im_w, float* depth,
                       float* normals, unsigned char* colors, dvmvs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DVMVS_B200_H */
