"""Tensor-level wrappers over the C ABI.  Internal activations are channel-last fp32 torch tensors of shape
(B, H, W, C); the reference-facing API hands out / accepts (B, C, H, W) tensors, which are zero-copy permuted
views of the same storage (torch.channels_last strides).  torch is used for device memory and the current
stream only."""
import ctypes
import os as _os_mod


def _os_environ_get(k, d):
    return _os_mod.environ.get(k, d)


import torch

from . import _native as N


def _stream():
    if N.DRYRUN:
        return None
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _first_tensor(args):
    for a in args:
        if isinstance(a, torch.Tensor):
            return a
        if isinstance(a, (list, tuple)):
            t = _first_tensor(a)
            if t is not None:
                return t
        f32 = getattr(a, "f32", None)            # Act
        if isinstance(f32, torch.Tensor):
            return f32
        planes = getattr(a, "planes", None)
        if isinstance(planes, torch.Tensor):
            return planes
    return None


def on_tensor_device(fn):
    """Native calls enqueue on the CURRENT device's current stream and allocate their outputs next to their inputs: when the
    first tensor argument lives on another CUDA device than the current one (modules built on cuda:1 in a process whose
    current device is cuda:0), run the call under torch.cuda.device(that device) -- stream, workspace and per-device kernel
    attributes then all belong to the device the pointers are on."""
    import functools

    @functools.wraps(fn)
    def wrapped(*args, **kwargs):
        t = None if N.DRYRUN else _first_tensor(args)
        if t is not None and t.is_cuda and t.device.index != torch.cuda.current_device():
            with torch.cuda.device(t.device):
                return fn(*args, **kwargs)
        return fn(*args, **kwargs)
    return wrapped


_WORKSPACE = {}
WORKSPACE_BYTES = 32 << 20
_STAND_IN = __import__("threading").local()


class stand_in_for:
    """Context manager: work enqueued inside runs on a stream that stands in for `stream` -- the side stream of a Fork, the
    capture stream of an auto-graph -- and gets a split-K workspace of its own.  torch hands out its pooled streams
    round-robin, so a stand-in can be the very CUDA stream an engine stage runs on; keyed by the stream alone, the stage's
    graph and the stand-in's graph (replayed on another stream) would share partial sums while running concurrently."""

    def __init__(self, stream):
        self.tag = stream.cuda_stream

    def __enter__(self):
        self.prev = getattr(_STAND_IN, "tags", ())
        _STAND_IN.tags = self.prev + (self.tag,)

    def __exit__(self, *exc):
        _STAND_IN.tags = self.prev
        return False


def workspace(device):
    """Scratch for the deterministic split-K reductions of small-map convolutions: one buffer per (device, stream) --
    kernels on different streams (the two stages of PipelinedFusionnet, or a user's own streams) may run concurrently
    and must not share partial-sum storage.  Allocated once per stream (and per stand_in_for chain on it)."""
    key = (device.type, device.index, 0 if N.DRYRUN else torch.cuda.current_stream(device).cuda_stream,
           getattr(_STAND_IN, "tags", ()))
    ws = _WORKSPACE.get(key)
    if ws is None:
        # zero-initialised: its first 16 KiB hold the split-K arrival counters of conv_tc_kernel (self-cleaning)
        ws = _WORKSPACE[key] = torch.zeros(WORKSPACE_BYTES // 4, dtype=torch.float32, device=device)
    return ws


def require_cuda_f32(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor, got %s" % (name, type(t)))
    if not t.is_cuda and not N.DRYRUN:
        raise RuntimeError("%s must be a CUDA tensor (the native path has no CPU fallback)" % name)
    if t.dtype != torch.float32:
        raise RuntimeError("%s must be float32, got %s" % (name, t.dtype))
    return t


@on_tensor_device
def to_nhwc(x, name="input"):
    """(B,C,H,W) logical tensor -> contiguous (B,H,W,C) tensor (zero-copy when already channels_last)."""
    require_cuda_f32(x, name)
    if x.dim() != 4:
        raise ValueError("%s must have shape (B, C, H, W), got %s" % (name, tuple(x.shape)))
    v = x.permute(0, 2, 3, 1)
    if v.is_contiguous():
        return v
    B, C, H, W = x.shape
    if C == 1:
        return x.contiguous().view(B, H, W, 1)
    xc = x.contiguous()
    y = torch.empty((B, H, W, C), dtype=torch.float32, device=x.device)
    N.check(N.lib().dvmvs_nchw_to_nhwc(xc.data_ptr(), y.data_ptr(), B, C, H, W, _stream()), "nchw_to_nhwc")
    return y


def to_api(x_nhwc):
    """(B,H,W,C) contiguous -> (B,C,H,W) view (channels_last strides), no copy."""
    return x_nhwc.permute(0, 3, 1, 2)


@on_tensor_device
def to_nchw_contiguous(x_nhwc):
    B, H, W, C = x_nhwc.shape
    y = torch.empty((B, C, H, W), dtype=torch.float32, device=x_nhwc.device)
    N.check(N.lib().dvmvs_nhwc_to_nchw(x_nhwc.data_ptr(), y.data_ptr(), B, C, H, W, _stream()), "nhwc_to_nchw")
    return y


class PackedConv:
    """Dense conv weights in the kernel layout [k][k][Cin][Cout] with eval-mode BatchNorm folded in
    (scale into the weights, shift into the bias; folded in fp64, stored fp32)."""

    def __init__(self, conv_weight, conv_bias=None, bn=None, stride=1, act=N.ACT_NONE):
        w = conv_weight.detach().to(torch.float64)
        cout = w.shape[0]
        b = conv_bias.detach().to(torch.float64) if conv_bias is not None else None
        if bn is not None:
            scale = bn.weight.detach().to(torch.float64) / torch.sqrt(bn.running_var.detach().to(torch.float64) + bn.eps)
            shift = bn.bias.detach().to(torch.float64) - bn.running_mean.detach().to(torch.float64) * scale
            w = w * scale.view(-1, 1, 1, 1)
            b = shift if b is None else b * scale + shift
        self.ksize = int(w.shape[2])
        self.cin = int(w.shape[1])
        self.cout = int(cout)
        self.stride = int(stride)
        self.act = act
        self.weight = w.permute(2, 3, 1, 0).contiguous().to(torch.float32)          # [k][k][Cin][Cout]
        self.bias = b.to(torch.float32).contiguous() if b is not None else None


class PackedDepthwise:
    def __init__(self, conv_weight, bn, stride, act=N.ACT_RELU):
        w = conv_weight.detach().to(torch.float64)                                  # (C,1,k,k)
        scale = bn.weight.detach().to(torch.float64) / torch.sqrt(bn.running_var.detach().to(torch.float64) + bn.eps)
        shift = bn.bias.detach().to(torch.float64) - bn.running_mean.detach().to(torch.float64) * scale
        w = w * scale.view(-1, 1, 1, 1)
        self.ksize = int(w.shape[2])
        self.channels = int(w.shape[0])
        self.stride = int(stride)
        self.act = act
        self.weight = w[:, 0].permute(1, 2, 0).contiguous().to(torch.float32)       # [k][k][C]
        self.bias = shift.to(torch.float32).contiguous()


@on_tensor_device
def conv2d(sources, pc, residual=None, residual_mode=N.RES_NONE, aux=None):
    """sources: list of (nhwc tensor, mode) with mode SRC_DIRECT / SRC_UPSAMPLE2X (tensor at half resolution).
    Returns out (B,Hout,Wout,Cout) [, aux_out] -- aux = (mult, base) emits 1/(mult*act(y)+base) as well."""
    d = N.ConvDesc()
    first, mode0 = sources[0]
    B = first.shape[0]
    Hin = first.shape[1] * (2 if mode0 == N.SRC_UPSAMPLE2X else 1)
    Win = first.shape[2] * (2 if mode0 == N.SRC_UPSAMPLE2X else 1)
    cin = 0
    for i, (t, mode) in enumerate(sources):
        f = 2 if mode == N.SRC_UPSAMPLE2X else 1
        if t.shape[0] != B or t.shape[1] * f != Hin or t.shape[2] * f != Win:
            raise ValueError("conv2d: source %d has shape %s, expected spatial %dx%d (mode %d)" % (i, tuple(t.shape), Hin, Win, mode))
        d.src[i] = t.data_ptr()
        d.src_channels[i] = t.shape[3]
        d.src_mode[i] = mode
        cin += t.shape[3]
    if cin != pc.cin:
        raise ValueError("conv2d: %d input channels given, weights expect %d" % (cin, pc.cin))
    d.n_src = len(sources)
    pad = (pc.ksize - 1) // 2
    Hout = (Hin + 2 * pad - pc.ksize) // pc.stride + 1
    Wout = (Win + 2 * pad - pc.ksize) // pc.stride + 1
    out = torch.empty((B, Hout, Wout, pc.cout), dtype=torch.float32, device=first.device)
    d.weight = pc.weight.data_ptr()
    d.bias = pc.bias.data_ptr() if pc.bias is not None else None
    d.residual_mode = residual_mode
    if residual is not None:
        d.residual = residual.data_ptr()
        d.Hr, d.Wr = residual.shape[1], residual.shape[2]
    d.out = out.data_ptr()
    aux_out = None
    if aux is not None:
        aux_out = torch.empty_like(out)
        d.aux_out = aux_out.data_ptr()
        d.aux_mult, d.aux_base = aux
    d.B, d.Hin, d.Win, d.Cout = B, Hin, Win, pc.cout
    d.ksize, d.stride, d.act = pc.ksize, pc.stride, pc.act
    ws = workspace(first.device)
    d.workspace, d.workspace_bytes = ws.data_ptr() + 16384, WORKSPACE_BYTES - 16384      # head = tensor-core path's counters
    N.check(N.lib().dvmvs_conv2d(ctypes.byref(d), _stream()), "conv2d")
    return (out, aux_out) if aux is not None else out


@on_tensor_device
def stem_conv(image_nchw, pc):
    """MnasNet stem on the NCHW image (contiguous) -> channel-last (B, H/2, W/2, 32)."""
    B, C, H, W = image_nchw.shape
    y = torch.empty((B, (H - 1) // 2 + 1, (W - 1) // 2 + 1, 32), dtype=torch.float32, device=image_nchw.device)
    N.check(N.lib().dvmvs_stem_conv(image_nchw.data_ptr(), pc.weight.data_ptr(), pc.bias.data_ptr(), y.data_ptr(), B, H, W, _stream()),
            "stem_conv")
    return y


@on_tensor_device
def dwconv2d(x, pd, want_f32=True, want_planes=False):
    """Returns y (fp32) by default; with want_planes also / only the fp16-pair planes: (y or None, planes)."""
    B, H, W, C = x.shape
    pad = pd.ksize // 2
    Hout = (H + 2 * pad - pd.ksize) // pd.stride + 1
    Wout = (W + 2 * pad - pd.ksize) // pd.stride + 1
    y = torch.empty((B, Hout, Wout, C), dtype=torch.float32, device=x.device) if want_f32 else None
    planes = torch.empty((2, B, Hout, Wout, C), dtype=torch.float16, device=x.device) if want_planes else None
    N.check(N.lib().dvmvs_dwconv2d(x.data_ptr(), pd.weight.data_ptr(), pd.bias.data_ptr(), y.data_ptr() if want_f32 else None,
                                   planes.data_ptr() if want_planes else None, B, H, W, C, pd.ksize, pd.stride, pd.act, _stream()),
            "dwconv2d")
    return (y, planes) if want_planes else y


@on_tensor_device
def plane_sweep(ref_nhwc, meas_nhwc_list, pose1, pose2_list, K, min_depth, max_depth, n_depth_levels, dot_product=True,
                force_generic=False):
    B, h, w, C = ref_nhwc.shape
    M = len(meas_nhwc_list)
    if M < 1 or M != len(pose2_list):
        raise ValueError("plane_sweep: need >= 1 measurement frame and as many poses (got %d, %d)" % (M, len(pose2_list)))
    for m in meas_nhwc_list:
        if tuple(m.shape) != (B, h, w, C):
            raise ValueError("plane_sweep: measurement features %s != reference features %s" % (tuple(m.shape), (B, h, w, C)))
    pose1 = require_cuda_f32(pose1, "pose1").contiguous()
    K = require_cuda_f32(K, "K").contiguous()
    poses = [require_cuda_f32(p, "pose2").contiguous() for p in pose2_list]
    if tuple(pose1.shape) != (B, 4, 4) or tuple(K.shape) != (B, 3, 3) or any(tuple(p.shape) != (B, 4, 4) for p in poses):
        raise ValueError("plane_sweep: poses must be (B,4,4) and K (B,3,3)")
    out = torch.empty((B, h, w, int(n_depth_levels)), dtype=torch.float32, device=ref_nhwc.device)
    meas_ptrs = (ctypes.c_void_p * M)(*[m.data_ptr() for m in meas_nhwc_list])
    pose_ptrs = (ctypes.c_void_p * M)(*[p.data_ptr() for p in poses])
    fn = N.lib().dvmvs_plane_sweep_generic if force_generic else N.lib().dvmvs_plane_sweep_fused
    N.check(fn(ref_nhwc.data_ptr(), meas_ptrs, pose1.data_ptr(), pose_ptrs, K.data_ptr(), out.data_ptr(), B, C, h, w,
               int(n_depth_levels), M, float(min_depth), float(max_depth), N.SWEEP_DOT if dot_product else N.SWEEP_SAD, _stream()),
            "plane_sweep_fused")
    return out


@on_tensor_device
def plane_sweep_h16(ref_nhwc, meas_h16_list, pose1, pose2_list, K, min_depth, max_depth, n_depth_levels):
    """EXPERIMENTAL (opt-in, DVMVS_SWEEP_FP16=1): the fused plane sweep gathering fp16 measurement features -- (B,h,w,32)
    float16 tensors, e.g. the hi plane of a tensor-core convolution's output; dot-product cost only."""
    B, h, w, C = ref_nhwc.shape
    M = len(meas_h16_list)
    for m in meas_h16_list:
        if m.dtype != torch.float16 or tuple(m.shape) != (B, h, w, C) or not m.is_contiguous():
            raise ValueError("plane_sweep_h16: measurement features must be contiguous float16 %s" % ((B, h, w, C),))
    pose1 = require_cuda_f32(pose1, "pose1").contiguous()
    K = require_cuda_f32(K, "K").contiguous()
    poses = [require_cuda_f32(p, "pose2").contiguous() for p in pose2_list]
    out = torch.empty((B, h, w, int(n_depth_levels)), dtype=torch.float32, device=ref_nhwc.device)
    meas_ptrs = (ctypes.c_void_p * M)(*[m.data_ptr() for m in meas_h16_list])
    pose_ptrs = (ctypes.c_void_p * M)(*[p.data_ptr() for p in poses])
    N.check(N.lib().dvmvs_plane_sweep_fused_h16(ref_nhwc.data_ptr(), meas_ptrs, pose1.data_ptr(), pose_ptrs, K.data_ptr(), out.data_ptr(), B, C,
                                                h, w, int(n_depth_levels), M, float(min_depth), float(max_depth), _stream()), "plane_sweep_h16")
    return out


@on_tensor_device
def plane_sweep_tc(ref_planes, meas_planes_list, pose1, pose2_list, K, min_depth, max_depth, n_depth_levels, terms=3, out=None):
    """The fused plane sweep in its tensor-core form (correlate the epipolar band on the tensor cores, then blend four scalars per
    sample; csrc/sweep_tc.cu).  ref_planes / meas_planes_list[m]: fp16 (hi, lo) planes of the 32-channel half-resolution
    features -- either a (2,B,h,w,32) tensor or a (hi, lo) pair of (B,h,w,32) tensors (batch slices of a stacked tensor).
    terms=3: fp32-equivalent dot products; terms=1: plain fp16 features (hi planes only).  Dot-product cost only."""
    def pair(t):
        hi, lo = (t[0], t[1]) if not isinstance(t, torch.Tensor) or t.dim() == 5 else (t, None)
        for x in (hi, lo):
            if x is not None and (x.dtype != torch.float16 or x.dim() != 4 or x.shape[3] != 32 or not x.is_contiguous()):
                raise ValueError("plane_sweep_tc: feature planes must be contiguous float16 (B,h,w,32), got %s %s" % (tuple(x.shape), x.dtype))
        return hi, lo
    rhi, rlo = pair(ref_planes)
    meas = [pair(t) for t in meas_planes_list]
    B, h, w, _ = rhi.shape
    M = len(meas)
    if M < 1 or M != len(pose2_list):
        raise ValueError("plane_sweep_tc: need >= 1 measurement frame and as many poses (got %d, %d)" % (M, len(pose2_list)))
    if any(tuple(hi.shape) != (B, h, w, 32) for hi, _ in meas):
        raise ValueError("plane_sweep_tc: measurement features differ in shape from the reference features %s" % ((B, h, w, 32),))
    if terms == 3 and (rlo is None or any(lo is None for _, lo in meas)):
        raise ValueError("plane_sweep_tc: terms=3 needs the lo planes")
    pose1 = require_cuda_f32(pose1, "pose1").contiguous()
    K = require_cuda_f32(K, "K").contiguous()
    poses = [require_cuda_f32(p, "pose2").contiguous() for p in pose2_list]
    if tuple(pose1.shape) != (B, 4, 4) or tuple(K.shape) != (B, 3, 3) or any(tuple(p.shape) != (B, 4, 4) for p in poses):
        raise ValueError("plane_sweep_tc: poses must be (B,4,4) and K (B,3,3)")
    if out is None:
        out = torch.empty((B, h, w, int(n_depth_levels)), dtype=torch.float32, device=rhi.device)
    hi_ptrs = (ctypes.c_void_p * M)(*[hi.data_ptr() for hi, _ in meas])
    lo_ptrs = (ctypes.c_void_p * M)(*[(lo.data_ptr() if lo is not None else None) for _, lo in meas])
    pose_ptrs = (ctypes.c_void_p * M)(*[p.data_ptr() for p in poses])
    N.check(N.lib().dvmvs_plane_sweep_tc(rhi.data_ptr(), rlo.data_ptr() if rlo is not None else None, hi_ptrs, lo_ptrs, pose1.data_ptr(), pose_ptrs,
                                         K.data_ptr(), out.data_ptr(), B, h, w, int(n_depth_levels), M, float(min_depth), float(max_depth),
                                         int(terms), _stream()), "plane_sweep_tc")
    return out


SWEEP_TC_MAX_PLANES = 128
SWEEP_FP16 = _os_environ_get("DVMVS_SWEEP_FP16", "0") == "1"      # experimental, see plane_sweep_h16


@on_tensor_device
def preprocess_rgb(image_hwc, crop_x, crop_y, out_h, out_w, scale, mean, std, normalize=True, bgr=None, out=None):
    """Device pre-processing of one decoded frame (dataset_loader.py:260-263,322-334 + run-testing.py:127): image_hwc is a
    CUDA tensor (H,W,3), uint8 (as cv2.imread returns it: BGR unless bgr=False) or float32 (as load_image returns it: RGB
    unless bgr=True).  Returns / fills a (1,3,out_h,out_w) fp32 tensor."""
    if not image_hwc.is_cuda:
        raise RuntimeError("preprocess_rgb: image must be a CUDA tensor (no CPU fallback; use PreprocessImage.apply_rgb on the host)")
    if image_hwc.dim() != 3 or image_hwc.shape[2] != 3 or image_hwc.dtype not in (torch.uint8, torch.float32):
        raise RuntimeError("preprocess_rgb: expected an (H,W,3) uint8 or float32 tensor, got %s %s" % (tuple(image_hwc.shape), image_hwc.dtype))
    is_u8 = image_hwc.dtype == torch.uint8
    if bgr is None:
        bgr = is_u8
    image_hwc = image_hwc.contiguous()
    in_h, in_w = int(image_hwc.shape[0]), int(image_hwc.shape[1])
    if out is None:
        out = torch.empty((1, 3, int(out_h), int(out_w)), dtype=torch.float32, device=image_hwc.device)
    elif tuple(out.shape) != (1, 3, int(out_h), int(out_w)) or out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous():
        raise RuntimeError("preprocess_rgb: out must be a contiguous CUDA fp32 (1,3,%d,%d) tensor" % (out_h, out_w))
    m3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in std])
    N.check(N.lib().dvmvs_preprocess_rgb(image_hwc.data_ptr(), 1 if is_u8 else 0, 1 if bgr else 0, in_h, in_w, int(crop_x), int(crop_y),
                                         out.data_ptr(), int(out_h), int(out_w), 1 if normalize else 0, float(scale), m3, s3, _stream()),
            "preprocess_rgb")
    return out


@on_tensor_device
def hidden_warp(h_nhwc, depth_b1hw, prev_pose, cur_pose, K, invalid_thresh):
    B, h, w, C = h_nhwc.shape
    depth = require_cuda_f32(depth_b1hw, "depth").contiguous()
    K = require_cuda_f32(K, "camera_matrix").contiguous()
    cur_pose = require_cuda_f32(cur_pose, "pose").contiguous()
    prev_ptr = None
    if prev_pose is not None:
        prev_pose = require_cuda_f32(prev_pose, "previous_pose").contiguous()
        prev_ptr = prev_pose.data_ptr()
    out = torch.empty_like(h_nhwc)
    N.check(N.lib().dvmvs_hidden_warp(h_nhwc.data_ptr(), depth.data_ptr(), prev_ptr, cur_pose.data_ptr(), K.data_ptr(),
                                      out.data_ptr(), B, C, h, w, float(invalid_thresh), _stream()), "hidden_warp")
    return out


@on_tensor_device
def depth_reproject(cur_pose, prev_pose, prev_depth, full_K, half_K, H, W):
    B = cur_pose.shape[0]
    args = [require_cuda_f32(t, n).contiguous() for t, n in ((cur_pose, "reference_pose"), (prev_pose, "measurement_pose"),
                                                             (prev_depth, "previous_depth"), (full_K, "full_K"), (half_K, "half_K"))]
    out = torch.empty((B, 1, H // 2, W // 2), dtype=torch.float32, device=cur_pose.device)
    N.check(N.lib().dvmvs_depth_reproject(args[0].data_ptr(), args[1].data_ptr(), args[2].data_ptr(), args[3].data_ptr(),
                                          args[4].data_ptr(), out.data_ptr(), B, H, W, _stream()), "depth_reproject")
    return out


@on_tensor_device
def lstm_gates(gates_nhwc, c_nhwc, parts=None, addend=None):
    """ConvLSTM gate epilogue (convlstm.py:45-59).  gates_nhwc: (B,h,w,4C) gate pre-activations -- or, with parts=(workspace
    tensor, byte offset, n_parts, part_stride), the split-K partial sums a deferred gate convolution left in its workspace: the
    epilogue is then the finishing pass of that GEMM (sum of the parts in split order + `addend`, the state-independent half)."""
    B, h, w, C = c_nhwc.shape
    h_out = torch.empty((B, h, w, C), dtype=torch.float32, device=c_nhwc.device)
    c_out = torch.empty_like(h_out)
    if parts is None:
        N.check(N.lib().dvmvs_lstm_gates(gates_nhwc.data_ptr(), c_nhwc.data_ptr(), h_out.data_ptr(), c_out.data_ptr(), B, h, w, C,
                                         _stream()), "lstm_gates")
    else:
        ws, offset, n_parts, stride = parts
        N.check(N.lib().dvmvs_lstm_gates_parts(ws.data_ptr() + offset, int(n_parts), int(stride), addend.data_ptr() if addend is not None else None,
                                               c_nhwc.data_ptr(), h_out.data_ptr(), c_out.data_ptr(), B, h, w, C, _stream()), "lstm_gates_parts")
    return h_out, c_out


@on_tensor_device
def upsample2x(x_nhwc):
    B, H, W, C = x_nhwc.shape
    y = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float32, device=x_nhwc.device)
    N.check(N.lib().dvmvs_upsample2x(x_nhwc.data_ptr(), y.data_ptr(), B, H, W, C, _stream()), "upsample2x")
    return y


# ================================================================================================ tensor-core path
def round_up(x, m):
    return (x + m - 1) // m * m


@on_tensor_device
def split_planes(x_nhwc, upsample=False):
    """fp32 (B,H,W,C) -> fp16 (hi, lo) planes (2,B,H',W',Cs), Cs = C rounded up to 8 (zero channels)."""
    B, H, W, C = x_nhwc.shape
    Cs = round_up(C, 8)
    f = 2 if upsample else 1
    planes = torch.empty((2, B, H * f, W * f, Cs), dtype=torch.float16, device=x_nhwc.device)
    N.check(N.lib().dvmvs_split_planes(x_nhwc.data_ptr(), planes.data_ptr(), B, H, W, C, Cs, 1 if upsample else 0, 0, Cs, _stream()),
            "split_planes")
    return planes


@on_tensor_device
def concat_planes(sources):
    """torch.cat([...], dim=channels) staged directly as ONE fp16-pair operand tensor: sources = [(fp32 nhwc, upsample)]."""
    shapes = [(t.shape[1] * (2 if up else 1), t.shape[2] * (2 if up else 1)) for t, up in sources]
    B, (Ho, Wo) = sources[0][0].shape[0], shapes[0]
    if any(s != (Ho, Wo) for s in shapes):
        raise ValueError("concat_planes: spatial sizes differ: %s" % (shapes,))
    c_total = sum(t.shape[3] for t, _ in sources)
    Cs = round_up(c_total, 8)
    planes = torch.empty((2, B, Ho, Wo, Cs), dtype=torch.float16, device=sources[0][0].device)
    off = 0
    for i, (t, up) in enumerate(sources):
        C = t.shape[3]
        cover = C if i + 1 < len(sources) else Cs - off          # the last source also zero-fills the padding channels
        N.check(N.lib().dvmvs_split_planes(t.data_ptr(), planes.data_ptr(), B, t.shape[1], t.shape[2], C, Cs, 1 if up else 0, off, cover,
                                           _stream()), "split_planes")
        off += C
    return planes


def tc_chunking(cs):
    kchunk = 64 if cs % 64 == 0 else 32
    return kchunk, (cs + kchunk - 1) // kchunk


class PackedConvTC:
    """Weights for dvmvs_conv2d_tc: fp16 (hi, lo) matrices [rows][K] with the K axis ordered tap-major, then source,
    then 32/64-channel chunks (each chunk zero-padded to full width), BN folded in fp64 beforehand."""

    def __init__(self, pc, src_channels, device):
        """pc: PackedConv (fp32, [k][k][Cin][Cout]); src_channels: real channel count of every concatenated source."""
        k, cin, cout = pc.ksize, pc.cin, pc.cout
        assert sum(src_channels) == cin, (src_channels, cin)
        w = pc.weight.detach().to("cpu", torch.float32).reshape(k * k, cin, cout)       # [tap][cin][cout]
        cols = []
        off = 0
        self.src_stored = []
        for cr in src_channels:
            cs = round_up(cr, 8)
            kchunk, nch = tc_chunking(cs)
            blk = torch.zeros(k * k, nch * kchunk, cout, dtype=torch.float32)
            blk[:, :cr, :] = w[:, off:off + cr, :]
            cols.append(blk)
            off += cr
            self.src_stored.append(cs)
        wk = torch.cat(cols, dim=1)                                 # [tap][k_per_tap][cout]
        self.k_per_tap = wk.shape[1]
        self.ktot = k * k * self.k_per_tap
        rows = round_up(cout, 128)
        w2d = torch.zeros(rows, self.ktot, dtype=torch.float32)
        w2d[:cout] = wk.reshape(self.ktot, cout).t()
        hi = w2d.to(torch.float16)
        lo = (w2d - hi.to(torch.float32)).to(torch.float16)
        self.w_hi = hi.contiguous().to(device)
        self.w_lo = lo.contiguous().to(device)
        self.rows = rows
        self.ksize, self.cin, self.cout, self.stride, self.act = k, cin, cout, pc.stride, pc.act
        self.bias = pc.bias.to(device) if pc.bias is not None else None
        self.src_channels = list(src_channels)


@on_tensor_device
def conv2d_tc(sources, ptc, residual=None, residual_mode=N.RES_NONE, aux=None, want_f32=True, want_planes=True, terms=3,
              block_n=None, allow_split=True, blk_out=None, defer_finish=False):
    """sources: list of fp16-pair plane tensors (2,B,Hin,Win,Cs_i) matching ptc.src_stored.  Returns
    (out_f32 or None, out_planes or None[, aux_out])."""
    d = N.ConvTcDesc()
    first = sources[0]
    B, Hin, Win = first.shape[1], first.shape[2], first.shape[3]
    if len(sources) != len(ptc.src_stored):
        raise ValueError("conv2d_tc: %d sources given, weights packed for %d" % (len(sources), len(ptc.src_stored)))
    for i, t in enumerate(sources):
        if t.dtype != torch.float16 or tuple(t.shape[:4]) != (2, B, Hin, Win) or t.shape[4] != ptc.src_stored[i]:
            raise ValueError("conv2d_tc: source %d has shape %s / %s, expected (2,%d,%d,%d,%d) fp16"
                             % (i, tuple(t.shape), t.dtype, B, Hin, Win, ptc.src_stored[i]))
        d.src_planes[i] = t.data_ptr()
        d.src_channels[i] = t.shape[4]
    d.n_src = len(sources)
    pad = (ptc.ksize - 1) // 2
    Hout = (Hin + 2 * pad - ptc.ksize) // ptc.stride + 1
    Wout = (Win + 2 * pad - ptc.ksize) // ptc.stride + 1
    if block_n is None:
        tiles = B * ((Hout + 7) // 8) * ((Wout + 15) // 16)
        if ptc.cout >= 1024 and tiles < 16:
            block_n = 128          # e.g. the ConvLSTM gate conv (Cout 2048 on an 8x8 map): amortise the activation tile over
                                   # 128 output channels and let split-K over the taps provide the CTAs
        elif ptc.cout <= 32 or tiles < 16:
            block_n = 32
        elif ptc.cout <= 64 or tiles < 64:
            block_n = 64
        else:
            block_n = 128
    if want_planes and ptc.cout % 8 != 0:
        raise ValueError("conv2d_tc: fp16-pair output needs Cout % 8 == 0")
    dev = first.device
    out_f32 = torch.empty((B, Hout, Wout, ptc.cout), dtype=torch.float32, device=dev) if want_f32 else None
    out_planes = torch.empty((2, B, Hout, Wout, ptc.cout), dtype=torch.float16, device=dev) if want_planes else None
    d.w_hi, d.w_lo = ptc.w_hi.data_ptr(), ptc.w_lo.data_ptr()
    d.w_rows, d.ktot, d.block_n, d.terms, d.allow_split = ptc.rows, ptc.ktot, block_n, terms, 1 if allow_split else 0
    d.bias = ptc.bias.data_ptr() if ptc.bias is not None else None
    d.residual_mode = residual_mode
    if residual is not None:
        d.residual = residual.data_ptr()
        d.Hr, d.Wr = residual.shape[1], residual.shape[2]
    d.out_f32 = out_f32.data_ptr() if out_f32 is not None else None
    d.out_planes = out_planes.data_ptr() if out_planes is not None else None
    if blk_out is not None:            # caller-provided (2,B,Cout/8,Hout,Wout,8) tensor, filled alongside out_planes
        d.out_blk = blk_out.data_ptr()
    aux_out = None
    if aux is not None:
        aux_out = torch.empty((B, Hout, Wout, ptc.cout), dtype=torch.float32, device=dev)
        d.aux_out = aux_out.data_ptr()
        d.aux_mult, d.aux_base = aux
    d.B, d.Hin, d.Win, d.Cout = B, Hin, Win, ptc.cout
    d.ksize, d.stride, d.act = ptc.ksize, ptc.stride, ptc.act
    ws = None
    if allow_split:
        ws = workspace(dev)
        d.workspace, d.workspace_bytes = ws.data_ptr(), WORKSPACE_BYTES
    d.out_hi_only = 0 if lo_planes_needed() else 1
    if defer_finish:
        # split-K launch whose finishing pass the caller fuses into its own epilogue (ConvLSTM gates): partial sums stay in the workspace
        k = N.lib().dvmvs_conv2d_tc_ksplit(ctypes.byref(d)) if (ws is not None and not N.DRYRUN) else 1
        if k > 1 and residual is None and aux is None:
            d.defer_finish = 1
            d.out_f32 = d.out_planes = d.out_blk = None
            N.check(N.lib().dvmvs_conv2d_tc(ctypes.byref(d), _stream()), "conv2d_tc(deferred finish)")
            return ("parts", (ws, 16384, k, B * Hout * Wout * ptc.cout))
        return None                 # this launch would not split: the caller runs the ordinary path
    N.check(N.lib().dvmvs_conv2d_tc(ctypes.byref(d), _stream()), "conv2d_tc")
    if aux is not None:
        return out_f32, out_planes, aux_out
    return out_f32, out_planes


@on_tensor_device
def expand_dwconv(act, expand_layer, dw, terms=None):
    """MnasNet block front half in one launch: the 1x1 expansion `expand_layer` (a ConvLayer on the tensor-core path) of the Act
    `act`, then the depthwise convolution `dw` (PackedDepthwise).  Returns the fp16 (hi, lo) planes (2,B,Hout,Wout,mid) that the
    block's projection reads -- equal to conv2d_tc(..., want_f32=True) followed by dwconv2d(..., want_planes=True).  The lo plane
    is written only for terms=3 (the projection runs the same terms); terms=None uses the current family's terms."""
    terms = _TC_TERMS if terms is None else int(terms)
    pc = expand_layer.pc
    if pc.ksize != 1 or pc.stride != 1 or not expand_layer.tc_eligible() or dw.channels != pc.cout:
        raise ValueError("expand_dwconv: needs a tensor-core 1x1 expansion to %d channels, got k=%d stride=%d cout=%d"
                         % (dw.channels, pc.ksize, pc.stride, pc.cout))
    if expand_layer._ptc is None:
        expand_layer._ptc = PackedConvTC(pc, expand_layer.src_channels, pc.weight.device)
    ptc = expand_layer._ptc
    x = act.get_planes()
    _, B, H, W, Cs = x.shape
    if Cs != ptc.src_stored[0]:
        raise ValueError("expand_dwconv: input has %d channels, weights packed for %d" % (Cs, ptc.src_stored[0]))
    pad = dw.ksize // 2
    Hout = (H + 2 * pad - dw.ksize) // dw.stride + 1
    Wout = (W + 2 * pad - dw.ksize) // dw.stride + 1
    planes = torch.empty((2, B, Hout, Wout, dw.channels), dtype=torch.float16, device=x.device)
    N.check(N.lib().dvmvs_expand_dwconv(x.data_ptr(), B, H, W, Cs, ptc.w_hi.data_ptr(), ptc.w_lo.data_ptr(), ptc.rows, ptc.ktot,
                                        ptc.bias.data_ptr(), ptc.act, dw.weight.data_ptr(), dw.bias.data_ptr(), dw.ksize, dw.stride,
                                        dw.act, dw.channels, terms, 1 if terms == 3 else 0, planes.data_ptr(), _stream()),
            "expand_dwconv")
    return planes


# ================================================================================================ halo (blocked-layout) path
@on_tensor_device
def split_blocked(sources, only=None, into=None):
    """sources: [(fp32 nhwc tensor, upsample)] -> blocked fp16 pair planes (2, B, C8, H', W', 8) of their channel
    concatenation (torch.cat staged straight into the operand layout of conv_halo_kernel).  Every source starts on an
    8-channel block boundary: narrow sources (the 1-channel depth, the RGB image) are padded to 8 with zero channels --
    PackedConvHalo(pad_sources_to_8=True) lays the weights out the same way.
    only / into: stage just the listed source indices into an existing operand tensor (sources not staged yet may be
    given as (shape tuple, upsample)) -- lets independent producers fill one concatenated operand at different times.
    While no kernel reads lo planes (1-term operands everywhere) only the hi plane is written."""
    shp = lambda t: tuple(t) if isinstance(t, (tuple, list)) else tuple(t.shape)
    shapes = [(shp(t)[1] * (2 if up else 1), shp(t)[2] * (2 if up else 1)) for t, up in sources]
    B, (Ho, Wo) = shp(sources[0][0])[0], shapes[0]
    if any(sh != (Ho, Wo) for sh in shapes):
        raise ValueError("split_blocked: spatial sizes differ: %s" % (shapes,))
    C8 = sum((shp(t)[3] + 7) // 8 for t, _ in sources)
    if into is None:
        dev = next(t.device for t, _ in sources if isinstance(t, torch.Tensor))
        into = torch.empty((2, B, C8, Ho, Wo, 8), dtype=torch.float16, device=dev)
    planes = into
    hi_only = 0 if lo_planes_needed() else N.SPLIT_HI_ONLY
    off = 0
    for i, (t, up) in enumerate(sources):
        C = shp(t)[3]
        cover = (C + 7) // 8 * 8
        if only is None or i in only:
            flags = (N.SPLIT_UPSAMPLE2X if up else 0) | hi_only
            N.check(N.lib().dvmvs_split_blocked(t.data_ptr(), planes.data_ptr(), B, t.shape[1], t.shape[2], C, C8, flags, off, cover,
                                                _stream()), "split_blocked")
        off += cover
    return planes


class PackedConvHalo:
    """Weights for dvmvs_conv2d_halo in their shared-memory image [n-tile][group][ky][kx][kc/8][block_n][8] (fp16 hi / lo)."""

    def __init__(self, pc, src_channels, device, kc=None, block_n=None, concat_padded=False):
        """src_channels: real channels of each source.  concat_padded=False: every source is its own blocked tensor
        (kernel-level K-split).  concat_padded=True: the sources are staged by split_blocked() into ONE blocked tensor
        in which each source starts on an 8-channel boundary."""
        k, cin, cout = pc.ksize, pc.cin, pc.cout
        assert sum(src_channels) == cin and pc.stride == 1
        self.kc = kc or (16 if k == 5 else 32)
        self.block_n = block_n or (32 if cout <= 32 else 64)
        kc, bn = self.kc, self.block_n
        w = pc.weight.detach().to("cpu", torch.float32)                    # [k][k][cin][cout]
        n_tiles = (cout + bn - 1) // bn
        if concat_padded:                                                    # one operand tensor, sources padded to 8 channels
            padded = torch.zeros(k, k, sum((c + 7) // 8 * 8 for c in src_channels), cout, dtype=torch.float32)
            src_off, dst_off = 0, 0
            for cr in src_channels:
                padded[:, :, dst_off:dst_off + cr, :] = w[:, :, src_off:src_off + cr, :]
                src_off, dst_off = src_off + cr, dst_off + (cr + 7) // 8 * 8
            w, src_channels = padded, [padded.shape[2]]
        groups = []                                                          # (cin offset, valid channels) per kc-group
        self.src_c8 = []
        off = 0
        for cr in src_channels:
            c8 = (cr + 7) // 8
            self.src_c8.append(c8)
            for cg in range((c8 * 8 + kc - 1) // kc):
                lo_c = cg * kc
                groups.append((off + lo_c, max(0, min(kc, cr - lo_c))))
            off += cr
        self.n_groups = len(groups)
        packed = torch.zeros(n_tiles, self.n_groups, k, k, kc // 8, bn, 8, dtype=torch.float32)
        for gi, (c0, nvalid) in enumerate(groups):
            if nvalid == 0:
                continue
            blk = torch.zeros(k, k, kc, n_tiles * bn, dtype=torch.float32)
            blk[:, :, :nvalid, :cout] = w[:, :, c0:c0 + nvalid, :]
            # [k][k][kc][ntile*bn] -> [ntile][k][k][kc/8][bn][8]
            blk = blk.reshape(k, k, kc // 8, 8, n_tiles, bn).permute(4, 0, 1, 2, 5, 3)
            packed[:, gi] = blk
        hi = packed.to(torch.float16)
        lo = (packed - hi.to(torch.float32)).to(torch.float16)
        self.w_hi, self.w_lo = hi.contiguous().to(device), lo.contiguous().to(device)
        self.ksize, self.cin, self.cout, self.act = k, cin, cout, pc.act
        self.bias = pc.bias.to(device) if pc.bias is not None else None
        self.src_channels = list(src_channels)


@on_tensor_device
def conv2d_halo(sources_blk, ph, residual=None, terms=3, want_f32=True, want_blk=False, want_nhwc=True):
    """sources_blk: list of blocked plane tensors (2,B,C8_i,H,W,8).  Returns (f32 or None, blk or None, nhwc planes or None)."""
    d = N.ConvHaloDesc()
    first = sources_blk[0]
    B, H, W = first.shape[1], first.shape[3], first.shape[4]
    if len(sources_blk) != len(ph.src_c8):
        raise ValueError("conv2d_halo: %d sources given, weights packed for %d" % (len(sources_blk), len(ph.src_c8)))
    for i, t in enumerate(sources_blk):
        if t.dtype != torch.float16 or tuple(t.shape) != (2, B, ph.src_c8[i], H, W, 8):
            raise ValueError("conv2d_halo: source %d has shape %s, expected %s" % (i, tuple(t.shape), (2, B, ph.src_c8[i], H, W, 8)))
        d.src_blk[i] = t.data_ptr()
        d.src_c8[i] = ph.src_c8[i]
    d.n_src = len(sources_blk)
    dev = first.device
    out_f32 = torch.empty((B, H, W, ph.cout), dtype=torch.float32, device=dev) if want_f32 else None
    out_blk = torch.empty((2, B, ph.cout // 8, H, W, 8), dtype=torch.float16, device=dev) if want_blk else None
    out_nhwc = torch.empty((2, B, H, W, ph.cout), dtype=torch.float16, device=dev) if want_nhwc else None
    d.w_hi, d.w_lo = ph.w_hi.data_ptr(), ph.w_lo.data_ptr()
    d.n_groups, d.kc, d.block_n, d.terms = ph.n_groups, ph.kc, ph.block_n, terms
    d.bias = ph.bias.data_ptr() if ph.bias is not None else None
    d.residual = residual.data_ptr() if residual is not None else None
    d.out_f32 = out_f32.data_ptr() if want_f32 else None
    d.out_blk = out_blk.data_ptr() if want_blk else None
    d.out_nhwc = out_nhwc.data_ptr() if want_nhwc else None
    d.B, d.H, d.W, d.Cout, d.ksize, d.act = B, H, W, ph.cout, ph.ksize, ph.act
    d.out_hi_only = 0 if lo_planes_needed() else 1
    N.check(N.lib().dvmvs_conv2d_halo(ctypes.byref(d), _stream()), "conv2d_halo")
    return out_f32, out_blk, out_nhwc


# ================================================================================================ backend dispatch
import os as _os

# "tc" (default): wgmma implicit-GEMM kernels wherever a layer is eligible, CUDA-core kernels for the rest (stem, depthwise,
# depth heads); "fp32": exact-fp32 CUDA-core kernels everywhere -- the device-side cross-check the parity tests pin the
# tensor path against (tests/conftest.py selects it for the op-level tests).
_BACKEND = _os.environ.get("DVMVS_CONV_BACKEND", "tc")
_TC_TERMS = int(_os.environ.get("DVMVS_TC_TERMS", "3"))        # 3: fp16 (hi, lo) pairs ~ fp32 accuracy; 1: plain fp16 operands
_TC_STRIDE2 = _os.environ.get("DVMVS_TC_STRIDE2", "1") == "1"  # stride-2 convolutions on the tensor path too
_HALO = _os.environ.get("DVMVS_HALO", "1") == "1"          # blocked-layout halo kernel for large stride-1 k>=3 convolutions
_HALO_MIN_PIXELS = int(_os.environ.get("DVMVS_HALO_MIN_PIXELS", "4096"))   # >= 64x64 maps; smaller maps: split-K conv_tc


def set_conv_backend(name, terms=None, stride2=None):
    """'fp32' = exact-fp32 CUDA-core convolutions everywhere; 'tc' = wgmma implicit GEMM (fp16-pair operands, fp32
    accumulate) for every dense convolution it supports, CUDA-core kernels for the rest."""
    global _BACKEND, _TC_TERMS, _TC_STRIDE2
    if name not in ("fp32", "tc"):
        raise ValueError("backend must be 'fp32' or 'tc'")
    global _TC_TERMS_BASE, _CONFIG_EPOCH
    _CONFIG_EPOCH += 1
    _BACKEND = name
    if terms is not None:
        _TC_TERMS = int(terms)
        _TC_TERMS_BASE = int(terms)
    if stride2 is not None:
        _TC_STRIDE2 = bool(stride2)


def conv_backend():
    return _BACKEND


_CONFIG_EPOCH = 0


def config_epoch():
    """Bumped by every change of the backend / precision configuration (captured auto-graphs are keyed by it)."""
    return _CONFIG_EPOCH


_TC_TERMS_BASE = _TC_TERMS          # the terms set_conv_backend chose (family_terms() changes _TC_TERMS while a module runs)


def lo_planes_needed():
    """fp16 lo planes are only read by 3-term products: when the base precision and every family policy are 1-term, producers
    skip writing them (and never read them)."""
    return _TC_TERMS_BASE == 3 or _TC_TERMS == 3 or any(v == 3 for v in _TERMS_POLICY.values())


# Per-family operand precision of the tensor-core path: module family ("fe", "fpn", "cve", "lstm", "cvd") -> terms
# (3 = fp16 (hi, lo) pairs, three products, ~fp32 accuracy; 1 = plain fp16 operands, fp32 accumulate).  Families not
# listed use the global `terms` of set_conv_backend.  The top-level modules' forwards run under family_terms(), so the
# shared building blocks (StandardLayer, EncoderBlock, ...) follow the module they are used in.
_TERMS_POLICY = {}


def set_precision_policy(policy=None):
    """policy: dict family -> 1 | 3, or None / {} to clear.  Also accepts "fe=1,fpn=1,cve=1" (DVMVS_TC_POLICY syntax)."""
    global _TERMS_POLICY, _CONFIG_EPOCH
    _CONFIG_EPOCH += 1
    if isinstance(policy, str):
        policy = {k.strip(): int(v) for k, v in (item.split("=") for item in policy.split(",") if item.strip())}
    policy = dict(policy or {})
    for k, v in policy.items():
        if k not in ("fe", "fpn", "cve", "lstm", "cvd", "sweep") or v not in (1, 3):
            raise ValueError("precision policy: family in fe/fpn/cve/lstm/cvd/sweep, terms 1 or 3 (got %r=%r)" % (k, v))
    _TERMS_POLICY = policy


def precision_policy():
    return dict(_TERMS_POLICY)


if _os.environ.get("DVMVS_TC_POLICY"):
    set_precision_policy(_os.environ["DVMVS_TC_POLICY"])


def family_terms(family):
    """Decorator for the forward of a top-level module: convolutions launched inside use the family's terms."""
    def deco(fn):
        import functools

        @functools.wraps(fn)
        def wrapped(*a, **k):
            global _TC_TERMS
            t = _TERMS_POLICY.get(family)
            if t is None:
                return fn(*a, **k)
            saved, _TC_TERMS = _TC_TERMS, t
            try:
                return fn(*a, **k)
            finally:
                _TC_TERMS = saved
        return wrapped
    return deco


class Act:
    """An activation inside a module: fp32 channel-last tensor and/or its fp16 (hi, lo) planes (created on demand,
    cached).  `up` planes = planes of the x2-bilinear-upsampled tensor (F.interpolate materialised for the TMA loader)."""
    __slots__ = ("f32", "planes", "planes_up", "blk", "blk_up", "version", "pair")

    def __init__(self, f32=None, planes=None, blk=None, pair=None):
        self.f32, self.planes, self.planes_up, self.blk, self.blk_up, self.version = f32, planes, None, blk, None, None
        self.pair = pair          # (hi, lo) fp16 (B,H,W,C) tensors when the planes are a batch slice of a bigger tensor's planes

    @property
    def channels(self):
        return self.f32.shape[3] if self.f32 is not None else self.planes.shape[4]

    def get_planes(self, upsample=False):
        if self.f32 is None and (upsample or self.planes is None):
            raise RuntimeError("activation has no fp32 representation to derive planes from")
        if upsample:
            if self.planes_up is None:
                self.planes_up = split_planes(self.f32, upsample=True)
            return self.planes_up
        if self.planes is None:
            self.planes = split_planes(self.f32)
        return self.planes

    def get_blk_up(self):
        """blocked pair planes of the x2-upsampled tensor (operand of conv_halo_kernel), cached"""
        if self.blk_up is None:
            self.blk_up = split_blocked([(self.f32, True)])
        return self.blk_up


# ---- fork / join of independent work inside one module call (e.g. a decoder depth head next to the next block's
# up-convolution): the forked part runs on a per-(device, stream) side stream between two events.  Works eagerly and
# under CUDA-graph capture (the events become graph edges, the two parts parallel branches).  Protocol that keeps the
# caching allocator safe without record_stream: every fork starts with the side stream waiting on a fresh event of the
# main stream, every fork is joined before its results are used, and tensors crossing streams stay referenced until the
# join.
_SIDE_STREAMS = {}
_FORK = _os_environ_get("DVMVS_DECODER_FORK", "1") == "1"


class Fork:
    def __init__(self):
        self.active = _FORK and not N.DRYRUN and torch.cuda.is_available()
        if self.active:
            self.main = torch.cuda.current_stream()
            key = (self.main.device.index, self.main.cuda_stream)
            side = _SIDE_STREAMS.get(key)
            if side is None:
                side = _SIDE_STREAMS[key] = torch.cuda.Stream(device=self.main.device)
            self.side = side

    def __enter__(self):
        if self.active:
            ev = torch.cuda.Event()
            ev.record(self.main)
            self.side.wait_event(ev)
            self._ctx = torch.cuda.stream(self.side)
            self._ctx.__enter__()
            self._tag = stand_in_for(self.main)
            self._tag.__enter__()
        return self

    def __exit__(self, *exc):
        if self.active:
            self._done = torch.cuda.Event()
            self._done.record(self.side)
            self._tag.__exit__(*exc)
            self._ctx.__exit__(*exc)
        return False

    def join(self):
        if self.active:
            self.main.wait_event(self._done)


def to_act(x, name="input"):
    """API tensor (B,C,H,W) -> Act.  When the tensor is the untouched output of one of our modules (same storage, same
    autograd version), the operand layouts the PRODUCER KERNEL emitted next to the fp32 values (fp16 pair planes, blocked
    planes) come along; the Act handed back is a fresh object, so layouts derived later on demand (split kernels,
    x2-upsampled planes) live and die with the consumer's call and are never cached on a tensor the caller can reach --
    a CUDA-graph replay or an out-of-band write rewrites such a tensor without any notification.
    Caveat (INTEGRATION.md): a write through `.data` does not bump the version either; call dvmvs._ops.invalidate(t) after
    one, or the producer-emitted fp16 planes of `t` are stale."""
    a = getattr(x, "_dvmvs_act", None)
    if a is not None and a.f32.data_ptr() == x.data_ptr() and a.version == x._version and tuple(a.f32.shape) == (
            x.shape[0], x.shape[2], x.shape[3], x.shape[1]):
        return Act(a.f32, a.planes, a.blk, a.pair)
    return Act(to_nhwc(x, name))


def act_to_api(a):
    t = to_api(a.f32)
    keep = Act(a.f32, a.planes, a.blk, a.pair)  # what the producer emitted; nothing derived later is attached to it
    keep.version = t._version
    t._dvmvs_act = keep
    return t


def batch_slice(t, lo, hi):
    """t[lo:hi] along the batch axis of an API tensor, keeping the operand layouts its producer emitted as views (the engines run
    FeatureExtractor + FeatureShrinker once over the reference and measurement images stacked on the batch axis and hand the
    slices to the plane sweep; LookaheadFusionnet runs the encoder over several keyframes and hands slices to the decoder).
    The (hi, lo) pair planes always come along as two separate tensors (`pair`).  The stacked forms `planes` (2,B,H,W,C) and
    `blk` (2,B,C/8,H,W,8) come along as strided views only while no kernel reads lo planes (1-term operands everywhere): the
    kernels locate the lo plane at +B*H*W*C from the hi plane, which a batch slice of a bigger tensor does not satisfy; in
    3-term configurations the consumer derives contiguous planes from the fp32 slice instead (one split launch)."""
    v = t[lo:hi]
    a = getattr(t, "_dvmvs_act", None)
    if a is not None and a.f32.data_ptr() == t.data_ptr() and a.version == t._version and a.planes is not None:
        act = Act(a.f32[lo:hi], pair=(a.planes[0, lo:hi], a.planes[1, lo:hi]))
        if not lo_planes_needed():
            act.planes = a.planes[:, lo:hi]
            if a.blk is not None:
                act.blk = a.blk[:, lo:hi]
        act.version = v._version
        v._dvmvs_act = act
    return v


def act_pair(a):
    """(hi, lo) fp16 planes of an Act as two contiguous (B,H,W,C) tensors (a split kernel runs when the producer emitted none)."""
    if a.pair is not None:
        return a.pair
    p = a.get_planes()
    return p[0], p[1]


_SWEEP = _os_environ_get("DVMVS_SWEEP", "tc")      # "tc": tensor-core form of the plane sweep on the tc backend; "gather": always the fp32 gather kernel


def sweep_uses_tc(dot_product, channels, n_depth_levels, n_meas):
    return (_SWEEP == "tc" and _BACKEND == "tc" and dot_product and channels == 32 and 2 <= n_depth_levels <= SWEEP_TC_MAX_PLANES and
            n_meas * n_depth_levels <= 512 and n_meas <= 8)


def sweep_terms():
    return _TERMS_POLICY.get("sweep", _TC_TERMS)


def invalidate(t):
    """Drops the operand layouts attached to an API tensor (after modifying it through `.data`)."""
    if hasattr(t, "_dvmvs_act"):
        del t._dvmvs_act
    return t


class ConvLayer:
    """One dense convolution of the network: BN-folded weights for both backends + the channel split of its sources."""

    def __init__(self, pc, src_channels=None, pack_sources=False):
        """pack_sources: on the tensor-core path stage all sources into ONE concatenated operand tensor (fewer, fuller K
        chunks when the sources are narrow, e.g. refine.0's [32, 1, 3])."""
        self.pc = pc
        self.src_channels = list(src_channels) if src_channels is not None else [pc.cin]
        self.pack_sources = pack_sources
        self._ptc = None
        self._phalo = None

    def tc_eligible(self):
        pc = self.pc
        return pc.cout % 8 == 0 and pc.cout >= 16 and (pc.stride == 1 or _TC_STRIDE2) and pc.cin >= 16

    def uses_tc(self):
        return _BACKEND == "tc" and self.tc_eligible()

    def uses_halo(self, hout, wout, residual_mode, aux):
        pc = self.pc
        return (_HALO and self.uses_tc() and pc.stride == 1 and pc.ksize >= 3 and hout * wout >= _HALO_MIN_PIXELS and
                residual_mode in (N.RES_NONE, N.RES_SAME) and aux is None)

    def path(self, hout, wout, residual_mode=N.RES_NONE, aux=None):
        """which kernel family run() uses for an output map of hout x wout: 'halo', 'tc' or 'fp32'"""
        if self.uses_halo(hout, wout, residual_mode, aux):
            return "halo"
        return "tc" if self.uses_tc() else "fp32"

    def prestage_upsampled(self, act):
        """Stage the x2-upsampled operand of `act` (a source this layer reads with SRC_UPSAMPLE2X) now, on the current
        stream, in the layout run() will want; cached on the Act.  No-op on the fp32 path / for packed-source layers."""
        if self.pack_sources:
            return
        kind = self.path(2 * act.f32.shape[1], 2 * act.f32.shape[2])
        if kind == "halo":
            act.get_blk_up()
        elif kind == "tc":
            act.get_planes(upsample=True)

    def run_deferred(self, sources):
        """Tensor-core path only, single source: launches the convolution WITHOUT its split-K finishing pass when it splits and
        returns ("parts", (workspace, byte offset, n_parts, part_stride)); otherwise (no split / other path) returns None and the
        caller uses run()."""
        if not self.uses_tc() or self.pack_sources or len(sources) != 1:
            return None
        pc = self.pc
        a0, m0 = sources[0]
        hin = (a0.f32 if a0.f32 is not None else a0.planes[0]).shape[1]
        win = (a0.f32 if a0.f32 is not None else a0.planes[0]).shape[2]
        if m0 != N.SRC_DIRECT or self.uses_halo(hin, win, N.RES_NONE, None):
            return None
        if self._ptc is None:
            self._ptc = PackedConvTC(pc, self.src_channels, pc.weight.device)
        r = conv2d_tc([a0.get_planes()], self._ptc, terms=_TC_TERMS, want_f32=False, want_planes=False, defer_finish=True)
        if isinstance(r, tuple) and len(r) == 2 and r[0] == "parts":
            return r
        return None

    def run(self, sources, residual=None, residual_mode=N.RES_NONE, aux=None, want_f32=True, want_planes=True, want_blk=True,
            prestaged=None):
        """sources: list of (Act, mode).  Returns Act (or (Act, aux tensor)).  want_* only prune outputs of the
        tensor-core path (the fp32 path always produces fp32): want_f32 the fp32 tensor, want_planes the fp16 pair
        planes (what tensor-core consumers read), want_blk (halo path only) the blocked planes (what halo consumers read
        for SRC_DIRECT).  Callers prune an output only when they know every consumer of the result reads another one.
        prestaged: the concatenated blocked operand of a pack_sources layer on the halo path, already filled by the
        caller (split_blocked(..., only=, into=))."""
        pc = self.pc
        a0, m0 = sources[0]
        if a0.f32 is not None:
            hin, win = a0.f32.shape[1], a0.f32.shape[2]
        elif a0.planes is not None:
            hin, win = a0.planes.shape[2], a0.planes.shape[3]
        else:
            hin, win = a0.blk.shape[3], a0.blk.shape[4]
        if m0 == N.SRC_UPSAMPLE2X:
            hin, win = 2 * hin, 2 * win
        if self.uses_halo(hin, win, residual_mode, aux):
            if self._phalo is None:
                self._phalo = PackedConvHalo(pc, self.src_channels, pc.weight.device, concat_padded=self.pack_sources)
            # sources that already carry blocked planes (outputs of tensor-core layers on large maps) are used as they
            # are -- the kernel concatenates up to three sources along K; upsampled / fp32-only sources are staged
            if self.pack_sources:
                blks = [prestaged if prestaged is not None else split_blocked([(a.f32, mode == N.SRC_UPSAMPLE2X) for a, mode in sources])]
            else:
                blks = [a.blk if (mode == N.SRC_DIRECT and a.blk is not None) else
                        (a.blk_up if (mode == N.SRC_UPSAMPLE2X and a.blk_up is not None) else split_blocked([(a.f32, mode == N.SRC_UPSAMPLE2X)]))
                        for a, mode in sources]
            f32, oblk, onhwc = conv2d_halo(blks, self._phalo, residual=residual.f32 if residual is not None else None,
                                           terms=_TC_TERMS, want_f32=want_f32, want_blk=want_blk, want_nhwc=want_planes)
            return Act(f32, onhwc, oblk)
        if self.uses_tc():
            if self._ptc is None:
                self._ptc = PackedConvTC(pc, [pc.cin] if self.pack_sources else self.src_channels, pc.weight.device)
            if self.pack_sources:
                planes = [concat_planes([(a.f32, mode == N.SRC_UPSAMPLE2X) for a, mode in sources])]
            else:
                planes = [a.get_planes(upsample=(mode == N.SRC_UPSAMPLE2X)) for a, mode in sources]
            res = residual.f32 if residual is not None else None
            hout = (hin + 2 * ((pc.ksize - 1) // 2) - pc.ksize) // pc.stride + 1
            wout = (win + 2 * ((pc.ksize - 1) // 2) - pc.ksize) // pc.stride + 1
            blk_out = None
            if _HALO and want_planes and hout * wout >= _HALO_MIN_PIXELS and pc.cout % 8 == 0:
                # large map: its consumers are halo convolutions -> emit their operand layout from this epilogue too
                blk_out = torch.empty((2, planes[0].shape[1], pc.cout // 8, hout, wout, 8), dtype=torch.float16, device=planes[0].device)
            r = conv2d_tc(planes, self._ptc, residual=res, residual_mode=residual_mode, aux=aux, terms=_TC_TERMS,
                          want_f32=want_f32, want_planes=want_planes, blk_out=blk_out)
            out = Act(r[0], r[1], blk_out)
            return (out, r[2]) if aux is not None else out
        r = conv2d([(a.f32, mode) for a, mode in sources], pc, residual=residual.f32 if residual is not None else None,
                   residual_mode=residual_mode, aux=aux)
        if aux is not None:
            return Act(r[0]), r[1]
        return Act(r)
