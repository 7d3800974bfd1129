"""ctypes binding of libdvmvs_sm90.so (C ABI declared in include/dvmvs_b200.h).  Fails loudly when the library
has not been built: the product path has no fallback."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libdvmvs_sm90.so")

c_float_p = ctypes.c_void_p
ABI_VERSION = 6      # dvmvs_abi_version() the descriptor mirrors below were written for; bump with every descriptor / signature change
_lib = None

ACT_NONE, ACT_RELU, ACT_SIGMOID = 0, 1, 2
SRC_DIRECT, SRC_UPSAMPLE2X = 0, 1
SPLIT_UPSAMPLE2X, SPLIT_HI_ONLY = 1, 2
RES_NONE, RES_SAME, RES_NEAREST_UP = 0, 1, 2
SWEEP_DOT, SWEEP_SAD = 0, 1
LOSS_L1, LOSS_L1_INV, LOSS_L1_REL, LOSS_HUBER = 0, 1, 2, 3

# every symbol include/dvmvs_b200.h declares (tests check that the library exports all of them)
EXPORTED_SYMBOLS = [
    "dvmvs_abi_version", "dvmvs_set_programmatic_launch", "dvmvs_last_error_string", "dvmvs_kernel_launch_count", "dvmvs_plane_sweep_fused",
    "dvmvs_hidden_warp", "dvmvs_depth_reproject", "dvmvs_conv2d", "dvmvs_conv2d_tc", "dvmvs_conv2d_halo", "dvmvs_split_blocked", "dvmvs_split_planes", "dvmvs_stem_conv", "dvmvs_dwconv2d", "dvmvs_expand_dwconv", "dvmvs_lstm_gates",
    "dvmvs_upsample2x", "dvmvs_nchw_to_nhwc", "dvmvs_nhwc_to_nchw", "dvmvs_preprocess_rgb", "dvmvs_tsdf_integrate",
    "dvmvs_plane_sweep_backward", "dvmvs_hidden_warp_backward", "dvmvs_lstm_gates_backward", "dvmvs_depth_loss_forward",
    "dvmvs_depth_loss_backward", "dvmvs_plane_sweep_fused_h16", "dvmvs_plane_sweep_tc", "dvmvs_lstm_gates_parts", "dvmvs_conv2d_tc_ksplit", "dvmvs_plane_sweep_tc_set_timeline",
    "dvmvs_mesh_scratch_bytes", "dvmvs_mesh_count", "dvmvs_mesh_extract", "dvmvs_tsdf_raycast",
]


class ConvDesc(ctypes.Structure):
    """mirror of dvmvs_conv_desc"""
    _fields_ = [
        ("src", ctypes.c_void_p * 3), ("src_channels", ctypes.c_int * 3), ("src_mode", ctypes.c_int * 3),
        ("n_src", ctypes.c_int),
        ("weight", ctypes.c_void_p), ("bias", ctypes.c_void_p), ("residual", ctypes.c_void_p),
        ("residual_mode", ctypes.c_int), ("Hr", ctypes.c_int), ("Wr", ctypes.c_int),
        ("out", ctypes.c_void_p), ("aux_out", ctypes.c_void_p),
        ("aux_mult", ctypes.c_float), ("aux_base", ctypes.c_float),
        ("B", ctypes.c_int), ("Hin", ctypes.c_int), ("Win", ctypes.c_int), ("Cout", ctypes.c_int),
        ("ksize", ctypes.c_int), ("stride", ctypes.c_int), ("act", ctypes.c_int),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_longlong),
    ]


class ConvTcDesc(ctypes.Structure):
    """mirror of dvmvs_conv_tc_desc"""
    _fields_ = [
        ("src_planes", ctypes.c_void_p * 3), ("src_channels", ctypes.c_int * 3), ("n_src", ctypes.c_int),
        ("w_hi", ctypes.c_void_p), ("w_lo", ctypes.c_void_p),
        ("w_rows", ctypes.c_int), ("ktot", ctypes.c_int), ("block_n", ctypes.c_int), ("terms", ctypes.c_int),
        ("allow_split", ctypes.c_int),
        ("bias", ctypes.c_void_p), ("residual", ctypes.c_void_p),
        ("residual_mode", ctypes.c_int), ("Hr", ctypes.c_int), ("Wr", ctypes.c_int),
        ("out_f32", ctypes.c_void_p), ("out_planes", ctypes.c_void_p), ("aux_out", ctypes.c_void_p),
        ("aux_mult", ctypes.c_float), ("aux_base", ctypes.c_float),
        ("B", ctypes.c_int), ("Hin", ctypes.c_int), ("Win", ctypes.c_int), ("Cout", ctypes.c_int),
        ("ksize", ctypes.c_int), ("stride", ctypes.c_int), ("act", ctypes.c_int),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_longlong),
        ("out_blk", ctypes.c_void_p),
        ("out_hi_only", ctypes.c_int), ("defer_finish", ctypes.c_int),
    ]


DRYRUN = os.environ.get("DVMVS_DRYRUN") == "1"     # host-logic smoke tests only: kernels are not executed, results are garbage


class _DryRunLib:
    """Stands in for the shared library when DVMVS_DRYRUN=1: every entry point returns 0 without doing anything, so the
    Python plumbing (shapes, descriptors, module wiring) can be exercised on a machine without a GPU.  Never used by the
    product path."""

    def __getattr__(self, name):
        if name == "dvmvs_last_error_string":
            return lambda: b"dry run"
        if name == "dvmvs_kernel_launch_count":
            return lambda: 0
        return lambda *a, **k: 0


class ConvHaloDesc(ctypes.Structure):
    """mirror of dvmvs_conv_halo_desc"""
    _fields_ = [
        ("src_blk", ctypes.c_void_p * 3), ("src_c8", ctypes.c_int * 3), ("n_src", ctypes.c_int),
        ("w_hi", ctypes.c_void_p), ("w_lo", ctypes.c_void_p),
        ("n_groups", ctypes.c_int), ("kc", ctypes.c_int), ("block_n", ctypes.c_int), ("terms", ctypes.c_int),
        ("bias", ctypes.c_void_p), ("residual", ctypes.c_void_p),
        ("out_f32", ctypes.c_void_p), ("out_blk", ctypes.c_void_p), ("out_nhwc", ctypes.c_void_p),
        ("B", ctypes.c_int), ("H", ctypes.c_int), ("W", ctypes.c_int), ("Cout", ctypes.c_int),
        ("ksize", ctypes.c_int), ("act", ctypes.c_int),
        ("w_cat", ctypes.c_void_p),
        ("out_hi_only", ctypes.c_int),
    ]


def lib():
    global _lib
    if _lib is None and DRYRUN:
        _lib = _DryRunLib()
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError("dvmvs: %s not found -- build it with `python deep-video-mvs_b200/build_native.py` "
                               "(there is no CPU / eager fallback)" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        if L.dvmvs_abi_version() != ABI_VERSION:
            raise RuntimeError("dvmvs: %s has ABI version %d, this binding was written for %d -- rebuild it with "
                               "`python deep-video-mvs_b200/build_native.py --force`" % (LIB_PATH, L.dvmvs_abi_version(), ABI_VERSION))
        i, f, p = ctypes.c_int, ctypes.c_float, ctypes.c_void_p
        L.dvmvs_last_error_string.restype = ctypes.c_char_p
        L.dvmvs_set_programmatic_launch.argtypes = [i]
        L.dvmvs_plane_sweep_fused.argtypes = [p, p, p, p, p, p, i, i, i, i, i, i, f, f, i, p]
        L.dvmvs_plane_sweep_generic.argtypes = [p, p, p, p, p, p, i, i, i, i, i, i, f, f, i, p]
        L.dvmvs_plane_sweep_fused_h16.argtypes = [p, p, p, p, p, p, i, i, i, i, i, i, f, f, p]
        L.dvmvs_plane_sweep_tc.argtypes = [p, p, p, p, p, p, p, p, i, i, i, i, i, f, f, i, p]
        L.dvmvs_plane_sweep_tc_set_timeline.argtypes = [p]
        L.dvmvs_hidden_warp.argtypes = [p, p, p, p, p, p, i, i, i, i, f, p]
        L.dvmvs_depth_reproject.argtypes = [p, p, p, p, p, p, i, i, i, p]
        L.dvmvs_conv2d.argtypes = [ctypes.POINTER(ConvDesc), p]
        L.dvmvs_conv2d_tc.argtypes = [ctypes.POINTER(ConvTcDesc), p]
        L.dvmvs_conv2d_halo.argtypes = [ctypes.POINTER(ConvHaloDesc), p]
        L.dvmvs_split_blocked.argtypes = [p, p, i, i, i, i, i, i, i, i, p]
        L.dvmvs_split_planes.argtypes = [p, p, i, i, i, i, i, i, i, i, p]
        L.dvmvs_stem_conv.argtypes = [p, p, p, p, i, i, i, p]
        L.dvmvs_dwconv2d.argtypes = [p, p, p, p, p, i, i, i, i, i, i, i, p]
        L.dvmvs_expand_dwconv.argtypes = [p, i, i, i, i, p, p, i, i, p, i, p, p, i, i, i, i, i, i, p, p]
        L.dvmvs_lstm_gates.argtypes = [p, p, p, p, i, i, i, i, p]
        L.dvmvs_lstm_gates_parts.argtypes = [p, i, ctypes.c_longlong, p, p, p, p, i, i, i, i, p]
        L.dvmvs_conv2d_tc_ksplit.argtypes = [ctypes.POINTER(ConvTcDesc)]
        L.dvmvs_upsample2x.argtypes = [p, p, i, i, i, i, p]
        L.dvmvs_preprocess_rgb.argtypes = [p, i, i, i, i, i, i, p, i, i, i, f, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), p]
        L.dvmvs_nchw_to_nhwc.argtypes = [p, p, i, i, i, i, p]
        L.dvmvs_nhwc_to_nchw.argtypes = [p, p, i, i, i, i, p]
        d = ctypes.c_double
        L.dvmvs_tsdf_integrate.argtypes = [p, p, p, i, i, i, ctypes.POINTER(ctypes.c_float), d, d, p, i, p, i, i, i,
                                           ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double), d, p, p]
        ll = ctypes.c_longlong
        L.dvmvs_mesh_scratch_bytes.argtypes = [i, i, i, ctypes.POINTER(ll)]
        L.dvmvs_mesh_count.argtypes = [p, i, i, i, p, ll, p]
        L.dvmvs_mesh_extract.argtypes = [p, p, i, i, i, ctypes.POINTER(ctypes.c_float), f, p, ll, i, i, p, p, p, p, p, p]
        L.dvmvs_tsdf_raycast.argtypes = [p, p, i, i, i, ctypes.POINTER(ctypes.c_float), d, d, p, i, i, i, p, p, p, p]
        L.dvmvs_plane_sweep_backward.argtypes = [p, p, p, p, p, p, p, p, i, i, i, i, i, i, f, f, i, p]
        L.dvmvs_hidden_warp_backward.argtypes = [p, p, p, p, p, p, i, i, i, i, f, p]
        L.dvmvs_lstm_gates_backward.argtypes = [p, p, p, p, p, p, i, i, i, i, p]
        ip, fp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_float)
        L.dvmvs_depth_loss_forward.argtypes = [p, ip, ip, i, p, p, i, i, i, p]
        L.dvmvs_depth_loss_backward.argtypes = [p, p, ip, ip, fp, i, p, p, p, i, i, i, i, p]
        _lib = L
    return _lib


def check(rc, what):
    if rc != 0:
        raise RuntimeError("dvmvs native call %s failed (%d): %s" % (what, rc, lib().dvmvs_last_error_string().decode()))


def launch_count():
    return lib().dvmvs_kernel_launch_count()
