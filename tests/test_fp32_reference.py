"""The fp32 CUDA-core kernels (depth heads and direct convolution of dvmvs_conv2d, stem, depthwise, x2 upsampling) against the fp64
reference of tests/fp32_reference.py element by element, and the operand staging (dvmvs_split_planes, dvmvs_split_blocked) bit for
bit against fp16_split of the values it stages.  Prints the worst err / bound of every case."""

import numpy as np
import pytest
import torch

from tests import fp32_reference as R
from tests.tc_reference import ACT_NONE, ACT_RELU, ACT_SIGMOID, check

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENTINEL = torch.tensor(7.0).half().view(torch.int16)


def _randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


class _NoWorkspace:
    """dvmvs_conv2d without its split-K workspace while active"""

    def __enter__(self):
        from dvmvs import _native as N
        self.L = N.lib()
        self.real = self.L.dvmvs_conv2d

        def conv(dref, stream):
            dref._obj.workspace, dref._obj.workspace_bytes = None, 0
            return self.real(dref, stream)
        self.L.dvmvs_conv2d = conv
        return self

    def __exit__(self, *exc):
        self.L.dvmvs_conv2d = self.real
        return False


# ------------------------------------------------------------------------------------------------ dvmvs_conv2d
CONV_CASES = [
    # name, B, H, W, [(channels, upsampled)], Cout, k, stride, act, aux, residual mode
    ("head32_16x16_cin128_aux", 1, 16, 16, [(128, False)], 1, 3, 1, ACT_SIGMOID, (3.9, 0.05), 0),
    ("head8_40x48_cin64_aux", 1, 40, 48, [(64, False)], 1, 3, 1, ACT_SIGMOID, (3.9, 0.05), 0),
    ("head8_full_res_256x256_cin32", 1, 256, 256, [(32, False)], 1, 3, 1, ACT_SIGMOID, (3.9, 0.05), 0),
    ("direct_cout1_cin20_odd", 2, 13, 11, [(20, False)], 1, 3, 1, ACT_SIGMOID, (2.0, 0.5), 0),
    ("direct_cout3_k5_s2_odd", 1, 19, 23, [(16, False)], 3, 5, 2, ACT_RELU, None, 0),
    ("direct_cout40_k1_res_same", 1, 8, 8, [(192, False)], 40, 1, 1, ACT_NONE, None, 1),
    ("direct_cout40_k3_s2_upsampled_concat", 1, 18, 22, [(16, True), (24, False), (1, True)], 40, 3, 2, ACT_RELU, None, 0),
    ("direct_cout32_k1_nearest_up", 1, 16, 16, [(24, False)], 32, 1, 1, ACT_NONE, None, 2),
    ("direct_deep_k3_split", 1, 8, 10, [(512, False), (64, False)], 96, 3, 1, ACT_RELU, None, 0),
    ("direct_k5_split_odd", 1, 7, 9, [(256, False)], 3, 5, 1, ACT_NONE, None, 0),
]


def _conv_case(ops, case):
    name, B, H, W, srcs, Cout, k, stride, act, aux, res_mode = case
    seed = sum(map(ord, name))
    xs = [_randn((B, H // (2 if up else 1), W // (2 if up else 1), c), seed + i) for i, (c, up) in enumerate(srcs)]
    cin = sum(c for c, _ in srcs)
    pc = ops.PackedConv(_randn((Cout, cin, k, k), seed + 10, (2.0 / (cin * k * k)) ** 0.5), _randn((Cout,), seed + 11, 0.1), None,
                        stride=stride, act=act)
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    res = None
    if res_mode == 1:
        res = _randn((B, Ho, Wo, Cout), seed + 12)
    elif res_mode == 2:
        res = _randn((B, Ho // 2, Wo // 2, Cout), seed + 12)
    return xs, pc, res, (Ho, Wo)


def _path(case):
    name, B, H, W, srcs, Cout, k, stride, act, aux, res_mode = case
    cin = sum(c for c, _ in srcs)
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    if Cout == 1 and len(srcs) == 1 and not srcs[0][1] and k == 3 and stride == 1 and cin % 32 == 0 and res_mode == 0:
        return "head%d" % R.head_lanes(B, Ho, Wo, cin), 1
    from dvmvs import _ops as ops
    return "direct", R.direct_ksplit(B, Ho, Wo, Cout, [c for c, _ in srcs], ops.WORKSPACE_BYTES - 16384)


def launched_conv_branch(fn):
    """runs fn (one dvmvs_conv2d call) under torch.profiler; returns (the branch the library launched: "head8" / "head32" /
    "direct K/S" / "direct K/S split", fn's result) from the names of the kernels it ran"""
    import re
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):         # the call is repeatable; the profiler now and then delivers no kernel record for it: run it again
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with torch.no_grad():
                r = fn()
                torch.cuda.synchronize()
        names = " ".join(e.key for e in prof.key_averages())
        head = re.search(r"conv_head_kernel<\s*(\d+)\s*>", names)
        direct = re.search(r"conv2d_direct_kernel<\s*(\d+)\s*,\s*(\d+)\s*>", names)
        if head or direct:
            break
    assert bool(head) != bool(direct), "dvmvs_conv2d launched %s" % names
    if head:
        return "head" + head.group(1), r
    return "direct %s/%s%s" % (direct.group(1), direct.group(2), " split" if "conv_epilogue_kernel" in names else ""), r


def conv_chain(branch, cin_total, src_channels, k):
    """the longest fmaf chain of the launched branch; a split launch is charged its longest possible part (one chunk per part is the
    shortest, the whole K the longest) plus one addition per chunk, whatever split count the host chose"""
    if branch.startswith("head"):
        lanes = int(branch[4:])
        return 3 * cin_total // lanes + 2 + int(np.log2(lanes))
    chunks = sum((c + R.CK - 1) // R.CK for c in src_channels)
    return k * k * R.CK * chunks + (chunks if branch.endswith("split") else 0)


def test_conv_cases_reach_every_path():
    paths = {_path(c)[0] for c in CONV_CASES}
    assert paths == {"head8", "head32", "direct"}
    assert {c[5] for c in CONV_CASES if _path(c)[0] == "direct"} >= {1, 3, 40}
    assert any(_path(c)[1] > 1 for c in CONV_CASES) and {c[6] for c in CONV_CASES} == {1, 3, 5} and {c[7] for c in CONV_CASES} == {1, 2}
    assert any(_path(c)[0] == "head8" and c[2] * c[3] == 256 * 256 for c in CONV_CASES)


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv2d_vs_fp64_reference(case):
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    name, B, H, W, srcs, Cout, k, stride, act, aux, res_mode = case
    xs, pc, res, _ = _conv_case(ops, case)
    path, ksplit = _path(case)
    expected = path if path.startswith("head") else "direct %d/%d%s" % (k, stride, " split" if ksplit > 1 else "")
    srcs_args = lambda: [(x, N.SRC_UPSAMPLE2X if up else N.SRC_DIRECT) for x, (_, up) in zip(xs, srcs)]
    for with_ws in (True, False):
        if with_ws:
            branch, r = launched_conv_branch(lambda: ops.conv2d(srcs_args(), pc, residual=res, residual_mode=res_mode, aux=aux))
            assert branch == expected, "%s: the library launched %s, the case expects %s" % (name, branch, expected)
        else:
            with _NoWorkspace():
                branch, r = launched_conv_branch(lambda: ops.conv2d(srcs_args(), pc, residual=res, residual_mode=res_mode, aux=aux))
            assert not branch.endswith("split"), "%s: split without a workspace" % name
        out, aux_out = r if aux is not None else (r, None)
        ref = R.conv_reference([(_nchw(x), up) for x, (_, up) in zip(xs, srcs)], pc.weight, stride, pc.bias,
                               None if res is None else _nchw(res), res_mode, act, aux, chain=conv_chain(branch, pc.cin, [c for c, _ in srcs], k))
        worst = check("%s %s" % (name, branch), _nchw(out), ref.y, ref.bound)[0]
        if aux is not None:
            worst = max(worst, check("%s aux" % name, _nchw(aux_out), ref.aux, ref.aux_bound)[0])
        print("\nconv2d %-40s %-16s err/bound %.3f" % (name, branch, worst))
        if path.startswith("head") or ksplit == 1:
            break


# ------------------------------------------------------------------------------------------------ stem, depthwise, upsample
@pytest.mark.parametrize("bias", [True, False])
def test_stem_conv_vs_fp64_reference(bias):
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    B, H, W = 2, 37, 29
    img = _randn((B, 3, H, W), 1)
    w = _randn((3, 3, 3, 32), 2, 0.3)
    b = _randn((32,), 3, 0.1) if bias else None
    y = torch.empty((B, (H - 1) // 2 + 1, (W - 1) // 2 + 1, 32), device=DEV)
    N.check(N.lib().dvmvs_stem_conv(img.data_ptr(), w.data_ptr(), b.data_ptr() if bias else None, y.data_ptr(), B, H, W, ops._stream()),
            "stem_conv")
    torch.cuda.synchronize()
    ref = R.stem_reference(img, w, b)
    print("\nstem B=%d %dx%d bias=%s  err/bound %.3f" % (B, H, W, bias, check("stem", _nchw(y), ref.y, ref.bound)[0]))


DW_CASES = [  # B, H, W, C, k, stride, act, bias
    (1, 17, 15, 4, 3, 2, ACT_RELU, True),
    (1, 9, 11, 1152, 5, 1, ACT_NONE, False),
    (2, 13, 9, 72, 5, 2, ACT_RELU, True),
    (1, 16, 16, 32, 3, 1, ACT_NONE, True),
]


@pytest.mark.parametrize("case", DW_CASES)
def test_dwconv_vs_fp64_reference(case):
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    B, H, W, C, k, stride, act, bias = case
    x = _randn((B, H, W, C), C + k)
    w = _randn((k, k, C), C + k + 1, 0.3)
    b = _randn((C,), C + k + 2, 0.1) if bias else None
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    y = torch.empty((B, Ho, Wo, C), device=DEV)
    planes = torch.empty((2, B, Ho, Wo, C), dtype=torch.float16, device=DEV) if C % 8 == 0 else None
    N.check(N.lib().dvmvs_dwconv2d(x.data_ptr(), w.data_ptr(), b.data_ptr() if bias else None, y.data_ptr(),
                                   planes.data_ptr() if planes is not None else None, B, H, W, C, k, stride, act, ops._stream()), "dwconv2d")
    torch.cuda.synchronize()
    ref = R.dwconv_reference(_nchw(x), w, b, stride, act)
    worst = check("dwconv %s" % (case,), _nchw(y), ref.y, ref.bound)[0]
    if planes is not None:           # the fp16 pair is the split of the same call's fp32 output, bit for bit
        eh, el = R.split_expected(y)
        assert torch.equal(planes[0].view(torch.int16), eh.view(torch.int16)) and torch.equal(planes[1].view(torch.int16), el.view(torch.int16))
    print("\ndwconv %s  err/bound %.3f" % (case, worst))


@pytest.mark.parametrize("shape", [(2, 5, 7, 3), (1, 8, 10, 32), (1, 64, 64, 1)])
def test_upsample2x_vs_fp64_reference(shape):
    from dvmvs import _ops as ops
    x = _randn(shape, sum(shape))
    with torch.no_grad():
        y = ops.upsample2x(x)
        torch.cuda.synchronize()
    ref, bound = R.upsample_reference(_nchw(x))
    print("\nupsample2x %s  err/bound %.3f" % (shape, check("upsample2x %s" % (shape,), _nchw(y), ref, bound)[0]))


def test_layout_transposes_exact():
    from dvmvs import _ops as ops
    x = _randn((2, 37, 9, 13), 4)
    nhwc = ops.to_nhwc(x)
    assert torch.equal(nhwc, x.permute(0, 2, 3, 1))
    assert torch.equal(ops.to_nchw_contiguous(nhwc), x)


# ------------------------------------------------------------------------------------------------ operand staging
def _blk_channels_last(p):
    """blocked planes (2,B,C8,H,W,8) -> (2,B,H,W,C8*8)"""
    two, B, C8, H, W, _ = p.shape
    return p.permute(0, 1, 3, 4, 2, 5).reshape(two, B, H, W, C8 * 8)


def _stage(kind, x, up, Cs, off, cover, hi_only=False):
    """one sentinel-filled staging call; returns the (hi, lo) planes channel-last and the staged fp32 values"""
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    B, H, W, C = x.shape
    f = 2 if up else 1
    if kind == "planes":
        planes = torch.empty((2, B, H * f, W * f, Cs), dtype=torch.float16, device=DEV)
        planes.view(torch.int16).fill_(int(SENTINEL))
        N.check(N.lib().dvmvs_split_planes(x.data_ptr(), planes.data_ptr(), B, H, W, C, Cs, 1 if up else 0, off, cover, ops._stream()), "split_planes")
        cl = planes
    else:
        planes = torch.empty((2, B, Cs // 8, H * f, W * f, 8), dtype=torch.float16, device=DEV)
        planes.view(torch.int16).fill_(int(SENTINEL))
        flags = (N.SPLIT_UPSAMPLE2X if up else 0) | (N.SPLIT_HI_ONLY if hi_only else 0)
        N.check(N.lib().dvmvs_split_blocked(x.data_ptr(), planes.data_ptr(), B, H, W, C, Cs // 8, flags, off, cover, ops._stream()), "split_blocked")
        cl = _blk_channels_last(planes)
    torch.cuda.synchronize()
    return cl[0], cl[1], ops.upsample2x(x) if up else x


@pytest.mark.parametrize("kind", ["planes", "blocked"])
@pytest.mark.parametrize("C", [1, 3, 12, 32, 72])
@pytest.mark.parametrize("up", [False, True])
def test_staging_bit_exact(kind, C, up):
    x = _randn((2, 5, 7, C), C)
    Cs = -(-(C + 8) // 8) * 8 + 8                   # room on both sides of the window
    for off, cover in ((0, -(-C // 8) * 8), (8, -(-C // 8) * 8 + 8)):
        hi, lo, values = _stage(kind, x, up, Cs, off, cover)
        R.check_staged("%s C=%d up=%s window [%d,+%d)" % (kind, C, up, off, cover), hi, lo, values, off, cover, SENTINEL)
    if up:
        ref, bound = R.upsample_reference(_nchw(x))
        check("upsample2x C=%d" % C, _nchw(values), ref, bound)
    if kind == "blocked":
        hi, lo, values = _stage(kind, x, up, Cs, 8, -(-C // 8) * 8, hi_only=True)
        R.check_staged("blocked hi-only C=%d" % C, hi, lo, values, 8, -(-C // 8) * 8, SENTINEL, hi_only=True)


@pytest.mark.parametrize("kind", ["planes", "blocked"])
@pytest.mark.parametrize("up", [False, True])
def test_staging_misaligned_view(kind, up):
    """a view 4 bytes past a 16-byte boundary (what to_nhwc can return for a channels_last slice): the scalar loads"""
    B, H, W, C = 1, 6, 5, 32
    buf = _randn((B * H * W * C + 1,), 77)
    x = buf[1:].view(B, H, W, C)
    assert x.data_ptr() % 16 == 4
    hi, lo, values = _stage(kind, x, up, 40, 0, 40)
    R.check_staged("misaligned %s up=%s" % (kind, up), hi, lo, values, 0, 40, SENTINEL)


def test_concat_planes_three_sources_last_zero_fills():
    from dvmvs import _ops as ops
    a, b, c = _randn((1, 8, 6, 12), 1), _randn((1, 4, 3, 5), 2), _randn((1, 8, 6, 3), 3)
    with torch.no_grad():
        planes = ops.concat_planes([(a, False), (b, True), (c, False)])
        torch.cuda.synchronize()
    assert planes.shape[-1] == 24
    R.check_staged("concat_planes source 0", planes[0], planes[1], a, 0, 12, SENTINEL, others=False)
    R.check_staged("concat_planes source 1", planes[0], planes[1], ops.upsample2x(b), 12, 5, SENTINEL, others=False)
    R.check_staged("concat_planes source 2", planes[0], planes[1], c, 17, 7, SENTINEL, others=False)


def test_split_blocked_only_into_two_calls():
    """the decoder's staging: sources 0 and 2 first, source 1 later into the same tensor (_blocks.py)"""
    from dvmvs import _ops as ops
    d4, s2, image = _randn((1, 16, 20, 1), 4), _randn((1, 16, 20, 32), 5), _randn((1, 32, 40, 3), 6)
    srcs = [(d4, True), (s2, True), (image, False)]
    meta = [(tuple(t.shape) if i == 1 else t, up) for i, (t, up) in enumerate(srcs)]
    with torch.no_grad():
        buf = ops.split_blocked(meta, only=(0, 2))
        buf.view(torch.int16)[:, :, 1:5].fill_(int(SENTINEL))     # source 1's blocks are staged by the second call only
        ops.split_blocked(srcs, only=(1,), into=buf)
        torch.cuda.synchronize()
    check_blocked_staging("decoder staging", buf, srcs, None)


def check_blocked_staging(what, buf, sources, only):
    """a split_blocked operand tensor against the fp16 split of each staged source (upsample2x's output for an upsampled one)"""
    from dvmvs import _ops as ops
    cl = _blk_channels_last(buf)
    hi_only = not ops.lo_planes_needed()
    off = 0
    for i, (t, up) in enumerate(sources):
        C = (tuple(t) if isinstance(t, (tuple, list)) else tuple(t.shape))[3]
        cover = -(-C // 8) * 8
        if only is None or i in only:
            lo = torch.full_like(cl[1], 7.0) if hi_only else cl[1]       # the lo plane is not written at 1 term: not checked then
            R.check_staged("%s source %d" % (what, i), cl[0], lo, ops.upsample2x(t) if up else t, off, cover, SENTINEL, hi_only=hi_only,
                           others=False)
        off += cover
