"""conv_tc_kernel (+ its finishing kernel), conv_halo_kernel, expand_dw_kernel and lstm_gates_kernel against a float64 reference
computed from the fp16 operands the kernels multiply (tests/tc_reference.py): every element within the stated accumulation
bound, fp16 outputs bit-exact against the fp32 output of the same call.  Prints the worst err / bound and the worst
err / (u * n * S) -- the accumulation constant the bound charges C_ACC for -- of every case."""
import pytest
import torch
import torch.nn.functional as F

from tests import tc_reference as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENTINEL = 7.0


@pytest.fixture
def ops():
    from dvmvs import _ops
    old = (_ops._BACKEND, _ops._TC_TERMS_BASE, _ops._TC_STRIDE2)
    try:
        yield _ops
    finally:
        _ops.set_conv_backend(old[0], terms=old[1], stride2=old[2])


def _randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _blk_to_nchw(blk):
    """one plane of a blocked tensor (B,C8,H,W,8) -> (B,C8*8,H,W)"""
    B, C8, H, W, _ = blk.shape
    return blk.permute(0, 1, 4, 2, 3).reshape(B, C8 * 8, H, W)


class _Raw:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f2", "data": (ptr, False), "version": 2}


def _fill_lo(ptr, n):
    if ptr:
        torch.as_tensor(_Raw(ptr + 2 * n, n), device=DEV).fill_(SENTINEL)


class NativeSpy:
    """Wraps the library's dvmvs_conv2d_tc / dvmvs_conv2d_halo while active: records the split count (dvmvs_conv2d_tc_ksplit on
    the same descriptor), the output tile, block_n, terms and batch of every conv2d_tc launch, and fills the lo plane of every fp16 output of a
    hi-plane-only launch with SENTINEL first, so that a test can tell the plane was left alone."""

    def __enter__(self):
        from dvmvs import _native as N
        self.L = L = N.lib()
        self.real = {"dvmvs_conv2d_tc": L.dvmvs_conv2d_tc, "dvmvs_conv2d_halo": L.dvmvs_conv2d_halo}
        self.tc = []

        def tc(dref, stream):
            d = dref._obj
            pad = (d.ksize - 1) // 2
            Ho, Wo = (d.Hin + 2 * pad - d.ksize) // d.stride + 1, (d.Win + 2 * pad - d.ksize) // d.stride + 1
            self.tc.append({"ksplit": int(L.dvmvs_conv2d_tc_ksplit(dref)), "tile": "8x16" if (Wo <= 8 and Ho > 8) else "16x8",
                            "block_n": int(d.block_n), "terms": int(d.terms), "B": int(d.B)})
            if d.out_hi_only:
                n = d.B * Ho * Wo * d.Cout
                _fill_lo(d.out_planes, n)
                _fill_lo(d.out_blk, n)
            return self.real["dvmvs_conv2d_tc"](dref, stream)

        def halo(dref, stream):
            d = dref._obj
            if d.out_hi_only:
                n = d.B * d.H * d.W * d.Cout
                _fill_lo(d.out_nhwc, n)
                _fill_lo(d.out_blk, n)
            return self.real["dvmvs_conv2d_halo"](dref, stream)

        L.dvmvs_conv2d_tc, L.dvmvs_conv2d_halo = tc, halo
        return self

    def __exit__(self, *exc):
        for k, v in self.real.items():
            setattr(self.L, k, v)
        return False


def _report(line):
    print(line, flush=True)


def _check_outputs(what, ref, f32=None, planes=None, blk=None, aux=None, hi_only=False):
    """f32 (B,H,W,C) fp32, planes (2,B,H,W,C) fp16, blk (2,B,C/8,H,W,8) fp16 of one call against `ref` (NCHW fp64).
    Returns (worst err / bound, worst accumulation constant)."""
    scale = ref.eps_acc / R.C_ACC
    rows = []
    if f32 is not None:
        R.check(what + " fp32", _nchw(f32), ref.y, ref.bound, ref.S, scale, rows)
    for name, t in (("planes", planes), ("blk", blk)):
        if t is None:
            continue
        hi = _nchw(t[0]) if name == "planes" else _blk_to_nchw(t[0])
        lo = None if hi_only else (_nchw(t[1]) if name == "planes" else _blk_to_nchw(t[1]))
        if hi_only:
            assert bool((t[1] == SENTINEL).all()), "%s: hi-only launch wrote the lo plane of its %s output" % (what, name)
        if f32 is not None:             # the fp16 outputs are the rounding of the fp32 output of the same call, bit for bit
            x = _nchw(f32)
            assert torch.equal(hi, x.half()), "%s: %s hi plane != fp16_rn(fp32 output)" % (what, name)
            if lo is not None:
                assert torch.equal(lo, (x - hi.float()).half()), "%s: %s lo plane != fp16_rn(fp32 - hi)" % (what, name)
        elif lo is None:
            R.check(what + " " + name + " hi", hi.float(), ref.y, R.fp16_bound(ref.y, ref.bound), report=rows)
        else:
            R.check(what + " " + name + " hi+lo", hi.float() + lo.float(), ref.y, R.fp16_bound(ref.y, ref.bound, pair=True), report=rows)
    if aux is not None:
        R.check(what + " aux", _nchw(aux), ref.aux, ref.aux_bound, report=rows)
    return max(r[1] for r in rows), max(r[2] for r in rows)


# ------------------------------------------------------------------------------------------------ conv_tc_kernel
TC_CASES = [
    # name, B, H, W, [src channels], Cout, k, stride, bias, residual mode, act, aux, outputs (f: fp32, p: planes, b: blocked), block_n
    ("k3_mixed_chunks_res_same", 2, 13, 21, [64, 40, 8], 96, 3, 1, True, R.RES_SAME, R.ACT_RELU, None, "fpb", 32),
    ("k3_tile8x16_nearest_up", 2, 20, 7, [32], 64, 3, 1, False, R.RES_NEAREST_UP, R.ACT_NONE, None, "fp", 64),
    ("k1_sigmoid_aux_partial_ntile", 3, 9, 17, [64], 40, 1, 1, True, R.RES_NONE, R.ACT_SIGMOID, (3.9, 0.05), "f", 32),
    ("k5_s2_odd_cout20_res_same", 2, 23, 19, [32, 24], 20, 5, 2, True, R.RES_SAME, R.ACT_RELU, None, "f", 32),
    ("k3_cout12_nearest_up_sigmoid_aux", 1, 15, 9, [16], 12, 3, 1, False, R.RES_NEAREST_UP, R.ACT_SIGMOID, (2.0, 0.5), "f", 32),
    ("k3_s2_n128_blk", 2, 17, 33, [128], 256, 3, 2, True, R.RES_NONE, R.ACT_RELU, None, "fpb", 128),
    ("k5_three_sources_planes_only_n64", 1, 16, 24, [64, 1, 3], 72, 5, 1, True, R.RES_NONE, R.ACT_RELU, None, "p", 64),
    ("k1_nobias_res_same_n64", 2, 8, 8, [96], 64, 1, 1, False, R.RES_SAME, R.ACT_NONE, None, "fpb", 64),
    ("k3_tile8x16_s2_odd_blk_n64", 1, 33, 15, [32, 32], 64, 3, 2, True, R.RES_NEAREST_UP, R.ACT_RELU, None, "fpb", 64),
]


def _tc_operands(ops, case):
    name, B, H, W, chans, Cout, k, stride, bias, res_mode, act, aux, outs, block_n = case
    seed = sum(map(ord, name))
    xs = [_randn((B, H, W, c), seed + i) for i, c in enumerate(chans)]
    cin = sum(chans)
    w = _randn((Cout, cin, k, k), seed + 10, (2.0 / (cin * k * k)) ** 0.5)
    b = _randn((Cout,), seed + 11, 0.1) if bias else None
    pc = ops.PackedConv(w, b, None, stride=stride, act=act)
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    res = None
    if res_mode == R.RES_SAME:
        res = _randn((B, Ho, Wo, Cout), seed + 12)
    elif res_mode == R.RES_NEAREST_UP:
        res = _randn((B, (Ho + 1) // 2, (Wo + 1) // 2, Cout), seed + 12)
    return xs, pc, res, (Ho, Wo)


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("case", TC_CASES, ids=[c[0] for c in TC_CASES])
def test_conv2d_tc_vs_fp64_reference(ops, case, terms):
    name, B, H, W, chans, Cout, k, stride, bias, res_mode, act, aux, outs, block_n = case
    ops.set_conv_backend("tc", terms=terms)          # terms=1: no consumer reads lo planes -> the launches write hi planes only
    xs, pc, res, (Ho, Wo) = _tc_operands(ops, case)
    ptc = ops.PackedConvTC(pc, chans, DEV)
    planes = [ops.split_planes(x) for x in xs]
    xh, xl = zip(*[R.fp16_split(_nchw(x)) for x in xs])
    ksplits = []
    for allow_split in (False, True):
        with NativeSpy() as spy, torch.no_grad():
            blk = torch.empty((2, B, Cout // 8, Ho, Wo, 8), dtype=torch.float16, device=DEV) if "b" in outs else None
            r = ops.conv2d_tc(planes, ptc, residual=res, residual_mode=res_mode, aux=aux, want_f32="f" in outs, want_planes="p" in outs,
                              terms=terms, block_n=block_n, allow_split=allow_split, blk_out=blk)
            torch.cuda.synchronize()
        (launch,) = spy.tc
        ksplits.append(launch["ksplit"])
        ref = R.conv_reference(torch.cat(xh, 1), torch.cat(xl, 1), pc.weight, terms, stride, pc.bias, None if res is None else _nchw(res),
                               res_mode, act, aux, k_padded=ptc.ktot, ksplit=launch["ksplit"])
        worst, acc = _check_outputs("%s terms=%d split=%d" % (name, terms, launch["ksplit"]), ref, f32=r[0], planes=r[1], blk=blk,
                                    aux=r[2] if aux is not None else None, hi_only=terms == 1)
        _report("conv_tc %-36s terms=%d tile=%s ksplit=%d  err/bound %.3f  err/(u n S) %.3f" % (name, terms, launch["tile"], launch["ksplit"],
                                                                                           worst, acc))
    assert ksplits[0] == 1
    if k > 1:      # the split is over filter taps: every k>1 case is small enough to split on an H100
        assert ksplits[1] > 1, "%s: the split-K launch did not split (%d)" % (name, ksplits[1])


def test_conv2d_tc_cases_reach_both_tiles_and_every_option():
    tiles = {"8x16" if (((W + 2 * ((k - 1) // 2) - k) // s + 1) <= 8 and ((H + 2 * ((k - 1) // 2) - k) // s + 1) > 8) else "16x8"
             for _, B, H, W, _, _, k, s, *_ in TC_CASES}
    assert tiles == {"8x16", "16x8"}
    assert {c[6] for c in TC_CASES} == {1, 3, 5} and {c[13] for c in TC_CASES} == {32, 64, 128}
    assert {c[9] for c in TC_CASES} == {R.RES_NONE, R.RES_SAME, R.RES_NEAREST_UP}
    assert {c[10] for c in TC_CASES} == {R.ACT_NONE, R.ACT_RELU, R.ACT_SIGMOID}
    assert any(c[5] % 8 for c in TC_CASES) and any(len(c[4]) == 3 for c in TC_CASES)


@pytest.mark.parametrize("terms", [1, 3])
def test_conv2d_tc_deferred_finish_parts(ops, terms):
    """defer_finish: the launch leaves its split-K partial sums in the workspace; their sum in split order matches the reference"""
    ops.set_conv_backend("tc", terms=terms)
    B, H, W, cin, cout = 1, 8, 8, 512, 256
    x = _randn((B, H, W, cin), 5)
    pc = ops.PackedConv(_randn((cout, cin, 3, 3), 6, (2.0 / (cin * 9)) ** 0.5), None, None)
    ptc = ops.PackedConvTC(pc, [cin], DEV)
    with NativeSpy() as spy, torch.no_grad():
        r = ops.conv2d_tc([ops.split_planes(x)], ptc, terms=terms, want_f32=False, want_planes=False, defer_finish=True)
        assert r is not None and r[0] == "parts"
        ws, offset, n_parts, stride = r[1]
        total = B * H * W * cout
        parts = ws[offset // 4:offset // 4 + n_parts * stride].view(n_parts, stride)[:, :total]
        acc = torch.zeros(total, device=DEV)
        for p in parts:
            acc = acc + p
        torch.cuda.synchronize()
    assert n_parts > 1 and spy.tc[0]["ksplit"] == n_parts
    xh, xl = R.fp16_split(_nchw(x))
    ref = R.conv_reference(xh, xl, pc.weight, terms, k_padded=ptc.ktot, ksplit=n_parts)
    worst, accw = _check_outputs("deferred parts terms=%d" % terms, ref, f32=acc.view(B, H, W, cout))
    _report("conv_tc deferred parts terms=%d ksplit=%d  err/bound %.3f  err/(u n S) %.3f" % (terms, n_parts, worst, accw))


# ------------------------------------------------------------------------------------------------ conv_halo_kernel, separate sources
HALO_CASES = [
    # name, B, H, W, [src channels], Cout, k, block_n, bias, residual, act
    ("k5_kc16_three_sources_rgb_depth", 1, 40, 36, [32, 1, 3], 32, 5, 32, True, True, R.ACT_RELU),
    ("k3_kc32_two_sources_n64_partial", 2, 24, 20, [32, 64], 72, 3, 64, True, False, R.ACT_NONE),
    ("k5_kc16_two_sources_n64_partial", 1, 33, 27, [24, 8], 40, 5, 64, False, True, R.ACT_RELU),
    ("k3_kc32_decoder_like_n32_partial", 1, 32, 48, [32, 32, 1], 40, 3, 32, True, True, R.ACT_RELU),
]


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("case", HALO_CASES, ids=[c[0] for c in HALO_CASES])
def test_conv2d_halo_separate_sources_vs_fp64_reference(ops, case, terms):
    name, B, H, W, chans, Cout, k, block_n, bias, use_res, act = case
    ops.set_conv_backend("tc", terms=terms)
    seed = sum(map(ord, name))
    xs = [_randn((B, H, W, c), seed + i) for i, c in enumerate(chans)]
    cin = sum(chans)
    w = _randn((Cout, cin, k, k), seed + 10, (2.0 / (cin * k * k)) ** 0.5)
    pc = ops.PackedConv(w, _randn((Cout,), seed + 11, 0.1) if bias else None, None, act=act)
    ph = ops.PackedConvHalo(pc, chans, DEV, block_n=block_n, concat_padded=False)
    assert ph.kc == (16 if k == 5 else 32) and len(ph.src_c8) == len(chans)
    res = _randn((B, H, W, Cout), seed + 12) if use_res else None
    blks = [ops.split_blocked([(x, False)]) for x in xs]
    xh, xl = zip(*[R.fp16_split(_nchw(x)) for x in xs])
    ref = R.conv_reference(torch.cat(xh, 1), torch.cat(xl, 1), pc.weight, terms, 1, pc.bias, None if res is None else _nchw(res),
                           R.RES_SAME if use_res else R.RES_NONE, act, k_padded=k * k * ph.n_groups * ph.kc)
    for flags in ((True, True, True), (False, True, False), (False, False, True)):      # blocked-only: the pixels-fastest stores
        with NativeSpy(), torch.no_grad():
            f32, oblk, onhwc = ops.conv2d_halo(blks, ph, residual=res, terms=terms, want_f32=flags[0], want_blk=flags[1], want_nhwc=flags[2])
            torch.cuda.synchronize()
        worst, acc = _check_outputs("%s terms=%d outputs=%s" % (name, terms, flags), ref, f32=f32, planes=onhwc, blk=oblk, hi_only=terms == 1)
        _report("conv_halo %-34s terms=%d outputs=%-18s err/bound %.3f  err/(u n S) %.3f" % (name, terms, flags, worst, acc))


# ------------------------------------------------------------------------------------------------ lstm_gates_kernel
def _lstm_instantiation(B, C, hw):
    """<PPW, CPB> dvmvs_lstm_gates_parts launches for (B, C, h*w)"""
    if B * (C // 32) < 74 and hw <= 512:
        ppw = -(-hw // 32)
        return (2 if ppw <= 2 else 4 if ppw <= 4 else 16), 8
    ppw = -(-hw // 8)
    return (2 if ppw <= 2 else 8 if ppw <= 8 else 16 if ppw <= 16 else 64), 32


LSTM_SHAPES = [  # B, C, h, w: every instantiation on both sides of each threshold, and both sides of the narrow / wide switch
    (1, 64, 1, 1), (1, 64, 8, 8), (1, 64, 5, 13), (1, 64, 8, 16), (1, 64, 3, 43), (1, 64, 16, 32),
    (5, 512, 1, 1), (5, 512, 4, 4), (5, 512, 1, 17), (5, 512, 8, 8), (5, 512, 5, 13), (5, 512, 8, 16), (5, 512, 3, 43), (5, 512, 16, 32),
    (4, 512, 8, 8), (2, 96, 4, 5),
]
ALL_LSTM_INSTANTIATIONS = {(2, 8), (4, 8), (16, 8), (2, 32), (8, 32), (16, 32), (64, 32)}


def _check_lstm(what, g32, c, h_out, c_out):
    hn, cn, bh, bc = R.lstm_reference(g32, c)
    rows = []
    R.check(what + " h", h_out, hn, bh, report=rows)
    R.check(what + " c", c_out, cn, bc, report=rows)
    return max(r[1] for r in rows)


def test_lstm_gates_every_instantiation(ops):
    reached = set()
    for B, C, h, w in LSTM_SHAPES:
        seed = B * 1000 + C + h * 37 + w
        g = _randn((B, h, w, 4 * C), seed, 2.0)
        c = _randn((B, h, w, C), seed + 1)
        with torch.no_grad():
            h_out, c_out = ops.lstm_gates(g, c)
        inst = _lstm_instantiation(B, C, h * w)
        reached.add(inst)
        worst = _check_lstm("lstm_gates B=%d C=%d %dx%d <%d,%d>" % ((B, C, h, w) + inst), g, c, h_out, c_out)
        _report("lstm_gates <%2d,%2d> B=%d C=%3d %2dx%-2d  err/bound %.3f" % (inst + (B, C, h, w, worst)))
    assert reached == ALL_LSTM_INSTANTIATIONS
    assert _lstm_instantiation(4, 512, 64) == (2, 8) and _lstm_instantiation(5, 512, 64) == (8, 32)


@pytest.mark.parametrize("with_addend", [False, True])
@pytest.mark.parametrize("n_parts", [1, 3, 9])
def test_lstm_gates_parts_form(ops, n_parts, with_addend):
    """the finishing pass of a deferred gate GEMM: the parts summed in split order (+ the addend), then the epilogue"""
    B, C, h, w = 1, 512, 8, 8
    total = B * h * w * 4 * C
    stride = total + 96
    seed = n_parts * 10 + with_addend
    ws = _randn((n_parts * stride + 64,), seed, 0.7)
    addend = _randn((B, h, w, 4 * C), seed + 1) if with_addend else None
    c = _randn((B, h, w, C), seed + 2)
    with torch.no_grad():
        h_out, c_out = ops.lstm_gates(None, c, parts=(ws, 64 * 4, n_parts, stride), addend=addend)
    g = torch.zeros(total, device=DEV)
    for sp in range(n_parts):
        g = g + ws[64 + sp * stride:64 + sp * stride + total]
    g = g.view(B, h, w, 4 * C)
    if addend is not None:
        g = g + addend
    worst = _check_lstm("lstm_gates parts=%d addend=%s" % (n_parts, with_addend), g, c, h_out, c_out)
    _report("lstm_gates parts n=%d addend=%-5s err/bound %.3f" % (n_parts, with_addend, worst))


@pytest.mark.parametrize("terms", [1, 3])
def test_lstm_deferred_gate_gemm_and_epilogue(ops, terms):
    """what the recurrent stage runs: conv_h.run_deferred (split-K gate GEMM without its finishing pass), then lstm_gates(parts=...)"""
    from dvmvs import _native as N
    ops.set_conv_backend("tc", terms=terms)
    B, C, h, w = 1, 512, 8, 8
    hid = _randn((B, h, w, C), 21)
    c = _randn((B, h, w, C), 22)
    gx = _randn((B, h, w, 4 * C), 23)
    conv_h = ops.ConvLayer(ops.PackedConv(_randn((4 * C, C, 3, 3), 24, (1.0 / (C * 9)) ** 0.5), None, None))
    with torch.no_grad():
        r = conv_h.run_deferred([(ops.Act(hid), N.SRC_DIRECT)])
        assert r is not None, "the gate GEMM at the benchmark's bottleneck no longer splits"
        ws, offset, n_parts, stride = r[1]
        total = B * h * w * 4 * C
        parts = torch.zeros(total, device=DEV)
        for sp in range(n_parts):
            parts = parts + ws[offset // 4 + sp * stride:offset // 4 + sp * stride + total]
        h_out, c_out = ops.lstm_gates(None, c, parts=r[1], addend=gx)
        torch.cuda.synchronize()
    assert n_parts > 1
    xh, xl = R.fp16_split(_nchw(hid))
    ref = R.conv_reference(xh, xl, conv_h.pc.weight, terms, k_padded=conv_h._ptc.ktot, ksplit=n_parts)
    wg, acc = _check_outputs("gate GEMM parts terms=%d" % terms, ref, f32=parts.view(B, h, w, 4 * C))
    we = _check_lstm("deferred gate epilogue terms=%d" % terms, parts.view(B, h, w, 4 * C) + gx, c, h_out, c_out)
    _report("lstm deferred terms=%d ksplit=%d  GEMM err/bound %.3f err/(u n S) %.3f  epilogue err/bound %.3f" % (terms, n_parts, wg, acc, we))


# ------------------------------------------------------------------------------------------------ every layer the benchmark runs
def _real_channels(planes_list, src_channels, blocked, packed, plane=0):
    """hi (plane 0) or lo (plane 1) planes of the operands -> (B, Cin, H, W) of the real channels in the weights' order"""
    hi = [_blk_to_nchw(t[plane]) if blocked else _nchw(t[plane]) for t in planes_list]
    if packed:        # one operand tensor holding every source (at 8-channel boundaries on the blocked path, back to back otherwise)
        out, off = [], 0
        for cr in src_channels:
            out.append(hi[0][:, off:off + cr])
            off += (cr + 7) // 8 * 8 if blocked else cr
        return torch.cat(out, 1).double()
    return torch.cat([t[:, :cr] for t, cr in zip(hi, src_channels)], 1).double()


def _at(t, rows, dim=0):
    return None if t is None else t.index_select(dim, rows)


def _operands(planes_list, src_channels, blocked, packed, terms, rows):
    """(hi, lo) operands of the batch rows `rows` in fp64; lo is None for 1-term products (its plane is not written then)"""
    hi = _at(_real_channels(planes_list, src_channels, blocked, packed), rows)
    lo = _at(_real_channels(planes_list, src_channels, blocked, packed, 1), rows) if terms == 3 else None
    R.check_live("operands", hi)
    return hi, lo


def _replay_tc(args, kw, lay, spy, rows):
    from dvmvs import _ops as ops
    planes, ptc = args[0], args[1]
    terms = kw.get("terms", 3)
    x, xl = _operands(planes, [ptc.cin] if lay.pack_sources else lay.src_channels, False, lay.pack_sources, terms, rows)
    with torch.no_grad():
        r = ops.conv2d_tc(*args, **kw)
        torch.cuda.synchronize()
    ks = spy.tc[-1]["ksplit"]
    res = kw.get("residual")
    ref = R.conv_reference(x, xl, lay.pc.weight, terms, ptc.stride, ptc.bias, None if res is None else _nchw(_at(res, rows)),
                           kw.get("residual_mode", R.RES_NONE), ptc.act, kw.get("aux"), k_padded=ptc.ktot, ksplit=ks)
    w, a = _check_outputs("", ref, f32=_at(r[0], rows), planes=_at(r[1], rows, 1), blk=_at(kw.get("blk_out"), rows, 1),
                          aux=_at(r[2], rows) if kw.get("aux") else None, hi_only=terms == 1)
    return spy.tc[-1], w, a


def _replay_deferred(args, kw, lay, gates_call, spy, rows):
    from dvmvs import _ops as ops
    planes, ptc = args[0], args[1]
    terms = kw.get("terms", 3)
    x, xl = _operands(planes, lay.src_channels, False, False, terms, rows)
    (_, c), gkw = gates_call[0], gates_call[1]
    R.check_live("deferred gate epilogue", _at(c, rows), _at(gkw.get("addend"), rows))
    with torch.no_grad():
        r = ops.conv2d_tc(*args, **kw)
        ws, offset, n_parts, stride = r[1]
        B, h, w, C = c.shape
        total = B * h * w * 4 * C
        g = torch.zeros(total, device=DEV)
        for sp in range(n_parts):
            g = g + ws[offset // 4 + sp * stride:offset // 4 + sp * stride + total]
        h_out, c_out = ops.lstm_gates(None, c, parts=r[1], addend=gkw.get("addend"))
        torch.cuda.synchronize()
    ref = R.conv_reference(x, xl, lay.pc.weight, terms, k_padded=ptc.ktot, ksplit=n_parts)
    g = g.view(B, h, w, 4 * C)
    wg, acc = _check_outputs("", ref, f32=_at(g, rows))
    if gkw.get("addend") is not None:
        g = g + gkw["addend"]
    we = _check_lstm("gate epilogue", _at(g, rows), _at(c, rows), _at(h_out, rows), _at(c_out, rows))
    return dict(spy.tc[-1], gates=_lstm_instantiation(B, C, h * w)), max(wg, we), acc


def _replay_gates(args, rows):
    """the plain gate epilogue (the gate convolution did not split, so it ran with its own finishing pass and the state-
    independent half as its residual): lstm_gates on the pre-activations the engine handed it"""
    from dvmvs import _ops as ops
    g, c = args
    R.check_live("lstm_gates", _at(g, rows), _at(c, rows))
    with torch.no_grad():
        h_out, c_out = ops.lstm_gates(g, c)
        torch.cuda.synchronize()
    B, h, w, C = c.shape
    return _lstm_instantiation(B, C, h * w), _check_lstm("gate epilogue", _at(g, rows), _at(c, rows), _at(h_out, rows), _at(c_out, rows))


def _replay_halo(args, kw, lay, rows):
    from dvmvs import _ops as ops
    blks, ph = args[0], args[1]
    terms = kw.get("terms", 3)
    x, xl = _operands(blks, lay.src_channels, True, lay.pack_sources, terms, rows)
    with torch.no_grad():
        f32, oblk, onhwc = ops.conv2d_halo(*args, **kw)
        torch.cuda.synchronize()
    res = kw.get("residual")
    ref = R.conv_reference(x, xl, lay.pc.weight, terms, 1, ph.bias, None if res is None else _nchw(_at(res, rows)),
                           R.RES_NONE if res is None else R.RES_SAME, ph.act, k_padded=ph.ksize ** 2 * ph.n_groups * ph.kc)
    return _check_outputs("", ref, f32=_at(f32, rows), planes=_at(onhwc, rows, 1), blk=_at(oblk, rows, 1), hi_only=terms == 1)


def _replay_expand(args, kw, rows):
    from dvmvs import _ops as ops
    act, expand, dw = args[0], args[1], args[2]
    terms = kw.get("terms", args[3] if len(args) > 3 else None)
    terms = ops._TC_TERMS if terms is None else terms               # None: the terms of the call's family, as the engine ran it
    pc = expand.pc
    x, xl = (_at(_nchw(p)[:, :pc.cin].double(), rows) for p in act.get_planes())
    R.check_live("expand_dwconv", x)
    with torch.no_grad():
        out = ops.expand_dwconv(*args, **kw)
        torch.cuda.synchronize()
    e = R.conv_reference(x, xl, pc.weight, terms, 1, pc.bias, act=pc.act, k_padded=expand._ptc.ktot)
    k = dw.ksize
    wd = dw.weight.permute(2, 0, 1).unsqueeze(1).double()             # [k][k][C] -> (C,1,k,k)
    y = F.conv2d(e.y, wd, dw.bias.double(), dw.stride, k // 2, groups=dw.channels)
    b = F.conv2d(e.bound, wd.abs(), None, dw.stride, k // 2, groups=dw.channels)
    b = b + (k * k + 2) * R.U * (F.conv2d(e.y.abs(), wd.abs(), None, dw.stride, k // 2, groups=dw.channels) + dw.bias.double().abs().view(1, -1, 1, 1))
    y, b = R.activation(y, b, dw.act)
    rows_ = []
    R.check("expand_dwconv", _nchw(_at(out[0], rows)).float(), y, R.fp16_bound(y, b), report=rows_)
    return rows_[0][1], e.eps_acc, terms


def _point_params():
    """bench.py's operating points (tools/engine_record.py POINTS) at their own input sizes, and the headline engine at 256x320
    and 320x256: the portrait size is the only one whose 10x8 bottleneck runs the 8-wide tile"""
    from tools.engine_record import POINTS
    return ([pytest.param("value", 256, 320, id="256-320"), pytest.param("value", 320, 256, id="320-256")] +
            [pytest.param(p, None, None, id=p) for p in POINTS])


@pytest.mark.parametrize("point,height,width", _point_params())
def test_every_benchmark_layer_vs_fp64_reference(ops, point, height, width):
    """Records every conv2d_tc, conv2d_halo, expand_dwconv and ConvLSTM gate call (deferred pair or plain epilogue) of the engine
    bench.py runs at this operating point (seed-7 weights, the point's operand terms and batch, clip b in batch row b), and replays
    each on its recorded operands against the fp64 reference, on the batch rows tools.engine_record.batch_rows picks.  One line
    per layer; a failure names the layer.  Then checks the facts that make the point differ from the headline (batch, split
    counts, block_n, gate path and instantiation, terms, aggregator0's cost-volume channels)."""
    import time
    from tools.engine_record import batch_rows, engine_calls, layer_names, point_config, trunk_batch
    t0 = time.perf_counter()
    cfg = point_config(point, height, width)
    mods, calls = engine_calls(("conv2d_tc", "conv2d_halo", "expand_dwconv", "lstm_gates"), point=point, height=height, width=width)
    names = layer_names(mods)
    gate_layer = mods["lstm"].lstm_cell.packed()[1]             # conv(W[:, Cin:], h): the gate convolution on the recurrent state
    agg0 = mods["cve"].packed()[0]
    gates_calls = [v for k, v in calls.items() if k[0] == "lstm_gates" and k[2]]
    seen = {"conv2d_tc": 0, "conv2d_halo": 0, "expand_dwconv": 0, "deferred": 0, "lstm_gates": 0}
    tiles, worst_all, acc_all = set(), 0.0, 0.0
    trunk, terms_seen, tc_launches, gate, agg0_seen = set(), set(), [], {}, False
    print()
    for key, (args, kw, lay, on_rec) in calls.items():
        kind = key[0]
        if kind == "lstm_gates" and key[2]:
            continue                    # replayed with its gate GEMM
        layer = names.get(id(lay if lay is not None else args[1]), "?") if kind != "lstm_gates" else "lstm gates"
        if kind == "conv2d_halo":
            path, shape = "halo", (args[0][0].shape[1],) + tuple(args[0][0].shape[3:5])
        elif kind == "conv2d_tc":
            path, shape = "tc deferred+gates" if kw.get("defer_finish") else "tc", tuple(args[0][0].shape[1:4])
        elif kind == "lstm_gates":
            path, shape = "gates", tuple(args[1].shape[:3])
        else:
            path, shape = "expand_dw", tuple(args[0].get_planes().shape[1:4])
        rows = torch.tensor(batch_rows(shape[0]), device=DEV)
        launch, acc, extra = {}, 0.0, ""
        try:
            with NativeSpy() as spy:
                if path == "tc deferred+gates":
                    assert len(gates_calls) == 1, "expected one deferred gate epilogue, recorded %d" % len(gates_calls)
                    launch, worst, acc = _replay_deferred(args, kw, lay, gates_calls[0], spy, rows)
                    assert launch["ksplit"] > 1
                    seen["deferred"] += 1
                    extra = " gates=<%d,%d>" % launch["gates"]
                elif path == "tc":
                    launch, worst, acc = _replay_tc(args, kw, lay, spy, rows)
                elif path == "gates":
                    inst, worst = _replay_gates(args, rows)
                    gate["plain"] = inst
                    extra = " gates=<%d,%d>" % inst
                elif path == "halo":
                    worst, acc = _replay_halo(args, kw, lay, rows)
                else:
                    worst, _, expand_terms = _replay_expand(args, kw, rows)
        except AssertionError as e:
            raise AssertionError("%s: layer %s (%s%s, input B,H,W=%s): %s" % (point, layer, path, ", recurrent stage" if on_rec else "", shape, e)) from None
        seen[kind] += 1
        if path.startswith("tc"):
            tiles.add(launch["tile"])
            tc_launches.append((layer, launch))
            terms_seen.add(launch["terms"])
            if lay is gate_layer:
                gate["conv"] = launch
        elif path == "halo":
            terms_seen.add(kw["terms"])
        elif path == "expand_dw":
            terms_seen.add(expand_terms)
        if layer.startswith("fe"):
            trunk.add(shape[0])
        if lay is agg0:
            agg0_seen = True
            assert lay.src_channels == [32, cfg["n_depth_levels"]], "%s: aggregator0 reads %s" % (point, lay.src_channels)
        worst_all, acc_all = max(worst_all, worst), max(acc_all, acc)
        facts = ("ksplit=%d block_n=%-3d terms=%d tile=%-4s" % (launch["ksplit"], launch["block_n"], launch["terms"], launch["tile"])
                 if launch else "%-34s" % "")
        _report("%-34s %-18s B,H,W=%-15s %s rows=%d err/bound %.3f  err/(u n S) %.3f%s" % (layer, path, shape, facts, len(rows), worst, acc, extra))
    deferred = seen["deferred"] > 0
    _report("%s %dx%d B=%d terms=%d: %s; trunk batch %s; gate %s; worst err/bound %.3f, worst err/(u n S) %.3f (C_ACC = %g); %.1f s" % (
        point, cfg["height"], cfg["width"], cfg["batch"], cfg["terms"], seen, sorted(trunk),
        "deferred+gates ksplit=%d" % gate["conv"]["ksplit"] if deferred else "plain block_n=%d ksplit=%d <%d,%d>" % (
            (gate["conv"]["block_n"], gate["conv"]["ksplit"]) + gate["plain"]), worst_all, acc_all, R.C_ACC, time.perf_counter() - t0))
    # what makes this point this point
    assert all(seen[k] > 0 for k in ("conv2d_tc", "conv2d_halo", "expand_dwconv")), seen
    assert "conv" in gate and agg0_seen, "%s: the gate convolution or aggregator0 was not replayed" % point
    assert trunk == {trunk_batch(cfg)}, "%s: trunk batch %s, expected %d" % (point, sorted(trunk), trunk_batch(cfg))
    assert terms_seen == {cfg["terms"]}, "%s: tensor-core calls at terms %s, expected %d" % (point, terms_seen, cfg["terms"])
    assert gate["conv"]["B"] == cfg["batch"]
    if cfg["batch"] == 1:         # the gate GEMM (Cout 2048 on the 8x8 map) has 16 CTAs: it splits and the epilogue is its finishing pass
        assert deferred and seen["lstm_gates"] == 0, "%s: no deferred gate GEMM + epilogue pair (%s)" % (point, seen)
        assert gate["conv"]["block_n"] == 128
    else:                         # >= 66 CTAs: no split, so no deferred pair; the plain epilogue, wide instantiation
        assert not deferred and seen["lstm_gates"] == 1, "%s: expected the plain gate epilogue (%s)" % (point, seen)
        assert gate["conv"]["ksplit"] == 1 and gate["plain"] == (8, 32), (gate["conv"], gate["plain"])
        assert gate["conv"]["block_n"] == (64 if cfg["batch"] >= 16 else 128), gate["conv"]
    if cfg["batch"] == 32:
        split = [(n, l["ksplit"]) for n, l in tc_launches if l["ksplit"] != 1]
        assert not split, "%s: conv2d_tc calls that split: %s" % (point, split)
    if (cfg["height"], cfg["width"]) == (320, 256):
        assert "8x16" in tiles, "the 10x8 bottleneck of a portrait input no longer runs the 8-wide tile"
