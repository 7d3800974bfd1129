"""conv_ws_kernel -- the weight-streaming split-K kernel dvmvs_conv2d_tc picks for small-map k x k layers -- against the float64
reference on its own fp16 operands (tests/tc_reference.py); every call's plan (NativeSpy: dvmvs_conv2d_tc_ksplit on the launched
descriptor) is checked against the selection rule below, so each case asserts that conv_ws_kernel ran; its workspace rows and
outputs under guarded allocations; its determinism; and (without a GPU) the selection rule against dvmvs_conv2d_tc_ksplit."""
import pytest
import torch

from tests import tc_reference as R
from tests.test_tc_reference import NativeSpy, _check_outputs, _nchw, _randn, _report

DEV = "cuda"
gpu = pytest.mark.gpu


@pytest.fixture
def ops():
    from dvmvs import _ops
    old = (_ops._BACKEND, _ops._TC_TERMS_BASE, _ops._TC_STRIDE2)
    try:
        yield _ops
    finally:
        _ops.set_conv_backend(old[0], terms=old[1], stride2=old[2])


# name, B, H, W, [(src channels, upsampled from H/2 x W/2)], Cout
WS_CASES = [
    ("gate_hidden_half_8x8", 1, 8, 8, [(512, False)], 2048),
    ("gate_both_halves_8x8_b4", 4, 8, 8, [(512, False), (512, False)], 2048),
    ("decoder1_up_16x16", 1, 16, 16, [(512, True)], 256),
    ("decoder1_conv1_16x16", 1, 16, 16, [(256, False), (256, False)], 256),
    ("decoder2_conv1_32x32_depth", 1, 32, 32, [(128, False), (128, False), (1, False)], 128),
    ("ragged_7x9_cout200_b4", 4, 7, 9, [(64, False)], 200),
    ("ragged_15x17_cout136_32chunks", 1, 15, 17, [(96, False), (32, False)], 136),
]


def _ws_operands(ops, case, k=3, stride=1):
    name, B, H, W, srcs, Cout = case
    seed = sum(map(ord, name))
    xs = [_randn((B, H // 2, W // 2, c) if up else (B, H, W, c), seed + i) for i, (c, up) in enumerate(srcs)]
    cin = sum(c for c, _ in srcs)
    pc = ops.PackedConv(_randn((Cout, cin, k, k), seed + 10, (2.0 / (cin * k * k)) ** 0.5), _randn((Cout,), seed + 11, 0.1), None,
                        stride=stride, act=R.ACT_RELU)
    ptc = ops.PackedConvTC(pc, [c for c, _ in srcs], DEV)
    planes = [ops.split_planes(x, upsample=up) for x, (_, up) in zip(xs, srcs)]
    return pc, ptc, planes


def _run_case(ops, case, terms, k=3, stride=1):
    """one split launch of the case: checks the fp32 and fp16 outputs against the fp64 reference and that conv_ws_kernel ran"""
    name, B, H, W, srcs, Cout = case
    ops.set_conv_backend("tc", terms=terms)
    pc, ptc, planes = _ws_operands(ops, case, k, stride)
    with NativeSpy() as spy, torch.no_grad():
        f32, pl = ops.conv2d_tc(planes, ptc, terms=terms, want_f32=True, want_planes=Cout % 8 == 0, allow_split=True)
        torch.cuda.synchronize()
    (launch,) = spy.tc
    assert expected_ksplit(B, *planes[0].shape[2:4], Cout, k, stride, launch["block_n"], ptc.rows) == (launch["ksplit"], "ws"), name
    # the reference reads the operands the kernel multiplies: the staged (upsampled, channel-padded) planes
    xh = torch.cat([_nchw(p[0])[:, :c].double() for p, (c, _) in zip(planes, srcs)], 1)
    xl = torch.cat([_nchw(p[1])[:, :c].double() for p, (c, _) in zip(planes, srcs)], 1) if terms == 3 else None
    ref = R.conv_reference(xh, xl, pc.weight, terms, stride, pc.bias, None, R.RES_NONE, R.ACT_RELU, None, k_padded=ptc.ktot,
                           ksplit=launch["ksplit"])
    worst, acc = _check_outputs("%s terms=%d" % (name, terms), ref, f32=f32, planes=pl, hi_only=terms == 1)
    _report("conv_ws %-32s terms=%d ksplit=%d  err/bound %.3f  err/(u n S) %.3f" % (name, terms, launch["ksplit"], worst, acc))
    return f32


@gpu
@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("case", WS_CASES, ids=[c[0] for c in WS_CASES])
def test_conv_ws_vs_fp64_reference(ops, case, terms):
    _run_case(ops, case, terms)


@gpu
@pytest.mark.parametrize("terms", [1, 3])
def test_conv_ws_5x5(ops, terms):
    _run_case(ops, ("k5_12x12", 2, 12, 12, [(64, False)], 128), terms, k=5)


@gpu
@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("case", [("encoder3_down_16_to_8_b4", 4, 16, 16, [(256, False)], 512),
                                  ("down_ragged_33x19_to_17x10", 1, 33, 19, [(64, False), (32, False)], 136)], ids=lambda c: c[0])
def test_conv_ws_stride2(ops, case, terms):
    """the encoder's stride-2 convolutions: strided activation boxes on the same kernel"""
    _run_case(ops, case, terms, stride=2)


@gpu
@pytest.mark.parametrize("terms", [1, 3])
def test_conv_ws_deferred_parts_and_lstm_gates(ops, terms):
    """the recurrent stage's gate path: run_deferred on conv_ws_kernel, parts summed in split order, dvmvs_lstm_gates_parts"""
    from tests import test_tc_reference as T
    with NativeSpy() as spy:
        T.test_lstm_deferred_gate_gemm_and_epilogue(ops, terms)
        T.test_conv2d_tc_deferred_finish_parts(ops, terms)
    gate, parts = spy.tc[-2:]
    assert expected_ksplit(1, 8, 8, 2048, 3, 1, gate["block_n"], 2048) == (gate["ksplit"], "ws")
    assert expected_ksplit(1, 8, 8, 256, 3, 1, parts["block_n"], 256) == (parts["ksplit"], "ws")


@gpu
def test_conv_ws_is_deterministic(ops):
    case = WS_CASES[1]
    a = _run_case(ops, case, 1)
    b = _run_case(ops, case, 1)
    assert torch.equal(a, b)


@gpu
@pytest.mark.parametrize("terms", [1, 3])
def test_conv_ws_guarded(ops, terms):
    """every case with its operands, outputs and the split-K workspace in guarded buffers: no read outside the operands (poisoned
    fringes would turn outputs into NaN), no store outside the outputs and the workspace rows of its split count"""
    from tests import guarded as G
    with G.guard_allocations():
        for case in WS_CASES:
            _run_case(ops, case, terms)
            G.verify()


# ------------------------------------------------------------------------------------------------ selection rule (no GPU)
N_SMS = 132
WORKSPACE = 32 << 20          # dvmvs._ops.WORKSPACE_BYTES: what conv2d_tc passes (the head of 16 KiB included)


def expected_ksplit(B, H, W, Cout, k, stride, block_n, w_rows, residual=False, aux=False, allow_split=True, ws_bytes=WORKSPACE):
    """dvmvs_conv2d_tc's split count and kernel (csrc/conv_tc.cu tc_plan): returns (ksplit, 'ws' or 'tc')"""
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    tw = 8 if (Wo <= 8 and Ho > 8) else 16
    th = 128 // tw
    ctas = -(-Wo // tw) * -(-Ho // th) * B * -(-Cout // block_n)
    taps = k * k
    if not (allow_split and ws_bytes > 16384 and ctas < N_SMS // 2 and taps > 1):
        return 1, "tc"
    fit = (ws_bytes - 16384) // (B * Ho * Wo * Cout * 4)
    if not residual and not aux and Cout % 8 == 0 and w_rows % 128 == 0 and Ho * Wo <= 1024:
        if Ho <= 8 and Wo <= 8:
            tw = th = 8
        base = -(-Wo // tw) * -(-Ho // th) * B * -(-Cout // 128)
        ks = min(min(taps, max(2, -(-64 // base))), fit)
        if ks >= 2:
            per = -(-taps // ks)
            return -(-taps // per), "ws"
    ks = max(1, min(min(taps, -(-N_SMS // ctas)), fit))
    per = -(-taps // ks)
    return -(-taps // per), "tc"


# B, H(in), W(in), Cout, k, stride, block_n, w_rows, residual, aux, allow_split, workspace bytes
RULE_CASES = [
    (1, 8, 8, 2048, 3, 1, 128, 2048, False, False, True, WORKSPACE),      # gate GEMM
    (4, 8, 8, 2048, 3, 1, 128, 2048, False, False, True, WORKSPACE),
    (1, 16, 16, 256, 3, 1, 32, 256, False, False, True, WORKSPACE),       # decoder block 1
    (1, 32, 32, 128, 3, 1, 64, 128, False, False, True, WORKSPACE),       # decoder block 2
    (1, 16, 24, 72, 5, 1, 64, 128, False, False, True, WORKSPACE),
    (1, 32, 32, 128, 3, 1, 64, 128, False, False, False, WORKSPACE),      # no split allowed: conv_tc_kernel, unsplit
    (1, 16, 16, 256, 3, 2, 32, 256, False, False, True, WORKSPACE),       # stride 2: conv_ws_kernel too
    (1, 16, 16, 256, 3, 1, 32, 256, True, False, True, WORKSPACE),        # residual: conv_tc_kernel
    (1, 16, 16, 12, 3, 1, 32, 128, False, True, True, WORKSPACE),         # aux, Cout % 8 != 0
    (1, 16, 16, 64, 3, 1, 32, 64, False, False, True, WORKSPACE),         # weight rows not a multiple of 128
    (1, 64, 64, 32, 3, 1, 32, 128, False, False, True, WORKSPACE),        # map above 32x32
    (2, 16, 16, 256, 1, 1, 64, 256, False, False, True, WORKSPACE),       # 1x1: never split
    (1, 8, 8, 2048, 3, 1, 128, 2048, False, False, True, 16384 + 2 * 64 * 2048 * 4),   # workspace holds 2 splits
    (1, 8, 8, 2048, 3, 1, 128, 2048, False, False, True, 16384 + 64 * 2048 * 4),       # workspace holds one split only
    (32, 8, 8, 512, 3, 1, 32, 512, False, False, True, WORKSPACE),       # enough CTAs unsplit
]


@pytest.mark.parametrize("case", RULE_CASES)
def test_selection_rule_matches_dvmvs_conv2d_tc_ksplit(case):
    from dvmvs import _native as N
    B, H, W, Cout, k, stride, block_n, w_rows, res, aux, allow, ws_bytes = case
    d = N.ConvTcDesc()
    d.B, d.Hin, d.Win, d.Cout, d.ksize, d.stride, d.block_n, d.w_rows = B, H, W, Cout, k, stride, block_n, w_rows
    d.residual_mode = R.RES_SAME if res else R.RES_NONE
    d.aux_out = 16 if aux else None
    d.allow_split = 1 if allow else 0
    d.workspace, d.workspace_bytes = 4096, ws_bytes
    import ctypes
    got = N.lib().dvmvs_conv2d_tc_ksplit(ctypes.byref(d))
    want, kernel = expected_ksplit(B, H, W, Cout, k, stride, block_n, w_rows, res, aux, allow, ws_bytes)
    assert got == want, (case, got, want, kernel)


def test_rule_cases_reach_both_kernels():
    kinds = {expected_ksplit(*c)[1] for c in RULE_CASES}
    assert kinds == {"ws", "tc"}
    assert expected_ksplit(*RULE_CASES[0])[1] == "ws" and expected_ksplit(*RULE_CASES[0])[0] >= 2
