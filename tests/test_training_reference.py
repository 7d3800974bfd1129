"""The training-step kernels against the fp64 references of tests/training_reference.py, element by element: the plane-sweep backward,
the ConvLSTM gate backward and the multi-scale depth loss (sums and gradient), called through dvmvs.training -- and through the C ABI
where only it reaches a path (one measurement buffer passed twice, grad_c = nullptr).  Every case first asserts the edges it claims
to reach, from the fp64 geometry or its inputs, and prints one line: worst err / bound, the ill-conditioned / ambiguous counts and
the kernel instantiation."""
import ctypes

import numpy as np
import pytest
import torch

from tests import training_reference as R
from tests.sweep_reference import positions

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------ plane-sweep backward
SWEEP_REACH = {                         # what each case must reach (counts from the fp64 geometry, > 0)
    "batch2_w33_D13_M3": ("left", "right", "top", "bottom", "n_outside"),
    "w40_D2_M1": ("n_outside",),
    "w64_D64_M3": ("n_outside",),
    "smem_max_D256_M8": ("n_outside",),
    "crossing_borders": ("n_behind", "n_outside", "left", "top", "bottom"),
    "forward_motion": ("n_live",),
    "zero_baseline": ("n_live",),
    "far_out_of_view": ("n_outside",),
    "grad_zeros_B2": ("n_gzero",),
    "train_128x128_D64_M2": ("n_outside",),
    "train_128x160_D96_M4": ("n_outside",),
}


def _assert_sweep_reach(name, c, ref):
    B, h, w, D, M = c["B"], c["h"], c["w"], c["D"], c["M"]
    for k in SWEEP_REACH[name]:
        assert getattr(ref, k) > 0, "%s reaches no %s sample" % (name, k)
    if name == "batch2_w33_D13_M3":
        assert B > 1 and w % 32 and D % R.K_GROUP and not torch.equal(c["pose1"][0], c["pose1"][1])
    if name == "smem_max_D256_M8":
        smem = (32 * 32 + M * D * 4 + 8 * 12 + 32 * D) * 4 + R.K_GROUP * 32 * 32
        assert D == 256 and M == 8 and smem > 64 * 1024
    if name == "crossing_borders":                # the denominator changes sign on the plane range
        den = positions(c["pose1"], c["pose2s"][0], c["K"], ref.depths, h, w)["den"]
        assert bool((den < 0).any()) and bool((den > 0).any())
    if name == "zero_baseline":
        assert torch.equal(c["pose1"], c["pose2s"][0])
    if name == "grad_zeros_B2":
        assert bool((c["g"] == 0).all(-1).any()) and bool((c["g"] == 0).any())


def _sweep_through_training(c, layout):
    from dvmvs.training import plane_sweep_cost_volume
    conv = (lambda t: t.contiguous(memory_format=torch.channels_last)) if layout == "channels_last" else (lambda t: t.contiguous())
    f1 = conv(_nchw(c["f1"].to(DEV))).requires_grad_(True)
    f2s = [conv(_nchw(f.to(DEV))).requires_grad_(True) for f in c["f2s"]]
    cost = plane_sweep_cost_volume(f1, f2s, c["pose1"].to(DEV), [p.to(DEV) for p in c["pose2s"]], c["K"].to(DEV), R.SWEEP_MIN_DEPTH,
                                   R.SWEEP_MAX_DEPTH, c["D"])
    cost.backward(conv(_nchw(c["g"].to(DEV))))
    torch.cuda.synchronize()
    return _nhwc(f1.grad), [_nhwc(f.grad) for f in f2s]


@pytest.mark.parametrize("name", list(R.SWEEP_CASES))
def test_plane_sweep_backward_vs_fp64_reference(name):
    c = R.sweep_case(name)
    ref = R.sweep_case_reference(c, DEV)
    _assert_sweep_reach(name, c, ref)
    layouts = ("nchw", "channels_last") if name == "grad_zeros_B2" else ("nchw",)
    for layout in layouts:
        gref, gmeas = _sweep_through_training(c, layout)
        worst, nz = R.check_sweep_backward("%s %s" % (name, layout), ref, gref, gmeas)
        print("\nsweep backward %-22s %-13s err/bound %.4f  ill-conditioned %d  exact +0 %d  live %d  outside %d  behind %d  "
              "straddling L/R/T/B %d/%d/%d/%d  plane_sweep_backward_c32_kernel D=%d (%d groups) M=%d w=%d"
              % (name, layout, worst, ref.n_ill, nz, ref.n_live, ref.n_outside, ref.n_behind, ref.left, ref.right, ref.top, ref.bottom,
                 c["D"], (c["D"] + 7) // 8, c["M"], c["w"]))


def test_plane_sweep_backward_same_buffer_twice_through_the_abi():
    """grad_meas_host with one buffer for frames 0 and 1 (the same measurement tensor): zeroed once, both contributions accumulate"""
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    c = R.sweep_case("batch2_w33_D13_M3")
    c["f2s"][1] = c["f2s"][0]
    ref = R.sweep_case_reference(c, DEV)
    B, h, w, D, M = c["B"], c["h"], c["w"], c["D"], c["M"]
    f1 = c["f1"].to(DEV).contiguous()
    meas = [c["f2s"][0].to(DEV).contiguous(), None, c["f2s"][2].to(DEV).contiguous()]
    meas[1] = meas[0]
    pose1, K = c["pose1"].to(DEV).contiguous(), c["K"].to(DEV).contiguous()
    pose2s = [p.to(DEV).contiguous() for p in c["pose2s"]]
    g = c["g"].to(DEV).contiguous()
    g_ref = torch.full_like(f1, float("nan"))
    shared, other = torch.full_like(f1, float("nan")), torch.full_like(f1, float("nan"))      # the entry point must zero them
    arr = lambda ts: (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
    N.check(N.lib().dvmvs_plane_sweep_backward(f1.data_ptr(), arr(meas), pose1.data_ptr(), arr(pose2s), K.data_ptr(), g.data_ptr(),
                                               g_ref.data_ptr(), arr([shared, shared, other]), B, 32, h, w, D, M, R.SWEEP_MIN_DEPTH,
                                               R.SWEEP_MAX_DEPTH, N.SWEEP_DOT, ops._stream()), "plane_sweep_backward")
    torch.cuda.synchronize()
    worst, nz = R.check_sweep_backward("aliased", ref, g_ref, [shared, other], buffers=[[0, 1], [2]])
    print("\nsweep backward aliased buffer (frames 0, 1)  err/bound %.4f  exact +0 %d" % (worst, nz))


# ------------------------------------------------------------------------------------------------ ConvLSTM gate backward
@pytest.mark.parametrize("name", list(R.LSTM_CASES))
def test_lstm_gates_backward_vs_fp64_reference(name):
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    from dvmvs.training import lstm_gate_epilogue
    gates, c_in, gh, gc = R.lstm_case(name)
    B, h, w, C = c_in.shape
    reach = R.lstm_reach(gates, C)
    assert reach["const_g"] >= B and reach["const_cp"] >= B and reach["saturated"] > 0, reach
    # grad_c present: through dvmvs.training under autograd
    a = _nchw(gates.to(DEV)).contiguous().requires_grad_(True)
    cc = _nchw(c_in.to(DEV)).contiguous().requires_grad_(True)
    hn, cn = lstm_gate_epilogue(a, cc)
    torch.autograd.backward([hn, cn], [_nchw(gh.to(DEV)).contiguous(), _nchw(gc.to(DEV)).contiguous()])
    torch.cuda.synchronize()
    gv, gb, cv, cb = (t.to(DEV) for t in R.lstm_backward_reference(gates, c_in, gh, gc))
    w1 = R.check_bound(name + " grad_gates", _nhwc(a.grad), gv, gb)
    w2 = R.check_bound(name + " grad_c_in", _nhwc(cc.grad), cv, cb)
    # grad_c absent: grad_c = nullptr through the C ABI (autograd materialises a zero gradient instead)
    g_d, c_d, gh_d = gates.to(DEV).contiguous(), c_in.to(DEV).contiguous(), gh.to(DEV).contiguous()
    out_g, out_c = torch.full_like(g_d, float("nan")), torch.full_like(c_d, float("nan"))
    N.check(N.lib().dvmvs_lstm_gates_backward(g_d.data_ptr(), c_d.data_ptr(), gh_d.data_ptr(), None, out_g.data_ptr(), out_c.data_ptr(),
                                              B, h, w, C, ops._stream()), "lstm_gates_backward")
    torch.cuda.synchronize()
    gv, gb, cv, cb = (t.to(DEV) for t in R.lstm_backward_reference(gates, c_in, gh, None))
    w3 = R.check_bound(name + " grad_gates (no grad_c)", out_g, gv, gb)
    w4 = R.check_bound(name + " grad_c_in (no grad_c)", out_c, cv, cb)
    print("\nlstm backward %-14s err/bound grad_c %.4f / %.4f  no grad_c %.4f / %.4f  constant-g channels %d  constant-cp channels %d  "
          "saturated %d  lstm_gates_backward_kernel<%d>" % (name, w1, w2, w3, w4, reach["const_g"], reach["const_cp"], reach["saturated"],
                                                          R.lstm_instantiation(h * w)))


def test_lstm_cases_cross_every_instantiation_boundary():
    hws = sorted({h * w for (_, h, w, _) in R.LSTM_CASES.values()})
    assert hws == [1, 16, 17, 64, 65, 80, 128]
    assert {R.lstm_instantiation(x) for x in hws} == {2, 8, 16}
    for lo, hi in ((16, 17), (64, 65)):
        assert R.lstm_instantiation(lo) != R.lstm_instantiation(hi)
    assert {c for (_, _, _, c) in R.LSTM_CASES.values()} == {32, 512} and {b for (b, _, _, _) in R.LSTM_CASES.values()} == {1, 4}


# ------------------------------------------------------------------------------------------------ depth loss
@pytest.mark.parametrize("loss_type", list(R.LOSS_COLUMN))
@pytest.mark.parametrize("case", list(R.LOSS_CASES))
def test_depth_loss_vs_fp64_reference(case, loss_type):
    from dvmvs.training import multi_scale_depth_loss
    preds, gt, weights, up = R.loss_case(case)
    reach = R.loss_reach(preds, gt)
    need = {"one_scale_B2_20x20": ("straddle", "neg", "zeros", "equal", "one_apart"),
            "five_scales_odd_ratios": ("straddle", "non_integer", "upsampled", "neg", "equal", "one_apart"),
            "eight_scales_one_empty": ("straddle", "non_integer", "empty", "neg"),
            "nan_groundtruth": ("nan",),
            "train_bench_B4_256": ()}[case]
    for k in need:
        assert reach[k] > 0, "%s reaches no %s" % (case, k)
    if case == "eight_scales_one_empty":
        assert len(preds) == R.MAX_SCALES
    if case == "train_bench_B4_256":
        assert len(preds) == 5 and gt.shape == (4, 256, 256)
    pt = [torch.from_numpy(p).to(DEV).requires_grad_(True) for p in preds]
    loss, sums = multi_scale_depth_loss(pt, weights, torch.from_numpy(gt).to(DEV), loss_type)
    (loss * up).backward()
    torch.cuda.synchronize()
    ref_sums, bound = R.loss_forward_reference(preds, gt)
    wf = R.check_loss_sums("%s %s sums" % (case, loss_type), sums.cpu().numpy(), ref_sums, bound)
    got_counts = sums[:, 4].cpu().numpy().astype(np.float64)
    ref = R.loss_backward_reference(preds, gt, weights, up, loss_type, got_counts)
    wb, amb = R.check_loss_grad("%s %s grad" % (case, loss_type), [p.grad.cpu().numpy() for p in pt], ref)
    print("\nloss %-24s %-7s sums err/bound %.4f  grad err/bound %.4f  ambiguous %d  scales %d  blocks %s  %s"
          % (case, loss_type, wf, wb, amb, len(preds), R.loss_blocks(gt.shape[0], [p.shape[1:] for p in preds]),
             {k: v for k, v in reach.items() if k != "scales"}))
