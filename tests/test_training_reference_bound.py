"""The bounds of tests/training_reference.py are honest and not vacuous (no GPU needed): an fp32 emulation of each training-step kernel,
in its own operation order, passes the comparator; each planted defect fails it.  Prints the worst err / bound of every emulation
(each constant is >= 8x what it measures) and the factor by which each defect is rejected."""
import numpy as np
import pytest
import torch

from tests import training_reference as R
from tests.tc_reference import U


# ------------------------------------------------------------------------------------------------ plane-sweep backward
@pytest.mark.parametrize("name", R.CPU_SWEEP_CASES)
def test_sweep_backward_emulation_within_bound(name):
    c = R.sweep_case(name)
    ref = R.sweep_case_reference(c)
    gref, gmeas = R.sweep_case_emulation(c, seed=1)
    worst, nz = R.check_sweep_backward(name, ref, torch.from_numpy(gref), [torch.from_numpy(t) for t in gmeas])
    print("\nsweep backward %-20s emulation err/bound %.4f  exact +0 %d  ill-conditioned %d" % (name, worst, nz, ref.n_ill))
    assert worst * 8 <= 1.0


def test_sweep_backward_aliased_buffer_emulation_within_bound():
    """one measurement buffer passed for frames 0 and 1: both contributions accumulate into it"""
    c = R.sweep_case("batch2_w33_D13_M3")
    c["f2s"][1] = c["f2s"][0]
    ref = R.sweep_case_reference(c)
    gref, gmeas = R.sweep_case_emulation(c, buffers=[[0, 1], [2]], seed=2)
    worst, _ = R.check_sweep_backward("aliased", ref, torch.from_numpy(gref), [torch.from_numpy(t) for t in gmeas], buffers=[[0, 1], [2]])
    print("\nsweep backward aliased buffer  emulation err/bound %.4f" % worst)
    assert worst * 8 <= 1.0


SWEEP_DEFECT_CASES = {
    "clamp_border": "batch2_w33_D13_M3",       # taps straddling every border
    "swap_01_10": "batch2_w33_D13_M3",
    "scale_32": "batch2_w33_D13_M3",           # M = 3
    "drop_last_group": "batch2_w33_D13_M3",    # D = 13: a partial plane group
    "drop_frame_ref": "batch2_w33_D13_M3",
    "meas_next_frame": "batch2_w33_D13_M3",
}


def _rejection(fn):
    """the factor by which the comparator rejects: the worst err / bound it reports (inf for an exact-zero violation)"""
    try:
        fn()
    except AssertionError as e:
        msg = str(e)
        if "by x" in msg:
            return float(msg.split("by x")[1].split()[0])
        return float("inf")
    raise AssertionError("planted defect not rejected")


@pytest.mark.parametrize("defect", R.SWEEP_DEFECTS)
def test_sweep_backward_planted_defect_rejected(defect):
    c = R.sweep_case(SWEEP_DEFECT_CASES[defect])
    assert c["D"] % R.K_GROUP != 0 and c["M"] > 1
    ref = R.sweep_case_reference(c)
    gref, gmeas = R.sweep_case_emulation(c, variant=defect)
    f = _rejection(lambda: R.check_sweep_backward(defect, ref, torch.from_numpy(gref), [torch.from_numpy(t) for t in gmeas]))
    print("\nsweep backward defect %-16s rejected by x%.3g" % (defect, f))
    assert f > 1.0


# ------------------------------------------------------------------------------------------------ ConvLSTM gate backward
def _lstm_check(what, case, variant=None, with_gc=True):
    gates, c_in, gh, gc = R.lstm_case(case)
    gc = gc if with_gc else None
    ggv, ggb, gcv, gcb = R.lstm_backward_reference(gates, c_in, gh, gc)
    eg, ec = R.emulate_lstm_backward(gates.numpy(), c_in.numpy(), gh.numpy(), None if gc is None else gc.numpy(), variant)
    w1 = R.check_bound(what + " grad_gates", torch.from_numpy(eg), ggv, ggb)
    w2 = R.check_bound(what + " grad_c_in", torch.from_numpy(ec), gcv, gcb)
    return max(w1, w2)


@pytest.mark.parametrize("with_gc", [True, False])
@pytest.mark.parametrize("name", list(R.LSTM_CASES))
def test_lstm_backward_emulation_within_bound(name, with_gc):
    worst = _lstm_check(name, name, with_gc=with_gc)
    print("\nlstm backward %-14s grad_c %-5s emulation err/bound %.4f" % (name, with_gc, worst))
    assert worst * 8 <= 1.0


@pytest.mark.parametrize("defect", R.LSTM_DEFECTS)
def test_lstm_backward_planted_defect_rejected(defect):
    f = _rejection(lambda: _lstm_check(defect, "hw64_C32_B4", variant=defect))
    print("\nlstm backward defect %-20s rejected by x%.3g" % (defect, f))
    assert f > 1.0


# ------------------------------------------------------------------------------------------------ depth loss
def _loss_check(case, loss_type, variant=None, seed=0):
    preds, gt, weights, up = R.loss_case(case)
    sums, bound = R.loss_forward_reference(preds, gt)
    es, eg = R.emulate_loss(preds, gt, weights, up, loss_type, variant, seed)
    wf = R.check_loss_sums("%s %s sums" % (case, loss_type), es, sums, bound)
    ref = R.loss_backward_reference(preds, gt, weights, up, loss_type, sums[:, 4])
    wb, amb = R.check_loss_grad("%s %s grad" % (case, loss_type), eg, ref)
    return wf, wb, amb


@pytest.mark.parametrize("loss_type", list(R.LOSS_COLUMN))
@pytest.mark.parametrize("case", R.CPU_LOSS_CASES)
def test_loss_emulation_within_bound(case, loss_type):
    preds, gt, _, _ = R.loss_case(case)
    reach = R.loss_reach(preds, gt)
    wf, wb, amb = _loss_check(case, loss_type, seed=3)
    print("\nloss %-24s %-7s emulation sums err/bound %.4f  grad err/bound %.4f  ambiguous %d  %s" % (case, loss_type, wf, wb, amb, reach))
    assert wf * 8 <= 1.0 and wb * 8 <= 1.0


def test_loss_gradient_constant():
    """the worst |emulated gradient - fp64| in units of u |gradient| over every case and loss type: C_GRAD is >= 8x it"""
    worst = 0.0
    for case in R.CPU_LOSS_CASES:
        for lt in R.LOSS_COLUMN:
            worst = max(worst, _loss_check(case, lt)[1] * R.C_GRAD)
    print("\nloss gradient: worst err / (u |gradient|) = %.3f (C_GRAD = %g)" % (worst, R.C_GRAD))
    assert worst * 8 <= R.C_GRAD


LOSS_DEFECT_CASES = {                           # (case, loss type)
    "other_count": ("five_scales_odd_ratios", "L1"),
    "sign0": ("one_scale_B2_20x20", "L1"),      # p = g at 10 % of the pixels
    "round_index": ("five_scales_odd_ratios", "L1-inv"),
    "inv_g2": ("one_scale_B2_20x20", "L1-inv"),
    "neg_invalid": ("one_scale_B2_20x20", "L1"),
}


@pytest.mark.parametrize("defect", sorted(LOSS_DEFECT_CASES))
def test_loss_planted_defect_rejected(defect):
    case, lt = LOSS_DEFECT_CASES[defect]
    f = _rejection(lambda: _loss_check(case, lt, variant=defect))
    print("\nloss defect %-12s rejected by x%.3g" % (defect, f))
    assert f > 1.0


@pytest.mark.parametrize("loss_type", ["Huber"])
def test_loss_huber_le_is_unobservable(loss_type):
    """'<=' instead of '<' at Huber's |d| < 1 changes nothing: at |d| = 1 both branches give 0.5 in the forward and d = sign(d) in the
    backward, so the sums and gradients agree bit for bit, on a case that puts |p - g| exactly at 1"""
    preds, gt, weights, up = R.loss_case("one_scale_B2_20x20")
    assert R.loss_reach(preds, gt)["one_apart"] > 0
    a_s, a_g = R.emulate_loss(preds, gt, weights, up, loss_type)
    b_s, b_g = R.emulate_loss(preds, gt, weights, up, loss_type, variant="huber_le")
    assert np.array_equal(a_s.view(np.uint32), b_s.view(np.uint32))
    assert all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a_g, b_g))


def test_nearest_index_rule_matches_torch_on_every_case():
    for case in R.LOSS_CASES:
        B, H, W, sizes, _, _ = R.LOSS_CASES[case]
        for hs, ws in sizes:
            R.assert_nearest_matches_torch(H, W, hs, ws)
    assert U == 2.0 ** -24
