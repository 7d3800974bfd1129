"""The fp64 reference and error bound of tests/tc_reference.py are neither vacuous nor tighter than honest fp32 accumulation:
a stand-in "kernel" (fp32 im2col matmul over the same fp16-rounded operands, split-K partial sums added in order, fp32
epilogue) passes the comparator, and each planted defect of the kind a tensor-core kernel rewrite could introduce is rejected."""
import pytest
import torch
import torch.nn.functional as F

from tests import tc_reference as R


def _round_toward_zero(x):
    """fp16 rounding toward zero instead of to nearest"""
    h = x.half()
    away = h.float().abs() > x.abs()
    bits = h.view(torch.int16)
    return torch.where(away, bits - 1, bits).view(torch.float16)       # sign-magnitude: one step down in magnitude


def standin(x32, w32, terms, stride, bias, residual, residual_mode, act, ksplit, defect=None):
    """x32 (B,Cin,H,W) fp32, w32 [k][k][Cin][Cout] fp32 -> (B,Cout,Ho,Wo) fp32, computed in fp32 like the kernels"""
    k = w32.shape[0]
    pad = (k - 1) // 2
    B, Cin, H, W = x32.shape
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    xh = _round_toward_zero(x32) if defect == "round_toward_zero" else x32.half()
    xl = (x32 - xh.float()).half()
    wh = w32.half()
    wl = (w32 - wh.float()).half()
    cols_h = F.unfold(xh.float(), k, padding=pad, stride=stride)          # (B, Cin*k*k, L), rows ordered (cin, ky, kx)
    cols_l = F.unfold(xl.float(), k, padding=pad, stride=stride)
    mat = lambda w: w.float().permute(3, 2, 0, 1).reshape(w.shape[3], -1)   # (Cout, Cin*k*k)
    taps = torch.arange(Cin * k * k) % (k * k)
    if defect == "lost_edge_tap":
        # tap (0, 0) skipped for the output pixels of the bottom row and the right column
        edge = torch.zeros(Ho, Wo, dtype=torch.bool)
        edge[-1, :] = True
        edge[:, -1] = True
        drop = (taps == 0).float()[None, :, None] * edge.reshape(1, 1, -1).float()
        cols_h = cols_h * (1 - drop)
        cols_l = cols_l * (1 - drop)
    per = (k * k + ksplit - 1) // ksplit
    parts = []
    for sp in range(ksplit):
        sel = ((taps >= sp * per) & (taps < (sp + 1) * per)).float()[None, :, None]
        p = mat(wh) @ (cols_h * sel)
        if terms == 3:
            if defect != "drop_lo_hi":
                p = p + mat(wh) @ (cols_l * sel)
            p = p + mat(wl) @ (cols_h * sel)
        parts.append(p)
    if defect == "split_part_twice":
        parts.append(parts[0])
    y = torch.zeros_like(parts[0])
    for p in parts:
        y = y + p
    y = y.reshape(B, -1, Ho, Wo)
    if bias is not None:
        b = torch.roll(bias, -1) if defect == "bias_from_next_channel" else bias
        y = y + b.view(1, -1, 1, 1)
    if residual_mode == R.RES_SAME:
        y = y + residual
    elif residual_mode == R.RES_NEAREST_UP:
        Hr, Wr = residual.shape[2:]
        ry = torch.arange(Ho) * Hr // Ho
        rx = torch.arange(Wo) * Wr // Wo
        if defect == "residual_neighbour_pixel":
            rx = (rx + 1).clamp_max(Wr - 1)
        y = y + residual[:, :, ry][:, :, :, rx]
    if act == R.ACT_RELU:
        y = y.clamp_min(0)
    elif act == R.ACT_SIGMOID:
        y = torch.sigmoid(y)
    return y


# name, B, Cin, Cout, H, W, k, stride, terms, residual mode, act, ksplit
CASES = [
    ("k3_res_nearest_relu", 2, 8, 16, 11, 13, 3, 1, 1, R.RES_NEAREST_UP, R.ACT_RELU, 1),
    ("k3_terms3_bias", 2, 8, 16, 11, 13, 3, 1, 3, R.RES_NONE, R.ACT_NONE, 1),
    ("k3_split3_same", 1, 16, 16, 9, 10, 3, 1, 1, R.RES_SAME, R.ACT_NONE, 3),
    ("k5_s2_sigmoid", 2, 8, 8, 13, 11, 5, 2, 3, R.RES_NONE, R.ACT_SIGMOID, 2),
]

DEFECTS = {  # defect -> the case that must reject it
    "round_toward_zero": "k3_res_nearest_relu",
    "drop_lo_hi": "k3_terms3_bias",
    "lost_edge_tap": "k3_res_nearest_relu",
    "residual_neighbour_pixel": "k3_res_nearest_relu",
    "bias_from_next_channel": "k3_terms3_bias",
    "split_part_twice": "k3_split3_same",
}


def _run(case, defect=None):
    name, B, Cin, Cout, H, W, k, stride, terms, res_mode, act, ksplit = case
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(k, k, Cin, Cout, generator=g) * (2.0 / (Cin * k * k)) ** 0.5
    bias = torch.randn(Cout, generator=g) * 0.1
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    residual = None
    if res_mode == R.RES_SAME:
        residual = torch.randn(B, Cout, Ho, Wo, generator=g)
    elif res_mode == R.RES_NEAREST_UP:
        residual = torch.randn(B, Cout, (Ho + 1) // 2, (Wo + 1) // 2, generator=g)
    got = standin(x, w, terms, stride, bias, residual, res_mode, act, ksplit, defect)
    xh, xl = R.fp16_split(x)
    ref = R.conv_reference(xh, xl, w, terms, stride, bias, residual, res_mode, act, ksplit=ksplit)
    return R.check(name, got, ref.y, ref.bound, ref.S, ref.eps_acc / R.C_ACC)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_honest_fp32_accumulation_passes(case):
    worst, acc = _run(case)
    assert worst <= 1.0


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_planted_defect_is_rejected(defect):
    case = next(c for c in CASES if c[0] == DEFECTS[defect])
    with pytest.raises(AssertionError, match="exceeds the bound"):
        _run(case, defect)


def test_lstm_reference_matches_the_epilogue_in_fp32():
    """an fp32 evaluation of the gate epilogue (the kernel's arithmetic, other summation order) stays inside lstm_reference's bound"""
    g = torch.Generator().manual_seed(5)
    B, h, w, C = 2, 5, 7, 32
    gates = torch.randn(B, h, w, 4 * C, generator=g) * 2
    c = torch.randn(B, h, w, C, generator=g)
    hn, cn, bh, bc = R.lstm_reference(gates, c)
    x = gates.reshape(B, h * w, 4 * C)
    gi, gf, go, gg = x.split(C, -1)

    def ln(t):
        m = t.mean(1, keepdim=True)
        return (t - m) * torch.rsqrt(((t - m) ** 2).mean(1, keepdim=True) + 1e-5)

    cnext = ln(torch.sigmoid(gf) * c.reshape(B, h * w, C) + torch.sigmoid(gi) * F.celu(ln(gg)))
    h32 = torch.sigmoid(go) * F.celu(cnext)
    R.check("lstm h fp32", h32.reshape(B, h, w, C), hn, bh)
    R.check("lstm c fp32", cnext.reshape(B, h, w, C), cn, bc)
    with pytest.raises(AssertionError):                       # the forget and input gates swapped
        bad = ln(torch.sigmoid(gi) * c.reshape(B, h * w, C) + torch.sigmoid(gf) * F.celu(ln(gg)))
        R.check("lstm c swapped gates", bad.reshape(B, h, w, C), cn, bc)
