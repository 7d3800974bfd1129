"""fp64 reference of the tensor-core convolutions and of the ConvLSTM gate epilogue, computed from the fp16 operands the kernels
multiply, with an element-wise error bound.  Shared by the GPU tests (tests/test_tc_reference.py) and by the CPU test that
checks the bound rejects planted defects (tests/test_tc_reference_bound.py); nothing here needs a GPU.

Error model of a tensor-core convolution (fp16 x fp16 products are exact in fp32; only the fp32 accumulation rounds):

    |y_kernel - y_ref| <= eps_acc * S + EPS_EP * (|conv| + |bias| + |residual|)

    S        = conv64(|x^|, |w^|) over the same terms (the magnitude the accumulation error scales with)
    eps_acc  = C_ACC * u * n,  u = 2^-24, n = terms * K / 16 + ksplit: one accumulation step per k16 MMA (wgmma adds 16
               products into the fp32 accumulator per step; Hopper's adder is not an IEEE sequential sum, so the model charges a
               full step, not one addition, with C_ACC units of u) plus one fp32 addition per split-K partial sum
    EPS_EP   = the fp32 bias / residual additions of the epilogue.

The bound is carried through ReLU (1-Lipschitz), the sigmoid and aux = 1/(mult * act + base) by their derivatives, and
fp16 outputs add their representation error."""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24          # fp32 unit roundoff
C_ACC = 32.0            # units of u per accumulation step: >= 8x the worst err / (u * n * S) measured on an H100 SXM (2.71, 700 W);
                        # the GPU tests print the measured value of every case
EPS_EP = 4 * U
EPS_FN = 8 * U          # expf / expm1f / rsqrtf / division: a few ulp each
H16 = 2.0 ** -11        # fp16 unit roundoff
H16_TINY = 2.0 ** -25   # half the fp16 subnormal spacing: absolute rounding error below 2^-14

ACT_NONE, ACT_RELU, ACT_SIGMOID = 0, 1, 2
RES_NONE, RES_SAME, RES_NEAREST_UP = 0, 1, 2


def fp16_split(x):
    """x (fp32) -> (fp16_rn(x), fp16_rn(x - hi)) as float64; the subtraction is exact in fp32"""
    x = x.float()
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi.double(), lo.double()


def conv64(x, w_kkio, stride):
    """float64 convolution, x (B,Cin,H,W), weights [k][k][Cin][Cout], zero padding (k-1)/2"""
    w = w_kkio.permute(3, 2, 0, 1).contiguous()
    return F.conv2d(x, w, None, stride, (w.shape[-1] - 1) // 2)


def nearest_up(r, size):
    """RES_NEAREST_UP: the residual map (B,C,Hr,Wr) read at the nearest coarse pixel of every output pixel"""
    return F.interpolate(r, size=size, mode="nearest")


class Ref:
    """y: reference output; bound: element-wise bound on |kernel - y|; S: the accumulation magnitude; z: pre-activation"""

    def __init__(self, y, bound, S, z, eps_acc, aux=None, aux_bound=None):
        self.y, self.bound, self.S, self.z, self.eps_acc, self.aux, self.aux_bound = y, bound, S, z, eps_acc, aux, aux_bound


def conv_reference(xh, xl, w32, terms, stride=1, bias=None, residual=None, residual_mode=RES_NONE, act=ACT_NONE, aux=None,
                   k_padded=None, ksplit=1):
    """xh / xl: (B,Cin,H,W) float64 hi / lo operands (xl unused for terms=1); w32: fp32 [k][k][Cin][Cout] (BN folded), split here;
    bias (Cout,), residual (B,C,Hout,Wout) for RES_SAME or (B,C,Hr,Wr) for RES_NEAREST_UP; aux = (mult, base).
    k_padded: GEMM K the kernel runs (channel padding included; default k*k*Cin)."""
    wh, wl = fp16_split(w32.to(xh.device))
    y = conv64(xh, wh, stride)
    S = conv64(xh.abs(), wh.abs(), stride)
    if terms == 3:          # tc_mma_chunk's order: hi*hi, lo*hi, hi*lo
        y = y + conv64(xl, wh, stride) + conv64(xh, wl, stride)
        S = S + conv64(xl.abs(), wh.abs(), stride) + conv64(xh.abs(), wl.abs(), stride)
    k = w32.shape[0]
    K = k_padded if k_padded is not None else k * k * w32.shape[2]
    eps_acc = C_ACC * U * (terms * math.ceil(K / 16) + ksplit)
    z, mag = y, y.abs()
    if bias is not None:
        b = bias.double().to(y.device).view(1, -1, 1, 1)
        z, mag = z + b, mag + b.abs()
    if residual_mode != RES_NONE:
        r = residual.double().to(y.device)
        if residual_mode == RES_NEAREST_UP:
            r = nearest_up(r, z.shape[2:])
        z, mag = z + r, mag + r.abs()
    bz = eps_acc * S + EPS_EP * mag
    out, bound = activation(z, bz, act)
    ref = Ref(out, bound, S, z, eps_acc)
    if aux is not None:
        ref.aux, ref.aux_bound = aux_reference(out, bound, *aux)
    return ref


def activation(z, bz, act):
    if act == ACT_RELU:
        return z.clamp_min(0.0), bz
    if act == ACT_SIGMOID:
        s = torch.sigmoid(z)
        return s, (s * (1 - s) + 0.1 * bz) * bz + EPS_FN * s          # |sigmoid''| <= 0.1
    return z, bz


def aux_reference(a, ba, mult, base):
    d = mult * a + base
    slack = d.abs() - abs(mult) * ba
    assert bool((slack > 0).all()), "aux denominator within the error bound of zero"
    aux = 1.0 / d
    return aux, abs(mult) * ba / (d.abs() * slack) + EPS_FN * aux.abs()


def fp16_bound(y, bound, pair=False):
    """bound on |fp16 output - y|: the kernel's fp32 value is within `bound`, then rounded to fp16 (or to an fp16 pair hi + lo)"""
    if pair:
        return bound + H16 * H16 * 2 * (y.abs() + bound) + H16_TINY
    return bound + H16 * (y.abs() + bound) + H16_TINY


def check(what, got, ref_y, bound, S=None, eps_scale=None, report=None):
    """Asserts |got - ref_y| <= bound element-wise (got: float tensor of the reference's shape).  Returns (worst err / bound,
    worst err / (u * n * S) -- the measured accumulation constant in units of the model's C_ACC) and names the worst element."""
    got = got.double().to(ref_y.device)
    err = (got - ref_y).abs()
    finite = bool(torch.isfinite(got).all())
    ratio = err / bound.clamp_min(1e-300)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    acc = 0.0
    if S is not None and eps_scale is not None:
        acc = float((err / (eps_scale * S).clamp_min(1e-300)).max())
    if report is not None:
        report.append((what, worst, acc))
    if not finite or worst > 1.0:
        idx = tuple(int(i) for i in torch.nonzero(ratio == ratio.max())[0]) if finite else None
        raise AssertionError("%s: |kernel - fp64 reference| exceeds the bound by x%.3g at index %s (kernel %r, reference %r, bound %.3e)%s"
                             % (what, worst, idx, float(got[idx]) if idx else None, float(ref_y[idx]) if idx else None,
                                float(bound[idx]) if idx else 0.0, "" if finite else " -- non-finite output"))
    return worst, acc


# ------------------------------------------------------------------------------------------------ ConvLSTM gate epilogue
EPS_LSTM = 8 * U        # per elementary fp32 operation; see lstm_reference


def lstm_reference(g, c):
    """float64 restatement of the gate epilogue (reference convlstm.py:45-59, csrc/conv.cu lstm_gates_kernel) on the kernel's
    own fp32 pre-activations g (B,h,w,4C) and cell state c (B,h,w,C).  Returns (h, c_next, bound_h, bound_c).

    Bound: the sums over the n = h*w positions of the two-pass statistics err by <= n*u of the summed magnitudes, the pointwise
    functions by EPS_LSTM relative.  For x^ = (x - mean) * rstd that gives |dx^| <= e_n * (kappa + |x^|), e_n = (n + 8) * EPS_LSTM,
    kappa = rstd * mean|x| (how much a relative error of x is amplified by the centring); errors of the LayerNorm input dc add
    rstd * (|dc_p| + max dc) * (1 + |x^|)."""
    B, h, w, C4 = g.shape
    C = C4 // 4
    n = h * w
    g = g.double().reshape(B, n, C4)
    c = c.double().reshape(B, n, C)
    gi, gf, go, gg = g[..., :C], g[..., C:2 * C], g[..., 2 * C:3 * C], g[..., 3 * C:]
    e_n = (n + 8) * EPS_LSTM

    def ln(x):
        m = x.mean(1, keepdim=True)
        r = 1.0 / torch.sqrt(((x - m) ** 2).mean(1, keepdim=True) + 1e-5)
        xn = (x - m) * r
        return xn, r, r * x.abs().mean(1, keepdim=True)

    def celu(x):
        return torch.where(x > 0, x, torch.expm1(x))

    si, sf, so = torch.sigmoid(gi), torch.sigmoid(gf), torch.sigmoid(go)
    gn, _, kappa_g = ln(gg)
    b_gn = e_n * (kappa_g + gn.abs())
    cg = celu(gn)
    b_cg = b_gn + EPS_LSTM * (cg.abs() + 1)
    cn_pre = sf * c + si * cg
    b_pre = si * b_cg + EPS_LSTM * 4 * (sf * c.abs() + si * cg.abs() + si + sf)
    cn, r_c, kappa_c = ln(cn_pre)
    b_cn = e_n * (kappa_c + cn.abs()) + r_c * (b_pre + b_pre.amax(1, keepdim=True)) * (1 + cn.abs())
    hn = so * celu(cn)
    b_h = so * (b_cn + EPS_LSTM * (cn.abs() + 1)) + EPS_LSTM * 4 * (hn.abs() + so)
    shape = (B, h, w, C)
    return hn.reshape(shape), cn.reshape(shape), b_h.reshape(shape), b_cn.reshape(shape)


def check_live(what, *tensors):
    """operands replayed from an engine's buffers are finite and not all zero: a replay on a zero hidden state or on a buffer
    nothing wrote proves nothing"""
    for i, t in enumerate(tensors):
        if t is None:
            continue
        assert bool(torch.isfinite(t).all()), "%s: operand %d is not finite" % (what, i)
        assert bool((t != 0).any()), "%s: operand %d is all zero" % (what, i)
