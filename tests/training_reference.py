"""fp64 references of the training-step kernels (csrc/geometry.cu plane_sweep_backward_c32_kernel, csrc/training.cu
lstm_gates_backward_kernel, depth_loss_forward_kernel, depth_loss_backward_kernel), each with a per-element bound, and fp32
emulations of the kernels in their own operation order.  Shared by the GPU tests (tests/test_training_reference.py) and by the CPU
test that checks the bounds against the emulations and against planted defects (tests/test_training_reference_bound.py); nothing
here needs a GPU.

Plane-sweep backward, g the upstream gradient (B,h,w,D), positions, deltas and the ill-conditioned test of tests/sweep_reference.py:
    grad_ref[p, c]    = 1/(32 M) sum_{m,d} g[p,d] sum_t w_t f2_m[q_t, c]
    grad_meas_m[q, c] = 1/(32 M) sum_{p,d: q a tap of (p,d,m)} g[p,d] w_t f1[p, c]
    grad_ref bound    (M D + C_BLEND + 1) u sum |g| sum_t w_t |f2| / (32 M)   (one fmaf chain over M D steps, the blend, gscale)
                      + per channel delta_x Lx + delta_y Ly + delta_x delta_y Lc, L the largest tap differences of that channel over
                      the cells the delta box touches; an ill-conditioned sample: 2 |g| max|f2_m| of the channel, counted
    grad_meas bound   2 (delta_x + delta_y + delta_x delta_y) |g f1| / (32 M), summed over the samples whose 4x4 block contains q
                      + (C_BLEND + n_q) u w |g f1| / (32 M), n_q the atomic additions into q (any order)
                      + |g f1| / (32 M) of every ill-conditioned sample on every pixel of its batch entry
    exact +0          grad_meas pixels no tap can reach; grad_ref pixels none of whose samples with g != 0 can touch the image.

ConvLSTM gate backward: the derivative of the gate epilogue (tests/tc_reference.py lstm_reference) at the kernel's fp32 inputs,
LayerNorm dx = rstd (dy - mean dy - x^ mean(dy x^)), sigmoid' = s (1 - s), celu' = exp(x) for x <= 0.  The bound is a running
error carried as (value, bound) through the kernel's own expression order: every fp32 operation charges EPS_LSTM relative, the
hw-position means (hw + 8) EPS_LSTM sum|.| / hw, rsqrtf / expf / expm1f EPS_FN.  The rstd amplification of near-constant channels
comes out of the propagation.

Depth loss: per scale j, over the pixels whose nearest-down-sampled ground truth is non-zero (NaN is non-zero, as in the reference),
the sums [l1, huber, l1_inv, l1_rel, count].  Nearest index: torch's fp32 rule min(floorf(dst * (float)in / out), in - 1).
    sums bound        C_TERM u per term (l1_inv: u (|1/g| + |1/p|), the subtraction cancels) + (5 + 8 + blocks_j) u sum |terms|
                      (shuffle tree, 8-warp sum, one atomic per block of the scale); counts exact (< 2^24 per scale, asserted)
    gradient          up w_j / count_j dl within C_GRAD u relative; the sign of p - g is exact in fp32, the sign of 1/g - 1/p and the
                      side of Huber's |d| < 1 are not: within rounding of the branch point either branch is accepted (counted).
                      g = 0 and every element of a scale without a valid pixel is +0.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from tests.sweep_reference import C_BLEND, _f32, _patch_index, emulate_positions, fmaf, plane_depths, positions
from tests.tc_reference import EPS_FN, EPS_LSTM, U

C_TERM = 4.0            # units of u per loss term: |g - p| (1), 0.5 d d (3), d / g (2), 1/g - 1/p (2 of |1/g| + |1/p|)
C_GRAD = 32.0           # units of u of |gradient|: >= 8x the worst measured by the emulation (the CPU test prints it)
K_GROUP = 8             # planes per step of plane_sweep_backward_c32_kernel
LOSS_THREADS = 256      # threads per block of the loss kernels
MAX_SCALES = 8


def _bits_zero(t):
    return t.contiguous().view(torch.int32) == 0


def check_exact_zero(what, got, zero):
    """got (torch float32) is +0 bit for bit wherever zero (got's shape, or got's without the channel) is set"""
    if zero.dim() < got.dim():
        zero = zero[..., None].expand_as(got)
    bad = zero & ~_bits_zero(got)
    if bool(bad.any()):
        i = tuple(int(v) for v in torch.nonzero(bad)[0])
        raise AssertionError("%s: element %s must be +0, kernel %r" % (what, i, float(got[i])))
    return int(zero.sum())


def check_bound(what, got, y, bound):
    """|got - y| <= bound element-wise, non-finite got fails; returns the worst err / bound"""
    got = got.double().to(y.device)
    err = (got - y).abs()
    ratio = torch.where(torch.isfinite(got), err / bound.clamp_min(1e-300), torch.full_like(err, math.inf))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if worst > 1.0:
        i = tuple(int(v) for v in torch.nonzero(ratio == ratio.max())[0])
        raise AssertionError("%s: |kernel - fp64 reference| exceeds the bound by x%.3g at %s (kernel %r, reference %r, bound %.3e)"
                             % (what, worst, i, float(got[i]), float(y[i]), float(bound[i])))
    return worst


# ------------------------------------------------------------------------------------------------ plane-sweep backward
class SweepBwdRef:
    def __init__(self, **kw):
        self.__dict__.update(kw)

    def meas(self, frames):
        """(y, bound, zero) of a gradient buffer the listed frames accumulate into (one frame, or an aliased buffer)"""
        y = sum(self.meas_y[m] for m in frames)
        S = sum(self.meas_S[m] for m in frames)
        cnt = sum(self.meas_cnt[m] for m in frames)
        pos = sum(self.meas_pos[m] for m in frames)
        ill = sum(self.meas_ill[m] for m in frames)
        bound = (C_BLEND + cnt[..., None]) * U * (S + ill) + pos + ill
        reach = torch.stack([self.meas_reach[m] for m in frames]).any(0)
        return y, bound, ~reach


def sweep_backward_reference(f1, f2s, pose1, pose2s, K, min_depth, max_depth, D, g):
    """f1, f2s[m] (B,h,w,32) and g (B,h,w,D) fp32, pose1 (B,4,4), pose2s [M x (B,4,4)], K (B,3,3) fp32, all on one device.
    Returns SweepBwdRef: ref_y / ref_bound / ref_zero (B,h,w,C), per frame the parts of its gradient (combined by .meas), and the
    sample classes: n_live, n_outside, n_ill, per-border straddle counts, n_behind (den < 0, live) -- what a case can assert."""
    B, h, w, C = f1.shape
    M = len(f2s)
    dev = f1.device
    depths = plane_depths(min_depth, max_depth, D)
    gs = 1.0 / (32 * M)
    npix = B * h * w
    f1d = f1.double()
    g64 = g.double()
    y_ref = torch.zeros(B, h, w, C, dtype=torch.float64, device=dev)
    acc_ref, pos_ref, ill_ref = torch.zeros_like(y_ref), torch.zeros_like(y_ref), torch.zeros_like(y_ref)
    reach_ref = torch.zeros(B, h, w, dtype=torch.bool, device=dev)
    meas_y, meas_S, meas_cnt, meas_pos, meas_ill, meas_reach = [], [], [], [], [], []
    stats = dict(n_live=0, n_outside=0, n_ill=0, n_behind=0, left=0, right=0, top=0, bottom=0, n_gzero=0)
    b_off = (torch.arange(B, device=dev) * (h * w)).view(B, 1, 1, 1)
    chunk = max(1, min(D, (1 << 22) // (npix * 16 * C)))
    inner = [5, 6, 9, 10]
    for m in range(M):
        f2z = torch.cat([f2s[m].double().reshape(npix, C), f2s[m].new_zeros(1, C, dtype=torch.float64)])
        cap = f2s[m].double().abs().reshape(B, h * w, C).amax(1)                      # (B,C)
        y_m = torch.zeros(npix + 1, C, dtype=torch.float64, device=dev)
        S_m, pos_m = torch.zeros_like(y_m), torch.zeros_like(y_m)
        cnt_m = torch.zeros(npix + 1, dtype=torch.float64, device=dev)
        reach_m = torch.zeros(npix + 1, dtype=torch.float64, device=dev)
        ill_m = torch.zeros(B, C, dtype=torch.float64, device=dev)
        nill_m = torch.zeros(B, dtype=torch.float64, device=dev)
        for d0 in range(0, D, chunk):
            ds = torch.arange(d0, min(D, d0 + chunk))
            P = positions(pose1, pose2s[m], K, depths, h, w, ds)
            xs, ys, dx, dy = P["xs"], P["ys"], P["delta_x"], P["delta_y"]
            gd = g64[..., ds.to(dev)].permute(0, 3, 1, 2)                             # (B,d,h,w)
            act = gd != 0
            fin = torch.isfinite(xs) & torch.isfinite(ys)
            outside = fin & ((xs + dx <= -1) | (xs - dx >= w) | (ys + dy <= -1) | (ys - dy >= h))
            ill = act & ~outside & ~(fin & (dx < 1) & (dy < 1))
            live = act & ~outside & ~ill
            stats["n_gzero"] += int((~act).sum())
            stats["n_live"] += int(live.sum())
            stats["n_outside"] += int((act & outside).sum())
            stats["n_ill"] += int(ill.sum())
            stats["n_behind"] += int((live & (P["den"] < 0)).sum())
            stats["left"] += int((live & (xs < 0)).sum())
            stats["right"] += int((live & (xs > w - 1)).sum())
            stats["top"] += int((live & (ys < 0)).sum())
            stats["bottom"] += int((live & (ys > h - 1)).sum())
            xs_c, ys_c = torch.where(live, xs, -5.0), torch.where(live, ys, -5.0)
            idx, x0, y0 = _patch_index(xs_c, ys_c, h, w, npix, b_off)                  # (B,d,h,w,16)
            fx, fy = xs_c - x0, ys_c - y0
            wt = torch.stack([(1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy], -1)
            wt = torch.where(live[..., None], wt, torch.zeros_like(wt))
            ga = (gd.abs() * gs)[..., None]                                            # (B,d,h,w,1)
            gv = (gd * gs)[..., None]
            # ---- grad_ref: gather
            pat = f2z[idx]                                                             # (B,d,h,w,16,C)
            val = (wt[..., None] * pat[..., inner, :]).sum(-2)
            mag = (wt[..., None] * pat[..., inner, :].abs()).sum(-2)
            p4 = pat.reshape(*pat.shape[:-2], 4, 4, C)
            dxm = (p4[..., :, 1:, :] - p4[..., :, :-1, :]).abs()                       # (..,4,3,C)
            dym = (p4[..., 1:, :, :] - p4[..., :-1, :, :]).abs()                       # (..,3,4,C)
            crm = (p4[..., 1:, 1:, :] - p4[..., 1:, :-1, :] - p4[..., :-1, 1:, :] + p4[..., :-1, :-1, :]).abs()
            del pat, p4
            dx_, dy_ = dx.clamp(max=1.0), dy.clamp(max=1.0)
            cx_lo, cx_hi = torch.floor(xs_c - dx_) - x0, torch.floor(xs_c + dx_) - x0
            cy_lo, cy_hi = torch.floor(ys_c - dy_) - y0, torch.floor(ys_c + dy_) - y0
            o = torch.arange(-1, 2, device=dev, dtype=torch.float64)
            col = (o >= cx_lo[..., None]) & (o <= cx_hi[..., None])
            row = (o >= cy_lo[..., None]) & (o <= cy_hi[..., None])
            cell = (row[..., :, None] & col[..., None, :])[..., None]                   # (..,3,3,1)
            Lx = (torch.maximum(dxm[..., :3, :, :], dxm[..., 1:, :, :]) * cell).amax((-2, -3))
            Ly = (torch.maximum(dym[..., :, :3, :], dym[..., :, 1:, :]) * cell).amax((-2, -3))
            Lc = (crm * cell).amax((-2, -3))
            del dxm, dym, crm
            pos = dx_[..., None] * Lx + dy_[..., None] * Ly + (dx_ * dy_)[..., None] * Lc
            y_ref += (gv * val).sum(1)
            acc_ref += (ga * mag).sum(1)
            pos_ref += torch.where(live[..., None], ga * pos, torch.zeros_like(pos)).sum(1)
            ill_ref += torch.where(ill[..., None], 2.0 * ga * cap[:, None, None, None, :], torch.zeros_like(pos)).sum(1)
            reach_ref |= (live | ill).any(1)
            # ---- grad_meas: scatter
            f1b = f1d[:, None].expand(B, len(ds), h, w, C)
            for t, k in enumerate(inner):
                it = idx[..., k].reshape(-1)
                y_m.index_add_(0, it, (gv * wt[..., t, None] * f1b).reshape(-1, C))
                S_m.index_add_(0, it, (ga * wt[..., t, None] * f1b.abs()).reshape(-1, C))
                cnt_m.index_add_(0, it, (live & (wt[..., t] > 0)).double().reshape(-1))
            pf = torch.where(live[..., None], 2.0 * (dx_ + dy_ + dx_ * dy_)[..., None] * ga * f1b.abs(), torch.zeros_like(f1b))
            pf = pf.reshape(-1, C)
            for k in range(16):
                it = idx[..., k].reshape(-1)
                pos_m.index_add_(0, it, pf)
                reach_m.index_add_(0, it, live.double().reshape(-1))
            ill_m += torch.where(ill[..., None], ga * f1b.abs(), torch.zeros_like(f1b)).sum((1, 2, 3))
            nill_m += ill.double().sum((1, 2, 3))
        ill_pix = (ill_m[:, None, :].expand(B, h * w, C)).reshape(npix, C)
        meas_y.append(y_m[:npix].reshape(B, h, w, C))
        meas_S.append(S_m[:npix].reshape(B, h, w, C))
        meas_cnt.append((cnt_m[:npix].reshape(B, h * w) + 4 * nill_m[:, None]).reshape(B, h, w))
        meas_pos.append(pos_m[:npix].reshape(B, h, w, C))
        meas_ill.append(ill_pix.reshape(B, h, w, C))
        meas_reach.append(((reach_m[:npix].reshape(B, h * w) > 0) | (nill_m[:, None] > 0)).reshape(B, h, w))
    ref_bound = (M * D + C_BLEND + 1) * U * acc_ref + pos_ref + ill_ref
    return SweepBwdRef(ref_y=y_ref, ref_bound=ref_bound, ref_zero=~reach_ref, meas_y=meas_y, meas_S=meas_S, meas_cnt=meas_cnt,
                       meas_pos=meas_pos, meas_ill=meas_ill, meas_reach=meas_reach, depths=depths, **stats)


def check_sweep_backward(what, ref, grad_ref, grad_meas, buffers=None):
    """grad_ref (B,h,w,C) and the measurement gradient buffers (list of (B,h,w,C)) of one backward call against the reference;
    buffers[i]: the frames accumulated into grad_meas[i] (default: one per frame).  Returns (worst err / bound, exact +0 count)."""
    grad_ref = grad_ref.to(ref.ref_y.device)
    worst = check_bound(what + " grad_ref", grad_ref, ref.ref_y, ref.ref_bound)
    nz = check_exact_zero(what + " grad_ref", grad_ref, ref.ref_zero)
    buffers = buffers or [[m] for m in range(len(ref.meas_y))]
    for frames, got in zip(buffers, grad_meas):
        got = got.to(ref.ref_y.device)
        y, bound, zero = ref.meas(frames)
        worst = max(worst, check_bound("%s grad_meas%s" % (what, frames), got, y, bound))
        nz += check_exact_zero("%s grad_meas%s" % (what, frames), got, zero)
    return worst, nz


SWEEP_DEFECTS = ("clamp_border", "swap_01_10", "scale_32", "drop_last_group", "drop_frame_ref", "meas_next_frame")


def _phase_a(xs, ys, h, w, variant=None):
    """sweep_phase_a in fp32: the four flat tap indices (within the batch entry) and weights (B,h,w,4)"""
    with np.errstate(invalid="ignore"):
        inside = (xs > -1) & (xs < w) & (ys > -1) & (ys < h)
    xs, ys = np.where(inside, xs, 0).astype(np.float32), np.where(inside, ys, 0).astype(np.float32)
    x0f, y0f = np.floor(xs), np.floor(ys)
    fx, fy = _f32(xs - x0f), _f32(ys - y0f)
    gx, gy = _f32(_f32(x0f + 1) - xs), _f32(_f32(y0f + 1) - ys)
    x0, y0 = x0f.astype(np.int64), y0f.astype(np.int64)
    vx0, vx1, vy0, vy1 = x0 >= 0, x0 + 1 < w, y0 >= 0, y0 + 1 < h
    if variant == "clamp_border":         # taps outside the image read the clamped edge pixel with their weight
        vx0 = vx1 = vy0 = vy1 = np.ones_like(inside)
    xa, xb, ya, yb = np.maximum(x0, 0), np.minimum(x0 + 1, w - 1), np.maximum(y0, 0), np.minimum(y0 + 1, h - 1)
    off = np.stack([ya * w + xa, ya * w + xb, yb * w + xa, yb * w + xb], -1)
    wt = np.stack([np.where(vy0 & vx0, _f32(gx * gy), 0), np.where(vy0 & vx1, _f32(fx * gy), 0),
                   np.where(vy1 & vx0, _f32(gx * fy), 0), np.where(vy1 & vx1, _f32(fx * fy), 0)], -1).astype(np.float32)
    if variant == "swap_01_10":
        wt = wt[..., [0, 2, 1, 3]]
    off = np.where(inside[..., None], off, 0)
    wt = np.where(inside[..., None], wt, np.float32(0)).astype(np.float32)
    return off, wt


def emulate_sweep_backward(f1, f2s, pose1, pose2s, K, min_depth, max_depth, D, g, variant=None, seed=0, buffers=None):
    """plane_sweep_backward_c32_kernel in fp32 numpy, in its order: plane groups, frames, the 8 planes of a group; one fmaf chain
    per (pixel, channel) for grad_ref; grad_meas products added in a shuffled order.  buffers: as check_sweep_backward.
    Returns (grad_ref (B,h,w,C), [grad_meas buffer (B,h,w,C)])."""
    f1, g = np.asarray(f1, np.float32), np.asarray(g, np.float32)
    f2s = [np.asarray(f, np.float32) for f in f2s]
    B, h, w, C = f1.shape
    M = len(f2s)
    buffers = buffers or [[m] for m in range(M)]
    depths = plane_depths(min_depth, max_depth, D).numpy()
    pos = [emulate_positions(np.asarray(pose1), np.asarray(p2), np.asarray(K), depths, h, w, "st") for p2 in pose2s]
    gscale = _f32(np.float32(1) / np.float32(32 if variant == "scale_32" else 32 * M))
    gd_all = _f32(g * gscale)
    gref = np.zeros((B, h, w, C), np.float32)
    b_off = (np.arange(B) * h * w)[:, None, None, None]
    f2flat = [f.reshape(B * h * w, C) for f in f2s]
    contrib = [[] for _ in range(M)]
    n_groups = D // K_GROUP if variant == "drop_last_group" else (D + K_GROUP - 1) // K_GROUP
    for gi in range(n_groups):
        for m in range(M):
            for k in range(K_GROUP):
                d = gi * K_GROUP + k
                if d >= D:
                    break
                off, wt = _phase_a(pos[m][0][:, d], pos[m][1][:, d], h, w, variant)
                gd = gd_all[..., d]
                act = gd != 0
                t = f2flat[m][b_off + off]                                         # (B,h,w,4,C)
                wt_c = wt[..., None]
                blend = fmaf(t[..., 3, :], wt_c[..., 3, :], fmaf(t[..., 2, :], wt_c[..., 2, :],
                             fmaf(t[..., 1, :], wt_c[..., 1, :], _f32(t[..., 0, :] * wt_c[..., 0, :]))))
                if not (variant == "drop_frame_ref" and m == M - 1):
                    gref = np.where(act[..., None], fmaf(gd[..., None], blend, gref), gref)
                tgt = m + 1 if (variant == "meas_next_frame" and m + 1 < M) else m
                for tp in range(4):
                    c = _f32(gd * wt[..., tp])
                    sel = act & (c != 0)
                    if sel.any():
                        contrib[tgt].append(((b_off[..., 0] + off[..., tp])[sel], _f32(c[sel][:, None] * f1[sel])))
    rng = np.random.RandomState(seed)
    out = []
    for frames in buffers:
        buf = np.zeros((B * h * w, C), np.float32)
        parts = [c for m in frames for c in contrib[m]]
        if parts:
            idx = np.concatenate([p[0] for p in parts])
            val = np.concatenate([p[1] for p in parts])
            perm = rng.permutation(len(idx))
            np.add.at(buf, idx[perm], val[perm])            # fp32 additions one by one, in the shuffled order
        out.append(buf.reshape(B, h, w, C))
    return gref, out


# ------------------------------------------------------------------------------------------------ ConvLSTM gate backward
class _RE:
    """(value, bound) of a quantity the kernel computes in fp32, both float64 tensors (B, hw, C) or (B, 1, C)"""

    def __init__(self, v, e=None):
        self.v, self.e = v, (torch.zeros_like(v) if e is None else e)

    def __add__(self, o):
        o = o if isinstance(o, _RE) else _RE(torch.full_like(self.v, float(o)))
        v = self.v + o.v
        return _RE(v, self.e + o.e + EPS_LSTM * v.abs())

    def __sub__(self, o):
        o = o if isinstance(o, _RE) else _RE(torch.full_like(self.v, float(o)))
        v = self.v - o.v
        return _RE(v, self.e + o.e + EPS_LSTM * v.abs())

    def __mul__(self, o):
        v = self.v * o.v
        return _RE(v, self.v.abs() * o.e + o.v.abs() * self.e + self.e * o.e + EPS_LSTM * v.abs())


def _mean(a):
    """block_sum(...) * inv_n over the hw positions"""
    n = a.v.shape[1]
    return _RE(a.v.mean(1, keepdim=True), a.e.sum(1, keepdim=True) / n + (n + 8) * EPS_LSTM * a.v.abs().sum(1, keepdim=True) / n)


def _rsqrt(a):
    """rsqrtf of var + 1e-5: the kernel's argument is >= 1e-5 whatever its error"""
    v = 1.0 / torch.sqrt(a.v)
    lo = torch.clamp(a.v - a.e, min=1e-5 * (1 - 1e-6))
    return _RE(v, (1.0 / torch.sqrt(lo) - v) + EPS_FN * (1.0 / torch.sqrt(lo)))


def _sigmoid(x):
    """1 / (1 + expf(-x)) of an exact fp32 input; where expf may overflow (x < -88) the kernel's s is 0 and the true s < 2^-126"""
    s = torch.sigmoid(x)
    e = s * (1 - s) * EPS_FN + 2 * EPS_LSTM * s + torch.where(x < -88.0, torch.full_like(s, 2.0 ** -126), torch.zeros_like(s))
    return _RE(s, e)


def _celu(a):
    v = torch.where(a.v > 0, a.v, torch.expm1(a.v))
    return _RE(v, a.e + EPS_FN * v.abs())           # 1-Lipschitz


def _celu_grad(a):
    v = torch.where(a.v > 0, torch.ones_like(a.v), torch.exp(a.v))
    return _RE(v, a.e + EPS_FN * v)                  # 1-Lipschitz, continuous at 0


def lstm_backward_reference(gates, c_in, grad_h, grad_c=None):
    """gates (B,h,w,4C) pre-activations (i, f, o, g), c_in, grad_h, grad_c (B,h,w,C) fp32 (grad_c None: absent).  Returns
    (grad_gates, bound_gates (B,h,w,4C), grad_c_in, bound_c_in (B,h,w,C)) in float64."""
    B, h, w, C4 = gates.shape
    C = C4 // 4
    n = h * w
    g = gates.double().reshape(B, n, C4)
    ai, af, ao, ag = (_RE(g[..., k * C:(k + 1) * C]) for k in range(4))
    vc = _RE(c_in.double().reshape(B, n, C))
    gh = _RE(grad_h.double().reshape(B, n, C))
    gc = _RE(grad_c.double().reshape(B, n, C)) if grad_c is not None else _RE(torch.zeros_like(vc.v))

    def layernorm(x):
        m = _mean(x)
        d = x - m
        r = _rsqrt(_mean(d * d) + 1e-5)
        return d * r, r

    def ln_backward(dy, xh, r):
        m1, m2 = _mean(dy), _mean(dy * xh)
        return r * ((dy - m1) - xh * m2)

    nn, rstd_g = layernorm(ag)
    si, sf, so = _sigmoid(ai.v), _sigmoid(af.v), _sigmoid(ao.v)
    gg = _celu(nn)
    cp = sf * vc + si * gg
    cn, rstd_c = layernorm(cp)
    d_o = gh * _celu(cn)
    dcn = gh * so * _celu_grad(cn) + gc
    one = _RE(torch.ones_like(vc.v))
    grad_ao = d_o * so * (one - so)
    dcp = ln_backward(dcn, cn, rstd_c)
    grad_c_in = dcp * sf
    grad_af = dcp * vc * sf * (one - sf)
    grad_ai = dcp * gg * si * (one - si)
    dn = dcp * si * _celu_grad(nn)
    grad_ag = ln_backward(dn, nn, rstd_g)
    shape4, shape = (B, h, w, C4), (B, h, w, C)
    gv = torch.cat([grad_ai.v, grad_af.v, grad_ao.v, grad_ag.v], -1).reshape(shape4)
    ge = torch.cat([grad_ai.e, grad_af.e, grad_ao.e, grad_ag.e], -1).reshape(shape4)
    return gv, ge, grad_c_in.v.reshape(shape), grad_c_in.e.reshape(shape)


LSTM_DEFECTS = ("drop_mean_xy", "celu_grad_at_cp", "sigmoid_grad_s", "ignore_grad_c", "grad_c_in_without_f")


def _block_sum(x):
    """block_sum over positions p = warp + 8 j: each warp's serial sum over j, then the 8 warps in order (fp32)"""
    B, n, C = x.shape
    t = np.zeros((B, C), np.float32)
    for wp in range(8):
        s = np.zeros((B, C), np.float32)
        for p in range(wp, n, 8):
            s = _f32(s + x[:, p])
        t = _f32(t + s)
    return t[:, None]


def emulate_lstm_backward(gates, c_in, grad_h, grad_c=None, variant=None):
    """lstm_gates_backward_kernel in fp32 numpy (expression order of the kernel; the compiler may contract some a * b + c into fmaf,
    which the bound covers).  Returns (grad_gates (B,h,w,4C), grad_c_in (B,h,w,C))."""
    gates = np.asarray(gates, np.float32)
    B, h, w, C4 = gates.shape
    C = C4 // 4
    n = h * w
    g = gates.reshape(B, n, C4)
    ai, af, ao, ag = (g[..., k * C:(k + 1) * C] for k in range(4))
    vc = np.asarray(c_in, np.float32).reshape(B, n, C)
    gh = np.asarray(grad_h, np.float32).reshape(B, n, C)
    gc = np.asarray(grad_c, np.float32).reshape(B, n, C) if (grad_c is not None and variant != "ignore_grad_c") else np.zeros_like(vc)
    inv_n = _f32(np.float32(1) / np.float32(n))
    eps = np.float32(1e-5)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        sig = lambda x: _f32(np.float32(1) / _f32(np.float32(1) + np.exp(-x)))
        celu = lambda x: np.where(x > 0, x, np.expm1(x)).astype(np.float32)
        celu_grad = lambda x: np.where(x > 0, np.float32(1), np.exp(x)).astype(np.float32)
        rsqrt = lambda x: _f32(1.0 / np.sqrt(x.astype(np.float64)))
        mean_g = _f32(_block_sum(ag) * inv_n)
        d = _f32(ag - mean_g)
        rstd_g = rsqrt(_f32(_f32(_block_sum(_f32(d * d)) * inv_n) + eps))
        nn = _f32(d * rstd_g)
        si, sf, so = sig(ai), sig(af), sig(ao)
        gg = celu(nn)
        cp = _f32(_f32(sf * vc) + _f32(si * gg))
        mean_c = _f32(_block_sum(cp) * inv_n)
        dc = _f32(cp - mean_c)
        rstd_c = rsqrt(_f32(_f32(_block_sum(_f32(dc * dc)) * inv_n) + eps))
        cn = _f32(dc * rstd_c)
        d_o = _f32(gh * celu(cn))
        dcn = _f32(_f32(_f32(gh * so) * celu_grad(cp if variant == "celu_grad_at_cp" else cn)) + gc)
        grad_ao = _f32(d_o * so) if variant == "sigmoid_grad_s" else _f32(_f32(d_o * so) * _f32(np.float32(1) - so))
        m1 = _f32(_block_sum(dcn) * inv_n)
        m2 = _f32(_block_sum(_f32(dcn * cn)) * inv_n)
        if variant == "drop_mean_xy":
            m2 = np.zeros_like(m2)
        dcp = _f32(rstd_c * _f32(_f32(dcn - m1) - _f32(cn * m2)))
        grad_c_in = dcp if variant == "grad_c_in_without_f" else _f32(dcp * sf)
        grad_af = _f32(_f32(_f32(dcp * vc) * sf) * _f32(np.float32(1) - sf))
        grad_ai = _f32(_f32(_f32(dcp * gg) * si) * _f32(np.float32(1) - si))
        dn = _f32(_f32(dcp * si) * celu_grad(nn))
        k1 = _f32(_block_sum(dn) * inv_n)
        k2 = _f32(_block_sum(_f32(dn * nn)) * inv_n)
        grad_ag = _f32(rstd_g * _f32(_f32(dn - k1) - _f32(nn * k2)))
    gg_out = np.concatenate([grad_ai, grad_af, grad_ao, grad_ag], -1).reshape(B, h, w, C4)
    return gg_out, grad_c_in.reshape(B, h, w, C)


# ------------------------------------------------------------------------------------------------ multi-scale depth loss
L1, L1_INV, L1_REL, HUBER = "L1", "L1-inv", "L1-rel", "Huber"
LOSS_COLUMN = {L1: 0, HUBER: 1, L1_INV: 2, L1_REL: 3}


def nearest_index(out, inn, rounded=False):
    """torch's nearest source index in fp32: min(floorf(dst * (float)in / out), in - 1) (rounded: the planted defect)"""
    s = np.float32(inn) / np.float32(out)
    src = _f32(np.arange(out, dtype=np.float32) * s)
    src = np.floor(src + np.float32(0.5)) if rounded else np.floor(src)
    return np.minimum(src.astype(np.int64), inn - 1)


def downsampled_gt(gt, hs, ws, rounded=False):
    """gt (B,H,W) fp32 numpy read at the nearest index of every (y, x) of an (hs, ws) scale"""
    H, W = gt.shape[1:]
    return gt[:, nearest_index(hs, H, rounded)][:, :, nearest_index(ws, W, rounded)]


def assert_nearest_matches_torch(H, W, hs, ws):
    """the fp32 rule picks the pixels F.interpolate(mode='nearest') picks at this size"""
    grid = torch.arange(H * W, dtype=torch.float64).reshape(1, 1, H, W)
    want = F.interpolate(grid, size=(hs, ws), mode="nearest")[0, 0].long().numpy()
    got = nearest_index(hs, H)[:, None] * W + nearest_index(ws, W)[None, :]
    assert np.array_equal(want, got), "nearest index rule differs from F.interpolate at %dx%d -> %dx%d" % (H, W, hs, ws)


def loss_blocks(B, sizes):
    return [(B * hs * ws + LOSS_THREADS - 1) // LOSS_THREADS for hs, ws in sizes]


def loss_forward_reference(preds, gt):
    """preds [(B,hs,ws) fp32 numpy], gt (B,H,W) fp32 numpy -> (sums (n,5) float64, bound (n,5))"""
    B, H, W = gt.shape
    n = len(preds)
    sizes = [p.shape[1:] for p in preds]
    blocks = loss_blocks(B, sizes)
    sums, bound = np.zeros((n, 5)), np.zeros((n, 5))
    for j, p in enumerate(preds):
        assert_nearest_matches_torch(H, W, *sizes[j])
        g = downsampled_gt(gt, *sizes[j]).astype(np.float64)
        p = p.astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            valid = g != 0
            g, p = g[valid], p[valid]
            d = np.abs(g - p)
            terms = [d, np.where(d < 1, 0.5 * d * d, d - 0.5), np.abs(1 / g - 1 / p), d / g]
            mags = [np.abs(terms[0]), np.abs(terms[1]), np.abs(1 / g) + np.abs(1 / p), np.abs(terms[3])]
        assert valid.sum() < 2 ** 24, "fp32 atomics count exactly only below 2^24 valid pixels per scale"
        for k in range(4):
            sums[j, k] = terms[k].sum()
            bound[j, k] = C_TERM * U * mags[k].sum() + (5 + 8 + blocks[j]) * U * np.abs(terms[k]).sum()
        sums[j, 4] = valid.sum()
    return sums, bound


def check_loss_sums(what, got, sums, bound):
    """sums (n,5): counts bit-exact, NaN exactly where the reference is NaN, the rest within the bound; returns worst err / bound"""
    got = np.asarray(got, np.float64)
    nan = np.isnan(sums)
    if not np.array_equal(np.isnan(got), nan):
        raise AssertionError("%s: NaN pattern of the sums differs: kernel %s, reference %s" % (what, np.isnan(got).tolist(), nan.tolist()))
    if not np.array_equal(got[:, 4], sums[:, 4]):
        raise AssertionError("%s: valid counts differ: kernel %s, reference %s" % (what, got[:, 4].tolist(), sums[:, 4].tolist()))
    err = np.where(nan, 0.0, np.abs(got - np.where(nan, 0.0, sums)))
    ratio = np.where(nan | (np.arange(5) == 4), 0.0, err / np.maximum(bound, 1e-300))
    worst = float(ratio.max())
    if worst > 1.0:
        j, k = np.unravel_index(np.argmax(ratio), ratio.shape)
        raise AssertionError("%s: scale %d column %d exceeds the bound by x%.3g (kernel %r, reference %r, bound %.3e)"
                             % (what, j, k, worst, got[j, k], sums[j, k], bound[j, k]))
    return worst


def loss_backward_reference(preds, gt, weights, up, loss_type, counts):
    """d loss / d p per scale: up * w_j / count_j * dl with the kernel's counts.  Returns a list of (cands (k,B,hs,ws) float64 -- the
    values either branch may give --, zero (B,hs,ws) bool -- must be +0 --, ambiguous (B,hs,ws) bool -- more than one candidate)"""
    out = []
    for j, p in enumerate(preds):
        g = downsampled_gt(gt, *p.shape[1:]).astype(np.float64)
        p = p.astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            scale = float(up) * float(weights[j]) / counts[j]
            diff = p - g
            sgn = np.sign(diff)
            amb = np.zeros(g.shape, bool)
            if loss_type == L1:
                cands = [sgn]
            elif loss_type == L1_REL:
                cands = [sgn / g]
            elif loss_type == HUBER:
                cands = [np.where(np.abs(diff) < 1, diff, sgn)]
                amb = np.abs(np.abs(diff) - 1) <= 2 * U * np.abs(diff)            # fl(p - g) may land on either side of 1
                cands.append(np.where(amb, np.where(np.abs(diff) < 1, sgn, diff), cands[0]))
            else:
                e = 1 / g - 1 / p
                inv = 1 / (p * p)
                cands = [np.sign(e) * inv]
                amb = np.abs(e) <= 2 * U * (np.abs(1 / g) + np.abs(1 / p))        # the fp32 e may have either sign or be 0
                for s in (-1.0, 0.0, 1.0):
                    cands.append(np.where(amb, s * inv, cands[0]))
            valid = g != 0
            cands = np.stack([np.where(valid, scale * c, 0.0) for c in cands])
        out.append((cands, ~valid | (counts[j] == 0), amb & valid))
    return out


def check_loss_grad(what, grads, ref):
    """grads [(B,hs,ws) fp32 numpy]: +0 bit for bit where required, within C_GRAD u of some candidate elsewhere (rows with NaN ground
    truth are not checked).  Returns (worst err / bound, ambiguous count)."""
    worst, n_amb = 0.0, 0
    for j, (got, (cands, zero, amb)) in enumerate(zip(grads, ref)):
        got = np.asarray(got, np.float32)
        bad = zero & (got.view(np.uint32) != 0)
        if bad.any():
            i = tuple(int(v) for v in np.argwhere(bad)[0])
            raise AssertionError("%s: scale %d element %s must be +0, kernel %r" % (what, j, i, float(got[i])))
        live = ~zero & np.isfinite(cands).all(0)
        with np.errstate(invalid="ignore"):
            ratio = (np.abs(got.astype(np.float64)[None] - cands) / np.maximum(C_GRAD * U * np.abs(cands), 1e-300)).min(0)
        ratio = np.where(live, np.where(np.isnan(ratio), np.inf, ratio), 0.0)
        n_amb += int(amb.sum())
        if ratio.size and ratio.max() > 1.0:
            i = tuple(int(v) for v in np.unravel_index(np.argmax(ratio), ratio.shape))
            raise AssertionError("%s: scale %d element %s exceeds the bound by x%.3g (kernel %r, reference %s)"
                                 % (what, j, i, float(ratio[i]), float(got[i]), [float(c[i]) for c in cands]))
        worst = max(worst, float(ratio.max()) if ratio.size else 0.0)
    return worst, n_amb


LOSS_DEFECTS = ("other_count", "sign0", "huber_le", "round_index", "inv_g2", "neg_invalid")


def _tree_sum(v, blocks):
    """per block: the 32-lane shuffle butterfly, lane 0 of each warp, the 8 warps in order (fp32).  v (blocks * 256,)"""
    t = v.reshape(blocks, LOSS_THREADS // 32, 32).astype(np.float32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        t = _f32(t + t[..., lane ^ o])
    s = np.zeros(blocks, np.float32)
    for i in range(LOSS_THREADS // 32):
        s = _f32(s + t[:, i, 0])
    return s


def emulate_loss(preds, gt, weights, up, loss_type, variant=None, seed=0):
    """depth_loss_forward_kernel and depth_loss_backward_kernel in fp32 numpy: per-block trees, the blocks of a scale atomically in
    a random order.  Returns (sums (n,5) fp32, [grad (B,hs,ws) fp32])."""
    rng = np.random.RandomState(seed)
    n = len(preds)
    B = gt.shape[0]
    blocks = loss_blocks(B, [p.shape[1:] for p in preds])
    sums = np.zeros((n, 5), np.float32)
    gts = []
    one = np.float32(1)
    for j, p in enumerate(preds):
        g = downsampled_gt(gt, *p.shape[1:], rounded=variant == "round_index").astype(np.float32)
        gts.append(g)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            valid = (g > 0) if variant == "neg_invalid" else (g != 0)
            d = np.abs(_f32(g - p))
            huber = np.where(d <= 1 if variant == "huber_le" else d < 1, _f32(_f32(np.float32(0.5) * d) * d), _f32(d - np.float32(0.5)))
            terms = [d, huber, np.abs(_f32(_f32(one / g) - _f32(one / p))), _f32(d / g), np.ones_like(d)]
        per = np.zeros(blocks[j] * LOSS_THREADS, np.float32)
        for k in range(5):
            per[:] = 0
            per[:g.size] = np.where(valid, terms[k], 0).ravel()
            part = _tree_sum(per, blocks[j])
            for b in rng.permutation(blocks[j]):
                if part[b] != 0:
                    sums[j, k] = _f32(sums[j, k] + part[b])
    grads = []
    for j, p in enumerate(preds):
        g = gts[j]
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            valid = (g > 0) if variant == "neg_invalid" else (g != 0)
            diff = _f32(p - g)
            sgn = np.where(diff > 0, one, np.where(diff < 0, -one, np.float32(1 if variant == "sign0" else 0))).astype(np.float32)
            if loss_type == L1:
                dl = sgn
            elif loss_type == HUBER:
                dl = np.where(np.abs(diff) <= 1 if variant == "huber_le" else np.abs(diff) < 1, diff, sgn)
            elif loss_type == L1_INV:
                e = _f32(_f32(one / g) - _f32(one / p))
                s = np.where(e > 0, one, np.where(e < 0, -one, np.float32(0)))
                dl = _f32(s / _f32((g * g) if variant == "inv_g2" else (p * p)))
            else:
                dl = _f32(sgn / g)
            cnt = sums[(j + 1) % n, 4] if variant == "other_count" else sums[j, 4]
            out = _f32(_f32(_f32(np.float32(up) * np.float32(weights[j])) / cnt) * dl)
        grads.append(np.where(valid, out, np.float32(0)).astype(np.float32))
    return sums, grads


# ------------------------------------------------------------------------------------------------ cases (shared by both tests)
def _t32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))


def _rel(t, yaw=0.0):
    P = np.eye(4)
    c, s = np.cos(yaw), np.sin(yaw)
    P[:3, :3] = [[c, 0, s], [0, 1, 0], [-s, 0, c]]
    P[:3, 3] = t
    return P


def _half_K(h, w, B=1):
    import synth_data as synth
    K = _t32(synth.intrinsics(2 * h, 2 * w))[None].repeat(B, 1, 1)
    K[:, 0:2] /= 2.0
    return K


SWEEP_MIN_DEPTH, SWEEP_MAX_DEPTH = 0.25, 20.0
# name: (B, h, w, D, M, geometry); geometry "moderate": distinct random poses per batch entry, "clip": synthetic clip poses,
# otherwise the measurement cameras relative to the reference camera
SWEEP_CASES = {
    "batch2_w33_D13_M3": (2, 20, 33, 13, 3, "moderate"),
    "w40_D2_M1": (1, 12, 40, 2, 1, "moderate"),
    "w64_D64_M3": (1, 16, 64, 64, 3, "moderate"),
    "smem_max_D256_M8": (1, 6, 40, 256, 8, "moderate"),
    "crossing_borders": (1, 24, 40, 13, 2, [_rel([0.05, 0.02, 1.0], yaw=0.3), _rel([0.1, 0, 0.1])]),
    "forward_motion": (1, 24, 40, 16, 2, [_rel([0.02, 0.01, -0.3]), _rel([0, 0, -0.15])]),
    "zero_baseline": (1, 16, 40, 8, 1, [np.eye(4)]),
    "far_out_of_view": (1, 16, 40, 13, 2, [_rel([2.0, 0.0, 0.0]), _rel([0.0, -3.0, 0.5], yaw=1.2)]),
    "grad_zeros_B2": (2, 16, 33, 13, 2, "moderate"),
    "train_128x128_D64_M2": (1, 128, 128, 64, 2, "clip"),
    "train_128x160_D96_M4": (1, 128, 160, 96, 4, "clip"),
}
CPU_SWEEP_CASES = ("batch2_w33_D13_M3", "w40_D2_M1", "crossing_borders", "forward_motion", "zero_baseline", "far_out_of_view",
                   "grad_zeros_B2")


def sweep_case(name):
    """fp32 CPU tensors of one case: dict f1, f2s (B,h,w,32), g (B,h,w,D), pose1, pose2s, K and the shape"""
    from tests.sweep_reference import moderate_geometry, rigid
    B, h, w, D, M, geo = SWEEP_CASES[name]
    seed = sum(map(ord, name))
    if geo == "moderate":
        pose1, pose2s, K = moderate_geometry(B, h, w, M, seed)
    elif geo == "clip":
        import synth_data as synth
        pose1 = _t32(np.stack([synth.camera_pose(M)] * B))
        pose2s = [_t32(np.stack([synth.camera_pose(M - k)] * B)) for k in range(1, M + 1)]
        K = _half_K(h, w, B)
    else:
        pose1 = torch.eye(4)[None] if name == "zero_baseline" else _t32(rigid(np.random.RandomState(seed), 0.5, 0.3))[None]
        pose2s = [pose1 @ _t32(r)[None] for r in geo]
        K = _half_K(h, w)
    gen = torch.Generator().manual_seed(seed)
    f1 = torch.randn(B, h, w, 32, generator=gen) * 2
    f2s = [torch.randn(B, h, w, 32, generator=gen) * 2 for _ in range(M)]
    g = torch.randn(B, h, w, D, generator=gen)
    if name == "grad_zeros_B2":          # exact zeros: single samples, whole planes, and every plane of some pixels
        g = torch.where(torch.rand(B, h, w, D, generator=gen) < 0.4, torch.zeros_like(g), g)
        g[..., 3] = 0
        g[:, 2:5, 7:30] = 0
    return dict(name=name, B=B, h=h, w=w, D=D, M=M, pose1=pose1, pose2s=pose2s, K=K, f1=f1, f2s=f2s, g=g)


def sweep_case_reference(c, dev="cpu"):
    to = lambda t: t.to(dev)
    return sweep_backward_reference(to(c["f1"]), [to(f) for f in c["f2s"]], to(c["pose1"]), [to(p) for p in c["pose2s"]], to(c["K"]),
                                    SWEEP_MIN_DEPTH, SWEEP_MAX_DEPTH, c["D"], to(c["g"]))


def sweep_case_emulation(c, variant=None, buffers=None, seed=0):
    return emulate_sweep_backward(c["f1"].numpy(), [f.numpy() for f in c["f2s"]], c["pose1"].numpy(), [p.numpy() for p in c["pose2s"]],
                                  c["K"].numpy(), SWEEP_MIN_DEPTH, SWEEP_MAX_DEPTH, c["D"], c["g"].numpy(), variant, seed, buffers)


# (B, h, w, C): hw crosses each instantiation boundary of the kernel (PPW = 2 up to 16 positions, 8 up to 64, 16 up to 128)
LSTM_CASES = {
    "hw1_C32_B1": (1, 1, 1, 32), "hw1_C512_B4": (4, 1, 1, 512),
    "hw16_C32_B4": (4, 4, 4, 32), "hw16_C512_B1": (1, 4, 4, 512),
    "hw17_C32_B1": (1, 1, 17, 32), "hw17_C512_B4": (4, 17, 1, 512),
    "hw64_C32_B4": (4, 8, 8, 32), "hw64_C512_B1": (1, 8, 8, 512),
    "hw65_C32_B1": (1, 5, 13, 32), "hw65_C512_B4": (4, 13, 5, 512),
    "hw80_C32_B4": (4, 8, 10, 32), "hw80_C512_B1": (1, 8, 10, 512),
    "hw128_C32_B1": (1, 8, 16, 32), "hw128_C512_B4": (4, 16, 8, 512),
}


def lstm_instantiation(hw):
    ppw = (hw + 7) // 8
    return 2 if ppw <= 2 else (8 if ppw <= 8 else 16)


def lstm_case(name):
    """fp32 (gates (B,h,w,4C), c_in, grad_h, grad_c) with, in every batch entry: channel 0's g pre-activation constant over the
    positions; channel 1's f c + i celu(n) constant (i = sigmoid(-100) = 0 in fp32, f and c constant); channels 2-5 saturated
    sigmoids (|a| = 20 +- 0.5) on the i, f, o gates"""
    B, h, w, C = LSTM_CASES[name]
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    n = h * w
    gates = torch.randn(B, n, 4 * C, generator=gen) * 1.5
    c_in = torch.randn(B, n, C, generator=gen)
    gates[:, :, 3 * C + 0] = 0.7
    gates[:, :, 0 * C + 1] = -100.0
    gates[:, :, 1 * C + 1] = 0.3
    c_in[:, :, 1] = -1.25
    for ch, sgn in ((2, 1), (3, -1), (4, 1), (5, -1)):
        for k in range(3):
            gates[:, :, k * C + ch] = sgn * (20.0 + torch.rand(B, n, generator=gen) - 0.5) * (1 if k != 1 else -1)
    grad_h = torch.randn(B, n, C, generator=gen)
    grad_c = torch.randn(B, n, C, generator=gen)
    sh = lambda t, c: t.reshape(B, h, w, c).contiguous()
    return sh(gates, 4 * C), sh(c_in, C), sh(grad_h, C), sh(grad_c, C)


def lstm_reach(gates, C):
    """the edges a case reaches, from its inputs"""
    B, h, w, _ = gates.shape
    g = gates.reshape(B, h * w, 4 * C)
    gg = g[..., 3 * C:]
    const_g = int(((gg.amax(1) - gg.amin(1)) == 0).sum())
    const_cp = int(((g[..., :C] <= -88).all(1) & ((g[..., C:2 * C].amax(1) - g[..., C:2 * C].amin(1)) == 0)).sum())
    sat = int((g[..., :3 * C].abs() >= 19).sum())
    return dict(const_g=const_g, const_cp=const_cp, saturated=sat)


# name: (B, H, W, scale sizes, weights, upstream); the ground truth has zeros and negative values, and predictions equal to it or
# exactly 1 away at chosen pixels
LOSS_CASES = {
    "one_scale_B2_20x20": (2, 20, 20, [(20, 20)], [1.0], 1.0),
    "five_scales_odd_ratios": (2, 50, 70, [(50, 70), (25, 35), (13, 17), (7, 9), (60, 90)], [1.0, 0.5, 0.0, 2.0, 0.25], 3.0),
    "eight_scales_one_empty": (3, 30, 40, [(30, 40), (15, 20), (11, 13), (8, 10), (5, 7), (3, 3), (2, 2), (1, 1)],
                               [1, 1, 1, 1, 1, 1, 1, 1.5], -0.5),
    "nan_groundtruth": (2, 24, 24, [(24, 24), (12, 12), (5, 5)], [1.0, 1.0, 1.0], 1.0),
    "train_bench_B4_256": (4, 256, 256, [(16, 16), (32, 32), (64, 64), (128, 128), (256, 256)], [1, 1, 1, 1, 1], 1.0),
}
CPU_LOSS_CASES = ("one_scale_B2_20x20", "five_scales_odd_ratios", "eight_scales_one_empty", "nan_groundtruth")


def loss_case(name):
    """fp32 numpy (preds [(B,hs,ws)], gt (B,H,W), weights, upstream)"""
    B, H, W, sizes, weights, up = LOSS_CASES[name]
    rng = np.random.RandomState(sum(map(ord, name)))
    gt = (rng.rand(B, H, W) * 5 + 0.3).astype(np.float32)
    gt = np.round(gt * 8) / 8                                    # dyadic: p = g + 1 is exact
    gt[rng.rand(B, H, W) < 0.1] = 0
    gt[rng.rand(B, H, W) < 0.05] *= -1
    gt = gt.astype(np.float32)
    if name == "eight_scales_one_empty":
        gt[:, 0, 0] = 0                                          # the 1x1 scale reads only (0, 0): no valid pixel
    if name == "nan_groundtruth":
        gt[0, 6, 6] = np.nan                                     # read by the 24x24 and 12x12 scales, not by 5x5
    preds = []
    for hs, ws in sizes:
        g = downsampled_gt(gt, hs, ws)
        p = (rng.rand(B, hs, ws) * 5 + 0.3).astype(np.float32)
        r = rng.rand(B, hs, ws)
        p = np.where(r < 0.1, g, np.where(r < 0.2, g + np.float32(1), np.where(r < 0.25, g - np.float32(1), p)))
        p = np.where(np.isfinite(p) & (p != 0), p, np.float32(1.5)).astype(np.float32)
        preds.append(p)
    return preds, gt, weights, up


def loss_reach(preds, gt):
    """the edges a case reaches, from its inputs"""
    B, H, W = gt.shape
    r = dict(scales=len(preds), straddle=0, non_integer=0, upsampled=0, empty=0, neg=0, zeros=0, equal=0, one_apart=0, nan=0)
    for p in preds:
        hs, ws = p.shape[1:]
        g = downsampled_gt(gt, hs, ws)
        r["straddle"] += (B * hs * ws) % LOSS_THREADS != 0
        r["non_integer"] += (H % hs != 0) or (W % ws != 0)
        r["upsampled"] += hs > H or ws > W
        r["empty"] += int(not (g != 0).any())
        r["neg"] += int((g < 0).sum())
        r["zeros"] += int((g == 0).sum())
        with np.errstate(invalid="ignore"):
            r["equal"] += int(((p == g) & (g != 0)).sum())
            r["one_apart"] += int((np.abs(p.astype(np.float64) - g) == 1).sum())
        r["nan"] += int(np.isnan(g).sum())
    return r
