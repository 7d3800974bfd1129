"""fp64 reference of the plane sweeps (plane_sweep_tc_kernel at 1 and 3 terms, plane_sweep_c32_kernel, plane_sweep_generic_kernel)
computed from the operands each kernel multiplies, with a per-sample error bound.  Shared by the GPU tests
(tests/test_sweep_reference.py) and by the CPU test that checks the bound against an emulation of the kernels' arithmetic and
against planted defects (tests/test_sweep_reference_bound.py); nothing here needs a GPU.

Semantics: oracle/dvmvs_oracle.py calculate_cost_volume_by_warping / cost_volume_fusion.  For every sample (b, v, u, plane d,
frame m) the position (xs, ys) = (w-1)/w * (q0, q1) / (q2 + 1e-8), q = G (u, v, 1) + Kt / depth_d, G = K R K^-1, Kt = K t, is
evaluated in fp64 from the fp32 poses and K, at the fp32 plane depths both kernels use.  The cost is linear in the four taps, so
per frame it is sum_t w_t s_t with s_t the dot product of the reference pixel's features with tap t's (0 outside the image),
divided by C; the frames are summed in order and divided by M.  s_t is formed from the operands of each form:

    "tc1"     hi2 . fp16_rn(hi1 * 2^-5)            (the consumer pre-scales the reference tile in fp16)
    "tc3"     (hi2 . hi1 + lo2 . hi1 + hi2 . lo1) / 32   (no lo . lo)
    "gather"  f2 . f1 / C                          (fp32 features)

Error bound per sample, in the units of the output:

    accumulation  C_ACC * u * n * P_t per tap, P_t = sum |products|; n = terms * 2 k16 steps on the band path, one step per
                  channel on the gather and direct paths.  A tensor-core sample may take either the band or the direct path
                  (decided per chunk by the planner), and the two differ: the direct path multiplies hi1 / 32 (not the fp16
                  pre-scaled operand) at 1 term and includes lo . lo at 3 terms, and at 1 term the band path stores S in fp16
                  (H16 * |s| + H16_TINY).  The tap bound takes the larger of the two paths' terms, accumulation and rounding
                  differences separately (>= the larger of the two paths' bounds).
    blend         C_BLEND * u * sum_t w_t |s_t| (four fmaf, the frame sum and 1/M).
    position      the fp32 position is off by delta = C_POS * u * (sx * (Q0 + |x| Q2) / |den| + w) in x (same in y), Q the
                  running magnitudes of q (|K| |R| |K^-1| and |K| |t| from |pose2^-1| |pose1|, times |u|, |v|, 1 / depth).
                  Charged delta_x * Lx + delta_y * Ly + delta_x * delta_y * |cross term|, L the largest tap difference over
                  the cells the delta box touches.  Where delta >= 1 px (|den| near 0) the sample is ill-conditioned: the
                  frame's cost is bounded by Cauchy-Schwarz (|f1| * max |f2|) and the sample is counted.
"""
import math

import numpy as np
import torch

from tests.tc_reference import C_ACC, H16, H16_TINY, U, check

C_POS = 16.0            # units of u of the position magnitude: >= 8x the worst measured by the fp32 emulation of the kernels'
                        # position arithmetic (tests/test_sweep_reference_bound.py prints it)
C_BLEND = 16.0          # units of u of sum_t w_t |s_t|: four fmaf, the frame sum (M <= 8 additions) and 1/M
TILE_W, TILE_H, BAND_ROWS, RUN = 16, 4, 64, 32      # plane_sweep_tc_kernel's tile, band row slots and TMA runs (sweep_tc.cu)

FORMS = {            # n_band: k16 steps of the band path (None: no band path); store16: S stored in fp16
    "tc1": dict(n_band=2, store16=True),
    "tc3": dict(n_band=6, store16=False),
    "gather": dict(n_band=None, store16=False),
}


def plane_depths(min_depth, max_depth, D):
    """the fp32 plane depths both kernels use: 1 / (inv_base + d * inv_step) in double from the fp32 depth range, then fp32"""
    mn, mx = float(np.float32(min_depth)), float(np.float32(max_depth))
    inv_base, inv_step = 1.0 / mx, (1.0 / mn - 1.0 / mx) / (D - 1)
    return torch.tensor([float(np.float32(1.0 / (inv_base + d * inv_step))) for d in range(D)], dtype=torch.float64)


def frame_geometry(pose1, pose2, K):
    """fp64 G = K R K^-1 (B,3,3), Kt (B,3) and their running magnitudes from fp32 poses (B,4,4) and K (B,3,3)"""
    p1, p2, K = pose1.double(), pose2.double(), K.double()
    inv2 = torch.linalg.inv(p2)
    E = inv2 @ p1
    Kinv = torch.linalg.inv(K)
    G = K @ E[:, :3, :3] @ Kinv
    Kt = (K @ E[:, :3, 3:])[..., 0]
    Emag = inv2.abs() @ p1.abs()
    Gmag = K.abs() @ Emag[:, :3, :3] @ Kinv.abs()
    Ktmag = (K.abs() @ Emag[:, :3, 3:])[..., 0]
    return G, Kt, Gmag, Ktmag


def positions(pose1, pose2, K, depths, h, w, d_sel=None):
    """fp64 sample positions of one frame: dict of (B, D', h, w) tensors xs, ys, den, delta_x, delta_y (d_sel: plane indices)"""
    dev = pose1.device
    G, Kt, Gmag, Ktmag = frame_geometry(pose1, pose2, K)
    dep = depths.to(dev) if d_sel is None else depths.to(dev)[d_sel]
    v, u = torch.meshgrid(torch.arange(h, dtype=torch.float64, device=dev), torch.arange(w, dtype=torch.float64, device=dev), indexing="ij")
    base = G[:, :, 0, None, None] * u + G[:, :, 1, None, None] * v + G[:, :, 2, None, None]            # (B,3,h,w)
    bmag = Gmag[:, :, 0, None, None] * u + Gmag[:, :, 1, None, None] * v + Gmag[:, :, 2, None, None]
    q = base[:, None] + Kt[:, None, :, None, None] / dep[None, :, None, None, None]                     # (B,D,3,h,w)
    Q = bmag[:, None] + Ktmag[:, None, :, None, None] / dep[None, :, None, None, None]
    den = q[:, :, 2] + 1e-8
    sx, sy = (w - 1) / w, (h - 1) / h
    x, y = q[:, :, 0] / den, q[:, :, 1] / den
    dx = C_POS * U * (sx * (Q[:, :, 0] + x.abs() * Q[:, :, 2]) / den.abs() + w)
    dy = C_POS * U * (sy * (Q[:, :, 1] + y.abs() * Q[:, :, 2]) / den.abs() + h)
    return dict(xs=x * sx, ys=y * sy, den=den, delta_x=dx, delta_y=dy)


def form_operands(form, f1=None, f2s=None, planes1=None, planes2=None):
    """(ref operands, meas operands, alt ref operands, alt meas operands, scale) as float64 (B,h,w,C) lists; s = scale * sum_i
    ref[i] . meas[i]; alt: the direct path's product list (None: no second path).  planes: (hi, lo) fp16 tensors"""
    if form == "gather":
        return [f1.double()], [[f.double()] for f in f2s], None, None, 1.0 / f1.shape[-1]
    hi1, lo1 = planes1[0].double(), planes1[1].double() if planes1[1] is not None else None
    meas = [(p[0].double(), p[1].double() if p[1] is not None else None) for p in planes2]
    if form == "tc1":
        r = (planes1[0].float() * 2.0 ** -5).half().double()
        return [r], [[hi] for hi, _ in meas], [hi1 / 32], [[hi] for hi, _ in meas], 1.0
    return ([hi1, hi1, lo1], [[hi, lo, hi] for hi, lo in meas], [hi1, hi1, lo1, lo1], [[hi, lo, hi, lo] for hi, lo in meas], 1.0 / 32)


class SweepRef:
    """y (B,h,w,D): reference; bound: per-sample bound on |kernel - y|; acc: the accumulation part of the bound over C_ACC (the
    u * n * S the measured constant is expressed in); other: the rest of the bound; wabs: sum_m sum_t w_t |s_t| / M; n_ill:
    ill-conditioned samples; smax: the largest |s| of any tap (dot mode; at 1 term the kernel stores it in fp16)"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _patch_index(xs, ys, h, w, npix_b, b_off):
    """flat indices (.., 16) of the 4 x 4 pixels around the cell of (xs, ys) (rows y0-1..y0+2, cols x0-1..x0+2), the zero row
    (index B*h*w) outside the image"""
    x0, y0 = torch.floor(xs).long(), torch.floor(ys).long()
    o = torch.arange(-1, 3, device=xs.device)
    X = x0[..., None, None] + o[None, :]                   # (..,1,4) cols
    Y = y0[..., None, None] + o[:, None]                   # (..,4,1) rows
    inside = (X >= 0) & (X < w) & (Y >= 0) & (Y < h)
    idx = b_off[..., None, None] + Y.clamp(0, h - 1) * w + X.clamp(0, w - 1)
    return torch.where(inside, idx, torch.full_like(idx, npix_b)).reshape(*xs.shape, 16), x0, y0


def sweep_reference(form, pose1, pose2s, K, min_depth, max_depth, D, f1=None, f2s=None, planes1=None, planes2=None,
                    dot=True, plane_chunk=None):
    """fp64 reference and bound of one sweep.  pose1 (B,4,4), pose2s [M x (B,4,4)], K (B,3,3) fp32; f1 / f2s fp32 (B,h,w,C)
    for the gather form; planes1 / planes2 (hi, lo) fp16 (B,h,w,32) for the tensor-core forms.  All on one device."""
    ref_ops, meas_ops, alt_ref, alt_meas, scale = form_operands(form, f1, f2s, planes1, planes2)
    B, h, w, C = ref_ops[0].shape
    M = len(pose2s)
    dev = ref_ops[0].device
    cfg = FORMS[form]
    depths = plane_depths(min_depth, max_depth, D)
    if plane_chunk is None:          # at most 2^25 gathered operand elements at a time
        plane_chunk = max(1, min(D, (1 << 25) // (B * h * w * 16 * C)))
    y = torch.zeros(B, D, h, w, dtype=torch.float64, device=dev)
    acc_b, oth_b, wabs = torch.zeros_like(y), torch.zeros_like(y), torch.zeros_like(y)
    n_ill, smax = 0, 0.0
    b_off = (torch.arange(B, device=dev) * (h * w)).view(B, 1, 1, 1)
    zero = lambda t: torch.cat([t.reshape(B * h * w, -1), t.new_zeros(1, t.shape[-1])])
    ref_norm = [r.norm(dim=-1) for r in ref_ops]                    # (B,h,w) for the Cauchy-Schwarz bound
    for m in range(M):
        mflat = [zero(t) for t in meas_ops[m]]
        aflat = [zero(t) for t in alt_meas[m]] if alt_meas is not None else None
        cs = sum(rn * t.norm(dim=-1).amax() for rn, t in zip(ref_norm, meas_ops[m])) * scale * (1 + H16)     # |s| <= cs
        for d0 in range(0, D, plane_chunk):
            ds = torch.arange(d0, min(D, d0 + plane_chunk), device=dev)
            P = positions(pose1, pose2s[m], K, depths, h, w, ds.cpu())
            xs, ys = P["xs"], P["ys"]
            ill = ~(torch.isfinite(xs) & torch.isfinite(ys) & (P["delta_x"] < 1) & (P["delta_y"] < 1))
            xs_c = torch.nan_to_num(xs, nan=-4.0).clamp(-4.0, w + 3.0)
            ys_c = torch.nan_to_num(ys, nan=-4.0).clamp(-4.0, h + 3.0)
            idx, x0, y0 = _patch_index(xs_c, ys_c, h, w, B * h * w, b_off)          # (B,d,h,w,16)
            fx, fy = xs_c - x0, ys_c - y0
            wt = torch.stack([(1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy], -1)      # taps 00, 01, 10, 11
            inner = [5, 6, 9, 10]

            if dot:
                def dots(refs, meas, absval=False):
                    s = 0
                    for r, mf in zip(refs, meas):
                        g = mf[idx]                                           # (B,d,h,w,16,C)
                        rr = r[:, None, :, :, None, :]
                        s = s + ((g.abs() * rr.abs()) if absval else (g * rr)).sum(-1)
                    return s * scale
                s = dots(ref_ops, mflat)                                      # (B,d,h,w,16)
                smax = max(smax, float(s.abs().max()))
                Pp = dots(ref_ops, mflat, True)
                if cfg["n_band"] is None:
                    tap_acc = C_ACC * U * C * Pp / C_ACC
                    tap_oth = torch.zeros_like(s)
                else:
                    band_acc = U * cfg["n_band"] * Pp
                    band_oth = (H16 * (s.abs() + C_ACC * band_acc) + H16_TINY) if cfg["store16"] else torch.zeros_like(s)
                    alt = dots(alt_ref, aflat)
                    dir_acc = U * C * dots(alt_ref, aflat, True)
                    dir_oth = (alt - s).abs()
                    # either path, part by part: the accumulation of the direct path (one step per channel) and the fp16 store
                    # or the lo . lo / pre-scale difference, whichever is larger
                    tap_acc = torch.maximum(dir_acc, band_acc)
                    tap_oth = torch.maximum(dir_oth, band_oth)
                val = (wt * s[..., inner]).sum(-1)
                sabs = (wt * s[..., inner].abs()).sum(-1)
                accm = (wt * tap_acc[..., inner]).sum(-1)
                othm = (wt * tap_oth[..., inner]).sum(-1)
                pat = s.reshape(*s.shape[:-1], 4, 4)
                dxm = (pat[..., :, 1:] - pat[..., :, :-1]).abs()
                dym = (pat[..., 1:, :] - pat[..., :-1, :]).abs()
                crm = (pat[..., 1:, 1:] - pat[..., 1:, :-1] - pat[..., :-1, 1:] + pat[..., :-1, :-1]).abs()
                ill_b = val.abs() + cs[:, None]
            else:
                f1d = ref_ops[0]
                g = mflat[0][idx]                                             # (B,d,h,w,16,C)
                warped = (wt[..., None] * g[..., inner, :]).sum(-2)
                f1b = f1d[:, None]
                val = (f1b - warped).abs().sum(-1)
                mag = (f1b.abs() + (wt[..., None] * g[..., inner, :].abs()).sum(-2)).sum(-1)
                accm, othm, sabs = U * C * mag, torch.zeros_like(val), val
                pat = g.reshape(*g.shape[:-2], 4, 4, C)
                dxm = (pat[..., :, 1:, :] - pat[..., :, :-1, :]).abs().sum(-1)
                dym = (pat[..., 1:, :, :] - pat[..., :-1, :, :]).abs().sum(-1)
                crm = (pat[..., 1:, 1:, :] - pat[..., 1:, :-1, :] - pat[..., :-1, 1:, :] + pat[..., :-1, :-1, :]).abs().sum(-1)
                ill_b = val.abs() + f1d.abs().sum(-1)[:, None] + mflat[0].abs().sum(-1).amax()
            # cells of the 4 x 4 patch the delta box touches: cell (i, j) has its top-left pixel at (y0 - 1 + i, x0 - 1 + j)
            dx_, dy_ = P["delta_x"].clamp(max=1.0), P["delta_y"].clamp(max=1.0)
            cx_lo, cx_hi = torch.floor(xs_c - dx_) - x0, torch.floor(xs_c + dx_) - x0        # in {-1, 0, 1}
            cy_lo, cy_hi = torch.floor(ys_c - dy_) - y0, torch.floor(ys_c + dy_) - y0
            o = torch.arange(-1, 2, device=dev, dtype=torch.float64)
            col = (o >= cx_lo[..., None]) & (o <= cx_hi[..., None])                          # (..,3)
            row = (o >= cy_lo[..., None]) & (o <= cy_hi[..., None])
            cell = row[..., :, None] & col[..., None, :]                                     # (..,3,3)
            Lx = (torch.maximum(dxm[..., :3, :], dxm[..., 1:, :]) * cell).amax((-1, -2))
            Ly = (torch.maximum(dym[..., :, :3], dym[..., :, 1:]) * cell).amax((-1, -2))
            Lc = (crm * cell).amax((-1, -2))
            pos = dx_ * Lx + dy_ * Ly + dx_ * dy_ * Lc
            crossing = cell.sum((-1, -2)) > 1
            if dot:      # the kernel may blend the taps of a neighbouring cell: charge the largest tap bound of the patch
                accm = torch.where(crossing, torch.maximum(accm, tap_acc.amax(-1)), accm)
                othm = torch.where(crossing, torch.maximum(othm, tap_oth.amax(-1)), othm)
            sl = slice(d0, d0 + len(ds))
            fin = ~ill
            val = torch.where(torch.isfinite(xs) & torch.isfinite(ys), val, torch.zeros_like(val))     # non-finite: contributes 0
            y[:, sl] += val
            wabs[:, sl] += torch.where(fin, sabs, torch.zeros_like(val))
            acc_b[:, sl] += torch.where(fin, accm, torch.zeros_like(val))
            oth_b[:, sl] += torch.where(fin, othm + pos, ill_b)
            n_ill += int(ill.sum())
    y, acc_b, oth_b, wabs = (t.permute(0, 2, 3, 1) / M for t in (y, acc_b, oth_b, wabs))
    oth_b = oth_b + C_BLEND * U * wabs
    return SweepRef(y=y, bound=C_ACC * acc_b + oth_b, acc=acc_b, other=oth_b, wabs=wabs, n_ill=n_ill, smax=smax, form=form,
                    depths=depths)


def check_sweep(what, got, ref, describe=None, report=None):
    """|got - ref.y| <= ref.bound for every sample (got: (B,h,w,D) kernel output), non-finite output always fails.  Returns
    (worst err / bound, worst err / (u n S) not explained by the other terms of the bound, median bound / sum w|s|); a failure
    names the sample (b, v, u, d) and, through describe(idx), its tile, chunk geometry and path class."""
    got = got.double().to(ref.y.device)
    err = (got - ref.y).abs()
    resid = (err - ref.other).clamp_min(0)
    acc = float((resid / ref.acc.clamp_min(1e-300)).max()) if err.numel() else 0.0
    nz = ref.wabs > 0
    tight = float((ref.bound[nz] / ref.wabs[nz]).median()) if bool(nz.any()) else 0.0
    try:
        worst, _ = check(what, got, ref.y, ref.bound)
    except AssertionError as e:
        finite = torch.isfinite(got)
        ratio = torch.where(finite, err / ref.bound.clamp_min(1e-300), torch.full_like(err, math.inf))
        idx = tuple(int(i) for i in torch.nonzero(ratio == ratio.max())[0])
        msg = "%s; sample (b, v, u, d) = %s: kernel %r, reference %r, bound %.3e" % (e, idx, float(got[idx]), float(ref.y[idx]),
                                                                                  float(ref.bound[idx]))
        raise AssertionError(msg + ("; " + describe(idx) if describe else "")) from None
    if report is not None:
        report.append((what, worst, acc, tight))
    return worst, acc, tight


# ------------------------------------------------------------------------------------------------ fp32 emulation of the kernels
def _f32(x):
    return np.asarray(x, dtype=np.float32)


def fmaf(a, b, c):
    """fmaf evaluated in float64 (exact product of two fp32), then rounded to fp32"""
    f64 = lambda x: np.asarray(x, dtype=np.float64)
    return _f32(f64(a) * f64(b) + f64(c))


def emulate_matrices(pose1, pose2, K):
    """sweep_matrices / st_matrices (common.cuh): double inverses rounded to fp32, fmaf chains.  numpy fp32 (B,4,4),(B,4,4),(B,3,3)
    -> G (B,3,3), Kt (B,3) fp32"""
    inv2 = _f32(np.linalg.inv(pose2.astype(np.float64)))
    Kinv = _f32(np.linalg.inv(K.astype(np.float64)))

    def mul(a, b):
        n = a.shape[-1]
        o = np.zeros(a.shape[:-1] + (b.shape[-1],), np.float32)
        for i in range(a.shape[-2]):
            for j in range(b.shape[-1]):
                s = np.zeros(a.shape[0], np.float32)
                for k in range(n):
                    s = fmaf(a[:, i, k], b[:, k, j], s)
                o[:, i, j] = s
        return o

    E = mul(inv2, pose1)
    R, t = E[:, :3, :3].copy(), E[:, :3, 3]
    G = mul(mul(K, R), Kinv)
    Kt = np.stack([fmaf(K[:, i, 2], t[:, 2], fmaf(K[:, i, 1], t[:, 1], _f32(K[:, i, 0] * t[:, 0]))) for i in range(3)], -1)
    return G, Kt


def emulate_positions(pose1, pose2, K, depths, h, w, variant="st"):
    """fp32 positions (B,D,h,w) as the kernels compute them: "st" = st_position / sweep_phase_a (fmaf chains, __frcp_rn, one
    (w-1)/w scale), "generic" = plane_sweep_generic_kernel's sweep_sample_pos"""
    G, Kt = emulate_matrices(pose1, pose2, K)
    dep = _f32(np.asarray(depths))
    kd = _f32(Kt[:, None, :] / dep[None, :, None])                           # (B,D,3)
    v, u = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    q = []
    for k in range(3):
        base = fmaf(G[:, k, 0, None, None], u, fmaf(G[:, k, 1, None, None], v, G[:, k, 2, None, None]))      # (B,h,w)
        q.append(_f32(base[:, None] + kd[:, :, k, None, None]))
    den = _f32(q[2] + np.float32(1e-8))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if variant == "st":
            r = _f32(1.0 / den.astype(np.float64))
            sx, sy = np.float32(w - 1) / np.float32(w), np.float32(h - 1) / np.float32(h)
            return _f32(_f32(q[0] * r) * sx), _f32(_f32(q[1] * r) * sy)
        wn, hn = np.float32(w * 0.5), np.float32(h * 0.5)
        x, y = _f32(q[0] / den), _f32(q[1] / den)
        gx, gy = _f32(_f32(x - wn) / wn), _f32(_f32(y - hn) / hn)
        return (_f32(_f32(_f32(gx + np.float32(1)) * np.float32(0.5)) * np.float32(w - 1)),
                _f32(_f32(_f32(gy + np.float32(1)) * np.float32(0.5)) * np.float32(h - 1)))


# ------------------------------------------------------------------------------------------------ plane_sweep_tc's tile plan
def tile_boxes(pose1, pose2, K, depths, h, w, slack=0.0):
    """per (b, tile, plane) of one frame, from the fp64 geometry: the planner's box {x_lo, x_hi, y_lo, y_hi} of the tile's four
    corners (positions clamped to [-1, w] x [-1, h]; slack widens (> 0) or narrows (< 0) it by that many pixels) and whether the
    denominator changes sign over the tile (clear of zero by 1e-3 of its magnitude).  Returns numpy arrays (B, ty, tx, D)."""
    tx, ty = (w + TILE_W - 1) // TILE_W, (h + TILE_H - 1) // TILE_H
    G, Kt, _, _ = frame_geometry(pose1, pose2, K)
    G, Kt = G.cpu().numpy(), Kt.cpu().numpy()
    dep = depths.cpu().numpy()
    u0 = np.arange(tx) * TILE_W
    v0 = np.arange(ty) * TILE_H
    cu = np.stack([u0, np.minimum(u0 + TILE_W, w) - 1])           # (2, tx) corner columns
    cv = np.stack([v0, np.minimum(v0 + TILE_H, h) - 1])           # (2, ty)
    U_ = cu[None, :, None, :] + 0 * cv[:, None, :, None]          # (2cv,2cu,ty,tx)
    V_ = cv[:, None, :, None] + 0 * cu[None, :, None, :]
    q = np.einsum("bij,jcdyx->bicdyx", G, np.stack([U_, V_, np.ones_like(U_)]).astype(np.float64))      # (B,3,2,2,ty,tx)
    q = q[..., None] + (Kt[:, :, None, None, None, None, None] / dep)           # (B,3,2,2,ty,tx,D)
    den = q[:, 2] + 1e-8
    with np.errstate(divide="ignore", invalid="ignore"):
        xs = np.clip(np.nan_to_num(q[:, 0] / den * ((w - 1) / w), nan=-1.0), -1.0, w)
        ys = np.clip(np.nan_to_num(q[:, 1] / den * ((h - 1) / h), nan=-1.0), -1.0, h)
    xs, ys, den = (a.reshape(a.shape[0], 4, *a.shape[3:]) for a in (xs, ys, den))     # (B,4,ty,tx,D)
    scale = np.abs(den).max(1)
    pos, neg = (den > 1e-3 * scale[:, None]).sum(1), (den < -1e-3 * scale[:, None]).sum(1)
    sign_change = (pos > 0) & (neg > 0)
    box = np.stack([np.floor(xs.min(1) - 1e-3 - slack), np.floor(xs.max(1) + 1e-3 + slack) + 1,
                    np.floor(ys.min(1) - 1e-3 - slack), np.floor(ys.max(1) + 1e-3 + slack) + 1], -1).astype(np.int64)
    return box, sign_change, (pos == 4) | (neg == 4), neg == 4


def plan_tile(boxes, degenerate, D, M, qcap, est):
    """plane_sweep_tc's chunk planner on one tile (st_plan_tile), on given per-(frame, plane) boxes: boxes [M][D] of (xl, xh,
    yl, yh), degenerate [M][D] (direct path for the plane), est[m] = planes per chunk of the first guess.  Returns (chunks as
    (m, d0, nd, band), replanned, stuck frames)"""
    n = list(est)
    stuck = [False] * M
    replanned = False
    while True:
        chunks, fail = [], [False] * M
        for m in range(M):
            for d0 in range(0, D, n[m]):
                nd = min(n[m], D - d0)
                bx = boxes[m][d0:d0 + nd]
                deg = bool(degenerate[m][d0:d0 + nd].any())
                fits = False
                if not deg:
                    ylo, yhi = int(bx[:, 2].min()), int(bx[:, 3].max())
                    total = 0
                    if yhi - ylo + 1 <= BAND_ROWS:
                        for yy in range(ylo, yhi + 1):
                            sel = (bx[:, 2] <= yy) & (bx[:, 3] >= yy)
                            if sel.any():
                                total += (int(bx[sel, 1].max()) - int(bx[sel, 0].min()) + RUN) // RUN * RUN
                        fits = 0 < total <= qcap
                chunks.append((m, d0, nd, fits))
                if not fits and not deg and not stuck[m] and nd > 1:
                    fail[m] = True
        if not any(fail):
            return chunks, replanned, stuck
        replanned = True
        for m in range(M):
            if not fail[m]:
                continue
            n_new = max(1, (n[m] * 3) >> 2)
            total = sum((D + (n_new if j == m else n[j]) - 1) // (n_new if j == m else n[j]) for j in range(M))
            if n_new < n[m] and total <= 32:
                n[m] = n_new
            else:
                stuck[m] = True


def first_guess(pose1, pose2, K, depths, h, w, qcap, D, M):
    """planes per chunk of the planner's first guess (st_band_estimate), per (b, ty, tx), from the fp64 tile-centre motion"""
    tx, ty = (w + TILE_W - 1) // TILE_W, (h + TILE_H - 1) // TILE_H
    G, Kt, _, _ = frame_geometry(pose1, pose2, K)
    G, Kt = G.cpu().numpy(), Kt.cpu().numpy()
    dep = depths.cpu().numpy()[[0, D - 1]]
    u0, v0 = np.arange(tx) * TILE_W, np.arange(ty) * TILE_H
    uc = u0 + 0.5 * (np.minimum(TILE_W, w - u0) - 1)
    vc = v0 + 0.5 * (np.minimum(TILE_H, h - v0) - 1)
    p = np.stack(np.broadcast_arrays(uc[None, :], vc[:, None], np.ones((ty, tx))))        # (3,ty,tx)
    q = np.einsum("bij,jyx->biyx", G, p)[..., None] + Kt[:, :, None, None, None] / dep        # (B,3,ty,tx,2)
    with np.errstate(divide="ignore", invalid="ignore"):
        xs = np.clip(np.nan_to_num(q[:, 0] / (q[:, 2] + 1e-8) * ((w - 1) / w), nan=-1.0), -1.0, w)
        ys = np.clip(np.nan_to_num(q[:, 1] / (q[:, 2] + 1e-8) * ((h - 1) / h), nan=-1.0), -1.0, h)
    ddx = np.abs(xs[..., 1] - xs[..., 0]) / (D - 1)
    ddy = np.abs(ys[..., 1] - ys[..., 0]) / (D - 1)
    budget = max(1, 32 // M)
    out = np.zeros(ddx.shape, np.int64)
    for idx in np.ndindex(ddx.shape):
        dx, dy = ddx[idx], ddy[idx]
        nch = min(budget, 32)
        for j in range(32):
            nt = j + 1
            n_try = (D + nt - 1) // nt
            rows = (TILE_H + 2) + dy * n_try
            ppr = min(n_try, (TILE_H + 2) / max(dy, 1e-6))
            width = (TILE_W + 1) + dx * ppr
            if nt >= budget or rows * RUN * math.ceil(width / RUN) <= qcap:
                nch = nt
                break
        out[idx] = (D + nch - 1) // nch
    return out


# ------------------------------------------------------------------------------------------------ test geometry
def rigid(rng, trans, rot):
    """random rigid pose: rotation by rot * U(0.3, 1) rad about a random axis, translation trans * U(-1, 1)^3"""
    ax = rng.randn(3)
    ax /= np.linalg.norm(ax)
    ang = rot * rng.uniform(0.3, 1.0)
    Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    P = np.eye(4)
    P[:3, :3] = np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * Kx @ Kx
    P[:3, 3] = trans * rng.uniform(-1, 1, size=3)
    return P


def moderate_geometry(B, h, w, M, seed, trans=0.15, rot=0.05):
    """per-batch K (focal 0.9 w +-10 %, principal point +-2 px) and poses, measurement frames displaced by `trans` m and `rot`
    rad: (pose1 (B,4,4), [M x pose2 (B,4,4)], K (B,3,3)) as fp32 torch tensors"""
    rng = np.random.RandomState(seed)
    pose1 = np.stack([rigid(rng, 0.5, 0.3) for _ in range(B)])
    pose2s = [np.stack([pose1[b] @ rigid(rng, trans, rot) for b in range(B)]) for _ in range(M)]
    K = np.stack([np.array([[0.9 * w * rng.uniform(0.9, 1.1), 0, w / 2 + rng.uniform(-2, 2)],
                            [0, 0.9 * w * rng.uniform(0.9, 1.1), h / 2 + rng.uniform(-2, 2)], [0, 0, 1]]) for _ in range(B)])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    return t(pose1), [t(p) for p in pose2s], t(K)
