"""fp64 reference of the hidden-state warp (hidden_warp_kernel, hidden_warp_backward_kernel) and of the depth re-projection
(depth_reproject_kernel), with a per-element bound.  Shared by the GPU tests (tests/test_geometry_reference.py) and by the CPU test
that checks the bounds against an fp32 emulation of the kernels and against planted defects (tests/test_geometry_reference_bound.py);
nothing here needs a GPU.  numpy throughout; poses (B,4,4), K (B,3,3) and depths are the fp32 arrays the kernels read.

Hidden warp (oracle/dvmvs_oracle.py warp_frame_depth, plus the `depth <= thresh` mask of convlstm.py): T = inv(prev) @ cur in
fp64 (cur itself when prev is None); every pixel (u, v) of depth d is unprojected with K, transformed, z <- relu(z), projected with
scale = 1/z (1 where |z| <= 1e-8) and h is sampled there bilinearly with zero padding (align_corners=True: at the pixel itself).

    position  delta = C_POS * u * (f * (P_a + |a| P_z / |z|) / |z| + |us| + |c| + w) per axis, P the running magnitudes of the
              transformed point (|inv(prev)| |cur| times |X|, |Y|, |Z|, 1); the last two terms are the kernel's normalise /
              unnormalise round trip.  Charged (delta_x + delta_y + delta_x delta_y) times the largest difference between the
              values of the 4x4 pixels around the sample (zeros outside the image): every cell the delta box can touch.
    blend     C_BLEND * u * sum_t w_t |h_t| (one product of weights, four fmaf).
    exact     masked pixels (d <= fp32 thresh), samples whose whole delta box lies outside (-1, w) x (-1, h), and samples at a
              non-finite position (NaN depth is not masked either) are +0 in every channel.
    ill       samples whose fp64 z lies within delta_z of the 1e-8 branch point (relu makes 0 and negative z take the scale-1
              branch too), or whose delta reaches half a pixel: only |out| <= max |h| of the channel is asserted; counted.

Backward: the fp64 transpose of the same weights, grad_in[q] = sum_p w_pq g_p.  Per q the bound sums, over the samples p whose
4x4 block contains q, 2 (delta_x + delta_y + delta_x delta_y) |g_p| (the weight moved by the position error) plus
(C_BLEND + n_q) u w_pq |g_p| (products and the n_q atomic additions in any order); an ill-conditioned sample may land anywhere
and is charged |g_p| on every pixel of its batch entry.

Re-projection (oracle get_non_differentiable_rectangle_depth_estimation): T = inv(cur) @ prev; every source pixel is projected with
the UN-relu'd z into the half-resolution grid (torch.round = half to even), and each target keeps the largest zr = max(z, 0).
A source is ambiguous if its projected position lies within delta of a .5 boundary (the image edges are such boundaries) or its
|z| within delta_z of 1e-8.  Per target, `sure` = the sources that certainly land there, `maybe` = sure + the ambiguous sources
that could; the kernel's value must lie in [max(sure) - eps, max(maybe) + eps], within eps of the zr of a member of maybe or +0
when sure is empty, be +0 when maybe is empty, and never carry a sign bit.  eps = C_ZR * u * P_z of that source.
"""
import numpy as np

from tests.sweep_reference import C_BLEND, _f32, fmaf, rigid
from tests.tc_reference import U

C_POS = 16.0            # units of u of the position magnitude: >= 8x the worst measured by the fp32 emulation (the CPU test prints it)
C_ZR = 32.0             # units of u of P_z for the kernel's z (and zr): >= 8x the worst measured by the emulation (3.27)
Z_TINY = 1e-8           # the projection's guard: scale = 1 where |z| <= 1e-8


def transforms(first, second):
    """fp64 T = inv(first) @ second and its running magnitude |inv(first)| |second| (B,4,4); first None: T = second"""
    s = np.asarray(second, np.float64)
    if first is None:
        return s, np.abs(s)
    inv = np.linalg.inv(np.asarray(first, np.float64))
    return inv @ s, np.abs(inv) @ np.abs(s)


def camera_points(T, Tmag, depth, K):
    """fp32 depth (B,h,w) -> fp64 transformed points p (B,3,h,w) and their running magnitudes P (B,3,h,w)"""
    B, h, w = depth.shape
    K = np.asarray(K, np.float64)
    d = depth.astype(np.float64)
    v, u = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    fx, fy, cx, cy = (K[:, 0, 0, None, None], K[:, 1, 1, None, None], K[:, 0, 2, None, None], K[:, 1, 2, None, None])
    with np.errstate(invalid="ignore"):
        X = (u - cx) / fx * d
        Y = (v - cy) / fy * d
        Pt = np.stack([X, Y, d, np.ones_like(d)], 1)
        p = np.einsum("bij,bjhw->bihw", T[:, :3], Pt)
        P = np.einsum("bij,bjhw->bihw", Tmag[:, :3], np.abs(Pt))
    return p, P


def project(p, P, K, relu, extent, branch=None):
    """fp64 pixel position (a_u, a_v) of the points, its bound (delta_u, delta_v), z as the projection sees it, delta_z and the
    ill-conditioned flag (the 1e-8 branch within reach, or delta >= 0.5 px).  relu: the warp's z <- relu(z); extent: the
    normalise / unnormalise round trip's (w, h), or (0, 0).  branch: None, or the side of the 1e-8 guard to evaluate whatever z
    is -- "one" (scale 1) or "inv" (scale 1 / z, z taken just above 1e-8 where it is not)."""
    K = np.asarray(K, np.float64)
    z = np.maximum(p[:, 2], 0.0) if relu else p[:, 2]
    dz = C_POS * U * P[:, 2]
    if branch == "inv":
        z = np.where(np.abs(z) > Z_TINY, z, Z_TINY * (1 + 1e-6))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        big = np.abs(z) > Z_TINY
        if branch == "one":
            big = np.zeros_like(big)
        scale = np.where(big, 1.0 / np.where(big, z, 1.0), 1.0)
        out, delta = [], []
        for a, f, c, ext in ((0, K[:, 0, 0], K[:, 0, 2], extent[0]), (1, K[:, 1, 1], K[:, 1, 2], extent[1])):
            f, c = f[:, None, None], c[:, None, None]
            pos = p[:, a] * scale * f + c
            az = np.abs(np.where(big, z, 1.0))
            mag = np.where(big, f * (P[:, a] + np.abs(p[:, a]) * P[:, 2] / az) / az, f * P[:, a])
            out.append(pos)
            delta.append(C_POS * U * (mag + np.abs(pos) + np.abs(c) + ext))
        # the warp's relu sends z <= 0 to the scale-1 branch too: only the 1e-8 threshold of the raw z can flip
        near = np.abs((p[:, 2] if relu else np.abs(z)) - Z_TINY) <= dz
        ill = (delta[0] >= 0.5) | (delta[1] >= 0.5)
        if branch is None:
            ill |= near
    return out[0], out[1], delta[0], delta[1], z, dz, ill


# ------------------------------------------------------------------------------------------------ hidden-state warp
class WarpGeometry:
    """per (b, pixel) fp64 sample position, bounds and the classification of the samples"""

    def __init__(self, depth, prev_pose, cur_pose, K, thresh, branch=None):
        depth = np.asarray(depth, np.float32)
        self.B, self.h, self.w = depth.shape
        T, Tmag = transforms(prev_pose, cur_pose)
        self.T = T
        p, P = camera_points(T, Tmag, depth, K)
        self.z_raw = p[:, 2]
        self.xs, self.ys, self.dx, self.dy, _, self.dz, ill = project(p, P, K, True, (self.w, self.h), branch)
        with np.errstate(invalid="ignore"):
            self.masked = depth <= np.float32(thresh)
            finite = np.isfinite(self.xs) & np.isfinite(self.ys)
            outside = ((self.xs + self.dx <= -1) | (self.xs - self.dx >= self.w) | (self.ys + self.dy <= -1) | (self.ys - self.dy >= self.h))
            zbranch = (np.abs(self.z_raw - Z_TINY) <= self.dz) & (branch is None)      # either side of the 1e-8 guard within reach
        self.zero = self.masked | ~finite | (outside & ~zbranch)
        self.ill = ill & ~self.zero
        self.live = ~self.zero & ~self.ill              # the samples checked against the bound
        xs, ys = np.where(self.live, self.xs, -5.0), np.where(self.live, self.ys, -5.0)
        self.x0, self.y0 = np.floor(xs).astype(np.int64), np.floor(ys).astype(np.int64)
        lx, ly = xs - self.x0, ys - self.y0
        self.wx = (1.0 - lx, lx)
        self.wy = (1.0 - ly, ly)

    def taps(self):
        """the four (dy, dx, weight, valid, flat index) taps of every sample (weight 0 where not live)"""
        for ty in (0, 1):
            for tx in (0, 1):
                yy, xx = self.y0 + ty, self.x0 + tx
                valid = self.live & (yy >= 0) & (yy < self.h) & (xx >= 0) & (xx < self.w)
                wt = np.where(valid, self.wy[ty] * self.wx[tx], 0.0)
                yield wt, valid, np.where(valid, yy * self.w + xx, 0)

    def block(self):
        """the 16 flat indices of the 4x4 pixels around every live sample, and whether each is inside the image"""
        for oy in (-1, 0, 1, 2):
            for ox in (-1, 0, 1, 2):
                yy, xx = self.y0 + oy, self.x0 + ox
                valid = self.live & (yy >= 0) & (yy < self.h) & (xx >= 0) & (xx < self.w)
                yield valid, np.where(valid, yy * self.w + xx, 0)

    def pos_factor(self):
        with np.errstate(invalid="ignore"):
            return np.where(self.live, self.dx + self.dy + self.dx * self.dy, 0.0)


class WarpRef:
    def __init__(self, geo, y, bound, cap, branches=()):
        self.geo, self.y, self.bound, self.cap, self.branches = geo, y, bound, cap, branches


def _gather(hf, b_idx, idx):
    return hf[b_idx, idx]                     # (B, npix, C)


def warp_reference(h_in, depth, prev_pose, cur_pose, K, thresh, branch=None):
    """h_in (B,h,w,C) fp32 -> WarpRef: y (B,h,w,C) fp64, bound, cap (B,C) = max |h| per channel; where samples are ill-conditioned
    by the 1e-8 guard, also the references of both of its branches"""
    geo = WarpGeometry(depth, prev_pose, cur_pose, K, thresh, branch)
    h64 = np.asarray(h_in, np.float64)
    B, hh, ww, C = h64.shape
    hf = h64.reshape(B, hh * ww, C)
    bi = np.arange(B)[:, None]
    y = np.zeros((B, hh * ww, C))
    mag = np.zeros((B, hh * ww, C))
    for wt, valid, idx in geo.taps():
        t = _gather(hf, bi, idx.reshape(B, -1))
        wt = wt.reshape(B, -1, 1)
        y += wt * t
        mag += wt * np.abs(t)
    hi = np.full((B, hh * ww, C), -np.inf)
    lo = np.full((B, hh * ww, C), np.inf)
    for valid, idx in geo.block():
        t = np.where(valid.reshape(B, -1, 1), _gather(hf, bi, idx.reshape(B, -1)), 0.0)
        hi, lo = np.maximum(hi, t), np.minimum(lo, t)
    rng = np.where(geo.live.reshape(B, -1, 1), hi - lo, 0.0)
    bound = C_BLEND * U * mag + 2.0 * geo.pos_factor().reshape(B, -1, 1) * rng
    cap = np.abs(h64).reshape(B, -1, C).max(1)
    branches = ()
    if branch is None and geo.ill.any():
        branches = tuple(warp_reference(h_in, depth, prev_pose, cur_pose, K, thresh, b) for b in ("one", "inv"))
    return WarpRef(geo, y.reshape(B, hh, ww, C), bound.reshape(B, hh, ww, C), cap, branches)


def warp_backward_reference(g_out, depth, prev_pose, cur_pose, K, thresh):
    """g_out (B,h,w,C) fp32 -> WarpRef of grad_h_in (B,h,w,C)"""
    geo = WarpGeometry(depth, prev_pose, cur_pose, K, thresh)
    g64 = np.asarray(g_out, np.float64)
    B, hh, ww, C = g64.shape
    gf = np.abs(g64.reshape(B, hh * ww, C))
    n = hh * ww
    y = np.zeros((B * n, C))
    S = np.zeros((B * n, C))
    cnt = np.zeros(B * n)
    off = (np.arange(B) * n)[:, None]
    for wt, valid, idx in geo.taps():
        flat = (idx.reshape(B, -1) + off).ravel()
        wv = wt.reshape(-1, 1)
        np.add.at(y, flat, wv * g64.reshape(B * n, C))
        np.add.at(S, flat, wv * gf.reshape(B * n, C))
        np.add.at(cnt, flat, valid.ravel().astype(np.float64))
    pos = np.zeros((B * n, C))
    pf = (2.0 * geo.pos_factor()).reshape(-1, 1) * gf.reshape(B * n, C)
    for valid, idx in geo.block():
        flat = (idx.reshape(B, -1) + off).ravel()
        np.add.at(pos, flat, np.where(valid.reshape(-1, 1), pf, 0.0))
    ill = (np.where(geo.ill.reshape(B, -1, 1), gf, 0.0)).sum(1)             # (B,C)
    bound = (C_BLEND + cnt[:, None]) * U * S + pos + np.repeat(ill, n, axis=0)
    return WarpRef(geo, y.reshape(B, hh, ww, C), bound.reshape(B, hh, ww, C), None)


def check_warp(what, got, ref, report=None, backward=False):
    """|kernel - y| <= bound on the live samples, +0 bit for bit on the exact-zero ones, |out| <= max |h| on the ill-conditioned
    ones (forward).  Returns the worst err / bound."""
    got = np.asarray(got, np.float32)
    geo = ref.geo
    if not backward:
        bits = got.view(np.uint32)
        zbad = geo.zero[..., None] & (bits != 0)
        if zbad.any():
            i = tuple(int(v) for v in np.argwhere(zbad)[0])
            raise AssertionError("%s: sample %s must be +0 (%s), kernel %r" % (what, i, "masked" if geo.masked[i[:3]] else
                                                                                 "outside the image / non-finite position", float(got[i])))
        # an ill-conditioned sample takes one side of the 1e-8 guard: its value must be that side's (a side that is itself
        # ill-conditioned -- a position error of half a pixel or more -- only bounds it by max |h|)
        ok = np.zeros(got.shape, bool)
        g64 = got.astype(np.float64)
        for alt in ref.branches:
            ag = alt.geo
            with np.errstate(invalid="ignore"):
                ok |= ag.zero[..., None] & (bits == 0)
                ok |= ag.live[..., None] & (np.abs(g64 - alt.y) <= alt.bound)
                ok |= ag.ill[..., None] & (np.abs(g64) <= ref.cap[:, None, None, :] * (1 + 8 * U))
        ill = geo.ill[..., None] & ~ok
        if ill.any():
            i = tuple(int(v) for v in np.argwhere(ill)[0])
            raise AssertionError("%s: ill-conditioned sample %s = %r is neither side's value of the 1e-8 guard" % (what, i, float(got[i])))
        sel = geo.live[..., None] & np.ones(got.shape, bool)
    else:
        sel = np.ones(got.shape, bool)
    err = np.abs(got.astype(np.float64) - ref.y)
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(sel, err / np.maximum(ref.bound, 1e-300), 0.0)
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    worst = float(ratio.max()) if ratio.size else 0.0
    if report is not None:
        report.append((what, worst))
    if worst > 1.0:
        i = tuple(int(v) for v in np.unravel_index(np.argmax(ratio), ratio.shape))
        raise AssertionError("%s: |kernel - fp64 reference| exceeds the bound by x%.3g at %s (kernel %r, reference %r, bound %.3e)"
                             % (what, worst, i, float(got[i]), float(ref.y[i]), float(ref.bound[i])))
    return worst


# ------------------------------------------------------------------------------------------------ depth re-projection
class ReprojectRef:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def reproject_reference(cur_pose, prev_pose, prev_depth, full_K, half_K, H, W):
    """the sure / maybe sets of every half-resolution target (see the module docstring)"""
    depth = np.asarray(prev_depth, np.float32).reshape(-1, H, W)
    B = depth.shape[0]
    hw, hh = W // 2, H // 2
    T, Tmag = transforms(cur_pose, prev_pose)
    p, P = camera_points(T, Tmag, depth, full_K)
    pu, pv, du, dv, z, dz, ill_z = project(p, P, half_K, False, (0, 0))
    with np.errstate(invalid="ignore"):
        zr = np.maximum(z, 0.0)
        eps = C_ZR * U * P[:, 2]
        zamb = ill_z                                     # near the 1e-8 branch, or a position error of half a pixel and more
        tu, tv = np.round(pu), np.round(pv)              # numpy rounds half to even, as torch.round
        amb_u = np.abs(np.abs(pu - np.floor(pu)) - 0.5) <= du
        amb_v = np.abs(np.abs(pv - np.floor(pv)) - 0.5) <= dv
    amb = amb_u | amb_v | zamb
    sure = ~amb & (tu >= 0) & (tv >= 0) & (tu < hw) & (tv < hh)
    cells, vals, epss, sure_flag = [], [], [], []
    bidx = np.broadcast_to(np.arange(B)[:, None, None], pu.shape)
    for su in (-1, 0, 1):
        for sv in (-1, 0, 1):
            if su == 0 and sv == 0:
                cu, cv, sel = tu, tv, ~np.isnan(tu) & ~np.isnan(tv)
                sel = sel & ~zamb
            else:
                cu, cv = tu + su, tv + sv
                sel = (amb_u | (su == 0)) & (amb_v | (sv == 0)) & ~zamb & (amb_u | amb_v)
            sel = sel & (cu >= 0) & (cv >= 0) & (cu < hw) & (cv < hh)
            cells.append((bidx[sel] * hh * hw + cv[sel].astype(np.int64) * hw + cu[sel].astype(np.int64)))
            vals.append(zr[sel])
            epss.append(eps[sel])
            sure_flag.append(sure[sel] if (su == 0 and sv == 0) else np.zeros(int(sel.sum()), bool))
    cells, vals, epss, sure_flag = (np.concatenate(a) for a in (cells, vals, epss, sure_flag))
    n = B * hh * hw
    lo = np.full(n, -np.inf)
    np.maximum.at(lo, cells[sure_flag], vals[sure_flag] - epss[sure_flag])
    has_sure = np.zeros(n, bool)
    has_sure[cells[sure_flag]] = True
    hi = np.full(n, -np.inf)
    np.maximum.at(hi, cells, vals + epss)
    # sources whose z is within reach of the 1e-8 branch may land anywhere: their zr (tiny) is a candidate of every target
    zamb_b = [zr[b][zamb[b]] for b in range(B)]
    zamb_max = np.array([(v.max() + eps[b][zamb[b]].max()) if v.size else -np.inf for b, v in enumerate(zamb_b)])
    hi = np.maximum(hi, np.repeat(zamb_max, hh * hw))
    return ReprojectRef(cells=cells, vals=vals, eps=epss, lo=lo, hi=hi, has_sure=has_sure, sure_cells=cells[sure_flag], zamb_b=zamb_b, zamb_eps=[eps[b][zamb[b]] for b in range(B)],
                        shape=(B, hh, hw), n_amb=int(amb.sum()), n_zamb=int(zamb.sum()), n_sure=int(sure.sum()),
                        n_behind=int((z < 0).sum()), tu=tu, tv=tv, z=z, amb=amb)


def check_reproject(what, got, ref, report=None):
    """the rules of the module docstring; returns the number of targets checked against a non-empty `sure`"""
    got = np.asarray(got, np.float32).reshape(-1)
    B, hh, hw = ref.shape
    bits = got.view(np.uint32)
    g = got.astype(np.float64)

    def fail(msg, i):
        b, r = divmod(int(i), hh * hw)
        raise AssertionError("%s: target (b=%d, row %d, col %d) = %r: %s" % (what, b, r // hw, r % hw, float(got[i]), msg))

    neg = np.nonzero(bits >> 31)[0]
    if neg.size:
        fail("sign bit set", neg[0])
    empty = ~np.isfinite(ref.hi)
    bad = np.nonzero(empty & (bits != 0))[0]
    if bad.size:
        fail("no source can land here: must be +0", bad[0])
    bad = np.nonzero(ref.has_sure & (g < ref.lo))[0]
    if bad.size:
        fail("below the largest sure source %r" % float(ref.lo[bad[0]]), bad[0])
    bad = np.nonzero(~empty & (g > ref.hi))[0]
    if bad.size:
        fail("above every source that may land here (%r)" % float(ref.hi[bad[0]]), bad[0])
    # the value is one source's zr (or +0 with no sure source)
    best = np.full(g.shape, np.inf)
    np.minimum.at(best, ref.cells, np.abs(g[ref.cells] - ref.vals) - ref.eps)
    for b in range(B):
        if ref.zamb_b[b].size:
            sl = slice(b * hh * hw, (b + 1) * hh * hw)
            d = (np.abs(g[sl][:, None] - ref.zamb_b[b][None, :]) - ref.zamb_eps[b][None, :]).min(1)
            best[sl] = np.minimum(best[sl], d)
    ok = (best <= 0) | (~ref.has_sure & (bits == 0))
    bad = np.nonzero(~ok)[0]
    if bad.size:
        fail("not the zr of any source that may land here", bad[0])
    if report is not None:
        report.append((what, int(ref.has_sure.sum())))
    return int(ref.has_sure.sum())


# ------------------------------------------------------------------------------------------------ fp32 emulation of the kernels
def _mat4_mul(a, b):
    o = np.zeros(a.shape, np.float32)
    for i in range(4):
        for j in range(4):
            s = np.zeros(a.shape[0], np.float32)
            for k in range(4):
                s = fmaf(a[:, i, k], b[:, k, j], s)
            o[:, i, j] = s
    return o


def emulate_transform(first, second):
    """mat4_rigid_free_inverse (double, rounded to fp32) then mat4_mul's fmaf chains; first None: second"""
    second = _f32(second)
    if first is None:
        return second.copy()
    return _mat4_mul(_f32(np.linalg.inv(np.asarray(first, np.float64))), second)


def _emulate_points(T, depth, K, b_T=None):
    B, h, w = depth.shape
    K = _f32(K)
    v, u = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    fx, fy, cx, cy = K[:, 0, 0, None, None], K[:, 1, 1, None, None], K[:, 0, 2, None, None], K[:, 1, 2, None, None]
    if b_T is not None:
        T = np.broadcast_to(T[b_T:b_T + 1], T.shape)
    t = lambda i: T[:, i // 4, i % 4, None, None]
    with np.errstate(invalid="ignore", over="ignore"):
        X = _f32(_f32(_f32(u - cx) / fx) * depth)
        Y = _f32(_f32(_f32(v - cy) / fy) * depth)
        Z = depth
        x = _f32(fmaf(t(0), X, fmaf(t(1), Y, _f32(t(2) * Z))) + t(3))
        y = _f32(fmaf(t(4), X, fmaf(t(5), Y, _f32(t(6) * Z))) + t(7))
        z = _f32(fmaf(t(8), X, fmaf(t(9), Y, _f32(t(10) * Z))) + t(11))
    return x, y, z, fx, fy, cx, cy


def emulate_warp_positions(depth, prev_pose, cur_pose, K, variant=None):
    """hidden_warp_kernel's fp32 sample positions (xs, ys) (B,h,w); variant: a planted defect (see emulate_warp)"""
    depth = _f32(depth)
    B, h, w = depth.shape
    T = emulate_transform(prev_pose, cur_pose)
    x, y, z, fx, fy, cx, cy = _emulate_points(T, depth, K, 0 if variant == "batch0_transform" else None)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if variant != "no_relu":
            z = np.maximum(z, np.float32(0))
        scale = np.where(np.abs(z) > np.float32(Z_TINY), _f32(np.float32(1) / z), np.float32(1))
        us = fmaf(_f32(x * scale), fx, cx)
        vs = fmaf(_f32(y * scale), fy, cy)
        sw, sh = _f32(np.float32(2) / np.float32(w - 1)), _f32(np.float32(2) / np.float32(h - 1))
        gx, gy = fmaf(us, sw, np.float32(-1)), fmaf(vs, sh, np.float32(-1))
        if variant == "align_corners_false":
            xs = _f32(_f32(_f32(_f32(gx + np.float32(1)) * np.float32(w)) - np.float32(1)) * np.float32(0.5))
            ys = _f32(_f32(_f32(_f32(gy + np.float32(1)) * np.float32(h)) - np.float32(1)) * np.float32(0.5))
        else:
            xs = _f32(_f32(_f32(gx + np.float32(1)) * np.float32(0.5)) * np.float32(w - 1))
            ys = _f32(_f32(_f32(gy + np.float32(1)) * np.float32(0.5)) * np.float32(h - 1))
    return xs, ys


def _emulate_taps(xs, ys, h, w, variant=None):
    with np.errstate(invalid="ignore"):
        if variant == "int_truncation":
            x0, y0 = _f32(np.trunc(xs)), _f32(np.trunc(ys))
        else:
            x0, y0 = _f32(np.floor(xs)), _f32(np.floor(ys))
        wx = (_f32(_f32(x0 + np.float32(1)) - xs), _f32(xs - x0))
        wy = (_f32(_f32(y0 + np.float32(1)) - ys), _f32(ys - y0))
        for dy in (0, 1):
            for dx in (0, 1):
                xf, yf = x0 + dx, y0 + dy
                ok = (xf >= 0) & (xf <= w - 1) & (yf >= 0) & (yf <= h - 1)
                wt = _f32(wx[dy] * wy[dx]) if variant == "swap_xy_weights" else _f32(wx[dx] * wy[dy])
                idx = np.where(ok, np.nan_to_num(yf) * w + np.nan_to_num(xf), 0).astype(np.int64)
                yield ok, wt, idx


WARP_DEFECTS = ("int_truncation", "batch0_transform", "mask_lt", "no_relu", "swap_xy_weights", "align_corners_false")


def emulate_warp(h_in, depth, prev_pose, cur_pose, K, thresh, variant=None):
    """hidden_warp_kernel in fp32 numpy, operation for operation; variant: one of WARP_DEFECTS"""
    h_in, depth = _f32(h_in), _f32(depth)
    B, h, w, C = h_in.shape
    xs, ys = emulate_warp_positions(depth, prev_pose, cur_pose, K, variant)
    with np.errstate(invalid="ignore"):
        masked = (depth < np.float32(thresh)) if variant == "mask_lt" else (depth <= np.float32(thresh))
    o = np.zeros((B, h * w, C), np.float32)
    hf = h_in.reshape(B, h * w, C)
    bi = np.arange(B)[:, None]
    for ok, wt, idx in _emulate_taps(xs, ys, h, w, variant):
        ok = ok & ~masked
        t = hf[bi, idx.reshape(B, -1)]
        o = np.where(ok.reshape(B, -1, 1), fmaf(t, wt.reshape(B, -1, 1), o), o)
    return o.reshape(B, h, w, C)


def emulate_warp_backward(g_out, depth, prev_pose, cur_pose, K, thresh):
    """hidden_warp_backward_kernel in fp32 numpy: wt * g rounded, then added (atomics) in pixel order"""
    g_out, depth = _f32(g_out), _f32(depth)
    B, h, w, C = g_out.shape
    xs, ys = emulate_warp_positions(depth, prev_pose, cur_pose, K)
    with np.errstate(invalid="ignore"):
        masked = depth <= np.float32(thresh)
    out = np.zeros((B * h * w, C), np.float32)
    off = (np.arange(B) * h * w)[:, None]
    for ok, wt, idx in _emulate_taps(xs, ys, h, w):
        ok = (ok & ~masked).ravel()
        flat = (idx.reshape(B, -1) + off).ravel()[ok]
        contrib = _f32(wt.reshape(-1, 1)[ok] * g_out.reshape(-1, C)[ok])
        for i, f in enumerate(flat):          # sequential fp32 additions (the atomics' order is arbitrary; this is one order)
            out[f] = _f32(out[f] + contrib[i])
    return out.reshape(B, h, w, C)


REPROJECT_DEFECTS = ("floor", "min", "bound_le", "relu_projection")


def emulate_reproject(cur_pose, prev_pose, prev_depth, full_K, half_K, H, W, variant=None):
    """depth_reproject_kernel in fp32 numpy: z-as-uint atomicMax of zr onto the rintf-rounded half-resolution target"""
    depth = _f32(prev_depth).reshape(-1, H, W)
    B = depth.shape[0]
    hw, hh = W // 2, H // 2
    T = emulate_transform(cur_pose, prev_pose)
    x, y, z, *_ = _emulate_points(T, depth, full_K)
    Kh = _f32(half_K)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        zr = np.maximum(z, np.float32(0))
        zp = zr if variant == "relu_projection" else z
        scale = np.where(np.abs(zp) > np.float32(Z_TINY), _f32(np.float32(1) / zp), np.float32(1))
        rnd = np.floor if variant == "floor" else np.rint
        pu = _f32(rnd(fmaf(_f32(x * scale), Kh[:, 0, 0, None, None], Kh[:, 0, 2, None, None])))
        pv = _f32(rnd(fmaf(_f32(y * scale), Kh[:, 1, 1, None, None], Kh[:, 1, 2, None, None])))
        ok = (pu >= 0) & (pv >= 0) & (pv < hh) & ((pu <= hw) if variant == "bound_le" else (pu < hw))
    flat = (np.arange(B)[:, None, None] * hh * hw + np.where(ok, pv, 0).astype(np.int64) * hw + np.where(ok, pu, 0).astype(np.int64))[ok]
    vals = zr[ok].view(np.uint32)
    keep = flat < B * hh * hw
    if variant == "min":
        out = np.full(B * hh * hw, np.uint32(0xFFFFFFFF))
        np.minimum.at(out, flat[keep], vals[keep])
        out[out == np.uint32(0xFFFFFFFF)] = 0
    else:
        out = np.zeros(B * hh * hw, np.uint32)
        np.maximum.at(out, flat[keep], vals[keep])
    return out.view(np.float32).reshape(B, 1, hh, hw)


# ------------------------------------------------------------------------------------------------ test cases
F32_THRESH = float(np.float32(0.01))         # convlstm.py's invalid-depth threshold as the kernel compares it

WARP_CASES = {
    # name: B, C, h, w, trans, rot, seed, kind ("prev": inv(prev) @ cur, thresh 0.01; "edges": + depths at the threshold and NaN;
    # "raw": prev_pose = NULL, thresh = -inf, a transform that puts z below, at and just above 0 and at the 1e-8 guard)
    "bench_256_8x8": (1, 512, 8, 8, 0.10, 0.05, 1, "prev"),
    "bench_landscape_8x10": (1, 512, 8, 10, 0.10, 0.05, 2, "prev"),
    "bench_portrait_10x8": (1, 512, 10, 8, 0.10, 0.05, 3, "prev"),
    "batch3_distinct_poses": (3, 64, 8, 8, 0.30, 0.20, 4, "prev"),
    "c4_partial_last_cta": (2, 4, 23, 19, 0.25, 0.10, 5, "prev"),
    "threshold_and_nan_depth": (1, 8, 12, 16, 0.002, 0.002, 6, "edges"),      # slight motion: depth 0.01 stays in view
    "raw_transform_z_signs": (1, 8, 9, 12, 0.0, 0.0, 7, "raw"),
}


def warp_case(name):
    """(h_in (B,h,w,C), depth (B,h,w), prev_pose or None, cur_pose, K, thresh) as fp32 numpy"""
    B, C, h, w, trans, rot, seed, kind = WARP_CASES[name]
    rng = np.random.RandomState(100 + seed)
    h_in = rng.randn(B, h, w, C).astype(np.float32)
    depth = (0.3 + 4.0 * np.abs(rng.randn(B, h, w))).astype(np.float32)
    K = np.stack([np.array([[0.9 * w * rng.uniform(0.9, 1.1), 0, w / 2 + rng.uniform(-1, 1)],
                            [0, 0.9 * w * rng.uniform(0.9, 1.1), h / 2 + rng.uniform(-1, 1)], [0, 0, 1]]) for _ in range(B)]).astype(np.float32)
    if kind == "raw":
        # z = 2^-24 d - 2^-23: negative below d = 2, exactly 0 at d = 2, 2^-46 at the next float up, 6e-8 (> 1e-8) at d = 3
        T = np.eye(4)
        T[2, 2], T[2, 3] = 2.0 ** -24, -(2.0 ** -23)
        T[0, 3], T[1, 3] = 0.05, -0.03
        depth.reshape(-1)[0:4] = [2.0, np.nextafter(np.float32(2.0), np.float32(3.0)), 1.5, 3.0]
        depth.reshape(-1)[4] = 2.0 + 1e-8 * 2 ** 24        # z within rounding of the 1e-8 guard: ill-conditioned, either side
        depth.reshape(-1)[5:40] = 1.0 + rng.uniform(0, 0.9, 35)
        depth.reshape(-1)[40] = np.nan
        return h_in, depth, None, T[None].repeat(B, 0).astype(np.float32), K, float("-inf")
    prev = np.stack([rigid(rng, 0.5, 0.3) for _ in range(B)])
    cur = np.stack([prev[b] @ rigid(rng, trans, rot) for b in range(B)])
    if kind == "edges":
        d = depth.reshape(-1)
        d[0] = np.float32(0.01)
        d[1] = np.nextafter(np.float32(0.01), np.float32(1.0))
        d[2] = 0.0
        d[3] = np.nan
    return h_in, depth, prev.astype(np.float32), cur.astype(np.float32), K, F32_THRESH


def warp_reach(geo):
    """what a case's fp64 geometry reaches (asserted by the tests)"""
    live = geo.live
    r = {}
    for ax, pos, n in (("x", geo.xs, geo.w), ("y", geo.ys, geo.h)):
        with np.errstate(invalid="ignore"):
            r["neg_frac_" + ax] = bool((live & (pos > -1) & (pos < 0)).any())
            r["past_last_" + ax] = bool((live & (pos > n - 1) & (pos < n)).any())
    with np.errstate(invalid="ignore"):
        r["z_negative"] = bool((~geo.masked & (geo.z_raw < 0)).any())
        r["z_zero"] = bool((~geo.masked & (geo.z_raw == 0)).any())
        r["z_tiny"] = bool((~geo.masked & (geo.z_raw > 0) & (geo.z_raw < Z_TINY)).any())
        r["z_at_guard"] = bool(geo.ill.any())
    return r


REPROJECT_CASES = {
    # name: B, H, W, kind, seed
    "clip_256_keyframes_0_1": (1, 256, 256, "clip", 1),
    "batch2_distinct_poses": (2, 64, 96, "random", 2),
    "forward_motion": (1, 64, 64, "forward", 3),
    "behind_camera": (1, 48, 64, "behind", 4),
    "odd_half_size_depth_zeros": (1, 54, 70, "random", 5),
}


def reproject_case(name, synth=None):
    """(cur_pose, prev_pose, prev_depth (B,1,H,W), full_K, half_K, H, W) as fp32 numpy; "clip" needs synth_data"""
    B, H, W, kind, seed = REPROJECT_CASES[name]
    rng = np.random.RandomState(200 + seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    depth = np.stack([1.5 + 0.6 * np.sin(3 * xx + b) * np.cos(2 * yy) + 0.05 * rng.randn(H, W) for b in range(B)])[:, None]
    K = np.array([[0.9 * W, 0, W / 2.0 + 1.3], [0, 0.9 * W, H / 2.0 - 0.7], [0, 0, 1]])
    if kind == "clip":
        clip = synth.make_clip(0, 2, H, W, 1)
        cur, prev = clip["poses"][1][None], clip["poses"][0][None]
        K = clip["K"].astype(np.float64)
    elif kind == "forward":
        cur = np.stack([rigid(rng, 0.5, 0.3) for _ in range(B)])
        step = np.eye(4)
        step[2, 3] = 0.4                           # the previous camera stood 0.4 m further forward: its view shrinks into ours
        prev = np.stack([cur[b] @ step for b in range(B)])
    elif kind == "behind":
        cur = np.stack([rigid(rng, 0.5, 0.3) for _ in range(B)])
        turn = np.eye(4)
        turn[0, 0] = turn[2, 2] = -1.0             # the previous camera looked the other way from 1 m ahead: most of its view
        turn[:3, 3] = [0.05, 0.0, 1.0]             # lies behind us and projects, mirrored, into the image
        prev = np.stack([cur[b] @ turn for b in range(B)])
    else:
        cur = np.stack([rigid(rng, 0.5, 0.3) for _ in range(B)])
        prev = np.stack([cur[b] @ rigid(rng, 0.15, 0.08) for b in range(B)])
    if kind != "clip":
        depth[:, :, 0:2, :] = 0.0                  # invalid (zero) depths of the previous prediction
    full_K = np.stack([K] * B).astype(np.float32)
    half_K = full_K.copy()
    half_K[:, 0:2, :] /= 2.0
    return cur.astype(np.float32), prev.astype(np.float32), depth.astype(np.float32), full_K, half_K, H, W


def reproject_reach(ref):
    """sources per target, behind-camera sources landing inside, targets on the last row / column"""
    B, hh, hw = ref.shape
    counts = np.bincount(ref.sure_cells, minlength=B * hh * hw)          # sources certain to land on each target
    inside = (ref.tu >= 0) & (ref.tv >= 0) & (ref.tu < hw) & (ref.tv < hh)
    with np.errstate(invalid="ignore"):
        return dict(max_sources=int(counts.max()), behind_inside=int((inside & (ref.z < 0)).sum()),
                    last_col=bool((inside & (ref.tu == hw - 1)).any()), last_row=bool((inside & (ref.tv == hh - 1)).any()))
