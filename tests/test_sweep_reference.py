"""plane_sweep_tc_kernel (1 and 3 terms), plane_sweep_c32_kernel and plane_sweep_generic_kernel against the fp64 reference of
tests/sweep_reference.py, sample by sample, on their own operands: the benchmark's launch, the BASELINE config 3 shape, partial
tiles, the M * D and D limits, tall bands, a denominator that changes sign on a tile, converging bands, zero baseline and extreme
feature magnitudes; the band-capacity limits of the planner (DVMVS_SWEEP_QCAP, read once per process) in subprocesses; and the
sweep bench.py's engine launches, replayed on its own buffers.  Every case first asserts, from the fp64 geometry, that it reaches
the paths it is meant to reach.  Prints per case, kernel and terms: worst err / bound, worst err / (u n S) not explained by the
other terms of the bound, the ill-conditioned samples and the median bound / sum w|s|."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import sweep_reference as R
from tests.tc_reference import C_ACC

pytestmark = pytest.mark.gpu

DEV = "cuda"
REPO_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIN_DEPTH, MAX_DEPTH = 0.25, 20.0
FP16_MAX = 65504.0


@pytest.fixture
def ops():
    from dvmvs import _ops
    old = (_ops._BACKEND, _ops._TC_TERMS_BASE, _ops._TC_STRIDE2)
    try:
        yield _ops
    finally:
        _ops.set_conv_backend(old[0], terms=old[1], stride2=old[2])


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))


def _clip_geometry(n_keyframes, H, W, M):
    """poses and half-resolution K of keyframes 0.. of a synthetic clip as synth.make_clip poses it (keyframe t: pose t + M, its
    measurement frames: poses t + M - k), stacked over the batch: the group bench.py's lookahead engine sweeps in one launch"""
    import synth_data as synth
    ref = [t + M for t in range(n_keyframes)]
    pose1 = _t(np.stack([synth.camera_pose(i) for i in ref]))
    pose2s = [_t(np.stack([synth.camera_pose(i - k) for i in ref])) for k in range(1, M + 1)]
    K = _t(np.stack([synth.intrinsics(H, W)] * n_keyframes))
    K[:, 0:2] /= 2.0
    return pose1, pose2s, K


def _relative(pose1, rel):
    """measurement poses pose1 @ rel (rel: 4x4, the measurement camera in the reference camera's frame)"""
    return pose1 @ _t(rel)[None]


def _rel(t, yaw=0.0):
    P = np.eye(4)
    c, s = np.cos(yaw), np.sin(yaw)
    P[:3, :3] = [[c, 0, s], [0, 1, 0], [-s, 0, c]]
    P[:3, 3] = t
    return P


def _half_K(h, w, B=1):
    import synth_data as synth
    K = _t(synth.intrinsics(2 * h, 2 * w))[None].repeat(B, 1, 1)
    K[:, 0:2] /= 2.0
    return K


# name: B, h, w, D, M
CASES = {
    "benchmark_group": (4, 128, 128, 64, 2),
    "c3": (1, 128, 160, 96, 4),
    "partial_tiles": (2, 37, 53, 32, 3),
    "tiny": (1, 3, 9, 2, 1),
    "max_frames": (1, 64, 96, 64, 8),
    "max_planes": (2, 48, 80, 128, 4),
    "vertical_motion": (1, 96, 64, 64, 2),
    "crossing": (1, 64, 64, 64, 2),
    "forward_motion": (1, 64, 96, 64, 2),
    "identity": (1, 32, 48, 16, 1),
    "magnitudes": (1, 64, 64, 32, 2),
    # bench.py's roofline launches (time_sweep): nb clips at 128x128, D = 64, M = 2, features randn x 4 seeded with nb, clip 0's
    # keyframe-0 poses repeated over the batch
    "roofline_1": (1, 128, 128, 64, 2),
    "roofline_8": (8, 128, 128, 64, 2),
    "roofline_32": (32, 128, 128, 64, 2),
}


def make_case(name):
    """geometry (fp32, CPU) and seeded features (scale 4 unless the case says otherwise) of one case"""
    B, h, w, D, M = CASES[name]
    seed = B if name.startswith("roofline_") else sum(map(ord, name))
    if name.startswith("roofline_"):
        pose1, pose2s, K = _clip_geometry(1, 2 * h, 2 * w, M)
        pose1, pose2s, K = pose1.repeat(B, 1, 1), [p.repeat(B, 1, 1) for p in pose2s], K.repeat(B, 1, 1)
    elif name == "benchmark_group":
        pose1, pose2s, K = _clip_geometry(4, 2 * h, 2 * w, M)
    elif name == "c3":
        pose1, pose2s, K = _clip_geometry(1, 2 * h, 2 * w, M)
    elif name in ("vertical_motion", "crossing", "forward_motion", "identity"):
        pose1, K = _t(R.rigid(np.random.RandomState(seed), 0.5, 0.3))[None], _half_K(h, w)
        if name == "identity":          # an exactly invertible pose: E = I and Kt = 0 in every precision
            pose1 = torch.eye(4)[None]
        rel = {"vertical_motion": [_rel([0, 9.0, 0]), _rel([0.05, 6.5, 0])],       # ~30 rows per plane: chunks > 64 rows
               "crossing": [_rel([0.05, 0.02, 1.0], yaw=0.3), _rel([0.1, 0, 0.1])],  # 1 m ahead: near planes behind the camera
               "forward_motion": [_rel([0.02, 0.01, -0.3]), _rel([0, 0, -0.15])],    # epipole inside the image
               "identity": [np.eye(4)]}[name]
        pose2s = [_relative(pose1, r) for r in rel]
    else:
        pose1, pose2s, K = R.moderate_geometry(B, h, w, M, seed)
    g = torch.Generator().manual_seed(seed)
    f1 = torch.randn(B, h, w, 32, generator=g) * 4
    f2s = [torch.randn(B, h, w, 32, generator=g) * 4 for _ in range(M)]
    if name == "magnitudes":
        # half the pixels around 1e-3 (fp16 subnormal after the 1-term pre-scale by 2^-5), the rest positive with a mean product of
        # about 2^13 per channel, so that S = sum_c f2 f1 / 32 reaches ~2^13 -- 1/8 of the fp16 range the 1-term kernel stores S in
        def mix(f):
            small = torch.rand(B, h, w, 1, generator=g) < 0.5
            return torch.where(small, f * 2.5e-4, f.abs() * 28.0)
        f1, f2s = mix(f1), [mix(f) for f in f2s]
    return dict(name=name, B=B, h=h, w=w, D=D, M=M, pose1=pose1, pose2s=pose2s, K=K, f1=f1, f2s=f2s)


def run_kernels(c, ops, forms=("tc1", "tc3", "fused", "generic")):
    """the kernels' outputs (B,h,w,D) on the case's operands, and the (hi, lo) planes they were given"""
    cu = lambda t: t.to(DEV)
    f1, f2s = cu(c["f1"]), [cu(f) for f in c["f2s"]]
    p1, p2s, K = cu(c["pose1"]), [cu(p) for p in c["pose2s"]], cu(c["K"])
    planes1, planes2 = ops.split_planes(f1), [ops.split_planes(f) for f in f2s]
    args = (p1, p2s, K, MIN_DEPTH, MAX_DEPTH, c["D"])
    out = {}
    for form in forms:
        if form in ("tc1", "tc3"):
            out[form] = ops.plane_sweep_tc(planes1, planes2, *args, terms=int(form[2]))
        else:
            out[form] = ops.plane_sweep(f1, f2s, *args, dot_product=True, force_generic=form == "generic")
    torch.cuda.synchronize()
    return out, planes1, planes2


def references(c, planes1, planes2):
    cu = lambda t: t.to(DEV)
    geo = (cu(c["pose1"]), [cu(p) for p in c["pose2s"]], cu(c["K"]), MIN_DEPTH, MAX_DEPTH, c["D"])
    pl = lambda p: (p[0], p[1])
    return {"tc1": R.sweep_reference("tc1", *geo, planes1=pl(planes1), planes2=[pl(p) for p in planes2]),
            "tc3": R.sweep_reference("tc3", *geo, planes1=pl(planes1), planes2=[pl(p) for p in planes2]),
            "gather": R.sweep_reference("gather", *geo, f1=cu(c["f1"]), f2s=[cu(f) for f in c["f2s"]])}


# ------------------------------------------------------------------------------------------------ paths the cases reach
def tc_qcap(terms, D, M):
    """the band capacity dvmvs_plane_sweep_tc picks by default (sweep_tc.cu host side; sizeof(StSmem) = 19736 bytes)"""
    fixed = 1024 + (2 if terms == 3 else 1) * 64 * 64 + ((D * 65 + 3) & ~3) * 4 + M * D * 48 + 19736 + 64
    per_q = 272 + 128 if terms == 3 else 144 + 64
    return min(int((227 * 1024 - fixed) // per_q) & ~31, 512 if terms == 3 else 1024)


def path_census(c, qcap):
    """plane_sweep_tc's plan of every tile, emulated from the fp64 geometry with the boxes widened and narrowed by 0.01 px: a
    property is counted only where both agree.  Returns counts of planes / chunks / tiles by path class."""
    B, h, w, D, M = c["B"], c["h"], c["w"], c["D"], c["M"]
    depths = R.plane_depths(MIN_DEPTH, MAX_DEPTH, D)
    per = {}
    for slack in (0.01, -0.01):
        geo = [R.tile_boxes(c["pose1"], p, c["K"], depths, h, w, slack) for p in c["pose2s"]]
        est = [R.first_guess(c["pose1"], p, c["K"], depths, h, w, qcap, D, M) for p in c["pose2s"]]
        box = np.stack([g[0] for g in geo], 3)                 # (B,ty,tx,M,D,4)
        sign_change = np.stack([g[1] for g in geo], 3)
        one_sign = np.stack([g[2] for g in geo], 3)
        all_neg = np.stack([g[3] for g in geo], 3)
        tall = box[..., 3] - box[..., 2] >= R.BAND_ROWS
        degenerate = ~one_sign | tall
        single = ((box[..., 1] - box[..., 0] + R.RUN) // R.RUN * R.RUN) * (box[..., 3] - box[..., 2] + 1)
        res = dict(sign_change=sign_change.sum(), negative_band=(all_neg & ~tall & (single <= qcap)).sum(),
                   tall_plane=tall.sum(), mixed_tiles=0, replanned_tiles=0, stuck_frames=0, direct_chunks=0, tall_chunks=0)
        for b, ty, tx in np.ndindex(box.shape[:3]):
            chunks, replanned, stuck = R.plan_tile(box[b, ty, tx], degenerate[b, ty, tx], D, M, qcap, [e[b, ty, tx] for e in est])
            kinds = {band for _, _, _, band in chunks}
            res["mixed_tiles"] += kinds == {True, False}
            res["replanned_tiles"] += replanned
            res["stuck_frames"] += sum(stuck)
            res["direct_chunks"] += sum(not band for _, _, _, band in chunks)
            for m, d0, nd, band in chunks:
                bx = box[b, ty, tx, m, d0:d0 + nd]
                res["tall_chunks"] += (not band) and nd > 1 and int(bx[:, 3].max() - bx[:, 2].min()) + 1 > R.BAND_ROWS
        per[slack] = res
    return {k: int(min(per[0.01][k], per[-0.01][k])) for k in per[0.01]}


CLAIMS = {   # case -> properties of the default-capacity plan that must be present (counted with a margin)
    "crossing": ("sign_change", "negative_band", "direct_chunks"),
    "vertical_motion": ("tall_chunks", "stuck_frames", "direct_chunks"),
}
QCAP_CLAIMS = {224: ("mixed_tiles", "replanned_tiles", "stuck_frames"), 64: ("direct_chunks",)}


def _assert_reach(c):
    B, h, w, D, M = c["B"], c["h"], c["w"], c["D"], c["M"]
    name = c["name"]
    G, Kt, _, _ = R.frame_geometry(c["pose1"], c["pose2s"][0], c["K"])
    if name == "benchmark_group":
        assert B * ((w + 15) // 16) * ((h + 3) // 4) >= 6 * 132, "fewer than ~8 tiles per persistent CTA"
    if name.startswith("roofline_"):
        assert (h, w, D, M) == (128, 128, 64, 2) and bool((c["pose1"] == c["pose1"][:1]).all())
    if name == "partial_tiles":
        assert h % 4 and w % 16 and M & (M - 1) and B > 1
    if name == "tiny":
        assert h < R.TILE_H and w < R.TILE_W and D == 2
    if name == "max_frames":
        assert M * D == 512 and 32 // M == 4
    if name == "max_planes":
        assert D == 128
    if name == "forward_motion":
        e = (Kt[0, :2] / Kt[0, 2]).tolist()
        assert 0 < e[0] < w and 0 < e[1] < h, "epipole %s outside the image" % e
    if name == "identity":
        assert float(Kt.abs().max()) == 0.0, "non-zero baseline"
    if name in CLAIMS:
        census = path_census(c, tc_qcap(1, D, M))
        print("%s: plan at the default band capacity %s" % (name, census))
        for k in CLAIMS[name]:
            assert census[k] > 0, "%s reaches no %s: %s" % (name, k, census)


def _describe(c):
    """failure context of a sample: its tile and, per frame, the plane's box, sign change and single-plane band size"""
    depths = R.plane_depths(MIN_DEPTH, MAX_DEPTH, c["D"])
    geo = [R.tile_boxes(c["pose1"], p, c["K"], depths, c["h"], c["w"]) for p in c["pose2s"]]

    def describe(idx):
        b, v, u, d = idx
        ty, tx = v // R.TILE_H, u // R.TILE_W
        parts = []
        for m, (box, sc, one, neg) in enumerate(geo):
            bx = box[b, ty, tx, d]
            single = (bx[1] - bx[0] + R.RUN) // R.RUN * R.RUN * (bx[3] - bx[2] + 1)
            parts.append("frame %d: box x [%d, %d] y [%d, %d], band %d px, %s" % (
                m, bx[0], bx[1], bx[2], bx[3], single, "sign change (direct)" if sc[b, ty, tx, d] else
                ("tall (direct)" if bx[3] - bx[2] >= R.BAND_ROWS else ("negative den" if neg[b, ty, tx, d] else "band"))))
        return "tile (b %d, ty %d, tx %d); %s" % (b, ty, tx, "; ".join(parts))
    return describe


def _check_all(c, outs, refs, tag=""):
    rows = []
    describe = _describe(c)
    for form, got in outs.items():
        ref = refs["gather" if form in ("fused", "generic") else form]
        what = "%s%s %s" % (c["name"], tag, form)
        worst, acc, tight = R.check_sweep(what, got, ref, describe)
        print("%-40s err/bound %.3f  err/(u n S) %.3f  ill-conditioned %d  median bound/sum w|s| %.2e" % (
            what, worst, acc, ref.n_ill, tight), flush=True)
        assert acc <= C_ACC / 8, "%s: measured accumulation constant %.3f > C_ACC / 8" % (what, acc)
        rows.append((what, worst, acc))
    return rows


def on_rows(c, outs, planes1, planes2):
    """the case, the kernels' outputs and operands restricted to the batch rows tools.engine_record.batch_rows picks: the sweep
    computes every output row from its own operand row, so the reference over these rows is exact for them"""
    from tools.engine_record import batch_rows
    rows = batch_rows(c["B"])
    if len(rows) == c["B"]:
        return c, outs, planes1, planes2
    r = torch.tensor(rows)
    c = dict(c, B=len(rows), pose1=c["pose1"][r], pose2s=[p[r] for p in c["pose2s"]], K=c["K"][r], f1=c["f1"][r], f2s=[f[r] for f in c["f2s"]])
    r = r.to(DEV)
    return c, {k: v.index_select(0, r) for k, v in outs.items()}, planes1.index_select(1, r), [p.index_select(1, r) for p in planes2]


@pytest.mark.parametrize("name", list(CASES))
def test_sweep_kernels_vs_fp64_reference(name, ops):
    c = make_case(name)
    _assert_reach(c)
    outs, planes1, planes2 = run_kernels(c, ops)
    c, outs, planes1, planes2 = on_rows(c, outs, planes1, planes2)
    refs = references(c, planes1, planes2)
    if name == "magnitudes":
        r = (planes1[0].float() * 2.0 ** -5).half()
        sub = float(((r != 0) & (r.abs() < 2.0 ** -14)).float().mean())
        print("magnitudes: %.0f %% of the pre-scaled reference operands subnormal, largest |S| %.4g (fp16 max %g)" % (
            100 * sub, refs["tc1"].smax, FP16_MAX))
        assert sub > 0.2 and 2.0 ** 13 <= refs["tc1"].smax < FP16_MAX
    _check_all(c, outs, refs)


_QCAP_SCRIPT = r"""
import sys, torch
sys.path[:0] = [%r, %r]
from dvmvs import _ops as ops
from tests import test_sweep_reference as T
for name in sys.argv[2:]:
    outs, _, _ = T.run_kernels(T.make_case(name), ops, forms=("tc1", "tc3"))
    torch.save({k: v.cpu() for k, v in outs.items()}, "%%s/%%s.pt" %% (sys.argv[1], name))
"""


@pytest.mark.parametrize("qcap", [224, 64])
def test_sweep_tc_band_capacity_vs_fp64_reference(qcap, ops, tmp_path):
    """the benchmark-group, max-frames and vertical-motion cases with the band capacity forced down (DVMVS_SWEEP_QCAP, read once per
    process: a subprocess per value).  224 (not a multiple of 64: the last MMA slice reads rows past the band) lets single-plane
    chunks fit, so the planner shortens chunks, runs out of chunk-list room and leaves frames stuck: band and direct chunks in one
    tile.  64: every plane takes the direct path."""
    names = ("benchmark_group", "max_frames", "vertical_motion")
    cases = {n: make_case(n) for n in names}
    census = {n: path_census(cases[n], qcap) for n in names}
    print("qcap %d plans: %s" % (qcap, census))
    for k in QCAP_CLAIMS[qcap]:
        assert sum(cs[k] for cs in census.values()) > 0, "qcap %d: no %s in %s" % (qcap, k, census)
    env = dict(os.environ, DVMVS_SWEEP_QCAP=str(qcap))
    code = _QCAP_SCRIPT % (REPO_DIR, os.path.join(REPO_DIR, "deep-video-mvs_b200"))
    out = subprocess.run([sys.executable, "-c", code, str(tmp_path)] + list(names), env=env, capture_output=True, text=True,
                         timeout=900, cwd=REPO_DIR)
    assert out.returncode == 0, out.stderr[-3000:]
    for n in names:
        c = cases[n]
        outs = torch.load(tmp_path / ("%s.pt" % n))
        _, planes1, planes2 = run_kernels(c, ops, forms=())
        _check_all(c, outs, references(c, planes1, planes2), tag=" qcap=%d" % qcap)


def test_sweep_of_the_benchmarked_engine_vs_fp64_reference(ops):
    """the sweep of every operating point bench.py reports (tools/engine_record.py POINTS), each checked by _engine_sweep_at; every
    point that fails is reported"""
    sys.path.insert(0, REPO_DIR)
    from tools.engine_record import POINTS
    failed = {}
    for point in POINTS:
        try:
            _engine_sweep_at(ops, point)
        except AssertionError as e:
            failed[point] = str(e)
        torch.cuda.empty_cache()
    assert not failed, "\n".join("%s: %s" % kv for kv in failed.items())


def _engine_sweep_at(ops, point):
    """the plane_sweep_tc launch of the engine bench.py runs at this operating point, recorded while it runs as bench.py runs it
    and replayed on its own buffers: the FPN features it really sweeps, under the bound of the point's terms, on the batch rows
    tools.engine_record.batch_rows picks.  Checks the sweep's batch, D, M and terms against the point's configuration."""
    import time
    from tools.engine_record import batch_rows, engine_calls, point_config
    t0 = time.perf_counter()
    cfg = point_config(point)
    _, calls = engine_calls(("plane_sweep_tc",), point=point)
    sweeps = [v for k, v in calls.items() if k[0] == "plane_sweep_tc"]
    assert len(sweeps) == 1, "%s: the engine launched %d plane_sweep_tc call sites" % (point, len(sweeps))
    for args, kw, _, _ in sweeps:
        ref_pair, meas_pairs, pose1, pose2s, K, mn, mx, D = args[:8]
        terms = kw.get("terms", 3)
        B, h, w, _ = ref_pair[0].shape
        expect_B = cfg["batch"] * (cfg["lookahead"] if cfg["engine"] == "lookahead" else 1)
        assert (B, D, len(pose2s), terms) == (expect_B, cfg["n_depth_levels"], cfg["n_measurement_frames"], cfg["terms"]), (
            "%s: sweep B, D, M, terms = %s, expected %s" % (point, (B, D, len(pose2s), terms),
                                                          (expect_B, cfg["n_depth_levels"], cfg["n_measurement_frames"], cfg["terms"])))
        rows = torch.tensor(batch_rows(B), device=DEV)
        sel = lambda t: t.index_select(0, rows)
        pl = lambda p: (sel(p[0]), sel(p[1]) if terms == 3 else None)
        from tests.tc_reference import check_live
        check_live("%s sweep" % point, sel(ref_pair[0]), *[sel(p[0]) for p in meas_pairs])
        got = ops.plane_sweep_tc(ref_pair, meas_pairs, pose1, pose2s, K, mn, mx, D, terms=terms)
        torch.cuda.synchronize()
        ref = R.sweep_reference("tc%d" % terms, sel(pose1).float(), [sel(p).float() for p in pose2s], sel(K).float(), mn, mx, D,
                                planes1=pl(ref_pair), planes2=[pl(p) for p in meas_pairs])
        c = dict(name="engine", B=len(rows), h=h, w=w, D=D, M=len(pose2s), pose1=sel(pose1).cpu(), pose2s=[sel(p).cpu() for p in pose2s],
                 K=sel(K).cpu())
        worst, acc, tight = R.check_sweep("%s sweep B=%d %dx%d terms=%d" % (point, B, h, w, terms), sel(got), ref, _describe(c))
        feat = max(float(ref_pair[0].float().abs().max()), max(float(p[0].float().abs().max()) for p in meas_pairs))
        print("%s sweep B=%d (rows %s) %dx%d D=%d M=%d terms=%d: err/bound %.3f  err/(u n S) %.3f  ill-conditioned %d  median bound/sum "
              "w|s| %.2e; largest |feature| %.4g, largest |S| %.4g (fp16 max %g); %.1f s" % (
                  point, B, batch_rows(B), h, w, D, len(pose2s), terms, worst, acc, ref.n_ill, tight, feat, ref.smax, FP16_MAX,
                  time.perf_counter() - t0))
        assert acc <= C_ACC / 8
        assert ref.smax < FP16_MAX / 8, "the engine's correlations come within 8x of the fp16 range of the 1-term S"
