"""The fp64 reference and per-sample bound of tests/sweep_reference.py are the unmodified reference's semantics, neither vacuous nor
tighter than honest fp32 arithmetic: the reference matches the oracle and the golden vectors, an fp32 emulation of the kernels'
position arithmetic stays within the position term, an fp32 stand-in of the band algorithm passes, and each planted defect of the
kind a plane-sweep kernel could have is rejected."""
import numpy as np
import pytest
import torch

from tests import sweep_reference as R


def _nhwc(x):
    return torch.from_numpy(np.ascontiguousarray(x)).permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------ the reference itself
def test_reference_matches_oracle_and_golden(oracle, synth, cases, golden_ops):
    """every golden plane-sweep case (dot and SAD): the fp64 reference on the fp32 features is within the gather bound of the
    golden vectors of the unmodified reference and of oracle.cost_volume_fusion"""
    for name, c in cases.PLANE_SWEEP_CASES.items():
        inp = cases.plane_sweep_inputs(synth, c)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
        pose1, pose2s, K = t(inp["pose1"]), [t(p) for p in inp["pose2s"]], t(inp["K"])
        ref = R.sweep_reference("gather", pose1, pose2s, K, c["min_depth"], c["max_depth"], c["D"], f1=_nhwc(inp["image1"]),
                                f2s=[_nhwc(x) for x in inp["image2s"]], dot=c["dot"])
        gold = torch.from_numpy(golden_ops["plane_sweep/" + name]).permute(0, 2, 3, 1)
        worst_g, _, _ = R.check_sweep("golden plane_sweep/" + name, gold, ref)
        orc = oracle.cost_volume_fusion(t(inp["image1"]), [t(x) for x in inp["image2s"]], pose1, pose2s, K,
                                        oracle.get_warp_grid_for_cost_volume_calculation(c["w"], c["h"]), c["min_depth"],
                                        c["max_depth"], c["D"], "cpu", c["dot"]).permute(0, 2, 3, 1)
        worst_o, _, _ = R.check_sweep("oracle plane_sweep/" + name, orc, ref)
        print("plane_sweep/%s: err/bound golden %.3f, oracle %.3f, ill-conditioned samples %d" % (name, worst_g, worst_o, ref.n_ill))


# ------------------------------------------------------------------------------------------------ CPU cases
# name, B, h, w, D, M, trans, rot, seed
CASES = [
    ("moderate", 2, 13, 37, 12, 3, 0.15, 0.05, 11),
    ("wide", 1, 12, 20, 10, 2, 1.5, 0.5, 12),
    ("single", 1, 9, 18, 9, 1, 0.3, 0.1, 13),
]


def _case(name):
    _, B, h, w, D, M, trans, rot, seed = next(c for c in CASES if c[0] == name)
    pose1, pose2s, K = R.moderate_geometry(B, h, w, M, seed, trans, rot)
    g = torch.Generator().manual_seed(seed)
    f1 = torch.randn(B, h, w, 32, generator=g) * 4
    f2s = [torch.randn(B, h, w, 32, generator=g) * 4 for _ in range(M)]
    return dict(B=B, h=h, w=w, D=D, M=M, pose1=pose1, pose2s=pose2s, K=K, f1=f1, f2s=f2s)


def test_position_emulation_within_delta():
    """the kernels' fp32 positions (st_position / sweep_phase_a and sweep_sample_pos, emulated in numpy fp32) differ from the fp64
    positions by less than delta at every well-conditioned sample; prints the measured constant, which C_POS exceeds 8x"""
    worst = 0.0
    for name in [c[0] for c in CASES] + ["benchmark_geometry"]:
        if name == "benchmark_geometry":          # 128 x 128 half-resolution geometry of the synthetic clip, forward and crossing poses too
            import synth_data as synth
            h = w = 128
            K = torch.from_numpy(synth.intrinsics(256, 256))[None].clone()
            K[:, 0:2] /= 2
            pose1 = torch.from_numpy(synth.camera_pose(3))[None]
            fwd = pose1.clone()
            fwd[:, 2, 3] -= 1.0
            pose2s, D = [torch.from_numpy(synth.camera_pose(3 - k))[None] for k in (1, 2)] + [fwd], 64
        else:
            c = _case(name)
            h, w, D, K, pose1, pose2s = c["h"], c["w"], c["D"], c["K"], c["pose1"], c["pose2s"]
        depths = R.plane_depths(0.25, 20.0, D)
        for p2 in pose2s:
            P = R.positions(pose1, p2, K, depths, h, w)
            ok = torch.isfinite(P["xs"]) & (P["delta_x"] < 1) & (P["delta_y"] < 1)
            for variant in ("st", "generic"):
                xe, ye = R.emulate_positions(pose1.numpy(), p2.numpy(), K.numpy(), depths.numpy(), h, w, variant)
                for e, ref, dl in ((xe, P["xs"], P["delta_x"]), (ye, P["ys"], P["delta_y"])):
                    err = (torch.from_numpy(e.astype(np.float64)) - ref).abs()
                    ratio = (err / dl)[ok]
                    assert bool((ratio <= 1).all()), "%s %s: fp32 position outside delta by x%.3g" % (name, variant, float(ratio.max()))
                    worst = max(worst, float(ratio.max()) * R.C_POS)
    print("position error: measured constant %.3f units of u (C_POS = %g, ratio %.1f)" % (worst, R.C_POS, R.C_POS / max(worst, 1e-30)))
    assert R.C_POS >= 8 * worst


# ------------------------------------------------------------------------------------------------ fp32 stand-in of the band algorithm
PLANES = slice(4, 8)      # the chunk the chunk defects hit


def standin(c, terms, defect=None):
    """plane_sweep_tc's algorithm in torch fp32: S from the fp16 operands (fp16 store at 1 term), blended at the emulated fp32
    positions with zero padding, frames summed in order, divided by M.  -> (B,h,w,D) fp32"""
    B, h, w, D, M = c["B"], c["h"], c["w"], c["D"], c["M"]
    hi1 = c["f1"].half().float()
    lo1 = (c["f1"] - hi1).half().float()
    r = (hi1 * 2.0 ** -5).half().float()
    depths = R.plane_depths(0.25, 20.0, D).numpy()
    acc = torch.zeros(B, D, h, w)
    u_idx = torch.arange(w).view(1, 1, 1, w)
    for m in range(M):
        hi2 = c["f2s"][m].half().float()
        lo2 = (c["f2s"][m] - hi2).half().float()
        dep = depths.copy()
        if defect == "d0_off_by_one" and m == 0:
            dep[PLANES] = depths[PLANES.start + 1:PLANES.stop + 1]
        xs, ys = R.emulate_positions(c["pose1"].numpy(), c["pose2s"][m].numpy(), c["K"].numpy(), dep, h, w)
        xs, ys = torch.from_numpy(xs), torch.from_numpy(ys)
        if defect == "no_shrink":
            xs, ys = xs / np.float32((w - 1) / w), ys / np.float32((h - 1) / h)
        xs = torch.nan_to_num(xs, nan=-1.0).clamp(-1.0, float(w))
        ys = torch.nan_to_num(ys, nan=-1.0).clamp(-1.0, float(h))
        x0f, y0f = torch.floor(xs), torch.floor(ys)
        fx, fy, gx, gy = xs - x0f, ys - y0f, (x0f + 1) - xs, (y0f + 1) - ys
        s = []
        for t in range(4):
            x, y = x0f.long() + (t & 1), y0f.long() + (t >> 1)
            if defect == "tap_one_over_at_tile_edge" and (t & 1):
                x = torch.where(u_idx % R.TILE_W == R.TILE_W - 1, x + 1, x)
            inside = (x >= 0) & (x < w) & (y >= 0) & (y < h)
            if defect == "clamp_to_edge":
                inside = inside | (x == -1) | (y == h)
            idx = torch.arange(B).view(B, 1, 1, 1) * (h * w) + y.clamp(0, h - 1) * w + x.clamp(0, w - 1)
            g_hi = hi2.reshape(-1, 32)[idx] * inside[..., None]
            ref_hi = hi1[:, None]
            if terms == 1:
                st = (g_hi * r[:, None]).sum(-1).half().float()
            else:
                g_lo = lo2.reshape(-1, 32)[idx] * inside[..., None]
                st = (g_hi * ref_hi).sum(-1) + (g_hi * lo1[:, None]).sum(-1)
                if defect != "drop_lo_hi":
                    st = st + (g_lo * ref_hi).sum(-1)
            s.append(st)
        v = s[3] * (fx * fy) + s[2] * (gx * fy) + s[1] * (fx * gy) + s[0] * (gx * gy)
        if terms == 3:
            v = v * (1.0 / 32)
        if defect == "chunk_dropped" and m == M - 1:
            v[:, PLANES] = 0
        if defect == "chunk_twice" and m == 0:
            v[:, PLANES] *= 2
        acc = acc + v
    out = acc / (M - 1 if defect == "divide_by_M_minus_1" else M)
    return out.permute(0, 2, 3, 1)


def _reference(c, terms):
    hi1 = c["f1"].half()
    planes = lambda f: (f.half(), (f - f.half().float()).half())
    return R.sweep_reference("tc%d" % terms, c["pose1"], c["pose2s"], c["K"], 0.25, 20.0, c["D"], planes1=planes(c["f1"]),
                             planes2=[planes(f) for f in c["f2s"]])


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_honest_fp32_standin_passes(name, terms):
    c = _case(name)
    ref = _reference(c, terms)
    worst, acc, tight = R.check_sweep("stand-in %s terms=%d" % (name, terms), standin(c, terms), ref)
    print("stand-in %s terms=%d: err/bound %.3f, err/(u n S) %.3f, median bound/sum w|s| %.2e, ill-conditioned %d" % (
        name, terms, worst, acc, tight, ref.n_ill))


DEFECTS = {  # defect -> terms it is planted at (on the "moderate" case)
    "tap_one_over_at_tile_edge": 1,
    "clamp_to_edge": 1,
    "no_shrink": 1,
    "chunk_dropped": 1,
    "chunk_twice": 3,
    "d0_off_by_one": 1,
    "drop_lo_hi": 3,
    "divide_by_M_minus_1": 1,
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_planted_defect_is_rejected(defect):
    c = _case("moderate")
    terms = DEFECTS[defect]
    with pytest.raises(AssertionError, match="exceeds the bound"):
        R.check_sweep("stand-in with %s" % defect, standin(c, terms, defect), _reference(c, terms))
