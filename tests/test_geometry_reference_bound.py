"""The hidden-warp and re-projection bounds of tests/geometry_reference.py are honest and not vacuous (no GPU needed): an fp32
emulation of each kernel, operation for operation, passes the comparator on every case the GPU tests run; each planted defect
fails it.  Also measures the position and z constants the bounds charge (C_POS, C_ZR >= 8x the worst measured)."""
import numpy as np
import pytest

from tests import geometry_reference as G
from tests.tc_reference import U

# the cases each planted warp defect is run on: ones whose geometry reaches what the defect gets wrong
WARP_DEFECT_CASES = {
    "int_truncation": "c4_partial_last_cta",            # samples in (-1, 0)
    "batch0_transform": "batch3_distinct_poses",
    "mask_lt": "threshold_and_nan_depth",                # a depth exactly at fp32(0.01)
    "no_relu": "raw_transform_z_signs",                  # z < 0 inside the image
    "swap_xy_weights": "bench_landscape_8x10",
    "align_corners_false": "bench_256_8x8",
}


@pytest.mark.parametrize("name", list(G.WARP_CASES))
def test_warp_emulation_within_bound(name):
    h_in, depth, prev, cur, K, thresh = G.warp_case(name)
    ref = G.warp_reference(h_in, depth, prev, cur, K, thresh)
    worst = G.check_warp(name, G.emulate_warp(h_in, depth, prev, cur, K, thresh), ref)
    g = np.random.RandomState(9).randn(*h_in.shape).astype(np.float32)
    bref = G.warp_backward_reference(g, depth, prev, cur, K, thresh)
    bworst = G.check_warp(name + " backward", G.emulate_warp_backward(g, depth, prev, cur, K, thresh), bref, backward=True)
    print("%-26s emulation err/bound %.3f  backward %.3f  ill-conditioned %d" % (name, worst, bworst, int(ref.geo.ill.sum())))


def test_warp_position_constant():
    """the worst |fp32 position - fp64 position| of the emulation in units of u times the position magnitude: C_POS is >= 8x it"""
    worst = 0.0
    for name in G.WARP_CASES:
        h_in, depth, prev, cur, K, thresh = G.warp_case(name)
        geo = G.WarpGeometry(depth, prev, cur, K, thresh)
        xs, ys = G.emulate_warp_positions(depth, prev, cur, K)
        live = geo.live
        for got, ref, d in ((xs, geo.xs, geo.dx), (ys, geo.ys, geo.dy)):
            worst = max(worst, float((np.abs(got[live] - ref[live]) / (d[live] / G.C_POS)).max()))
    print("warp position: worst err / (u * magnitude) = %.3f (C_POS = %g)" % (worst, G.C_POS))
    assert worst * 8 <= G.C_POS


@pytest.mark.parametrize("defect", G.WARP_DEFECTS)
def test_warp_planted_defect_rejected(defect):
    name = WARP_DEFECT_CASES[defect]
    h_in, depth, prev, cur, K, thresh = G.warp_case(name)
    ref = G.warp_reference(h_in, depth, prev, cur, K, thresh)
    with pytest.raises(AssertionError):
        G.check_warp(name + " " + defect, G.emulate_warp(h_in, depth, prev, cur, K, thresh, variant=defect), ref)


@pytest.mark.parametrize("name", list(G.REPROJECT_CASES))
def test_reproject_emulation_within_bound(name, synth):
    args = G.reproject_case(name, synth)
    ref = G.reproject_reference(*args)
    G.check_reproject(name, G.emulate_reproject(*args), ref)
    print("%-28s ambiguous sources %d (near the 1e-8 branch %d), sure %d" % (name, ref.n_amb, ref.n_zamb, ref.n_sure))


def test_reproject_z_constant(synth):
    """the worst |fp32 z - fp64 z| of the emulation in units of u * P_z: C_ZR is >= 8x it"""
    worst = 0.0
    for name in G.REPROJECT_CASES:
        cur, prev, depth, fK, hK, H, W = G.reproject_case(name, synth)
        T, Tmag = G.transforms(cur, prev)
        p, P = G.camera_points(T, Tmag, depth.reshape(-1, H, W), fK)
        _, _, z, *_ = G._emulate_points(G.emulate_transform(cur, prev), depth.reshape(-1, H, W), fK)
        worst = max(worst, float((np.abs(z - p[:, 2]) / (U * P[:, 2])).max()))
    print("re-projection z: worst err / (u * P_z) = %.3f (C_ZR = %g)" % (worst, G.C_ZR))
    assert worst * 8 <= G.C_ZR


@pytest.mark.parametrize("defect", ["floor", "min", "bound_le"])
def test_reproject_planted_defect_rejected(defect, synth):
    case = {"floor": "batch2_distinct_poses", "min": "forward_motion", "bound_le": "batch2_distinct_poses"}[defect]
    args = G.reproject_case(case, synth)
    ref = G.reproject_reference(*args)
    with pytest.raises(AssertionError):
        G.check_reproject(case + " " + defect, G.emulate_reproject(*args, variant=defect), ref)


def test_reproject_relu_projection_is_unobservable(synth):
    """Projecting with the relu'd z moves only the sources with z < 0, and those carry zr = +0 -- the value of an unfilled target --
    so no output can tell the defect apart: the emulations agree bit for bit even where such sources land inside the image."""
    args = G.reproject_case("behind_camera", synth)
    ref = G.reproject_reference(*args)
    assert G.reproject_reach(ref)["behind_inside"] > 0
    a, b = G.emulate_reproject(*args), G.emulate_reproject(*args, variant="relu_projection")
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
