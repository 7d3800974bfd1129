"""hidden_warp_kernel, hidden_warp_backward_kernel and depth_reproject_kernel against the fp64 reference of
tests/geometry_reference.py, element by element.  Each case first asserts, from its fp64 geometry, the situations it is there to
reach.  Prints the worst err / bound of every case and the ill-conditioned / ambiguous counts."""

import numpy as np
import pytest
import torch

from tests import geometry_reference as G

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)


def _warp_reach_all():
    reached = {}
    for name in G.WARP_CASES:
        _, depth, prev, cur, K, thresh = G.warp_case(name)
        for k, v in G.warp_reach(G.WarpGeometry(depth, prev, cur, K, thresh)).items():
            reached[k] = reached.get(k, False) or v
    return reached


def test_warp_cases_reach_every_edge():
    r = _warp_reach_all()
    assert all(r.values()), r
    _, depth, prev, _, _, thresh = G.warp_case("threshold_and_nan_depth")
    d = depth.reshape(-1)
    assert d[0] == np.float32(thresh) and d[1] == np.nextafter(np.float32(thresh), np.float32(1)) and np.isnan(d).any()
    B, C, h, w = G.WARP_CASES["c4_partial_last_cta"][:4]
    assert C == 4 and (h * w * C // 4) % 128 != 0 and (h * w * C // 4) // 128 >= 2
    assert G.warp_case("raw_transform_z_signs")[2] is None and G.warp_case("raw_transform_z_signs")[5] == float("-inf")
    _, _, prev, cur, _, _ = G.warp_case("batch3_distinct_poses")
    T = G.transforms(prev, cur)[0]
    assert np.abs(T[1] - T[0]).max() > 1e-2 and np.abs(T[2] - T[0]).max() > 1e-2


@pytest.mark.parametrize("name", list(G.WARP_CASES))
def test_hidden_warp_vs_fp64_reference(name):
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    h_in, depth, prev, cur, K, thresh = G.warp_case(name)
    with torch.no_grad():
        out = ops.hidden_warp(_t(h_in), _t(depth), _t(prev), _t(cur), _t(K), thresh)
        B, h, w, C = h_in.shape
        g = np.random.RandomState(9).randn(*h_in.shape).astype(np.float32)
        gt, d, K_, cur_ = _t(g), _t(depth), _t(K), _t(cur)
        prev_ = _t(prev)
        gin = torch.empty_like(gt)
        N.check(N.lib().dvmvs_hidden_warp_backward(gt.data_ptr(), d.data_ptr(), prev_.data_ptr() if prev_ is not None else None, cur_.data_ptr(),
                                                   K_.data_ptr(), gin.data_ptr(), B, C, h, w, float(thresh), ops._stream()), "hidden_warp_backward")
        torch.cuda.synchronize()
    ref = G.warp_reference(h_in, depth, prev, cur, K, thresh)
    worst = G.check_warp("hidden_warp " + name, out.cpu().numpy(), ref)
    bref = G.warp_backward_reference(g, depth, prev, cur, K, thresh)
    bworst = G.check_warp("hidden_warp_backward " + name, gin.cpu().numpy(), bref, backward=True)
    geo = ref.geo
    print("\nhidden_warp %-26s err/bound %.3f  backward err/bound %.3f  live %d  exact +0 %d  ill-conditioned %d"
          % (name, worst, bworst, int(geo.live.sum()), int(geo.zero.sum()), int(geo.ill.sum())))


def test_reproject_cases_reach_every_edge(synth):
    reach = {G.REPROJECT_CASES[n][3]: G.reproject_reach(G.reproject_reference(*G.reproject_case(n, synth))) for n in G.REPROJECT_CASES}
    assert reach["forward"]["max_sources"] >= 16, reach["forward"]
    assert reach["behind"]["behind_inside"] > 0
    assert any(r["last_col"] for r in reach.values()) and any(r["last_row"] for r in reach.values())
    B, H, W = G.REPROJECT_CASES["odd_half_size_depth_zeros"][:3]
    assert (H // 2) % 2 == 1 and (W // 2) % 2 == 1
    cur, prev = G.reproject_case("batch2_distinct_poses")[:2]
    T = G.transforms(cur, prev)[0]
    assert np.abs(T[1] - T[0]).max() > 1e-2


@pytest.mark.parametrize("name", list(G.REPROJECT_CASES))
def test_depth_reproject_vs_fp64_reference(name, synth):
    from dvmvs import _ops as ops
    cur, prev, depth, fK, hK, H, W = G.reproject_case(name, synth)
    with torch.no_grad():
        out = ops.depth_reproject(_t(cur), _t(prev), _t(depth), _t(fK), _t(hK), H, W)
        torch.cuda.synchronize()
    ref = G.reproject_reference(cur, prev, depth, fK, hK, H, W)
    n = G.check_reproject("depth_reproject " + name, out.cpu().numpy(), ref)
    print("\ndepth_reproject %-28s targets with a sure source %d  ambiguous sources %d (near the 1e-8 branch %d)  behind the camera %d"
          % (name, n, ref.n_amb, ref.n_zamb, ref.n_behind))
