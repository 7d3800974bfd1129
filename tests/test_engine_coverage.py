"""Every native entry point bench.py's default engine launches is covered by an fp64 reference test, and the fp32 CUDA-core, staging
and geometry calls of the engine pass those references on the engine's own buffers.

ENTRY_TESTS maps each dvmvs_* entry point (and each branch of dvmvs_conv2d) to the test that checks it against fp64; an entry point
the engine starts launching without one fails test_engine_entry_points_are_covered."""
import importlib

import numpy as np
import pytest
import torch

from tests import fp32_reference as R
from tests import geometry_reference as G
from tests.tc_reference import check
from tests.test_fp32_reference import check_blocked_staging, conv_chain, launched_conv_branch

pytestmark = pytest.mark.gpu

_REPLAY = "tests.test_engine_coverage::test_engine_calls_replayed_vs_fp64_reference"
ENTRY_TESTS = {
    "dvmvs_conv2d_tc": "tests.test_tc_reference::test_every_benchmark_layer_vs_fp64_reference",
    "dvmvs_conv2d_halo": "tests.test_tc_reference::test_every_benchmark_layer_vs_fp64_reference",
    "dvmvs_expand_dwconv": "tests.test_tc_reference::test_every_benchmark_layer_vs_fp64_reference",
    "dvmvs_lstm_gates_parts": "tests.test_tc_reference::test_every_benchmark_layer_vs_fp64_reference",
    "dvmvs_lstm_gates": "tests.test_tc_reference::test_lstm_gates_every_instantiation",
    "dvmvs_plane_sweep_tc": "tests.test_sweep_reference::test_sweep_of_the_benchmarked_engine_vs_fp64_reference",
    "dvmvs_stem_conv": _REPLAY,
    "dvmvs_dwconv2d": _REPLAY,
    "dvmvs_split_planes": _REPLAY,
    "dvmvs_split_blocked": _REPLAY,
    "dvmvs_upsample2x": _REPLAY,
    "dvmvs_hidden_warp": _REPLAY,
    "dvmvs_depth_reproject": _REPLAY,
    "dvmvs_conv2d": _REPLAY,
    "dvmvs_conv2d head8": _REPLAY,
    "dvmvs_conv2d head32": _REPLAY,
    "dvmvs_nchw_to_nhwc": "tests.test_fp32_reference::test_layout_transposes_exact",
    "dvmvs_nhwc_to_nchw": "tests.test_fp32_reference::test_layout_transposes_exact",
}
for _k in (1, 3, 5):
    for _s in (1, 2):
        for _split in ("", " split"):
            ENTRY_TESTS["dvmvs_conv2d direct %d/%d%s" % (_k, _s, _split)] = _REPLAY
HOST_ONLY = {"dvmvs_conv2d_tc_ksplit", "dvmvs_kernel_launch_count", "dvmvs_last_error_string", "dvmvs_abi_version",
             "dvmvs_set_programmatic_launch"}      # queries and switches: they launch no kernel

OPS_REPLAYED = ("stem_conv", "dwconv2d", "split_planes", "concat_planes", "split_blocked", "conv2d", "upsample2x", "hidden_warp", "depth_reproject")


@pytest.fixture(autouse=True)
def _restore_backend():
    """recording primes bench.py's engine, which selects the 1-term tensor-core backend: the tests after these keep theirs"""
    from dvmvs import _ops
    old = (_ops._BACKEND, _ops._TC_TERMS_BASE, _ops._TC_STRIDE2)
    try:
        yield
    finally:
        _ops.set_conv_backend(old[0], terms=old[1], stride2=old[2])


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def uncovered(recorded):
    """the recorded entry points (and dvmvs_conv2d branches) that ENTRY_TESTS does not map to a test"""
    return sorted(k for k in recorded if k not in ENTRY_TESTS and k not in HOST_ONLY)


def test_coverage_map_names_existing_tests():
    for entry, test in ENTRY_TESTS.items():
        mod, fn = test.split("::")
        assert callable(getattr(importlib.import_module(mod), fn, None)), "%s: %s does not exist" % (entry, test)


def test_engine_entry_points_are_covered():
    from tools.engine_record import engine_calls
    native = {}
    engine_calls((), height=256, width=256, native=native)
    print()
    for k in sorted(native):
        print("%-40s x%-4d %s" % (k, native[k], ENTRY_TESTS.get(k, "host only" if k in HOST_ONLY else "NOT COVERED")))
    assert not uncovered(native), "the 256x256 engine launches entry points no fp64 test covers: %s" % uncovered(native)
    for must in ("dvmvs_stem_conv", "dvmvs_split_blocked", "dvmvs_hidden_warp", "dvmvs_depth_reproject", "dvmvs_conv2d", "dvmvs_conv2d_tc"):
        assert must in native, "the engine no longer calls %s: update ENTRY_TESTS and this list" % must
    dropped = dict(ENTRY_TESTS)
    dropped.pop("dvmvs_stem_conv")           # the check is not vacuous: an entry point missing from the map is reported
    assert [k for k in native if k not in dropped and k not in HOST_ONLY] == ["dvmvs_stem_conv"]


# ------------------------------------------------------------------------------------------------ replays
def _np(t):
    return None if t is None else t.detach().float().cpu().numpy()


def _check_warp(what, args, prev=None, cur=None):
    from dvmvs import _ops as ops
    h, depth, p, c, K, thresh = args
    if prev is not None:
        p, c = prev, cur
    with torch.no_grad():
        out = ops.hidden_warp(h, depth, p, c, K, thresh)
        torch.cuda.synchronize()
    B, hh, ww, _ = h.shape
    ref = G.warp_reference(_np(h), _np(depth).reshape(B, hh, ww), _np(p), _np(c), _np(K), thresh)
    return G.check_warp(what, out.cpu().numpy(), ref), int(ref.geo.ill.sum())


def _check_reproject(what, args, prev=None, cur=None):
    from dvmvs import _ops as ops
    c, p, depth, fK, hK, H, W = args
    if prev is not None:
        p, c = prev, cur
    with torch.no_grad():
        out = ops.depth_reproject(c, p, depth, fK, hK, H, W)
        torch.cuda.synchronize()
    ref = G.reproject_reference(_np(c), _np(p), _np(depth), _np(fK), _np(hK), H, W)
    G.check_reproject(what, out.cpu().numpy(), ref)
    return ref.n_amb


def _replay(name, a, kw):
    """one recorded call, rerun on its buffers and checked; returns (what, worst err / bound or None, note)"""
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    if name == "stem_conv":
        image, pc = a
        with torch.no_grad():
            y = ops.stem_conv(image, pc)
            torch.cuda.synchronize()
        ref = R.stem_reference(image, pc.weight, pc.bias)
        return check("stem", _nchw(y), ref.y, ref.bound)[0], ""
    if name == "dwconv2d":
        x, pd = a[0], a[1]
        planes = x.shape[3] % 8 == 0
        with torch.no_grad():
            r = ops.dwconv2d(x, pd, want_f32=True, want_planes=planes)
            torch.cuda.synchronize()
        y, p = r if planes else (r, None)
        ref = R.dwconv_reference(_nchw(x), pd.weight, pd.bias, pd.stride, pd.act)
        if p is not None:
            eh, el = R.split_expected(y)
            assert torch.equal(p[0].view(torch.int16), eh.view(torch.int16)) and torch.equal(p[1].view(torch.int16), el.view(torch.int16))
        return check("dwconv", _nchw(y), ref.y, ref.bound)[0], ""
    if name == "split_planes":
        x, up = a[0], (a[1] if len(a) > 1 else kw.get("upsample", False))
        with torch.no_grad():
            planes = ops.split_planes(x, upsample=up)
            torch.cuda.synchronize()
        R.check_staged("split_planes", planes[0], planes[1], ops.upsample2x(x) if up else x, 0, planes.shape[-1], None, others=False)
        return None, "bit-exact"
    if name == "concat_planes":
        (sources,) = a
        with torch.no_grad():
            planes = ops.concat_planes(sources)
            torch.cuda.synchronize()
        off = 0
        for i, (t, up) in enumerate(sources):
            cover = t.shape[3] if i + 1 < len(sources) else planes.shape[-1] - off
            R.check_staged("concat_planes source %d" % i, planes[0], planes[1], ops.upsample2x(t) if up else t, off, cover, None, others=False)
            off += t.shape[3]
        return None, "bit-exact"
    if name == "split_blocked":
        sources = a[0]
        with torch.no_grad():
            buf = ops.split_blocked(*a, **kw)
            torch.cuda.synchronize()
        check_blocked_staging("split_blocked", buf, sources, kw.get("only"))
        return None, "bit-exact"
    if name == "upsample2x":
        (x,) = a
        with torch.no_grad():
            y = ops.upsample2x(x)
            torch.cuda.synchronize()
        ref, bound = R.upsample_reference(_nchw(x))
        return check("upsample2x", _nchw(y), ref, bound)[0], ""
    if name == "conv2d":
        sources, pc = a
        res, res_mode, aux = kw.get("residual"), kw.get("residual_mode", N.RES_NONE), kw.get("aux")
        branch, r = launched_conv_branch(lambda: ops.conv2d(sources, pc, residual=res, residual_mode=res_mode, aux=aux))
        out, aux_out = r if aux is not None else (r, None)
        chain = conv_chain(branch, pc.cin, [t.shape[3] for t, _ in sources], pc.ksize)
        ref = R.conv_reference([(_nchw(t), m == N.SRC_UPSAMPLE2X) for t, m in sources], pc.weight, pc.stride, pc.bias,
                               None if res is None else _nchw(res), res_mode, pc.act, aux, chain=chain)
        worst = check("conv2d", _nchw(out), ref.y, ref.bound)[0]
        if aux is not None:
            worst = max(worst, check("conv2d aux", _nchw(aux_out), ref.aux, ref.aux_bound)[0])
        return worst, branch
    if name == "hidden_warp":
        worst, ill = _check_warp("hidden_warp", a)
        return worst, "ill-conditioned %d" % ill
    if name == "depth_reproject":
        return None, "ambiguous sources %d" % _check_reproject("depth_reproject", a)
    raise AssertionError("no replay for %s" % name)


@pytest.mark.parametrize("height,width", [(256, 256), (320, 256)])
def test_engine_calls_replayed_vs_fp64_reference(height, width, synth):
    """Records every stem, depthwise, staging, dvmvs_conv2d (depth head), upsampling, hidden-warp and re-projection call of the engine
    while it primes at this size and replays each on its buffers against the fp64 reference; the warp and the re-projection once
    more with the poses of the clip's keyframes 0 -> 1 (priming repeats one frame: the recorded poses are an identity motion)."""
    from tools.engine_record import engine_calls
    mods, calls = engine_calls(OPS_REPLAYED, height=height, width=width)
    seen = {}
    print()
    for key, (args, kw, lay, on_rec) in calls.items():
        name = key[0]
        try:
            worst, note = _replay(name, args, kw)
        except AssertionError as e:
            raise AssertionError("%s call %s: %s" % (name, key[1:], e)) from None
        seen[name] = seen.get(name, 0) + 1
        print("%-16s %-60s %s %s" % (name, str(key[1:])[:60], "err/bound %.3f" % worst if worst is not None else "", note))
    clip = synth.make_clip(0, 2, height, width, 1)
    p0, p1 = (torch.from_numpy(np.ascontiguousarray(clip["poses"][i], dtype=np.float32))[None].cuda() for i in (0, 1))
    for key, (args, kw, _, _) in calls.items():
        if key[0] in ("hidden_warp", "depth_reproject"):
            B = args[0].shape[0]
        if key[0] == "hidden_warp":
            worst, ill = _check_warp("hidden_warp keyframes 0->1", args, prev=p0.expand(B, 4, 4).contiguous(), cur=p1.expand(B, 4, 4).contiguous())
            print("hidden_warp keyframes 0->1  err/bound %.3f  ill-conditioned %d" % (worst, ill))
        elif key[0] == "depth_reproject":
            n = _check_reproject("depth_reproject keyframes 0->1", args, prev=p0.expand(B, 4, 4).contiguous(), cur=p1.expand(B, 4, 4).contiguous())
            print("depth_reproject keyframes 0->1  ambiguous sources %d" % n)
    print("%dx%d replayed: %s" % (height, width, seen))
    for must in ("stem_conv", "split_blocked", "conv2d", "hidden_warp", "depth_reproject"):
        assert seen.get(must), "the engine made no %s call at %dx%d" % (must, height, width)
