"""Every native entry point bench.py's default engine launches is covered by an fp64 reference test, and the fp32 CUDA-core, staging
and geometry calls of the engine pass those references on the engine's own buffers; the same at the lookahead engine
configurations of tools/engine_record.py's ENGINE_POINTS.

ENTRY_TESTS maps each dvmvs_* entry point (and each branch of dvmvs_conv2d) to the test that checks it against fp64; an entry point
the engine starts launching without one fails test_engine_entry_points_are_covered.  An entry point mapped to the replay test below
counts as covered at an operating point of bench.py only if that point's replay reaches it.  The tests named here run over
bench.py's points; ENGINE_POINT_TESTS names their counterparts over ENGINE_POINTS, which run the same replay code."""
import importlib

import numpy as np
import pytest
import torch

from tests import fp32_reference as R
from tests import geometry_reference as G
from tests.tc_reference import check, check_live
from tests.test_fp32_reference import check_blocked_staging, conv_chain
from tools.engine_record import branch_of

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
# the direct-convolution branches tests/test_fp32_reference.py's CONV_CASES reach (test_unit_direct_branches_are_reached checks it);
# the engine's other branches are covered where the replay of an operating point reaches them
_CONV_UNIT = "tests.test_fp32_reference::test_conv2d_vs_fp64_reference"
UNIT_DIRECT = {"direct 1/1", "direct 1/1 split", "direct 3/1", "direct 3/1 split", "direct 3/2", "direct 5/1 split", "direct 5/2"}
for _k in (1, 3, 5):
    for _s in (1, 2):
        for _split in ("", " split"):
            _b = "direct %d/%d%s" % (_k, _s, _split)
            ENTRY_TESTS["dvmvs_conv2d " + _b] = _CONV_UNIT if _b in UNIT_DIRECT else _REPLAY
HOST_ONLY = {"dvmvs_conv2d_tc_ksplit", "dvmvs_kernel_launch_count", "dvmvs_last_error_string", "dvmvs_abi_version",
             "dvmvs_set_programmatic_launch"}      # queries and switches: they launch no kernel
ENGINE_POINT_TESTS = {
    "tests.test_tc_reference::test_every_benchmark_layer_vs_fp64_reference": "tests.test_tc_reference::test_every_engine_point_layer_vs_fp64_reference",
    "tests.test_sweep_reference::test_sweep_of_the_benchmarked_engine_vs_fp64_reference":
        "tests.test_sweep_reference::test_sweep_of_each_engine_point_vs_fp64_reference",
    _REPLAY: "tests.test_engine_coverage::test_engine_point_calls_replayed_vs_fp64_reference",
}
# what only fusionnet's recurrent stage launches (hidden-state warp, depth re-projection, ConvLSTM gates): pairnet launches none of it
RECURRENT_ENTRY_POINTS = ("dvmvs_hidden_warp", "dvmvs_depth_reproject", "dvmvs_lstm_gates", "dvmvs_lstm_gates_parts")

OPS_REPLAYED = ("stem_conv", "dwconv2d", "split_planes", "concat_planes", "split_blocked", "conv2d", "upsample2x", "hidden_warp", "depth_reproject")
OP_ENTRY = {"stem_conv": "dvmvs_stem_conv", "dwconv2d": "dvmvs_dwconv2d", "split_planes": "dvmvs_split_planes", "concat_planes": "dvmvs_split_planes",
            "split_blocked": "dvmvs_split_blocked", "conv2d": "dvmvs_conv2d", "upsample2x": "dvmvs_upsample2x", "hidden_warp": "dvmvs_hidden_warp",
            "depth_reproject": "dvmvs_depth_reproject"}


def _point_params(with_sizes=()):
    """bench.py's operating points (tools/engine_record.py POINTS); the headline keeps its historical id (its input size), and
    with_sizes adds it at other input sizes"""
    from tools.engine_record import POINTS
    return ([pytest.param("value", None, None, id="256-256")] + [pytest.param("value", h, w, id="%d-%d" % (h, w)) for h, w in with_sizes] +
            [pytest.param(p, None, None, id=p) for p in POINTS if p != "value"])


def _engine_point_params():
    from tools.engine_record import ENGINE_POINTS
    return list(ENGINE_POINTS)


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
    for entry, test in list(ENTRY_TESTS.items()) + list(ENGINE_POINT_TESTS.items()):
        mod, fn = test.split("::")
        assert callable(getattr(importlib.import_module(mod), fn, None)), "%s: %s does not exist" % (entry, test)
    assert set(ENGINE_POINT_TESTS) <= set(ENTRY_TESTS.values())


def test_unit_direct_branches_are_reached():
    """UNIT_DIRECT is what tests/test_fp32_reference.py's CONV_CASES reach, no more"""
    from tests.test_fp32_reference import CONV_CASES, _path
    reached = set()
    for c in CONV_CASES:
        path, ksplit = _path(c)
        if path == "direct":
            reached.add("direct %d/%d%s" % (c[6], c[7], " split" if ksplit > 1 else ""))
    assert reached == UNIT_DIRECT, sorted(reached ^ UNIT_DIRECT)


def replayed_entry_points(calls):
    """the entry points, and dvmvs_conv2d branches, that test_engine_calls_replayed_vs_fp64_reference reaches when it replays
    these recorded calls (each dvmvs_conv2d call is run once more to read its branch)"""
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    reached = set()
    for key, (a, kw, _, _) in calls.items():
        reached.add(OP_ENTRY[key[0]])
        if key[0] == "conv2d":
            sources, pc = a
            branch, _ = branch_of(lambda: ops.conv2d(sources, pc, residual=kw.get("residual"), residual_mode=kw.get("residual_mode", N.RES_NONE),
                                                     aux=kw.get("aux")))
            reached.add("dvmvs_conv2d " + branch)
    return reached


def uncovered_at(native, reached, tests=None):
    """the launched entry points / branches that are neither mapped to a unit test nor reached by the replay at this point"""
    tests = ENTRY_TESTS if tests is None else tests
    return sorted(k for k in native if k not in HOST_ONLY and (k not in tests or (tests[k] == _REPLAY and k not in reached)))


def _each_point(check):
    """runs check(point) for every operating point of bench.py (tools/engine_record.py POINTS) and reports every point that fails"""
    from tools.engine_record import POINTS
    failed = {}
    for point in POINTS:
        try:
            check(point)
        except AssertionError as e:
            failed[point] = str(e)
        torch.cuda.empty_cache()
    assert not failed, "\n".join("%s: %s" % kv for kv in failed.items())


def test_engine_entry_points_are_covered():
    """at every operating point bench.py reports: every native entry point (and dvmvs_conv2d branch) the point's engine launches is
    mapped to an fp64 test, and one mapped to the replay test is reached by that point's replay"""
    _each_point(_entry_points_at)


@pytest.mark.parametrize("point", _engine_point_params())
def test_engine_point_entry_points_are_covered(point):
    """test_engine_entry_points_are_covered at a lookahead engine configuration of tools/engine_record.py's ENGINE_POINTS"""
    _entry_points_at(point)
    torch.cuda.empty_cache()


def _entry_points_at(point):
    from tools.engine_record import ENGINE_POINTS, engine_calls
    print("\n" + point)
    native = {}
    mods, calls = engine_calls(OPS_REPLAYED, point=point, native=native)
    reached = replayed_entry_points(calls)
    for k in sorted(native):
        test = ENTRY_TESTS.get(k, "host only" if k in HOST_ONLY else "NOT COVERED")
        if point in ENGINE_POINTS:
            test = ENGINE_POINT_TESTS.get(test, test)
        replay = test in (_REPLAY, ENGINE_POINT_TESTS[_REPLAY])
        print("%-40s x%-5d %s%s" % (k, native[k], test, " (NOT REPLAYED HERE)" if replay and k not in reached else ""))
    assert not uncovered(native), "%s: the engine launches entry points no fp64 test covers: %s" % (point, uncovered(native))
    assert not uncovered_at(native, reached), "%s: launched, mapped to the replay, but not replayed at this point: %s" % (point, uncovered_at(native, reached))
    recurrent = "lstm" in mods
    for must in ("dvmvs_stem_conv", "dvmvs_split_blocked", "dvmvs_conv2d", "dvmvs_conv2d_tc") + (
            ("dvmvs_hidden_warp", "dvmvs_depth_reproject") if recurrent else ()):
        assert must in native, "%s: the engine no longer calls %s: update ENTRY_TESTS and this list" % (point, must)
    if not recurrent:
        launched = [k for k in RECURRENT_ENTRY_POINTS if k in native]
        assert not launched, "%s: pairnet launches recurrent-stage entry points %s" % (point, launched)
    dropped = dict(ENTRY_TESTS)
    dropped.pop("dvmvs_stem_conv")           # the check is not vacuous: an entry point missing from the map is reported
    assert [k for k in native if k not in dropped and k not in HOST_ONLY] == ["dvmvs_stem_conv"]
    heads = [k for k in native if k.startswith("dvmvs_conv2d head")]
    assert heads and uncovered_at(native, reached - {heads[0]}) == [heads[0]]      # nor is the replay check


# ------------------------------------------------------------------------------------------------ replays
def _np(t):
    return None if t is None else t.detach().float().cpu().numpy()


def _at(t, rows):
    return t.index_select(0, rows)


def _check_warp(what, args, rows, prev=None, cur=None):
    from dvmvs import _ops as ops
    h, depth, p, c, K, thresh = args
    if prev is not None:
        p, c = prev, cur
    check_live(what, _at(h, rows), _at(depth, rows))
    with torch.no_grad():
        out = ops.hidden_warp(h, depth, p, c, K, thresh)
        torch.cuda.synchronize()
    _, hh, ww, _ = h.shape
    ref = G.warp_reference(_np(_at(h, rows)), _np(_at(depth, rows)).reshape(len(rows), hh, ww), _np(_at(p, rows)), _np(_at(c, rows)),
                           _np(_at(K, rows)), thresh)
    return G.check_warp(what, _at(out, rows).cpu().numpy(), ref), int(ref.geo.ill.sum())


def _check_reproject(what, args, rows, prev=None, cur=None):
    from dvmvs import _ops as ops
    c, p, depth, fK, hK, H, W = args
    if prev is not None:
        p, c = prev, cur
    check_live(what, _at(depth, rows))
    with torch.no_grad():
        out = ops.depth_reproject(c, p, depth, fK, hK, H, W)
        torch.cuda.synchronize()
    ref = G.reproject_reference(_np(_at(c, rows)), _np(_at(p, rows)), _np(_at(depth, rows)), _np(_at(fK, rows)), _np(_at(hK, rows)), H, W)
    G.check_reproject(what, _at(out, rows).cpu().numpy(), ref)
    return ref.n_amb


def _replay(name, a, kw, rows):
    """one recorded call, rerun on its buffers and checked on the batch rows `rows`; returns (worst err / bound or None, note)"""
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    if name == "stem_conv":
        image, pc = a
        check_live("stem", _at(image, rows))
        with torch.no_grad():
            y = ops.stem_conv(image, pc)
            torch.cuda.synchronize()
        ref = R.stem_reference(_at(image, rows), pc.weight, pc.bias)
        return check("stem", _nchw(_at(y, rows)), ref.y, ref.bound)[0], ""
    if name == "dwconv2d":
        x, pd = a[0], a[1]
        check_live("dwconv", _at(x, rows))
        planes = x.shape[3] % 8 == 0
        with torch.no_grad():
            r = ops.dwconv2d(x, pd, want_f32=True, want_planes=planes)
            torch.cuda.synchronize()
        y, p = r if planes else (r, None)
        ref = R.dwconv_reference(_nchw(_at(x, rows)), pd.weight, pd.bias, pd.stride, pd.act)
        if p is not None:
            eh, el = R.split_expected(y)
            assert torch.equal(p[0].view(torch.int16), eh.view(torch.int16)) and torch.equal(p[1].view(torch.int16), el.view(torch.int16))
        return check("dwconv", _nchw(_at(y, rows)), ref.y, ref.bound)[0], ""
    if name == "split_planes":
        x, up = a[0], (a[1] if len(a) > 1 else kw.get("upsample", False))
        check_live("split_planes", x)
        with torch.no_grad():
            planes = ops.split_planes(x, upsample=up)
            torch.cuda.synchronize()
        R.check_staged("split_planes", planes[0], planes[1], ops.upsample2x(x) if up else x, 0, planes.shape[-1], None, others=False)
        return None, "bit-exact"
    if name == "concat_planes":
        (sources,) = a
        check_live("concat_planes", *[t for t, _ in sources])
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
        check_live("split_blocked", *[t for i, (t, _) in enumerate(sources) if torch.is_tensor(t) and (kw.get("only") is None or i in kw["only"])])
        with torch.no_grad():
            buf = ops.split_blocked(*a, **kw)
            torch.cuda.synchronize()
        check_blocked_staging("split_blocked", buf, sources, kw.get("only"))
        return None, "bit-exact"
    if name == "upsample2x":
        (x,) = a
        check_live("upsample2x", _at(x, rows))
        with torch.no_grad():
            y = ops.upsample2x(x)
            torch.cuda.synchronize()
        ref, bound = R.upsample_reference(_nchw(_at(x, rows)))
        return check("upsample2x", _nchw(_at(y, rows)), ref, bound)[0], ""
    if name == "conv2d":
        sources, pc = a
        check_live("conv2d", *[_at(t, rows) for t, _ in sources])
        res, res_mode, aux = kw.get("residual"), kw.get("residual_mode", N.RES_NONE), kw.get("aux")
        with torch.no_grad():
            branch, r = branch_of(lambda: ops.conv2d(sources, pc, residual=res, residual_mode=res_mode, aux=aux))
        out, aux_out = r if aux is not None else (r, None)
        chain = conv_chain(branch, pc.cin, [t.shape[3] for t, _ in sources], pc.ksize)
        ref = R.conv_reference([(_nchw(_at(t, rows)), m == N.SRC_UPSAMPLE2X) for t, m in sources], pc.weight, pc.stride, pc.bias,
                               None if res is None else _nchw(_at(res, rows)), res_mode, pc.act, aux, chain=chain)
        worst = check("conv2d", _nchw(_at(out, rows)), ref.y, ref.bound)[0]
        if aux is not None:
            worst = max(worst, check("conv2d aux", _nchw(_at(aux_out, rows)), ref.aux, ref.aux_bound)[0])
        return worst, branch
    if name == "hidden_warp":
        worst, ill = _check_warp("hidden_warp", a, rows)
        return worst, "ill-conditioned %d" % ill
    if name == "depth_reproject":
        return None, "ambiguous sources %d" % _check_reproject("depth_reproject", a, rows)
    raise AssertionError("no replay for %s" % name)


def _row_motion(synth, B):
    """per-row (previous, current) poses: row b moves from frame b to frame b + 1 + b % 3 of the synthetic trajectory, so that every
    row has its own motion (the synthetic clips share one trajectory: their keyframe 0 -> 1 poses are the same in every row)"""
    pose = lambda i: torch.from_numpy(np.ascontiguousarray(synth.camera_pose(i), dtype=np.float32))
    prev = torch.stack([pose(b) for b in range(B)]).cuda()
    cur = torch.stack([pose(b + 1 + b % 3) for b in range(B)]).cuda()
    rel = torch.linalg.inv(prev) @ cur
    assert B == 1 or not torch.equal(rel[0], rel[1]), "rows share one motion"
    return prev, cur


def _replay_engine_calls(point, synth, height=None, width=None):
    """Records every stem, depthwise, staging, dvmvs_conv2d (depth head), upsampling, hidden-warp and re-projection call of the
    engine of this operating point (tools/engine_record.py POINTS or ENGINE_POINTS), and replays each on its buffers against the
    fp64 reference, on the batch rows tools.engine_record.batch_rows picks; the warp and the re-projection once more with a
    different camera motion in every batch row (priming repeats one frame: the recorded poses are an identity motion).  One line
    per call.  Returns (cfg, calls replayed per op, stem batches, batches of the dvmvs_conv2d calls of the decoder's layers)."""
    from tools.engine_record import batch_rows, engine_calls, layer_names, point_config
    cfg = point_config(point, height, width)
    mods, calls = engine_calls(OPS_REPLAYED, point=point, height=height, width=width)
    names = layer_names(mods)
    seen, stem_batch, head_batch = {}, set(), set()
    print()
    for key, (args, kw, lay, on_rec) in calls.items():
        name = key[0]
        first = args[0][0][0] if name in ("concat_planes", "split_blocked", "conv2d") else args[0]
        B = first.shape[0] if torch.is_tensor(first) else first[0]          # split_blocked: a source not staged yet is its shape
        rows = torch.tensor(batch_rows(B), device="cuda")
        try:
            worst, note = _replay(name, args, kw, rows)
        except AssertionError as e:
            raise AssertionError("%s: %s call %s: %s" % (point, name, key[1:], e)) from None
        seen[name] = seen.get(name, 0) + 1
        if name == "stem_conv":
            stem_batch.add(B)
        if name == "conv2d" and names.get(id(lay), "").startswith("cvd"):
            head_batch.add(B)
        print("%-16s %-60s B=%-3d rows=%d %s %s" % (name, str(key[1:])[:60], B, len(rows), "err/bound %.3f" % worst if worst is not None else "", note))
    for key, (args, kw, _, _) in calls.items():
        if key[0] not in ("hidden_warp", "depth_reproject"):
            continue
        B = args[0].shape[0]
        rows = torch.tensor(batch_rows(B), device="cuda")
        prev, cur = _row_motion(synth, B)
        if key[0] == "hidden_warp":
            worst, ill = _check_warp("hidden_warp, a motion per row", args, rows, prev=prev, cur=cur)
            print("hidden_warp, a motion per row  B=%d err/bound %.3f  ill-conditioned %d" % (B, worst, ill))
        else:
            n = _check_reproject("depth_reproject, a motion per row", args, rows, prev=prev, cur=cur)
            print("depth_reproject, a motion per row  B=%d ambiguous sources %d" % (B, n))
    return cfg, seen, stem_batch, head_batch


@pytest.mark.parametrize("point,height,width", _point_params(with_sizes=[(320, 256)]))
def test_engine_calls_replayed_vs_fp64_reference(point, height, width, synth):
    """Every stem, depthwise, staging, dvmvs_conv2d (depth head), upsampling, hidden-warp and re-projection call of the engine
    bench.py runs at this operating point, replayed against the fp64 reference (_replay_engine_calls).  Checks the trunk batch of
    the point."""
    import time
    from tools.engine_record import trunk_batch
    t0 = time.perf_counter()
    cfg, seen, stem_batch, _ = _replay_engine_calls(point, synth, height, width)
    print("%s %dx%d B=%d: replayed %s; stem batch %s; %.1f s" % (point, cfg["height"], cfg["width"], cfg["batch"], seen, sorted(stem_batch),
                                                              time.perf_counter() - t0))
    for must in ("stem_conv", "split_blocked", "conv2d", "hidden_warp", "depth_reproject"):
        assert seen.get(must), "%s: the engine made no %s call" % (point, must)
    assert stem_batch == {trunk_batch(cfg)}, "%s: stem batch %s, expected %d" % (point, sorted(stem_batch), trunk_batch(cfg))


@pytest.mark.parametrize("point", _engine_point_params())
def test_engine_point_calls_replayed_vs_fp64_reference(point, synth):
    """test_engine_calls_replayed_vs_fp64_reference at a lookahead engine configuration of tools/engine_record.py's ENGINE_POINTS.
    Checks the trunk batches, the batch of the decoder's depth heads, and that pairnet runs no hidden warp or re-projection."""
    import time
    from tools.engine_record import decoder_batch, trunk_batches
    t0 = time.perf_counter()
    cfg, seen, stem_batch, head_batch = _replay_engine_calls(point, synth)
    print("%s %dx%d B=%d lookahead=%d cache=%d: replayed %s; stem batch %s; depth-head batch %s; %.1f s" % (
        point, cfg["height"], cfg["width"], cfg["batch"], cfg["lookahead"], cfg["feature_cache"], seen, sorted(stem_batch), sorted(head_batch),
        time.perf_counter() - t0))
    recurrent = ("hidden_warp", "depth_reproject")
    for must in ("stem_conv", "split_blocked", "conv2d") + (recurrent if cfg["engine"] != "pairnet" else ()):
        assert must in seen, "%s: the engine made no %s call" % (point, must)
    if cfg["engine"] == "pairnet":
        assert not set(recurrent) & set(seen), "%s: pairnet made recurrent-stage calls %s" % (point, seen)
    assert stem_batch == trunk_batches(cfg), "%s: stem batch %s, expected %s" % (point, sorted(stem_batch), sorted(trunk_batches(cfg)))
    assert head_batch == {decoder_batch(cfg)}, "%s: depth-head (cvd.*) batch %s, expected %d" % (point, sorted(head_batch), decoder_batch(cfg))
