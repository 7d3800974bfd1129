"""LookaheadPairnet (dvmvs.pipeline): pairnet with every stage, the decoder included, batched over groups of keyframes.

- Against eager keyframe() on the same backend, and against the CPU oracle (oracle.pairnet_step) at c1 and at the c2 shape.
- Bit for bit against an eager replay of its own schedule, undelayed and with each of its streams delayed (the bounded
  torch.cuda._sleep helpers of test_engine_ordering.py); a planted skipped wait must change the delayed run.
- Row independence: a keyframe's depth does not depend on its position in the group, its neighbours, or whether flush()
  launched its group incomplete.
- The caller contract of submit() and depth_of(), the shipped pairnet weights on the fixture scene, constructor errors.
"""
import numpy as np
import pytest
import torch

from tests import helpers, scene_fixture
from tests.test_engine_ordering import (NAN, _Delay, _Skips, _assert_same, _calibrate, _diff, _frames, _late, _lookahead_script,
                                        _map, _run, _stage_graphs, _tc, _tensors, _under_delays)

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture
def delay(monkeypatch):
    return _Delay(monkeypatch)


@pytest.fixture
def skips(monkeypatch):
    return _Skips(monkeypatch)


def _pairnet_modules(oracle, synth, D, seed=11):
    w = helpers.oracle_weights(oracle, synth, seed, n_depth_levels=D)
    return helpers.build_product_modules(w, n_depth_levels=D, pairnet=True), w


def _engine(mods, B, H, W, M, D, T=3, G=2):
    from dvmvs import pipeline
    return pipeline.LookaheadPairnet(mods, batch=B, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, lookahead=T, n_groups=G)


def _replay(mods, frames, script, T, B, H, W, M, D):
    """What LookaheadPairnet.flush() runs, eagerly on the current stream and without graphs: per group the five stage bodies
    over one T*B batch holding the buffered keyframes' inputs, each keyframe's depth read from its rows.  Rows no keyframe
    filled hold the fresh buffers' inputs (the engine's hold an earlier keyframe's): rows are independent, which
    test_rows_are_independent checks on its own.  reset() and sync only end a group early through the script's layout."""
    from dvmvs import pipeline
    from dvmvs._base import no_auto_graph
    depths, buffered = [], []

    def flush():
        grp = pipeline._group_buffers(T, B, H, W, M, DEV)
        for j, k in enumerate(buffered):
            pipeline._upload(pipeline._keyframe_rows(grp, j, B), frames[k])
        for key, body in pipeline._pairnet_group_stages(mods, (0.25, 20.0, D)):
            grp[key] = body(grp)
        depths.extend(grp["depth"][j * B:(j + 1) * B].clone() for j in range(len(buffered)))
        buffered.clear()

    with no_auto_graph():
        for op in script:
            if op == "sync":
                if buffered:
                    flush()
            elif op != "reset":
                buffered.append(op)
                if len(buffered) == T:
                    flush()
        if buffered:
            flush()
    torch.cuda.synchronize()
    return depths


def _clip_args(clip, k):
    ref_i, meas_i = clip["frames"][k]
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)[None]
    return c(clip["images"][ref_i]), c(clip["poses"][ref_i]), [c(clip["images"][j]) for j in meas_i], [c(clip["poses"][j]) for j in meas_i], c(clip["K"])


# ------------------------------------------------------------------------------------------------ accuracy
# backend, terms, bound, B, (H, W, D, M), lookahead; the last one is c1 at pairnet_bench.py's largest group (8 clips x lookahead 8)
EAGER_CASES = [pytest.param(backend, terms, bound, B, (64, 96, 64, 2), 3, id="%s-%d-%g-%d" % (backend, terms, bound, B))
               for backend, terms, bound in [("fp32", 3, 1e-5), ("tc", 3, 1e-5), ("tc", 1, 1e-4)] for B in (1, 2)]
EAGER_CASES.append(pytest.param("tc", 1, 1e-4, 8, (128, 128, 32, 1), 8, id="c1-tc-1-0.0001-8-lookahead8"))


@pytest.mark.parametrize("backend,terms,bound,B,shape,T", EAGER_CASES)
def test_pairnet_engine_matches_eager_keyframe(oracle, synth, backend, terms, bound, B, shape, T):
    """Two synthetic clips back to back (7 + 4 keyframes in groups of T: the last group incomplete) against eager keyframe()
    with pairnet modules on the same backend: every keyframe's rows of the group read its own inputs and land in its own
    output.  Not bit for bit: the split-K choice of a few convolutions depends on the batch."""
    from dvmvs import _ops as ops
    from dvmvs import pipeline
    H, W, D, M = shape
    old = ops.conv_backend()
    ops.set_conv_backend(backend, terms=terms, stride2=True)
    try:
        with torch.no_grad():
            mods, _ = _pairnet_modules(oracle, synth, D)
            frames = _frames(synth, B, 7, H, W, M) + _frames_of_seed(synth, 20, B, 4, H, W, M)
            eng = _engine(mods, B, H, W, M, D, T=T)
            eng.prime(*frames[0])
            expected, got = [], []
            for i, f in enumerate(frames):
                if i == 7:
                    eng.reset()
                expected.append(pipeline.keyframe(mods, pipeline.KeyframeState(), *f, n_depth_levels=D)[0].clone())
                out = torch.empty((B, H, W), dtype=torch.float32, device=DEV)
                got.append((eng.submit(*f, out=out), out))
            eng.synchronize()
        assert B == 1 or not torch.equal(expected[-1][0], expected[-1][-1]), "the batch rows hold the same clip"
        errs = [float((o - e).abs().sum() / e.abs().sum()) for (_, o), e in zip(got, expected)]
        print("pairnet lookahead engine vs eager keyframe (%s, %d terms, B=%d, %dx%d D=%d M=%d, lookahead %d): rel-L1 per keyframe"
              % (backend, terms, B, H, W, D, M, T),
              ["%.1e" % e for e in errs])
        assert max(errs) <= bound, errs
        assert torch.equal(eng.depth_of(got[-1][0]), got[-1][1])
        assert eng.kernels_per_keyframe > 0
    finally:
        ops.set_conv_backend(old, terms=3)


def _frames_of_seed(synth, seed, B, n, H, W, M):
    """_frames with clips seed + c instead of 5 + c (a second clip sequence)."""
    clips = [synth.make_clip(seed + c, n, H, W, M) for c in range(B)]
    stack = lambda pick: torch.from_numpy(np.ascontiguousarray(np.stack([pick(c) for c in clips]))).to(DEV)
    out = []
    for t in range(n):
        ref = lambda c: c["frames"][t][0]
        meas = lambda c, m: c["frames"][t][1][m]
        out.append((stack(lambda c: c["images"][ref(c)]), stack(lambda c: c["poses"][ref(c)]),
                    [stack(lambda c: c["images"][meas(c, m)]) for m in range(M)],
                    [stack(lambda c: c["poses"][meas(c, m)]) for m in range(M)], stack(lambda c: c["K"])))
    return out


_ORACLE_GOLD = {}


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("point", ["c1", "c2"])
def test_pairnet_engine_vs_oracle(oracle, synth, point, terms):
    """BASELINE c1 (128x128, 32 planes, 1 measurement frame) and the c2 shape for pairnet (256x256, 64 planes, 2 measurement
    frames) through the engine on the tensor-core backend, 5 keyframes in groups of 2 (the last incomplete), against
    oracle.pairnet_step: the north-star budget, 1e-3 rel-L1 on inverse depth.  The tighter fusionnet bounds (TC_PRECISIONS
    of test_gpu_parity.py) were measured for fusionnet only and are not assumed here; the measured maxima are printed."""
    from dvmvs import _ops as ops
    H, W, D, M = (128, 128, 32, 1) if point == "c1" else (256, 256, 64, 2)
    n = 5
    T = torch.from_numpy
    old = ops.conv_backend()
    ops.set_conv_backend("tc", terms=terms, stride2=True)
    try:
        with torch.no_grad():
            mods, w = _pairnet_modules(oracle, synth, D, seed=7)
            clip = synth.make_clip(0, n, H, W, M)
            eng = _engine(mods, 1, H, W, M, D, T=2, G=2)
            eng.prime(*_clip_args(clip, 0))
            outs = []
            for k in range(n):
                out = torch.empty((1, H, W), dtype=torch.float32, device=DEV)
                eng.submit(*_clip_args(clip, k), out=out)
                outs.append(out)
            eng.synchronize()
            if point not in _ORACLE_GOLD:
                K = T(clip["K"])[None]
                _ORACLE_GOLD[point] = [oracle.pairnet_step(w, T(clip["images"][r])[None], T(clip["poses"][r])[None],
                                                           [T(clip["images"][j])[None] for j in ms], [T(clip["poses"][j])[None] for j in ms],
                                                           K, n_depth_levels=D).numpy() for r, ms in clip["frames"]]
        errs = [oracle.rel_l1_inverse_depth(o.cpu().numpy(), g) for o, g in zip(outs, _ORACLE_GOLD[point])]
        print("pairnet lookahead engine vs oracle, %s, %d terms: max rel-L1(inverse depth) %.3e, per keyframe %s"
              % (point, terms, max(errs), ["%.2e" % e for e in errs]))
        assert max(errs) <= 1e-3, errs
    finally:
        ops.set_conv_backend(old, terms=3)


def test_pairnet_engine_shipped_weights_vs_oracle():
    """The reference's shipped pairnet weights on the fixture scene (320x256, 64 planes), the index lines with 3 measurement
    frames through the engine (tensor cores, fp16 operands) against oracle.pairnet_step with the same weights: <= 1e-3."""
    w = scene_fixture.load_shipped_weights("pairnet")
    if w is None:
        pytest.skip("shipped weights not fetched (DVMVS_REFERENCE_ROOT=<reference checkout> python tools/fetch_fixtures.py)")
    from dvmvs import _ops as ops
    from oracle import dvmvs_oracle as oracle
    old = ops.conv_backend()
    ops.set_conv_backend("tc", terms=1, stride2=True)
    try:
        mods = helpers.build_product_modules(w, pairnet=True)
        frames, full_K, _ = scene_fixture.load_scene()
        steady = [fr for fr in frames if len(fr["measurement_images"]) == 3]
        assert steady
        H, W = steady[0]["reference_image"].shape[-2:]
        T = torch.from_numpy
        args = lambda fr, dev: (T(fr["reference_image"])[None].to(dev), T(fr["reference_pose"])[None].to(dev),
                                [T(x)[None].to(dev) for x in fr["measurement_images"]], [T(p)[None].to(dev) for p in fr["measurement_poses"]],
                                T(full_K)[None].to(dev))
        with torch.no_grad():
            eng = _engine(mods, 1, H, W, 3, 64, T=4, G=2)
            eng.prime(*args(steady[0], DEV))
            outs = []
            for fr in steady:
                out = torch.empty((1, H, W), dtype=torch.float32, device=DEV)
                eng.submit(*args(fr, DEV), out=out)
                outs.append(out)
            eng.synchronize()
            errs = [oracle.rel_l1_inverse_depth(o.cpu().numpy(), oracle.pairnet_step(w, *args(fr, "cpu")).numpy())
                    for o, fr in zip(outs, steady)]
        print("pairnet lookahead engine + shipped weights vs oracle (%d keyframes):" % len(errs), ["%.2e" % e for e in errs])
        assert max(errs) <= 1e-3, errs
    finally:
        ops.set_conv_backend(old, terms=3)


# ------------------------------------------------------------------------------------------------ stream ordering
ORDERING = [  # H, W, D, M, terms, B, T, G
    pytest.param((64, 96, 64, 2, 1, 1, 3, 2), id="64x96-1term"),
    pytest.param((64, 96, 64, 2, 3, 2, 3, 2), id="64x96-3terms-B2"),
    pytest.param((128, 128, 32, 1, 1, 1, 4, 3), id="c1-T4-G3"),
]


@pytest.mark.parametrize("cfg", ORDERING)
def test_pairnet_engine_equals_its_schedule_replay_under_delayed_streams(oracle, synth, delay, cfg):
    """The engine against _replay with torch.equal on every keyframe, undelayed, with each of its five streams delayed alone,
    all but the decoder's stream delayed, and the caller's stream delayed.  The replay runs the engine's batches, so every
    split-K decision is the engine's and no tolerance is needed."""
    H, W, D, M, terms, B, T, G = cfg
    script, n = _lookahead_script(T, G)
    with _tc(terms), torch.no_grad():
        mods, _ = _pairnet_modules(oracle, synth, D)
        frames = _frames(synth, B, n, H, W, M)
        eng = _engine(mods, B, H, W, M, D, T, G)
        eng.prime(*frames[0])
        ref = _replay(mods, frames, script, T, B, H, W, M, D)
        assert B == 1 or not torch.equal(ref[-1][0], ref[-1][-1]), "the batch rows hold the same clip"
        _assert_same(_run(eng, frames, script), ref, "undelayed")
        assert len(_stage_graphs(eng)) == 5 * eng.G
        cycles = _calibrate(eng, "pairnet lookahead %s" % (cfg,))
        delay.install()
        _under_delays(eng, frames, script, ref, delay, cycles, "pairnet lookahead %s" % (cfg,))


def test_planted_ordering_defects_change_the_delayed_run(oracle, synth, delay, skips):
    """Each planted defect skips one wait of the engine; with the stream that produces what the wait guards delayed (for the
    group-reuse wait: the decoder's stream, which still reads the reused group), the run must differ from the bit-exact
    replay.  So the delayed runs of the schedule-replay test would catch a missing wait."""
    H, W, D, M, T, G = 64, 96, 64, 2, 3, 2
    script, n = _lookahead_script(T, G)
    with _tc(1), torch.no_grad():
        mods, _ = _pairnet_modules(oracle, synth, D)
        frames = _frames(synth, 1, n, H, W, M)
        eng = _engine(mods, 1, H, W, M, D, T, G)
        eng.prime(*frames[0])
        ref = _replay(mods, frames, script, T, 1, H, W, M, D)
        _assert_same(_run(eng, frames, script), ref, "undelayed, no defect")
        assert len(_stage_graphs(eng)) == 5 * eng.G
        cycles = _calibrate(eng, "pairnet defects")
        delay.install()
        s = eng.streams
        defects = [("the decoder does not wait for the encoder (done[3])", dict(on=s[4], events=[g["done"][3] for g in eng.groups]), [s[3]]),
                   ("the plane sweep does not wait for the pyramid (done[1])", dict(on=s[2], events=[g["done"][1] for g in eng.groups]), [s[1]]),
                   ("the group-reuse wait on done[4] is skipped", dict(on=None, events=[g["done"][4] for g in eng.groups]), [s[4]])]
        missed = []
        for name, plant, streams in defects:
            with skips.planted(**plant) as sk:
                with delay.on(streams, cycles):
                    delayed = _run(eng, frames, script)
                hit = sk.skipped
            _run(eng, frames, script)                 # a clean run after the defect's
            assert hit > 0, "%s: the planted defect skipped no wait" % name
            bad = _diff(delayed, ref)[0]
            print("pairnet, planted defect '%s': delayed run %s (%d of %d keyframes differ)"
                  % (name, "catches it" if bad else "DOES NOT catch it", len(bad), len(ref)))
            if not bad:
                missed.append(name)
        assert not missed, "planted defects the delayed run did not catch: %s" % missed


# ------------------------------------------------------------------------------------------------ row independence
@pytest.mark.parametrize("B", [1, 2])
def test_rows_are_independent(oracle, synth, B):
    """Keyframe X submitted at every position of a group of 3, next to different neighbours each time, and launched by
    flush() in incomplete groups of 1 and 2 whose other rows hold stale inputs: its depth is the same bit for bit every time,
    i.e. no kernel of the five stages makes a batch row depend on another."""
    H, W, D, M, T = 64, 96, 64, 2, 3
    with _tc(1), torch.no_grad():
        mods, _ = _pairnet_modules(oracle, synth, D)
        frames = _frames(synth, B, 10, H, W, M)
        X = frames[9]
        eng = _engine(mods, B, H, W, M, D, T, 2)
        eng.prime(*frames[0])
        groups = [[X, frames[0], frames[1]], [frames[2], X, frames[3]], [frames[4], frames[5], X], [X], [frames[6], X], [frames[7], frames[8], X]]
        seen = []
        for grp in groups:
            for f in grp:
                out = torch.full((B, H, W), NAN, device=DEV)
                eng.submit(*f, out=out)
                if f is X:
                    seen.append(out)
            eng.synchronize()
        torch.cuda.synchronize()
    assert bool(torch.isfinite(seen[0]).all())
    differ = [i for i, o in enumerate(seen) if not torch.equal(o, seen[0])]
    print("pairnet rows, B=%d: keyframe X in %d placements, %d differ from the first" % (B, len(seen), len(differ)))
    assert not differ, "placements %s of keyframe X differ (max |diff| %.3e)" % (
        differ, max(float((seen[i] - seen[0]).abs().max()) for i in differ))


# ------------------------------------------------------------------------------------------------ caller contract
def test_submit_consumes_inputs_on_the_callers_stream(oracle, synth, delay):
    """As test_engine_ordering's test of that name: (a) inputs produced late on the caller's stream; (b) inputs freed right
    after submit() and their memory reused and filled with NaN, stream 0 delayed; (c) CUDA inputs overwritten with NaN after
    every submit(), and pinned host inputs rewritten once the caller's stream has passed the submit(), stream 0 delayed;
    (d) one `out` for every submit(), the decoder's stream delayed: after each synchronize() it holds the last keyframe's depth."""
    H, W, D, M, T, G = 64, 96, 64, 2, 3, 2
    script, n = _lookahead_script(T, G)
    with _tc(1), torch.no_grad():
        mods, _ = _pairnet_modules(oracle, synth, D)
        frames = _frames(synth, 1, n, H, W, M)
        eng = _engine(mods, 1, H, W, M, D, T, G)
        eng.prime(*frames[0])
        ref = _replay(mods, frames, script, T, 1, H, W, M, D)
        _assert_same(_run(eng, frames, script), ref, "undelayed")
        assert len(_stage_graphs(eng)) == 5 * eng.G
        cycles = _calibrate(eng, "pairnet contract")
        delay.install()
        first, last = eng.streams[:1], eng.streams[-1:]
        failures = []

        def check(what, got):
            bad, worst = _diff(got, ref)
            print("pairnet, %s: %s" % (what, "bit-identical" if not bad else "keyframes %s differ (max |diff| %.3e)" % (bad, worst)))
            if bad:
                failures.append(what)

        check("(a) inputs produced late", _run(eng, frames, script, _late(frames, cycles)))

        held, reused = {}, [0, 0]

        def fresh(k):
            args = _map(lambda t: t.clone(), frames[k])
            held["ptrs"] = {t.data_ptr() for t in _tensors(args)}
            return args, {}

        def free_and_poison():
            nan = [torch.full_like(t, NAN) for t in _tensors(frames[0])]
            reused[0] += sum(t.data_ptr() in held["ptrs"] for t in nan)
            reused[1] += len(nan)
            held["nan"] = nan

        with delay.on(first, cycles):
            check("(b) inputs freed, memory reused and filled with NaN", _run(eng, frames, script, fresh, free_and_poison))
        print("pairnet, (b): %d of %d NaN-filled allocations reused an input's memory" % (reused[0], reused[1]))
        if not reused[0]:
            failures.append("(b) never reused an input's memory, so it does not test what it says")

        buf = _map(lambda t: t.clone(), frames[0])

        def overwrite_feed(k):
            for dst, src in zip(_tensors(buf), _tensors(frames[k])):
                dst.copy_(src)
            return buf, {}

        def poison():
            for t in _tensors(buf):
                t.fill_(NAN)

        with delay.on(first, cycles):
            check("(c) CUDA inputs overwritten after submit()", _run(eng, frames, script, overwrite_feed, poison))

        host = [_map(lambda t: t.cpu(), f) for f in frames]
        pinned = _map(lambda t: t.cpu().pin_memory(), frames[0])

        def pinned_feed(k):
            for dst, src in zip(_tensors(pinned), _tensors(host[k])):
                dst.copy_(src)
            return pinned, {}

        def host_poison():
            torch.cuda.current_stream().synchronize()
            for t in _tensors(pinned):
                t.fill_(NAN)

        with delay.on(first, cycles):
            check("(c) pinned host inputs rewritten after the caller's stream passed submit()", _run(eng, frames, script, pinned_feed, host_poison))

        out = torch.full((1, H, W), NAN, device=DEV)
        seen, i = [], -1
        with delay.on(last, cycles):
            for op in script + ["sync"]:
                if op == "sync":
                    eng.synchronize()
                    torch.cuda.synchronize()
                    seen.append((i, out.clone()))
                elif op != "reset":
                    eng.submit(*frames[op], out=out)
                    i += 1
        bad = [j for j, o in seen if not torch.equal(o, ref[j])]
        print("pairnet, (d) one out for every submit(): %s" % ("bit-identical at every synchronize()" if not bad else "differs after keyframes %s" % bad))
        if bad:
            failures.append("(d) one out")
        assert not failures, "the pairnet engine breaks the caller contract: %s" % failures


def test_depth_of_stale_buffered_and_launched_keyframes(oracle, synth):
    """depth_of(t): a keyframe buffered in a group not launched yet raises KeyError; once its group is launched it returns a
    buffer equal to the keyframe's own `out`; once a later keyframe launched in its slot it raises KeyError (stale).  Checked
    after every submit and synchronize of a run that wraps around both groups with incomplete groups."""
    H, W, D, M, T, G = 64, 96, 64, 2, 3, 2
    script, n = _lookahead_script(T, G)
    with _tc(1), torch.no_grad():
        mods, _ = _pairnet_modules(oracle, synth, D)
        frames = _frames(synth, 1, n, H, W, M)
        eng = _engine(mods, 1, H, W, M, D, T, G)
        eng.prime(*frames[0])
        t0 = eng.t
        outs, launched, slot_of, counts = {}, set(), {}, {"buffered": 0, "launched": 0, "stale": 0}
        for op in script + ["sync"]:
            if op == "sync":
                eng.synchronize()
            elif op != "reset":
                slot = (eng._gi % G) * T + eng._fill          # the keyframe slot this submit fills
                out = torch.full((1, H, W), NAN, device=DEV)
                t = eng.submit(*frames[op], out=out)
                outs[t], slot_of[t] = out, slot
            if eng._fill == 0:              # the open group was launched (or nothing is buffered)
                launched.update(outs)
            torch.cuda.synchronize()
            newest = {}
            for t in sorted(launched):
                newest[slot_of[t]] = t
            for t in range(t0, eng.t):
                if t not in launched:
                    with pytest.raises(KeyError):
                        eng.depth_of(t)
                    counts["buffered"] += 1
                elif newest[slot_of[t]] == t:
                    assert torch.equal(eng.depth_of(t), outs[t]), "launched keyframe %d" % t
                    counts["launched"] += 1
                else:
                    with pytest.raises(KeyError):
                        eng.depth_of(t)
                    counts["stale"] += 1
        print("pairnet depth_of checks:", counts)
        assert all(counts.values())


def test_constructor_rejects_fusionnet_modules_and_bad_sizes(oracle, synth):
    from dvmvs import pipeline
    D = 64
    w = helpers.oracle_weights(oracle, synth, 11, n_depth_levels=D)
    kw = dict(batch=1, height=64, width=96, n_measurement_frames=2, n_depth_levels=D)
    with pytest.raises(ValueError, match="LookaheadFusionnet"):
        pipeline.LookaheadPairnet(helpers.build_product_modules(w, n_depth_levels=D), **kw)
    pairnet = helpers.build_product_modules(w, n_depth_levels=D, pairnet=True)
    with pytest.raises(ValueError):
        pipeline.LookaheadPairnet(pairnet, lookahead=0, **kw)
    with pytest.raises(ValueError):
        pipeline.LookaheadPairnet(pairnet, n_groups=1, **kw)
