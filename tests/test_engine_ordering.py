"""Stream ordering of the keyframe engines (dvmvs.pipeline): their cross-stream events, slot and group reuse, static
recurrent state and input uploads are checked under timings a quiet GPU does not produce.

- LookaheadFusionnet against an eager replay of its own schedule, bit for bit on every keyframe.  PipelinedFusionnet and
  GraphedFusionnet against eager keyframe(), bit for bit.
- Every engine again with one or more of its streams delayed: a patched CUDAGraph.replay / pipeline._upload first enqueues
  a bounded torch.cuda._sleep on the streams chosen, calibrated to at least 5x the longest stage-graph replay of the engine.
  The caller's stream is delayed by the test itself, before it writes the inputs it submits.
- Planted ordering defects (one skipped wait each) must change the delayed run's depth: the delays can expose a missing wait.
- The caller contract of submit(): inputs produced late, freed, or overwritten after submit(), and one `out` for all.
- depth_of(t) returns keyframe t's depth or raises.

The engines draw their streams from torch's round-robin stream pool, so which CUDA streams a test's engine gets depends
on every stream created before it in the process.  In this file's order the 5-stage engine of
test_submit_consumes_inputs_on_the_callers_stream[pipelined] got, as one stage stream, the stream that an earlier
engine's decoder fork used as its side stream; with the split-K workspace keyed by stream alone, that stage's graph and
the recurrent stage's forked convolutions shared partial sums while running concurrently (see dvmvs._ops.stand_in_for).
"""
import contextlib
import math

import numpy as np
import pytest
import torch

from tests import helpers

pytestmark = pytest.mark.gpu

DEV = "cuda"
NAN = float("nan")


# ------------------------------------------------------------------------------------------------ inputs and scripts
@contextlib.contextmanager
def _tc(terms):
    from dvmvs import _ops as ops
    old = ops.conv_backend()
    ops.set_conv_backend("tc", terms=terms, stride2=True)
    try:
        yield
    finally:
        ops.set_conv_backend(old, terms=3)


def _frames(synth, B, n, H, W, M):
    """n keyframes of B clips (clip 5 + c in batch row c) as bench.py stacks them: (ref, ref_pose, [meas], [meas_poses], K)."""
    clips = [synth.make_clip(5 + c, n, H, W, M) for c in range(B)]
    stack = lambda pick: torch.from_numpy(np.ascontiguousarray(np.stack([pick(c) for c in clips]))).to(DEV)
    K = stack(lambda c: c["K"])
    out = []
    for t in range(n):
        ref = lambda c: c["frames"][t][0]
        meas = lambda c, m: c["frames"][t][1][m]
        out.append((stack(lambda c: c["images"][ref(c)]), stack(lambda c: c["poses"][ref(c)]),
                    [stack(lambda c: c["images"][meas(c, m)]) for m in range(M)],
                    [stack(lambda c: c["poses"][meas(c, m)]) for m in range(M)], K))
    return out


def _lookahead_script(T, G):
    """Keyframe indices with "reset" / "sync" between them, 3 G groups: every group is used three times and a run ends at the
    group it started in (so every run captures nothing new after the first).  Group 1 has a reset() in its middle, group 2 is
    flushed incomplete by a synchronize() after T - 1 keyframes, and the last group is incomplete."""
    script, k = [], 0
    for gi in range(3 * G):
        for j in range(T - 1 if gi in (2, 3 * G - 1) else T):
            if gi == 1 and j == T // 2:
                script.append("reset")
            script.append(k)
            k += 1
        if gi == 2:
            script.append("sync")
    return script, k


def _pipelined_script(n):
    """3 n keyframes (every slot used three times, a run ends in the slot it started in), a reset() in the middle and a
    synchronize() in the middle of the second pass over the slots."""
    script = list(range(3 * n))
    script.insert(2 * n + 1, "sync")
    script.insert(n + 1, "reset")
    return script, 3 * n


def _map(fn, frame):
    ref, rpose, meas, mposes, K = frame
    return fn(ref), fn(rpose), [fn(x) for x in meas], [fn(x) for x in mposes], fn(K)


def _tensors(frame):
    ref, rpose, meas, mposes, K = frame
    return [ref, rpose, *meas, *mposes, K]


# ------------------------------------------------------------------------------------------------ references
def _replay_lookahead(mods, frames, script, T, B, H, W, M, D):
    """What LookaheadFusionnet.flush() runs, eagerly on the current stream and without graphs: per group the trunk head (with
    the side inputs), trunk tail + pyramid, plane sweep and encoder over the same stacked T*B batch, then the recurrent
    stage of each buffered keyframe in order on batch slices of the group's outputs, carrying a KeyframeState that reset()
    drops.  Rows of an incomplete group that no keyframe filled hold zeros (the engine's hold an earlier keyframe): every
    operation reads only its own batch row, so they do not reach a submitted keyframe's depth."""
    from dvmvs import _ops as ops
    from dvmvs import pipeline
    from dvmvs._base import no_auto_graph
    TB = T * B
    depths, state, buffered = [], pipeline.KeyframeState(), []

    def flush():
        images = torch.zeros(((M + 1) * TB, 3, H, W), device=DEV)
        eye = lambda: torch.eye(4, device=DEV).repeat(TB, 1, 1)
        grp = {"images": images, "ref_image": images[:TB], "meas_images": [images[(m + 1) * TB:(m + 2) * TB] for m in range(M)],
               "ref_pose": eye(), "meas_poses": [eye() for _ in range(M)],
               "full_K": torch.tensor([[float(W), 0.0, W / 2.0], [0.0, float(W), H / 2.0], [0.0, 0.0, 1.0]], device=DEV).repeat(TB, 1, 1)}
        for j, (k, _) in enumerate(buffered):
            ref, rpose, meas, mposes, K = frames[k]
            lo, hi = j * B, (j + 1) * B
            grp["ref_image"][lo:hi].copy_(ref)
            grp["ref_pose"][lo:hi].copy_(rpose)
            grp["full_K"][lo:hi].copy_(K)
            for m in range(M):
                grp["meas_images"][m][lo:hi].copy_(meas[m])
                grp["meas_poses"][m][lo:hi].copy_(mposes[m])
        pipeline._stage_side_inputs(grp)
        head = mods["fe"].forward_head(grp["images"])
        pyramid = mods["fpn"](*mods["fe"].forward_tail(head))
        swept = pipeline._sweep_from_pyramid(grp, pyramid, 0, 0.25, 20.0, D)
        enc, half_K = pipeline._stage_enc(mods, grp, swept)
        nonlocal state
        for j, (k, with_state) in enumerate(buffered):
            lo, hi = j * B, (j + 1) * B
            if not with_state:
                state = pipeline.KeyframeState()
            view = {"ref_image": grp["ref_image"][lo:hi], "ref_pose": grp["ref_pose"][lo:hi], "full_K": grp["full_K"][lo:hi],
                    "ref_cl": grp["ref_cl"][lo:hi], "lstm_K": grp["lstm_K"][lo:hi], "input_gates": grp["input_gates"][lo:hi]}
            pred, state = pipeline._stage_rec(mods, state, view, tuple(ops.batch_slice(e, lo, hi) for e in enc), half_K[lo:hi])
            depths.append(pred.clone())
        buffered.clear()

    has_state = False
    with no_auto_graph():
        for op in script:
            if op == "reset":
                has_state = False
            elif op == "sync":
                if buffered:
                    flush()
            else:
                buffered.append((op, has_state))
                has_state = True
                if len(buffered) == T:
                    flush()
        if buffered:
            flush()
    torch.cuda.synchronize()
    return depths


def _eager_keyframes(mods, frames, script, D):
    """keyframe() per submitted keyframe, eagerly and without graphs, carrying the state that reset() drops."""
    from dvmvs import pipeline
    from dvmvs._base import no_auto_graph
    st, depths = pipeline.KeyframeState(), []
    with no_auto_graph():
        for op in script:
            if op == "reset":
                st = pipeline.KeyframeState()
            elif op != "sync":
                pred, st = pipeline.keyframe(mods, st, *frames[op], n_depth_levels=D)
                depths.append(pred.clone())
    torch.cuda.synchronize()
    return depths


# ------------------------------------------------------------------------------------------------ driving an engine
class _Graphed:
    """GraphedFusionnet behind the submit / reset / synchronize surface of the other engines."""

    def __init__(self, eng):
        self.eng = eng

    def reset(self):
        self.eng.reset()

    def submit(self, *args, out):
        out.copy_(self.eng.step(*args))

    def synchronize(self):
        pass


def _run(eng, frames, script, feed=None, after=None):
    """Drives `eng` through `script` from a fresh clip state; returns each submitted keyframe's depth (its own `out`).
    feed(k) -> (args, kwargs) of submit(), after() runs on the caller's side right after each submit()."""
    eng.reset()
    B, _, H, W = frames[0][0].shape
    outs = []
    for op in script:
        if op == "reset":
            eng.reset()
        elif op == "sync":
            eng.synchronize()
        else:
            args, kw = feed(op) if feed is not None else (frames[op], {})
            out = torch.full((B, H, W), NAN, device=DEV)
            eng.submit(*args, out=out, **kw)
            del args
            if after is not None:
                after()
            outs.append(out)
    eng.synchronize()
    torch.cuda.synchronize()
    return outs


def _late(frames, cycles):
    """The caller's stream sleeps, then produces the inputs it submits as fresh tensors."""
    def feed(k):
        torch.cuda._sleep(cycles)
        return _map(lambda t: t.clone(), frames[k]), {}
    return feed


def _diff(got, ref):
    """Indices of the keyframes whose depth is not bit-identical to the reference, and the largest difference."""
    bad = [i for i, (g, r) in enumerate(zip(got, ref)) if not torch.equal(g, r)]
    worst = max((float((got[i] - ref[i]).abs().nan_to_num(nan=math.inf).max()) for i in bad), default=0.0)
    return bad, worst


def _assert_same(got, ref, what):
    assert len(got) == len(ref)
    bad, worst = _diff(got, ref)
    assert not bad, "%s: keyframes %s differ from the reference (max |diff| %.3e)" % (what, bad, worst)


class _Delay:
    """After install(): every CUDAGraph.replay() and pipeline._upload() issued on one of `streams` first enqueues
    torch.cuda._sleep(cycles) there.  Installed after prime(), so that no captured graph contains a sleep; lazily captured
    graphs go through pipeline._capture_graph, which replays nothing."""

    def __init__(self, monkeypatch):
        self.monkeypatch, self.streams, self.cycles, self.sleeps = monkeypatch, [], 0, 0

    def install(self):
        from dvmvs import pipeline
        replay, upload = torch.cuda.CUDAGraph.replay, pipeline._upload

        def delayed_replay(graph):
            self._sleep()
            return replay(graph)

        def delayed_upload(*args, **kwargs):
            self._sleep()
            return upload(*args, **kwargs)

        self.monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", delayed_replay)
        self.monkeypatch.setattr(pipeline, "_upload", delayed_upload)

    def _sleep(self):
        if self.cycles and torch.cuda.current_stream() in self.streams:
            torch.cuda._sleep(self.cycles)
            self.sleeps += 1

    @contextlib.contextmanager
    def on(self, streams, cycles):
        self.streams, self.cycles, self.sleeps = list(streams), cycles, 0
        try:
            yield self
        finally:
            self.streams, self.cycles = [], 0


@pytest.fixture
def delay(monkeypatch):
    return _Delay(monkeypatch)


class _Skips:
    """Planted ordering defects: Stream.wait_event(ev) skipped for ev in `events` (on stream `on`, or on any stream when `on`
    is None), Stream.wait_stream(other) skipped on stream `on`."""

    def __init__(self, monkeypatch):
        self.events, self.on, self.other, self.skipped = (), None, None, 0
        wait_event, wait_stream = torch.cuda.Stream.wait_event, torch.cuda.Stream.wait_stream

        def skip_event(stream, event):
            if any(event is e for e in self.events) and (self.on is None or stream == self.on):
                self.skipped += 1
                return None
            return wait_event(stream, event)

        def skip_stream(stream, other):
            if self.other is not None and stream == self.on and other == self.other:
                self.skipped += 1
                return None
            return wait_stream(stream, other)

        monkeypatch.setattr(torch.cuda.Stream, "wait_event", skip_event)
        monkeypatch.setattr(torch.cuda.Stream, "wait_stream", skip_stream)

    @contextlib.contextmanager
    def planted(self, on, events=(), other=None):
        self.on, self.events, self.other, self.skipped = on, tuple(events), other, 0
        try:
            yield self
        finally:
            self.on, self.events, self.other = None, (), None


@pytest.fixture
def skips(monkeypatch):
    return _Skips(monkeypatch)


def _stage_graphs(eng):
    """(graph, stream) of every captured stage graph of an engine."""
    from dvmvs import pipeline
    if isinstance(eng, (pipeline.LookaheadFusionnet, pipeline.LookaheadPairnet)):
        out = [(gr, eng.streams[i]) for g in eng.groups for i, gr in enumerate(g["graph"]) if gr is not None]
        return out + [(gr, eng.streams[4]) for ks in eng.kslots for gr in ks["graph"].values()]
    if isinstance(eng, pipeline.PipelinedFusionnet):
        return [(gr, eng.streams[i]) for slot in eng.slots for i, d in enumerate(slot["graph"]) for gr in d.values()]
    return [(gr, torch.cuda.current_stream()) for gr in eng.eng._graphs.values()]


def _elapsed_ms(stream, fn, reps=3):
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record()
            fn()
            e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def _calibrate(eng, label):
    """Sleep cycles worth at least 5x (aimed at 6x) the longest stage-graph replay of `eng`, each graph replayed alone on its
    own stream with the engine otherwise idle (median of 3).  Replaying a stage graph rewrites only buffers that the
    engine's next run rewrites before reading (a run starts with reset()), so this changes no later result."""
    torch.cuda.synchronize()
    graphs = _stage_graphs(eng)
    assert graphs
    longest = max(_elapsed_ms(s, g.replay) for g, s in graphs)
    side = torch.cuda.Stream()
    cycles = 2_000_000
    for _ in range(4):
        sleep = _elapsed_ms(side, lambda: torch.cuda._sleep(cycles), reps=1)
        if sleep >= 6.0 * longest:
            break
        cycles = int(cycles * 6.6 * longest / sleep) + 1
    print("%s: %d stage graphs, longest replay %.3f ms; sleep of %d cycles %.3f ms (%.1fx)"
          % (label, len(graphs), longest, cycles, sleep, sleep / longest))
    assert sleep >= 5.0 * longest, "sleep %.3f ms is not 5x the longest stage replay %.3f ms" % (sleep, longest)
    return cycles


def _variants(eng, frames, cycles):
    """(name, delayed engine streams, feed): each engine stream alone, every stream but the last, the caller's stream."""
    streams = list(getattr(getattr(eng, "eng", eng), "streams", []))
    out = [("stream %d" % i, [s], None) for i, s in enumerate(streams)]
    if streams:
        out.append(("streams 0..%d" % (len(streams) - 2), streams[:-1], None))
    out.append(("caller's stream", [], _late(frames, cycles)))
    return out


def _under_delays(eng, frames, script, ref, delay, cycles, what):
    for name, streams, feed in _variants(eng, frames, cycles):
        with delay.on(streams, cycles):
            got = _run(eng, frames, script, feed)
            slept = delay.sleeps
        assert feed is not None or slept > 0, "%s, %s delayed: no sleep was enqueued" % (what, name)
        _assert_same(got, ref, "%s, %s delayed" % (what, name))


def _modules(oracle, synth, D):
    return helpers.build_product_modules(helpers.oracle_weights(oracle, synth, 11, n_depth_levels=D), n_depth_levels=D)


# ------------------------------------------------------------------------------------------------ engine matrix
LOOKAHEAD = [  # H, W, D, M, terms, B, T, G
    pytest.param((256, 256, 64, 2, 1, 1, 4, 3), id="headline-256x256-T4-G3"),
    pytest.param((64, 96, 64, 2, 1, 1, 3, 2), id="64x96-1term"),
    pytest.param((64, 96, 64, 2, 3, 1, 3, 2), id="64x96-3terms"),
    pytest.param((64, 96, 96, 4, 1, 1, 3, 2), id="64x96-M4-D96"),
    pytest.param((64, 96, 64, 2, 1, 2, 3, 2), id="64x96-B2"),
]


@pytest.mark.parametrize("cfg", LOOKAHEAD)
def test_lookahead_engine_equals_its_schedule_replay_under_delayed_streams(oracle, synth, delay, cfg):
    """LookaheadFusionnet against _replay_lookahead with torch.equal on every keyframe, undelayed and with each of its
    streams delayed alone, all but the recurrent stream delayed, and the caller's stream delayed.  The replay runs the
    engine's batches, so every split-K decision is the engine's and no tolerance is needed.  64x96-M4-D96 is c3's engine
    configuration (4 measurement frames, 96 planes) at a small size; B2 has a distinct clip in each batch row."""
    from dvmvs import pipeline
    H, W, D, M, terms, B, T, G = cfg
    script, n = _lookahead_script(T, G)
    with _tc(terms), torch.no_grad():
        mods = _modules(oracle, synth, D)
        frames = _frames(synth, B, n, H, W, M)
        eng = pipeline.LookaheadFusionnet(mods, batch=B, height=H, width=W, n_measurement_frames=M, n_depth_levels=D,
                                          lookahead=T, n_groups=G)
        eng.prime(*frames[0])
        ref = _replay_lookahead(mods, frames, script, T, B, H, W, M, D)
        assert B == 1 or not torch.equal(ref[-1][0], ref[-1][-1]), "the batch rows hold the same clip"
        _assert_same(_run(eng, frames, script), ref, "undelayed")
        cycles = _calibrate(eng, "lookahead %s" % (cfg,))
        delay.install()
        _under_delays(eng, frames, script, ref, delay, cycles, "lookahead %s" % (cfg,))


PIPELINED = [  # n_stages, B, H, W
    pytest.param((2, 1, 64, 96), id="2-stages-64x96"),
    pytest.param((3, 1, 64, 96), id="3-stages-64x96"),
    pytest.param((4, 1, 64, 96), id="4-stages-64x96"),
    pytest.param((5, 1, 64, 96), id="5-stages-64x96"),
    pytest.param((5, 8, 256, 256), id="batched_8-5-stages-256x256"),
]


@pytest.mark.parametrize("cfg", PIPELINED)
def test_pipelined_engine_equals_eager_keyframe_under_delayed_streams(oracle, synth, delay, cfg):
    """PipelinedFusionnet against eager keyframe() with torch.equal on every keyframe, undelayed and under every delay
    variant; batched_8 is bench.py's point of that name (a distinct clip in each of the 8 rows)."""
    from dvmvs import pipeline
    ns, B, H, W = cfg
    D, M = 64, 2
    script, n = _pipelined_script(ns)
    with _tc(1), torch.no_grad():
        mods = _modules(oracle, synth, D)
        frames = _frames(synth, B, n, H, W, M)
        eng = pipeline.PipelinedFusionnet(mods, batch=B, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, n_stages=ns)
        eng.prime(*frames[0])
        ref = _eager_keyframes(mods, frames, script, D)
        assert B == 1 or not torch.equal(ref[-1][0], ref[-1][-1]), "the batch rows hold the same clip"
        _assert_same(_run(eng, frames, script), ref, "undelayed")
        cycles = _calibrate(eng, "pipelined %s" % (cfg,))
        delay.install()
        _under_delays(eng, frames, script, ref, delay, cycles, "pipelined %s" % (cfg,))


def test_feature_cache_engine_under_delayed_streams(oracle, synth, delay):
    """PipelinedFusionnet(feature_cache=8): a keyframe's measurement frames are the previous keyframes' reference frames
    (hits, submitted without an image), except after the jumps in the sequence (misses, computed eagerly on the sweep
    stage's stream), and the ring of 8 evicts.  Its reference is the engine's own undelayed run: eager keyframe() computes
    a hit's features in another batch."""
    from dvmvs import pipeline
    H, W, D, M, ns = 64, 96, 64, 2, 5
    ks = list(range(0, 6)) + list(range(9, 15)) + list(range(18, 21))          # 15 keyframes: 3 passes over the 5 slots
    script = ks[:7] + ["reset"] + ks[7:11] + ["sync"] + ks[11:]
    with _tc(1), torch.no_grad():
        mods = _modules(oracle, synth, D)
        clip = synth.make_clip(5, 21, H, W, M)
        frames = _frames(synth, 1, 21, H, W, M)
        ids = {k: (clip["frames"][k][0], clip["frames"][k][1]) for k in ks}
        eng = pipeline.PipelinedFusionnet(mods, batch=1, height=H, width=W, n_measurement_frames=M, n_depth_levels=D,
                                          n_stages=ns, feature_cache=8)
        eng.prime(*frames[0])

        def feed(k, src=None):
            ref, rpose, meas, mposes, K = frames[k] if src is None else src(k)
            meas = [None if i in eng.cache else x for i, x in zip(ids[k][1], meas)]
            return (ref, rpose, meas, mposes, K), {"reference_id": ids[k][0], "measurement_ids": ids[k][1]}

        def run(src=None):
            eng.cache.clear()
            eng.cache.hits = eng.cache.misses = 0
            got = _run(eng, frames, script, lambda k: feed(k, src))
            assert eng.cache.hits > 0 and eng.cache.misses > 0, (eng.cache.hits, eng.cache.misses)
            return got

        ref = run()
        assert all(bool(torch.isfinite(r).all()) for r in ref)
        assert _diff(run(), ref)[0] == [], "the feature cache engine is not deterministic undelayed"
        cycles = _calibrate(eng, "feature cache")
        delay.install()
        for name, streams, late in _variants(eng, frames, cycles):
            with delay.on(streams, cycles):
                got = run(None if late is None else (lambda k: late(k)[0]))
            _assert_same(got, ref, "feature cache, %s delayed" % name)


# ------------------------------------------------------------------------------------------------ planted defects
def _defects(eng, kind):
    """(name, planted(skips) kwargs, delayed streams, caller delayed) per planted ordering defect of `eng`."""
    s = eng.streams
    if kind == "lookahead":
        return [("the recurrent stream does not wait for done[3]", dict(on=s[4], events=[g["done"][3] for g in eng.groups]), [s[3]], False),
                ("the group-reuse wait on done[4] is skipped", dict(on=None, events=[g["done"][4] for g in eng.groups]), [s[4]], False),
                ("stage 2 does not wait for done[1]", dict(on=s[2], events=[g["done"][1] for g in eng.groups]), [s[1]], False),
                ("stream 0 does not wait for the caller's stream", dict(on=s[0], other=torch.cuda.current_stream()), [], True)]
    last = eng.n_stages - 1
    out = [("stage %d does not wait for done[%d]" % (i, i - 1), dict(on=s[i], events=[sl["done"][i - 1] for sl in eng.slots]), [s[i - 1]], False)
           for i in range(1, eng.n_stages)]
    return out + [("the slot-reuse wait on done[%d] is skipped" % last, dict(on=None, events=[sl["done"][last] for sl in eng.slots]), [s[last]], False),
                  ("stream 0 does not wait for the caller's stream", dict(on=s[0], other=torch.cuda.current_stream()), [], True)]


@pytest.mark.parametrize("kind", ["lookahead", "pipelined"])
def test_planted_ordering_defects_change_the_delayed_run(oracle, synth, delay, skips, kind):
    """Each planted defect skips one wait of the engine.  With the stream that produces what the wait guards delayed (for the
    reuse waits: the stream that still reads the reused buffers), the run must differ from the bit-exact reference; whether
    the undelayed run also differs is printed, to show what the delay adds."""
    from dvmvs import pipeline
    H, W, D, M = 64, 96, 64, 2
    if kind == "lookahead":
        T, G = 3, 2
        script, n = _lookahead_script(T, G)
    else:
        script, n = _pipelined_script(5)
    with _tc(1), torch.no_grad():
        mods = _modules(oracle, synth, D)
        frames = _frames(synth, 1, n, H, W, M)
        kw = dict(batch=1, height=H, width=W, n_measurement_frames=M, n_depth_levels=D)
        if kind == "lookahead":
            eng = pipeline.LookaheadFusionnet(mods, lookahead=T, n_groups=G, **kw)
            eng.prime(*frames[0])
            ref = _replay_lookahead(mods, frames, script, T, 1, H, W, M, D)
        else:
            eng = pipeline.PipelinedFusionnet(mods, n_stages=5, **kw)
            eng.prime(*frames[0])
            ref = _eager_keyframes(mods, frames, script, D)
        _assert_same(_run(eng, frames, script), ref, "undelayed, no defect")
        cycles = _calibrate(eng, "%s defects" % kind)
        delay.install()
        missed = []
        for name, plant, streams, caller in _defects(eng, kind):
            feed = _late(frames, cycles) if caller else None
            with skips.planted(**plant) as sk:
                undelayed = _run(eng, frames, script, _late(frames, 0) if caller else None)
                with delay.on(streams, cycles):
                    delayed = _run(eng, frames, script, feed)
                hit = sk.skipped
            _run(eng, frames, script)                 # a clean run after the defect's
            assert hit > 0, "%s: the planted defect skipped no wait" % name
            bad_u, bad_d = _diff(undelayed, ref)[0], _diff(delayed, ref)[0]
            print("%s, planted defect '%s': undelayed run %s, delayed run %s (%d of %d keyframes differ)"
                  % (kind, name, "catches it" if bad_u else "does not catch it", "catches it" if bad_d else "DOES NOT catch it",
                     len(bad_d), len(ref)))
            if not bad_d:
                missed.append(name)
        assert not missed, "planted defects the delayed run did not catch: %s" % missed


# ------------------------------------------------------------------------------------------------ caller contract
def _contract_engine(kind, mods, H, W, D, M):
    from dvmvs import pipeline
    kw = dict(batch=1, height=H, width=W, n_measurement_frames=M, n_depth_levels=D)
    if kind == "lookahead":
        return pipeline.LookaheadFusionnet(mods, lookahead=3, n_groups=2, **kw)
    if kind == "pipelined":
        return pipeline.PipelinedFusionnet(mods, n_stages=5, **kw)
    return _Graphed(pipeline.GraphedFusionnet(mods, **kw))


@pytest.mark.parametrize("kind", ["lookahead", "pipelined", "graphed"])
def test_submit_consumes_inputs_on_the_callers_stream(oracle, synth, delay, kind):
    """The contract of submit() (and GraphedFusionnet.step()): the engine behaves as if it had consumed its inputs on the
    caller's current stream at the time of the call.
    (a) inputs produced late on the caller's stream (it sleeps first);
    (b) inputs freed right after submit(), their memory immediately reused on the caller's stream and filled with NaN,
        stream 0 delayed;
    (c) the same CUDA input tensors overwritten with NaN on the caller's stream after every submit(), stream 0 delayed;
        the same with pinned host inputs rewritten on the host once the caller's stream has passed the submit();
    (d) one `out` for every submit() (as bench.py does), the last stream delayed: after each synchronize() it holds the
        last submitted keyframe's depth."""
    H, W, D, M = 64, 96, 64, 2
    script, n = _lookahead_script(3, 2) if kind == "lookahead" else _pipelined_script(5)
    with _tc(1), torch.no_grad():
        mods = _modules(oracle, synth, D)
        frames = _frames(synth, 1, n, H, W, M)
        eng = _contract_engine(kind, mods, H, W, D, M)
        if kind == "graphed":
            _run(eng, frames, script)             # captures both graphs
            ref = _eager_keyframes(mods, frames, script, D)
        else:
            eng.prime(*frames[0])
            ref = (_replay_lookahead(mods, frames, script, 3, 1, H, W, M, D) if kind == "lookahead"
                   else _eager_keyframes(mods, frames, script, D))
        _assert_same(_run(eng, frames, script), ref, "undelayed")
        cycles = _calibrate(eng, "%s contract" % kind)
        delay.install()
        streams = list(getattr(eng, "streams", []))
        first, last = streams[:1], streams[-1:]
        failures = []

        def check(what, got):
            bad, worst = _diff(got, ref)
            print("%s, %s: %s" % (kind, what, "bit-identical" if not bad else "keyframes %s differ (max |diff| %.3e)" % (bad, worst)))
            if bad:
                failures.append(what)

        # (a)
        check("(a) inputs produced late", _run(eng, frames, script, _late(frames, cycles)))

        # (b)
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
        print("%s, (b): %d of %d NaN-filled allocations reused an input's memory" % (kind, reused[0], reused[1]))
        if not reused[0]:
            failures.append("(b) never reused an input's memory, so it does not test what it says")

        # (c), CUDA inputs
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

        # (c), pinned host inputs
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
            check("(c) pinned host inputs rewritten after the caller's stream passed submit()",
                  _run(eng, frames, script, pinned_feed, host_poison))

        # (d)
        out = torch.full((1, H, W), NAN, device=DEV)
        seen, i = [], -1
        with delay.on(last, cycles):
            eng.reset()
            for op in script + ["sync"]:
                if op == "reset":
                    eng.reset()
                elif op == "sync":
                    eng.synchronize()
                    torch.cuda.synchronize()
                    seen.append((i, out.clone()))
                else:
                    eng.submit(*frames[op], out=out)
                    i += 1
        bad = [j for j, o in seen if not torch.equal(o, ref[j])]
        print("%s, (d) one out for every submit(): %s" % (kind, "bit-identical at every synchronize()" if not bad else "differs after keyframes %s" % bad))
        if bad:
            failures.append("(d) one out")
        assert not failures, "%s engine breaks the caller contract: %s" % (kind, failures)


# ------------------------------------------------------------------------------------------------ depth_of
@pytest.mark.parametrize("kind", ["lookahead", "pipelined"])
def test_depth_of_returns_the_keyframes_depth_or_raises(oracle, synth, kind):
    """After every submit / reset / synchronize of a sequence that wraps around the slots with incomplete groups, with the
    device synchronised but nothing flushed, depth_of(t) for every t of the sequence, one before it and two after it either
    raises KeyError or returns a buffer equal to keyframe t's own `out` (which starts as NaN, so a keyframe whose group was
    not launched yet cannot pass)."""
    from dvmvs import pipeline
    H, W, D, M = 64, 96, 64, 2
    script, n = _lookahead_script(3, 2) if kind == "lookahead" else _pipelined_script(3)
    with _tc(1), torch.no_grad():
        mods = _modules(oracle, synth, D)
        frames = _frames(synth, 1, n, H, W, M)
        kw = dict(batch=1, height=H, width=W, n_measurement_frames=M, n_depth_levels=D)
        eng = (pipeline.LookaheadFusionnet(mods, lookahead=3, n_groups=2, **kw) if kind == "lookahead"
               else pipeline.PipelinedFusionnet(mods, n_stages=3, **kw))
        eng.prime(*frames[0])
        t0 = eng.t
        outs, returned, raised, wrong = {}, 0, 0, []
        for step, op in enumerate(script + ["sync"]):
            if op == "reset":
                eng.reset()
            elif op == "sync":
                eng.synchronize()
            else:
                out = torch.full((1, H, W), NAN, device=DEV)
                outs[eng.submit(*frames[op], out=out)] = out
            torch.cuda.synchronize()
            for t in [-1] + list(range(t0, eng.t + 2)):
                try:
                    depth = eng.depth_of(t)
                except KeyError:
                    raised += 0 <= t < eng.t
                    continue
                returned += 1
                if t not in outs or not torch.equal(depth, outs[t]):
                    wrong.append((step, t))
        assert torch.equal(eng.depth_of(eng.t - 1), outs[eng.t - 1])
        print("%s depth_of: %d calls returned the keyframe's depth, %d calls for submitted keyframes raised, %d returned another"
              " depth" % (kind, returned, raised, len(wrong)))
        assert not wrong, "depth_of(t) returned a depth that is not keyframe t's at (step, t) = %s" % wrong[:10]
        assert returned > 0 and raised > 0
