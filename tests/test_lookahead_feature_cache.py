"""The lookahead engines' feature cache (LookaheadFusionnet / LookaheadPairnet with feature_cache=N, row f1): the trunk and
the feature pyramid over the reference images only, measurement features gathered from the cache's device ring.

- Against the same engine without the cache, on synthetic clips whose keyframes read the previous frames.
- The ring's content, exactly: stored reference features and gathered measurement features.
- Bit for bit against an eager replay of the engine's own schedule, undelayed and with each stream (and the caller's)
  delayed; a planted defect -- the ring store moved into the trunk-tail stage, on another stream -- must be caught.
- Hits and misses, row independence (pairnet), the CPU oracle at c1 / c2 / c3 shapes, the shipped weights.
"""
import os

import numpy as np
import pytest
import torch

from tests import helpers, scene_fixture
from tests.test_engine_ordering import (NAN, _Delay, _assert_same, _calibrate, _diff, _frames, _lookahead_script, _map, _tc,
                                        _variants)

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture
def delay(monkeypatch):
    return _Delay(monkeypatch)


def _modules(oracle, synth, D, pairnet, seed=11):
    w = helpers.oracle_weights(oracle, synth, seed, n_depth_levels=D)
    return helpers.build_product_modules(w, n_depth_levels=D, pairnet=pairnet), w


def _engine(mods, pairnet, B, H, W, M, D, T, G=2, cache=0):
    from dvmvs import pipeline
    cls = pipeline.LookaheadPairnet if pairnet else pipeline.LookaheadFusionnet
    return cls(mods, batch=B, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, lookahead=T, n_groups=G,
               feature_cache=cache)


def _ids(k, M):
    """Frame ids of keyframe k of synth.make_clip (the same in every batch row): reference frame k + M, measurement frames the
    M frames before it."""
    return {"reference_id": k + M, "measurement_ids": [k + M - i for i in range(1, M + 1)]}


def _feed(eng, frames, M, key=None):
    """feed(k) for the engines' submit(): keyframe `key(k)`'s inputs and ids, None for every measurement image the engine
    holds."""
    def feed(k):
        kf = k if key is None else key(k)
        ref, rpose, meas, mposes, K = frames[kf]
        ids = _ids(kf, M)
        return (ref, rpose, [None if i in eng.cache else x for i, x in zip(ids["measurement_ids"], meas)], mposes, K), ids
    return feed


def _run(eng, script, feed):
    """Drives `eng` through `script` from a fresh clip state and an empty cache; returns each keyframe's depth."""
    eng.reset()
    eng.cache.clear()
    eng.cache.hits = eng.cache.misses = 0
    B, H, W = eng.B, eng.H, eng.W
    outs = []
    for op in script:
        if op == "reset":
            eng.reset()
        elif op == "sync":
            eng.synchronize()
        else:
            args, kw = feed(op)
            out = torch.full((B, H, W), NAN, device=DEV)
            eng.submit(*args, out=out, **kw)
            outs.append(out)
    eng.synchronize()
    torch.cuda.synchronize()
    return outs


def _rel_l1_inv(a, b):
    from oracle import dvmvs_oracle as oracle
    return oracle.rel_l1_inverse_depth(a.cpu().numpy(), b.cpu().numpy())


# ------------------------------------------------------------------------------------------------ against the cache-less engine
CASES = [  # backend, terms, bound, B, T, M, D
    pytest.param(("fp32", 3, 1e-5, 1, 3, 2, 64), id="fp32-B1-T3"),
    pytest.param(("tc", 3, 1e-5, 1, 3, 2, 64), id="tc3-B1-T3"),
    pytest.param(("tc", 1, 1e-4, 1, 3, 2, 64), id="tc1-B1-T3"),
    pytest.param(("tc", 1, 1e-4, 2, 4, 2, 64), id="tc1-B2-T4"),
    pytest.param(("tc", 3, 1e-5, 2, 1, 2, 64), id="tc3-B2-T1"),
    pytest.param(("tc", 1, 1e-4, 1, 3, 4, 96), id="tc1-M4-D96"),
]


@pytest.mark.parametrize("pairnet", [False, True], ids=["fusionnet", "pairnet"])
@pytest.mark.parametrize("case", CASES)
def test_cache_engine_matches_cacheless_engine(oracle, synth, case, pairnet):
    """11 keyframes of synthetic clips (a reset after 7, the last group incomplete) through the engine with and without the
    cache.  The trunk batch differs (T*B against (M+1)*T*B images), so the split-K choice of a few convolutions
    does too: the bounds of test_lookahead_engine_matches_eager_keyframe.  A cold start misses the M frames never seen; the
    steady state passes no measurement image."""
    from dvmvs import _ops as ops
    backend, terms, bound, B, T, M, D = case
    H, W = 64, 96
    old = ops.conv_backend()
    ops.set_conv_backend(backend, terms=terms, stride2=True)
    try:
        with torch.no_grad():
            mods, _ = _modules(oracle, synth, D, pairnet)
            frames = _frames(synth, B, 11, H, W, M)
            plain = _engine(mods, pairnet, B, H, W, M, D, T)
            cached = _engine(mods, pairnet, B, H, W, M, D, T, cache=T * (M + 1) + 2)
            plain.prime(*frames[0])
            cached.prime(*frames[0])
            assert cached.cache.hits == cached.cache.misses == 0 and len(cached.cache._index) == 0
            script = list(range(7)) + ["reset"] + list(range(7, 11))
            feed = _feed(cached, frames, M)
            got = _run(cached, script, feed)
            assert (cached.cache.misses, cached.cache.hits) == (M, M * 10), (cached.cache.misses, cached.cache.hits)
            plain.reset()
            ref = []
            for op in script:
                if op == "reset":
                    plain.reset()
                    continue
                out = torch.full((B, H, W), NAN, device=DEV)
                plain.submit(*frames[op], out=out)
                ref.append(out)
            plain.synchronize()
        errs = [_rel_l1_inv(g, r) for g, r in zip(got, ref)]
        print("%s cache engine vs cache-less (%s): rel-L1(inverse depth) per keyframe %s"
              % ("pairnet" if pairnet else "fusionnet", case, ["%.1e" % e for e in errs]))
        assert all(bool(torch.isfinite(g).all()) for g in got)
        assert max(errs) <= bound, errs
    finally:
        ops.set_conv_backend(old, terms=3)


# ------------------------------------------------------------------------------------------------ ring content
@pytest.mark.parametrize("pairnet", [False, True], ids=["fusionnet", "pairnet"])
def test_ring_holds_the_pyramid_features_and_gathers_its_entries(oracle, synth, pairnet):
    """One group of 3 keyframes x 2 clips: the ring entry of each reference id equals that keyframe's rows of the group's
    pyramid a2, every gathered measurement row equals its ring entry, and a missed frame's entry equals FeatureShrinker(
    FeatureExtractor(image)) of its image (torch.equal throughout)."""
    H, W, D, M, T, B = 64, 96, 64, 2, 3, 2
    with _tc(1), torch.no_grad():
        mods, _ = _modules(oracle, synth, D, pairnet)
        frames = _frames(synth, B, T, H, W, M)
        eng = _engine(mods, pairnet, B, H, W, M, D, T, cache=T * (M + 1))
        eng.prime(*frames[0])
        _run(eng, list(range(T)), _feed(eng, frames, M))
        grp = eng.groups[(eng._gi - 1) % eng.G]
        ring, index = eng.cache.ring, grp["ring_index"]
        a2 = grp["pyramid"][0].permute(0, 2, 3, 1)
        for j in range(T):
            e = eng.cache._index[_ids(j, M)["reference_id"]]
            assert int(index[0, j]) == e
            assert torch.equal(ring[e], a2[j * B:(j + 1) * B]), "keyframe %d: ring entry != pyramid rows" % j
            for m in range(M):
                assert torch.equal(grp["meas_half"][m][j * B:(j + 1) * B], ring[int(index[1 + m, j])]), (j, m)
        for m, fid in enumerate(_ids(0, M)["measurement_ids"]):       # keyframe 0's frames missed
            half = mods["fpn"](*mods["fe"](frames[0][2][m]))[0]
            assert torch.equal(ring[eng.cache._index[fid]], half.permute(0, 2, 3, 1))


# ------------------------------------------------------------------------------------------------ schedule replay
def _replay(mods, pairnet, frames, script, key, cap, T, B, H, W, M, D):
    """What the engine runs, eagerly on the current stream and without graphs: per keyframe the reservation of submit(); per
    group the rows of the buffered keyframes, the miss stores, then the stage bodies (store, gather and sweep in the sweep
    stage) over the same T*B batch, and for fusionnet the recurrent stage of each keyframe on its batch slice, carrying a
    KeyframeState that reset() drops.  Its own FeatureCache of the same capacity goes through the same reservations, so
    every ring entry is the engine's.  Rows no keyframe filled hold zeros (the engine's hold earlier inputs) and gather
    the sink: every operation reads only its own batch row."""
    from dvmvs import _ops as ops
    from dvmvs import pipeline
    from dvmvs._base import no_auto_graph
    cache = pipeline.FeatureCache(cap)
    cache.allocate((B, H // 2, W // 2, 32), DEV)
    depths, state, buffered, grp = [], pipeline.KeyframeState(), [], None
    stages = (pipeline._pairnet_group_stages if pairnet else pipeline._group_stages)(mods, (0.25, 20.0, D), cache)

    def flush():
        nonlocal state
        for j, (kf, _, hits) in enumerate(buffered):
            pipeline._upload(pipeline._keyframe_rows(grp, j, B), frames[kf], hits)
        grp["ring_index"].copy_(grp["ring_table"])
        pipeline._store_misses(mods, cache, grp, B)
        for k, body in stages:
            grp[k] = body(grp)
        cache.unpin()
        if pairnet:
            depths.extend(grp["depth"][j * B:(j + 1) * B].clone() for j in range(len(buffered)))
        else:
            enc, half_K = grp["enc"]
            for j, (_, with_state, _) in enumerate(buffered):
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
                kf = key(op)
                ids = _ids(kf, M)
                if not buffered:
                    grp = pipeline._group_buffers(T, B, H, W, M, DEV)
                    pipeline._ring_buffers(grp, cache, T, B, H, W, M)
                hits = pipeline._cache_hits(cache, M, frames[kf][2], ids["reference_id"], ids["measurement_ids"])
                pipeline._reserve_keyframe(cache, grp, len(buffered), ids["reference_id"], ids["measurement_ids"], hits)
                buffered.append((kf, has_state, hits))
                has_state = True
                if len(buffered) == T:
                    flush()
        if buffered:
            flush()
    torch.cuda.synchronize()
    return depths


def _jumpy(k):
    """Keyframe index of script step k: pairs of consecutive keyframes two apart, so that every pair starts with M misses and
    each group takes more ring entries than the smallest ring keeps free -- it evicts entries the previous group reads."""
    return k + 2 * (k // 2)


def _late_feed(feed, cycles):
    """The caller's stream sleeps, then produces the inputs it submits as fresh tensors."""
    def late(k):
        torch.cuda._sleep(cycles)
        args, kw = feed(k)
        return _map(lambda t: None if t is None else t.clone(), args), kw
    return late


REPLAY = [  # pairnet, B, T, G
    pytest.param((False, 1, 3, 2), id="fusionnet-B1-T3-G2"),
    pytest.param((False, 2, 3, 2), id="fusionnet-B2-T3-G2"),
    pytest.param((True, 1, 3, 2), id="pairnet-B1-T3-G2"),
]


@pytest.mark.parametrize("cfg", REPLAY)
def test_cache_engine_equals_its_schedule_replay_under_delayed_streams(oracle, synth, delay, cfg):
    """The engine with the smallest ring (lookahead * (M + 1), so groups evict) against _replay with torch.equal on every
    keyframe of a script with a reset, an incomplete flush() and misses in every second keyframe: undelayed, with each of
    its streams delayed alone, all but the last, and the caller's stream delayed."""
    pairnet, B, T, G = cfg
    H, W, D, M = 64, 96, 64, 2
    cap = T * (M + 1)
    script, n = _lookahead_script(T, G)
    with _tc(1), torch.no_grad():
        mods, _ = _modules(oracle, synth, D, pairnet)
        frames = _frames(synth, B, _jumpy(n) + 2, H, W, M)
        eng = _engine(mods, pairnet, B, H, W, M, D, T, G, cache=cap)
        eng.prime(*frames[0])
        ref = _replay(mods, pairnet, frames, script, _jumpy, cap, T, B, H, W, M, D)
        feed = _feed(eng, frames, M, _jumpy)
        _assert_same(_run(eng, script, feed), ref, "undelayed")
        assert eng.cache.misses > M and eng.cache.hits > 0
        cycles = _calibrate(eng, "cache engine %s" % (cfg,))
        delay.install()
        for name, streams, late in _variants(eng, frames, cycles):
            with delay.on(streams, cycles):
                got = _run(eng, script, feed if late is None else _late_feed(feed, cycles))
                slept = delay.sleeps
            assert late is not None or slept > 0, name
            _assert_same(got, ref, "%s delayed" % name)


def test_planted_ring_store_on_the_trunk_stream_is_caught(oracle, synth, delay, monkeypatch):
    """The planted defect: the ring store moved from the sweep stage's graph into the trunk-tail + pyramid stage's graph, on
    another stream than the gathers.  Undelayed it may go unnoticed; with the sweep stage's stream delayed, a later group's
    store overwrites entries an earlier group has yet to gather, and the run must differ from the replay."""
    from dvmvs import pipeline
    H, W, D, M, T, G, B = 64, 96, 64, 2, 3, 2, 1
    cap = T * (M + 1)
    script, n = _lookahead_script(T, G)
    real_stages = pipeline._group_stages

    def store_in_pyramid_stage(mods, depth_args, cache=None):
        stages = real_stages(mods, depth_args, cache)
        key, pyramid = stages[1]

        def pyramid_then_store(grp):
            out = pyramid(grp)
            idx = grp["ring_index"][0]
            cache.ring.index_copy_(0, idx, out[0].permute(0, 2, 3, 1).reshape((idx.numel(), -1) + tuple(cache.ring.shape[2:])))
            return out
        return [stages[0], (key, pyramid_then_store)] + stages[2:]

    with _tc(1), torch.no_grad():
        mods, _ = _modules(oracle, synth, D, False)
        frames = _frames(synth, B, _jumpy(n) + 2, H, W, M)
        ref = _replay(mods, False, frames, script, _jumpy, cap, T, B, H, W, M, D)
        monkeypatch.setattr(pipeline, "_group_stages", store_in_pyramid_stage)
        monkeypatch.setattr(pipeline, "_ring_store", lambda grp, ring: None)
        eng = _engine(mods, False, B, H, W, M, D, T, G, cache=cap)
        eng.prime(*frames[0])
        feed = _feed(eng, frames, M, _jumpy)
        undelayed = _run(eng, script, feed)
        cycles = _calibrate(eng, "planted defect")
        delay.install()
        with delay.on([eng.streams[2]], cycles):
            delayed = _run(eng, script, feed)
    bad_u, bad_d = _diff(undelayed, ref)[0], _diff(delayed, ref)[0]
    print("planted ring store on the trunk stream: undelayed run %s, delayed run %s (%d of %d keyframes differ)"
          % ("catches it" if bad_u else "does not catch it", "catches it" if bad_d else "DOES NOT catch it", len(bad_d), len(ref)))
    assert bad_d, "the delayed run did not catch the ring store on the trunk stream"


# ------------------------------------------------------------------------------------------------ hits and misses
@pytest.mark.parametrize("pairnet", [False, True], ids=["fusionnet", "pairnet"])
def test_old_ids_hit_and_cold_start_misses_only_new_ids(oracle, synth, pairnet):
    """40 keyframes, lookahead 4, a ring of 30: keyframe t reads the reference frames of keyframes t - 1 and t - 20 (t - 2
    before t = 20), without images.  Only the two ids keyframe 0 reads, never seen before, miss; every later read hits, the
    20-keyframe-old ones included."""
    H, W, D, M, T, B = 64, 96, 64, 2, 4, 1
    with _tc(1), torch.no_grad():
        mods, _ = _modules(oracle, synth, D, pairnet)
        frames = _frames(synth, B, 40, H, W, M)
        eng = _engine(mods, pairnet, B, H, W, M, D, T, cache=30)
        eng.prime(*frames[0])
        outs, images = [], {}
        for t in range(40):
            ref, rpose, meas, mposes, K = frames[t]
            images[t] = ref
            mids = [t - 1, t - 20 if t >= 20 else t - 2]
            held = [i in eng.cache for i in mids]
            assert held == [t > 0, t > 0], (t, held)
            mimgs = [None if h else meas[m] for m, h in enumerate(held)]
            out = torch.full((B, H, W), NAN, device=DEV)
            eng.submit(ref, rpose, mimgs, mposes, K, out=out, reference_id=t, measurement_ids=mids)
            outs.append(out)
        eng.synchronize()
    assert (eng.cache.misses, eng.cache.hits) == (2, 2 * 40 - 2), (eng.cache.misses, eng.cache.hits)
    assert all(bool(torch.isfinite(o).all()) for o in outs)


# ------------------------------------------------------------------------------------------------ row independence
@pytest.mark.parametrize("B", [1, 2])
def test_pairnet_rows_are_independent_with_the_cache(oracle, synth, B):
    """Keyframe X at every position of a group of 3 and in incomplete groups of 1 and 2, the cache cleared before each group
    so that every keyframe's measurement frames miss and are computed alone: X's depth is the same bit for bit every time,
    whichever ring entries and gathered rows it gets."""
    H, W, D, M, T = 64, 96, 64, 2, 3
    with _tc(1), torch.no_grad():
        mods, _ = _modules(oracle, synth, D, True)
        frames = _frames(synth, B, 10, H, W, M)
        eng = _engine(mods, True, B, H, W, M, D, T, cache=T * (M + 1))
        eng.prime(*frames[0])
        placements = [[9, 0, 1], [2, 9, 3], [4, 5, 9], [9], [6, 9], [2, 0, 9]]      # no neighbour's reference frame is one of X's
        seen = []
        for grp in placements:
            eng.cache.clear()
            for k in grp:
                out = torch.full((B, H, W), NAN, device=DEV)
                eng.submit(*frames[k], out=out, **_ids(k, M))
                if k == 9:
                    seen.append(out)
            eng.synchronize()
        torch.cuda.synchronize()
    assert bool(torch.isfinite(seen[0]).all())
    differ = [i for i, o in enumerate(seen) if not torch.equal(o, seen[0])]
    assert not differ, "placements %s of keyframe X differ" % differ


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("point", ["c1-pairnet", "c2", "c3"])
def test_cache_engine_vs_oracle(oracle, synth, point):
    """The cache engines on the tensor-core backend with fp16 operands (bench.py's), 5 keyframes in groups of 2 (the last
    incomplete; from the second keyframe on every measurement frame hits), against the CPU oracle: oracle.pairnet_step at
    c1, oracle.fusionnet_step at the c2 and c3 shapes, within the north-star 1e-3 rel-L1 on inverse depth the engine tests
    use."""
    H, W, D, M = {"c1-pairnet": (128, 128, 32, 1), "c2": (256, 256, 64, 2), "c3": (256, 320, 96, 4)}[point]
    pairnet = point.endswith("pairnet")
    n, T = 5, 2
    Tn = torch.from_numpy
    with _tc(1), torch.no_grad():
        mods, w = _modules(oracle, synth, D, pairnet, seed=7)
        clip = synth.make_clip(0, n, H, W, M)
        frames = _frames_of(clip, M)
        eng = _engine(mods, pairnet, 1, H, W, M, D, T, cache=T * (M + 1))
        eng.prime(*frames[0])
        outs = _run(eng, list(range(n)), _feed(eng, frames, M))
        assert eng.cache.misses == M
        K = Tn(clip["K"])[None]
        st = oracle.FusionnetState()
        gold = []
        for r, ms in clip["frames"]:
            args = (Tn(clip["images"][r])[None], Tn(clip["poses"][r])[None], [Tn(clip["images"][j])[None] for j in ms],
                    [Tn(clip["poses"][j])[None] for j in ms], K)
            if pairnet:
                gold.append(oracle.pairnet_step(w, *args, n_depth_levels=D).numpy())
            else:
                g, st = oracle.fusionnet_step(w, st, *args, n_depth_levels=D)
                gold.append(g.numpy())
    errs = [oracle.rel_l1_inverse_depth(o.cpu().numpy(), g) for o, g in zip(outs, gold)]
    print("cache engine vs oracle, %s: rel-L1(inverse depth) per keyframe %s" % (point, ["%.2e" % e for e in errs]))
    assert max(errs) <= 1e-3, errs


def _frames_of(clip, M):
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)[None]
    return [(c(clip["images"][r]), c(clip["poses"][r]), [c(clip["images"][j]) for j in ms], [c(clip["poses"][j]) for j in ms],
             c(clip["K"])) for r, ms in clip["frames"]]


# ------------------------------------------------------------------------------------------------ shipped weights
@pytest.mark.parametrize("terms,bound", [(1, 3.3e-4), (3, 1e-4)])
def test_shipped_weights_reproduce_golden_with_the_cache(terms, bound):
    """The fixture scene's 10 golden keyframes through the shipped fusionnet weights: the index lines with fewer than 3
    measurement frames eagerly (keyframe()), the rest through LookaheadFusionnet(feature_cache=30, lookahead=4) continuing
    their recurrent state (load_state), with the image names as frame ids.  The misses are exactly 00003.png and the reference
    frames of the eager lines -- the frames that never passed through the engine's ring."""
    w = scene_fixture.load_shipped_weights("fusionnet")
    if w is None:
        pytest.skip("shipped weights not fetched (DVMVS_REFERENCE_ROOT=<reference checkout> python tools/fetch_fixtures.py)")
    from dvmvs import pipeline
    from oracle import dvmvs_oracle as oracle
    with open(os.path.join(scene_fixture.SCENE, "keyframe+hololens-dataset+000+nmeas+3")) as fh:
        lines = [ln.split(" ") for ln in fh.read().splitlines()]
    frames, full_K, gold = scene_fixture.load_scene()
    Tn = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)[None]
    K = Tn(full_K)
    with _tc(terms), torch.no_grad():
        mods = helpers.build_product_modules(w)
        H, W = frames[0]["reference_image"].shape[-2:]
        eng = pipeline.LookaheadFusionnet(mods, batch=1, height=H, width=W, n_measurement_frames=3, lookahead=4, feature_cache=30)
        steady = [i for i, ln in enumerate(lines) if len(ln) == 4]
        fr = frames[steady[0]]
        eng.prime(Tn(fr["reference_image"]), Tn(fr["reference_pose"]), [Tn(x) for x in fr["measurement_images"]],
                  [Tn(p) for p in fr["measurement_poses"]], K)
        preds, st = [], pipeline.KeyframeState()
        for i, fr in enumerate(frames):
            if i < steady[0]:
                pred, st = pipeline.keyframe(mods, st, Tn(fr["reference_image"]), Tn(fr["reference_pose"]),
                                             [Tn(x) for x in fr["measurement_images"]], [Tn(p) for p in fr["measurement_poses"]], K)
                preds.append(pred)
                continue
            if i == steady[0]:
                eng.load_state(st.lstm_state, st.previous_depth, st.previous_pose)
            ids = lines[i]
            images = [None if n in eng.cache else Tn(x) for n, x in zip(ids[1:], fr["measurement_images"])]
            out = torch.full((1, H, W), NAN, device=DEV)
            eng.submit(Tn(fr["reference_image"]), Tn(fr["reference_pose"]), images, [Tn(p) for p in fr["measurement_poses"]], K,
                       out=out, reference_id=ids[0], measurement_ids=ids[1:])
            preds.append(out)
        eng.synchronize()
    errs = [oracle.rel_l1_inverse_depth(p[0].cpu().numpy(), g) for p, g in zip(preds, gold)]
    print("shipped weights, cache engine, %d terms: rel-L1(inverse depth) vs golden %s" % (terms, ["%.2e" % e for e in errs]))
    assert len(preds) == len(gold) == 10
    assert max(errs) <= bound, errs
    never_in_ring = {"00003.png"} | {lines[i][0] for i in range(steady[0])}
    seen_in_engine = set()
    expected_misses = 0
    for i in steady:
        expected_misses += sum(n in never_in_ring and n not in seen_in_engine for n in lines[i][1:])
        seen_in_engine |= set(lines[i])
    assert eng.cache.misses == expected_misses == len(never_in_ring), (eng.cache.misses, expected_misses, never_in_ring)
