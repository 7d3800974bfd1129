"""The lookahead engines' feature cache without a GPU: with DVMVS_DRYRUN=1 (native entry points stubbed, see
test_dryrun_plumbing.py) one group with the cache is composed from the engines' stage bodies, eagerly and without graphs,
on CPU tensors.  Checks that the trunk runs over the T*B reference images only, that the sweep stage stores, then gathers,
then sweeps, the ring index table of a scripted id schedule (sink columns included), what the gather copies, the ring's
reservation and pinning, and every ValueError of the constructor and of submit().  Depth values are meaningless here (the
stubs write nothing); the GPU side is tests/test_lookahead_feature_cache.py.  Runs in a subprocess because the switch is
read at import time."""
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import sys, torch
sys.path.insert(0, %r); sys.path.insert(0, %r)
import synth_data as synth
from dvmvs import _ops as ops, pipeline
from oracle import dvmvs_oracle as oracle
H, W, D, M, T, B = 64, 96, 32, 2, 3, 2
TB, h, w = T * B, H // 2, W // 2
clips = [synth.make_clip(3 + c, T, H, W, M) for c in range(B)]

def weights(with_lstm):
    shapes = oracle.state_dict_shapes(D, with_lstm=with_lstm)
    return {t: {k: torch.from_numpy(v) for k, v in synth.make_state_dict(shapes[t], seed=1).items()} for t in shapes}

def frame(j):
    st = lambda pick: torch.stack([torch.from_numpy(pick(c)) for c in clips])
    ref = lambda c: c["frames"][j][0]
    meas = lambda c, m: c["frames"][j][1][m]
    return (st(lambda c: c["images"][ref(c)]), st(lambda c: c["poses"][ref(c)]), [st(lambda c: c["images"][meas(c, m)]) for m in range(M)],
            [st(lambda c: c["poses"][meas(c, m)]) for m in range(M)], st(lambda c: c["K"]))

def expect_value_error(fn, what):
    try:
        fn()
    except ValueError as e:
        print("ValueError (%%s): %%s" %% (what, e))
    else:
        raise AssertionError("no ValueError: " + what)

frames = [frame(j) for j in range(T)]
ops.set_conv_backend("tc", terms=1, stride2=True)

# ---- one group with the cache, composed from the stage bodies the engines capture
calls = []
real = {name: getattr(pipeline, name) for name in ("_ring_store", "_ring_gather", "_sweep_from_pyramid")}
for name, fn in real.items():
    setattr(pipeline, name, lambda *a, _n=name, _f=fn, **k: (calls.append(_n), _f(*a, **k))[1])
for pairnet in (True, False):
    mods = pipeline.build_modules(weights(not pairnet), device="cpu", n_depth_levels=D, pairnet=pairnet)
    cache = pipeline.FeatureCache(T * (M + 1))
    cache.allocate((B, h, w, 32), "cpu")
    grp = pipeline._group_buffers(T, B, H, W, M, "cpu")
    pipeline._ring_buffers(grp, cache, T, B, H, W, M)
    # ids: keyframe 0 misses both measurement frames; keyframe 1 reads keyframe 0's reference frame, stored by this group
    ids = [("r0", ["a", "b"]), ("r1", ["r0", "a"])]
    for j, (rid, mids) in enumerate(ids):
        hits = pipeline._cache_hits(cache, M, frames[j][2], rid, mids)
        assert hits == ([False, False] if j == 0 else [True, True]), hits
        dev_index, table = pipeline._reserve_keyframe(cache, grp, j, rid, mids, hits)
        pipeline._upload(pipeline._keyframe_rows(grp, j, B), frames[j], hits)
        dev_index.copy_(table)
    assert (cache.hits, cache.misses) == (2, 2)
    e = cache._index
    S = cache.sink
    # row 0: reference entries, rows 1 + m: measurement entries; column 2 (no keyframe) names the sink
    assert grp["ring_index"].tolist() == [[e["r0"], e["r1"], S], [e["a"], e["r0"], S], [e["b"], e["a"], S]], grp["ring_index"].tolist()
    assert grp["misses"] == [(0, 0, e["a"]), (0, 1, e["b"])], grp["misses"]
    assert cache._pinned == {e["r0"], e["r1"], e["a"], e["b"]}
    # measurement images are written only for misses: keyframe 1's rows keep the zeros of the fresh buffers
    assert torch.equal(grp["meas_images"][0][0:B], frames[0][2][0]) and float(grp["meas_images"][0][B:2 * B].abs().max()) == 0.0
    stages = (pipeline._pairnet_group_stages if pairnet else pipeline._group_stages)(mods, (0.25, 20.0, D), cache)
    calls.clear()
    for key, body in stages:
        grp[key] = body(grp)
    assert calls == ["_ring_store", "_ring_gather", "_sweep_from_pyramid"], calls
    assert [t.shape[0] for t in grp["head"]] == [TB] * len(grp["head"]), "trunk batch is not T*B"
    assert [tuple(t.shape) for t in grp["pyramid"]] == [(TB, 32, H // s, W // s) for s in (2, 4, 8, 16)]
    (f2, f4, f8, f16, cv), half_K = grp["swept"]
    assert tuple(f2.shape) == (TB, 32, h, w) and tuple(cv.shape) == (TB, D, h, w)
    enc, _ = grp["enc"]
    assert [t.shape[0] for t in enc] == [TB] * 5
    # the store writes each keyframe's B rows of a2 into its reference entry, the sink for the unfilled column
    a2 = grp["pyramid"][0].permute(0, 2, 3, 1)
    for j, rid in enumerate(["r0", "r1"]):
        assert torch.equal(cache.ring[e[rid]], a2[j * B:(j + 1) * B])
    # the gather, on its own with distinct ring contents: meas_half row block (m, j) <- ring entry ring_index[1 + m, j]
    for k in range(cache.capacity + 1):
        cache.ring[k].fill_(float(k))
    real["_ring_gather"](grp, cache.ring)
    for m in range(M):
        for j in range(T):
            rows = grp["meas_half"][m][j * B:(j + 1) * B]
            assert torch.equal(rows, cache.ring[int(grp["ring_index"][1 + m, j])]), (m, j)
    cache.unpin()
    # the next group's first keyframe starts a fresh table: every other column names the sink again
    hits = pipeline._cache_hits(cache, M, [None, None], "r2", ["r1", "r0"])
    _, table = pipeline._reserve_keyframe(cache, grp, 0, "r2", ["r1", "r0"], hits)
    assert table[:, 1:].eq(S).all() and table[:, 0].tolist() == [e["r2"], e["r1"], e["r0"]] and grp["misses"] == []
for name, fn in real.items():
    setattr(pipeline, name, fn)

# ---- reservation and pinning: no pinned entry is evicted, FIFO order otherwise
cap = 6
cache = pipeline.FeatureCache(cap)
order = []                                    # ids in the order they took an entry (FIFO reference)
for g in range(12):
    pinned_ids = []
    for k in range(3):
        fid = (g, k)
        if k == 0 and g > 0:
            fid = (g - 1, 2)                  # a hit on an id of the previous group, pinned before the new ids take entries
            assert fid in cache
        before = dict(cache._index)
        cache.reserve(fid)
        pinned_ids.append(fid)
        if fid not in before:
            gone = set(before) - set(cache._index)
            assert not gone & set(pinned_ids), (g, gone)
            unpinned = [i for i in order if i in before and i not in pinned_ids]
            assert len(before) < cap or gone == {unpinned[0]}, (g, gone, unpinned[:2])
            order.append(fid)
    assert all(i in cache for i in pinned_ids)
    cache.unpin()
# a pinned id outlives younger unpinned ones; once unpinned it is the oldest and goes first
cache = pipeline.FeatureCache(3)
cache.reserve("x")
for i in range(5):
    cache.reserve(i)
    cache._pinned.discard(cache._index[i])
assert "x" in cache and 3 in cache and 4 in cache
cache.unpin()
cache.reserve(5)
assert "x" not in cache and 3 in cache and 4 in cache
cache.unpin()
try:
    full = pipeline.FeatureCache(2)
    full.reserve(0), full.reserve(1), full.reserve(2)
except RuntimeError as e:
    print("RuntimeError:", e)
else:
    raise AssertionError("a reservation evicted a pinned entry")

# ---- ValueErrors: the constructor's capacity check, and submit()'s id rules before anything is copied
pmods = pipeline.build_modules(weights(False), device="cpu", n_depth_levels=D, pairnet=True)
fmods = pipeline.build_modules(weights(True), device="cpu", n_depth_levels=D)
for cls, mods in ((pipeline.LookaheadFusionnet, fmods), (pipeline.LookaheadPairnet, pmods)):
    for bad in (T * (M + 1) - 1, -1):
        expect_value_error(lambda: cls(mods, batch=B, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, lookahead=T,
                                       feature_cache=bad), "%%s(feature_cache=%%d)" %% (cls.__name__, bad))
    assert pipeline._lookahead_cache(T * (M + 1), T, B, H, W, M, "cpu").ring.shape == (T * (M + 1) + 1, B, h, w, 32)
    for with_cache in (True, False):
        eng = object.__new__(cls)             # only what submit() reads before its checks: a copy or launch would fail
        eng.cache, eng.M = (pipeline.FeatureCache(T * (M + 1)) if with_cache else None), M
        if with_cache:
            eng.cache.allocate((B, h, w, 32), "cpu")
            eng.cache.reserve("held")
        ref, rpose, meas, mposes, K = frames[0]
        if with_cache:
            expect_value_error(lambda: eng.submit(ref, rpose, meas, mposes, K, reference_id="r", measurement_ids=["held"]), "one id")
            expect_value_error(lambda: eng.submit(ref, rpose, meas, mposes, K, reference_id="r"), "no ids")
            expect_value_error(lambda: eng.submit(ref, rpose, [None, None], mposes, K, reference_id="r", measurement_ids=["held", "new"]),
                               "miss without an image")
            assert eng.cache.hits == eng.cache.misses == 0 and set(eng.cache._index) == {"held"}
        else:
            expect_value_error(lambda: eng.submit(ref, rpose, meas, mposes, K, measurement_ids=["a", "b"]), "ids, no cache")
            expect_value_error(lambda: eng.submit(ref, rpose, meas, mposes, K, reference_id="r"), "reference id, no cache")
print("lookahead feature cache plumbing ok")
"""


def test_lookahead_feature_cache_group_composes_without_gpu():
    env = dict(os.environ, DVMVS_DRYRUN="1")
    code = SCRIPT % (REPO, os.path.join(REPO, "deep-video-mvs_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "lookahead feature cache plumbing ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
