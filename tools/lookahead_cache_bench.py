"""The lookahead engines with and without the feature cache (row f1) on the GPU: LookaheadFusionnet at c2 (256x256, 64 planes,
2 measurement frames) and c3 (256x320, 96 planes, 4 measurement frames), LookaheadPairnet at c1 (128x128, 32 planes, 1
measurement frame) and the c2 shape; lookahead 4 and 8, batch 1.  Prints one JSON line with the card name, power limit and
maximum SM clock read in the same run.

The keyframe schedule is a real one: tests/golden/keyframes/poses_000.npy replayed through dvmvs.keyframe_buffer.KeyframeBuffer
(the reference's selection, M measurement frames; keyframes with fewer are skipped), cycled, each cycle a new clip (reset(),
fresh frame ids).  Images are seeded synthetic images per frame id, device-resident; weights are seeded (random-init).
Tensor-core backend with fp16 operands, as bench.py.  Per point and engine:
  keyframes_per_s     CUDA events around --steps submits plus flush(), after prime() and a warm-up; median of --repeats
  hits / misses       the cache's counters over the timed windows
  stage_ms_per_keyframe  each stage graph of group 0 replayed alone (20 replays) over the lookahead; for fusionnet the
                     recurrent stage's graph per keyframe last
  check_rel_l1        max rel-L1 (inverse depth) of the first 2 x lookahead keyframes against the cache-less engine
  profile_us_per_keyframe  a separate torch.profiler window: CUDA time per keyframe of the ring gather (index_select), the ring
                     store (index_copy_) and the fp32 -> fp16 operand splits (split_planes kernels, in both engines: the
                     difference is the split of the gathered rows)

    python tools/lookahead_cache_bench.py [--steps 96] [--warmup 16] [--repeats 3] [--lookaheads 4,8] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (REPO, os.path.join(REPO, "deep-video-mvs_b200"), os.path.join(REPO, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from pairnet_bench import card  # noqa: E402

POINTS = {"fusionnet-c2": (256, 256, 64, 2, False), "fusionnet-c3": (256, 320, 96, 4, False),
          "pairnet-c1": (128, 128, 32, 1, True), "pairnet-c2": (256, 256, 64, 2, True)}      # H, W, D, M, pairnet
PROFILE_KERNELS = {"gather": ("indexselect",), "store": ("index_copy", "indexcopy", "indexfunc"), "split": ("split_planes",)}


def schedule(M):
    """(reference id, reference pose, [measurement ids], [measurement poses]) of every keyframe the reference's keyframe buffer
    selects on the committed pose track with M measurement frames."""
    from dvmvs.config import Config
    from dvmvs.keyframe_buffer import KeyframeBuffer
    poses = np.load(os.path.join(REPO, "tests", "golden", "keyframes", "poses_000.npy"))
    buf = KeyframeBuffer(buffer_size=Config.test_keyframe_buffer_size, keyframe_pose_distance=Config.test_keyframe_pose_distance,
                         optimal_t_score=Config.test_optimal_t_measure, optimal_R_score=Config.test_optimal_R_measure,
                         store_return_indices=False)
    out = []
    for pose in poses:
        if buf.try_new_keyframe(pose, None) != 1:
            continue
        frames, ids = buf.get_best_measurement_frames(M, with_ids=True)
        if len(ids) == M:
            out.append((buf.last_frame_id, pose, list(ids), [f[0] for f in frames]))
    return out


class Feeder:
    """Keyframe t of the cycled schedule as submit() arguments; cycle c's frame ids are (c, id), so that each cycle is a new
    clip whose first measurement frames miss."""

    def __init__(self, sched, H, W):
        import synth_data as synth
        ids = sorted({i for r, _, ms, _ in sched for i in [r] + ms})
        self.images = {i: torch.from_numpy(synth.smooth_image("kb/%d" % i, H, W, seed=i))[None].cuda() for i in ids}
        pose = lambda p: torch.from_numpy(np.ascontiguousarray(p, dtype=np.float32))[None].cuda()
        self.sched = [(r, pose(rp), ms, [pose(p) for p in mp]) for r, rp, ms, mp in sched]
        self.K = torch.from_numpy(synth.intrinsics(H, W))[None].cuda()

    def plain(self, t):
        r, rp, ms, mp = self.sched[t % len(self.sched)]
        return self.images[r], rp, [self.images[i] for i in ms], mp, self.K

    def __call__(self, eng, t):
        """(args, kwargs, new clip?) of keyframe t for `eng` (ids only when it has a cache)."""
        c, k = divmod(t, len(self.sched))
        r, rp, ms, mp = self.sched[k]
        if eng.cache is None:
            return self.plain(t), {}, k == 0
        mids = [(c, i) for i in ms]
        imgs = [None if i in eng.cache else self.images[i[1]] for i in mids]
        return (self.images[r], rp, imgs, mp, self.K), {"reference_id": (c, r), "measurement_ids": mids}, k == 0


def events_ms(fn, start, end):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(start)
    fn()
    e1.record(end)
    e1.synchronize()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def stage_ms(eng):
    graphs = [(g, eng.streams[i]) for i, g in enumerate(eng.groups[0]["graph"])]
    rec = [ks["graph"][True] for ks in eng.kslots if True in ks.get("graph", {})]
    if rec:
        graphs.append((rec[0], eng.streams[4]))
    out = []
    for g, s in graphs:
        def replays():
            for _ in range(20):
                g.replay()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            g.replay()
            out.append(events_ms(replays, s, s) / 20.0)
    return [ms / eng.T for ms in out[:len(eng.groups[0]["graph"])]] + out[len(eng.groups[0]["graph"]):]


def run(eng, feed, t0, n, out):
    for t in range(t0, t0 + n):
        args, kw, new_clip = feed(eng, t)
        if new_clip:
            eng.reset()
        eng.submit(*args, out=out, **kw)


def first_depths(eng, feed, n, B, H, W):
    eng.reset()
    if eng.cache is not None:
        eng.cache.clear()
    outs = [torch.empty((B, H, W), device="cuda") for _ in range(n)]
    for t in range(n):
        args, kw, _ = feed(eng, t)
        eng.submit(*args, out=outs[t], **kw)
    eng.synchronize()
    return outs


def profile_us(eng, feed, t0, n, out):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(eng, feed, t0, n, out)
        eng.synchronize()
        torch.cuda.synchronize()
    tot = {k: 0.0 for k in PROFILE_KERNELS}
    names = {k: set() for k in PROFILE_KERNELS}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        low = ev.name.lower()
        for k, pats in PROFILE_KERNELS.items():
            if any(p in low for p in pats):
                tot[k] += ev.device_time
                names[k].add(ev.name[:80])
    return {k: tot[k] / n for k in tot}, {k: sorted(v) for k, v in names.items()}


def bench_point(name, T, args):
    from dvmvs import pipeline
    from oracle import dvmvs_oracle as oracle
    import synth_data as synth
    H, W, D, M, pairnet = POINTS[name]
    B = 1
    shapes = oracle.state_dict_shapes(D, with_lstm=not pairnet)
    w = {tag: {k: torch.from_numpy(v) for k, v in synth.make_state_dict(shapes[tag], seed=7).items()} for tag in shapes}
    mods = pipeline.build_modules(w, n_depth_levels=D, pairnet=pairnet)
    sched = schedule(M)
    feed = Feeder(sched, H, W)
    cls = pipeline.LookaheadPairnet if pairnet else pipeline.LookaheadFusionnet
    rec = {"point": name, "lookahead": T, "batch": B, "height": H, "width": W, "planes": D, "measurement_frames": M,
           "schedule_keyframes": len(sched), "timed_keyframes": args.steps, "repeats": args.repeats, "engines": {}}
    out = torch.empty((B, H, W), device="cuda")
    ref = None
    with torch.no_grad():
        for cache in (0, max(30, T * (M + 1))):
            eng = cls(mods, batch=B, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, lookahead=T, feature_cache=cache)
            eng.prime(*feed.plain(0))
            first = first_depths(eng, feed, 2 * T, B, H, W)
            if ref is None:
                ref = first
            check = max(oracle.rel_l1_inverse_depth(a.cpu().numpy(), b.cpu().numpy()) for a, b in zip(first, ref))
            if cache:
                eng.cache.clear()
            eng.reset()
            run(eng, feed, 0, args.warmup, out)
            eng.synchronize()
            h0, m0 = (eng.cache.hits, eng.cache.misses) if cache else (0, 0)
            t = args.warmup
            ms = []
            for _ in range(args.repeats):
                def window():
                    run(eng, feed, t, args.steps, out)
                    eng.flush()
                ms.append(events_ms(window, eng.stream_a, eng.stream_b))
                t += args.steps
            eng.synchronize()
            kps = args.steps / (float(np.median(ms)) * 1e-3)
            r = {"feature_cache": cache, "keyframes_per_s": kps, "windows_ms": ms, "check_rel_l1": check,
                 "stage_ms_per_keyframe": stage_ms(eng), "kernels_per_keyframe": eng.kernels_per_keyframe}
            if cache:
                r.update(hits=eng.cache.hits - h0, misses=eng.cache.misses - m0)
            r["profile_us_per_keyframe"], r["profile_kernels"] = profile_us(eng, feed, t, args.steps, out)
            rec["engines"]["cache" if cache else "no_cache"] = r
            del eng
            torch.cuda.empty_cache()
    if rec["engines"]["cache"]["check_rel_l1"] > 1e-3:
        raise SystemExit("%s lookahead %d: the cache engine deviates from the cache-less one: %s" % (name, T, rec))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=96, help="keyframes per timed window")
    ap.add_argument("--warmup", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--points", default=",".join(POINTS))
    ap.add_argument("--lookaheads", default="4,8")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lookahead_cache_bench.py needs a CUDA device")
    from dvmvs import _ops as ops
    ops.set_conv_backend("tc", terms=1, stride2=True)
    rec = dict(card(), backend="tc, 1-term fp16 operands", points=[])
    for name in a.points.split(","):
        for T in (int(x) for x in a.lookaheads.split(",")):
            rec["points"].append(bench_point(name, T, a))
            print(json.dumps(rec["points"][-1]), file=sys.stderr)
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
