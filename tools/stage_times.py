"""Where does the pipelined engine's keyframe time go?  Builds bench.py's engine (PipelinedFusionnet, 5 stages, tensor-core
backend, 1 product term, 256 x 256, M = 2, D = 64, seeded weights), then replays each stage's CUDA graph ALONE, back to
back, and reports microseconds and kernel launches per stage beside the steady-state keyframe period of the whole pipeline.
The last stage carries the loop dependence (ConvLSTM state + previous depth): the period cannot drop below its latency.

    python tools/stage_times.py [--clips 1] [--stages 5] [--out profiles/r02_stage_times.json]

--lookahead N times LookaheadFusionnet instead: its period, each batched stage's graph alone (per group of N keyframes) and the
recurrent stage's graph alone (per keyframe), whose share of the period says whether the loop-carried chain bounds it.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1)
    ap.add_argument("--stages", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--pairs", type=int, default=0)
    ap.add_argument("--lookahead", type=int, default=0, help="> 0: time LookaheadFusionnet(lookahead=N) instead and compare its depths with PipelinedFusionnet's")
    ap.add_argument("--groups", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import bench
    import synth_data as synth
    from dvmvs import _ops as ops
    from dvmvs import pipeline
    from dvmvs.fusionnet.model import CostVolumeDecoder, CostVolumeEncoder, FeatureExtractor, FeatureShrinker, LSTMFusion
    ops.set_conv_backend("tc", terms=1, stride2=True)
    dev = torch.device("cuda", 0)
    H, W, D, M = bench.H, bench.W, bench.D, bench.M
    mods = {"fe": FeatureExtractor(), "fpn": FeatureShrinker(), "cve": CostVolumeEncoder(), "lstm": LSTMFusion(), "cvd": CostVolumeDecoder()}
    for m in mods.values():
        shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.make_state_dict(shapes, seed=7).items()}, strict=True)
        m.to(dev).eval()
    n_frames = 40
    clips = [synth.make_clip(c, n_frames, H, W, M) for c in range(a.clips)]
    frames = []
    for t in range(n_frames):
        ref, rpose, meas, mpose, K = bench.stack_frame(clips, t)
        frames.append((torch.from_numpy(ref).to(dev), torch.from_numpy(rpose).to(dev), [torch.from_numpy(x).to(dev) for x in meas],
                       [torch.from_numpy(p).to(dev) for p in mpose], torch.from_numpy(K).to(dev)))
    if a.lookahead > 0:
        import time
        ref_eng = pipeline.PipelinedFusionnet(mods, batch=a.clips, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, n_stages=5)
        la = pipeline.LookaheadFusionnet(mods, batch=a.clips, height=H, width=W, n_measurement_frames=M, n_depth_levels=D,
                                         lookahead=a.lookahead, n_groups=a.groups)
        n_cmp = 14
        outs_a = [torch.empty((a.clips, H, W), device=dev) for _ in range(n_cmp)]
        outs_b = [torch.empty((a.clips, H, W), device=dev) for _ in range(n_cmp)]
        with torch.no_grad():
            ref_eng.prime(*frames[0])
            la.prime(*frames[0])
            for t in range(n_cmp):
                ref_eng.submit(*frames[t], out=outs_a[t])
                la.submit(*frames[t], out=outs_b[t])
            ref_eng.synchronize()
            la.synchronize()
            errs = [float((x - y).abs().sum() / x.abs().sum()) for x, y in zip(outs_a, outs_b)]
            la.reset()
            out = torch.empty((a.clips, H, W), dtype=torch.float32, device=dev)
            for t in range(8):
                la.submit(*frames[t], out=out)
            la.synchronize()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(la.stream_a)
            h0 = time.perf_counter()
            for rep in range(3):
                for t in range(8, n_frames):
                    la.submit(*frames[t], out=out)
            la.flush()
            host_us = (time.perf_counter() - h0) * 1e6 / (3 * (n_frames - 8))
            e1.record(la.stream_b)
            la.synchronize()
            torch.cuda.synchronize()
            period = e0.elapsed_time(e1) * 1e3 / (3 * (n_frames - 8))

            def alone(graph, stream, reps):
                with torch.cuda.stream(stream):
                    for _ in range(10):
                        graph.replay()
                    q0, q1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    q0.record(stream)
                    for _ in range(reps):
                        graph.replay()
                    q1.record(stream)
                    stream.synchronize()
                return q0.elapsed_time(q1) * 1e3 / reps

            # each stage's graph replayed alone: the batched stages once per group of `lookahead` keyframes, the recurrent
            # stage once per keyframe (its replays advance the static recurrent state, restored afterwards)
            grp = la.groups[0]
            batched = [alone(grp["graph"][i], la.streams[i], max(a.reps, 50)) for i in range(4)]
            saved = la._static_state.snapshot()
            ks = next(k for k in la.kslots if True in k["graph"])
            rec_us = alone(ks["graph"][True], la.streams[4], max(a.reps, 200))
            la._static_state.restore(saved)
            torch.cuda.synchronize()
        print(json.dumps({"engine": "LookaheadFusionnet", "lookahead": a.lookahead, "groups": a.groups, "clips": a.clips,
                          "period_us_per_keyframe_batch": period, "keyframes_per_s": a.clips * 1e6 / period, "host_enqueue_us_per_submit": host_us,
                          "recurrent_stage_us_alone": rec_us, "recurrent_stage_share_of_period": rec_us / period,
                          "batched_stages_us_alone_per_group": batched, "batched_stages_us_alone_per_keyframe": sum(batched) / a.lookahead,
                          "launches_per_keyframe": la.kernels_per_keyframe, "kernels": list(la._kernels),
                          "rel_l1_depth_vs_pipelined_engine_first_14_keyframes_max": max(errs), "finite": bool(torch.isfinite(out).all())}))
        return
    eng = pipeline.PipelinedFusionnet(mods, batch=a.clips, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, n_stages=a.stages)
    out = torch.empty((a.clips, H, W), dtype=torch.float32, device=dev)
    with torch.no_grad():
        eng.prime(*frames[0])
        for t in range(8):
            eng.submit(*frames[t], out=out)
        eng.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        import time
        e0.record(eng.stream_a)
        h0 = time.perf_counter()
        for t in range(8, n_frames):
            eng.submit(*frames[t], out=out)
        host_us = (time.perf_counter() - h0) * 1e6 / (n_frames - 8)       # enqueue cost only (no synchronisation inside)
        e1.record(eng.stream_b)
        eng.synchronize()
        torch.cuda.synchronize()
        period = e0.elapsed_time(e1) * 1e3 / (n_frames - 8)
    stages = []
    slot = eng.slots[0]
    last = a.stages - 1
    for i in range(a.stages):
        g = slot["graph"][i][True if i == last else False]
        s = eng.streams[i]
        with torch.cuda.stream(s):
            for _ in range(5):
                g.replay()
            s.synchronize()
            q0, q1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            q0.record(s)
            for _ in range(a.reps):
                g.replay()
            q1.record(s)
            s.synchronize()
        stages.append({"stage": i, "us_alone": q0.elapsed_time(q1) * 1e3 / a.reps, "launches": eng._kernels[i]})
    pairs = []
    if a.pairs:
        # stage i and stage j replayed concurrently on their own streams: wall = max(alone) means they share the GPU freely,
        # wall = sum(alone) means they serialise
        graphs = [slot["graph"][i][True if i == last else False] for i in range(a.stages)]
        for i in range(a.stages):
            for j in range(i + 1, a.stages):
                torch.cuda.synchronize()
                q0, q1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                q0.record()
                eng.streams[i].wait_event(q0)
                eng.streams[j].wait_event(q0)
                for _ in range(a.reps):
                    with torch.cuda.stream(eng.streams[i]):
                        graphs[i].replay()
                    with torch.cuda.stream(eng.streams[j]):
                        graphs[j].replay()
                torch.cuda.current_stream().wait_stream(eng.streams[i])
                torch.cuda.current_stream().wait_stream(eng.streams[j])
                q1.record()
                torch.cuda.synchronize()
                both = q0.elapsed_time(q1) * 1e3 / a.reps
                ai, aj = stages[i]["us_alone"], stages[j]["us_alone"]
                pairs.append({"pair": [i, j], "us_together": both, "max_alone": max(ai, aj), "sum_alone": ai + aj,
                              "overlap": (ai + aj - both) / min(ai, aj)})
    rec = {"clips": a.clips, "n_stages": a.stages, "period_us_per_keyframe_batch": period, "keyframes_per_s": a.clips * 1e6 / period,
           "host_enqueue_us_per_submit": host_us, "sum_of_stages_us": sum(s["us_alone"] for s in stages), "stages": stages,
           "launches_per_keyframe": eng.kernels_per_keyframe, "pairs": pairs}
    print(json.dumps(rec))
    if a.out:
        json.dump(rec, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
