"""Pairnet on the GPU: dvmvs.pipeline.LookaheadPairnet at lookahead 1, 2, 4 and 8 beside eager keyframe(), at c1 (128x128,
32 planes, 1 measurement frame) and at the c2 shape for pairnet (256x256, 64 planes, 2 measurement frames), batch 1 and 8.
Prints one JSON line with the card name, power limit and maximum SM clock read in the same run.

Per operating point (tensor-core backend, fp16 operands as bench.py; synthetic posed clips of synth_data; seeded weights,
or the reference's shipped pairnet weights at 64 planes when tests/golden/_ref_data has them):
  check              rel-L1 of the engine's first keyframe against eager keyframe(); the run stops above 1e-4
  lookahead[T]       keyframes/s (and frames/s = keyframes/s x B), device-resident inputs: CUDA events around the submit
                     loop plus flush(), after prime() and a warm-up; median of --repeats windows of --steps keyframes.
                     stage_ms_per_keyframe: each of the five stage graphs replayed alone (CUDA events, 20 replays) over T,
                     so the decoder's cost per keyframe batched over T keyframes stands beside its cost at T = 1
  sequential_ms      lookahead 1 with a synchronise after every submit: latency per keyframe
  eager_ms           keyframe() with pairnet modules (per-call CUDA graphs), CUDA events around --steps keyframes

    python tools/pairnet_bench.py [--steps 96] [--warmup 16] [--repeats 3] [--points c1,c2] [--batches 1,8] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (REPO, os.path.join(REPO, "deep-video-mvs_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

POINTS = {"c1": (128, 128, 32, 1), "c2": (256, 256, 64, 2)}      # H, W, D, M
LOOKAHEADS = (1, 2, 4, 8)
N_DISTINCT = 24            # distinct synthetic keyframes per point, cycled through the timed windows


def card():
    """Card name, power limit and maximum SM clock (a read-only nvidia-smi query)."""
    idx = torch.cuda.current_device()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(idx)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power, clock = [s.strip() for s in q.split(",")]
    except Exception as e:                                   # the numbers still stand; the record says why these are missing
        power = clock = "unknown (%s)" % e
    return {"card": torch.cuda.get_device_name(idx), "power_limit": power, "sm_clock_max": clock}


def weights(D):
    from oracle import dvmvs_oracle as oracle
    from tests import scene_fixture
    import synth_data as synth
    if D == 64:
        w = scene_fixture.load_shipped_weights("pairnet")
        if w is not None:
            return w, "reference's shipped pairnet weights"
    shapes = oracle.state_dict_shapes(D, with_lstm=False)
    return ({tag: {k: torch.from_numpy(v) for k, v in synth.make_state_dict(shapes[tag], seed=7).items()} for tag in shapes},
            "random-init (seeded, He-scaled) reference architecture")


def frames(B, H, W, M):
    """N_DISTINCT keyframes of B synthetic clips (clip seed = row), device-resident, as (ref, ref_pose, [meas], [poses], K)."""
    import synth_data as synth
    clips = [synth.make_clip(c, N_DISTINCT, H, W, M) for c in range(B)]
    st = lambda pick: torch.from_numpy(np.ascontiguousarray(np.stack([pick(c) for c in clips]))).cuda()
    out = []
    for t in range(N_DISTINCT):
        ref = lambda c: c["frames"][t][0]
        meas = lambda c, m: c["frames"][t][1][m]
        out.append((st(lambda c: c["images"][ref(c)]), st(lambda c: c["poses"][ref(c)]), [st(lambda c: c["images"][meas(c, m)]) for m in range(M)],
                    [st(lambda c: c["poses"][meas(c, m)]) for m in range(M)], st(lambda c: c["K"])))
    return out


def events_ms(fn, start_stream=None, end_stream=None):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(start_stream or torch.cuda.current_stream())
    end = fn()
    e1.record(end_stream or end or torch.cuda.current_stream())
    e1.synchronize()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def stage_ms(eng):
    """Each stage graph of group 0 replayed alone on its stream, 20 replays, ms per replay."""
    out = []
    for i in range(5):
        g, s = eng.groups[0]["graph"][i], eng.streams[i]

        def replays():
            for _ in range(20):
                g.replay()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            g.replay()
            out.append(events_ms(replays, s, s) / 20.0)
    return out


def bench_point(name, B, args):
    from dvmvs import pipeline
    H, W, D, M = POINTS[name]
    w, wdesc = weights(D)
    mods = pipeline.build_modules(w, n_depth_levels=D, pairnet=True)
    fr = frames(B, H, W, M)
    nf = len(fr)
    rec = {"point": name, "batch": B, "height": H, "width": W, "planes": D, "measurement_frames": M, "weights": wdesc,
           "timed_keyframes": args.steps, "repeats": args.repeats, "lookahead": {}}
    out = torch.empty((B, H, W), dtype=torch.float32, device="cuda")
    with torch.no_grad():
        # eager keyframe(): the reference's call sequence through the drop-in modules (per-call CUDA graphs)
        eager0 = pipeline.keyframe(mods, pipeline.KeyframeState(), *fr[0], n_depth_levels=D)[0].clone()
        for t in range(args.warmup):
            pipeline.keyframe(mods, pipeline.KeyframeState(), *fr[t % nf], n_depth_levels=D)
        def eager():
            for t in range(args.steps):
                pipeline.keyframe(mods, pipeline.KeyframeState(), *fr[t % nf], n_depth_levels=D)
        ms = [events_ms(eager) for _ in range(args.repeats)]
        rec["eager_ms"] = float(np.median(ms)) / args.steps
        rec["eager_keyframes_per_s"] = 1e3 / rec["eager_ms"]
        for T in LOOKAHEADS:
            eng = pipeline.LookaheadPairnet(mods, batch=B, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, lookahead=T)
            eng.prime(*fr[0])
            eng.submit(*fr[0], out=out)
            eng.synchronize()
            check = float((out - eager0).abs().sum() / eager0.abs().sum())
            if not check <= 1e-4:
                raise SystemExit("%s B=%d lookahead %d: the engine's first keyframe deviates from eager keyframe(): rel-L1 %g"
                                 % (name, B, T, check))
            for t in range(args.warmup):
                eng.submit(*fr[t % nf], out=out)
            eng.synchronize()

            def window():
                for t in range(args.steps):
                    eng.submit(*fr[t % nf], out=out)
                eng.flush()
                return eng.stream_b
            ms = [events_ms(window, eng.stream_a) for _ in range(args.repeats)]
            eng.synchronize()
            kps = args.steps / (float(np.median(ms)) * 1e-3)
            rec["lookahead"][str(T)] = {"keyframes_per_s": kps, "frames_per_s": kps * B, "check_rel_l1": check,
                                        "windows_ms": ms, "kernels_per_keyframe": eng.kernels_per_keyframe,
                                        "stage_ms_per_keyframe": [s / T for s in stage_ms(eng)]}
            if T == 1:
                def sequential():
                    for t in range(args.steps):
                        eng.submit(*fr[t % nf], out=out)
                        eng.synchronize()
                ms = [events_ms(sequential) for _ in range(args.repeats)]
                rec["sequential_ms"] = float(np.median(ms)) / args.steps
            del eng
            torch.cuda.empty_cache()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=96, help="keyframes per timed window")
    ap.add_argument("--warmup", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--points", default="c1,c2")
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pairnet_bench.py needs a CUDA device")
    from dvmvs import _ops as ops
    ops.set_conv_backend("tc", terms=1, stride2=True)
    rec = dict(card(), backend="tc, 1-term fp16 operands", points=[])
    for name in a.points.split(","):
        for B in (int(b) for b in a.batches.split(",")):
            rec["points"].append(bench_point(name, B, a))
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
