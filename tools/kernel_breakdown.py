"""Where does the GPU time of bench.py's default workload go, kernel by kernel?  Builds bench.py's engine the way
tools/stage_times.py does (LookaheadFusionnet, lookahead 4, tensor-core backend, 1 product term, 256 x 256, M = 2, D = 64,
seeded weights), runs it to steady state, then records `--keyframes` keyframes under torch.profiler (CUDA activities
only, in a run of its own: no timing is taken here) and prints one row per kernel name: launches, total us and share of
the kernel time, all per keyframe.  The last line is a JSON record; --out also writes it to a file.

    python tools/kernel_breakdown.py [--keyframes 48] [--out kernels.json]
"""
import argparse
import collections
import json
import os
import re
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))


def short_name(name):
    """'void dvmvs::conv_halo_kernel<32, 5, 16, 1>(dvmvs::HaloParams)' -> 'conv_halo_kernel<32, 5, 16, 1>'"""
    name = re.sub(r"^void ", "", name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):                 # drop the parameter list (the first '(' outside template brackets)
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    return name[:cut].replace("dvmvs::", "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=48, help="profiled keyframes (a multiple of the lookahead keeps groups whole)")
    ap.add_argument("--lookahead", type=int, default=4)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kernel_breakdown: needs a GPU")
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
    n_warm = 2 * a.lookahead * 3
    n_frames = n_warm + a.keyframes
    clips = [synth.make_clip(0, n_frames, H, W, M)]
    frames = []
    for t in range(n_frames):
        ref, rpose, meas, mpose, K = bench.stack_frame(clips, t)
        frames.append((torch.from_numpy(ref).to(dev), torch.from_numpy(rpose).to(dev), [torch.from_numpy(x).to(dev) for x in meas],
                       [torch.from_numpy(p).to(dev) for p in mpose], torch.from_numpy(K).to(dev)))
    eng = pipeline.LookaheadFusionnet(mods, batch=1, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, lookahead=a.lookahead)
    out = torch.empty((1, H, W), dtype=torch.float32, device=dev)
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        eng.prime(*frames[0])
        for t in range(n_warm):
            eng.submit(*frames[t], out=out)
        eng.flush()
        eng.synchronize()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for t in range(n_warm, n_frames):
                eng.submit(*frames[t], out=out)
            eng.flush()
            eng.synchronize()
            torch.cuda.synchronize()
    count, us = collections.Counter(), collections.Counter()
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        n = short_name(e.name)
        count[n] += 1
        us[n] += e.time_range.elapsed_us()
    total = sum(us.values())
    kf = float(a.keyframes)
    rows = [{"kernel": n, "launches_per_keyframe": count[n] / kf, "us_per_keyframe": us[n] / kf, "share": us[n] / total}
            for n in sorted(us, key=lambda n: -us[n])]
    print("%-60s %9s %10s %7s" % ("kernel", "launches", "us", "share"))
    for r in rows:
        print("%-60s %9.2f %10.1f %6.1f%%" % (r["kernel"][:60], r["launches_per_keyframe"], r["us_per_keyframe"], 100 * r["share"]))
    halo = [r for r in rows if r["kernel"].startswith("conv_halo_kernel")]
    halo_us = sum(r["us_per_keyframe"] for r in halo)
    print("kernel time per keyframe %.1f us; conv_halo_kernel %.1f us = %.1f%% (%.1f launches)"
          % (total / kf, halo_us, 100 * halo_us / (total / kf), sum(r["launches_per_keyframe"] for r in halo)))
    rec = {"device": torch.cuda.get_device_name(0), "keyframes": a.keyframes, "lookahead": a.lookahead,
           "kernel_us_per_keyframe": total / kf, "halo_us_per_keyframe": halo_us, "halo_share": halo_us / (total / kf), "kernels": rows}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
