"""Cost of a growable SparseTSDFVolume (max_capacity_blocks; dvmvs/tsdf.py, csrc/tsdf_sparse.cu) against a fixed pool.

Frames: tools/tsdf_sparse_bench.py's (the committed pose track of fixture scene 000 with analytic box-room depth at 540 x 340),
device-resident.  Reported, in one JSON line with the card name and power limit:
  no_growth   per-frame integrate time of a fixed volume and of a growable one, both with --capacity blocks (no growth happens):
              what the ring copy of depth and colour, the pinned copy of the counters and the event cost.  CUDA events around
              each call, median over --passes passes after one untimed pass (as tsdf_sparse_bench.py), the two volumes
              alternated --rounds times.
  growth      fresh volumes from capacity_blocks=64 to the whole scene (max_capacity_blocks=--capacity), --repeats times: the
              growths, the final capacity, the host wall time of the whole track ending with allocated_blocks() (which
              settles), the CUDA-event time of the integrate calls during which a growth and replay ran, and the peak device
              allocation above what was allocated before (torch.cuda.max_memory_allocated) against a fixed pool of --capacity.
              The run checks that the grown volume's export equals the fixed volume's.

    python tools/tsdf_sparse_grow_bench.py [--voxel 0.02] [--passes 5] [--rounds 2] [--repeats 5] [--capacity 65536]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import tsdf_sparse_bench as base  # noqa: E402


def growth_run(make, dev_frames, K):
    """one fresh volume through the track: (volume, wall ms, [(frame, event ms) of the calls that grew], growths in the final
    read, peak MiB)"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    vol = make()
    grew, events = [], []
    for i, (c, d, p) in enumerate(dev_frames):
        g = vol.growths
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        vol.integrate(c, d, K, p)
        e1.record()
        if vol.growths != g:
            grew.append(i)
            events.append((e0, e1))
    g = vol.growths
    vol.allocated_blocks()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    peak = (torch.cuda.max_memory_allocated() - before) / 2 ** 20
    return vol, wall, [(i, a.elapsed_time(b)) for i, (a, b) in zip(grew, events)], vol.growths - g, peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voxel", type=float, default=0.02)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--capacity", type=int, default=65536)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tsdf_sparse_grow_bench: needs a CUDA device")
    from dvmvs.tsdf import SparseTSDFVolume
    K, fr = base.frames()
    dev_frames = [(torch.from_numpy(c).cuda(), torch.from_numpy(d).cuda(), p) for c, d, p in fr]
    rec = {"voxel": a.voxel, "image": [base.H, base.W], "frames": len(fr), "passes": a.passes, "capacity_blocks": a.capacity}
    rec["card"], rec["power_limit"] = base.card()
    make = {"fixed": lambda: SparseTSDFVolume(a.voxel, capacity_blocks=a.capacity),
            "growable": lambda: SparseTSDFVolume(a.voxel, capacity_blocks=a.capacity, max_capacity_blocks=a.capacity)}
    for warm in (make["fixed"](), make["growable"](), SparseTSDFVolume(a.voxel, capacity_blocks=64, max_capacity_blocks=a.capacity)):
        for c, d, p in dev_frames[:3]:                          # first launches load modules; the last one grows
            warm.integrate(c, d, K, p)
        warm.allocated_blocks()
    del warm
    torch.cuda.synchronize()

    runs = {"fixed": [], "growable": []}
    for _ in range(a.rounds):
        for tag in ("fixed", "growable"):
            vol = make[tag]()
            first, steady = base.time_volume(vol, dev_frames, K, a.passes)
            assert vol.growths == 0
            runs[tag].append({"ms_per_frame_first_pass": first, "ms_per_frame": steady})
            del vol
    rec["no_growth"] = runs

    fixed = make["fixed"]()
    for c, d, p in dev_frames:
        fixed.integrate(c, d, K, p)
    blocks = fixed.allocated_blocks()
    want = fixed.to_dense().get_volume_tensors()
    del fixed
    torch.cuda.empty_cache()
    _, wall_fixed, _, _, peak_fixed = growth_run(make["fixed"], dev_frames, K)
    out = []
    for _ in range(a.repeats):
        vol, wall, grew, at_read, peak = growth_run(lambda: SparseTSDFVolume(a.voxel, capacity_blocks=64, max_capacity_blocks=a.capacity), dev_frames, K)
        same = vol.allocated_blocks() == blocks and all(torch.equal(x, y) for x, y in zip(vol.to_dense().get_volume_tensors(), want))
        out.append({"growths": vol.growths, "capacity": vol.capacity, "wall_ms": wall, "grew_in_frames": [i for i, _ in grew],
                    "ms_of_calls_that_grew": [t for _, t in grew], "growths_in_final_read": at_read, "peak_MiB": peak, "equals_fixed": same})
        del vol
        torch.cuda.empty_cache()
    rec["growth"] = {"blocks": blocks, "from_capacity": 64, "runs": out, "median_wall_ms": float(np.median([r["wall_ms"] for r in out])),
                     "fixed_pool_wall_ms": wall_fixed, "fixed_pool_peak_MiB": peak_fixed,
                     "device_bytes_MiB_fixed_pool": SparseTSDFVolume.device_bytes(a.capacity) / 2 ** 20}
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
