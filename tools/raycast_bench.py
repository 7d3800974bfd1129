"""Times TSDFVolume.render_tensors (ray casting on the device, csrc/raycast.cu) with CUDA events over many calls, on the room of
tools/tsdf_bench.py fused from 20 synthetic frames: 8 x 6.4 x 4.8 m at 4 cm (3.84 M voxels) and at 2 cm (30.7 M voxels).  The 20
poses are rendered at 256 x 320 one view per call and all 20 views in one call; each mode also runs through the C entry point
with preallocated outputs (no Python packing), which is the kernel time once the host outruns the device.  Rates: views/s, rays/s
and lattice samples/s, the samples counted by the numpy oracle on view 0 (tsdf evaluations of its march, jump probes
included); the oracle's time on that one view is the CPU figure.  Prints the card name and power limit of the run.

    python tools/raycast_bench.py [--voxels 0.04,0.02] [--frames 20] [--calls 50] [--out FILE.json]
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
sys.path.insert(0, os.path.join(REPO, "oracle"))
sys.path.insert(0, os.path.join(REPO, "tools"))
from mesh_bench import card  # noqa: E402
from tsdf_bench import frame  # noqa: E402


def timed(fn, calls):
    for _ in range(3):                                          # warm-up: module load, allocator, staging ring
        fn(0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for c in range(calls):
        fn(c)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / calls


def bench_room(voxel, n_frames, calls):
    from dvmvs import _native as N
    from dvmvs._ops import _stream
    from dvmvs.tsdf import TSDFVolume
    import raycast_oracle
    h, w = 256, 320
    K = np.array([[250.0, 0, 160.3], [0, 251.0, 127.6], [0, 0, 1]])
    vol = TSDFVolume(np.array([[-4.0, 4.0], [-3.2, 3.2], [0.0, 4.8]]), voxel)
    rng = np.random.RandomState(5)
    poses = []
    for i in range(n_frames):
        c, d, p = frame(i, h, w, rng)
        vol.integrate(c, d, K, p)
        poses.append(p)
    poses = np.stack(poses)
    n = len(poses)
    poses_dev = torch.from_numpy(poses).cuda()
    t_one = timed(lambda c: vol.render_tensors(K, poses_dev[c % n], h, w), calls)
    t_all = timed(lambda c: vol.render_tensors(K, poses_dev, h, w), calls) / n

    views = torch.from_numpy(raycast_oracle.views_of(K, poses)).cuda()
    depth = torch.empty((n, h, w), dtype=torch.float32, device="cuda")
    normals = torch.empty((n, h, w, 3), dtype=torch.float32, device="cuda")
    colors = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda")
    tsdf_t, _, color_t = vol.get_volume_tensors()
    dims = [int(v) for v in vol._vol_dim]

    def launch(first, count):
        N.check(N.lib().dvmvs_tsdf_raycast(tsdf_t.data_ptr(), color_t.data_ptr(), dims[0], dims[1], dims[2], vol._origin_c,
                                           vol._voxel_size, vol._trunc_margin, views[first:].data_ptr(), count, h, w,
                                           depth[first:].data_ptr(), normals[first:].data_ptr(), colors[first:].data_ptr(),
                                           _stream()), "tsdf_raycast")
    t_one_abi = timed(lambda c: launch(c % n, 1), calls)
    t_all_abi = timed(lambda c: launch(0, n), calls) / n
    hits = float((depth > 0).float().mean())

    tsdf, color = vol.get_volume()
    t0 = time.perf_counter()
    _, _, _, aux = raycast_oracle.render(tsdf, color, vol._vol_origin, vol._voxel_size, vol._trunc_margin, K, poses[0], h, w,
                                         return_aux=True)
    t_cpu = time.perf_counter() - t0
    samples = int(aux["samples"].sum())
    rays = h * w
    rec = {"voxel_m": voxel, "vol_dim": dims, "voxels": int(np.prod(dims)), "frames_fused": n_frames, "image": [h, w],
           "views": n, "hit_fraction": hits, "samples_view0": samples, "samples_per_ray_view0": samples / rays}
    for name, t in (("one_view_per_call", t_one), ("all_views_one_call", t_all), ("one_view_per_launch_c_abi", t_one_abi),
                    ("all_views_one_launch_c_abi", t_all_abi)):
        rec[name] = {"us_per_view": t * 1e6, "views_per_s": 1.0 / t, "rays_per_s": rays / t, "samples_per_s": samples / t}
    rec.update({"cpu_oracle_s_view0": t_cpu, "speedup_vs_cpu_oracle": t_cpu / t_all_abi})
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voxels", default="0.04,0.02")
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("raycast_bench.py needs a CUDA device")
    name, power = card()
    recs = []
    for v in (float(s) for s in a.voxels.split(",")):
        rec = bench_room(v, a.frames, a.calls)
        rec.update({"card": name, "power_limit": power})
        print(json.dumps(rec))
        recs.append(rec)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(recs, fh, indent=1)


if __name__ == "__main__":
    main()
