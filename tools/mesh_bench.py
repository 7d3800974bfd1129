"""Times TSDFVolume.get_mesh_tensors (marching cubes on the device, csrc/mesh.cu) with CUDA events over many calls, and
get_mesh end to end (device work, the one count read-back and the mesh copy to the host), on rooms fused from synthetic frames:
8 x 6.4 x 4.8 m at 4 cm (3.84 M voxels) and at 2 cm (30.7 M voxels).  Puts it against HBM (4 B per voxel read + the mesh
written) and times the numpy oracle beside it as the CPU figure.  Prints the card name and power limit of the run.

    python tools/mesh_bench.py [--voxels 0.04,0.02] [--frames 20] [--calls 50] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))
sys.path.insert(0, os.path.join(REPO, "oracle"))
sys.path.insert(0, os.path.join(REPO, "tools"))
from tsdf_bench import frame  # noqa: E402

HBM_GBPS = 3350.0            # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                      # the number still stands; the record says why the limit is missing
        power = "unknown (%s)" % e
    return name, power


def bench_room(voxel, n_frames, calls):
    from dvmvs.tsdf import TSDFVolume
    import mesh_oracle
    h, w = 256, 320
    K = np.array([[250.0, 0, 160.3], [0, 251.0, 127.6], [0, 0, 1]])
    vol = TSDFVolume(np.array([[-4.0, 4.0], [-3.2, 3.2], [0.0, 4.8]]), voxel)
    rng = np.random.RandomState(5)
    for i in range(n_frames):
        c, d, p = frame(i, h, w, rng)
        vol.integrate(c, d, K, p)
    n_vox = int(np.prod(vol._vol_dim))
    for _ in range(3):                                          # warm-up: module load, allocator
        mesh = vol.get_mesh_tensors()
    torch.cuda.synchronize()
    n_verts, n_faces = int(mesh[0].shape[0]), int(mesh[1].shape[0])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        vol.get_mesh_tensors()
    e1.record()
    e1.synchronize()
    t_dev = e0.elapsed_time(e1) * 1e-3 / calls
    t0 = time.perf_counter()
    for _ in range(calls):
        vol.get_mesh()
    t_e2e = (time.perf_counter() - t0) / calls
    tsdf, color = vol.get_volume()
    t0 = time.perf_counter()
    mesh_oracle.marching_cubes(tsdf, color, vol._voxel_size, vol._vol_origin)
    t_cpu = time.perf_counter() - t0
    mesh_bytes = n_verts * (12 + 12 + 3) + n_faces * 12
    alg = 4.0 * n_vox + mesh_bytes
    return {"voxel_m": voxel, "vol_dim": [int(v) for v in vol._vol_dim], "voxels": n_vox, "frames_fused": n_frames,
            "verts": n_verts, "faces": n_faces, "get_mesh_tensors_us": t_dev * 1e6, "voxels_per_s": n_vox / t_dev,
            "algorithmic_bytes": alg, "achieved_GBps": alg / t_dev * 1e-9, "hbm_share_of_datasheet": alg / t_dev * 1e-9 / HBM_GBPS,
            "get_mesh_end_to_end_us": t_e2e * 1e6, "cpu_oracle_s": t_cpu, "speedup_vs_cpu_oracle": t_cpu / t_dev}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voxels", default="0.04,0.02")
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench.py needs a CUDA device")
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
