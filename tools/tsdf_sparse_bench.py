"""Per-frame integrate time of SparseTSDFVolume against TSDFVolume over the same frames (dvmvs/tsdf.py, csrc/tsdf_sparse.cu).

Frames: the committed pose track of fixture scene 000 (tests/golden/scene000/poses_subset.npz, 11 poses, its intrinsics) with
analytic depth maps at 540 x 340: the camera inside a box room (the track's camera positions with 2 m of margin, 3 m high),
depth the distance along the optical axis to the first wall, random colours.  Dense volumes: the scene's bounds from the frames
(TSDFFusion.calculate_volume_bounds, as the reference's driver sizes its volume) and a box with 4x their voxel count (each extent
x 4^(1/3), same centre).  The sparse volume has the scene volume's origin; the run checks that its export over the scene bounds
equals the dense scene volume.

Timing: device tensors resident, CUDA events around each integrate call (the sparse call is its four allocation launches plus
the integration launch), median over `--passes` passes of the track after one untimed pass on the same volume; the first pass
into a fresh volume (every block new) is reported separately.  Prints one JSON line with the card name and power limit.

    python tools/tsdf_sparse_bench.py [--voxel 0.02] [--passes 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))

H, W = 340, 540


def card():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                      # the number still stands; the record says why the limit is missing
        power = "unknown (%s)" % e
    return name, power


def frames():
    """(colour, depth, pose) per pose of the track, depth of the box room around the track"""
    meta = np.load(os.path.join(REPO, "tests", "golden", "scene000", "poses_subset.npz"))
    K, poses = meta["K"], meta["poses"]
    centres = poses[:, :3, 3]
    lo, hi = centres.min(0) - 2.0, centres.max(0) + 2.0
    lo[1], hi[1] = centres[:, 1].mean() - 1.5, centres[:, 1].mean() + 1.5
    rng = np.random.RandomState(3)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    rays = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], axis=-1)      # camera frame, z = 1
    out = []
    for pose in poses:
        d = rays @ pose[:3, :3].T                                                                         # world directions
        c = pose[:3, 3]
        with np.errstate(divide="ignore"):
            t = np.min(np.where(d > 0, (hi - c) / d, np.where(d < 0, (lo - c) / d, np.inf)), axis=-1)     # exit from the box
        depth = t.astype(np.float32)                                                                      # z = 1 rays: t is depth
        color = rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8)
        out.append((color, depth, pose))
    return K, out


def time_volume(vol, dev_frames, K, passes):
    """(ms per frame of the first pass, median ms per frame of `passes` later passes)"""
    def one_pass():
        times = []
        for c, d, p in dev_frames:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            vol.integrate(c, d, K, p)
            e1.record()
            times.append((e0, e1))
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in times]
    first = one_pass()
    one_pass()
    later = [t for _ in range(passes) for t in one_pass()]
    return float(np.mean(first)), float(np.median(later))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voxel", type=float, default=0.02)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--capacity", type=int, default=65536)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tsdf_sparse_bench: needs a CUDA device")
    from dvmvs.tsdf import SparseTSDFVolume, TSDFFusion, TSDFVolume
    K, fr = frames()
    dev_frames = [(torch.from_numpy(c).cuda(), torch.from_numpy(d).cuda(), p) for c, d, p in fr]
    scene = TSDFFusion.calculate_volume_bounds([d for _, d, _ in fr], [p for _, _, p in fr], K)
    mid, half = scene.mean(1), (scene[:, 1] - scene[:, 0]) / 2 * 4 ** (1 / 3)
    large = np.stack([mid - half, mid + half], axis=1)
    rec = {"voxel": a.voxel, "image": [H, W], "frames": len(fr), "passes": a.passes}
    rec["card"], rec["power_limit"] = card()
    for warm in (TSDFVolume(scene, a.voxel), SparseTSDFVolume(a.voxel, capacity_blocks=a.capacity)):     # first launches load modules
        for c, d, p in dev_frames[:2]:
            warm.integrate(c, d, K, p)
    torch.cuda.synchronize()
    del warm
    for tag, bounds in (("dense_scene", scene), ("dense_4x", large)):
        vol = TSDFVolume(bounds, a.voxel)
        first, steady = time_volume(vol, dev_frames, K, a.passes)
        rec[tag] = {"bounds": bounds.tolist(), "voxels": int(np.prod(vol._vol_dim)), "MiB": 12 * int(np.prod(vol._vol_dim)) / 2 ** 20,
                    "ms_per_frame_first_pass": first, "ms_per_frame": steady}
        del vol
        torch.cuda.empty_cache()
    dense = TSDFVolume(scene, a.voxel)
    sparse = SparseTSDFVolume(a.voxel, origin=dense._vol_origin, capacity_blocks=a.capacity)
    first, steady = time_volume(sparse, dev_frames, K, a.passes)
    rec["sparse"] = {"blocks": sparse.allocated_blocks(), "capacity_blocks": a.capacity,
                     "MiB_allocated_blocks": SparseTSDFVolume.device_bytes(sparse.allocated_blocks()) / 2 ** 20,
                     "MiB_pool": SparseTSDFVolume.device_bytes(a.capacity) / 2 ** 20, "ms_per_frame_first_pass": first, "ms_per_frame": steady}
    for c, d, p in dev_frames:
        dense.integrate(c, d, K, p)
    check = SparseTSDFVolume(a.voxel, origin=dense._vol_origin, capacity_blocks=a.capacity)
    for c, d, p in dev_frames:
        check.integrate(c, d, K, p)
    rec["export_equals_dense_scene_volume"] = all(torch.equal(x, y) for x, y in zip(check.to_dense(scene).get_volume_tensors(),
                                                                                   dense.get_volume_tensors()))
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
