"""Mesh and ray casting of SparseTSDFVolume on its blocks against the dense route (dvmvs/tsdf.py, csrc/tsdf_sparse_view.cu).

Volume: tools/tsdf_sparse_bench.py's frames (the committed pose track, analytic box-room depth) at 2 cm and 4 cm.  Per voxel size:
  mesh    sparse get_mesh_tensors()  against  to_dense() + get_mesh_tensors()
  render  sparse render_tensors(every pose of the track, one call)  against  to_dense() + render_tensors(), and against
          render_tensors() on an already exported volume (kernel against kernel)
each timed with CUDA events after a warm-up call, median of --repeats, with the peak allocation of the call
(torch.cuda.max_memory_allocated after a reset, above what was allocated before) and a torch.equal check of the results.
Long path: the track replicated at --copies offsets --spacing metres apart along a diagonal, where the default box is too large
to export; only the sparse path runs.  Prints one JSON line with the card name and power limit.

    python tools/tsdf_sparse_view_bench.py [--repeats 10] [--copies 3] [--spacing 30]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import tsdf_sparse_bench as base  # noqa: E402

RH, RW = 240, 320


def timed(f, repeats):
    """(median ms, peak MiB above the allocation before the call, the last result)"""
    out = f()
    torch.cuda.synchronize()
    times, peak = [], 0
    for _ in range(repeats):
        del out
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        before = torch.cuda.memory_allocated()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = f()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
        peak = max(peak, torch.cuda.max_memory_allocated() - before)
    return float(np.median(times)), peak / 2 ** 20, out


def equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--copies", type=int, default=3)
    ap.add_argument("--spacing", type=float, default=30.0)
    ap.add_argument("--capacity", type=int, default=65536)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tsdf_sparse_view_bench: needs a CUDA device")
    from dvmvs.tsdf import SparseTSDFVolume
    K, fr = base.frames()
    dev = [(torch.from_numpy(c).cuda(), torch.from_numpy(d).cuda(), p) for c, d, p in fr]
    poses = np.stack([p for _, _, p in fr])
    Kr = K.copy()
    Kr[:2] *= RW / base.W
    rec = {"repeats": a.repeats, "render": [len(poses), RH, RW]}
    rec["card"], rec["power_limit"] = base.card()
    for voxel in (0.02, 0.04):
        vol = SparseTSDFVolume(voxel, capacity_blocks=a.capacity)
        for c, d, p in dev:
            vol.integrate(c, d, K, p)
        n = vol.allocated_blocks()
        dense = vol.to_dense()
        r = {"blocks": n, "box_voxels": int(np.prod(dense._vol_dim)), "block_voxels": n * 512}
        ms, mib, ms_ = timed(lambda: vol.get_mesh_tensors(), a.repeats)
        r["mesh_sparse"] = {"ms": ms, "peak_MiB": mib, "faces": int(ms_[1].shape[0])}
        ms, mib, md = timed(lambda: vol.to_dense().get_mesh_tensors(), a.repeats)
        r["mesh_export_then_dense"] = {"ms": ms, "peak_MiB": mib}
        r["mesh_equal"] = equal(ms_, md)
        ms, mib, rs = timed(lambda: vol.render_tensors(Kr, poses, RH, RW), a.repeats)
        r["render_sparse"] = {"ms": ms, "peak_MiB": mib, "hits": int((rs[0] > 0).sum())}
        ms, mib, rd = timed(lambda: vol.to_dense().render_tensors(Kr, poses, RH, RW), a.repeats)
        r["render_export_then_dense"] = {"ms": ms, "peak_MiB": mib}
        ms, mib, rk = timed(lambda: dense.render_tensors(Kr, poses, RH, RW), a.repeats)
        r["render_dense_kernel_only"] = {"ms": ms, "peak_MiB": mib}
        r["render_equal"] = equal(rs, rd) and equal(rs, rk)
        rec["voxel_%g" % voxel] = r
        del vol, dense, ms_, md, rs, rd, rk
        torch.cuda.empty_cache()
    # long path: the track copied along a diagonal; the default box cannot be exported
    voxel = 0.02
    vol = SparseTSDFVolume(voxel, capacity_blocks=a.capacity * a.copies)
    for i in range(a.copies):
        shift = np.full(3, a.spacing * i)
        for c, d, p in dev:
            q = p.copy()
            q[:3, 3] += shift
            vol.integrate(c, d, K, q)
    n = vol.allocated_blocks()
    _, _, vb = vol._box(None, "bench")
    dims = np.ceil((vb[:, 1] - vb[:, 0]) / voxel)
    r = {"copies": a.copies, "spacing_m": a.spacing, "blocks": n, "box_voxels": float(np.prod(dims)),
         "dense_export_GB": 12 * float(np.prod(dims)) / 1e9}
    ms, mib, m = timed(lambda: vol.get_mesh_tensors(), a.repeats)
    r["mesh_sparse"] = {"ms": ms, "peak_MiB": mib, "faces": int(m[1].shape[0])}
    long_poses = []
    for i in range(a.copies):
        q = poses.copy()
        q[:, :3, 3] += a.spacing * i
        long_poses.append(q)
    long_poses = np.concatenate(long_poses)
    ms, mib, rr = timed(lambda: vol.render_tensors(Kr, long_poses, RH, RW), a.repeats)
    r["render_sparse"] = {"ms": ms, "peak_MiB": mib, "views": len(long_poses), "hits": int((rr[0] > 0).sum())}
    rec["long_path"] = r
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
