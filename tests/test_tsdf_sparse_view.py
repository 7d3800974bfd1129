"""Mesh and ray casting of SparseTSDFVolume on its blocks (dvmvs/tsdf.py, csrc/tsdf_sparse_view.cu,
include/dvmvs_tsdf_sparse_view.h).  Their contract: over any lattice-aligned box, and the default box, get_mesh_tensors and
render_tensors return exactly what to_dense(box) followed by the dense method returns (torch.equal, order included); the dense
kernels are pinned to numpy oracles by tests/test_mesh.py and tests/test_raycast.py.

CPU: the header against the library and the ctypes binding, argument refusal without a GPU, and (DVMVS_DRYRUN=1, in a
subprocess) the box validation, the overflow flags and the render argument errors."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle"))
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))
import tsdf_cases  # noqa: E402

from tests.test_tsdf import _rot  # noqa: E402
from tests.test_tsdf_sparse import PATH_K, PATH_VOXEL, _adversarial_frames, _fuse, _path_frames, _production_frames  # noqa: E402

# every entry point of include/dvmvs_tsdf_sparse_view.h -> the test of this module that checks what it computes
VIEW_TESTS = {
    "dvmvs_tsdf_sparse_mesh_scratch_bytes": "test_gpu_memory_scales_with_the_blocks_not_the_box",
    "dvmvs_tsdf_sparse_mesh_count": "test_gpu_mesh_and_render_equal_the_export_on_every_box",
    "dvmvs_tsdf_sparse_mesh_extract": "test_gpu_mesh_and_render_equal_the_export_on_every_box",
    "dvmvs_tsdf_sparse_raycast": "test_gpu_mesh_and_render_equal_the_export_on_every_box",
}
VIEW_HOST_ONLY = set()


def _header_prototypes():
    header = open(os.path.join(REPO, "include", "dvmvs_tsdf_sparse_view.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    return re.findall(r"\bint\s+(dvmvs_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", header)


def test_view_header_library_binding_and_coverage_agree():
    """Every prototype of include/dvmvs_tsdf_sparse_view.h is exported, listed in SPARSE_VIEW_SYMBOLS, bound with as many
    arguments of the same C classes, mapped to a test here, and absent from the other headers' lists."""
    from dvmvs import _native as N
    protos = _header_prototypes()
    names = sorted(n for n, _ in protos)
    assert names == sorted(N.SPARSE_VIEW_SYMBOLS) and len(names) == 4
    assert not set(names) & (set(N.EXPORTED_SYMBOLS) | set(N.SPARSE_SYMBOLS))
    assert sorted(set(VIEW_TESTS) | VIEW_HOST_ONLY) == names
    assert all(callable(globals().get(t)) for t in VIEW_TESTS.values())
    lib = N.lib()
    kinds = {"ptr": (ctypes.c_void_p,), "int": (ctypes.c_int,), "longlong": (ctypes.c_longlong,), "double": (ctypes.c_double,),
             "float": (ctypes.c_float,)}
    for name, params in protos:
        want = []
        for q in params.split(","):
            q = q.strip()
            if "*" in q or "dvmvs_stream_t" in q:
                want.append("ptr")
            else:
                base = re.sub(r"\b(const|unsigned|signed)\b", "", q).split()
                want.append("longlong" if "long" in base else base[0])
        got = getattr(lib, name).argtypes
        assert got is not None and len(got) == len(want), (name, want, got)
        for i, (kind, at) in enumerate(zip(want, got)):
            is_ptr = isinstance(at, type) and (issubclass(at, ctypes._Pointer) or at is ctypes.c_void_p)
            assert (kind == "ptr" and is_ptr) or (kind != "ptr" and at in kinds[kind]), (name, i, kind, at)


def test_view_entry_points_refuse_bad_arguments_without_a_gpu():
    from dvmvs import _native as N
    lib = N.lib()
    n = ctypes.c_longlong(0)
    assert lib.dvmvs_tsdf_sparse_mesh_scratch_bytes(-1, ctypes.byref(n)) == -1
    assert lib.dvmvs_tsdf_sparse_mesh_scratch_bytes(1 << 22, ctypes.byref(n)) == -1
    assert lib.dvmvs_tsdf_sparse_mesh_scratch_bytes(4, None) == -1
    lo, f3 = (ctypes.c_longlong * 3)(0, 0, 0), (ctypes.c_float * 3)(0, 0, 0)
    assert lib.dvmvs_tsdf_sparse_mesh_count(None, None, 8, None, 4, None, None, 4, lo, 8, 8, 8, None, 1 << 20, None) == -1
    assert b"null" in lib.dvmvs_last_error_string()
    assert lib.dvmvs_tsdf_sparse_mesh_extract(None, None, 8, None, 4, None, None, None, 4, lo, 8, 8, 8, f3, 0.04, None, 1 << 20, 1, 1,
                                              None, None, None, None, None, None) == -1
    assert lib.dvmvs_tsdf_sparse_raycast(None, None, 8, None, 4, None, None, None, lo, 8, 8, 8, f3, 0.04, 0.2, None, 1, 8, 8,
                                         None, None, None, None) == -1
    # bad extents with non-null (never dereferenced) pointers
    p = ctypes.c_void_p(256)
    assert lib.dvmvs_tsdf_sparse_mesh_count(p, p, 6, p, 4, p, p, 4, lo, 8, 8, 8, p, 1 << 20, None) == -1       # table not 2^k
    assert lib.dvmvs_tsdf_sparse_mesh_count(p, p, 8, p, 4, p, p, 4, lo, -1, 8, 8, p, 1 << 20, None) == -1
    assert lib.dvmvs_tsdf_sparse_mesh_count(p, p, 8, p, 4, p, p, 4, lo, 1 << 30, 1 << 30, 8, p, 1 << 20, None) == -1   # > 2^61 voxels
    assert b"2^61" in lib.dvmvs_last_error_string()
    assert lib.dvmvs_tsdf_sparse_raycast(p, p, 8, p, 4, p, p, p, lo, 8, 0, 8, f3, 0.04, 0.2, p, 1, 8, 8, p, p, p, None) == -1
    assert lib.dvmvs_tsdf_sparse_raycast(p, p, 8, p, 4, p, p, p, lo, 8, 8, 8, f3, 0.0, 0.2, p, 1, 8, 8, p, p, p, None) == -1


DRYRUN_SCRIPT = r"""
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import numpy as np, torch
from dvmvs import _native as N
from dvmvs.tsdf import SparseTSDFVolume as S, TSDFVolume

assert N.DRYRUN

def raises(exc, f, match=""):
    try:
        f()
    except exc as e:
        assert match in str(e), (match, str(e))
        return str(e)
    raise AssertionError("no %%s" %% exc.__name__)

v = S(0.05, origin=(0.1, -0.2, 0.3), capacity_blocks=1000, device="cpu")
K, pose = np.array([[50.0, 0, 20], [0, 50.0, 15], [0, 0, 1]]), np.eye(4)
mesh = lambda b=None: v.get_mesh_tensors(b)
render = lambda b=None: v.render_tensors(K, pose, 30, 40, vol_bnds=b)
for f, what in ((mesh, "get_mesh"), (render, "render"), (v.get_mesh, "get_mesh"), (v.get_point_cloud, "get_mesh"),
                (lambda: v.render(K, pose, 30, 40), "render")):
    raises(ValueError, f, "SparseTSDFVolume.%%s: no block is allocated" %% what)           # the empty volume has no default box
o = np.float32([0.1, -0.2, 0.3]).astype(np.float64)
for f in (mesh, render):
    for lo in (o + 0.5 * 0.05, o + [0, 0.01 * 0.05, 0], o - [0, 0, 0.3 * 0.05]):
        raises(ValueError, lambda: f(np.stack([lo, lo + 1.0], axis=1)), "not on the voxel lattice")
    for b in (np.zeros((2, 3)), [[0, np.nan], [0, 1], [0, 1]], [[0, np.inf], [0, 1], [0, 1]], np.zeros(6)):
        raises(ValueError, lambda: f(b), "(3,2) finite bounds")
    raises(ValueError, lambda: f(np.stack([o, o + 1e9], axis=1)), "too large")
# an explicit box on an empty volume: an empty mesh without any launch
verts, faces, norms, colors = mesh(np.stack([o, o + 1.0], axis=1))
assert verts.shape == (0, 3) and faces.shape == (0, 3) and faces.dtype == torch.int32 and colors.dtype == torch.uint8

# every overflow flag raises before any launch, naming what allocated_blocks names
for n, flag, match in ((1500, N.SPARSE_POOL_FULL, "capacity_blocks >= 1500"), (2048, N.SPARSE_TABLE_FULL, "hash table of 2048"),
                       (3, N.SPARSE_FRUSTUM, "was not integrated")):
    v._counters[:2] = torch.tensor([n, flag], dtype=torch.int32)
    for f in (mesh, render, lambda: v.get_mesh(np.stack([o, o + 1.0], axis=1))):
        raises(RuntimeError, f, match)
v._counters[:2] = torch.tensor([0, 0], dtype=torch.int32)

# render's argument errors are TSDFVolume.render's, with the class name (both volumes run the base class's checks)
d = TSDFVolume([[0.1, 1.1], [-0.2, 0.8], [0.3, 1.3]], 0.05, device="cpu")
box = np.stack([o, o + 1.0], axis=1)
bad = [(np.eye(4)[:3], pose, 30, 40), (np.array([[0.0, 0, 20], [0, 50, 15], [0, 0, 1]]), pose, 30, 40),
       (np.array([[50.0, 0, np.nan], [0, 50, 15], [0, 0, 1]]), pose, 30, 40), (K, pose, 0, 40), (K, pose, 30, -1),
       (K, np.eye(3), 30, 40), (K, np.zeros((0, 4, 4)), 30, 40), (K, np.zeros((2, 4, 3)), 30, 40)]
for args in bad:
    want = raises(RuntimeError, lambda: d._views(*args))          # the checks TSDFVolume.render_tensors runs first
    got = raises(RuntimeError, lambda: v.render_tensors(*args, vol_bnds=box))
    assert want.startswith("TSDFVolume.render: ") and got == "SparseTSDFVolume" + want[len("TSDFVolume"):], (want, got)
print("dry run ok")
"""


def test_view_host_logic_dry_run():
    env = dict(os.environ, DVMVS_DRYRUN="1")
    script = DRYRUN_SCRIPT % (REPO, os.path.join(REPO, "deep-video-mvs_b200"))
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, cwd=REPO)
    assert r.returncode == 0 and "dry run ok" in r.stdout, r.stdout + r.stderr


# ------------------------------------------------------------------------------------------------------------------ GPU
def _views_around(center, radius, n=4):
    """camera-to-world poses: one at the centre looking along +z, one outside looking in, one looking away, an axis-parallel
    one, then more on a circle looking at the centre"""
    center = np.asarray(center, dtype=np.float64)
    out = []
    p = np.eye(4)
    p[:3, 3] = center
    out.append(p)                                               # inside, along +z (axis-parallel rays through the principal point)
    p = np.eye(4)
    p[:3, 3] = center - [0, 0, 2.5 * radius]
    out.append(p)                                               # outside, looking in
    p = np.eye(4)
    p[:3, :3] = _rot([0, 1, 0], np.pi)
    p[:3, 3] = center - [0, 0, 2.5 * radius]
    out.append(p)                                               # outside, looking away
    p = np.eye(4)
    p[:3, :3] = _rot([0, 1, 0], np.pi / 2)
    p[:3, 3] = center - [1.5 * radius, 0, 0]
    out.append(p)                                               # along +x
    for i in range(n):
        a = 2 * np.pi * i / n + 0.3
        p = np.eye(4)
        p[:3, :3] = _rot([0, 1, 0], -a + np.pi / 2) @ _rot([1, 0, 0], 0.2)
        p[:3, 3] = center + radius * np.array([np.cos(a), 0.3, np.sin(a)])
        out.append(p)
    return np.stack(out)


K_RENDER = np.array([[64.0, 0, 39.5], [0, 64.0, 29.5], [0, 0, 1]])      # 80 x 60; (39.5, 29.5) is not a pixel centre ...
K_AXIS = np.array([[64.0, 0, 40.0], [0, 64.0, 30.0], [0, 0, 1]])        # ... this one is: its centre ray is parallel to an axis


def _check(sparse, box, center, radius, what):
    """mesh and renders over `box` equal the export's, torch.equal; returns (mesh face count, hits)"""
    import torch
    dense = sparse.to_dense(box)
    got, want = sparse.get_mesh_tensors(box), dense.get_mesh_tensors()
    for name, a, b in zip(("verts", "faces", "norms", "colors"), got, want):
        assert a.shape == b.shape and torch.equal(a, b), "%s: mesh %s differs" % (what, name)
    n_faces = int(got[1].shape[0])
    poses = _views_around(center, radius)
    hits = 0
    for K in (K_RENDER, K_AXIS):
        got, want = sparse.render_tensors(K, poses, 60, 80, vol_bnds=box), dense.render_tensors(K, poses, 60, 80)
        for name, a, b in zip(("depth", "normals", "colors"), got, want):
            assert torch.equal(a, b), "%s: render %s differs in %d values" % (what, name, int((a != b).sum()))
        hits += int((got[0] > 0).sum())
    tposes = torch.from_numpy(poses).cuda()                     # tensor poses on the device; one view per call equals the batch
    got = sparse.render_tensors(torch.from_numpy(K_RENDER), tposes, 60, 80, vol_bnds=box)
    for i in (0, len(poses) - 1):
        one = sparse.render_tensors(K_RENDER, poses[i], 60, 80, vol_bnds=box)
        for a, b in zip(one, got):
            assert torch.equal(a, b[i]), what
    return n_faces, hits


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(tsdf_cases.CASES))
def test_gpu_mesh_and_render_equal_the_export_on_the_reference_cases(case):
    from dvmvs.tsdf import SparseTSDFVolume, TSDFVolume
    inp = tsdf_cases.inputs(case)
    dense = TSDFVolume(inp["bounds"], inp["voxel"])
    sparse = SparseTSDFVolume(inp["voxel"], origin=dense._vol_origin, capacity_blocks=4096)
    for fr in inp["frames"]:
        sparse.integrate(fr["color"], fr["depth"], inp["K"], fr["pose"], obs_weight=fr["weight"])
    b = np.asarray(inp["bounds"], dtype=np.float64)
    for box in (inp["bounds"], None):
        _check(sparse, box, b.mean(1), 0.5 * float(np.max(b[:, 1] - b[:, 0])), "%s box %s" % (case, box))


@pytest.mark.gpu
def test_gpu_mesh_and_render_equal_the_export_on_the_room_and_inside_cameras():
    """the 3.84 M-voxel room, and the adversarial cameras inside the volume at offsets 0 and 150 m"""
    bounds = np.array([[-4.0, 4.0], [-3.2, 3.2], [0.0, 4.8]])
    K = np.array([[250.0, 0, 160.3], [0, 251.0, 127.6], [0, 0, 1]])
    _, sparse = _fuse(_production_frames(), K, bounds, 0.04)
    n_faces, hits = _check(sparse, bounds, [0.0, 0.0, 1.5], 1.0, "room")
    assert n_faces > 10000 and hits > 1000
    for offset in (0.0, 150.0):
        b = np.array([[-2.0, 2.0], [-1.6, 1.6], [-2.0, 2.0]]) + offset
        _, sparse = _fuse(_adversarial_frames(offset), np.array([[100.0, 0, 63.5], [0, 100.0, 47.5], [0, 0, 1]]), b, 0.04)
        for box in (b, None):
            n_faces, hits = _check(sparse, box, [offset] * 3, 1.0, "offset %g box %s" % (offset, box))
            assert n_faces > 1000 and hits > 100


def _path_volume():
    from dvmvs.tsdf import SparseTSDFVolume
    sparse = SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384)
    for color, depth, pose, weight in _path_frames():
        sparse.integrate(color, depth, PATH_K, pose, obs_weight=weight)
    return sparse


@pytest.mark.gpu
def test_gpu_mesh_and_render_equal_the_export_on_every_box():
    """the boxes of the unbounded-path test of tests/test_tsdf_sparse.py: the default box, boxes cutting through the blocks,
    one reaching past them and one outside them"""
    sparse = _path_volume()
    boxes = [None, [[-1.0, 0.3], [-0.5, 0.2], [0.5, 1.6]], [[-3.5, -2.0], [-1.25, 0.4], [-0.75, 2.0]],
             [[1.0, 9.0], [-3.0, 3.0], [0.0, 2.5]], [[20.0, 21.0], [0.0, 1.0], [0.0, 1.0]]]
    faces = []
    for b in boxes:
        faces.append(_check(sparse, b, [0.0, 0.0, 0.5], 1.5, "box %s" % (b,))[0])
    assert faces[0] > 1000 and faces[-1] == 0


def _plant(sparse):
    """negative tsdf written straight into the pool next to missing blocks: on the -x / -y / -z faces of blocks whose lower
    neighbour is missing, at local index 7 next to a missing upper neighbour, and across 2 x 2 x 2 block corners"""
    import torch
    n = sparse.allocated_blocks()
    coords = sparse._coords[:n].cpu().numpy()
    have = {tuple(c) for c in coords}
    planted = 0
    rng = np.random.RandomState(5)
    for s in rng.permutation(n)[:400]:
        b = coords[s]
        for a in range(3):
            lo, hi = b.copy(), b.copy()
            lo[a] -= 1
            hi[a] += 1
            idx = [slice(None)] * 3
            if tuple(lo) not in have:                           # the lowest plane of the block, its lower neighbour missing
                idx[a] = 0
                sparse._tsdf[int(s)][tuple(idx)] = -0.5
                sparse._color[int(s)][tuple(idx)] = float(s % 65536) * 256 + 7
                planted += 1
            if tuple(hi) not in have:                           # local index 7, its upper neighbour missing
                idx[a] = 7
                sparse._tsdf[int(s)][tuple(idx)] = -0.25
                planted += 1
        if all(tuple(b - d) not in have for d in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1))):
            sparse._tsdf[int(s)][0, 0, 0] = -1.0                # a 2 x 2 x 2 block corner whose lower blocks are all missing
            planted += 1
    torch.cuda.synchronize()
    return planted


@pytest.mark.gpu
def test_gpu_missing_neighbour_cubes_are_meshed():
    """Surfaces planted against missing blocks: the cubes and grid edges whose lowest corner lies in a missing block must be
    meshed (and rendered) exactly as the export does.  Dropping the missing blocks from the work list fails this test."""
    sparse = _path_volume()
    assert _plant(sparse) > 200
    for b in (None, [[-1.0, 0.3], [-0.5, 0.2], [0.5, 1.6]]):
        _check(sparse, b, [0.0, 0.0, 0.5], 1.5, "planted, box %s" % (b,))


def _cluster_frames(shift):
    return [(c, d, np.concatenate([np.concatenate([p[:3, :3], (p[:3, 3] + shift)[:, None]], 1), p[3:]], 0), w)
            for c, d, p, w in _path_frames(n=4)]


@pytest.mark.gpu
def test_gpu_memory_scales_with_the_blocks_not_the_box():
    """Three clusters of the path far apart along a diagonal: the default box needs more than 50 GB dense.  Mesh and render
    succeed with a peak allocation of at most the scratch requested plus the outputs; each cluster's mesh over its block box
    padded by one block equals the export's bit for bit; the whole mesh is the concatenation of the clusters' meshes; a view of
    one cluster renders as over its padded box (within the lattice phase, see below)."""
    import torch
    from dvmvs import _native as N
    from dvmvs.tsdf import SparseTSDFVolume
    shifts = [np.zeros(3), np.array([60.0, 60.0, 60.0]), np.array([120.0, 120.0, 120.0])]
    sparse = SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384)
    counts = []
    for sh in shifts:
        for color, depth, pose, weight in _cluster_frames(sh):
            sparse.integrate(color, depth, PATH_K, pose, obs_weight=weight)
        counts.append(sparse.allocated_blocks())
    n = sparse.allocated_blocks()
    _, k, vb = sparse._box(None, "test")
    dims = np.ceil((vb[:, 1] - vb[:, 0]) / PATH_VOXEL)
    assert 12 * float(np.prod(dims)) > 50e9
    nbytes = ctypes.c_longlong(0)
    assert N.lib().dvmvs_tsdf_sparse_mesh_scratch_bytes(n, ctypes.byref(nbytes)) == 0
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    mesh = sparse.get_mesh_tensors()
    torch.cuda.synchronize()
    V, F = mesh[0].shape[0], mesh[1].shape[0]
    outputs = V * (12 + 12 + 3) + F * 12
    keys = 8 * (V + 3 * F)
    peak = torch.cuda.max_memory_allocated() - base
    slack = 1 << 20                                             # the caching allocator's rounding of the call's few allocations
    assert V > 0 and peak <= nbytes.value + keys + outputs + slack, (peak, nbytes.value, keys, outputs)
    coords = sparse._coords[:n].cpu().numpy().astype(np.int64)
    origin = sparse._origin.astype(np.float64)
    parts = []
    for i, sh in enumerate(shifts):
        c = coords[(np.abs(coords * 8 * PATH_VOXEL - sh) < 30).all(1)]
        lo, hi = (c.min(0) - 1) * 8, (c.max(0) + 2) * 8
        box = np.stack([origin + lo * PATH_VOXEL, origin + (hi - 0.5) * PATH_VOXEL], axis=1)
        got, want = sparse.get_mesh_tensors(box), sparse.to_dense(box).get_mesh_tensors()
        for a, b in zip(got, want):
            assert torch.equal(a, b), "cluster %d" % i
        parts.append((got, box))
    off = 0
    verts, faces, norms, colors = mesh
    for (v, f, nm, cl), box in parts:
        m = v.shape[0]
        sel = slice(off, off + m)
        # the box origins differ: positions agree to within float32 rounding of origin + index * voxel, here < 1e-3 voxel
        assert float((v - verts[sel]).abs().max()) < 1e-3 * PATH_VOXEL
        # normals and colours are equal except where the dense contract is box-relative: np.gradient is one-sided on the
        # whole box's faces (the padded cluster boxes have none at the surface), and the colour voxel is rint(index + t), whose
        # float32 rounding depends on the box origin at half-voxel ties
        idx = (verts[sel].double() - torch.tensor(vb[:, 0], device=v.device)) / PATH_VOXEL
        inner = ((idx > 1.5) & (idx < torch.tensor(dims, device=v.device) - 2.5)).all(1)
        assert torch.equal(nm[inner], norms[sel][inner])
        diff = (cl != colors[sel]).any(1) & inner
        frac = torch.remainder((v[diff].double() - torch.tensor(box[:, 0], device=v.device)) / PATH_VOXEL, 1.0)
        assert bool(((frac - 0.5).abs() < 1e-3).any(1).all()) and int(diff.sum()) <= 1e-3 * m, int(diff.sum())
        assert int(inner.sum()) > 0.9 * m
        off += m
    assert off == V
    cat_faces, voff = [], 0
    for (v, f, _, _), _ in parts:
        cat_faces.append(f + voff)
        voff += v.shape[0]
    assert torch.equal(torch.cat(cat_faces), faces)
    # renders: the whole box against the cluster's padded box from a view of cluster 1 only.  The two boxes put the ray's
    # half-voxel lattice at different phases (z_near differs), so samples differ; the crossing is interpolated linearly from
    # samples half a voxel apart, so depths agree to within a fraction of a voxel of camera depth: |dz| < 0.5 voxel * 2.
    poses = np.stack([p for _, _, p, _ in _cluster_frames(shifts[1])])        # the cluster's own cameras
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    whole = sparse.render_tensors(K_RENDER, poses, 60, 80)
    torch.cuda.synchronize()
    out_bytes = len(poses) * 60 * 80 * (4 + 12 + 3)
    assert torch.cuda.max_memory_allocated() - base <= out_bytes + slack
    part = sparse.render_tensors(K_RENDER, poses, 60, 80, vol_bnds=parts[1][1])
    both = (whole[0] > 0) & (part[0] > 0)
    assert int(both.sum()) > 500 and int((whole[0] > 0).sum()) >= 0.9 * int((part[0] > 0).sum())
    assert float((whole[0] - part[0])[both].abs().max()) <= PATH_VOXEL


@pytest.mark.gpu
def test_gpu_view_buffers_stay_in_their_bounds():
    """mesh and render with the pool, the scratch, the keys and the outputs in guarded buffers (tests/guarded.py): no fringe
    is touched and the results equal the unguarded ones"""
    import torch
    from dvmvs import tsdf as T
    from tests import guarded as G
    frames = _path_frames()
    plain = _path_volume()
    want_mesh = plain.get_mesh_tensors()
    poses = _views_around([0.0, 0.0, 0.5], 1.5)
    want_render = plain.render_tensors(K_RENDER, poses, 60, 80)
    with G.guard_allocations(modules=[T], guard_arguments=False):
        small = T.SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384)
        for color, depth, pose, weight in frames:
            small.integrate(color, depth, PATH_K, pose, obs_weight=weight)
        mesh = small.get_mesh_tensors()
        render = small.render_tensors(K_RENDER, poses, 60, 80)
        torch.cuda.synchronize()
        assert len(G.REGISTRY.guards) >= 12
        G.verify(clear=False)
        for a, b in zip(mesh + render, want_mesh + want_render):
            assert torch.equal(a, b)
        G.verify()


@pytest.mark.gpu
def test_gpu_mesh_and_render_are_deterministic():
    """two calls, and two volumes fused from the same frames (pool slots assigned by atomics), give identical bits"""
    import torch
    a, b = _path_volume(), _path_volume()
    poses = _views_around([0.0, 0.0, 0.5], 1.5)
    ra = a.get_mesh_tensors() + a.render_tensors(K_RENDER, poses, 60, 80)
    for vol in (a, b):
        rb = vol.get_mesh_tensors() + vol.render_tensors(K_RENDER, poses, 60, 80)
        for x, y in zip(ra, rb):
            assert torch.equal(x, y)
