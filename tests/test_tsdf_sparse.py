"""SparseTSDFVolume (dvmvs/tsdf.py, csrc/tsdf_sparse.cu, include/dvmvs_tsdf_sparse.h): TSDF fusion into 8 x 8 x 8-voxel blocks
allocated on the device.  Its contract: after any frames it holds, voxel for voxel, the tsdf, weight and colour a dense TSDFVolume
with the same origin holds after the same frames -- compared with array_equal on the cases of tests/test_tsdf.py (whose dense
volumes equal the reference's CPU path bit for bit), on a camera path no fixed box contains, and under a pool too small for the
frames.  A voxel the allocation missed would export weight 0 where the dense volume has weight > 0.

CPU: the header against the library and the ctypes binding, and (DVMVS_DRYRUN=1, in a subprocess) the constructor's argument
checks, the capacity arithmetic, the lattice check of to_dense and the overflow messages."""
import importlib
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

from tests.test_tsdf import _rot, _same  # noqa: E402

# every entry point of include/dvmvs_tsdf_sparse.h -> the test (of this module, or "module::test") that checks what it computes
SPARSE_TESTS = {
    "dvmvs_tsdf_sparse_allocate": "tests.test_tsdf_block_reference::test_gpu_allocation_frame_by_frame",
    "dvmvs_tsdf_sparse_integrate": "test_gpu_sparse_equals_dense_on_the_reference_cases",
    "dvmvs_tsdf_sparse_export": "test_gpu_unbounded_path_every_sub_box_equals_a_dense_volume_over_it",
    "dvmvs_tsdf_sparse_block_bounds": "test_gpu_unbounded_path_every_sub_box_equals_a_dense_volume_over_it",
}
SPARSE_HOST_ONLY = {"dvmvs_tsdf_sparse_scratch_bytes"}


def _header_prototypes():
    header = open(os.path.join(REPO, "include", "dvmvs_tsdf_sparse.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    return re.findall(r"\bint\s+(dvmvs_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", header)


def _names_a_test(t):
    if "::" in t:
        mod, fn = t.split("::")
        return callable(getattr(importlib.import_module(mod), fn, None))
    return callable(globals().get(t))


def test_sparse_header_library_binding_and_coverage_agree():
    """Every prototype of include/dvmvs_tsdf_sparse.h is exported, listed in SPARSE_SYMBOLS, bound with as many arguments of
    the same C classes, mapped to a test here (or host-only), and absent from dvmvs_b200.h's list."""
    import ctypes
    from dvmvs import _native as N
    protos = _header_prototypes()
    names = sorted(n for n, _ in protos)
    assert names == sorted(N.SPARSE_SYMBOLS) and len(names) == 5
    assert not set(names) & set(N.EXPORTED_SYMBOLS)
    assert sorted(set(SPARSE_TESTS) | SPARSE_HOST_ONLY) == names and not set(SPARSE_TESTS) & SPARSE_HOST_ONLY
    assert all(_names_a_test(t) for t in SPARSE_TESTS.values())
    lib = N.lib()
    kinds = {"ptr": (ctypes.c_void_p,), "int": (ctypes.c_int,), "longlong": (ctypes.c_longlong,), "double": (ctypes.c_double,)}
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


def test_sparse_entry_points_refuse_bad_arguments_without_a_gpu():
    import ctypes
    from dvmvs import _native as N
    lib = N.lib()
    n = ctypes.c_longlong(0)
    assert lib.dvmvs_tsdf_sparse_scratch_bytes(256, 320, ctypes.byref(n)) == 0 and n.value == 64 + 8 * 16 * 20
    assert lib.dvmvs_tsdf_sparse_scratch_bytes(0, 320, ctypes.byref(n)) == -1
    f3, f4 = (ctypes.c_float * 3)(0, 0, 0), (ctypes.c_float * 4)(100, 100, 50, 40)
    T = (ctypes.c_double * 16)(*np.eye(4).reshape(-1))
    assert lib.dvmvs_tsdf_sparse_allocate(None, None, 8, None, 4, None, None, None, 1024, f3, 0.04, 0.2, None, 0, 8, 8, f4, T, None) == -1
    assert b"null" in lib.dvmvs_last_error_string()
    assert lib.dvmvs_tsdf_sparse_integrate(None, None, None, None, 4, None, None, f3, 0.04, 0.2, None, 1, None, 0, 8, 8, f4, T, 1.0,
                                           None, None) == -1
    assert lib.dvmvs_tsdf_sparse_export(None, None, None, None, 4, None, (ctypes.c_int * 3)(), 8, 8, 8, None, None, None, None) == -1
    assert lib.dvmvs_tsdf_sparse_block_bounds(None, 4, None, None, None) == -1


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
        return
    raise AssertionError("no %%s" %% exc.__name__)

# constructor arguments
for kw in (dict(voxel_size=0), dict(voxel_size=-0.04), dict(voxel_size=float("nan")), dict(voxel_size=0.04, origin=(0, 0)),
           dict(voxel_size=0.04, origin=(0, np.inf, 0)), dict(voxel_size=0.04, capacity_blocks=0), dict(voxel_size=0.04, capacity_blocks=2.5),
           dict(voxel_size=0.04, capacity_blocks=True), dict(voxel_size=0.04, capacity_blocks=2 ** 29 + 1)):
    raises(ValueError, lambda: S(device="cpu", **kw))

# capacity arithmetic: the table is the smallest power of two >= 2 x capacity; device_bytes is what the constructor allocates
assert [S.table_size(c) for c in (1, 2, 3, 4, 5, 1000, 2 ** 29)] == [2, 4, 8, 8, 16, 2048, 2 ** 30]
assert S.device_bytes(1000) == 1000 * (512 * 12 + 16) + 2048 * 12 + 16
v = S(0.05, origin=(0.1, -0.2, 0.3), capacity_blocks=1000, device="cpu")
state = (v._keys, v._slots, v._coords, v._tsdf, v._weight, v._color, v._counters, v._visible)
assert sum(t.numel() * t.element_size() for t in state) == S.device_bytes(1000)
assert v._keys.numel() == 2048 and bool((v._keys == -1).all()) and tuple(v._tsdf.shape) == (1000, 8, 8, 8)
assert float(v._tsdf.min()) == 1.0 and float(v._weight.abs().max()) == 0.0 and float(v._color.abs().max()) == 0.0

# to_dense: lower bounds on the lattice origin + k * voxel_size (up to float32 rounding of the bounds), anything else refused
o = np.float32([0.1, -0.2, 0.3]).astype(np.float64)
raises(ValueError, lambda: v.to_dense(), "no block is allocated")
for b in (np.stack([o + np.array([2, -3, 0]) * 0.05, o + 1.0], axis=1),
          [[0.1, 0.5], [-0.2, 0.5], [0.3, 0.5]]):                     # float64 bounds whose float32 rounding is the origin
    d, want = v.to_dense(b), TSDFVolume(b, 0.05, device="cpu")
    assert isinstance(d, TSDFVolume) and np.array_equal(d._vol_dim, want._vol_dim) and np.array_equal(d._vol_origin, want._vol_origin)
    assert float(d.get_volume_tensors()[0].min()) == 1.0 and min(d._vol_dim) >= 4
for lo in (o + 0.5 * 0.05, o + [0, 0.01 * 0.05, 0], o - [0, 0, 0.3 * 0.05]):
    raises(ValueError, lambda: v.to_dense(np.stack([lo, lo + 1.0], axis=1)), "not on the voxel lattice")
raises(ValueError, lambda: v.to_dense(np.zeros((2, 3))))
raises(ValueError, lambda: v.to_dense([[0, np.nan], [0, 1], [0, 1]]))

# overflow: the next read-back raises, naming the capacity the frames need
v._counters[:2] = torch.tensor([1500, N.SPARSE_POOL_FULL], dtype=torch.int32)
raises(RuntimeError, v.allocated_blocks, "need 1500 blocks, the pool holds 1000: construct the volume with capacity_blocks >= 1500")
raises(RuntimeError, v.to_dense, "capacity_blocks >= 1500")
v._counters[:2] = torch.tensor([2048, N.SPARSE_TABLE_FULL | N.SPARSE_POOL_FULL], dtype=torch.int32)
raises(RuntimeError, v.allocated_blocks, "hash table of 2048 entries is full; the frames so far need more than 2048 blocks")
v._counters[:2] = torch.tensor([3, N.SPARSE_FRUSTUM], dtype=torch.int32)
raises(RuntimeError, lambda: v.to_dense([[0.1, 0.5], [-0.2, 0.5], [0.3, 0.5]]), "was not integrated")
v._counters[:2] = torch.tensor([3, 0], dtype=torch.int32)
assert v.allocated_blocks() == 3

# integrate: intrinsics the allocation's frustum cannot use are refused before any device work
w = S(0.05, device="cpu")
for (r, c, bad) in ((0, 0, 0.0), (1, 1, -5.0), (0, 2, np.nan), (1, 2, np.inf)):
    K = np.array([[50.0, 0, 20], [0, 50.0, 15], [0, 0, 1]])
    K[r, c] = bad
    raises(ValueError, lambda: w.integrate(np.zeros((30, 40, 3), np.uint8), np.ones((30, 40), np.float32), K, np.eye(4)), "focal lengths")
print("dry run ok")
"""


def test_sparse_volume_host_logic_dry_run():
    env = dict(os.environ, DVMVS_DRYRUN="1")
    script = DRYRUN_SCRIPT % (REPO, os.path.join(REPO, "deep-video-mvs_b200"))
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, cwd=REPO)
    assert r.returncode == 0 and "dry run ok" in r.stdout, r.stdout + r.stderr


# ------------------------------------------------------------------------------------------------------------------ GPU
def _fuse(frames, K, bounds, voxel, **sparse_kw):
    """the same frames into a dense TSDFVolume over bounds and a SparseTSDFVolume with the dense volume's origin"""
    from dvmvs.tsdf import SparseTSDFVolume, TSDFVolume
    dense = TSDFVolume(bounds, voxel)
    sparse = SparseTSDFVolume(voxel, origin=dense._vol_origin, **sparse_kw)
    for color, depth, pose, weight in frames:
        dense.integrate(color, depth, K, pose, obs_weight=weight)
        sparse.integrate(color, depth, K, pose, obs_weight=weight)
    return dense, sparse


def _assert_volumes_equal(got, want, what):
    assert np.array_equal(got._vol_dim, want._vol_dim) and np.array_equal(got._vol_origin, want._vol_origin), what
    for name, a, b in zip(("tsdf", "weight", "color"), got.get_volume_tensors(), want.get_volume_tensors()):
        a, b = a.cpu().numpy(), b.cpu().numpy()
        assert _same(a, b), "%s: %s differs in %d voxels" % (what, name, int((a != b).sum()))


def _production_frames():
    """the frames of tests/test_tsdf.py::test_gpu_volume_at_production_size_equals_oracle"""
    rng = np.random.RandomState(11)
    h, w = 256, 320
    out = []
    for i in range(3):
        yy, xx = np.mgrid[0:h, 0:w]
        depth = (2.0 + 0.8 * np.sin(xx / 40.0 + i) * np.cos(yy / 30.0) + 0.01 * rng.rand(h, w)).astype(np.float32)
        depth[rng.rand(h, w) < 0.05] = 0
        color = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
        pose = np.eye(4)
        pose[:3, 3] = [0.1 * i, -0.05 * i, 0.02 * i]
        c, s = np.cos(0.05 * i), np.sin(0.05 * i)
        pose[:3, :3] = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
        out.append((color, depth, pose, 1.0))
    return out


def _adversarial_frames(offset):
    """the frames of tests/test_tsdf.py::test_gpu_frustum_cull_never_drops_a_voxel_the_reference_updates: cameras inside the
    volume looking along every axis and obliquely"""
    rng = np.random.RandomState(23)
    h, w = 96, 128
    views = [([0, 1, 0], 0.0), ([0, 1, 0], np.pi / 2), ([0, 1, 0], np.pi), ([1, 0, 0], np.pi / 2), ([1, 0, 0], -np.pi / 2),
             ([1, 1, 0], 0.7), ([1, 2, 3], 2.1), ([0, 0, 1], np.pi / 4)]
    out = []
    for i, (axis, angle) in enumerate(views):
        depth = (0.3 + 1.5 * rng.rand(h, w)).astype(np.float32)
        color = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
        pose = np.eye(4)
        pose[:3, :3] = _rot(axis, angle)
        pose[:3, 3] = offset + rng.uniform(-0.5, 0.5, size=3)
        out.append((color, depth, pose, 1.0 + i))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(tsdf_cases.CASES))
def test_gpu_sparse_equals_dense_on_the_reference_cases(case):
    """oracle/tsdf_cases.py (uint8 and float32 colour, float32 and float64 depth, observation weights 0.3 and 2): the export
    over the dense volume's bounds equals the dense volume after every frame"""
    from dvmvs.tsdf import SparseTSDFVolume, TSDFVolume
    inp = tsdf_cases.inputs(case)
    dense = TSDFVolume(inp["bounds"], inp["voxel"])
    sparse = SparseTSDFVolume(inp["voxel"], origin=dense._vol_origin, capacity_blocks=4096)
    for i, fr in enumerate(inp["frames"]):
        dense.integrate(fr["color"], fr["depth"], inp["K"], fr["pose"], obs_weight=fr["weight"])
        sparse.integrate(fr["color"], fr["depth"], inp["K"], fr["pose"], obs_weight=fr["weight"])
        _assert_volumes_equal(sparse.to_dense(inp["bounds"]), dense, "%s frame %d" % (case, i))
    assert sparse.allocated_blocks() > 0 and sparse.updated_voxels() >= dense.updated_voxels() > 0


@pytest.mark.gpu
def test_gpu_sparse_equals_dense_at_production_size():
    """the 3.84 M-voxel room of tests/test_tsdf.py at 4 cm, 320 x 256 frames; every updated voxel is inside the room, so the
    update counts agree too, and the blocks allocated are a fraction of the room's"""
    bounds = np.array([[-4.0, 4.0], [-3.2, 3.2], [0.0, 4.8]])
    K = np.array([[250.0, 0, 160.3], [0, 251.0, 127.6], [0, 0, 1]])
    dense, sparse = _fuse(_production_frames(), K, bounds, 0.04)
    _assert_volumes_equal(sparse.to_dense(bounds), dense, "production size")
    assert sparse.updated_voxels() == dense.updated_voxels() > 100000
    n = sparse.allocated_blocks()
    assert 0 < n < 0.5 * (200 * 160 * 120) / 512, n


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0.0, 150.0])
def test_gpu_sparse_allocation_is_conservative_for_cameras_inside_the_volume(offset):
    """cameras inside the volume along every axis and obliquely, 150 m from the origin too: many voxels on the image border and
    next to the camera plane, where a block test that rounded the wrong way would drop voxels the dense volume updates"""
    bounds = np.array([[-2.0, 2.0], [-1.6, 1.6], [-2.0, 2.0]]) + offset
    K = np.array([[100.0, 0, 63.5], [0, 100.0, 47.5], [0, 0, 1]])
    dense, sparse = _fuse(_adversarial_frames(offset), K, bounds, 0.04)
    _assert_volumes_equal(sparse.to_dense(bounds), dense, "offset %g" % offset)
    assert dense.updated_voxels() > 50000


def _path_frames(n=9, h=60, w=80):
    """a camera sliding 6 m along x (and a little in y and z) past a wavy wall, turning slightly: no fixed box holds its path"""
    rng = np.random.RandomState(7)
    yy, xx = np.mgrid[0:h, 0:w]
    out = []
    for i in range(n):
        depth = (1.4 + 0.4 * np.sin(xx / 9.0 + i) * np.cos(yy / 7.0) + 0.02 * rng.rand(h, w)).astype(np.float32)
        depth[rng.rand(h, w) < 0.06] = 0
        color = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
        pose = np.eye(4)
        pose[:3, :3] = _rot([0.2, 1, 0.1], 0.15 * np.sin(i))
        pose[:3, 3] = [-3.0 + 0.75 * i, -0.4 + 0.1 * i, -0.5 + 0.05 * i]
        out.append((color, depth, pose, 1.0))
    return out


PATH_K = np.array([[60.0, 0, 39.5], [0, 60.0, 29.5], [0, 0, 1]])
PATH_VOXEL = 1.0 / 32            # dyadic: every lattice point origin + k * voxel is exact in float32, so a dense volume over any
                                 # lattice-aligned box has the sparse volume's world points


@pytest.mark.gpu
def test_gpu_unbounded_path_every_sub_box_equals_a_dense_volume_over_it():
    """A path through negative block coordinates.  The default export (the allocated blocks' bounding box), boxes cutting
    through it, one reaching past it and one outside it each equal a dense volume built over that box from the same frames,
    and the exported volume's mesh equals the dense volume's."""
    from dvmvs.tsdf import SparseTSDFVolume, TSDFVolume
    frames = _path_frames()
    sparse = SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384)
    for color, depth, pose, weight in frames:
        sparse.integrate(color, depth, PATH_K, pose, obs_weight=weight)
    full = sparse.to_dense()
    lo = full._vol_bnds[:, 0]
    assert lo[0] < -3.0 and lo[1] < 0 and full._vol_bnds[0, 1] > 3.0, full._vol_bnds
    assert np.all(full._vol_dim % 8 == 0) and np.all(np.rint(lo / PATH_VOXEL) % 8 == 0)
    boxes = [full._vol_bnds, [[-1.0, 0.3], [-0.5, 0.2], [0.5, 1.6]], [[-3.5, -2.0], [-1.25, 0.4], [-0.75, 2.0]],
             [[1.0, 9.0], [-3.0, 3.0], [0.0, 2.5]], [[20.0, 21.0], [0.0, 1.0], [0.0, 1.0]]]
    for b in boxes:
        dense = TSDFVolume(b, PATH_VOXEL)
        for color, depth, pose, weight in frames:
            dense.integrate(color, depth, PATH_K, pose, obs_weight=weight)
        got = full if b is full._vol_bnds else sparse.to_dense(b)
        _assert_volumes_equal(got, dense, "box %s" % (np.asarray(b).tolist(),))
        if b is full._vol_bnds:
            assert sparse.updated_voxels() == dense.updated_voxels() > 0
            for x, y in zip(full.get_mesh(), dense.get_mesh()):
                assert x.shape == y.shape and np.array_equal(x, y)
            assert len(full.get_mesh()[1]) > 1000
    assert float(sparse.to_dense(boxes[-1]).get_volume_tensors()[1].abs().max()) == 0.0


@pytest.mark.gpu
def test_gpu_pool_overflow_raises_with_the_needed_capacity_and_keeps_its_blocks():
    """A pool of about half the blocks the path needs, its state in guarded buffers (tests/guarded.py: sentinel fringes around
    the table, the pool and every other allocation): the read-back raises naming the capacity, every block that got a slot
    equals the dense volume there, and no fringe is touched.  A table too small for the keys raises too.  A pool of exactly
    the named capacity then fuses the path without error."""
    import torch
    from dvmvs import tsdf as T
    from tests import guarded as G
    frames = _path_frames()
    big = T.SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384)
    for color, depth, pose, weight in frames:
        big.integrate(color, depth, PATH_K, pose, obs_weight=weight)
    need = big.allocated_blocks()
    full = big.to_dense()
    k0 = torch.tensor(np.rint(full._vol_bnds[:, 0] / PATH_VOXEL).astype(np.int64), device="cuda")
    off = torch.stack(torch.meshgrid(*[torch.arange(8, device="cuda")] * 3, indexing="ij"), dim=-1)
    table = 1 << ((need - 1).bit_length() - 1)                 # the largest power of two < need: a table with no room for all keys
    for capacity, match in ((need // 2 + 1, "need %d blocks, the pool holds %d: construct the volume with capacity_blocks >= %d"
                             % (need, need // 2 + 1, need)), (table // 2, "hash table of %d entries is full" % table)):
        with G.guard_allocations(modules=[T], guard_arguments=False):
            small = T.SparseTSDFVolume(PATH_VOXEL, capacity_blocks=capacity)
            assert len(G.REGISTRY.guards) >= 8
            for color, depth, pose, weight in frames:
                small.integrate(color, depth, PATH_K, pose, obs_weight=weight)
            torch.cuda.synchronize()
            G.verify(clear=False)
            with pytest.raises(RuntimeError, match=re.escape(match)):
                small.allocated_blocks()
            with pytest.raises(RuntimeError, match=re.escape(match)):
                small.to_dense()
            n = min(int(small._counters[0]), capacity)
            assert n == capacity or capacity == table // 2
            idx = (small._coords[:n].long() * 8 - k0)[:, None, None, None, :] + off       # [n][8][8][8][3] dense voxel indices
            for name, pool, vol in zip(("tsdf", "weight", "color"), (small._tsdf, small._weight, small._color), full.get_volume_tensors()):
                want = vol[idx[..., 0], idx[..., 1], idx[..., 2]]
                assert torch.equal(pool[:n], want), "capacity %d: %s of a block with a slot differs" % (capacity, name)
            assert 0 < small.updated_voxels() < big.updated_voxels()
            G.verify()
    exact = T.SparseTSDFVolume(PATH_VOXEL, capacity_blocks=need)
    for color, depth, pose, weight in frames:
        exact.integrate(color, depth, PATH_K, pose, obs_weight=weight)
    assert exact.allocated_blocks() == need
    _assert_volumes_equal(exact.to_dense(), full, "capacity %d" % need)
