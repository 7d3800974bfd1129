"""Growing SparseTSDFVolume (dvmvs/tsdf.py, csrc/tsdf_sparse.cu, include/dvmvs_tsdf_sparse_grow.h).  The contract: after any
frames, a volume built with max_capacity_blocks holds, voxel for voxel, what a fixed volume large enough from the start holds
(and so what a TSDFVolume with the same origin holds), with the same update count, export, mesh and renders -- after many
growths, when the caller overwrites its input tensors right after integrate, when the first frame fills a 2-entry table.  At
the cap, the frames from the one that overflowed on are not integrated and the blocks with a slot hold what they held before it.

CPU: the header against the library and the ctypes binding, refusal of bad rehash arguments without a GPU, and
(DVMVS_DRYRUN=1, in a subprocess) the constructor's checks, the growth arithmetic, halt mode in counters[3] and the at-cap
message."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))

from tests.test_tsdf_sparse import PATH_K, PATH_VOXEL, _assert_volumes_equal, _fuse, _path_frames  # noqa: E402

# every entry point of include/dvmvs_tsdf_sparse_grow.h -> the test of this module that checks what it computes
GROW_TESTS = {
    "dvmvs_tsdf_sparse_rehash": "test_gpu_many_growths_equal_a_large_enough_volume",
}
CUT_BOX = [[-1.0, 0.3], [-0.5, 0.2], [0.5, 1.6]]


def _header_prototypes():
    header = open(os.path.join(REPO, "include", "dvmvs_tsdf_sparse_grow.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    return re.findall(r"\bint\s+(dvmvs_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", header)


def test_grow_header_library_binding_and_coverage_agree():
    """Every prototype of include/dvmvs_tsdf_sparse_grow.h is exported, listed in SPARSE_GROW_SYMBOLS, bound with as many
    arguments of the same C classes, mapped to a test here, and absent from the other headers' lists; the halt bit agrees."""
    from dvmvs import _native as N
    protos = _header_prototypes()
    names = sorted(n for n, _ in protos)
    assert names == sorted(N.SPARSE_GROW_SYMBOLS) and len(names) == 1
    assert not set(names) & (set(N.EXPORTED_SYMBOLS) | set(N.SPARSE_SYMBOLS) | set(N.SPARSE_VIEW_SYMBOLS))
    assert sorted(GROW_TESTS) == names
    assert all(callable(globals().get(t)) for t in GROW_TESTS.values())
    header = open(os.path.join(REPO, "include", "dvmvs_tsdf_sparse_grow.h")).read()
    assert re.search(r"DVMVS_SPARSE_HALT_ON_FULL = (\d+)", header).group(1) == str(N.SPARSE_HALT_ON_FULL)
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


def test_rehash_refuses_bad_arguments_without_a_gpu():
    from dvmvs import _native as N
    lib = N.lib()
    assert lib.dvmvs_tsdf_sparse_rehash(None, None, 8, None, 4, None, None) == -1
    assert b"null" in lib.dvmvs_last_error_string()
    p = ctypes.c_void_p(256)                                                # non-null, never dereferenced
    assert lib.dvmvs_tsdf_sparse_rehash(p, None, 8, p, 4, p, None) == -1
    for table, n in ((12, 4), (0, 0), (-8, 1), (3 << 29, 4), (8, 5), (8, -1), (1 << 30, (1 << 29) + 1)):
        assert lib.dvmvs_tsdf_sparse_rehash(p, p, table, p, n, p, None) == -1, (table, n)
        assert b"tsdf_sparse_rehash" in lib.dvmvs_last_error_string()


DRYRUN_SCRIPT = r"""
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import numpy as np, torch
from dvmvs import _native as N
from dvmvs.tsdf import SparseTSDFVolume as S

assert N.DRYRUN

def raises(exc, f, match=""):
    try:
        f()
    except exc as e:
        assert match in str(e), (match, str(e))
        return
    raise AssertionError("no %%s" %% exc.__name__)

# max_capacity_blocks: None or an integer >= capacity_blocks, at most 2^29
for m in (99, 100.5, True, 2 ** 29 + 1, "many"):
    raises(ValueError, lambda: S(0.05, capacity_blocks=100, max_capacity_blocks=m, device="cpu"))
raises(ValueError, lambda: S(0.05, capacity_blocks=100, max_capacity_blocks=99, device="cpu"), ">= capacity_blocks 100")
raises(ValueError, lambda: S(0.05, capacity_blocks=100, max_capacity_blocks=2 ** 29 + 1, device="cpu"), "exceeds 2^29")
assert S(0.05, capacity_blocks=8, max_capacity_blocks=2 ** 29, device="cpu").max_capacity_blocks == 2 ** 29
assert S(0.05, capacity_blocks=8, max_capacity_blocks=8.0, device="cpu").max_capacity_blocks == 8

# halt mode in counters[3] only for a growable volume; the fixed volume's state is as before
fixed, grow = S(0.05, capacity_blocks=100, device="cpu"), S(0.05, capacity_blocks=100, max_capacity_blocks=1000, device="cpu")
assert fixed.max_capacity_blocks is None and fixed._counters.tolist() == [0, 0, 0, 0]
assert grow._counters.tolist() == [0, 0, 0, N.SPARSE_HALT_ON_FULL] and N.SPARSE_HALT_ON_FULL == 1
for v in (fixed, grow):
    state = (v._keys, v._slots, v._coords, v._tsdf, v._weight, v._color, v._counters, v._visible)
    assert sum(t.numel() * t.element_size() for t in state) == S.device_bytes(100)

# growth arithmetic: min(max, max(2 x capacity, blocks needed)), then the table that follows
assert [S._grown_capacity(c, n, m) for c, n, m in ((64, 10, 16384), (64, 1000, 16384), (10000, 12000, 16384), (9000, 30000, 16384),
                                                    (1, 3, 2), (5, 0, 5))] == [128, 1000, 16384, 16384, 2, 5]
grow._tsdf[:] = torch.arange(100, dtype=torch.float32)[:, None, None, None]
grow._coords[:] = torch.arange(300, dtype=torch.int32).reshape(100, 3)
grow._counters[:2] = torch.tensor([150, N.SPARSE_POOL_FULL], dtype=torch.int32)
grow._grow(S._grown_capacity(grow.capacity, 150, 1000), 100)
assert grow.capacity == 200 and grow.growths == 1 and grow._keys.numel() == S.table_size(200) == 512 and grow._slots.numel() == 512
assert bool((grow._keys == -1).all())
for t, rows in ((grow._coords, 200), (grow._tsdf, 200), (grow._weight, 200), (grow._color, 200), (grow._visible, 200)):
    assert t.shape[0] == rows
assert torch.equal(grow._tsdf[:100, 0, 0, 0], torch.arange(100, dtype=torch.float32)) and float(grow._tsdf[100:].min()) == 1.0
assert torch.equal(grow._coords[:100].reshape(-1), torch.arange(300, dtype=torch.int32)) and int(grow._coords[100:].abs().max()) == 0
assert float(grow._weight.abs().max()) == 0.0 and grow._counters[3] == N.SPARSE_HALT_ON_FULL

# at the cap: the flag stays, the reads raise naming the need and the cap; updated_voxels still counts
cap = S(0.05, capacity_blocks=100, max_capacity_blocks=100, device="cpu")
cap._counters[:2] = torch.tensor([150, N.SPARSE_POOL_FULL], dtype=torch.int32)
msg = "the frames so far need 150 blocks, more than max_capacity_blocks 100: frame 0"
raises(RuntimeError, cap.allocated_blocks, msg)
raises(RuntimeError, cap.to_dense, msg)
raises(RuntimeError, cap.get_mesh_tensors, "were not integrated")
raises(RuntimeError, lambda: cap.render_tensors(np.array([[50.0, 0, 20], [0, 50.0, 15], [0, 0, 1]]), np.eye(4), 30, 40), msg)
assert cap.updated_voxels() == 0 and cap.capacity == 100 and cap.growths == 0
cap = S(0.05, capacity_blocks=1, max_capacity_blocks=1, device="cpu")
cap._counters[:2] = torch.tensor([2, N.SPARSE_TABLE_FULL | N.SPARSE_POOL_FULL], dtype=torch.int32)
raises(RuntimeError, cap.allocated_blocks, "need more than 2 blocks, more than max_capacity_blocks 1")
# the fixed pool's messages are unchanged
fixed._counters[:2] = torch.tensor([150, N.SPARSE_POOL_FULL], dtype=torch.int32)
raises(RuntimeError, fixed.allocated_blocks, "need 150 blocks, the pool holds 100: construct the volume with capacity_blocks >= 150")
print("dry run ok")
"""


def test_grow_host_logic_dry_run():
    env = dict(os.environ, DVMVS_DRYRUN="1")
    script = DRYRUN_SCRIPT % (REPO, os.path.join(REPO, "deep-video-mvs_b200"))
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, cwd=REPO)
    assert r.returncode == 0 and "dry run ok" in r.stdout, r.stdout + r.stderr


# ------------------------------------------------------------------------------------------------------------------ GPU
def _integrate_all(vol, frames):
    for color, depth, pose, weight in frames:
        vol.integrate(color, depth, PATH_K, pose, obs_weight=weight)
    return vol


def _assert_same_results(got, want, frames, what):
    """got and want: SparseTSDFVolumes after the same frames -- equal blocks, updates, export, mesh and renders"""
    assert got.allocated_blocks() == want.allocated_blocks() > 0, what
    assert got.updated_voxels() == want.updated_voxels() > 0, what
    _assert_volumes_equal(got.to_dense(), want.to_dense(), what)
    for x, y in zip(got.get_mesh(), want.get_mesh()):
        assert x.shape == y.shape and np.array_equal(x, y), what
    poses = np.stack([frames[i][2] for i in (0, 3, 8)])
    for x, y in zip(got.render(PATH_K, poses, 60, 80), want.render(PATH_K, poses, 60, 80)):
        assert np.array_equal(x, y), what


def _prefix_needs(frames):
    """blocks the first i + 1 frames need, for every i, and the fixed volume of 16 384 blocks fed all of them"""
    from dvmvs.tsdf import SparseTSDFVolume
    big = SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384)
    needs = []
    for color, depth, pose, weight in frames:
        big.integrate(color, depth, PATH_K, pose, obs_weight=weight)
        needs.append(big.allocated_blocks())
    return needs, big


@pytest.mark.gpu
def test_gpu_many_growths_equal_a_large_enough_volume():
    """From 64 blocks, with no read between frames: the same export, blocks, update count, mesh (order included) and renders
    as a fixed volume of 16 384 blocks, and the export of the default box and of a box cutting through the path equal dense
    volumes over those boxes."""
    from dvmvs.tsdf import SparseTSDFVolume, TSDFVolume
    frames = _path_frames()
    grow = _integrate_all(SparseTSDFVolume(PATH_VOXEL, capacity_blocks=64, max_capacity_blocks=16384), frames)
    fixed = _integrate_all(SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384), frames)
    _assert_same_results(grow, fixed, frames, "grown from 64")
    assert grow.capacity > 64 and grow.growths >= 3, (grow.capacity, grow.growths)
    full = grow.to_dense()
    dense = TSDFVolume(full._vol_bnds, PATH_VOXEL)
    for color, depth, pose, weight in frames:
        dense.integrate(color, depth, PATH_K, pose, obs_weight=weight)
    _assert_volumes_equal(full, dense, "default box")
    assert grow.updated_voxels() == dense.updated_voxels()
    dense, grow = _fuse(frames, PATH_K, CUT_BOX, PATH_VOXEL, capacity_blocks=64, max_capacity_blocks=16384)
    _assert_volumes_equal(grow.to_dense(CUT_BOX), dense, "cut box")
    assert grow.growths >= 3


@pytest.mark.gpu
def test_gpu_growth_replays_its_own_copy_when_the_caller_overwrites_its_input():
    """Every frame through one CUDA depth tensor and one colour tensor, overwritten right after each integrate; the pool
    overflows on a frame in the middle of the path, so the replay runs after the caller's tensors have changed."""
    import torch
    from dvmvs.tsdf import SparseTSDFVolume
    frames = _path_frames()
    needs, fixed = _prefix_needs(frames)
    assert needs[3] < needs[4] < needs[-1]
    grow = SparseTSDFVolume(PATH_VOXEL, capacity_blocks=needs[3], max_capacity_blocks=16384)
    depth = torch.empty(frames[0][1].shape, dtype=torch.float32, device="cuda")
    color = torch.empty(frames[0][0].shape, dtype=torch.uint8, device="cuda")
    for c, d, pose, weight in frames:
        depth.copy_(torch.from_numpy(d))
        color.copy_(torch.from_numpy(c))
        grow.integrate(color, depth, PATH_K, pose, obs_weight=weight)
        depth.fill_(0.7)
        color.fill_(9)
    _assert_same_results(grow, fixed, frames, "caller overwrites")
    assert grow.growths >= 1


@pytest.mark.gpu
def test_gpu_a_refused_frame_after_an_overflowing_one_is_not_held():
    """A frame the library refuses (a NaN in the pose: numpy inverts it without raising, dvmvs_tsdf_sparse_allocate refuses
    it) right after the frame that overflows the pool, and another as the last call before the reads.  Each raises from its
    own integrate call and takes no ring slot; no later call raises, and the volume ends equal to a fixed volume fed the
    accepted frames."""
    from dvmvs.tsdf import SparseTSDFVolume
    frames = _path_frames()
    needs, fixed = _prefix_needs(frames)
    j = next(i for i, n in enumerate(needs) if n > needs[2])
    assert j < len(frames) - 1
    bad = np.eye(4)
    bad[0, 3] = np.nan
    grow = SparseTSDFVolume(PATH_VOXEL, capacity_blocks=needs[2], max_capacity_blocks=16384)
    for i, (color, depth, pose, weight) in enumerate(frames):
        grow.integrate(color, depth, PATH_K, pose, obs_weight=weight)
        if i == j or i == len(frames) - 1:
            accepted = grow._frames
            with pytest.raises(RuntimeError, match="not an invertible finite transform"):
                grow.integrate(color, depth, PATH_K, bad, obs_weight=weight)
            assert grow._frames == accepted and all(f.index < accepted for f in grow._held)
    _assert_same_results(grow, fixed, frames, "refused frames")
    assert grow.growths >= 1 and len(grow._held) == 0


@pytest.mark.gpu
def test_gpu_growth_from_a_full_two_entry_table():
    """capacity_blocks=1: a 2-entry hash table the first frame fills (table-full flag); the volume still ends equal to the
    large fixed volume"""
    from dvmvs import _native as N
    from dvmvs.tsdf import SparseTSDFVolume
    frames = _path_frames()
    grow = SparseTSDFVolume(PATH_VOXEL, capacity_blocks=1, max_capacity_blocks=16384)
    assert grow._keys.numel() == 2
    grow.integrate(*frames[0][:2], PATH_K, frames[0][2])
    grow._synchronize()
    assert int(grow._counters[1]) & N.SPARSE_TABLE_FULL and int(grow._counters[0]) == 2 and grow.capacity == 1
    _integrate_all(grow, frames[1:])
    fixed = _integrate_all(SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384), frames)
    _assert_same_results(grow, fixed, frames, "from a 2-entry table")


@pytest.mark.gpu
def test_gpu_at_the_cap_the_frames_from_the_overflowing_one_are_not_integrated():
    """max_capacity_blocks below the path's need: the reads raise naming the need and the cap; with j the first frame whose
    prefix needs more blocks than the cap, every block with a slot equals a large volume fed only frames 0 ... j-1, so no voxel
    holds an update from frame j or later, and the update count is that volume's."""
    import torch
    from dvmvs.tsdf import SparseTSDFVolume
    frames = _path_frames()
    needs, big = _prefix_needs(frames)
    cap = needs[4]
    j = next(i for i, n in enumerate(needs) if n > cap)
    assert 0 < j < len(frames)
    grow = _integrate_all(SparseTSDFVolume(PATH_VOXEL, capacity_blocks=min(64, cap), max_capacity_blocks=cap), frames)
    match = "need %d blocks, more than max_capacity_blocks %d: frame %d " % (needs[j], cap, j)
    with pytest.raises(RuntimeError, match=re.escape(match)):
        grow.allocated_blocks()
    with pytest.raises(RuntimeError, match=re.escape(match)):
        grow.to_dense()
    assert grow.capacity == cap
    prefix = _integrate_all(SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384), frames[:j])
    assert grow.updated_voxels() == prefix.updated_voxels() < big.updated_voxels()
    box = big.to_dense()._vol_bnds                                                  # holds every block frame j allocates
    want = prefix.to_dense(box)
    k0 = torch.tensor(np.rint(box[:, 0] / PATH_VOXEL).astype(np.int64), device="cuda")
    off = torch.stack(torch.meshgrid(*[torch.arange(8, device="cuda")] * 3, indexing="ij"), dim=-1)
    n = min(int(grow._counters[0]), grow.capacity)
    assert n == cap
    idx = (grow._coords[:n].long() * 8 - k0)[:, None, None, None, :] + off       # [n][8][8][8][3] dense voxel indices
    for name, pool, vol in zip(("tsdf", "weight", "color"), (grow._tsdf, grow._weight, grow._color), want.get_volume_tensors()):
        assert torch.equal(pool[:n], vol[idx[..., 0], idx[..., 1], idx[..., 2]]), "%s of a block with a slot differs" % name


@pytest.mark.gpu
def test_gpu_halt_mode_leaves_every_byte_of_the_volume_alone():
    """At the ABI: with HALT_ON_FULL in counters[3] and POOL_FULL set by hand, one allocate + integrate changes no byte of
    the table, the pool, counters[0:2] or the update count; the box kernel still resets counters[2]."""
    import torch
    from dvmvs import _native as N
    from dvmvs.tsdf import SparseTSDFVolume
    frames = _path_frames()
    vol = _integrate_all(SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384), frames[:2])
    vol._counters[3] = N.SPARSE_HALT_ON_FULL
    vol._counters[1] |= N.SPARSE_POOL_FULL
    state = (vol._keys, vol._slots, vol._coords, vol._tsdf, vol._weight, vol._color, vol._counters[:2], vol._updated)
    before = [t.clone() for t in state]
    assert int(vol._counters[2]) > 0
    color, depth, pose, weight = frames[2]
    vol.integrate(color, depth, PATH_K, pose, obs_weight=weight)
    vol._synchronize()
    for name, a, b in zip(("keys", "slots", "coords", "tsdf", "weight", "color", "counters[0:2]", "updated"), state, before):
        assert torch.equal(a, b), name
    assert int(vol._counters[2]) == 0
    vol._counters[3] = 0                                                              # halt off: the same frame now runs
    vol._counters[1] = 0
    vol.integrate(color, depth, PATH_K, pose, obs_weight=weight)
    assert vol.allocated_blocks() > int(before[6][0]) and vol.updated_voxels() > int(before[7][0])


@pytest.mark.gpu
def test_gpu_growth_touches_no_fringe_of_the_old_or_new_buffers():
    """test_gpu_many_growths_equal_a_large_enough_volume's growth with every allocation of dvmvs.tsdf in a guarded buffer
    (tests/guarded.py): the old and new tables, pools and the frame ring are all guarded, and no fringe is touched."""
    import torch
    from dvmvs import tsdf as T
    from tests import guarded as G
    frames = _path_frames()
    fixed = _integrate_all(T.SparseTSDFVolume(PATH_VOXEL, capacity_blocks=16384), frames)
    want = fixed.to_dense()
    with G.guard_allocations(modules=[T], guard_arguments=False):
        grow = _integrate_all(T.SparseTSDFVolume(PATH_VOXEL, capacity_blocks=64, max_capacity_blocks=16384), frames)
        assert grow.allocated_blocks() == fixed.allocated_blocks() and grow.growths >= 3
        for t in (grow._keys, grow._slots, grow._coords, grow._tsdf, grow._counters) + tuple(grow._ring[0].values()):
            assert G.REGISTRY.lookup(t) is not None
        torch.cuda.synchronize()
        G.verify(clear=False)
        got = grow.to_dense(want._vol_bnds)
        torch.cuda.synchronize()
        G.verify()
    _assert_volumes_equal(got, want, "guarded growth")
