"""The voxel-block TSDF volume's allocation (csrc/tsdf_sparse.cu) stage by stage, against the reference's per-voxel rule
(tests/tsdf_block_reference.py).  SparseTSDFVolume equals a dense TSDFVolume with the same origin only if the allocation never
misses a block that the reference updates; the end-to-end tests of test_tsdf_sparse.py see only the blocks inside the dense box
they compare over, and only scenes near the origin.

CPU: the float64 restatements of the candidate box and the block test cover the ground truth on every frame set (exact), the
box's float32-spacing margin changes nothing near the origin, and the block test's depth test really drops blocks.
GPU, frame by frame on a fixed volume: each frame's visible list is duplicate-free, covers the ground truth and equals the
candidate box's blocks that pass the restated block test (up to blocks the device's contracted arithmetic may decide the
other way, counted and bounded); the allocated blocks are the union of the visible lists; the hash table's keys, slots and
coordinates agree and every key is where linear probing finds it -- also after every rehash of a growing volume.  Far from
the origin the export equals a dense volume, which in turn equals the oracle on a small box."""
import functools
import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle"))
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))
import tsdf_cases  # noqa: E402
import tsdf_oracle  # noqa: E402

from tests import tsdf_block_reference as R  # noqa: E402
from tests.test_tsdf import _rot  # noqa: E402
from tests.test_tsdf_sparse import PATH_K, PATH_VOXEL, _adversarial_frames, _path_frames  # noqa: E402


class FrameSet(object):
    def __init__(self, origin, voxel, K, frames, far_scale=None):
        self.origin = np.asarray(origin, dtype=np.float32)      # the volume's origin (float32, as the volume keeps it)
        self.voxel = float(voxel)
        self.K = np.asarray(K, dtype=np.float64)
        self.frames = frames                                      # [(colour, depth, pose, obs_weight)]
        self.far_scale = far_scale                                # far rows: metres per unit of their scene


def _colour(rng, h, w):
    return rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)


def _cases(name, offset):
    """oracle/tsdf_cases.py, the whole scene moved by offset metres"""
    inp = tsdf_cases.inputs(name)
    frames = []
    for fr in inp["frames"]:
        pose = fr["pose"].copy()
        pose[:3, 3] += offset
        frames.append((fr["color"], fr["depth"], pose, fr["weight"]))
    return FrameSet(inp["bounds"][:, 0] + offset, inp["voxel"], inp["K"], frames)


def _inside(offset):
    """the inside-the-volume cameras of test_tsdf_sparse.py (every axis and obliquely), origin at the dense volume's"""
    bounds = np.array([[-2.0, 2.0], [-1.6, 1.6], [-2.0, 2.0]]) + offset
    K = np.array([[100.0, 0, 63.5], [0, 100.0, 47.5], [0, 0, 1]])
    return FrameSet(bounds[:, 0], 0.04, K, _adversarial_frames(offset))


def _plane():
    """cameras at block corners, faces and inside blocks, with a wide field of view and depth from 3 cm: the camera plane cuts
    through blocks that hold updated voxels on both sides of it"""
    rng = np.random.RandomState(31)
    h, w, v = 40, 48, 0.04
    K = np.array([[0.45 * w, 0, w / 2.0 - 0.5], [0, 0.45 * w, h / 2.0 - 0.5], [0, 0, 1]])
    centres = [(0, 0, 0), (8 * v, -8 * v, 16 * v), (3.5 * v, 0.25 * v, -4 * v), (-8 * v, 2.7 * v, 8 * v), (0.013, -0.021, 0.007)]
    frames = []
    for i, c in enumerate(centres):
        depth = (0.03 + 0.6 * rng.rand(h, w)).astype(np.float32)
        pose = np.eye(4)
        pose[:3, :3] = _rot(rng.randn(3), [0.0, 0.3, np.pi / 2, 2.5, 1.1][i])
        pose[:3, 3] = c
        frames.append((_colour(rng, h, w), depth, pose, 1.0))
    return FrameSet((0.0, 0.0, 0.0), v, K, frames)


def _border():
    """axis-aligned cameras on the lattice of a dyadic voxel, with the image's border rays through voxel points: many voxels
    project exactly onto a half pixel at the border (rint's half-even tie decides), so blocks graze the image"""
    rng = np.random.RandomState(37)
    h, w, v = 15, 20, 1.0 / 32
    K = np.array([[20.0, 0, 9.5], [0, 20.0, 7.0], [0, 0, 1]])
    rots = [np.eye(3), np.array([[0.0, 0, 1], [0, 1, 0], [-1, 0, 0]]), np.array([[1.0, 0, 0], [0, 0, -1], [0, 1, 0]]),
            np.array([[-1.0, 0, 0], [0, -1, 0], [0, 0, 1]])]
    frames = []
    for i, rot in enumerate(rots):
        depth = (0.5 + 0.25 * (rng.rand(h, w) < 0.5)).astype(np.float32)
        pose = np.eye(4)
        pose[:3, :3] = rot
        pose[:3, 3] = np.array([8 * i, -4 * i, 3 * i]) * v
        frames.append((_colour(rng, h, w), depth, pose, 1.0))
    return FrameSet((0.0, 0.0, 0.0), v, K, frames)


def _ragged():
    """61 x 83 images: the last tile row and column are ragged"""
    rng = np.random.RandomState(41)
    h, w = 61, 83
    K = np.array([[0.8 * w, 0, 41.3], [0, 0.8 * w, 29.8], [0, 0, 1]])
    frames = []
    for i in range(3):
        yy, xx = np.mgrid[0:h, 0:w]
        depth = (1.0 + 0.6 * np.sin(xx / 7.0 + i) * np.cos(yy / 5.0) + 0.2 * rng.rand(h, w)).astype(np.float32)
        depth[-3:, :] = 2.4                                     # the ragged tiles hold the frame's largest depth
        depth[:, -2:] = 2.2
        pose = np.eye(4)
        pose[:3, :3] = _rot(rng.randn(3), 0.4 * i)
        pose[:3, 3] = rng.uniform(-0.3, 0.3, size=3)
        frames.append((_colour(rng, h, w), depth, pose, 1.0))
    return FrameSet((-0.013, 0.021, 0.0), 0.05, K, frames)


def _holes():
    """float64 depth with zero, negative and NaN pixels and a whole 16 x 16 tile without a valid pixel"""
    rng = np.random.RandomState(43)
    h, w = 40, 56
    K = np.array([[0.9 * w, 0, w / 2.0 + 0.3], [0, 0.9 * w, h / 2.0 - 0.2], [0, 0, 1]])
    frames = []
    for i in range(3):
        depth = 0.4 + 1.2 * rng.rand(h, w)
        r = rng.rand(h, w)
        depth[r < 0.1] = 0.0
        depth[(r >= 0.1) & (r < 0.2)] = -0.7
        depth[(r >= 0.2) & (r < 0.3)] = np.nan
        depth[16:32, 16:32] = np.where(rng.rand(16, 16) < 0.5, np.nan, -1.0)
        depth[0, 0] = 3.0 if i == 0 else depth[0, 0]           # one far pixel sets the frame's largest depth
        pose = np.eye(4)
        pose[:3, :3] = _rot(rng.randn(3), 0.5)
        pose[:3, 3] = rng.uniform(-0.2, 0.2, size=3)
        frames.append((_colour(rng, h, w).astype(np.float32), depth, pose, 1.0 + 0.5 * i))
    return FrameSet((0.0, 0.0, 0.0), 0.04, K, frames)


WALL = (16, 80, 16, 112)        # the wall's pixel rows and columns: whole 16 x 16 tiles


def _wall():
    """a near wall over whole tiles in the middle of the image and a far background: the block test's depth test (c) drops
    the blocks behind the wall"""
    rng = np.random.RandomState(47)
    h, w = 96, 128
    K = np.array([[100.0, 0, 63.5], [0, 100.0, 47.5], [0, 0, 1]])
    depth = np.full((h, w), 3.0, np.float32)
    depth[WALL[0]:WALL[1], WALL[2]:WALL[3]] = 0.6
    pose = np.eye(4)
    pose[:3, 3] = (0.011, -0.007, 0.003)
    return FrameSet((0.0, 0.0, 0.0), 0.04, K, [(_colour(rng, h, w), depth, pose, 1.0)])


FAR = {
    # origin, voxel: 1 mm at 1e5 m (float32 spacing 7.8 mm), 1 cm at 5e5 m (3.1 cm), a UTM-like origin (0.5 m in x) at 2 and 5 cm
    "far-1e5-1mm": ((1.0e5, -1.0e5, 3.7e4), 0.001),
    "far-5e5-1cm": ((5.0e5, 5.0e5, -5.0e5), 0.01),
    "far-utm-2cm": ((4.2e6, 5.1e5, 31.0), 0.02),
    "far-utm-5cm": ((4.2e6, 5.1e5, 31.0), 0.05),
}


AXIS_VIEWS = [np.array([[0.0, 0, 1], [0, 1, 0], [-1, 0, 0]]), np.array([[0.0, 0, -1], [0, 1, 0], [1, 0, 0]]),
              np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]]), np.array([[1.0, 0, 0], [0, -1, 0], [0, 0, -1]])]   # +x, -x, +y, -z


def _far(name):
    """24 x 32 frames with cameras within 0.7 s of origin + 2.8 s (1, 1, 1), s = 1 m at 2 cm and above, scaled with the voxel
    below, so every voxel they update has non-negative indices: 6 in random orientations with depth 0.3 s .. 1.2 s, then 4
    looking along +x, -x, +y and -z at a flat surface 1.1 s away, whose updated voxels fill the frustum box's far face (where
    float32 rounding carries voxels from outside an index-space margin into the box)"""
    origin, v = FAR[name]
    s = min(1.0, v / 0.02)
    rng = np.random.RandomState(53)
    h, w = 24, 32
    K = np.array([[0.9 * w, 0, w / 2.0 - 0.3], [0, 0.92 * w, h / 2.0 + 0.2], [0, 0, 1]])
    o = np.float32(origin).astype(np.float64)
    frames = []
    for i in range(6 + len(AXIS_VIEWS)):
        pose = np.eye(4)
        if i < 6:
            depth = (s * (0.3 + 0.9 * rng.rand(h, w))).astype(np.float32)
            pose[:3, :3] = _rot(rng.randn(3), rng.uniform(0, np.pi))
        else:
            depth = np.full((h, w), 1.1 * s, np.float32)
            pose[:3, :3] = AXIS_VIEWS[i - 6]
        depth[rng.rand(h, w) < 0.08] = 0.0
        pose[:3, 3] = o + s * (2.8 + rng.uniform(-0.7, 0.7, size=3))
        if i in (6, 7):
            reach = (float(depth.max()) + 5 * v) * (1 + 1e-9) + 1e-9
            pose[0, 3] = _edge_camera(o, v, pose[0, 3], reach, 1 if i == 6 else -1, s)
        frames.append((_colour(rng, h, w), depth, pose, 1.0))
    return FrameSet(o, v, K, frames, far_scale=s)


def _edge_camera(origin, v, base, reach, sign, s):
    """The camera x within 0.3 s of base that puts the far face of a view along +x (sign 1) or -x (-1), `reach` away, where
    float32 rounding carries the voxel just past a two-voxel index-space margin (rounded out to whole blocks) furthest into
    the face: such voxels are updated, and a box with only that margin misses their blocks.  base when no position does
    (the float32 spacing there is under four voxels)."""
    c = base + s * np.linspace(-0.3, 0.3, 6001)
    face = c + sign * reach
    q = (face - origin[0]) / v
    if sign > 0:
        g = R.BLOCK * (np.floor((np.floor(q) + 2) / R.BLOCK) + 1)
    else:
        g = R.BLOCK * np.floor((np.floor(q) - 2) / R.BLOCK) - 1
    gap = sign * (face - R.voxel_world(origin, v, g.astype(np.int64), 0)) - 1e-6 * s
    return float(c[np.argmax(gap)]) if gap.max() > 0 else base



def _path():
    """test_tsdf_sparse.py's camera path through negative block coordinates"""
    return FrameSet((0.0, 0.0, 0.0), PATH_VOXEL, PATH_K, _path_frames())


NEAR_ROWS = ["cases-%s-%d" % (c, o) for c in sorted(tsdf_cases.CASES) for o in (0, 150)] + [
    "inside-0", "inside-150", "plane", "border", "ragged-61x83", "holes", "wall"]
FAR_ROWS = sorted(FAR)
ROWS = NEAR_ROWS + FAR_ROWS


@functools.lru_cache(maxsize=None)
def frame_set(row):
    if row.startswith("cases-"):
        _, name, off = row.split("-")
        return _cases(name, float(off))
    if row.startswith("inside-"):
        return _inside(float(row.split("-")[1]))
    if row in FAR:
        return _far(row)
    return {"plane": _plane, "border": _border, "ragged-61x83": _ragged, "holes": _holes, "wall": _wall, "path": _path}[row]()


@functools.lru_cache(maxsize=None)
def needed(row, i):
    fs = frame_set(row)
    _, depth, pose, _ = fs.frames[i]
    return R.needed_blocks(depth, fs.K, pose, fs.origin, fs.voxel)


def _outside_box(blocks, lo, n):
    blocks = np.asarray(blocks).reshape(-1, 3)
    if lo is None:
        return blocks
    return blocks[np.any((blocks < lo) | (blocks >= lo + n), axis=1)]


def _allocation(f, widened=True):
    """the restated allocation of one frame: the candidate box's blocks that pass the block test, as a set"""
    kind, lo, n = R.candidate_box(f, widened=widened)
    if kind != "box":
        return set()
    blocks = R.box_blocks(lo, n)
    seen, _ = R.block_seen(f, blocks)
    return R.as_set(blocks[seen])


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_restated_hash_and_key_packing():
    """block_key packs 21 bits per axis biased by 2^20 (x highest) and decodes back; block_hash is the high half of the
    64-bit product; check_table accepts a table built by linear probing and names each broken invariant"""
    b = np.array([[0, 0, 0], [-1, 2, -3], [-(1 << 20), (1 << 20) - 1, 5], [1000, -1000, 77]])
    k = R.block_key(b)
    assert int(k[0]) == (1 << 20) << 42 | (1 << 20) << 21 | (1 << 20)
    assert int(k[2]) == 0 << 42 | ((1 << 21) - 1) << 21 | ((1 << 20) + 5)
    assert np.array_equal(R.decode_key(k), b) and int(k.max()) < 1 << 63
    assert int(R.block_hash(k[1:2], (1 << 30) - 1)[0]) == ((int(k[1]) * R.HASH_MUL) % (1 << 64)) >> 32 & ((1 << 30) - 1)
    size, coords = 16, np.array([[3, 1, 2], [-5, 0, 9], [7, 7, 7], [0, -2, 4], [1, 1, 1]])
    keys, slots = np.full(size, -1, np.int64), np.full(size, -1, np.int32)
    for s, key in enumerate(R.block_key(coords)):
        h = int(R.block_hash(np.array([key]), size - 1)[0])
        while keys[h] != -1:
            h = (h + 1) % size
        keys[h], slots[h] = np.int64(int(key)), s
    R.check_table(keys, slots, coords, len(coords))
    # slot 0's key moved past the first empty entry of its probe sequence: a lookup stops at that entry and misses it
    moved_keys, moved_slots = keys.copy(), slots.copy()
    at = int(np.nonzero(slots == 0)[0][0])
    moved_keys[at], moved_slots[at] = -1, -1
    h = int(R.block_hash(R.block_key(coords[:1]), size - 1)[0])
    empties = [(h + j) % size for j in range(size) if moved_keys[(h + j) % size] == -1]
    moved_keys[empties[1]], moved_slots[empties[1]] = keys[at], 0
    for broken, match in (((keys, slots, coords, 4), "non-empty keys"),
                          ((keys, np.where(slots == 0, 1, slots), coords, 5), "permutation"),
                          ((keys, slots, coords[[1, 0, 2, 3, 4]], 5), "decode"),
                          ((moved_keys, moved_slots, coords, 5), "after an empty entry")):
        with pytest.raises(AssertionError, match=match):
            R.check_table(*broken)


@pytest.mark.parametrize("row", ROWS)
def test_restated_box_and_block_test_cover_the_reference(row):
    """On every frame: every block holding a voxel the reference updates lies in the candidate box and passes the block test
    (both exact).  Near the origin, the float32-spacing term of the box's margin moves each face by at most one block and
    changes no frame's allocation."""
    fs = frame_set(row)
    total = 0
    for i, (_, depth, pose, _) in enumerate(fs.frames):
        f = R.Frame(depth, fs.K, pose, fs.origin, fs.voxel)
        need = needed(row, i)
        total += len(need)
        kind, lo, n = R.candidate_box(f)
        assert kind == "box" or len(need) == 0, (row, i, kind)
        missed = _outside_box(need, lo, n)
        assert len(missed) == 0, "%s frame %d: %d needed blocks outside the candidate box %s + %s: %s" % (
            row, i, len(missed), lo.tolist(), n.tolist(), missed[:8].tolist())
        seen, _ = R.block_seen(f, need)
        assert seen.all(), "%s frame %d: the block test drops %d needed blocks: %s" % (row, i, int((~seen).sum()),
                                                                                         need[~seen][:8].tolist())
        if row in NEAR_ROWS:
            kind0, lo0, n0 = R.candidate_box(f, widened=False)
            assert kind0 == kind
            if kind == "box":
                assert np.all(lo0 - lo <= 1) and np.all(lo0 - lo >= 0), (row, i, lo0, lo)
                assert np.all((lo + n) - (lo0 + n0) <= 1) and np.all((lo + n) - (lo0 + n0) >= 0), (row, i, lo0 + n0, lo + n)
                assert _allocation(f) == _allocation(f, widened=False), (row, i)
    assert total > 0


@pytest.mark.parametrize("row", ["far-1e5-1mm", "far-utm-2cm", "far-utm-5cm"])
def test_index_space_margin_misses_blocks_far_from_the_origin(row):
    """The box margin of two voxels in index space alone (the margin before the float32-spacing term): where the float32
    spacing of the world points exceeds four voxels (7.8 voxels at 1e5 m and 1 mm, 25 and 10 at the UTM-like x with 2 and 5
    cm), voxels from outside that box round into the frustum and the reference updates their blocks.  (At 5e5 m and 1 cm the
    spacing is 3.1 voxels: two voxels of margin suffice there.)"""
    fs = frame_set(row)
    missed = 0
    for i, (_, depth, pose, _) in enumerate(fs.frames):
        f = R.Frame(depth, fs.K, pose, fs.origin, fs.voxel)
        _, lo, n = R.candidate_box(f, widened=False)
        missed += len(_outside_box(needed(row, i), lo, n))
    assert missed > 0


def test_depth_test_drops_the_blocks_behind_a_near_wall():
    """Test (c) of the block test: behind the wall's tiles, from 0.6 m + trunc to the background's 3 m, no block is
    allocated unless another tile it projects into sees further; without (c) the frustum's blocks are all kept"""
    fs = frame_set("wall")
    _, depth, pose, _ = fs.frames[0]
    f = R.Frame(depth, fs.K, pose, fs.origin, fs.voxel)
    kind, lo, n = R.candidate_box(f)
    blocks = R.box_blocks(lo, n)
    seen, _ = R.block_seen(f, blocks)
    flat = R.Frame(np.full_like(depth, depth.max()), fs.K, pose, fs.origin, fs.voxel)
    kept, _ = R.block_seen(flat, blocks)                         # every tile at the largest depth: (c) drops nothing closer
    need = R.as_set(needed("wall", 0))
    assert need <= R.as_set(blocks[seen])
    # blocks whose every corner projects inside the wall's tiles, between 0.9 m and 2.7 m (the camera looks along +z)
    corners = np.stack([(blocks + np.array([cx, cy, cz])) * 8 * fs.voxel - pose[:3, 3]
                        for cx in (0, 1) for cy in (0, 1) for cz in (0, 1)])
    u = corners[..., 0] * fs.K[0, 0] / corners[..., 2] + fs.K[0, 2]
    v = corners[..., 1] * fs.K[1, 1] / corners[..., 2] + fs.K[1, 2]
    behind_wall = np.all((corners[..., 2] > 0.9) & (corners[..., 2] < 2.7) & (u > WALL[2]) & (u < WALL[3] - 1) & (v > WALL[0])
                         & (v < WALL[1] - 1), axis=0)
    assert behind_wall.sum() > 10 and not seen[behind_wall].any() and kept[behind_wall].all()
    ratio = seen.sum() / len(need)
    print("wall: %d blocks in the box, %d without test (c), %d allocated, %d needed: allocated / needed %.3f" % (
        len(blocks), int(kept.sum()), int(seen.sum()), len(need), ratio))
    assert not (seen & ~kept).any()                              # (c) only ever drops


# ------------------------------------------------------------------------------------------------------------------ GPU
def _state(vol):
    import torch
    torch.cuda.synchronize()
    return (vol._counters.cpu().numpy().astype(np.int64), vol._visible.cpu().numpy(), vol._coords.cpu().numpy().astype(np.int64),
            vol._keys.cpu().numpy(), vol._slots.cpu().numpy())


def _check_table(vol, what):
    counters, _, coords, keys, slots = _state(vol)
    assert counters[1] & 3 == 0, "%s: capacity flags %d" % (what, counters[1])
    n = int(counters[0])
    try:
        R.check_table(keys, slots, coords, n)
    except AssertionError as e:
        raise AssertionError("%s: %s" % (what, e))
    return R.as_set(coords[:n])


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS + ["path"])
def test_gpu_allocation_frame_by_frame(row):
    from dvmvs.tsdf import SparseTSDFVolume
    fs = frame_set(row)
    vol = SparseTSDFVolume(fs.voxel, origin=fs.origin, capacity_blocks=16384)
    union, need_union, tested, ambiguous, disagree = set(), set(), 0, 0, 0
    for i, (colour, depth, pose, weight) in enumerate(fs.frames):
        vol.integrate(colour, depth, fs.K, pose, obs_weight=weight)
        counters, visible, coords, _, _ = _state(vol)
        what = "%s frame %d" % (row, i)
        vis = visible[:counters[2]]
        assert len(np.unique(vis)) == len(vis), "%s: a slot is listed twice" % what
        got = R.as_set(coords[vis])
        need = R.as_set(needed(row, i))
        assert need <= got, "%s: %d needed blocks not visible: %s" % (what, len(need - got), sorted(need - got)[:8])
        f = R.Frame(depth, fs.K, pose, fs.origin, fs.voxel)
        kind, lo, n = R.candidate_box(f)
        _, lo_w, n_w = R.candidate_box(f, slack=1e-9)
        _, lo_n, n_n = R.candidate_box(f, slack=-1e-9)
        if kind != "box":
            assert not got, what
            continue
        blocks = R.box_blocks(lo_w, n_w)
        seen, amb = R.block_seen(f, blocks)
        in_box = np.all((blocks >= lo) & (blocks < lo + n), axis=1)
        amb |= ~np.all((blocks >= lo_n) & (blocks < lo_n + n_n), axis=1)
        want = in_box & seen
        assert got <= R.as_set(blocks), "%s: visible blocks outside the candidate box" % what
        is_got = np.array([tuple(b) in got for b in blocks.tolist()])
        wrong = (is_got != want) & ~amb
        assert not wrong.any(), "%s: %d blocks allocated against the restated block test, e.g. %s (allocated %s)" % (
            what, int(wrong.sum()), blocks[wrong][:4].tolist(), is_got[wrong][:4].tolist())
        tested += len(blocks)
        ambiguous += int(amb.sum())
        disagree += int(((is_got != want) & amb).sum())
        union |= got
        need_union |= need
        assert _check_table(vol, what) == union, "%s: the allocated blocks are not the union of the visible lists" % what
    print("%s: %d blocks allocated, %d needed, allocated / needed %.3f; %d of %d blocks tested ambiguous (%d decided the other "
          "way)" % (row, len(union), len(need_union), len(union) / max(len(need_union), 1), ambiguous, tested, disagree))
    assert ambiguous <= 0.1 * tested, "%s: %d of %d blocks ambiguous" % (row, ambiguous, tested)


@pytest.mark.gpu
@pytest.mark.parametrize("row", ["path", "far-utm-2cm"])
def test_gpu_rehash_keeps_the_table_invariants(row):
    """A volume growing from 64 blocks: the table after every rehash, and after every frame, passes the checks, and the
    blocks end as the fixed volume's"""
    from dvmvs.tsdf import SparseTSDFVolume
    fs = frame_set(row)
    fixed = SparseTSDFVolume(fs.voxel, origin=fs.origin, capacity_blocks=16384)
    grow = SparseTSDFVolume(fs.voxel, origin=fs.origin, capacity_blocks=64, max_capacity_blocks=16384)
    rehashed = []
    inner = grow._grow

    def checked_grow(capacity, n_blocks):
        inner(capacity, n_blocks)
        blocks = _check_table(grow, "%s after growth %d" % (row, grow.growths))
        assert len(blocks) == n_blocks
        rehashed.append(n_blocks)
    grow._grow = checked_grow
    for i, (colour, depth, pose, weight) in enumerate(fs.frames):
        fixed.integrate(colour, depth, fs.K, pose, obs_weight=weight)
        grow.integrate(colour, depth, fs.K, pose, obs_weight=weight)
        grow.allocated_blocks()
        _check_table(grow, "%s frame %d" % (row, i))
    assert grow.growths >= 3 and len(rehashed) == grow.growths
    assert _check_table(grow, row) == _check_table(fixed, row)


@pytest.mark.gpu
@pytest.mark.parametrize("row", FAR_ROWS)
def test_gpu_far_origin_sparse_equals_dense_and_dense_equals_oracle(row):
    """Far from the origin: the export over a dense volume's box (every updated voxel inside it) equals the dense volume and
    the update counts agree; on a small box the dense volume equals the oracle (its float32 frustum pre-test at these
    magnitudes)"""
    from dvmvs.tsdf import TSDFVolume
    from tests.test_tsdf import _same
    from tests.test_tsdf_sparse import _assert_volumes_equal, _fuse
    fs = frame_set(row)
    s = fs.far_scale
    o = fs.origin.astype(np.float64)
    bounds = np.stack([o, o + 5.6 * s], axis=1)
    frames = [(c, d, p, wt) for c, d, p, wt in fs.frames]
    dense, sparse = _fuse(frames, fs.K, bounds, fs.voxel, capacity_blocks=16384)
    assert np.array_equal(dense._vol_origin, fs.origin)
    _assert_volumes_equal(sparse.to_dense(bounds), dense, row)
    assert sparse.updated_voxels() == dense.updated_voxels() > 0
    small = np.stack([o + 2.2 * s, o + 3.4 * s], axis=1)
    gpu, orc = TSDFVolume(small, fs.voxel), tsdf_oracle.TSDFVolume(small, fs.voxel)
    total = 0
    for c, d, p, wt in frames:
        gpu.integrate(c, d, fs.K, p, obs_weight=wt)
        total += orc.integrate(c, d, fs.K, p, wt)
    tsdf, colour = gpu.get_volume()
    assert _same(gpu.get_volume_tensors()[1].cpu().numpy(), orc.weight), row
    assert _same(tsdf, orc.tsdf) and _same(colour, orc.color), row
    assert gpu.updated_voxels() == total > 0
