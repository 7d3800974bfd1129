"""Marching cubes behind TSDFVolume.get_mesh (reference: sample-data/run-tsdf-reconstruction.py:329-358; csrc/mesh.cu).
CPU: the generated table (tools/gen_mc_tables.py) and the numpy oracle (oracle/mesh_oracle.py): every case's triangles close
into consistently oriented loops over exactly its crossing edges; meshes of random volumes are watertight; analytic SDFs give
the right topology, area and normals.
GPU: get_mesh equals the oracle with array_equal on verts, faces, norms and colours."""
import collections
import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle"))
sys.path.insert(0, os.path.join(REPO, "tools"))
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))
import gen_mc_tables as T  # noqa: E402
import mesh_oracle  # noqa: E402
import tsdf_cases  # noqa: E402

GOLD = np.load(os.path.join(REPO, "tests", "golden", "tsdf.npz"))
CORNER = np.array([[c & 1, c >> 1 & 1, c >> 2 & 1] for c in range(8)], dtype=np.float64)


def random_volume(shape, seed, outside_border=True):
    """Values in {-1, 0, 1} (ties: 0 is outside, t = 0 or 1 exactly) mixed with continuous noise."""
    rng = np.random.RandomState(seed)
    ties = rng.choice(np.float32([-1, 0, 1]), size=shape)
    vol = np.where(rng.rand(*shape) < 0.5, ties, rng.randn(*shape)).astype(np.float32)
    if outside_border:
        vol[0] = vol[-1] = 1
        vol[:, 0] = vol[:, -1] = 1
        vol[:, :, 0] = vol[:, :, -1] = 1
    return vol


def random_colors(shape, seed):
    rng = np.random.RandomState(seed)
    rgb = rng.randint(0, 256, size=shape + (3,)).astype(np.float32)
    return (rgb[..., 2] * np.float32(65536) + rgb[..., 1] * np.float32(256) + rgb[..., 0]).astype(np.float32)


def sphere(n=32, r=10.0):
    c = (n - 1) / 2.0
    g = np.mgrid[0:n, 0:n, 0:n].astype(np.float64)
    return (np.sqrt(((g - c) ** 2).sum(0)) - r).astype(np.float32), c


def torus(n=32, big=9.0, small=4.0):
    c = (n - 1) / 2.0
    x, y, z = np.mgrid[0:n, 0:n, 0:n].astype(np.float64) - c
    return (np.sqrt((np.sqrt(x * x + y * y) - big) ** 2 + z * z) - small).astype(np.float32)


def directed_edges(faces):
    return collections.Counter((int(p), int(q)) for f in faces for p, q in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0])))


def euler_characteristic(verts, faces):
    undirected = {tuple(sorted(e)) for e in directed_edges(faces)}
    return len(verts) - len(undirected) + len(faces)


def crossing_edge_count(vol):
    inside = vol < 0
    return sum(int((np.diff(inside.astype(np.int8), axis=a) != 0).sum()) for a in range(3))


# ---- the table -------------------------------------------------------------------------------------------------------------
def test_committed_table_equals_generator_output():
    with open(T.HEADER) as fh:
        assert fh.read() == T.render(), "csrc/mc_tables.cuh is stale: run python tools/gen_mc_tables.py"


def _face_of(e1, e2):
    """(axis, side) of the cube face holding both edges."""
    corners = set(T.EDGES[e1]) | set(T.EDGES[e2])
    for a in range(3):
        sides = {(c >> a) & 1 for c in corners}
        if len(sides) == 1:
            return a, sides.pop()
    return None


@pytest.mark.parametrize("case", range(256))
def test_table_case_closes_oriented_loops_over_its_crossing_edges(case):
    tris = T.TRIANGLES[case]
    crossing = T.crossing_edges(case)
    assert sorted({e for t in tris for e in t}) == crossing
    assert len(tris) == len(crossing) - 2 * len(T.loops(case)) and len(tris) <= T.MAX_TRIS
    d = directed_edges(tris)
    assert all(n == 1 for n in d.values())
    boundary = [e for e in d if (e[1], e[0]) not in d]          # the loops; every other edge is a fan diagonal used both ways
    assert sorted(p for p, _ in boundary) == crossing and sorted(q for _, q in boundary) == crossing
    mid = {e: (CORNER[T.EDGES[e][0]] + CORNER[T.EDGES[e][1]]) / 2 for e in range(12)}
    for p, q in boundary:
        face = _face_of(p, q)
        assert face is not None, (case, p, q)                   # a loop edge runs over one cube face
        axis, side = face
        normal = np.zeros(3)
        normal[axis] = 1.0 if side else -1.0
        for c in set(T.EDGES[p]) | set(T.EDGES[q]):
            if (case >> c) & 1:                                 # inside corners lie to the right, seen from outside the cube
                assert np.dot(np.cross(mid[q] - mid[p], CORNER[c] - mid[p]), normal) < 0, (case, p, q, c)
    for p, q in d:
        if (q, p) in d:
            assert _face_of(p, q) is None                       # diagonals never join two edges of one face


# ---- the oracle on random and analytic volumes -------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1])
def test_random_volume_mesh_is_watertight_and_covers_every_case(seed):
    vol = random_volume((32, 32, 32), seed)
    verts, faces, norms, colors, aux = mesh_oracle.marching_cubes(vol, np.zeros_like(vol), 1.0, [0, 0, 0], return_aux=True)
    assert len(np.unique(aux["cases"])) == 256
    d = directed_edges(faces)
    assert all(n == 1 and d.get((e[1], e[0])) == 1 for e, n in d.items())
    assert len(verts) == crossing_edge_count(vol)
    assert np.all((aux["t"] >= 0) & (aux["t"] <= 1))
    assert faces.dtype == np.int32 and faces.min() >= 0 and faces.max() < len(verts)
    assert np.all(np.diff(aux["keys"]) > 0)


def test_sphere_topology_area_and_normals():
    vol, c = sphere()
    verts, faces, norms, _ = mesh_oracle.marching_cubes(vol, np.zeros_like(vol), 1.0, [0, 0, 0])
    assert euler_characteristic(verts, faces) == 2
    p = verts[faces].astype(np.float64)
    cross = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    area = 0.5 * np.linalg.norm(cross, axis=1).sum()
    assert abs(area / (4 * np.pi * 10.0 ** 2) - 1) < 0.01
    radial = (verts - c) / np.linalg.norm(verts - c, axis=1)[:, None]
    assert np.all((norms * radial).sum(1) > 0.9)                           # outward: toward increasing tsdf
    assert np.all((cross * (p.mean(1) - c)).sum(1) > 0)                    # counter-clockwise seen from outside


def test_torus_topology():
    vol = torus()
    verts, faces, _, _ = mesh_oracle.marching_cubes(vol, np.zeros_like(vol), 1.0, [0, 0, 0])
    assert euler_characteristic(verts, faces) == 0


@pytest.mark.parametrize("case", sorted(tsdf_cases.CASES))
def test_golden_tsdf_volumes_mesh_with_reference_colours(case):
    n = sum(1 for k in GOLD.files if k.startswith(case + "/tsdf_after_"))
    tsdf, color = GOLD["%s/tsdf_after_%d" % (case, n - 1)], GOLD["%s/color_after_%d" % (case, n - 1)]
    origin, voxel = GOLD[case + "/vol_origin"], tsdf_cases.CASES[case]["voxel"]
    verts, faces, norms, colors, aux = mesh_oracle.marching_cubes(tsdf, color, voxel, origin, return_aux=True)
    assert len(faces) > 0 and len(verts) == crossing_edge_count(tsdf)
    d = directed_edges(faces)
    assert any((e[1], e[0]) not in d for e in d)                           # open: the surface reaches the volume border
    ind = np.round(aux["vind"]).astype(int)                               # :352, half-even
    folded = color[ind[:, 0], ind[:, 1], ind[:, 2]].astype(np.int64)      # integral and < 2^24: exact integer unfold
    assert np.array_equal(colors, np.stack([folded % 256, folded // 256 % 256, folded // 65536], axis=1).astype(np.uint8))
    assert np.all(np.abs(np.linalg.norm(norms, axis=1) - 1) < 1e-5)


# ---- GPU: get_mesh against the oracle ---------------------------------------------------------------------------------------
def _gpu_volume(tsdf, color, voxel=0.04, origin=(-1.3, 0.2, 0.7)):
    import torch
    from dvmvs.tsdf import TSDFVolume
    shape = tsdf.shape
    bounds = np.array([[o, o + (d - 0.5) * voxel] for o, d in zip(origin, shape)])
    vol = TSDFVolume(bounds, voxel)
    assert tuple(vol._vol_dim) == shape
    t, _, c = vol.get_volume_tensors()
    t.copy_(torch.from_numpy(np.ascontiguousarray(tsdf, dtype=np.float32)))
    c.copy_(torch.from_numpy(np.ascontiguousarray(color, dtype=np.float32)))
    return vol


def _assert_mesh_equals_oracle(vol):
    tsdf, color = vol.get_volume()
    want = mesh_oracle.marching_cubes(tsdf, color, vol._voxel_size, vol._vol_origin)
    got = vol.get_mesh()
    for name, g, w in zip(("verts", "faces", "norms", "colors"), got, want):
        assert g.dtype == w.dtype and g.shape == w.shape, (name, g.dtype, g.shape, w.dtype, w.shape)
        assert np.array_equal(g, w), "%s differs in %d of %d rows" % (name, int((g != w).any(axis=1).sum()), len(w))
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1])
def test_gpu_random_volume_equals_oracle(seed):
    vol = random_volume((32, 32, 32), seed)
    verts, faces, _, _ = _assert_mesh_equals_oracle(_gpu_volume(vol, random_colors(vol.shape, seed)))
    assert len(verts) == crossing_edge_count(vol) and len(faces) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(37, 23, 50), (2, 2, 2), (2, 9, 3), (70, 5, 33), (17, 64, 2)])
def test_gpu_ragged_volume_equals_oracle(shape):
    vol = random_volume(shape, sum(shape), outside_border=False)
    _assert_mesh_equals_oracle(_gpu_volume(vol, random_colors(shape, 7)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_gpu_analytic_volume_equals_oracle(name):
    vol = sphere()[0] if name == "sphere" else torus()
    verts, faces, _, _ = _assert_mesh_equals_oracle(_gpu_volume(vol, random_colors(vol.shape, 3), voxel=0.5, origin=(-8.0, -8.0, -8.0)))
    assert euler_characteristic(verts, faces) == (2 if name == "sphere" else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 6, 7), (6, 1, 7), (6, 7, 1), (1, 1, 1)])
def test_gpu_volume_with_a_unit_dimension_has_an_empty_mesh(shape):
    vol = random_volume(shape, 4, outside_border=False)
    verts, faces, norms, colors = _gpu_volume(vol, random_colors(shape, 4)).get_mesh()
    assert verts.shape == (0, 3) and verts.dtype == np.float32
    assert faces.shape == (0, 3) and faces.dtype == np.int32
    assert norms.shape == (0, 3) and norms.dtype == np.float32
    assert colors.shape == (0, 3) and colors.dtype == np.uint8


@pytest.mark.gpu
def test_gpu_fresh_volume_has_an_empty_mesh_and_point_cloud():
    from dvmvs.tsdf import TSDFVolume
    vol = TSDFVolume(np.array([[0.0, 1.0], [0.0, 0.8], [0.0, 0.6]]), 0.05)          # all ones
    verts, faces, norms, colors = vol.get_mesh()
    assert verts.shape == faces.shape == norms.shape == colors.shape == (0, 3)
    assert vol.get_point_cloud().shape == (0, 6)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(tsdf_cases.CASES))
def test_gpu_integrated_golden_case_mesh_equals_oracle(case):
    from dvmvs.tsdf import TSDFVolume
    inp = tsdf_cases.inputs(case)
    vol = TSDFVolume(inp["bounds"], inp["voxel"])
    for fr in inp["frames"]:
        vol.integrate(fr["color"], fr["depth"], inp["K"], fr["pose"], obs_weight=fr["weight"])
    verts, faces, norms, colors = _assert_mesh_equals_oracle(vol)
    assert len(faces) > 0
    assert np.array_equal(vol.get_point_cloud(), np.hstack([verts, colors]))


@pytest.mark.gpu
def test_gpu_production_room_mesh_equals_oracle_and_repeats():
    """The 3.84 M-voxel room of test_tsdf (200 x 160 x 120 at 4 cm) after three fused frames.  Its 15 000 per-CTA counts take
    a two-level scan (15 000 pairs in 59 blocks of 256, then the 59 block sums in one); the scratch query says so."""
    import ctypes
    import torch
    from dvmvs import _native as N
    from dvmvs.tsdf import TSDFVolume
    rng = np.random.RandomState(11)
    h, w = 256, 320
    K = np.array([[250.0, 0, 160.3], [0, 251.0, 127.6], [0, 0, 1]])
    vol = TSDFVolume(np.array([[-4.0, 4.0], [-3.2, 3.2], [0.0, 4.8]]), 0.04)
    for i in range(3):
        yy, xx = np.mgrid[0:h, 0:w]
        depth = (2.0 + 0.8 * np.sin(xx / 40.0 + i) * np.cos(yy / 30.0) + 0.01 * rng.rand(h, w)).astype(np.float32)
        depth[rng.rand(h, w) < 0.05] = 0
        color = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
        pose = np.eye(4)
        pose[:3, 3] = [0.1 * i, -0.05 * i, 0.02 * i]
        c, s = np.cos(0.05 * i), np.sin(0.05 * i)
        pose[:3, :3] = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
        vol.integrate(color, depth, K, pose, obs_weight=1.0)
    nbytes = ctypes.c_longlong(0)
    N.check(N.lib().dvmvs_mesh_scratch_bytes(200, 160, 120, ctypes.byref(nbytes)), "mesh_scratch_bytes")
    assert nbytes.value == 8 * (1 + 15000 + 59)
    first = _assert_mesh_equals_oracle(vol)
    assert len(first[1]) > 50000
    again = vol.get_mesh_tensors()
    assert all(t.is_cuda for t in again)
    for a, b in zip(first, again):
        assert np.array_equal(a, b.cpu().numpy())
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_gpu_mesh_scan_spans_several_levels():
    """A 17.3 M-voxel volume holding a sphere and a random block: its 67 600 per-CTA counts take a three-level scan
    (67 600 pairs in 265 blocks, 265 sums in 2 blocks, 2 sums in one)."""
    n = (260, 260, 256)
    g = [np.arange(d, dtype=np.float32) for d in n]
    vol = np.sqrt((g[0][:, None, None] - 130) ** 2 + (g[1][None, :, None] - 100) ** 2 + (g[2][None, None, :] - 128) ** 2) - 60
    vol = vol.astype(np.float32)
    vol[200:240, 200:240, 20:60] = random_volume((40, 40, 40), 9, outside_border=False)
    assert (int(np.prod(n)) + 255) // 256 == 67600
    import ctypes
    from dvmvs import _native as N
    nbytes = ctypes.c_longlong(0)
    N.check(N.lib().dvmvs_mesh_scratch_bytes(*n, ctypes.byref(nbytes)), "mesh_scratch_bytes")
    assert nbytes.value == 8 * (1 + 67600 + 265 + 2)
    verts, faces, _, _ = _assert_mesh_equals_oracle(_gpu_volume(vol, random_colors(n, 1), voxel=0.02))
    assert len(verts) == crossing_edge_count(vol)


@pytest.mark.gpu
def test_gpu_get_mesh_needs_no_scikit_image(monkeypatch):
    monkeypatch.setitem(sys.modules, "skimage", None)                       # `import skimage` raises ImportError
    with pytest.raises(ImportError):
        import skimage  # noqa: F401
    vol, _ = sphere()
    verts, faces, _, colors = _assert_mesh_equals_oracle(_gpu_volume(vol, random_colors(vol.shape, 5), voxel=0.5, origin=(0.0, 0.0, 0.0)))
    assert np.array_equal(_gpu_volume(vol, random_colors(vol.shape, 5), voxel=0.5, origin=(0.0, 0.0, 0.0)).get_point_cloud(),
                          np.hstack([verts, colors]))
