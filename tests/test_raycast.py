"""Ray casting behind TSDFVolume.render (csrc/raycast.cu; no reference counterpart).
CPU: the numpy oracle (oracle/raycast_oracle.py) against analytic surfaces -- a plane (trilinear interpolation exact), a
Euclidean truncated sphere, a scene fused by the integration oracle -- plus the edge cases of the range clipping, and the march
with the empty-space skip equal to the march without it.
GPU: render equals the oracle with array_equal on depth, normals and colours; one launch of V views equals V launches; poses
as CUDA tensors equal poses as numpy arrays; malformed calls raise."""
import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle"))
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))
import raycast_oracle  # noqa: E402
import tsdf_cases  # noqa: E402
import tsdf_oracle  # noqa: E402

VOXEL = 0.05
ORIGIN = np.array([-0.8, -0.75, 0.3], dtype=np.float32)
H, W = 48, 64
K = np.array([[60.0, 0, 31.7], [0, 61.0, 23.4], [0, 0, 1]])


# ---- fixtures: volumes, cameras, analytic hits ---------------------------------------------------------------------------
def world_grid(shape, origin=ORIGIN, voxel=VOXEL):
    """float64 world coordinates of every voxel, (3, dx, dy, dz)."""
    return np.asarray(origin, np.float64)[:, None, None, None] + voxel * np.mgrid[0:shape[0], 0:shape[1], 0:shape[2]].astype(np.float64)


def plane_volume(shape, normal, offset, voxel=VOXEL):
    """tsdf = clip(signed distance to {x : n.x = offset} / (5 voxel), -1, 1): linear wherever the march interpolates."""
    n = np.asarray(normal, np.float64) / np.linalg.norm(normal)
    dist = np.tensordot(n, world_grid(shape, voxel=voxel), axes=1) - offset
    return np.clip(dist / (5 * voxel), -1, 1).astype(np.float32), n


def sphere_volume(shape, center, radius, voxel=VOXEL):
    """Euclidean truncated SDF of a sphere (world centre and radius), truncated at 5 voxel."""
    dist = np.sqrt(((world_grid(shape, voxel=voxel) - np.asarray(center, np.float64)[:, None, None, None]) ** 2).sum(0)) - radius
    return np.clip(dist / (5 * voxel), -1, 1).astype(np.float32)


def random_colors(shape, seed):
    rng = np.random.RandomState(seed)
    rgb = rng.randint(0, 256, size=tuple(shape) + (3,)).astype(np.float32)
    return (rgb[..., 2] * np.float32(65536) + rgb[..., 1] * np.float32(256) + rgb[..., 0]).astype(np.float32)


def look_at(eye, target, down=(0.0, 1.0, 0.0)):
    """camera-to-world pose: camera z toward target, x right, y as close to `down` as it gets."""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(np.asarray(down, np.float64), z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    pose = np.eye(4)
    pose[:3, :3] = np.stack([x, y, z], axis=1)
    pose[:3, 3] = eye
    return pose


def center_of(shape, origin=ORIGIN, voxel=VOXEL):
    return np.asarray(origin, np.float64) + voxel * (np.asarray(shape) - 1) / 2.0


def rays(pose, K=K, h=H, w=W):
    """world ray origin (3,) and directions (h, w, 3) per unit of camera depth, float64 (the float32 views the kernel reads)."""
    v = raycast_oracle.views_of(K, pose)[0].astype(np.float64)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    dc = np.stack([(xx - v[2]) / v[0], (yy - v[3]) / v[1], np.ones_like(xx)], axis=-1)
    return v[13:16], dc @ v[4:13].reshape(3, 3).T


def in_box(points, shape, origin=ORIGIN, voxel=VOXEL):
    g = (points - np.asarray(origin, np.float64)) / voxel
    return np.all((g >= 0) & (g <= np.asarray(shape) - 1), axis=-1)


def render(vol, color, pose, skip=True, K=K, h=H, w=W, voxel=VOXEL, origin=ORIGIN):
    return raycast_oracle.render(vol, color, origin, voxel, 5 * voxel, K, pose, h, w, skip=skip, return_aux=True)


PLANE_SHAPE = (40, 36, 32)
SPHERE_SHAPE = (32, 32, 32)
SPHERE_C = center_of(SPHERE_SHAPE) + np.array([0.011, -0.007, 0.004])
SPHERE_R = 10 * VOXEL


def plane_case():
    c = center_of(PLANE_SHAPE)
    vol, n = plane_volume(PLANE_SHAPE, [0.2, -0.3, -1.0], float(np.dot([0.2, -0.3, -1.0], c) / np.linalg.norm([0.2, -0.3, -1.0])))
    return vol, n, float(np.dot(n, c))


PLANE_POSES = [look_at(center_of(PLANE_SHAPE) + [0.3, 0.2, -2.2], center_of(PLANE_SHAPE)),
               look_at(center_of(PLANE_SHAPE) + [-0.5, -0.1, -1.6], center_of(PLANE_SHAPE) + [0.2, 0.1, 0.0])]
SPHERE_POSES = [look_at(SPHERE_C + [0.2, -0.3, -1.5], SPHERE_C), look_at(SPHERE_C + [-1.4, 0.4, 0.3], SPHERE_C),
                look_at(SPHERE_C + [0.0, 0.0, -0.6], SPHERE_C)]                 # the last one inside the volume


def sphere_hits(pose, center=SPHERE_C, radius=SPHERE_R):
    """analytic camera depth of the nearer sphere hit (nan = miss) and the ray's closest distance to the centre."""
    t, w = rays(pose)
    oc = t - center
    a, b, c = (w * w).sum(-1), 2 * (w * oc).sum(-1), (oc * oc).sum() - radius ** 2
    disc = b * b - 4 * a * c
    with np.errstate(invalid="ignore"):
        z = (-b - np.sqrt(disc)) / (2 * a)
    closest = np.linalg.norm(np.cross(-oc, w), axis=-1) / np.linalg.norm(w, axis=-1)
    return np.where(disc >= 0, z, np.nan), closest


# ---- CPU: the oracle against analytic surfaces ------------------------------------------------------------------------------
@pytest.mark.parametrize("view", range(len(PLANE_POSES)))
def test_plane_depth_is_the_analytic_intersection(view):
    vol, n, offset = plane_case()
    pose = PLANE_POSES[view]
    depth, normals, _, aux = render(vol, np.zeros_like(vol), pose)
    t, w = rays(pose)
    z = (offset - np.dot(n, t)) / (w @ n)
    on_lattice = (z >= aux["z_near"][0]) & (z <= aux["z_last"][0]) & in_box(t + z[..., None] * w, PLANE_SHAPE)
    assert on_lattice.sum() > 0.5 * H * W
    assert np.all(np.abs(depth[0][on_lattice] - z[on_lattice]) <= 1e-5 * z[on_lattice])
    assert np.all(depth[0][~on_lattice & ~in_box(t + z[..., None] * w, PLANE_SHAPE)] == 0)
    assert np.all(np.abs(normals[0][on_lattice] @ n - 1) < 1e-5)                 # toward increasing tsdf


@pytest.mark.parametrize("view", range(len(SPHERE_POSES)))
def test_sphere_hits_depth_and_normals_match_the_analytic_sphere(view):
    """Outside one voxel of the silhouette, hits are the analytic hits.  What trilinear interpolation of a sphere of radius r
    (in voxels) can do bounds the rest, and these bounds are tight for r = 10:
      * the interpolant of the convex distance exceeds it by at most trace(Hessian) / 8 = 1 / (4 r) voxel, so the crossing
        lies up to 1 / (4 r cos i) voxel deeper along the ray (i: incidence angle).  That is <= 0.05 voxel for i <= 60 deg,
        and 0.057 voxel one voxel from the silhouette (cos i = 0.44);
      * the gradient of the interpolant is the cell's finite difference: the true gradient up to half a voxel away on each
        axis, off by (1 - n_a^2) / (2 r) per axis, i.e. up to atan(sqrt(2) / (2 r)) = 4.05 deg, not 2 deg."""
    vol = sphere_volume(SPHERE_SHAPE, SPHERE_C, SPHERE_R)
    pose = SPHERE_POSES[view]
    depth, normals, _ = raycast_oracle.render(vol, np.zeros_like(vol), ORIGIN, VOXEL, 5 * VOXEL, K, pose, H, W)
    depth, normals = depth[0], normals[0]
    z, closest = sphere_hits(pose)
    near_silhouette = np.abs(closest - SPHERE_R) <= VOXEL
    hit = depth > 0
    assert np.array_equal(hit[~near_silhouette], np.isfinite(z)[~near_silhouette])
    both = hit & np.isfinite(z) & ~near_silhouette
    assert both.sum() > 100
    r = SPHERE_R / VOXEL
    cos_i = np.sqrt(1 - (closest[both] / SPHERE_R) ** 2)
    err = np.abs(depth[both] - z[both]) / VOXEL
    assert np.all(err <= np.maximum(0.05, 1 / (4 * r * cos_i)))
    t, w = rays(pose)
    n = t + z[both][:, None] * w[both] - SPHERE_C
    n /= np.linalg.norm(n, axis=1)[:, None]
    angle = np.degrees(np.arccos(np.clip((normals[both] * n).sum(1), -1, 1)))
    assert angle.max() <= np.degrees(np.arctan(np.sqrt(2) / (2 * r)))


@pytest.mark.parametrize("name", ["plane", "sphere"])
def test_empty_space_skip_changes_nothing(name):
    if name == "plane":
        vol, poses = plane_case()[0], PLANE_POSES
    else:
        vol, poses = sphere_volume(SPHERE_SHAPE, SPHERE_C, SPHERE_R), SPHERE_POSES
    color = random_colors(vol.shape, 1)
    with_skip = render(vol, color, np.stack(poses), skip=True)
    without = render(vol, color, np.stack(poses), skip=False)
    for a, b in zip(with_skip[:3], without[:3]):
        assert np.array_equal(a, b)
    assert with_skip[3]["samples"].sum() < 0.8 * without[3]["samples"].sum()   # it does skip


# ---- CPU: range clipping and degenerate volumes -----------------------------------------------------------------------------
def test_camera_inside_the_volume_finds_the_surface():
    vol = sphere_volume(SPHERE_SHAPE, SPHERE_C, SPHERE_R)
    pose = SPHERE_POSES[2]
    assert in_box(pose[:3, 3], SPHERE_SHAPE)
    depth, _, _, aux = render(vol, np.zeros_like(vol), pose)
    assert np.all(aux["z_near"] == 0)
    z, _ = sphere_hits(pose)
    centre = (slice(H // 2 - 4, H // 2 + 4), slice(W // 2 - 4, W // 2 + 4))
    assert np.all(np.abs(depth[0][centre] - z[centre]) <= 0.05 * VOXEL)


def test_camera_looking_away_gets_no_hits():
    vol = sphere_volume(SPHERE_SHAPE, SPHERE_C, SPHERE_R)
    pose = look_at(SPHERE_C + [0.0, 0.0, -1.5], SPHERE_C + [0.0, 0.0, -3.0])
    depth, normals, colors = raycast_oracle.render(vol, random_colors(vol.shape, 2), ORIGIN, VOXEL, 5 * VOXEL, K, pose, H, W)
    assert not depth.any() and not normals.any() and not colors.any()


def test_axis_parallel_rays():
    """Identity rotation, integral cx and cy: the rays of row cy and column cx have d = 0 on an axis.  Inside the slab they
    are admitted (a plane z = const is hit at its exact depth); outside it they are rejected."""
    shape = (30, 28, 26)
    z_plane = float(ORIGIN[2] + 17.3 * VOXEL)
    vol = np.clip((z_plane - world_grid(shape)[2]) / (5 * VOXEL), -1, 1).astype(np.float32)
    Ki = np.array([[40.0, 0, 20.0], [0, 40.0, 15.0], [0, 0, 1]])
    pose = np.eye(4)
    pose[:3, 3] = center_of(shape) + [0.013, -0.021, -1.0]
    depth = raycast_oracle.render(vol, np.zeros_like(vol), ORIGIN, VOXEL, 5 * VOXEL, Ki, pose, 30, 40)[0][0]
    want = np.float32(z_plane - pose[2, 3])
    assert np.all(np.abs(depth[15, :] - want) <= 1e-5 * want) and np.all(np.abs(depth[:, 20] - want) <= 1e-5 * want)
    pose[0, 3] = ORIGIN[0] - 0.2                                                   # column cx now runs beside the box
    depth = raycast_oracle.render(vol, np.zeros_like(vol), ORIGIN, VOXEL, 5 * VOXEL, Ki, pose, 30, 40)[0][0]
    assert not depth[:, 20].any() and depth[:, 33:].all()


@pytest.mark.parametrize("shape", [(1, 8, 9), (8, 1, 9), (8, 9, 1), (1, 1, 1)])
def test_volume_with_a_unit_dimension_gives_no_hits(shape):
    vol = -np.ones(shape, np.float32)
    vol[..., :1] = 1
    depth, normals, colors = raycast_oracle.render(vol, random_colors(shape, 3), ORIGIN, VOXEL, 5 * VOXEL, K,
                                                   look_at(center_of(shape) + [0.1, 0.1, -1.0], center_of(shape)), H, W)
    assert not depth.any() and not normals.any() and not colors.any()


def test_fresh_volume_gives_no_hits():
    vol = np.ones(SPHERE_SHAPE, np.float32)
    depth, normals, colors = raycast_oracle.render(vol, np.zeros_like(vol), ORIGIN, VOXEL, 5 * VOXEL, K, np.stack(SPHERE_POSES), H, W)
    assert not depth.any() and not normals.any() and not colors.any()


# ---- CPU: a scene fused by the integration oracle ---------------------------------------------------------------------------
FUSED_BOUNDS = np.array([[-0.6, 0.6], [-0.6, 0.6], [0.0, 1.0]])
FUSED_VOXEL = 0.02
BALL_C, BALL_R, WALL_Z = np.array([0.0, 0.05, 0.5]), 0.2, 0.85


def fused_poses():
    poses = []
    for i in range(12):
        a = 2 * np.pi * i / 12
        eye = np.array([0.2 * np.cos(a), 0.15 * np.sin(a), -0.35 + 0.03 * np.sin(3 * a)])
        poses.append(look_at(eye, BALL_C + [0.03 * np.sin(a), 0.0, 0.0]))
    return poses


def scene_depth(pose, K, h, w):
    """analytic depth of the ball in front of the wall z = WALL_Z (0 where neither is in front of the camera)."""
    t, dirs = rays(pose, K, h, w)
    oc = t - BALL_C
    a, b, c = (dirs * dirs).sum(-1), 2 * (dirs * oc).sum(-1), (oc * oc).sum() - BALL_R ** 2
    disc = b * b - 4 * a * c
    with np.errstate(invalid="ignore", divide="ignore"):
        ball = np.where(disc >= 0, (-b - np.sqrt(disc)) / (2 * a), np.inf)
        wall = np.where(dirs[..., 2] > 0, (WALL_Z - t[2]) / dirs[..., 2], np.inf)
    z = np.minimum(ball, wall)
    return np.where(np.isfinite(z) & (z > 0), z, 0.0)


def test_fused_scene_renders_the_depth_it_was_fused_from():
    h, w = 48, 64
    Kf = np.array([[55.0, 0, 31.6], [0, 55.0, 23.7], [0, 0, 1]])
    poses = fused_poses()
    orc = tsdf_oracle.TSDFVolume(FUSED_BOUNDS, FUSED_VOXEL)
    truth = [scene_depth(p, Kf, h, w).astype(np.float32) for p in poses]
    rng = np.random.RandomState(4)
    for d, p in zip(truth, poses):
        orc.integrate(rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8), d, Kf, p)
    depth, _, _ = raycast_oracle.render(orc.tsdf, orc.color, orc.vol_origin, FUSED_VOXEL, 5 * FUSED_VOXEL, Kf, np.stack(poses), h, w)
    errs = []
    for got, want in zip(depth, truth):
        pad = np.pad(want, 2, mode="edge")
        window = np.stack([pad[dy:dy + h, dx:dx + w] for dy in range(5) for dx in range(5)])
        smooth = (window.max(0) - window.min(0) <= 3 * FUSED_VOXEL) & (window.min(0) > 0)   # >= 2 px from a discontinuity
        valid = smooth & (got > 0)
        assert valid.sum() > 0.3 * h * w
        errs.append(np.abs(got[valid] - want[valid]))
    errs = np.concatenate(errs) / FUSED_VOXEL
    assert np.median(errs) <= 0.1 and np.percentile(errs, 99) <= 0.5, (np.median(errs), np.percentile(errs, 99))


# ---- GPU: render against the oracle -----------------------------------------------------------------------------------------
def _gpu_volume(tsdf, color, voxel=VOXEL, origin=ORIGIN):
    import torch
    from dvmvs.tsdf import TSDFVolume
    shape = tsdf.shape
    bounds = np.array([[o, o + (d - 0.5) * voxel] for o, d in zip(np.asarray(origin, np.float64), shape)])
    vol = TSDFVolume(bounds, voxel)
    assert tuple(vol._vol_dim) == shape
    t, _, c = vol.get_volume_tensors()
    t.copy_(torch.from_numpy(np.ascontiguousarray(tsdf, dtype=np.float32)))
    c.copy_(torch.from_numpy(np.ascontiguousarray(color, dtype=np.float32)))
    return vol


def _assert_render_equals_oracle(vol, K_, poses, h, w):
    tsdf, color = vol.get_volume()
    want = raycast_oracle.render(tsdf, color, vol._vol_origin, vol._voxel_size, vol._trunc_margin, K_, poses, h, w)
    got = vol.render(K_, poses, h, w)
    if np.asarray(poses).ndim == 2:
        want = tuple(x[0] for x in want)
    for name, g, e in zip(("depth", "normals", "colors"), got, want):
        assert g.dtype == e.dtype and g.shape == e.shape, (name, g.dtype, g.shape, e.dtype, e.shape)
        assert np.array_equal(g, e), "%s differs at %d of %d pixels" % (name, int((g != e).reshape(g.shape[:3] + (-1,)).any(-1).sum()), g.size)
    return got


def smooth_volume(shape, seed):
    """A sum of random plane waves: several surfaces, thin parts, fully truncated regions where it is clipped at 1."""
    rng = np.random.RandomState(seed)
    g = np.mgrid[0:shape[0], 0:shape[1], 0:shape[2]].astype(np.float64)
    f = np.full(shape, 0.3)
    for _ in range(6):
        k = rng.randn(3) * 0.25
        f += rng.uniform(0.3, 0.8) * np.sin(np.tensordot(k, g, axes=1) + rng.uniform(0, 2 * np.pi))
    return np.clip(f, -1, 1).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gpu_random_smooth_volume_equals_oracle(seed):
    shape = (36, 30, 33)
    vol = _gpu_volume(smooth_volume(shape, seed), random_colors(shape, seed))
    c = center_of(shape)
    poses = np.stack([look_at(c + [0.4, -0.3, -1.6], c), look_at(c + [-1.5, 0.2, 0.1], c + [0.1, 0, 0]), look_at(c + [0.05, 0.1, -0.2], c + [0.3, 0.2, 1.0])])
    depth = _assert_render_equals_oracle(vol, K, poses, H, W)[0]
    assert (depth > 0).mean() > 0.2


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["plane", "sphere"])
def test_gpu_analytic_volume_equals_oracle(name):
    if name == "plane":
        tsdf, poses = plane_case()[0], np.stack(PLANE_POSES)
    else:
        tsdf, poses = sphere_volume(SPHERE_SHAPE, SPHERE_C, SPHERE_R), np.stack(SPHERE_POSES)
    depth = _assert_render_equals_oracle(_gpu_volume(tsdf, random_colors(tsdf.shape, 5)), K, poses, H, W)[0]
    assert (depth > 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(37, 23, 50), (2, 2, 2), (2, 9, 3), (70, 5, 33), (17, 64, 2)])
def test_gpu_ragged_volume_equals_oracle(shape):
    rng = np.random.RandomState(sum(shape))
    tsdf = np.where(rng.rand(*shape) < 0.3, 1.0, rng.uniform(-1, 1, size=shape)).astype(np.float32)
    c = center_of(shape)
    poses = np.stack([look_at(c + [0.3, 0.2, -1.2], c), look_at(c + [1.3, -0.2, 0.1], c), look_at(c, c + [0.2, 0.1, 1.0])])
    _assert_render_equals_oracle(_gpu_volume(tsdf, random_colors(shape, 6)), K, poses, 37, 29)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 6, 7), (6, 1, 7), (6, 7, 1), (1, 1, 1)])
def test_gpu_volume_with_a_unit_dimension_gives_no_hits(shape):
    tsdf = -np.ones(shape, np.float32)
    vol = _gpu_volume(tsdf, random_colors(shape, 4))
    depth, normals, colors = _assert_render_equals_oracle(vol, K, look_at(center_of(shape) + [0.1, 0.1, -1.0], center_of(shape)), H, W)
    assert not depth.any() and not normals.any() and not colors.any()


@pytest.mark.gpu
def test_gpu_fresh_volume_gives_no_hits():
    from dvmvs.tsdf import TSDFVolume
    vol = TSDFVolume(np.array([[0.0, 1.0], [0.0, 0.8], [0.0, 0.6]]), 0.05)          # all ones
    depth, normals, colors = vol.render(K, np.stack([look_at([0.5, 0.4, -1.0], [0.5, 0.4, 0.3]), look_at([0.5, 0.4, 0.3], [0.5, 0.4, 1.0])]), H, W)
    assert depth.shape == (2, H, W) and normals.shape == colors.shape == (2, H, W, 3)
    assert not depth.any() and not normals.any() and not colors.any()


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(tsdf_cases.CASES))
def test_gpu_integrated_golden_case_renders_as_the_oracle(case):
    from dvmvs.tsdf import TSDFVolume
    inp = tsdf_cases.inputs(case)
    vol = TSDFVolume(inp["bounds"], inp["voxel"])
    for fr in inp["frames"]:
        vol.integrate(fr["color"], fr["depth"], inp["K"], fr["pose"], obs_weight=fr["weight"])
    h, w = inp["frames"][0]["depth"].shape
    depth = _assert_render_equals_oracle(vol, inp["K"], np.stack([fr["pose"] for fr in inp["frames"]]), h, w)[0]
    assert (depth > 0).any()


def _room():
    from dvmvs.tsdf import TSDFVolume
    rng = np.random.RandomState(11)
    h, w = 256, 320
    Kr = np.array([[250.0, 0, 160.3], [0, 251.0, 127.6], [0, 0, 1]])
    vol = TSDFVolume(np.array([[-4.0, 4.0], [-3.2, 3.2], [0.0, 4.8]]), 0.04)
    poses = []
    for i in range(3):
        yy, xx = np.mgrid[0:h, 0:w]
        depth = (2.0 + 0.8 * np.sin(xx / 40.0 + i) * np.cos(yy / 30.0) + 0.01 * rng.rand(h, w)).astype(np.float32)
        depth[rng.rand(h, w) < 0.05] = 0
        color = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
        pose = np.eye(4)
        pose[:3, 3] = [0.1 * i, -0.05 * i, 0.02 * i]
        c, s = np.cos(0.05 * i), np.sin(0.05 * i)
        pose[:3, :3] = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
        vol.integrate(color, depth, Kr, pose, obs_weight=1.0)
        poses.append(pose)
    return vol, Kr, np.stack(poses), h, w


@pytest.mark.gpu
def test_gpu_production_room_renders_as_the_oracle():
    """The 200 x 160 x 120 room of test_tsdf / test_mesh after three fused frames, rendered at its poses."""
    vol, Kr, poses, h, w = _room()
    depth = _assert_render_equals_oracle(vol, Kr, poses, h, w)[0]
    assert (depth > 0).mean() > 0.5


@pytest.mark.gpu
def test_gpu_call_consistency():
    """One launch of V views equals V one-view launches; CUDA-tensor poses equal numpy poses; two calls are bit-identical."""
    import torch
    vol, Kr, poses, h, w = _room()
    many = vol.render(Kr, poses, h, w)
    for i in range(len(poses)):
        one = vol.render(Kr, poses[i], h, w)
        for a, b in zip(many, one):
            assert np.array_equal(a[i], b)
    dev = vol.render_tensors(Kr, torch.from_numpy(poses).cuda(), h, w)
    assert all(t.is_cuda for t in dev)
    for a, b in zip(many, dev):
        assert np.array_equal(a, b.cpu().numpy())
    for a, b in zip(many, vol.render(Kr, poses, h, w)):
        assert np.array_equal(a, b)
    assert tuple(t.dtype for t in dev) == (torch.float32, torch.float32, torch.uint8)


@pytest.mark.gpu
def test_gpu_render_rejects_malformed_calls():
    import torch
    vol = _gpu_volume(sphere_volume(SPHERE_SHAPE, SPHERE_C, SPHERE_R), np.zeros(SPHERE_SHAPE, np.float32))
    pose = SPHERE_POSES[0]
    for bad in (pose[:3], np.stack([pose[:3, :3]] * 2), np.zeros((0, 4, 4)), pose.reshape(1, 1, 4, 4)):
        with pytest.raises(RuntimeError):
            vol.render(K, bad, H, W)
    for f in (0.0, -60.0, np.nan, np.inf):
        Kb = K.copy()
        Kb[0, 0] = f
        with pytest.raises(RuntimeError):
            vol.render(Kb, pose, H, W)
        Kb = K.copy()
        Kb[1, 1] = f
        with pytest.raises(RuntimeError):
            vol.render(Kb, pose, H, W)
    with pytest.raises(RuntimeError):
        vol.render(K, torch.from_numpy(pose).to("meta"), H, W)
    if torch.cuda.device_count() > 1:
        with pytest.raises(RuntimeError):
            vol.render(K, torch.from_numpy(pose).to("cuda:1"), H, W)
    with pytest.raises(RuntimeError):
        vol.render(K, pose, 0, W)
    assert vol.render(K, torch.from_numpy(pose), H, W)[0].shape == (H, W)       # a CPU tensor is a host array
