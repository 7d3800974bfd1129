"""TEST INFRASTRUCTURE ONLY -- never imported by the product (deep-video-mvs_b200/).  numpy restatement of the ray casting behind
dvmvs.tsdf.TSDFVolume.render (csrc/raycast.cu): the same float32 operations in the same order, vectorised over rays with one
loop iteration per march step, so the GPU result must equal this one with array_equal.  The contract is stated in the kernel's
header comment; `skip=False` turns the empty-space skip off (tests only: it shows that skipping changes nothing).
"""
import math

import numpy as np

import mesh_oracle

f32 = np.float32


def n_skip_for(voxel_size, trunc_margin):
    """Lattice steps of one empty-space jump, computed in float64 as the C entry point does."""
    n = math.floor((trunc_margin / voxel_size - 0.8660254037844386) / 0.5)
    return int(min(max(n, 1), 1 << 24))


def views_of(cam_intr, cam_poses):
    """(V, 16) float32: fx fy cx cy, R row-major, t -- what TSDFVolume.render_tensors packs."""
    intr = np.asarray(cam_intr).astype(np.float32)
    poses = np.asarray(cam_poses).reshape(-1, 4, 4).astype(np.float32)
    v = np.zeros((len(poses), 16), dtype=np.float32)
    v[:, :4] = [intr[0, 0], intr[1, 1], intr[0, 2], intr[1, 2]]
    v[:, 4:13] = poses[:, :3, :3].reshape(-1, 9)
    v[:, 13:16] = poses[:, :3, 3]
    return v


def _lerp(a, b, f):
    return a + f * (b - a)


class _Volume(object):
    def __init__(self, tsdf, origin, voxel):
        self.tsdf = np.ascontiguousarray(tsdf, dtype=np.float32)
        self.dims = np.array(self.tsdf.shape, dtype=np.int64)
        self.hi = self.dims.astype(np.float32) - f32(1)
        self.origin = np.asarray(origin, dtype=np.float32)
        self.voxel = f32(voxel)

    def point(self, o, d, z):
        """g = o + z d clamped into the box, (R, 3) float32."""
        return np.fmin(np.fmax(o + z[:, None] * d, f32(0)), self.hi)                # fminf / fmaxf

    def cell(self, o, d, z):
        """corners (R, 8) as c[i + 2j + 4k], fractions (R, 3)."""
        g = self.point(o, d, z)
        ci = np.minimum(np.floor(g).astype(np.int64), self.dims - 2)
        f = g - ci.astype(np.float32)
        c = np.stack([self.tsdf[ci[:, 0] + i, ci[:, 1] + j, ci[:, 2] + k] for k in (0, 1) for j in (0, 1) for i in (0, 1)], axis=1)
        return c, f

    def sample(self, o, d, z_near, dz, k):
        c, f = self.cell(o, d, z_near + k.astype(np.float32) * dz)
        x00, x10 = _lerp(c[:, 0], c[:, 1], f[:, 0]), _lerp(c[:, 2], c[:, 3], f[:, 0])
        x01, x11 = _lerp(c[:, 4], c[:, 5], f[:, 0]), _lerp(c[:, 6], c[:, 7], f[:, 0])
        F = _lerp(_lerp(x00, x10, f[:, 1]), _lerp(x01, x11, f[:, 1]), f[:, 2])
        return F, np.all(c == f32(1), axis=1)


def render(tsdf, color_vol, origin, voxel_size, trunc_margin, cam_intr, cam_poses, height, width, skip=True, return_aux=False):
    """depth (V,H,W) float32, normals (V,H,W,3) float32, colors (V,H,W,3) uint8 [, aux] for the (V,4,4) or (4,4) camera-to-world
    poses; aux: per ray `samples` (tsdf evaluations of the march, jump probes included) and `z_near`, `z_last` (first and last
    lattice depth; z_last < z_near where the ray misses the box)."""
    vol = _Volume(tsdf, origin, voxel_size)
    views = views_of(cam_intr, cam_poses)
    V, H, W = len(views), int(height), int(width)
    n_rays = V * H * W
    vv, yy, xx = np.meshgrid(np.arange(V), np.arange(H), np.arange(W), indexing="ij")
    view = views[vv.reshape(-1)]
    u, v = xx.reshape(-1).astype(np.float32), yy.reshape(-1).astype(np.float32)
    with np.errstate(all="ignore"):
        dcx = (u - view[:, 2]) / view[:, 0]
        dcy = (v - view[:, 3]) / view[:, 1]
        R = view[:, 4:13].reshape(-1, 3, 3)
        w = (R[:, :, 0] * dcx[:, None] + R[:, :, 1] * dcy[:, None]) + R[:, :, 2]
        d = w / vol.voxel
        o = (view[:, 13:16] - vol.origin) / vol.voxel
        length = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        dz = f32(0.5) / length
        inside = np.full(n_rays, bool(np.all(vol.dims >= 2)))
        z_near = np.zeros(n_rays, dtype=np.float32)
        z_far = np.full(n_rays, np.inf, dtype=np.float32)
        for a in range(3):
            flat = d[:, a] == 0
            inside &= ~flat | ((o[:, a] >= 0) & (o[:, a] <= vol.hi[a]))
            t0, t1 = (-o[:, a]) / d[:, a], (vol.hi[a] - o[:, a]) / d[:, a]
            z_near = np.where(flat, z_near, np.fmax(z_near, np.fmin(t0, t1)))
            z_far = np.where(flat, z_far, np.fmin(z_far, np.fmax(t0, t1)))
        n_f = np.floor((z_far - z_near) / dz)
    ok = inside & (z_near <= z_far) & (n_f < f32(2 ** 30))
    n = np.where(ok, n_f, -1).astype(np.int64)
    n_skip = n_skip_for(voxel_size, trunc_margin) if skip else None

    z_hit = np.zeros(n_rays, dtype=np.float32)
    hit = np.zeros(n_rays, dtype=bool)
    samples = np.zeros(n_rays, dtype=np.int64)
    act = np.nonzero(ok)[0]
    k = np.zeros(len(act), dtype=np.int64)
    f_prev, ones = vol.sample(o[act], d[act], z_near[act], dz[act], k)
    samples[act] += 1
    while len(act):
        live = k < n[act]
        act, k, f_prev, ones = act[live], k[live], f_prev[live], ones[live]
        if not len(act):
            break
        O, D, ZN, DZ = o[act], d[act], z_near[act], dz[act]
        jumped = np.zeros(len(act), dtype=bool)
        if skip:
            probe = np.nonzero(ones & (k + n_skip <= n[act]))[0]
            if len(probe):
                f_j, ones_j = vol.sample(O[probe], D[probe], ZN[probe], DZ[probe], k[probe] + n_skip)
                samples[act[probe]] += 1
                go = ~(f_j < 0)
                jp = probe[go]
                jumped[jp] = True
                k[jp] += n_skip
                f_prev[jp], ones[jp] = f_j[go], ones_j[go]
        step = np.nonzero(~jumped)[0]
        f_cur, ones_c = vol.sample(O[step], D[step], ZN[step], DZ[step], k[step] + 1)
        samples[act[step]] += 1
        crossing = (f_prev[step] >= 0) & (f_cur < 0)
        cs = step[crossing]
        with np.errstate(all="ignore"):
            fp, fc = f_prev[cs], f_cur[crossing]
            z_prev = ZN[cs] + k[cs].astype(np.float32) * DZ[cs]
            z_hit[act[cs]] = z_prev + (DZ[cs] * fp) / (fp - fc)
        hit[act[cs]] = True
        k[step] += 1
        f_prev[step], ones[step] = f_cur, ones_c
        keep = np.ones(len(act), dtype=bool)
        keep[cs] = False
        act, k, f_prev, ones = act[keep], k[keep], f_prev[keep], ones[keep]

    normals = np.zeros((n_rays, 3), dtype=np.float32)
    colors = np.zeros((n_rays, 3), dtype=np.uint8)
    h = np.nonzero(hit)[0]
    if len(h):
        c, f = vol.cell(o[h], d[h], z_hit[h])
        gx = _lerp(_lerp(c[:, 1] - c[:, 0], c[:, 3] - c[:, 2], f[:, 1]), _lerp(c[:, 5] - c[:, 4], c[:, 7] - c[:, 6], f[:, 1]), f[:, 2])
        gy = _lerp(_lerp(c[:, 2] - c[:, 0], c[:, 3] - c[:, 1], f[:, 0]), _lerp(c[:, 6] - c[:, 4], c[:, 7] - c[:, 5], f[:, 0]), f[:, 2])
        gz = _lerp(_lerp(c[:, 4] - c[:, 0], c[:, 5] - c[:, 1], f[:, 0]), _lerp(c[:, 6] - c[:, 2], c[:, 7] - c[:, 3], f[:, 0]), f[:, 1])
        with np.errstate(all="ignore"):
            glen = np.sqrt((gx * gx + gy * gy) + gz * gz)
            g = np.stack([gx, gy, gz], axis=1)
            normals[h] = np.where(glen[:, None] > 0, g / glen[:, None], f32(0))
        ind = np.rint(vol.point(o[h], d[h], z_hit[h])).astype(np.int64)
        colors[h] = mesh_oracle.colors_at(np.asarray(color_vol, dtype=np.float32), ind)
    out = (z_hit.reshape(V, H, W), normals.reshape(V, H, W, 3), colors.reshape(V, H, W, 3))
    if return_aux:
        with np.errstate(all="ignore"):
            z_last = np.where(ok, z_near + np.maximum(n, 0).astype(np.float32) * dz, -np.inf).astype(np.float32)
        return out + ({"samples": samples.reshape(V, H, W), "z_near": z_near.reshape(V, H, W), "z_last": z_last.reshape(V, H, W)},)
    return out
