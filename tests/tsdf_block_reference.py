"""TEST INFRASTRUCTURE ONLY -- never imported by the product (deep-video-mvs_b200/).  A float64 numpy restatement of the
voxel-block TSDF volume's allocation (csrc/tsdf_sparse.cu, csrc/tsdf_block_hash.cuh), stage by stage, and the ground truth it
must cover: the blocks holding a voxel that the reference's per-voxel rule (oracle/tsdf_oracle.py, TSDFVolume.integrate)
updates.

  needed_blocks   the ground truth, evaluated voxel by voxel over an index box derived here, not from the kernel's box
  candidate_box   sparse_frame + sparse_box_kernel: the frame's candidate blocks
  tile_max        sparse_tile_max_kernel: the largest valid depth of every 16 x 16-pixel tile
  block_seen      sparse_block_seen: the conservative per-block test (a) behind the camera, (b) outside the image, (c) behind
                  every tile's largest depth; with whether a threshold the block reached is too close to call
  block_key, block_hash, check_table
                  the 21-bit key packing, the multiplicative hash and linear probing of the hash table, and its invariants

The device code is compiled with multiply-add contraction and numpy evaluates without it, so a block whose decision lies
within a few ulps (or, far from the origin, within a sixteenth of the test's own slack) of a threshold is reported as
ambiguous instead of decided."""
import numpy as np

BLOCK = 8
TILE = 16
KEY_BITS = 21
KEY_BIAS = 1 << (KEY_BITS - 1)
MAX_CANDIDATES = 1 << 31
EMPTY = -1                       # all 64 bits set, as the volume's int64 key tensor holds it
HASH_MUL = 0x9E3779B97F4A7C15
AMBIGUOUS_REL = 1e-9


# ---------------------------------------------------------------------------------------------------------------- geometry
def camera(K, pose):
    """(fx, fy, cx, cy) as float32 widened and rows 0..2 of inv(pose) in float64, as SparseTSDFVolume.integrate passes them"""
    intr = np.asarray(K).astype(np.float32)
    fx, fy, cx, cy = (np.float64(v) for v in (intr[0, 0], intr[1, 1], intr[0, 2], intr[1, 2]))
    return (fx, fy, cx, cy), np.linalg.inv(np.asarray(pose, dtype=np.float64))


def voxel_world(origin, voxel, g, axis):
    """float64 value of the float32 world coordinate of voxel index g (int64 array) on one axis:
    f32(f64(origin32) + voxel_size * f64(g)), the oracle's and both kernels' rounding"""
    o = np.float64(np.float32(origin[axis]))
    return (o + np.float64(voxel) * np.asarray(g, dtype=np.int64).astype(np.float64)).astype(np.float32).astype(np.float64)


def index_range(origin, voxel, axis, lo, hi):
    """(first, last) voxel index whose world coordinate lies in [lo, hi], searched on the monotone float32 rounding (the
    bracket grows until it holds the answer); first > last when no index does"""
    o = float(np.float32(origin[axis]))

    def least(x, strict):
        e = int(np.floor((x - o) / voxel))
        s = 4
        while True:
            g = np.arange(e - s, e + s + 1, dtype=np.int64)
            w = voxel_world(origin, voxel, g, axis)
            above = w > x if strict else w >= x
            if not above[0] and above[-1]:
                return int(g[np.argmax(above)])
            s *= 4
    return least(lo, False), least(hi, True) - 1


def frustum_aabb(depth, K, pose, trunc, pixel_margin):
    """world AABB of the view frustum up to the frame's largest valid depth + trunc: the camera centre and the rays through the
    image corners `pixel_margin` pixels outside the pixel centres' extent, evaluated with pose (camera -> world).  None
    without a valid depth."""
    d = np.asarray(depth, dtype=np.float64)
    valid = d[d > 0]
    if valid.size == 0:
        return None
    zfar = float(valid.max()) + trunc
    (fx, fy, cx, cy), _ = camera(K, pose)
    h, w = d.shape
    pose = np.asarray(pose, dtype=np.float64)
    pts = [pose[:3, 3]]
    for u in (-pixel_margin, w - 1 + pixel_margin):
        for v in (-pixel_margin, h - 1 + pixel_margin):
            cam = np.array([(u - cx) / fx * zfar, (v - cy) / fy * zfar, zfar])
            pts.append(pose[:3, :3] @ cam + pose[:3, 3])
    pts = np.array(pts)
    return pts.min(0), pts.max(0)


# ------------------------------------------------------------------------------------------------------------ ground truth
def needed_blocks(depth, K, pose, origin, voxel, chunk=1 << 21):
    """The blocks (sorted unique (n,3) int64) holding a voxel that tsdf_oracle.TSDFVolume.integrate updates, step for step in
    its arithmetic: the float32 world point, np.dot(inv(pose), [world 1]) in float64, half-even np.round of the pixel, the
    image bounds and Z > 0, depth > 0 and depth - Z >= -trunc.  Evaluated over every voxel whose world point lies in the
    frustum's world AABB (to the largest depth + trunc, half a pixel outside the image) widened by one block, in chunks."""
    trunc = 5 * float(voxel)
    depth = np.asarray(depth)
    box = frustum_aabb(depth, K, pose, trunc, 0.5)
    if box is None:
        return np.zeros((0, 3), dtype=np.int64)
    lo, hi = box[0] - BLOCK * voxel, box[1] + BLOCK * voxel
    ranges = [index_range(origin, voxel, a, lo[a], hi[a]) for a in range(3)]
    if any(r[0] > r[1] for r in ranges):
        return np.zeros((0, 3), dtype=np.int64)
    gs = [np.arange(r[0], r[1] + 1, dtype=np.int64) for r in ranges]
    ws = [voxel_world(origin, voxel, g, a).astype(np.float32) for a, g in enumerate(gs)]
    (fx, fy, cx, cy), inv = camera(K, pose)
    h, w = depth.shape
    ny, nz = len(gs[1]), len(gs[2])
    per_x = max(1, chunk // (ny * nz))
    found = []
    for x0 in range(0, len(gs[0]), per_x):
        ix, iy, iz = np.meshgrid(np.arange(x0, min(x0 + per_x, len(gs[0]))), np.arange(ny), np.arange(nz), indexing="ij")
        ix, iy, iz = ix.reshape(-1), iy.reshape(-1), iz.reshape(-1)
        xyz_h = np.stack([ws[0][ix], ws[1][iy], ws[2][iz], np.ones(len(ix), dtype=np.float32)], axis=0)
        cam = np.dot(inv, xyz_h).T[:, :3]
        with np.errstate(all="ignore"):
            px = np.round(cam[:, 0] * fx / cam[:, 2] + cx)
            py = np.round(cam[:, 1] * fy / cam[:, 2] + cy)
        pz = cam[:, 2]
        ok = (px >= 0) & (px < w) & (py >= 0) & (py < h) & (pz > 0)
        dv = np.zeros(len(px))
        dv[ok] = depth[py[ok].astype(np.int64), px[ok].astype(np.int64)]
        with np.errstate(invalid="ignore"):
            upd = (dv > 0) & (dv - pz >= -trunc)
        if upd.any():
            g = np.stack([gs[0][ix[upd]], gs[1][iy[upd]], gs[2][iz[upd]]], axis=1)
            found.append(np.unique(np.floor_divide(g, BLOCK), axis=0))
    if not found:
        return np.zeros((0, 3), dtype=np.int64)
    return np.unique(np.concatenate(found), axis=0)


# ---------------------------------------------------------------------------------------------------------- the allocation
class Frame(object):
    """sparse_frame: the frame's parameters, the camera centre by the cofactor inverse and the world rays through the image
    corners 1.5 pixels outside it"""

    def __init__(self, depth, K, pose, origin, voxel):
        self.depth = np.asarray(depth)
        self.im_h, self.im_w = self.depth.shape
        (self.fx, self.fy, self.cx, self.cy), inv = camera(K, pose)
        self.T = inv[:3].reshape(-1).astype(np.float64)
        self.voxel = float(voxel)
        self.trunc = 5 * float(voxel)
        self.origin = np.asarray(origin, dtype=np.float32)
        self.tiles_x, self.tiles_y = -(-self.im_w // TILE), -(-self.im_h // TILE)
        T = self.T
        a, b, c, d, e, g, h, k, l = T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]
        det = a * (e * l - g * k) - b * (d * l - g * h) + c * (d * k - e * h)
        R = np.array([(e * l - g * k) / det, (c * k - b * l) / det, (b * g - c * e) / det,
                      (g * h - d * l) / det, (a * l - c * h) / det, (c * d - a * g) / det,
                      (d * k - e * h) / det, (b * h - a * k) / det, (a * e - b * d) / det])
        self.C = np.array([-(R[3 * r] * T[3] + R[3 * r + 1] * T[7] + R[3 * r + 2] * T[11]) for r in range(3)])
        us, vs = (-1.5, self.im_w + 0.5), (-1.5, self.im_h + 0.5)
        self.dir = np.zeros((4, 3))
        for q in range(4):
            cam = ((us[q & 1] - self.cx) / self.fx, (vs[q >> 1] - self.cy) / self.fy, 1.0)
            for r in range(3):
                self.dir[q, r] = R[3 * r] * cam[0] + R[3 * r + 1] * cam[1] + R[3 * r + 2] * cam[2]


def tile_max(depth):
    """sparse_tile_max_kernel: [tiles_y][tiles_x] float64, the largest depth > 0 of each 16 x 16 tile (NaN never counts), -1
    where there is none"""
    d = np.asarray(depth).astype(np.float64)
    h, w = d.shape
    ty, tx = -(-h // TILE), -(-w // TILE)
    pad = np.full((ty * TILE, tx * TILE), -1.0)
    with np.errstate(invalid="ignore"):
        pad[:h, :w] = np.where(d > 0, d, -1.0)
    return pad.reshape(ty, TILE, tx, TILE).max(axis=(1, 3))


def candidate_box(f, widened=True, slack=0.0):
    """sparse_box_kernel on Frame f: ("empty" | "frustum" | "box", lo (3,) int64 blocks, n (3,) int64).  widened=False is the
    margin before the float32 spacing term (two voxels in index space only).  slack moves every floor's argument outward
    (> 0) or inward (< 0) by slack * (|argument| + 1): the boxes at +-1e-9 bracket what the device's contracted arithmetic
    can give."""
    d = tile_max(f.depth).max()
    if not d > 0:
        return "empty", None, None
    zfar = (d + f.trunc) * (1.0 + 1e-9) + 1e-9
    if not np.isfinite(zfar):
        return "frustum", None, None
    lo3, n3, count = np.zeros(3, np.int64), np.zeros(3, np.int64), 1
    for a in range(3):
        p = f.C[a] + zfar * f.dir[:, a]
        lo, hi = min(f.C[a], p.min()), max(f.C[a], p.max())
        o = np.float64(f.origin[a])
        if widened:
            m = max(abs(lo), abs(hi)) + 2.0 * f.voxel
            spacing = np.ldexp(1.0, int(np.frexp(m)[1]) - 24)             # ldexp(1, ilogb(m) - 23)
        else:
            spacing = 0.0
        ql, qh = (lo - spacing - o) / f.voxel, (hi + spacing - o) / f.voxel
        ql, qh = ql - slack * (abs(ql) + 1), qh + slack * (abs(qh) + 1)
        vlo, vhi = np.floor(ql) - 2.0, np.floor(qh) + 2.0
        blo, bhi = np.floor(vlo / BLOCK), np.floor(vhi / BLOCK)
        if not (blo >= -KEY_BIAS and bhi < KEY_BIAS):
            return "frustum", None, None
        lo3[a], n3[a] = int(blo), int(bhi) - int(blo) + 1
        count *= int(n3[a])
        if count > MAX_CANDIDATES:
            return "frustum", None, None
    return "box", lo3, n3


def box_blocks(lo, n):
    """every block of a candidate box, (count,3) int64 in the allocation kernel's order (x, then y, then z fastest)"""
    g = np.meshgrid(*[np.arange(lo[a], lo[a] + n[a], dtype=np.int64) for a in range(3)], indexing="ij")
    return np.stack([x.reshape(-1) for x in g], axis=1)


def block_seen(f, blocks, tiles=None):
    """sparse_block_seen on Frame f for blocks (n,3): (seen (n,) bool, ambiguous (n,) bool).  A block is ambiguous when a test
    the device reaches for it lies within AMBIGUOUS_REL relative (plus a sixteenth of that test's slack) of its threshold."""
    blocks = np.asarray(blocks, dtype=np.int64).reshape(-1, 3)
    n = len(blocks)
    if tiles is None:
        tiles = tile_max(f.depth)
    T = f.T
    w = [[voxel_world(f.origin, f.voxel, blocks[:, a] * BLOCK + k, a) for k in (0, BLOCK - 1)] for a in range(3)]
    mag = [np.maximum(np.abs(w[a][0]), np.abs(w[a][1])) for a in range(3)]
    eps = [2.0 ** -40 * (abs(T[4 * r]) * mag[0] + abs(T[4 * r + 1]) * mag[1] + abs(T[4 * r + 2]) * mag[2] + abs(T[4 * r + 3]))
           for r in range(3)]
    X, Y, Z = np.zeros((8, n)), np.zeros((8, n)), np.zeros((8, n))
    for c in range(8):
        x, y, z = w[0][c & 1], w[1][(c >> 1) & 1], w[2][c >> 2]
        X[c] = T[0] * x + T[1] * y + T[2] * z + T[3]
        Y[c] = T[4] * x + T[5] * y + T[6] * z + T[7]
        Z[c] = T[8] * x + T[9] * y + T[10] * z + T[11]
    zmin, zmax = Z.min(0), Z.max(0)
    rel = AMBIGUOUS_REL

    def near(value, scale, own_slack):
        return np.abs(value) <= rel * scale + own_slack / 16

    # (a) behind the camera
    behind = zmax + eps[2] <= 0.0
    amb = near(zmax + eps[2], np.abs(zmax) + eps[2], eps[2])
    # (b) in front: the projected pixel rectangle
    front = zmin > 2.0 * eps[2]
    amb |= ~behind & near(zmin - 2.0 * eps[2], np.abs(zmin) + 2.0 * eps[2], eps[2])
    px0, px1 = np.zeros(n, np.int64), np.full(n, f.im_w - 1, np.int64)
    py0, py1 = np.zeros(n, np.int64), np.full(n, f.im_h - 1, np.int64)
    outside = np.zeros(n, bool)
    if front.any():
        with np.errstate(all="ignore"):
            zl = Z - eps[2]
            u = X * f.fx / Z + f.cx
            v = Y * f.fy / Z + f.cy
            su = f.fx * (eps[0] + np.abs(X) * eps[2] / zl) / zl + 1e-9 * (np.abs(u) + abs(f.cx) + 1.0)
            sv = f.fy * (eps[1] + np.abs(Y) * eps[2] / zl) / zl + 1e-9 * (np.abs(v) + abs(f.cy) + 1.0)
            u0, u1 = (u - su).min(0), (u + su).max(0)                    # meaningless (possibly NaN) where not in front
            v0, v1 = (v - sv).min(0), (v + sv).max(0)
        sumax, svmax = su.max(0), sv.max(0)
        for val, s in ((u0, sumax), (u1, sumax), (v0, svmax), (v1, svmax)):
            with np.errstate(invalid="ignore"):
                amb |= ~behind & front & near(val - np.rint(val), np.abs(val) + 1.0, s)
        u0, u1, v0, v1 = np.floor(u0), np.ceil(u1), np.floor(v0), np.ceil(v1)
        out = (u1 < 0.0) | (v1 < 0.0) | (u0 > f.im_w - 1) | (v0 > f.im_h - 1)
        outside = front & out
        sel = front & ~out
        px0[sel] = np.maximum(u0[sel], 0.0)
        px1[sel] = np.minimum(u1[sel], f.im_w - 1)
        py0[sel] = np.maximum(v0[sel], 0.0)
        py1[sel] = np.minimum(v1[sel], f.im_h - 1)
    # (c) the tiles' largest valid depth
    dmax = np.full(n, -1.0)
    reach = ~behind & ~outside
    for i in np.nonzero(reach)[0]:
        dmax[i] = tiles[py0[i] // TILE:py1[i] // TILE + 1, px0[i] // TILE:px1[i] // TILE + 1].max()
    slack_c = 1e-9 * (dmax + np.abs(zmin) + f.trunc)
    lhs, rhs = dmax + f.trunc + slack_c, zmin - eps[2]
    depth_ok = (dmax > 0.0) & (lhs >= rhs)
    amb |= reach & (dmax > 0.0) & near(lhs - rhs, np.abs(dmax) + np.abs(zmin) + f.trunc, slack_c + eps[2])
    return reach & depth_ok, amb


# ------------------------------------------------------------------------------------------------------------- hash table
def block_key(b):
    """tsdf_block_hash.cuh block_key of blocks (n,3) int64: 21 bits per axis, biased by 2^20, x highest; as uint64"""
    b = np.asarray(b, dtype=np.int64).reshape(-1, 3)
    m = (1 << KEY_BITS) - 1
    k = [((b[:, a] + KEY_BIAS) & m).astype(np.uint64) for a in range(3)]
    return (k[0] << np.uint64(2 * KEY_BITS)) | (k[1] << np.uint64(KEY_BITS)) | k[2]


def decode_key(key):
    """block_key's inverse: (n,3) int64"""
    key = np.asarray(key).astype(np.uint64)
    m = np.uint64((1 << KEY_BITS) - 1)
    return np.stack([((key >> np.uint64(2 * KEY_BITS)) & m).astype(np.int64), ((key >> np.uint64(KEY_BITS)) & m).astype(np.int64),
                     (key & m).astype(np.int64)], axis=1) - KEY_BIAS


def block_hash(key, mask):
    """tsdf_block_hash.cuh block_hash: the high half of key * 0x9E3779B97F4A7C15 (mod 2^64), masked"""
    key = np.asarray(key).astype(np.uint64)
    with np.errstate(over="ignore"):
        prod = key * np.uint64(HASH_MUL)
    return ((prod >> np.uint64(32)) & np.uint64(mask)).astype(np.int64)


def check_table(keys, slots, coords, n):
    """The invariants of a hash table holding n blocks: n non-empty keys; their slots a permutation of 0 .. n-1 (empty entries'
    slots -1); every key decodes to coords[slot]; every key found by the probe sequence from its hash with no empty entry
    before it.  keys int64 (EMPTY = -1), slots int32, coords (capacity,3); raises AssertionError naming the first violation."""
    keys, slots, coords = np.asarray(keys, dtype=np.int64), np.asarray(slots, dtype=np.int64), np.asarray(coords, dtype=np.int64)
    size = len(keys)
    assert size & (size - 1) == 0, "table size %d is not a power of two" % size
    full = keys != EMPTY
    assert int(full.sum()) == n, "%d non-empty keys, counters[0] = %d" % (int(full.sum()), n)
    pos = np.nonzero(full)[0]
    s = slots[pos]
    assert np.array_equal(np.sort(s), np.arange(n)), "the keys' slots are not a permutation of 0 .. %d" % (n - 1)
    assert np.all(slots[~full] == -1), "an empty entry has a slot"
    k = keys[pos].astype(np.uint64)
    got = decode_key(k)
    bad = np.nonzero(np.any(got != coords[s], axis=1))[0]
    assert bad.size == 0, "%d keys decode to other coordinates than their slot's, e.g. key %s -> %s, coords[%d] = %s" % (
        bad.size, hex(int(k[bad[0]])), got[bad[0]].tolist(), int(s[bad[0]]), coords[s[bad[0]]].tolist())
    assert len(np.unique(k)) == n, "a key is in the table twice"
    h = block_hash(k, size - 1)
    # empties in the cyclic range [h, pos): none may lie between a key's hash position and its entry
    empties = np.concatenate([[0], np.cumsum(np.tile(~full, 2))])
    end = np.where(pos >= h, pos, pos + size)
    between = empties[end] - empties[h]
    bad = np.nonzero(between)[0]
    assert bad.size == 0, "%d keys sit after an empty entry of their probe sequence, e.g. block %s at %d, hash %d" % (
        bad.size, got[bad[0]].tolist(), int(pos[bad[0]]), int(h[bad[0]]))


def as_set(blocks):
    return set(map(tuple, np.asarray(blocks, dtype=np.int64).reshape(-1, 3).tolist()))
