"""TEST INFRASTRUCTURE ONLY -- never imported by the product (deep-video-mvs_b200/).  numpy restatement of the marching cubes
behind dvmvs.tsdf.TSDFVolume.get_mesh (csrc/mesh.cu), the step that replaces scikit-image's marching cubes in the reference's
`get_mesh` (sample-data/run-tsdf-reconstruction.py:344-358).  Same tables (tools/gen_mc_tables.py), same float32 operations
in the same order, so the GPU result must equal this one with array_equal:
  * inside      = tsdf < 0 (NaN never inside); an edge crosses iff exactly one endpoint is inside
  * vertex      = one per crossing grid edge, sorted by key 3 * (C-order linear index of the lower voxel) + axis;
                  index space f32(i) + t along the edge's axis, t = -a / (b - a), a at the lower endpoint
  * world       = f32( f32(v * f32(voxel_size)) + origin )                                         (:351, NumPy-2 rules)
  * normal      = np.gradient (float32) at both endpoints, g_a + t * (g_b - g_a), divided by
                  sqrt((x*x + y*y) + z*z); a zero gradient gives (0, 0, 0)
  * colour      = the reference's lines (:352-357) at np.round(v)
  * faces       = cubes in C order, each case's triangles in table order, as vertex ids (int32)
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import gen_mc_tables as T  # noqa: E402

_TRI = np.zeros((256, T.MAX_TRIS, 3), dtype=np.int64)
_NTRI = np.array([len(t) for t in T.TRIANGLES], dtype=np.int64)
for _c, _tris in enumerate(T.TRIANGLES):
    if _tris:
        _TRI[_c, :len(_tris)] = _tris
_CORNER_OFF = np.array([[c & 1, c >> 1 & 1, c >> 2 & 1] for c in range(8)], dtype=np.int64)
_EDGE_AXIS = np.array([e // 4 for e in range(12)], dtype=np.int64)
_EDGE_LO = np.array([_CORNER_OFF[a] for a, _ in T.EDGES], dtype=np.int64)      # (12, 3) offset of the lower endpoint


def cube_cases(tsdf):
    """(dx-1, dy-1, dz-1) int array of case indices."""
    inside = tsdf < 0
    sx, sy, sz = (d - 1 for d in tsdf.shape)
    case = np.zeros((sx, sy, sz), dtype=np.int64)
    for c, (ox, oy, oz) in enumerate(_CORNER_OFF):
        case |= inside[ox:ox + sx, oy:oy + sy, oz:oz + sz].astype(np.int64) << c
    return case


def colors_at(color_vol, verts_ind):
    """The reference's colour lines (:352-357), verbatim in NumPy-2 semantics (colour_const a Python int)."""
    color_const = 256 * 256
    rgb_vals = color_vol[verts_ind[:, 0], verts_ind[:, 1], verts_ind[:, 2]]
    colors_b = np.floor(rgb_vals / color_const)
    colors_g = np.floor((rgb_vals - colors_b * color_const) / 256)
    colors_r = rgb_vals - colors_b * color_const - colors_g * 256
    colors = np.floor(np.asarray([colors_r, colors_g, colors_b])).T
    return colors.astype(np.uint8)


def marching_cubes(tsdf, color_vol, voxel_size, origin, return_aux=False):
    """verts (V,3) float32 world, faces (F,3) int32, norms (V,3) float32, colors (V,3) uint8 [, aux dict]."""
    tsdf = np.ascontiguousarray(tsdf, dtype=np.float32)
    dims = tsdf.shape
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8))
    if min(dims) < 2:
        aux = {"t": np.zeros(0, np.float32), "keys": np.zeros(0, np.int64), "cases": np.zeros(0, np.int64), "vind": np.zeros((0, 3), np.float32)}
        return empty + (aux,) if return_aux else empty
    inside = tsdf < 0
    keys, lows, axes = [], [], []
    for axis in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[axis], hi[axis] = slice(0, -1), slice(1, None)
        idx = np.stack(np.nonzero(inside[tuple(lo)] != inside[tuple(hi)]), axis=1)
        lows.append(idx)
        axes.append(np.full(len(idx), axis, dtype=np.int64))
        keys.append(3 * np.ravel_multi_index(idx.T, dims).astype(np.int64) + axis)
    keys, lows, axes = np.concatenate(keys), np.concatenate(lows), np.concatenate(axes)
    order = np.argsort(keys, kind="stable")
    keys, lows, axes = keys[order], lows[order], axes[order]
    ups = lows + np.eye(3, dtype=np.int64)[axes]
    a = tsdf[lows[:, 0], lows[:, 1], lows[:, 2]]
    b = tsdf[ups[:, 0], ups[:, 1], ups[:, 2]]
    with np.errstate(all="ignore"):
        t = (-a) / (b - a)                                                           # float32
    vind = lows.astype(np.float32)
    rows = np.arange(len(keys))
    vind[rows, axes] = vind[rows, axes] + t

    verts = vind * np.float32(voxel_size) + np.asarray(origin, dtype=np.float32)     # two float32 roundings

    grads = np.gradient(tsdf)
    ga = np.stack([g[lows[:, 0], lows[:, 1], lows[:, 2]] for g in grads], axis=1)
    gb = np.stack([g[ups[:, 0], ups[:, 1], ups[:, 2]] for g in grads], axis=1)
    with np.errstate(all="ignore"):
        n = ga + t[:, None] * (gb - ga)
        length = np.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2])
        norms = np.where(length[:, None] > 0, n / length[:, None], np.float32(0)).astype(np.float32)

    colors = colors_at(color_vol, np.round(vind).astype(int))

    case = cube_cases(tsdf)
    cubes = np.stack(np.nonzero(_NTRI[case] > 0), axis=1)                           # C order
    cc = case[cubes[:, 0], cubes[:, 1], cubes[:, 2]]
    ntri = _NTRI[cc]
    cube_of = np.repeat(np.arange(len(cubes)), ntri)
    tri_of = np.arange(len(cube_of)) - np.repeat(np.cumsum(ntri) - ntri, ntri)
    edges = _TRI[cc[cube_of], tri_of]                                                # (F, 3) edge ids
    low = cubes[cube_of][:, None, :] + _EDGE_LO[edges]                               # (F, 3, 3)
    fkeys = 3 * np.ravel_multi_index((low[..., 0], low[..., 1], low[..., 2]), dims).astype(np.int64) + _EDGE_AXIS[edges]
    faces = np.searchsorted(keys, fkeys)
    assert np.array_equal(keys[np.minimum(faces, len(keys) - 1)], fkeys), "a face uses an edge without a vertex"
    out = (verts.astype(np.float32), faces.astype(np.int32), norms, colors)
    if return_aux:
        return out + ({"t": t, "keys": keys, "cases": case, "vind": vind},)
    return out
