"""Generates deep-video-mvs_b200/csrc/mc_tables.cuh, the marching-cubes triangulation table of csrc/mesh.cu.  The numpy oracle
(oracle/mesh_oracle.py) imports the same tables, and tests/test_mesh.py checks that the committed header equals render().

    python tools/gen_mc_tables.py            # rewrites the header

Conventions (shared by the kernel and the oracle):
  corner c of the cube at voxel (x, y, z) is voxel (x + (c & 1), y + (c >> 1 & 1), z + (c >> 2 & 1)); case = sum of 1 << c over
  the INSIDE corners (tsdf < 0; NaN is never inside).
  edge e runs along axis a = e // 4 from corner EDGES[e][0] (its lower-index endpoint) to EDGES[e][1]; j = e % 4 gives the
  offsets along the other two axes in increasing axis order (bit 0 the first, bit 1 the second).

For each case the contour segments are traced on the six faces.  On a face, every maximal run of consecutive inside corners
(walking counter-clockwise as seen from outside the cube) gets one segment, from the crossing edge where the walk enters the
run to the one where it leaves: the inside corners lie to the right of the segment, and a face whose diagonal corners share
a sign keeps its two inside corners apart.  Neighbouring cubes trace the same segments on their common face, in opposite
directions, so the surface is closed wherever it does not reach the volume border.  Each crossing edge starts one segment
and ends one, so the segments chain into closed loops, ordered by their smallest edge id.  Each loop of n edges is fanned into
n - 2 triangles (v0, v_i, v_i+1), counter-clockwise as seen from the outside (increasing tsdf); v0 is the first edge, in loop
order from the smallest id, whose diagonals join no two edges of a common face (fan_apex).  So every mesh edge belongs to
exactly two triangles of opposite direction where the surface is closed."""
import os

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(REPO, "deep-video-mvs_b200", "csrc", "mc_tables.cuh")


def _edges():
    edges = []
    for axis in range(3):
        others = [a for a in range(3) if a != axis]
        for j in range(4):
            lo = ((j & 1) << others[0]) | ((j >> 1 & 1) << others[1])
            edges.append((lo, lo | (1 << axis)))
    return edges


EDGES = _edges()


def _edge_id(c0, c1):
    pair = (min(c0, c1), max(c0, c1))
    return EDGES.index(pair)


def _faces():
    """The six faces as corner cycles, counter-clockwise as seen from outside the cube."""
    faces = []
    for axis in range(3):
        u, v = [a for a in range(3) if a != axis]
        for side in (0, 1):
            base = side << axis
            cyc = [base, base | (1 << u), base | (1 << u) | (1 << v), base | (1 << v)]
            right_handed = (u, v, axis) in ((0, 1, 2), (1, 2, 0), (2, 0, 1))          # then cyc turns counter-clockwise about +axis
            ccw_about_plus = cyc if right_handed else cyc[::-1]
            faces.append(ccw_about_plus if side == 1 else ccw_about_plus[::-1])    # outward normal is +axis on side 1
    return faces


FACES = _faces()


def segments(case):
    """Directed contour segments (edge_from, edge_to) on the faces of the cube for one case."""
    segs = []
    for cyc in FACES:
        inside = [(case >> c) & 1 for c in cyc]
        if all(inside) or not any(inside):
            continue
        for k in range(4):
            if inside[k] and not inside[k - 1]:                      # a run of inside corners starts at k
                m = k
                while inside[(m + 1) % 4]:
                    m = (m + 1) % 4
                segs.append((_edge_id(cyc[k - 1], cyc[k]), _edge_id(cyc[m], cyc[(m + 1) % 4])))
    return segs


def crossing_edges(case):
    return [e for e, (a, b) in enumerate(EDGES) if ((case >> a) & 1) != ((case >> b) & 1)]


def loops(case):
    nxt = {}
    for a, b in segments(case):
        assert a not in nxt, (case, a)
        nxt[a] = b
    assert sorted(nxt) == crossing_edges(case) and sorted(nxt.values()) == crossing_edges(case), case
    out, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start, case
        out.append(loop)
    return out


def share_face(e1, e2):
    corners = set(EDGES[e1]) | set(EDGES[e2])
    return any(len({(c >> a) & 1 for c in corners}) == 1 for a in range(3))


def fan_apex(loop):
    """First position of the loop whose fan diagonals join no two edges of a common cube face.  Such a pair of edges is
    shared with the neighbouring cube across that face, which could join the same two vertices too: the mesh edge would then
    belong to four triangles.  A diagonal between edges with no common face exists in this cube only."""
    n = len(loop)
    for k in range(n):
        if all(not share_face(loop[k], loop[(k + i) % n]) for i in range(2, n - 1)):
            return k
    raise AssertionError(loop)


def triangles(case):
    tris = []
    for loop in loops(case):
        k = fan_apex(loop)
        loop = loop[k:] + loop[:k]
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


TRIANGLES = [triangles(c) for c in range(256)]
MAX_TRIS = max(len(t) for t in TRIANGLES)
assert MAX_TRIS == 5, MAX_TRIS        # the kernel sizes its per-cube work (and the count limits) from this


def render():
    lines = [
        "// GENERATED by tools/gen_mc_tables.py -- do not edit.  Marching-cubes tables of csrc/mesh.cu (conventions in the generator).",
        "#pragma once",
        "",
        "namespace dvmvs {",
        "",
        "constexpr int kMcMaxTris = %d;   // most triangles any case emits" % MAX_TRIS,
        "",
        "// edge e: lower-index corner, upper corner (corner c = voxel offset (c & 1, c >> 1 & 1, c >> 2 & 1)); axis = e / 4",
        "__constant__ unsigned char kMcEdgeCorner[12][2] = {%s};" % ", ".join("{%d, %d}" % e for e in EDGES),
        "",
        "// number of triangles per case",
        "__constant__ unsigned char kMcNumTris[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(TRIANGLES[c])) for c in range(r, r + 32)) + ",")
    lines += ["};", "", "// triangles per case: three edge ids each, in emission order (unused slots 0)",
              "__constant__ unsigned char kMcTris[256][kMcMaxTris * 3] = {"]
    for c in range(256):
        flat = [e for t in TRIANGLES[c] for e in t]
        flat += [0] * (MAX_TRIS * 3 - len(flat))
        lines.append("    {" + ", ".join(str(e) for e in flat) + "},")
    lines += ["};", "", "}  // namespace dvmvs", ""]
    return "\n".join(lines)


if __name__ == "__main__":
    with open(HEADER, "w") as fh:
        fh.write(render())
    print("wrote", HEADER, "max triangles per cube:", MAX_TRIS)
