"""Generate nerf_pl_b200/csrc/mc_table.h, the marching-cubes case table.

Conventions (shared by the table, the kernels in csrc/mesh_kernels.cuh and oracle/mesh_oracle.py):
- corner c of a cell has offsets (c & 1, (c >> 1) & 1, (c >> 2) & 1) along index axes (0, 1, 2);
  bit c of the case index is set when that corner is inside (sigma > threshold);
- edge e runs along axis e // 4; r = e % 4 gives the offsets of the two other axes (in increasing
  axis order) as (r & 1, r >> 1); its lower endpoint is the corner with offset 0 along the axis.

For every case the script traces, on each of the six faces, the segments joining that face's
sign-changing edges.  A face with four sign changes (inside corners on one diagonal) is resolved by
one rule that looks at that face's four corners only: the inside corners stay separated, so each
segment cuts off one inside corner.  Two cells sharing a face therefore draw the same segments there
and the surface has no cracks.  Each segment is oriented so that, with n the outward normal of the
face, n x (q - p) points away from the inside corners; the segments then chain into closed loops
whose fan triangles (v0, vi, vi+1) have normals (right-hand rule, index space) pointing from inside
to outside.

Run: python tools/gen_mc_table.py  (rewrites the header; tests/test_mesh_table.py checks it is current)
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "nerf_pl_b200", "csrc", "mc_table.h")


def corner_pos(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def edge_corners(e):
    """The two corners (lower, upper) of edge e."""
    axis, r = divmod(e, 4)
    others = [a for a in range(3) if a != axis]
    off = [0, 0, 0]
    off[others[0]] = r & 1
    off[others[1]] = r >> 1
    lo = off[0] + 2 * off[1] + 4 * off[2]
    return lo, lo | (1 << axis)


def edge_mid(e):
    a, b = edge_corners(e)
    pa, pb = corner_pos(a), corner_pos(b)
    return tuple((pa[i] + pb[i]) / 2 for i in range(3))


EDGE_OF = {frozenset(edge_corners(e)): e for e in range(12)}


def faces():
    """(outward normal, corners in cyclic order) of the six faces."""
    out = []
    for axis in range(3):
        for side in (0, 1):
            others = [a for a in range(3) if a != axis]
            cyc = []
            for u, v in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = [0, 0, 0]
                p[axis], p[others[0]], p[others[1]] = side, u, v
                cyc.append(p[0] + 2 * p[1] + 4 * p[2])
            n = [0, 0, 0]
            n[axis] = 1 if side else -1
            out.append((tuple(n), cyc))
    return out


FACES = faces()


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _sub(a, b):
    return tuple(x - y for x, y in zip(a, b))


def _dot(a, b):
    return sum(x * y for x, y in zip(a, b))


def face_segments(case, face):
    """Oriented segments (edge p, edge q) of one face under the separation rule."""
    n, cyc = face
    inside = [(case >> c) & 1 for c in cyc]
    # edges of the face in cyclic order: between cyc[i] and cyc[i+1]
    fedges = [EDGE_OF[frozenset((cyc[i], cyc[(i + 1) % 4]))] for i in range(4)]
    crossing = [i for i in range(4) if inside[i] != inside[(i + 1) % 4]]
    if not crossing:
        return []
    if len(crossing) == 2:
        pairs = [(crossing[0], crossing[1])]
    else:
        # ambiguous face: cut off each inside corner (corner i lies between face edges i-1 and i)
        pairs = [((i - 1) % 4, i) for i in range(4) if inside[i]]
    segs = []
    for a, b in pairs:
        ea, eb = fedges[a], fedges[b]
        shared = set(edge_corners(ea)) & set(edge_corners(eb))
        ref = shared.pop() if shared else edge_corners(ea)[0]
        ref_inside = (case >> ref) & 1
        pa, pb = edge_mid(ea), edge_mid(eb)
        side = _dot(_cross(n, _sub(pb, pa)), _sub(corner_pos(ref), pa))
        # n x t must point away from inside corners: an inside reference corner needs side < 0
        if (side < 0) != bool(ref_inside):
            ea, eb = eb, ea
        segs.append((ea, eb))
    return segs


def case_segments(case):
    segs = []
    for f in FACES:
        segs += face_segments(case, f)
    return segs


def case_loops(case):
    nxt = {}
    for p, q in case_segments(case):
        assert p not in nxt, (case, p)
        nxt[p] = q
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start, (case, loop)
        loops.append(loop)
    return loops


def case_triangles(case):
    tris = []
    for loop in case_loops(case):
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


def build_table():
    return [case_triangles(c) for c in range(256)]


def render_header(table) -> str:
    max_tris = max(len(t) for t in table)
    lines = [
        "// Generated by tools/gen_mc_table.py: do not edit.  Marching-cubes case table; conventions in that script.",
        "#ifndef NERFB200_MC_TABLE_H_",
        "#define NERFB200_MC_TABLE_H_",
        "#ifdef __CUDACC__",
        "#define NERFB200_MC_SPACE __constant__",
        "#else",
        "#define NERFB200_MC_SPACE",
        "#endif",
        f"#define NERFB200_MC_MAX_TRIS {max_tris}",
        "// number of triangles of each case",
        "static NERFB200_MC_SPACE const unsigned char nb_mc_tri_count[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("  " + ", ".join(str(len(t)) for t in table[r:r + 32]) + ",")
    lines.append("};")
    lines.append("// edges of each triangle (3 per triangle, -1 past the case's count)")
    lines.append(f"static NERFB200_MC_SPACE const signed char nb_mc_tri_edges[256][{3 * max_tris}] = {{")
    for c, tris in enumerate(table):
        flat = [e for t in tris for e in t] + [-1] * (3 * (max_tris - len(tris)))
        lines.append("  {" + ", ".join(str(e) for e in flat) + "},")
    lines.append("};")
    lines.append("#endif  // NERFB200_MC_TABLE_H_")
    return "\n".join(lines) + "\n"


def main(argv) -> int:
    text = render_header(build_table())
    with open(HEADER, "w") as f:
        f.write(text)
    print(f"wrote {os.path.normpath(HEADER)}")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
