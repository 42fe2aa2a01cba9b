"""Marching-cubes triangle table of csrc/watertight.cu, generated from one face rule instead of typed in.

    python -m meshanything_b200.mc_table          # rewrites meshanything_b200/csrc/mc_table.h

Cube conventions (shared by the kernel, the header and the numpy oracle):
  * corner c sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) from the cell's lower corner (x = i, y = j, z = k);
  * edge e = 4 * axis + m joins corner c0 (bit `axis` clear, the two other bits = m, lower axis first) and
    c1 = c0 | (1 << axis); edges 0, 4 and 8 leave corner 0 and are the three a cell owns;
  * bit c of the case index is set when corner c is inside (field < level).

Rule: on each of the 6 cube faces the crossed edges are joined by segments.  Two crossed edges make one segment.  Four
crossed edges (an ambiguous face: the two inside corners are diagonal) make two segments, each cutting off one inside
corner, so the inside corners are separated.  The rule reads only the face's four corners, so the two cells that share
a face draw the same segments and the surface has no cracks.  Every segment is directed so that, seen from outside the
cube, the inside corners of the face lie on its left; the directed segments then chain into closed loops (every crossed
edge starts one segment and ends one), and each loop is fan-triangulated from its first vertex (in loop order from the
lowest edge) whose chords all cross the cube's interior, so no chord lies on a cube face that the neighbour cell could
also draw.  With that direction the
right-hand normal of every triangle points from the inside corners to the outside ones, i.e. toward increasing field.

This is not Lewiner's topology (skimage.measure.marching_cubes): at ambiguous faces and cube saddles the connectivity can
differ, the surface itself stays closed and consistently oriented.
"""
from __future__ import annotations

import os

HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "mc_table.h")


def corner_offset(c: int):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def edges():
    """[(c0, c1, axis)] for the 12 cube edges, in edge-index order."""
    out = []
    for axis in range(3):
        others = [a for a in range(3) if a != axis]
        for m in range(4):
            c0 = ((m & 1) << others[0]) | (((m >> 1) & 1) << others[1])
            out.append((c0, c0 | (1 << axis), axis))
    return out


EDGES = edges()


def edge_midpoint(e: int):
    c0, _, axis = EDGES[e]
    p = list(corner_offset(c0))
    p[axis] += 0.5
    return p


def _edge_of(ca: int, cb: int) -> int:
    for e, (c0, c1, _) in enumerate(EDGES):
        if {c0, c1} == {ca, cb}:
            return e
    raise ValueError((ca, cb))


def faces():
    """[(axis, side, [4 corners in cyclic order])] for the 6 cube faces."""
    out = []
    for axis in range(3):
        b, c = [a for a in range(3) if a != axis]
        for side in (0, 1):
            cyc = [(0, 0), (1, 0), (1, 1), (0, 1)]
            out.append((axis, side, [(side << axis) | (u << b) | (v << c) for u, v in cyc]))
    return out


_FACE_EDGES = [{_edge_of(cyc[i], cyc[(i + 1) % 4]) for i in range(4)} for _, _, cyc in faces()]


def _sub(p, q):
    return [p[0] - q[0], p[1] - q[1], p[2] - q[2]]


def _cross(u, v):
    return [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]


def _dot(u, v):
    return u[0] * v[0] + u[1] * v[1] + u[2] * v[2]


def face_segments(case: int):
    """Directed segments [(edge_from, edge_to)] that the face rule draws for `case`, face by face."""
    segs = []
    for axis, side, cyc in faces():
        inside = [(case >> q) & 1 for q in cyc]
        fedges = [_edge_of(cyc[i], cyc[(i + 1) % 4]) for i in range(4)]   # fedges[i] joins cyc[i] and cyc[i+1]
        crossed = [i for i in range(4) if inside[i] != inside[(i + 1) % 4]]
        if not crossed:
            continue
        if len(crossed) == 2:
            pairs = [(fedges[crossed[0]], fedges[crossed[1]], [cyc[i] for i in range(4) if inside[i]])]
        else:                       # ambiguous face: cut off each inside corner on its own
            pairs = [(fedges[(i - 1) % 4], fedges[i], [cyc[i]]) for i in range(4) if inside[i]]
        normal = [0.0, 0.0, 0.0]
        normal[axis] = 1.0 if side else -1.0
        for p, q, ins in pairs:
            cen = [sum(corner_offset(c)[d] for c in ins) / len(ins) for d in range(3)]
            P, Q = edge_midpoint(p), edge_midpoint(q)
            s = _dot(_cross(_sub(Q, P), _sub(cen, P)), normal)
            assert s != 0.0
            segs.append((p, q) if s < 0 else (q, p))   # inside corners on the left, seen from outside the cube
    return segs


def case_triangles(case: int):
    """Oriented triangles [(e0, e1, e2)] of one case: segment loops, each fan-triangulated from its first edge."""
    nxt = {}
    for p, q in face_segments(case):
        assert p not in nxt
        nxt[p] = q
    assert sorted(nxt) == sorted(nxt.values())
    tris, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start and len(loop) >= 3
        k = len(loop)
        # fan apex: the first loop vertex whose chords all cross the cube's interior.  A chord between two edges of
        # one cube face would be drawn by the neighbour across that face as well, and four triangles would share it.
        s = next(s for s in range(k) if not any(_share_face(loop[s], loop[(s + i) % k]) for i in range(2, k - 1)))
        loop = loop[s:] + loop[:s]
        tris += [(loop[0], loop[i], loop[i + 1]) for i in range(1, k - 1)]
    return tris


def _share_face(ea: int, eb: int) -> bool:
    return any(ea in fe and eb in fe for fe in _FACE_EDGES)


def tables():
    """[256] lists of oriented edge triangles."""
    return [case_triangles(c) for c in range(256)]


def render_header() -> str:
    tab = tables()
    mx = max(len(t) for t in tab)
    lines = [
        "// mc_table.h -- GENERATED by `python -m meshanything_b200.mc_table`; do not edit.",
        "// Marching-cubes triangles per corner case (conventions in meshanything_b200/mc_table.py): kMcTriCount[case]",
        "// triangles, kMcTris[case][3 t + v] = cube edge of vertex v of triangle t.",
        "#pragma once",
        "",
        f"#define MA_MC_MAX_TRIS {mx}",
        "",
        "static __constant__ unsigned char kMcTriCount[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(t)) for t in tab[r:r + 32]) + ",")
    lines += ["};", "", f"static __constant__ signed char kMcTris[256][{3 * mx}] = {{"]
    for c, t in enumerate(tab):
        flat = [e for tri in t for e in tri] + [-1] * (3 * (mx - len(t)))
        lines.append("    {" + ", ".join(str(x) for x in flat) + f"}},  // {c}")
    lines += ["};", ""]
    return "\n".join(lines)


if __name__ == "__main__":
    with open(HEADER, "w") as f:
        f.write(render_header())
    print(HEADER)
