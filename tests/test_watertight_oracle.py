"""not gpu: the generated marching-cubes table, the numpy restatement of the watertight remesh (tests/watertight_oracle.py)
and its surface properties on analytic fields."""
import numpy as np

from meshanything_b200 import mc_table
from tests import watertight_oracle as W


def _crossed_edges(case):
    return {e for e, (c0, c1, _) in enumerate(mc_table.EDGES) if ((case >> c0) & 1) != ((case >> c1) & 1)}


def test_committed_header_is_the_generator_output():
    with open(mc_table.HEADER) as f:
        assert f.read() == mc_table.render_header()


def test_every_case_uses_exactly_its_crossed_edges():
    for case, tris in enumerate(mc_table.tables()):
        used = {e for t in tris for e in t}
        assert used == _crossed_edges(case), case
        assert all(len(set(t)) == 3 for t in tris)


def test_case_boundary_is_the_face_rule_and_neighbours_agree():
    """The directed edges used once by a case's triangles are exactly the segments the face rule draws; the rule on a
    face depends on its four corners only, and the cell across the face draws the same segments reversed."""
    for case, tris in enumerate(mc_table.tables()):
        directed = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
        boundary = {d for d in directed if (d[1], d[0]) not in directed}
        assert len(boundary) == len([d for d in directed if (d[1], d[0]) not in directed])
        assert boundary == set(mc_table.face_segments(case)), case
    faces = mc_table.faces()
    for axis in range(3):
        lo_face = next(f for f in faces if f[0] == axis and f[1] == 0)   # face x_axis = 0 of the upper cell
        hi_face = next(f for f in faces if f[0] == axis and f[1] == 1)   # face x_axis = 1 of the lower cell
        lo_edges = {mc_table._edge_of(lo_face[2][i], lo_face[2][(i + 1) % 4]) for i in range(4)}
        hi_edges = {mc_table._edge_of(hi_face[2][i], hi_face[2][(i + 1) % 4]) for i in range(4)}
        to_lo = {}                                                        # physical edge: upper-face edge -> lower
        for e in hi_edges:
            c0, c1, ax = mc_table.EDGES[e]
            to_lo[e] = mc_table._edge_of(c0 & ~(1 << axis), c1 & ~(1 << axis))
        assert set(to_lo.values()) == lo_edges
        for bits in range(16):
            lower = sum(((bits >> q) & 1) << c for q, c in enumerate(hi_face[2]))
            upper = sum(((bits >> q) & 1) << c for q, c in enumerate(lo_face[2]))
            for other in (0, 255 & ~sum(1 << c for c in hi_face[2])):     # the rest of the cube must not matter
                s_low = {(to_lo[p], to_lo[q]) for p, q in mc_table.face_segments(lower | other) if p in hi_edges and q in hi_edges}
                for other_up in (0, 255 & ~sum(1 << c for c in lo_face[2])):
                    s_up = {(p, q) for p, q in mc_table.face_segments(upper | other_up) if p in lo_edges and q in lo_edges}
                    assert s_low == {(q, p) for p, q in s_up}, (axis, bits)


def test_triangle_normals_point_from_inside_to_outside_corners():
    for case, tris in enumerate(mc_table.tables()):
        for t in tris:
            P = [np.array(mc_table.edge_midpoint(e)) for e in t]
            nrm = np.cross(P[1] - P[0], P[2] - P[0])
            toward_out = 0.0
            for e in t:
                c0, c1, _ = mc_table.EDGES[e]
                a, b = np.array(mc_table.corner_offset(c0)), np.array(mc_table.corner_offset(c1))
                toward_out += nrm @ ((b - a) if (case >> c0) & 1 else (a - b))
            assert toward_out > 0, (case, t)
    assert mc_table.tables()[1] and np.cross(*[np.array(mc_table.edge_midpoint(e)) - np.array(mc_table.edge_midpoint(
        mc_table.tables()[1][0][0])) for e in mc_table.tables()[1][0][1:]]) @ np.ones(3) > 0   # away from corner 0


def _closest_dist64(p, a, b, c):
    """Independent float64 point-triangle distance: Ericson's Voronoi-region closest point (Real-Time Collision
    Detection 5.1.5), with degenerate triangles taken as their three segments."""
    def seg(p, a, b):
        ab = b - a
        l = ab @ ab
        t = 0.0 if l == 0 else min(1.0, max(0.0, (p - a) @ ab / l))
        return np.linalg.norm(p - (a + t * ab))
    ab, ac, ap = b - a, c - a, p - a
    if np.linalg.norm(np.cross(ab, ac)) <= 1e-12 * max(1.0, ab @ ab + ac @ ac):
        return min(seg(p, a, b), seg(p, b, c), seg(p, c, a))
    d1, d2 = ab @ ap, ac @ ap
    if d1 <= 0 and d2 <= 0:
        return np.linalg.norm(p - a)
    bp = p - b
    d3, d4 = ab @ bp, ac @ bp
    if d3 >= 0 and d4 <= d3:
        return np.linalg.norm(p - b)
    vc = d1 * d4 - d3 * d2
    if vc <= 0 and d1 >= 0 and d3 <= 0:
        return np.linalg.norm(p - (a + d1 / (d1 - d3) * ab))
    cp = p - c
    d5, d6 = ab @ cp, ac @ cp
    if d6 >= 0 and d5 <= d6:
        return np.linalg.norm(p - c)
    vb = d5 * d2 - d1 * d6
    if vb <= 0 and d2 >= 0 and d6 <= 0:
        return np.linalg.norm(p - (a + d2 / (d2 - d6) * ac))
    va = d3 * d6 - d5 * d4
    if va <= 0 and (d4 - d3) >= 0 and (d5 - d6) >= 0:
        return np.linalg.norm(p - (b + (d4 - d3) / ((d4 - d3) + (d5 - d6)) * (c - b)))
    den = 1.0 / (va + vb + vc)
    return np.linalg.norm(p - (a + ab * vb * den + ac * vc * den))


def test_fp32_distance_matches_float64_closest_point():
    rng = np.random.RandomState(0)
    M = 3000
    tri = rng.uniform(-0.8, 0.8, (M, 3, 3)).astype(np.float32)
    tri[::10, 1] = tri[::10, 0]                                       # repeated vertex: a segment
    tri[1::10, 2] = tri[1::10, 0]
    tri[2::10, 1:] = tri[2::10, :1]                                   # a point
    t = rng.uniform(0, 1, (M // 10, 1)).astype(np.float32)
    tri[3::10, 2] = tri[3::10, 0] + t * (tri[3::10, 1] - tri[3::10, 0])   # collinear: zero area
    p = rng.uniform(-1, 1, (M, 3)).astype(np.float32)
    p[::3] = (tri[::3].mean(1) + 0.02 * rng.randn(len(tri[::3]), 3)).astype(np.float32)   # near the face
    d32 = W.tri_dist((p[:, 0], p[:, 1], p[:, 2]), *[(tri[:, v, 0], tri[:, v, 1], tri[:, v, 2]) for v in range(3)])
    assert d32.dtype == np.float32
    # relative to the coordinates' magnitude (1 here): the fp32 differences of the formula cancel at that scale
    for m in range(M):
        ref = _closest_dist64(p[m].astype(np.float64), *[tri[m, v].astype(np.float64) for v in range(3)])
        assert abs(float(d32[m]) - ref) <= 1e-5 * max(ref, 1.0), (m, float(d32[m]), ref)


def test_udf_grid_is_the_clamped_brute_force_minimum():
    rng = np.random.RandomState(1)
    v = rng.uniform(-0.6, 0.6, (30, 3)).astype(np.float32)
    f = rng.randint(0, 30, (25, 3))
    f[0] = [4, 4, 9]
    n = 16
    band = 3 * 2.0 / n
    fld = W.udf_grid(v, f, n, band)
    g = W.grid_coords(n)
    I, J, K = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
    p = (g[I.ravel()], g[J.ravel()], g[K.ravel()])
    brute = np.full(n ** 3, np.float32(band), np.float32)
    for tri in v[f]:
        d = W.tri_dist(p, *[tuple(np.full(n ** 3, tri[k, a], np.float32) for a in range(3)) for k in range(3)])
        brute = np.minimum(brute, d)
    assert np.array_equal(fld.reshape(-1), brute)


def _sphere_shell(n, R):
    g = W.grid_coords(n).astype(np.float64)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    return np.abs(np.sqrt(X * X + Y * Y + Z * Z) - R).astype(np.float32)


def test_sphere_shell_is_two_closed_outward_spheres():
    n, R = 64, 0.5
    dx = 2.0 / n
    verts, faces = W.marching_cubes(_sphere_shell(n, R), dx)
    assert W.is_watertight(faces)
    comps = W.components(faces, len(verts))
    assert len(comps) == 2 and all(W.euler_characteristic(faces[c]) == 2 for c in comps)
    w = verts.astype(np.float64) * dx - 1.0
    r = np.linalg.norm(w, axis=1)
    assert np.abs(np.abs(r - R) - dx).max() < 0.05 * dx
    cen = w[faces].mean(1)
    rc = np.linalg.norm(cen, axis=1)
    away = np.sign(rc - R)[:, None] * cen / rc[:, None]
    nrm = W.face_normals(w, faces)
    # grid points where the field equals the level exactly (on the axes here) collapse triangles to a point (t = 1 on
    # several edges), as in any marching cubes; every triangle with an area points away from radius R
    real = np.linalg.norm(nrm, axis=1) > 0
    assert real.mean() > 0.9
    assert (np.einsum("ij,ij->i", nrm[real], away[real]) > 0).all()


def test_single_open_triangle_becomes_one_closed_shell():
    n = 32
    tri = np.array([[-0.4, -0.3, 0.1], [0.5, -0.2, -0.1], [0.0, 0.45, 0.2]], np.float32)
    verts, faces = W.marching_cubes(W.udf_grid(tri, [[0, 1, 2]], n), 2.0 / n)
    assert W.is_watertight(faces)
    comps = W.components(faces, len(verts))
    assert len(comps) == 1 and W.euler_characteristic(faces) == 2
