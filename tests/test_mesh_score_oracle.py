"""not gpu: the numpy restatement of the best-of-N mesh score (tests/mesh_score_oracle.py) against independent float64
geometry, analytic cases, and its edge cases (absent faces, zero area, ties, the frame map)."""
import numpy as np
from scipy.spatial import cKDTree

from meshanything_b200.inputs import normalize_pc_normal
from tests import mesh_score_oracle as M
from tests.test_watertight_oracle import _closest_dist64

F32 = np.float32


def _cloud(P, seed, lo=-0.5, hi=0.5):
    rng = np.random.RandomState(seed)
    n = rng.randn(P, 3)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    return np.concatenate([rng.uniform(lo, hi, (P, 3)), n], axis=1).astype(F32)


def _soup(F, seed):
    rng = np.random.RandomState(seed)
    tri = rng.uniform(-0.5, 0.5, (F, 3, 3)).astype(F32)
    tri[::7, 1] = tri[::7, 0]                                  # repeated vertex: a segment
    tri[3::11] = tri[3::11, :1]                                # a point
    return tri


def _cube():
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)], F32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    return v[np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))])]


def test_point_to_mesh_matches_float64_closest_points():
    tri = _soup(40, 0)
    cloud = _cloud(300, 1, -0.7, 0.7)
    r = M.candidate(tri, cloud)
    t64 = tri.astype(np.float64)
    for i, p in enumerate(cloud[:, :3].astype(np.float64)):
        d = np.array([_closest_dist64(p, *t64[f]) for f in range(len(tri))])
        assert abs(float(r["point_dist"][i]) - d.min()) <= 1e-6, (i, float(r["point_dist"][i]), d.min())
        # the chosen face is a nearest one (up to the fp32 rounding of the two distances)
        assert d[r["point_face"][i]] <= d.min() + 1e-6
    assert abs(r["p2m"] - np.mean([min(_closest_dist64(p, *t) for t in t64)
                                   for p in cloud[:, :3].astype(np.float64)])) <= 1e-6


def test_mesh_to_point_matches_kdtree():
    tri = _soup(50, 2)
    cloud = _cloud(2000, 3)
    r = M.candidate(tri, cloud)
    pts, _ = M.quadrature(tri)
    d, j = cKDTree(cloud[:, :3].astype(np.float64)).query(pts.reshape(-1, 3).astype(np.float64))
    assert np.abs(r["quad_dist"].reshape(-1).astype(np.float64) - d).max() <= 1e-6
    # the chosen point is a nearest one (up to fp32 rounding)
    chosen = np.linalg.norm(cloud[r["quad_point"].reshape(-1), :3].astype(np.float64)
                            - pts.reshape(-1, 3).astype(np.float64), axis=1)
    assert (chosen <= d + 1e-6).all()
    agree = (r["quad_point"].reshape(-1) == j).mean()
    assert agree > 0.99, agree


def test_quadrature_points_are_the_sub_triangle_centroids_inside_the_face():
    tri = _soup(30, 4)
    pts, w = M.quadrature(tri)
    assert pts.shape == (30, 16, 3) and pts.dtype == F32 and w.shape == (30, 16)
    np.testing.assert_allclose(w.sum(1), M.face_area(tri), rtol=1e-15, atol=0)
    t = tri.astype(np.float64)
    ref64 = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
    np.testing.assert_allclose(M.face_area(tri), 0.5 * np.linalg.norm(ref64, axis=1), rtol=1e-12, atol=1e-18)
    s = M.S_SUB
    for f in range(len(tri)):
        a, b, c = t[f]
        grid = lambda i, j: a + (i / s) * (b - a) + (j / s) * (c - a)
        cents = [(grid(i, j) + grid(i + 1, j) + grid(i, j + 1)) / 3 for i in range(s) for j in range(s - i)]
        cents += [(grid(i + 1, j) + grid(i + 1, j + 1) + grid(i, j + 1)) / 3 for i in range(s - 1) for j in range(s - 1 - i)]
        np.testing.assert_allclose(pts[f].astype(np.float64), np.array(cents), atol=1e-7)
    # barycentrics of the 16 points: strictly inside, summing (with the weights) to the area
    assert (M.QUAD_U > 0).all() and (M.QUAD_V > 0).all() and (M.QUAD_U + M.QUAD_V < 1).all()
    assert len({(u, v) for u, v in zip(M.QUAD_U.tolist(), M.QUAD_V.tolist())}) == 16


def test_square_over_a_plane_cloud():
    delta = 0.01
    sq = np.array([[-0.4, -0.4], [0.4, -0.4], [0.4, 0.4], [-0.4, 0.4]])
    v = np.concatenate([sq, np.full((4, 1), delta)], axis=1).astype(F32)
    tri = v[np.array([[0, 1, 2], [0, 2, 3]])]
    rng = np.random.RandomState(5)
    xy = rng.uniform(-0.35, 0.35, (500, 2))
    nz = np.where(rng.rand(500) < 0.5, 1.0, -1.0)
    cloud = np.concatenate([xy, np.zeros((500, 1)), np.zeros((500, 2)), nz[:, None]], axis=1).astype(F32)
    r = M.candidate(tri, cloud)
    assert abs(r["p2m"] - delta) <= 1e-6 * delta
    assert np.all(np.abs(r["point_dist"] - F32(delta)) <= 1e-6 * delta)
    assert r["nc_p"] == 1.0 and r["nc_m"] == 1.0
    assert r["m2p"] >= delta * (1 - 1e-6)


def test_cube_against_points_on_its_surface():
    tri = _cube()
    rng = np.random.RandomState(6)
    axis = rng.randint(0, 3, 1000)
    side = np.where(rng.rand(1000) < 0.5, -0.5, 0.5)
    pts = rng.uniform(-0.5, 0.5, (1000, 3))
    pts[np.arange(1000), axis] = side
    nrm = np.zeros((1000, 3))
    nrm[np.arange(1000), axis] = np.sign(side)
    cloud = np.concatenate([pts, nrm], axis=1).astype(F32)
    r = M.candidate(tri, cloud)
    assert r["p2m"] <= 1e-6 and r["point_dist"].max() <= 1e-6
    assert r["nc_p"] == 1.0 and r["faces"] == 12


def test_absent_faces_are_ignored():
    tri = _soup(20, 7)
    cloud = _cloud(400, 8)
    with_nan = np.full((27, 3, 3), np.nan, F32)
    keep = np.sort(np.random.RandomState(9).choice(27, 20, replace=False))
    with_nan[keep] = tri
    with_nan[keep, 1:] = tri[:, 1:]
    a, b = M.candidate(tri, cloud), M.candidate(with_nan, cloud)
    assert b["faces"] == 20
    for k in ("p2m", "m2p", "nc_p", "nc_m"):
        assert a[k] == b[k], k
    assert np.array_equal(a["point_dist"], b["point_dist"]) and np.array_equal(keep[a["point_face"]], b["point_face"])
    assert np.array_equal(a["quad_dist"], b["quad_dist"][keep]) and np.array_equal(a["quad_point"], b["quad_point"][keep])
    absent = np.setdiff1d(np.arange(27), keep)
    assert np.isinf(b["quad_dist"][absent]).all() and (b["quad_point"][absent] == -1).all()
    # only the first coordinate marks a face absent: NaN elsewhere in a row would be invalid input, not a marker
    assert np.isnan(with_nan[absent, 0, 0]).all()


def test_empty_and_zero_area_candidates_score_inf():
    cloud = _cloud(200, 10)
    empty = np.full((6, 3, 3), np.nan, F32)
    flat = _soup(6, 11)
    flat[:, 2] = flat[:, 0]                                    # every face has a repeated vertex: zero area
    good = _soup(6, 12)
    chamfer, nc, res = M.score(np.stack([empty, flat, good])[None], cloud[None])
    assert np.isinf(chamfer[0, 0]) and np.isinf(chamfer[0, 1]) and np.isfinite(chamfer[0, 2])
    assert nc[0, 0] == 0.0 and nc[0, 1] == 0.0 and nc[0, 2] > 0
    assert res[0][0]["faces"] == 0 and (res[0][0]["point_face"] == -1).all()
    assert res[0][1]["faces"] == 6 and np.isfinite(res[0][1]["p2m"]) and np.isinf(res[0][1]["m2p"])
    assert M.select(chamfer)[0] == 2
    assert M.select(np.full((2, 4), np.inf)).tolist() == [0, 0]


def test_ties_pick_the_lowest_index():
    tri = _soup(10, 13)
    cloud = _cloud(300, 14)
    dup = np.concatenate([tri[:4], tri[2:3], tri[4:]])          # face 4 repeats face 2
    r = M.candidate(dup, cloud)
    assert (r["point_face"] != 4).all() and (r["point_face"] == 2).any()
    c2 = np.concatenate([cloud, cloud[::-1]])                   # every cloud point twice
    r2 = M.candidate(tri, c2)
    assert (r2["quad_point"] < len(cloud)).all()
    chamfer, _, _ = M.score(np.stack([tri, tri[::-1], tri])[None], cloud[None])
    assert chamfer[0, 0] == chamfer[0, 2]
    best = chamfer[0].min()
    assert M.select(chamfer)[0] == int(np.nonzero(chamfer[0] == best)[0][0])
    assert M.select(np.array([3.0, 1.0, 1.0, 2.0])) == 1


def test_frame_map_of_a_dataset_cloud():
    rng = np.random.RandomState(15)
    raw = np.concatenate([rng.uniform(-3, 7, (4096, 3)) * np.array([1.0, 0.3, 2.0]), rng.randn(4096, 3)], axis=1)
    raw[:, 3:] /= np.linalg.norm(raw[:, 3:], axis=1, keepdims=True)
    pc = normalize_pc_normal(raw)                               # what main.py's Dataset hands the model (fp16)
    m = M.frame_map(pc)
    assert m.dtype == F32
    xyz = m[:, :3].astype(np.float64)
    lo, hi = xyz.min(0), xyz.max(0)
    assert abs((hi - lo).max() - 1.0) <= 1e-6
    assert np.abs(lo + hi).max() <= 1e-6
    assert np.array_equal(m[:, 3:], pc[:, 3:].astype(F32))
    one = M.frame_map(np.array([[0.25, -0.5, 0.125, 0, 0, 1]], np.float16))
    assert np.array_equal(one, np.array([[0, 0, 0, 0, 0, 1]], F32))
