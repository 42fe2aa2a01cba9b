"""not gpu: the numpy restatement of the normal estimator (tests/normals_oracle.py) against scipy / LAPACK and analytic
clouds, its accuracy on the wand, and the bare-cloud readers of `--input_type pc`.  The GPU equals this oracle bit for
bit (tests/test_gpu_normals.py), so these bounds hold for the GPU too."""
import os

import numpy as np
import pytest

from tests import normals_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _sphere(n, seed, centre=(0.0, 0.0, 0.0), r=1.0):
    x = np.random.default_rng(seed).normal(size=(n, 3))
    return x / np.linalg.norm(x, axis=1, keepdims=True) * r + np.asarray(centre)


def _torus(n, seed, R=1.0, r=0.35):
    a, b = np.random.default_rng(seed).uniform(0, 2 * np.pi, (2, n))
    ring = np.stack([np.cos(a), np.sin(a), np.zeros(n)], axis=1)
    return ring * R + r * (np.cos(b)[:, None] * ring + np.sin(b)[:, None] * np.array([0.0, 0.0, 1.0])), ring * R


def _cube_surface(n, seed):
    rng = np.random.default_rng(seed)
    ax, sg = rng.integers(0, 3, n), rng.choice([-1.0, 1.0], n)
    p = rng.uniform(-1, 1, (n, 3))
    p[np.arange(n), ax] = sg
    nrm = np.zeros((n, 3))
    nrm[np.arange(n), ax] = sg
    return p, nrm


def _wand_samples(n, seed=0):
    from mesh_to_pc import SimpleMesh
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    mesh = SimpleMesh(z["vertices"], z["faces"])
    np.random.seed(seed)
    pts, idx = mesh.sample(n, return_index=True)
    return pts, mesh.face_normals[idx]


def _cov6(x):
    d = x - x.mean(axis=0)
    return np.array([d[:, a] @ d[:, b] for a, b in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))])


# ---------------------------------------------------------------- kNN


@pytest.mark.parametrize("k", [1, 8, 16, 64])
def test_knn_matches_a_kd_tree_away_from_ties(k):
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(k)
    p = O.frame_map(np.concatenate([_sphere(3000, k), rng.uniform(-1, 1, (1500, 3))]).astype(F32))
    nbr = O.knn(p, k)
    dist, ref = cKDTree(p.astype(np.float64)).query(p.astype(np.float64), k + 2)
    checked = 0
    for i in range(len(p)):
        d = dist[i][ref[i] != i]
        r = ref[i][ref[i] != i]
        if abs(d[k] - d[k - 1]) <= 1e-6 * d[k]:       # a tie at the boundary of the set: either choice is right
            continue
        assert set(nbr[i].tolist()) == set(r[:k].tolist()), i
        checked += 1
    assert checked > 0.99 * len(p)
    assert (np.diff(O._d2(p[:, None, :], p[nbr]), axis=1) >= 0).all()          # rank order


def test_fast_knn_equals_the_brute_force_definition_with_duplicates_and_clusters():
    rng = np.random.default_rng(7)
    p = rng.uniform(-1, 1, (6000, 3))
    p[100:400] = p[99]                                         # 301 identical points
    p[1000:3000] = p[1000] + rng.normal(scale=1e-4, size=(2000, 3))   # a dense cluster
    p = O.frame_map(p.astype(F32))
    for k in (1, 16, 64):
        assert np.array_equal(O.knn(p, k), O.knn_bruteforce(p, k)), k
    dup = O.knn_bruteforce(p, 8)[150]
    assert all(99 <= j < 400 for j in dup) and 150 not in dup and list(dup) == sorted(dup)   # ties: lowest index first


# ---------------------------------------------------------------- Jacobi


def _eigh_angle(cov):
    d, V = O.jacobi(cov[None])
    u = O.smallest_vector(d, V)[0].astype(np.float64)
    A = np.array([[cov[0], cov[1], cov[2]], [cov[1], cov[3], cov[4]], [cov[2], cov[4], cov[5]]])
    w, E = np.linalg.eigh(A)
    v = V[0, :, int(np.argmin(d[0]))]
    v = v / np.linalg.norm(v)
    return float(np.arcsin(min(1.0, np.linalg.norm(np.cross(v, E[:, 0]))))), w, u


def test_jacobi_matches_lapack_on_separated_spectra():
    rng = np.random.default_rng(0)
    worst = 0.0
    for t in range(2000):
        R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        x = (rng.normal(size=(17, 3)) * rng.uniform(0.01, 1.0, 3)) @ R.T
        ang, w, u = _eigh_angle(_cov6(x))
        if (w[1] - w[0]) > 1e-3 * w[2]:
            worst = max(worst, ang)
        assert abs(np.linalg.norm(u.astype(np.float64)) - 1) < 1e-6
    assert worst < 1e-9, worst


def test_jacobi_degenerate_covariances():
    rng = np.random.default_rng(1)
    same = np.repeat(rng.normal(size=(1, 3)), 17, axis=0)                      # rank 0: all points identical
    d, V = O.jacobi(_cov6(same)[None])
    assert np.array_equal(O.smallest_vector(d, V)[0], np.array([1, 0, 0], F32))   # documented: (1, 0, 0)
    line = np.outer(rng.normal(size=17), [1.0, 2.0, -0.5])                        # rank 1: a line
    plane = rng.normal(size=(17, 2)) @ np.array([[1.0, 0.0, 1.0], [0.0, 1.0, 1.0]])  # rank 2: a plane
    dupl = np.concatenate([rng.normal(size=(9, 3)) * [1, 1, 0.05]] * 2)        # duplicated points
    for x in (line, plane, dupl):
        ang, w, u = _eigh_angle(_cov6(x))
        assert abs(np.linalg.norm(u.astype(np.float64)) - 1) < 1e-6
        if w[1] - w[0] > 1e-6 * max(w[2], 1e-30):
            assert ang < 1e-9, ang
    _, _, u = _eigh_angle(_cov6(plane))
    assert abs(abs(float(u @ np.array([1.0, 1.0, -1.0]) / np.sqrt(3))) - 1) < 1e-6  # the plane's normal
    line_u = _eigh_angle(_cov6(line))[2].astype(np.float64)
    assert abs(line_u @ np.array([1.0, 2.0, -0.5])) < 1e-6                     # some direction across the line


# ---------------------------------------------------------------- forest


def test_kruskal_forest_has_the_minimum_total_weight():
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import minimum_spanning_tree
    p = O.frame_map(np.concatenate([_sphere(1500, 3), _sphere(700, 4, centre=(4.0, 0, 0))]).astype(F32))
    nbr = O.knn(p, 8)
    u = O.smallest_vector(*O.jacobi(O.pca(p, nbr)))
    ab, w = O.edges(nbr, u)
    keep = O.kruskal(len(p), ab, w)
    # scipy drops explicit zeros, and w = 0 is common: shift every weight by 1 (the forest does not change)
    g = coo_matrix((w.astype(np.float64) + 1.0, (ab[:, 0], ab[:, 1])), shape=(len(p), len(p)))
    ref = minimum_spanning_tree(g)
    assert keep.sum() == ref.nnz == len(p) - 2                                 # two components
    assert abs((w[keep].astype(np.float64) + 1.0).sum() - ref.sum()) < 1e-9 * ref.sum()


# ---------------------------------------------------------------- orientation on analytic clouds


def _oriented(points, k=16):
    p = O.frame_map(np.asarray(points).astype(F32))
    n, nbr, u = O.estimate_normals(p, k)
    assert np.all(np.abs(np.linalg.norm(n.astype(np.float64), axis=1) - 1) < 1e-6)
    return p, n


def test_sphere_normals_point_outward():
    p, n = _oriented(_sphere(4000, 0, centre=(0.3, -0.2, 5.0), r=2.0))
    assert (np.sum(n * p, axis=1) > 0).all()


def test_torus_normals_point_out_of_the_tube():
    pts, ring = _torus(6000, 1)
    p, n = _oriented(pts)
    ring_f = O.frame_map(np.concatenate([pts, ring]).astype(F32))[len(pts):]   # the tube's centre line, same frame
    assert (np.sum(n * (p - ring_f), axis=1) > 0).all()


def test_two_separate_spheres_are_two_components_both_outward():
    a, b = _sphere(2500, 2), _sphere(1500, 3, centre=(5.0, 1.0, 0.0), r=0.7)
    p, n = _oriented(np.concatenate([a, b]))
    nbr = O.knn(p, 16)
    *_, ncomp = O.orient(p, O.smallest_vector(*O.jacobi(O.pca(p, nbr))), nbr, return_forest=True)
    assert ncomp == 2
    ca = p[:2500].mean(axis=0)
    cb = p[2500:].mean(axis=0)
    assert (np.sum(n[:2500] * (p[:2500] - ca), axis=1) > 0).all()
    assert (np.sum(n[2500:] * (p[2500:] - cb), axis=1) > 0).all()


def test_cube_surface_sharp_edges():
    """The known weak spot of MST propagation: normals turn by 90 degrees across an edge.  The oracle measures 1 point
    in 6000 flipped (next to an edge); the bound leaves a margin of 5x."""
    pts, truth = _cube_surface(6000, 4)
    p, n = _oriented(pts)
    assert (np.sum(n * truth, axis=1) > 0).mean() >= 1 - 5 / 6000


def test_planar_patch_has_one_sign():
    rng = np.random.default_rng(5)
    pts = np.concatenate([rng.uniform(-1, 1, (3000, 2)), np.zeros((3000, 1))], axis=1) @ np.array(
        [[1.0, 0.0, 0.2], [0.0, 1.0, -0.3], [0.0, 0.0, 1.0]])
    p, n = _oriented(pts)
    plane_n = np.cross([1.0, 0.0, 0.2], [0.0, 1.0, -0.3])
    s = np.sum(n * plane_n, axis=1)
    assert (s > 0.999).all() or (s < -0.999).all()


# ---------------------------------------------------------------- accuracy on the wand


def test_wand_accuracy_at_100k_points():
    """Unoriented normals against the sampled faces' normals, 100k seeded samples, k = 16.  The oracle measures a median
    of 2.56 degrees and 93.9 % within 15 degrees; the bounds leave a margin (median < 3.5, share > 0.92).  At the 4096
    points the model sees, the same estimate gives a 29 degree median: estimate before subsampling."""
    pts, fn = _wand_samples(100_000)
    p = O.frame_map(pts.astype(F32))
    nbr = O.knn(p, 16)
    u = O.smallest_vector(*O.jacobi(O.pca(p, nbr)))
    ang = np.degrees(np.arccos(np.clip(np.abs(np.sum(u.astype(np.float64) * fn, axis=1)), 0, 1)))
    assert np.median(ang) < 3.5 and (ang < 15).mean() > 0.92, (np.median(ang), (ang < 15).mean())


# ---------------------------------------------------------------- readers


def _write_ply(path, xyz, binary, faces=None):
    n = len(xyz)
    head = ["ply", "format " + ("binary_little_endian 1.0" if binary else "ascii 1.0"), "comment bare scan",
            f"element vertex {n}", "property float x", "property float y", "property float z",
            "property uchar red"]
    if faces is not None:
        head += [f"element face {len(faces)}", "property list uchar int vertex_indices"]
    head.append("end_header")
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode())
        if binary:
            rec = np.zeros(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1")])
            rec["x"], rec["y"], rec["z"] = xyz.T
            f.write(rec.tobytes())
        else:
            for v in xyz:
                f.write(f"{float(v[0])!r} {float(v[1])!r} {float(v[2])!r} 7\n".encode())
        if faces is not None:
            for t in faces:
                f.write(f"3 {t[0]} {t[1]} {t[2]}\n".encode())


def test_load_points_reads_npy_and_vertex_only_ply(tmp_path):
    from mesh_to_pc import SimpleMesh, load_points
    xyz = np.random.default_rng(0).normal(size=(50, 3)).astype(F32)
    np.save(tmp_path / "a.npy", xyz)
    got = load_points(str(tmp_path / "a.npy"))
    assert got.dtype == F32 and np.array_equal(got, xyz)
    for binary in (False, True):
        path = tmp_path / f"b{int(binary)}.ply"
        _write_ply(path, xyz, binary)
        got = load_points(str(path))
        assert got.shape == (50, 3) and np.array_equal(got.astype(F32), xyz)
        with pytest.raises(ValueError, match="PLY without vertex/face"):      # the mesh reader keeps its error
            SimpleMesh.load_ply(str(path))
    _write_ply(tmp_path / "m.ply", xyz, False, faces=[[0, 1, 2]])
    with pytest.raises(ValueError, match="--input_type mesh"):
        load_points(str(tmp_path / "m.ply"))


def test_load_points_refuses_points_with_normals(tmp_path):
    from mesh_to_pc import load_points
    np.save(tmp_path / "pn.npy", np.zeros((5000, 6), F32))
    with pytest.raises(ValueError, match="--input_type pc_normal"):
        load_points(str(tmp_path / "pn.npy"))
    np.save(tmp_path / "bad.npy", np.zeros((5000, 4), F32))
    with pytest.raises(ValueError, match=r"\(N, 3\)"):
        load_points(str(tmp_path / "bad.npy"))


def test_pc_input_without_a_gpu_is_an_error(tmp_path, monkeypatch):
    import torch
    if torch.cuda.is_available():
        pytest.skip("this host has a GPU")
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    np.save(tmp_path / "s.npy", _sphere(5000, 0).astype(F32))
    with pytest.raises(RuntimeError, match="CUDA GPU"):
        cli.Dataset("pc", [str(tmp_path / "s.npy")])
