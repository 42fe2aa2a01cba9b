"""CPU: the numpy restatement of outlier removal (tests/outliers_oracle.py, DESIGN.md section 1.3) against float64
cKDTree / numpy statistics and scipy's components, and what it does to the clouds it is for: a stray point that
turns every normal of a sphere inward, a dense floating cluster, a cloud of identical points; and the command line's
refusal of `--remove_outliers` for mesh input."""
import argparse

import numpy as np
import pytest
from scipy.spatial import cKDTree

from tests import normals_oracle as NO
from tests import outliers_oracle as O

F32, F64 = np.float32, np.float64


def _sphere(n, rng, r=1.0):
    x = rng.normal(size=(n, 3))
    return x / np.linalg.norm(x, axis=1, keepdims=True) * r


def _ref_stats(p, k, std_ratio):
    """float64: kNN distances by cKDTree (self excluded), their means, numpy's mean and std(ddof=1)."""
    d, _ = cKDTree(np.asarray(p, F64)).query(np.asarray(p, F64), k + 1)
    dbar = d[:, 1:].mean(axis=1)
    mu, sigma = dbar.mean(), dbar.std(ddof=1)
    return dbar, mu, sigma, mu + std_ratio * sigma


def test_statistics_match_float64_on_exact_distances():
    """Integer coordinates on a line: every fp32 d^2 and sqrt is exact, so only the sums' order can differ."""
    rng = np.random.default_rng(0)
    x = rng.choice(100_000, 3000, replace=False).astype(F64)
    x[:5] = [300_000, 500_000, 700_000, 900_000, 1_100_000]          # stray points
    p = np.stack([x, np.zeros_like(x), np.zeros_like(x)], axis=1).astype(F32)
    for k in (1, 8, 16):
        r = O.remove_outliers(p, k, 2.0, 0.0)
        dbar, mu, sigma, thr = _ref_stats(p, k, 2.0)
        assert np.allclose(r["mean_dist"], dbar, rtol=1e-9, atol=0)
        for a, b in ((r["mu"], mu), (r["sigma"], sigma), (r["threshold"], thr)):
            assert abs(a - b) <= 1e-9 * abs(b)
        assert not r["keep"][:5].any()


def test_statistics_match_float64_on_a_scattered_cloud():
    """General coordinates: the fp32 distances carry ~1e-7 relative error, the fp64 sums nothing visible."""
    rng = np.random.default_rng(1)
    p = np.concatenate([_sphere(5000, rng), rng.uniform(-5, 5, (50, 3))]).astype(F32)
    r = O.remove_outliers(p, 16, 2.0, 0.0)
    dbar, mu, sigma, _ = _ref_stats(p, 16, 2.0)
    assert np.allclose(r["mean_dist"], dbar, rtol=1e-6, atol=0)
    assert abs(r["mu"] - mu) <= 1e-6 * mu and abs(r["sigma"] - sigma) <= 1e-6 * sigma
    # the fixed-order sums themselves, on the same values
    assert abs(O.fixed_sum(r["mean_dist"]) - np.sum(r["mean_dist"])) <= 1e-12 * np.sum(r["mean_dist"])
    assert abs(O.moments(r["mean_dist"], 2.0)[1] - np.std(r["mean_dist"], ddof=1)) <= 1e-12 * sigma


def _union_find_labels(n, nbr, inl):
    parent = list(range(n))

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a

    for i in range(n):
        if not inl[i]:
            continue
        for j in nbr[i].tolist():
            if inl[j]:
                a, b = find(i), find(j)
                if a != b:
                    parent[max(a, b)] = min(a, b)
    lab = np.array([find(i) for i in range(n)])
    low = {}
    for i in range(n):
        low.setdefault(lab[i], i)
    return np.where(inl, [low[v] for v in lab], -1)


def test_components_match_an_independent_union_find():
    rng = np.random.default_rng(2)
    parts = [_sphere(800, rng) + c for c in ((0, 0, 0), (5, 0, 0), (0, 7, 0))] + [rng.uniform(-1, 1, (30, 3)) * 0.01 + 20]
    p = np.concatenate(parts).astype(F32)[rng.permutation(2430)]
    nbr = NO.knn(p, 8)
    inl = rng.random(len(p)) > 0.05
    assert np.array_equal(O.components(len(p), nbr, inl), _union_find_labels(len(p), nbr, inl))


def _sphere_with_stray(seed, n=6000):
    rng = np.random.default_rng(seed)
    s = _sphere(n, rng)
    stray = _sphere(1, rng) * rng.uniform(7, 10)
    return np.concatenate([s, stray]).astype(F64)


@pytest.mark.parametrize("seed", range(6))
def test_one_stray_point_is_removed_and_the_sphere_comes_out_outward(seed):
    pts = _sphere_with_stray(seed)
    r = O.remove_outliers(O.frame_map(pts), 16, 2.0, 0.01)
    assert not r["keep"][-1] and r["keep"][:-1].all(), (r["inliers"], r["n_kept"])
    kept = pts[r["kept"]]
    frame = O.frame_map(kept)
    nrm, _, _ = NO.estimate_normals(frame, 16)
    assert (NO.dot32(nrm, frame) > 0).all()


def test_dense_floater_cluster_is_dropped_by_the_component_stage():
    rng = np.random.default_rng(3)
    s = _sphere(30_000, rng)
    cluster = rng.uniform(-0.02, 0.02, (200, 3)) + np.array([3.0, 0.0, 0.0])
    pts = np.concatenate([s, cluster]).astype(F64)
    off = O.remove_outliers(O.frame_map(pts), 16, 2.0, 0.0)
    assert off["keep"][-200:].all() and off["components"] == 0       # the statistical stage misses it
    r = O.remove_outliers(O.frame_map(pts), 16, 2.0, 0.01, nbr=off["knn"])
    assert not r["keep"][-200:].any()
    assert r["components"] >= 2 and r["dropped"] >= 1
    assert r["n_kept"] >= 29_000 and np.array_equal(r["keep"][:30_000], off["keep"][:30_000])


def test_identical_points_keep_everything():
    p = np.zeros((500, 3), F32)
    r = O.remove_outliers(O.frame_map(p), 16, 2.0, 0.01)
    assert r["sigma"] == 0 and r["threshold"] == 0 and r["keep"].all() and r["components"] == 1


def test_min_component_zero_switches_the_component_stage_off():
    rng = np.random.default_rng(4)
    pts = np.concatenate([_sphere(3000, rng), _sphere(20, rng) * 0.01 + 4]).astype(F32)
    frame = O.frame_map(pts)
    on = O.remove_outliers(frame, 8, 2.0, 0.05)
    off = O.remove_outliers(frame, 8, 2.0, 0.0, nbr=on["knn"])
    inl = off["mean_dist"] <= off["threshold"]
    assert np.array_equal(off["keep"], inl) and off["components"] == 0 and off["dropped"] == 0
    assert on["n_kept"] < off["n_kept"]


def test_mesh_input_refuses_remove_outliers(monkeypatch):
    import os
    monkeypatch.syspath_prepend(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import main as cli
    args = argparse.Namespace(num_samples=1, sampling=False, continuous_batching=False, input_type="mesh",
                              remove_outliers=True, outlier_neighbors=16, outlier_std_ratio=2.0,
                              outlier_min_component=0.01)
    with pytest.raises(ValueError, match="point-cloud input"):
        cli.check_args(args)
    with pytest.raises(ValueError, match="point-cloud input"):
        cli.Dataset("mesh", [], outliers={"k": 16})
    args.input_type, args.outlier_neighbors = "pc", 65
    with pytest.raises(ValueError, match="outlier_neighbors"):
        cli.check_args(args)
    args.outlier_neighbors, args.remove_outliers = 16, False
    cli.check_args(args)
    assert cli.outlier_options(args) is None
