"""CPU: the numpy restatement of plane removal (tests/plane_oracle.py, DESIGN.md section 1.6) against a direct Philox
evaluation, numpy's SVD and math.fsum, on a synthetic scan of an object on a table with legs and strays, on degenerate
input (collinear, identical, N = 3, tied hypotheses, points exactly at the threshold, the flip), and the command line's
handling of `--remove_plane`."""
import argparse
import math
import os
import sys

import numpy as np
import pytest

from tests import plane_oracle as P

F32, F64 = np.float32, np.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _philox_scalar(counter, key):
    """Philox4x32-10 of Random123 on Python integers, one counter at a time."""
    c, (k0, k1) = list(counter), key
    M = 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k0) & M, p1 & M, ((p0 >> 32) ^ c[3] ^ k1) & M, p0 & M]
        k0, k1 = (k0 + 0x9E3779B9) & M, (k1 + 0xBB67AE85) & M
    return c


@pytest.mark.parametrize("seed", [0, 5, (1 << 32) - 1, (1 << 32) + 7, (1 << 64) - 1])
def test_hypothesis_indices_against_a_direct_philox(seed):
    n, H = 12345, 40
    idx = P.hypothesis_indices(n, H, seed)
    for h in range(H):
        c = _philox_scalar((h, 0x504c414e, 0x4d455348, 0x414e5954), (seed & 0xFFFFFFFF, seed >> 32))
        assert idx[h].tolist() == [(c[j] * n) >> 32 for j in range(3)]
    assert idx.min() >= 0 and idx.max() < n


def test_refit_against_svd_and_fsum():
    rng = np.random.default_rng(0)
    n_true = np.array([0.3, -0.5, 0.8])
    n_true /= np.linalg.norm(n_true)
    e1 = np.cross(n_true, [1.0, 0, 0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(n_true, e1)
    uv = rng.uniform(-0.4, 0.4, (3000, 2))
    p = (uv[:, :1] * e1 + uv[:, 1:] * e2 + rng.normal(0, 1e-3, (3000, 1)) * n_true + [0.05, -0.02, 0.01]).astype(F32)
    on = rng.random(3000) < 0.8
    plane, cent, mom, n64 = P.refit(p, on)
    q = p[on].astype(F64)
    for a in range(3):                                            # the fixed-order sums against exact ones
        assert abs(cent[a] * on.sum() - math.fsum(q[:, a])) <= 1e-12 * math.fsum(np.abs(q[:, a]))
    d = q - cent
    for m, (a, b) in zip(mom, [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]):
        ref = math.fsum(d[:, a] * d[:, b])
        assert abs(m - ref) <= 1e-12 * math.fsum(np.abs(d[:, a] * d[:, b]))
    normal = np.linalg.svd(q - q.mean(0), full_matrices=False)[2][-1]
    angle = math.acos(min(1.0, abs(float(n64 @ normal))))
    assert angle < 1e-9, angle
    assert abs(float(np.linalg.norm(plane[:3].astype(F64))) - 1) < 1e-6


@pytest.mark.parametrize("obj", ["sphere", "wand"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_an_object_on_a_table_keeps_the_object(seed, obj):
    pts, lab, t = P.table_scene(seed, obj=obj)
    r = P.remove_plane(P.frame_map(pts), 0.01, 1000, 1000 + seed)
    assert r["found"] and r["valid_count"] >= 990                             # a repeated index is rare
    n = r["plane"][:3].astype(F64)
    assert math.degrees(math.acos(min(1.0, n[2] / np.linalg.norm(n)))) < 1.0      # from the table toward the object
    z = pts[:, 2]
    tab, obj_pts, legs = lab == 0, lab == 1, lab == 2
    assert not r["keep"][tab & (np.abs(z) <= 0.5 * t)].any()                   # the table goes
    assert not r["keep"][legs].any()                                           # and the legs under it
    assert r["keep"][obj_pts & (z > 2 * t)].all()                              # the object stays
    assert r["n_kept"] == r["above"] and r["on"] + r["above"] + r["below"] == len(pts)
    assert np.array_equal(r["kept"], np.nonzero(r["keep"])[0])


def test_collinear_and_identical_points_find_no_plane():
    # a line along x: every difference has y = z = 0, so every cross product is exactly 0 (a diagonal line is not
    # exactly collinear in fp32, and RANSAC rightly finds planes through its rounded points)
    line = np.stack([np.linspace(-1, 1, 500), np.full(500, 0.3), np.full(500, -2.0)], axis=1).astype(F32)
    for cloud in (line, np.zeros((300, 3), F32), np.tile([[0.2, 0.1, -0.3]], (50, 1)).astype(F32)):
        frame = P.frame_map(cloud)
        r = P.remove_plane(frame, 0.01, 200, 3)
        assert not r["found"] and r["valid_count"] == 0 and r["winner"] == 0 and r["winner_count"] == 0
        assert r["keep"].all() and r["n_kept"] == len(cloud) and (r["on"], r["above"], r["below"]) == (0, 0, 0)
        assert not r["plane"].any() and np.all(np.isinf(r["planes"][:, 3]))


def test_three_points():
    p = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], F32)
    r = P.remove_plane(P.frame_map(p), 0.01, 64, 9)
    valid = r["valid"]
    assert valid.any() and r["found"] and r["winner"] == int(np.argmax(valid)) and r["winner_count"] == 3
    assert r["on"] == 3 and r["n_kept"] == 0                                    # all three lie on their plane
    r = P.remove_plane(P.frame_map(p), 0.01, 1, 9)                              # one hypothesis: 3 distinct indices?
    assert r["found"] == bool(r["valid"][0])


def test_ties_go_to_the_lowest_hypothesis():
    """Every valid hypothesis of four coplanar points counts all four: the first valid one wins."""
    p = np.array([[-0.5, -0.5, 0], [0.5, -0.5, 0], [0.5, 0.5, 0], [-0.5, 0.5, 0]], F32)
    r = P.remove_plane(p, 0.01, 500, 4)
    valid = r["valid"]
    assert valid.sum() > 10 and not valid.all()
    assert np.all(r["counts"][valid] == 4) and np.all(r["counts"][~valid] == 0)
    assert r["winner"] == int(np.nonzero(valid)[0][0]) and r["winner_count"] == 4


def _grid(step=1 / 16):
    g = np.arange(-8, 9) * step
    return np.stack(np.meshgrid(g, g, indexing="ij"), axis=-1).reshape(-1, 2)


def test_points_exactly_at_the_threshold_are_on_the_plane():
    """Coordinates on a grid of 1/64: the frame map is the identity (centre 0, longest side 1) and every s is exact."""
    t = 1 / 64
    xy = _grid()
    layers = [(0.0, xy), (t, xy[::2]), (-t, xy[::2]), (2 * t, xy[::3]), (-2 * t, xy[::5])]
    p = np.concatenate([np.concatenate([q, np.full((len(q), 1), z)], axis=1) for z, q in layers]).astype(F32)
    assert np.array_equal(P.frame_map(p), p)
    r = P.remove_plane(p, t, 300, 1)
    assert r["found"] and r["planes"][r["winner"], :3].tolist() in ([0, 0, 1], [0, 0, -1])
    assert r["plane"].tolist() == [0, 0, 1, 0]
    assert r["winner_count"] == r["on"] == len(xy) + 2 * len(xy[::2])          # |s| = t counts as on
    assert r["above"] == len(xy[::3]) and r["below"] == len(xy[::5]) and not r["flipped"]
    assert np.all(p[r["keep"], 2] == 2 * t)


def test_the_plane_turns_toward_the_larger_side():
    t = 1 / 64
    xy = _grid()
    p = np.concatenate([np.concatenate([xy, np.zeros((len(xy), 1))], axis=1),
                        np.concatenate([xy[::5], np.full((len(xy[::5]), 1), 0.25)], axis=1),
                        np.concatenate([xy[::2], np.full((len(xy[::2]), 1), -0.25)], axis=1)]).astype(F32)
    r = P.remove_plane(P.frame_map(p), t, 300, 2)
    assert r["found"] and r["flipped"] == (r["refit"][2] > 0)
    assert r["plane"][2] < 0 and r["above"] == len(xy[::2]) and r["below"] == len(xy[::5])
    assert np.all(p[r["keep"], 2] == -0.25) and r["stats"][3] == r["plane"][2]


def _cli(monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    return cli


def _ns(**kw):
    base = dict(num_samples=1, sampling=False, continuous_batching=False, input_type="pc", remove_outliers=False,
                subsample="random", remove_plane=True, plane_distance=0.01, plane_iterations=1000)
    base.update(kw)
    return argparse.Namespace(**base)


def test_command_line_plane_flags(monkeypatch):
    cli = _cli(monkeypatch)
    monkeypatch.setattr(sys, "argv", ["main.py"])
    a = cli.get_args()
    assert (a.remove_plane, a.plane_distance, a.plane_iterations) == (False, 0.01, 1000)
    assert cli.plane_options(a) is None
    monkeypatch.setattr(sys, "argv", ["main.py", "--remove_plane", "--plane_distance", "0.02", "--plane_iterations", "64"])
    a = cli.get_args()
    assert cli.plane_options(a) == {"distance": 0.02, "iterations": 64}
    for kind in ("pc", "pc_normal"):
        cli.check_args(_ns(input_type=kind))
    with pytest.raises(ValueError, match="point-cloud input"):
        cli.check_args(_ns(input_type="mesh"))
    with pytest.raises(ValueError, match="point-cloud input"):
        cli.Dataset("mesh", [], plane={"distance": 0.01, "iterations": 1000})
    for bad in (0.0, -0.01, 1.5, float("nan"), float("inf"), 1e-50):
        with pytest.raises(ValueError, match="--plane_distance"):
            cli.check_args(_ns(plane_distance=bad))
    for bad in (0, -3, 65537):
        with pytest.raises(ValueError, match="--plane_iterations"):
            cli.check_args(_ns(plane_iterations=bad))
    cli.check_args(_ns(input_type="mesh", remove_plane=False, plane_distance=-1.0))   # unchecked without the flag
    old = argparse.Namespace(num_samples=1, sampling=False, continuous_batching=False, input_type="mesh",
                             remove_outliers=False)                                     # built without the new flags
    cli.check_args(old)
    assert cli.plane_options(old) is None


def test_without_the_flag_the_draw_is_unchanged(tmp_path, monkeypatch):
    cli = _cli(monkeypatch)
    cloud = np.random.default_rng(4).normal(size=(5000, 6)).astype(F32)
    np.save(tmp_path / "c.npy", cloud)
    np.random.seed(3)
    ref = cloud[np.random.choice(5000, 4096, replace=False)]
    for kw in ({}, {"plane": None}):
        np.random.seed(3)
        assert np.array_equal(cli.Dataset("pc_normal", [str(tmp_path / "c.npy")], **kw).data[0]["pc_normal"], ref)

