"""CPU: the numpy restatement of farthest-point subsampling (tests/subsample_oracle.py, DESIGN.md section 1.4) against a
hand-derived answer and float64 cKDTree covering radii, its behaviour on duplicates, edge cases and stray points, the
coverage it buys on a cloud of uneven density compared with np.random.choice, and the command line's handling of
`--subsample`."""
import argparse
import os
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

from tests import subsample_oracle as S

F32, F64 = np.float32, np.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _line(n):
    """Integer points on the x axis: every fp32 d^2 below 2^24 is exact."""
    return np.stack([np.arange(n), np.zeros(n), np.zeros(n)], axis=1).astype(F32)


def test_known_answer_on_a_line():
    idx, r2 = S.farthest_point_sample(_line(17), 17, 0)
    assert idx.tolist() == [0, 16, 8, 4, 12, 2, 6, 10, 14, 1, 3, 5, 7, 9, 11, 13, 15]
    assert r2.tolist() == [256, 64, 16, 16, 4, 4, 4, 4] + [1] * 8 + [0]
    idx, r2 = S.farthest_point_sample(_line(1000), 3, 0)            # 0, the far end, then the lowest of the two middles
    assert idx.tolist() == [0, 999, 499] and r2.tolist() == [999 ** 2, 499 ** 2, 250 ** 2]


def _sphere(n, rng):
    x = rng.normal(size=(n, 3))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def test_covering_radius_and_packing_against_float64():
    rng = np.random.default_rng(0)
    p = np.concatenate([rng.uniform(-0.5, 0.5, (3000, 3)), _sphere(2000, rng) * 0.4]).astype(F32)
    idx, r2 = S.farthest_point_sample(p, 600, 17)
    assert len(set(idx.tolist())) == 600 and np.all(np.diff(r2) <= 0)
    p64 = p.astype(F64)
    for t in (0, 1, 9, 99, 341, 599):
        picks = p64[idx[:t + 1]]
        cover = cKDTree(picks).query(p64)[0].max() ** 2
        assert abs(float(r2[t]) - cover) <= 1e-6 * cover, (t, float(r2[t]), cover)
        if t:                                                        # k-center packing: picks are >= sqrt(r2[t]) apart
            sep = cKDTree(picks).query(picks, 2)[0][:, 1].min()
            assert sep >= np.sqrt(float(r2[t])) * (1 - 1e-6), (t, sep, float(r2[t]))


def test_duplicates_are_taken_in_index_order_once():
    rng = np.random.default_rng(1)
    pos = rng.uniform(-0.5, 0.5, (10, 3)).astype(F32)
    p = np.repeat(pos, 100, axis=0)                                  # index i holds position i // 100
    idx, r2 = S.farthest_point_sample(p, 30, 0)
    first = idx[:10]
    assert sorted((first // 100).tolist()) == list(range(10))        # every distinct position once
    assert all(i % 100 == 0 for i in first.tolist())                # each by its lowest index
    rest = [i for i in range(len(p)) if i not in set(first.tolist())][:20]
    assert idx[10:].tolist() == rest and len(set(idx.tolist())) == 30
    assert np.all(r2[9:] == 0) and np.all(r2[:9] > 0)


def test_edge_cases():
    rng = np.random.default_rng(2)
    p = rng.uniform(-0.5, 0.5, (257, 3)).astype(F32)
    idx, r2 = S.farthest_point_sample(p, 257, 200)
    assert sorted(idx.tolist()) == list(range(257)) and idx[0] == 200 and r2[-1] == 0 and np.all(r2[:-1] > 0)
    idx, r2 = S.farthest_point_sample(p, 1, 5)
    d = p.astype(F64) - p[5].astype(F64)
    assert idx.tolist() == [5] and abs(float(r2[0]) - (d * d).sum(axis=1).max()) <= 1e-6 * float(r2[0])
    idx, r2 = S.farthest_point_sample(np.zeros((1, 3), F32), 1, 0)
    assert idx.tolist() == [0] and r2.tolist() == [0]
    idx, r2 = S.farthest_point_sample(np.zeros((50, 3), F32), 50, 7)   # all identical: index order after the start
    assert idx.tolist() == [7] + [i for i in range(50) if i != 7] and not r2.any()


@pytest.mark.parametrize("start", [0, 123, 4999, 5000])
def test_a_stray_point_is_among_the_first_two_picks(start):
    """The caveat of section 1.4: FPS takes the extremes first, so --remove_outliers belongs before it."""
    rng = np.random.default_rng(3)
    p = np.concatenate([_sphere(5000, rng), _sphere(1, rng) * 10]).astype(F64)
    idx, _ = S.farthest_point_sample(S.frame_map(p), 16, start)
    assert 5000 in idx[:2].tolist()


def _uneven_sphere(seed, draws=600_000):
    """About 100k points on the unit sphere with density proportional to e^(3z)."""
    rng = np.random.default_rng(seed)
    x = _sphere(draws, rng)
    keep = rng.random(draws) < np.exp(3 * x[:, 2]) / np.exp(3.0)
    return x[keep], rng


@pytest.mark.parametrize("seed", range(3))
def test_fps_covers_an_uneven_sphere_better_than_random_choice(seed):
    p, rng = _uneven_sphere(seed)
    ref = _sphere(200_000, np.random.default_rng(100 + seed))        # a uniform reference sample of the surface
    idx, _ = S.farthest_point_sample(p.astype(F32), 4096, int(rng.integers(len(p))))
    g_fps = cKDTree(p[idx]).query(ref)[0]
    g_rnd = cKDTree(p[rng.choice(len(p), 4096, replace=False)]).query(ref)[0]
    fps, rnd = (g_fps.max(), np.quantile(g_fps, 0.99)), (g_rnd.max(), np.quantile(g_rnd, 0.99))
    print(f"seed {seed}: {len(p)} points; largest / 99th-percentile gap: fps {fps[0]:.4f} / {fps[1]:.4f}, "
          f"np.random.choice {rnd[0]:.4f} / {rnd[1]:.4f}")
    assert fps[0] < rnd[0] and fps[1] < rnd[1]


def _cli(monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    return cli


def test_command_line_subsample_flag(monkeypatch):
    cli = _cli(monkeypatch)
    monkeypatch.setattr(sys, "argv", ["main.py"])
    assert cli.get_args().subsample == "random"                      # the default: the reference's draw
    monkeypatch.setattr(sys, "argv", ["main.py", "--subsample", "fps"])
    assert cli.get_args().subsample == "fps"
    args = argparse.Namespace(num_samples=1, sampling=False, continuous_batching=False, input_type="mesh",
                              remove_outliers=False, subsample="fps")
    with pytest.raises(ValueError, match="point-cloud input"):
        cli.check_args(args)
    with pytest.raises(ValueError, match="point-cloud input"):
        cli.Dataset("mesh", [], subsample="fps")
    with pytest.raises(ValueError, match="--subsample must be one of"):
        cli.Dataset("pc_normal", [], subsample="voxel")
    for kind in ("pc", "pc_normal"):
        args.input_type = kind
        cli.check_args(args)
    args.input_type, args.subsample = "mesh", "random"
    cli.check_args(args)


def test_random_subsample_is_the_unchanged_draw(tmp_path, monkeypatch):
    cli = _cli(monkeypatch)
    cloud = np.random.default_rng(4).normal(size=(5000, 6)).astype(F32)
    np.save(tmp_path / "c.npy", cloud)
    np.random.seed(3)
    ref = cloud[np.random.choice(5000, 4096, replace=False)]
    for kw in ({}, {"subsample": "random"}):
        np.random.seed(3)
        assert np.array_equal(cli.Dataset("pc_normal", [str(tmp_path / "c.npy")], **kw).data[0]["pc_normal"], ref)
