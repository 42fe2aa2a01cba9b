"""not gpu: the numpy restatement of object splitting (tests/objects_oracle.py, DESIGN.md section 1.7) against an
independent union-find, at the exact distance boundary, on ties, degenerate clouds and a tabletop scene; the
command-line handling of `--split_objects` / `--output_frame`; the arithmetic of the output-frame map."""
import argparse
import sys

import numpy as np
import pytest
import torch

from tests import objects_oracle as O
from tests import plane_oracle as P

F32, F64 = np.float32, np.float64


def _cli(monkeypatch):
    import os
    monkeypatch.syspath_prepend(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import main as cli
    return cli


def test_components_against_an_independent_union_find():
    rng = np.random.default_rng(0)
    p = rng.random((3000, 3)).astype(F32) - F32(0.5)
    for e in (0.01, 0.03, 0.06):
        pairs = O.edges(p, e)
        brute = [(i, j) for i in range(200) for j in range(i + 1, 200)
                 if O.d2(p[i:i + 1], p[j:j + 1])[0] <= O.e_and_e2(e)[1]]
        assert sorted(map(tuple, pairs[(pairs < 200).all(axis=1)].tolist())) == brute
        assert np.array_equal(O.component_minima(len(p), pairs), O.union_find_labels(len(p), pairs))


def test_pairs_exactly_at_e2_are_joined_and_one_ulp_beyond_are_not():
    e = 1 / 64
    _, e2 = O.e_and_e2(e)
    assert e2 == F32(1 / 4096)
    base = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [1, 1, 1]], F64) / 64          # chain of steps exactly e
    dl = float(np.nextafter(F32(e), F32(1)))                                          # one fp32 ulp beyond e
    far = np.array([[0, 0.25, 0], [dl, 0.25, 0], [0, 0.3, 0], [0, 0.3, dl]], F64)
    corners = np.array([[-0.5, -0.5, -0.5], [0.5, 0.5, 0.5]])
    p = O.frame_map(np.concatenate([base, far, corners]).astype(F32))
    assert np.array_equal(p, np.concatenate([base, far, corners]).astype(F32))          # the frame is the identity
    assert (O.d2(p[:3], p[1:4]) == e2).all()
    assert (O.d2(p[[4, 6]], p[[5, 7]]) > e2).all()
    lab = O.split_objects(p, e, 1)["labels"]
    assert (lab[:4] == 0).all() and np.array_equal(lab[4:8], np.arange(4, 8))


def test_ties_are_ordered_by_label():
    p = np.array([[0.5, 0, 0], [-0.5, 0, 0], [0.5, 0.01, 0], [-0.5, 0.01, 0], [0, 0.3, 0], [0, 0.3, 0.01]], F32)
    r = O.split_objects(O.frame_map(p), 0.02, 2)
    assert np.array_equal(r["clusters"], [0, 1, 4]) and np.array_equal(r["objects"], [0, 1, 4])
    assert np.array_equal(r["indices"], [0, 2, 1, 3, 4, 5]) and np.array_equal(r["offsets"], [0, 2, 4, 6])
    assert np.array_equal(r["stats"], [3, 3, 6, 0, 0, 0])


def test_all_identical_and_all_isolated():
    p = np.tile([[0.25, -1, 3]], (500, 1)).astype(F32)
    r = O.split_objects(O.frame_map(p), 1e-4, 500)
    assert (r["labels"] == 0).all() and np.array_equal(r["stats"], [1, 1, 500, 0, 0, 0])
    g = np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3) / 7 - 0.5
    r = O.split_objects(O.frame_map(g.astype(F32)), 0.1, 1)
    assert np.array_equal(r["labels"], np.arange(512)) and np.array_equal(r["indices"], np.arange(512))
    assert np.array_equal(r["stats"], [512, 512, 512, 0, 0, 0])
    r = O.split_objects(O.frame_map(g.astype(F32)), 0.1, 2)
    assert np.array_equal(r["stats"], [512, 0, 0, 512, 512, 1]) and np.array_equal(r["offsets"], [0])


def test_min_points_at_the_boundary():
    rng = np.random.default_rng(1)
    a = rng.random((40, 3)) * 0.01
    b = rng.random((39, 3)) * 0.01 + 0.9
    p = O.frame_map(np.concatenate([a, b]).astype(F32))
    for mp, want in ((39, [2, 2, 79, 0, 0, 0]), (40, [2, 1, 40, 1, 39, 39]), (41, [2, 0, 0, 2, 79, 40])):
        assert np.array_equal(O.split_objects(p, 0.05, mp)["stats"], want)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_a_table_scene_splits_into_its_three_objects(seed):
    pts, lab = O.table_scene(seed)
    k = P.remove_plane(P.frame_map(pts), 0.01, 1000, 7)["kept"]
    r = O.split_objects(O.frame_map(pts[k]), 0.02, 4096)
    assert r["stats"][1] == 3
    got = set()
    for j in range(3):
        part = lab[k][r["indices"][r["offsets"][j]:r["offsets"][j + 1]]]
        kinds = np.unique(part)
        assert len(kinds) == 1 and kinds[0] in (1, 2, 3)                  # none of another object's points
        assert len(part) == (lab[k] == kinds[0]).sum()                     # all of its own
        got.add(int(kinds[0]))
    assert got == {1, 2, 3}
    assert r["stats"][4] == (lab[k] >= 4).sum()                            # every stray dropped


def _ns(**kw):
    base = dict(num_samples=1, sampling=False, continuous_batching=False, input_type="pc", remove_outliers=False,
                subsample="random", split_objects=True, object_distance=0.02, output_frame="model")
    base.update(kw)
    return argparse.Namespace(**base)


def test_command_line_object_flags(monkeypatch):
    cli = _cli(monkeypatch)
    monkeypatch.setattr(sys, "argv", ["main.py"])
    a = cli.get_args()
    assert (a.split_objects, a.object_distance, a.output_frame) == (False, 0.02, "model")
    assert cli.object_options(a) is None
    monkeypatch.setattr(sys, "argv", ["main.py", "--split_objects", "--object_distance", "0.05", "--output_frame",
                                      "input"])
    a = cli.get_args()
    assert cli.object_options(a) == {"distance": 0.05} and a.output_frame == "input"
    for kind in ("pc", "pc_normal"):
        cli.check_args(_ns(input_type=kind))
    with pytest.raises(ValueError, match="point-cloud input"):
        cli.check_args(_ns(input_type="mesh"))
    with pytest.raises(ValueError, match="point-cloud input"):
        cli.Dataset("mesh", [], objects={"distance": 0.02})
    for bad in (0.0, -0.01, 1.5, float("nan"), float("inf"), 1e-50, 1e-25):
        with pytest.raises(ValueError, match="--object_distance"):
            cli.check_args(_ns(object_distance=bad))
    cli.check_args(_ns(object_distance=1.0))
    with pytest.raises(ValueError, match="--output_frame"):
        cli.check_args(_ns(output_frame="world"))
    cli.check_args(_ns(input_type="mesh", split_objects=False, output_frame="input"))   # any input type
    old = argparse.Namespace(num_samples=1, sampling=False, continuous_batching=False, input_type="mesh",
                             remove_outliers=False)                                     # built without the new flags
    cli.check_args(old)
    assert cli.object_options(old) is None


def test_without_the_flag_the_draw_is_unchanged(tmp_path, monkeypatch):
    cli = _cli(monkeypatch)
    cloud = np.random.default_rng(4).normal(size=(5000, 6)).astype(F32)
    np.save(tmp_path / "c.npy", cloud)
    np.random.seed(3)
    ref = cloud[np.random.choice(5000, 4096, replace=False)]
    np.random.seed(3)
    ds = cli.Dataset("pc_normal", [str(tmp_path / "c.npy")], objects=None)
    assert np.array_equal(ds.data[0]["pc_normal"], ref) and ds.data[0]["uid"] == "c"


def test_output_frame_map_arithmetic():
    from meshanything_b200 import metrics
    rng = np.random.default_rng(5)
    rows = (rng.random((4096, 3)) * [3.0, 0.5, 1.25] + [1e3, -7, 0.1]).astype(F32)
    centre, side = metrics.shape_frame(rows)
    r64 = rows.astype(F64)
    lo, hi = r64.min(0), r64.max(0)
    assert np.array_equal(centre.numpy(), (lo + hi) / 2) and side == (hi - lo).max()
    faces = torch.rand(7, 3, 3, dtype=torch.float32) - 0.5
    out = metrics.to_input_frame(faces, (centre, side))
    assert out.dtype == torch.float64
    assert np.array_equal(out.numpy(), (lo + hi) / 2 + (hi - lo).max() * faces.numpy().astype(F64))
    # the inverse of to_output_frame: the rows come back to within fp32 rounding
    back = metrics.to_input_frame(metrics.to_output_frame(torch.from_numpy(rows)[None])[0], (centre, side))
    assert np.abs(back.numpy() - r64).max() < 1e-3
    c1, s1 = metrics.shape_frame(np.tile([[1.0, 2.0, 3.0]], (5, 1)))
    assert s1 == 1.0 and np.array_equal(c1.numpy(), [1.0, 2.0, 3.0])                    # a single point: side 1
