"""CPU: the point-cloud pipeline of main.py's Dataset with its six GPU entry points (plane.remove_plane,
outliers.remove_outliers, smooth.smooth_points, objects.split_objects, normals.estimate_normals and
subsample.farthest_point_sample) replaced by deterministic numpy fakes.  Over both input types, float32 and float64
files and every subset of the optional stages, the order of the calls, the rows and options each call receives, the
items (rows, dtypes, colours on their rows, uids) and the global numpy RNG after the call are compared with a short
numpy restatement of the order plane -> outliers -> smooth -> split -> per object (normals, subset).  Also the
refusals of mesh input, the command line's checks and the "too few points" errors."""
import argparse
import itertools
import os
import sys

import numpy as np
import pytest
import torch

from meshanything_b200 import normals as normals_mod
from meshanything_b200 import objects as objects_mod
from meshanything_b200 import outliers as outliers_mod
from meshanything_b200 import plane as plane_mod
from meshanything_b200 import smooth as smooth_mod
from meshanything_b200 import subsample as subsample_mod

F32, F64 = np.float32, np.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M = 4096                   # the points the model takes
SHIFT = 0.25               # what the fake smoothing adds to every coordinate
PLANE = {"distance": 0.02, "iterations": 64}
OUTLIERS = {"k": 8, "std_ratio": 1.5, "min_component": 0.0}
SMOOTH = {"k": 12}
OBJECTS = {"distance": 0.05}
STAGES = ("plane", "outliers", "smooth", "objects", "fps", "colors")


# The fakes' rules: numpy functions of the values they receive; none of them draws from an RNG.
def _f64(points):
    return np.asarray(points, dtype=F64)


def plane_keep(points):
    z = _f64(points)[:, 2]
    return np.flatnonzero(z > np.sort(z)[len(z) // 10])            # the lowest tenth goes


def outlier_keep(points):
    p = _f64(points)
    d = np.linalg.norm(p - p.mean(axis=0), axis=1)
    return np.flatnonzero(d < np.sort(d)[len(d) * 19 // 20])       # the twentieth farthest from the centroid goes


def smoothed(points):
    p = np.asarray(points)
    return p + p.dtype.type(SHIFT)


def clusters(points):
    """The points with x < 0 and those with x >= 0, larger first."""
    x = _f64(points)[:, 0]
    parts = [c for c in (np.flatnonzero(x < 0), np.flatnonzero(x >= 0)) if len(c)]
    return sorted(parts, key=lambda c: (-len(c), c[0]))


def normals_of(points):
    v = _f64(points) - _f64(points).mean(axis=0) + (0.5, 0.25, 0.125)
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(F32)


def fps_picks(points, m, start):
    return np.roll(np.argsort(_f64(points)[:, 1], kind="stable"), -start)[:m]


@pytest.fixture
def calls(monkeypatch):
    """Installs the fakes; the list of (stage, rows received, options received) they append to, in call order."""
    log = []

    def remove_plane(points, distance=0.01, iterations=1000, seed=0):
        log.append(("plane", np.array(points), dict(distance=distance, iterations=iterations, seed=seed)))
        keep = plane_keep(points)
        n, kept = len(points), len(keep)
        return torch.from_numpy(keep), plane_mod.PlaneStats(
            found=True, normal=(0.0, 0.0, 1.0), offset=0.0, threshold=distance, hypothesis=0, hypothesis_count=n - kept,
            valid_hypotheses=iterations, on=n - kept, above=kept, below=0, kept=kept)

    def remove_outliers(points, k=16, std_ratio=2.0, min_component=0.01):
        log.append(("outliers", np.array(points), dict(k=k, std_ratio=std_ratio, min_component=min_component)))
        keep = outlier_keep(points)
        n, kept = len(points), len(keep)
        return torch.from_numpy(keep), outliers_mod.OutlierStats(
            n_points=n, removed_statistical=n - kept, removed_components=0, components=1, components_dropped=0,
            mean_distance=0.0, std_distance=0.0, threshold=0.0, kept=kept)

    def smooth_points(points, k=24):
        log.append(("smooth", np.array(points), dict(k=k)))
        n = len(points)
        return torch.from_numpy(smoothed(points)), smooth_mod.SmoothStats(
            n_points=n, k=k, quadratic=n, singular=0, far=0, mean_displacement=SHIFT, max_displacement=SHIFT)

    def split_objects(points, distance=0.02, min_points=4096):
        log.append(("objects", np.array(points), dict(distance=distance, min_points=min_points)))
        parts = clusters(points)
        kept = [c for c in parts if len(c) >= min_points]
        dropped = [len(c) for c in parts if len(c) < min_points]
        idx = np.concatenate(kept) if kept else np.zeros(0, np.int64)
        offsets = np.cumsum([0] + [len(c) for c in kept])
        return torch.from_numpy(idx), torch.from_numpy(offsets), objects_mod.ObjectStats(
            clusters=len(parts), objects=len(kept), object_points=len(idx), dropped_clusters=len(dropped),
            dropped_points=sum(dropped), largest_dropped=max(dropped, default=0), sizes=tuple(len(c) for c in kept),
            distance=distance)

    def estimate_normals(points, k=16):
        log.append(("normals", np.array(points), dict(k=k)))
        return torch.from_numpy(normals_of(points))

    def farthest_point_sample(points, m=4096, start=0):
        log.append(("fps", np.array(points), dict(m=m, start=start)))
        return torch.from_numpy(fps_picks(points, m, start)), torch.linspace(1.0, 0.01, m)

    for mod, fn in ((plane_mod, remove_plane), (outliers_mod, remove_outliers), (smooth_mod, smooth_points),
                    (objects_mod, split_objects), (normals_mod, estimate_normals),
                    (subsample_mod, farthest_point_sample)):
        monkeypatch.setattr(mod, fn.__name__, fn)
    return log


def restate(kind, paths, on):
    """What Dataset(kind, paths, ...) with the stages in `on` gives, drawing from the global RNG as it does:
    (entries, calls)."""
    entries, log = [], []
    for path in paths:
        raw = np.load(path)
        xyz = raw[:, :3]
        nrm = raw[:, 3:6] if kind == "pc_normal" else None
        rgb = raw[:, -3:].astype(F64) if "colors" in on else None

        def rows(keep):
            return [None if a is None else a[keep] for a in (xyz, nrm, rgb)]

        if "plane" in on:
            log.append(("plane", xyz, dict(PLANE, seed=int(np.random.randint(0, 2**62, dtype=np.int64)))))
            xyz, nrm, rgb = rows(plane_keep(xyz))
        if "outliers" in on:
            log.append(("outliers", xyz, OUTLIERS))
            xyz, nrm, rgb = rows(outlier_keep(xyz))
        if "smooth" in on:
            log.append(("smooth", xyz, SMOOTH))
            xyz = smoothed(xyz)
        parts = [np.arange(len(xyz))]
        if "objects" in on:
            log.append(("objects", xyz, dict(OBJECTS, min_points=M)))
            parts = [c for c in clusters(xyz) if len(c) >= M]
        uid = os.path.basename(path)[:-len(".npy")]
        for j, part in enumerate(parts):
            x = xyz[part]
            if kind == "pc":
                log.append(("normals", x, {"k": 16}))
                n = normals_of(x).astype(x.dtype)
            else:
                n = nrm[part]
            if "fps" in on:
                start = np.random.randint(len(x))
                log.append(("fps", x, {"m": M, "start": start}))
                pick = fps_picks(x, M, start)
            else:
                pick = np.random.choice(len(x), M, replace=False)
            entry = {"pc_normal": np.concatenate([x[pick], n[pick]], axis=1),
                     "uid": f"{uid}_obj{j}" if "objects" in on else uid}
            if "colors" in on:
                entry["colors"] = np.concatenate([x.astype(F64), rgb[part]], axis=1)
            entries.append(entry)
    return entries, log


def _cli(monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    return cli


def _write(path, kind, dtype, colors, n_neg, n_pos, seed):
    """Two blobs, one on each side of x = 0, on a slope in z, as an .npy of the layout `kind` and `colors` read."""
    rng = np.random.default_rng(seed)
    xyz = np.concatenate([rng.normal((-2.0, 0.0, 0.0), 0.6, (n_neg, 3)), rng.normal((2.0, 0.5, 0.3), 0.5, (n_pos, 3))])
    cols = [xyz]
    if kind == "pc_normal":
        nrm = rng.normal(size=xyz.shape)
        cols.append(nrm / np.linalg.norm(nrm, axis=1, keepdims=True))
    if colors:
        cols.append(rng.uniform(0, 1, xyz.shape))
    np.save(path, np.concatenate(cols, axis=1).astype(dtype))
    return str(path)


def _dataset_kw(on):
    return dict(plane=PLANE if "plane" in on else None, outliers=OUTLIERS if "outliers" in on else None,
                smooth=SMOOTH if "smooth" in on else None, objects=OBJECTS if "objects" in on else None,
                subsample="fps" if "fps" in on else "random", colors="colors" in on)


_MARKS = {"plane": ": plane n = (", "outliers": " by neighbour distance, ", "smooth": ": smoothed ",
          "objects": " clusters at e = ", "fps": " by farthest-point sampling; "}


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("kind", ["pc", "pc_normal"])
def test_every_stage_subset_against_the_restatement(tmp_path, monkeypatch, capsys, calls, kind, dtype):
    cli = _cli(monkeypatch)
    for r in range(len(STAGES) + 1):
        for on in itertools.combinations(STAGES, r):
            colors = "colors" in on
            paths = [_write(tmp_path / f"{name}.npy", kind, dtype, colors, n_neg, n_pos, seed)
                     for name, n_neg, n_pos, seed in (("scene", 6000, 7000, 1), ("shelf", 7500, 5200, 2))]
            calls.clear()
            capsys.readouterr()
            np.random.seed(11)
            ds = cli.Dataset(kind, paths, **_dataset_kw(on))
            after = np.random.get_state()
            printed = capsys.readouterr().out.splitlines()
            np.random.seed(11)
            want, want_calls = restate(kind, paths, on)
            got_state, want_state = after, np.random.get_state()
            assert got_state[0] == want_state[0] and np.array_equal(got_state[1], want_state[1]), on
            assert got_state[2:] == want_state[2:], on

            assert [c[0] for c in calls] == [c[0] for c in want_calls], on
            for (_, got_rows, got_opts), (name, want_rows, want_opts) in zip(calls, want_calls):
                assert got_rows.dtype == want_rows.dtype and np.array_equal(got_rows, want_rows), (on, name)
                assert got_opts == want_opts, (on, name)

            assert len(ds.data) == len(want) == (4 if "objects" in on else 2), on
            for got, exp in zip(ds.data, want):
                assert set(got) == ({"pc_normal", "uid", "colors"} if colors else {"pc_normal", "uid"}), on
                assert got["uid"] == exp["uid"], on
                assert got["pc_normal"].shape == (M, 6) and got["pc_normal"].dtype == dtype, on
                assert np.array_equal(got["pc_normal"], exp["pc_normal"]), on
                if colors:   # the restatement keeps every colour on the row it came with
                    assert got["colors"].dtype == F64 and np.array_equal(got["colors"], exp["colors"]), on

            per_input = [c[0] for c in want_calls if c[0] != "normals"]
            assert printed[-1] == f"dataset total data samples: {len(want)}"
            assert len(printed) == len(per_input) + 1, (on, printed)
            for line, stage in zip(printed, per_input):
                assert _MARKS[stage] in line and line.split(":")[0] in ("scene", "shelf"), (on, line)


_REFUSALS = {
    "outliers": ({"outliers": OUTLIERS}, {"remove_outliers": True},
                 "--remove_outliers applies to point-cloud input (--input_type pc or pc_normal): the points of a mesh "
                 "are sampled from its surface and have no outliers"),
    "subsample": ({"subsample": "fps"}, {"subsample": "fps"},
                  "--subsample fps applies to point-cloud input (--input_type pc or pc_normal): the points of a mesh "
                  "are already sampled uniformly by area"),
    "plane": ({"plane": PLANE}, {"remove_plane": True},
              "--remove_plane applies to point-cloud input (--input_type pc or pc_normal): the points of a mesh are "
              "sampled from its own surface, which has no scanned support under it"),
    "objects": ({"objects": OBJECTS}, {"split_objects": True},
                "--split_objects applies to point-cloud input (--input_type pc or pc_normal): splitting a mesh into "
                "its connected parts is not supported"),
    "smooth": ({"smooth": SMOOTH}, {"smooth": True},
               "--smooth applies to point-cloud input (--input_type pc or pc_normal): the points of a mesh are sampled "
               "exactly from its surface and carry no scanner noise"),
    "colors": ({"colors": True}, {"transfer_colors": True},
               "--transfer_colors applies to point-cloud input (--input_type pc or pc_normal): colours of a mesh's "
               "own vertices or textures are not read"),
}


def _ns(**kw):
    """A namespace of the command line's defaults, with `kw` on top."""
    base = dict(num_samples=1, sampling=False, continuous_batching=False, input_type="pc", remove_outliers=False,
                outlier_neighbors=16, outlier_std_ratio=2.0, outlier_min_component=0.01, subsample="random",
                remove_plane=False, plane_distance=0.01, plane_iterations=1000, split_objects=False,
                object_distance=0.02, smooth=False, smooth_neighbors=24, output_frame="model", transfer_colors=False,
                color_distance=0.05)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("stage", sorted(_REFUSALS))
def test_mesh_input_is_refused_with_the_same_message(monkeypatch, calls, stage):
    cli = _cli(monkeypatch)
    dataset_kw, flags, message = _REFUSALS[stage]
    with pytest.raises(ValueError) as e:
        cli.Dataset("mesh", ["never_read.obj"], **dataset_kw)
    assert str(e.value) == message
    with pytest.raises(ValueError) as e:
        cli.check_args(_ns(input_type="mesh", **flags))
    assert str(e.value) == message
    for kind in ("pc", "pc_normal"):
        cli.check_args(_ns(input_type=kind, **flags))
    assert calls == []


def test_check_args_ranges(monkeypatch):
    cli = _cli(monkeypatch)
    good = [dict(remove_outliers=True, outlier_neighbors=k) for k in (1, 64)]
    good += [dict(remove_outliers=True, outlier_std_ratio=-1.0, outlier_min_component=0.0)]
    good += [dict(remove_plane=True, plane_distance=d, plane_iterations=h) for d, h in ((1.0, 1), (1e-6, 65536))]
    good += [dict(split_objects=True, object_distance=d) for d in (1.0, 1e-6)]
    good += [dict(smooth=True, smooth_neighbors=k) for k in (5, 64, np.int64(24))]
    good += [dict(transfer_colors=True, color_distance=d) for d in (1.0, 1e-6)]
    good += [dict(subsample="fps"), dict(output_frame="input")]
    # out of range but with the stage off: not checked
    good += [dict(input_type="mesh", outlier_neighbors=0, plane_distance=-1.0, plane_iterations=0, object_distance=7.0,
                  smooth_neighbors=0, color_distance=0.0)]
    for kw in good:
        cli.check_args(_ns(**kw))
    nan, inf = float("nan"), float("inf")
    bad = [(dict(remove_outliers=True, outlier_neighbors=k), f"--outlier_neighbors must be in 1..64, got {k}")
           for k in (0, 65)]
    bad += [(dict(remove_outliers=True, **kw), "--outlier_std_ratio must be finite and --outlier_min_component finite "
             "and >= 0") for kw in ({"outlier_std_ratio": nan}, {"outlier_std_ratio": inf},
                                    {"outlier_min_component": -0.01}, {"outlier_min_component": nan})]
    bad += [(dict(remove_plane=True, plane_distance=d), "--plane_distance must be in (0, 1] (a share of the bounding "
             f"box's longest side), got {d}") for d in (0.0, -0.01, 1.5, nan, inf, 1e-50)]
    bad += [(dict(remove_plane=True, plane_iterations=h), f"--plane_iterations must be in 1..65536, got {h}")
            for h in (0, 65537)]
    bad += [(dict(split_objects=True, object_distance=d), "--object_distance must be in (0, 1] (a share of the "
             f"bounding box's longest side, with a square above 0 in fp32), got {d}") for d in (0.0, 1.5, nan, 1e-30)]
    bad += [(dict(smooth=True, smooth_neighbors=k), f"--smooth_neighbors must be in 5..64, got {k}")
            for k in (4, 65, True, 24.0)]
    bad += [(dict(transfer_colors=True, color_distance=d), "--color_distance must be in (0, 1] (a share of the "
             f"bounding box's longest side), got {d}") for d in (0.0, 1.5, nan, 1e-50)]
    bad += [(dict(subsample="voxel"), "--subsample must be one of random, fps, got 'voxel'"),
            (dict(output_frame="world"), "--output_frame must be one of model, input, got 'world'")]
    for kw, message in bad:
        with pytest.raises(ValueError) as e:
            cli.check_args(_ns(**kw))
        assert str(e.value) == message, kw


def test_options_from_the_command_line(monkeypatch):
    cli = _cli(monkeypatch)
    readers = (cli.outlier_options, cli.plane_options, cli.object_options, cli.smooth_options, cli.color_options)
    monkeypatch.setattr(sys, "argv", ["main.py"])
    assert [f(cli.get_args()) for f in readers] == [None, None, None, None, False]
    monkeypatch.setattr(sys, "argv", [
        "main.py", "--remove_outliers", "--outlier_neighbors", "9", "--outlier_std_ratio", "1.5",
        "--outlier_min_component", "0.2", "--remove_plane", "--plane_distance", "0.03", "--plane_iterations", "77",
        "--split_objects", "--object_distance", "0.04", "--smooth", "--smooth_neighbors", "30", "--transfer_colors",
        "--subsample", "fps"])
    a = cli.get_args()
    cli.check_args(a)
    assert [f(a) for f in readers] == [{"k": 9, "std_ratio": 1.5, "min_component": 0.2},
                                       {"distance": 0.03, "iterations": 77}, {"distance": 0.04}, {"k": 30}, True]
    # a namespace built without the newer flags: every stage off
    old = argparse.Namespace(num_samples=1, sampling=False, continuous_batching=False, input_type="mesh",
                             remove_outliers=False)
    cli.check_args(old)
    assert [f(old) for f in readers] == [None, None, None, None, False]


@pytest.mark.parametrize("on", [(), ("plane",), ("outliers",), ("smooth",), ("objects",), ("fps",), ("colors",),
                                ("plane", "outliers", "smooth", "objects", "fps", "colors")])
def test_too_few_points(tmp_path, monkeypatch, calls, on):
    """pc: refused before any stage (and before the plane seed is drawn).  pc_normal: plane and outlier removal refuse
    what they leave too small; otherwise the assertion fires after smoothing, before the split."""
    cli = _cli(monkeypatch)
    for kind in ("pc", "pc_normal"):
        path = _write(tmp_path / f"{kind}.npy", kind, F32, "colors" in on, 2000, 2000, 3)
        calls.clear()
        np.random.seed(5)
        before = np.random.get_state()[1].copy()
        if kind == "pc":
            expect, match, stages = AssertionError, "at least 4096 points", []
        elif "plane" in on:
            expect, match, stages = ValueError, "remain after plane removal", ["plane"]
        elif "outliers" in on:
            expect, match, stages = ValueError, "remain after outlier removal", ["outliers"]
        else:
            expect, match, stages = AssertionError, "at least 4096 points", ["smooth"] if "smooth" in on else []
        with pytest.raises(expect, match=match):
            cli.Dataset(kind, [path], **_dataset_kw(on))
        assert [c[0] for c in calls] == stages, (kind, on)
        if not stages:
            assert np.array_equal(np.random.get_state()[1], before)


def test_no_object_large_enough(tmp_path, monkeypatch, calls):
    cli = _cli(monkeypatch)
    for kind in ("pc", "pc_normal"):
        path = _write(tmp_path / f"{kind}.npy", kind, F64, False, 3000, 3000, 4)
        calls.clear()
        with pytest.raises(ValueError, match="no cluster of 4096 points"):
            cli.Dataset(kind, [path], objects=OBJECTS)
        assert [c[0] for c in calls] == ["objects"]
