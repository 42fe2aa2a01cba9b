"""-m gpu: moving-least-squares smoothing (csrc/smooth.cu) against its numpy restatement (tests/smooth_oracle.py) bit for
bit -- the kNN, the normals, the outcomes, the points and the stats, two calls identical -- over a grid of (N, k) and
hard clouds, 1M points, bad input refused before any launch, and the pipeline: `Dataset(..., smooth=...)` for `pc` and
`pc_normal` with and without outlier removal and object splitting, and `main.py --smooth`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from meshanything_b200 import capi
from meshanything_b200.pointcloud import frame_points
from meshanything_b200.smooth import DEFAULT_K, smooth_points
from tests import objects_oracle as JO
from tests import outliers_oracle as OO
from tests import smooth_oracle as S

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64
WAND = os.path.join(ROOT, "tests", "golden", "wand_mesh.npz")


def _dev():
    return torch.device("cuda", 0)


def _wand(n, seed, sigma=0.002):
    z = np.load(WAND)
    return S.add_noise(S.surface_points(z["vertices"], z["faces"], n, seed), sigma, seed + 1)


def _cloud(n, kind, seed):
    """The hard cases of the other stages' tests: the noisy wand (float64, offset by 1e4) with exact duplicates, a
    collinear line, a coplanar patch, a dense cluster in one cell, a far second component."""
    rng = np.random.default_rng(seed)
    if kind == "wand":
        p = _wand(n, seed)
        p[n // 7:n // 7 + n // 50] = p[:n // 50]
        return p + 1e4
    if kind == "line":
        return np.stack([rng.uniform(-1, 1, n), np.full(n, 0.25), np.full(n, 3.0)], axis=1).astype(F32)
    if kind == "coplanar":
        return np.concatenate([rng.uniform(-1, 1, (n, 2)), np.full((n, 1), 0.5)], axis=1).astype(F32)
    if kind == "cluster":
        p = _wand(n, seed)
        p[: n // 3] = rng.normal(0, 1e-4, (n // 3, 3)) + p[0]
        return p.astype(F32)
    if kind == "far":
        p = _wand(n, seed)
        p[n - n // 5:] = p[n - n // 5:] * 0.1 + [40.0, 0.0, 0.0]
        return p
    return np.repeat(rng.uniform(-1, 1, (max(1, n // 20), 3)), 20, axis=0)[:n].astype(F32)   # "duplicates"


CASES = ([(n, k, "wand") for n in (30, 1000, 20000, 100000) for k in (5, 16, 24, 64) if k < n]
         + [(n, k, kind) for kind in ("line", "coplanar", "cluster", "far", "duplicates")
            for n, k in ((2000, 8), (20000, 24))])


def _run(frame, k):
    out, st, nrm, flags, knn = capi.smooth_points(frame, k, want_terms=True)
    return [out.cpu().numpy(), st, nrm.cpu().numpy(), flags.cpu().numpy(), knn.cpu().numpy()]


@gpu
@pytest.mark.parametrize("n,k,kind", CASES)
def test_kernel_matches_the_oracle_bit_for_bit(n, k, kind):
    pts = _cloud(n, kind, CASES.index((n, k, kind)))
    frame = frame_points(pts, _dev()).contiguous()
    rf = S.frame_map(pts)
    assert np.array_equal(frame.cpu().numpy().view(np.uint32), rf.view(np.uint32))
    got, again = _run(frame, k), _run(frame, k)
    for x, y in zip(got, again):                                 # two calls: identical bits
        assert np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8))
    out, st, nrm, flags, knn = got
    r = S.smooth(rf, k)
    assert np.array_equal(knn, r["knn"])
    assert np.array_equal(nrm.view(np.uint32), r["normals"].view(np.uint32)), np.argwhere(nrm != r["normals"])[:5]
    assert np.array_equal(flags, r["flags"]), np.argwhere(flags != r["flags"])[:5]
    assert np.array_equal(out.view(np.uint32), r["points"].view(np.uint32)), np.argwhere(out != r["points"])[:5]
    assert st.tolist() == r["stats"].tolist()
    if kind in ("line", "duplicates"):
        assert st[0] == 0
    if kind == "duplicates":
        assert np.array_equal(out.view(np.uint32), rf.view(np.uint32))
    pub, pst = smooth_points(pts, k)                             # the public path
    ref, _ = S.smoothed_input(pts, k)
    assert pub.dtype == (torch.float64 if pts.dtype == F64 else torch.float32)
    assert np.array_equal(pub.cpu().numpy(), ref) and (pst.quadratic, pst.singular, pst.far) == tuple(st.tolist())


@gpu
def test_one_million_points_against_the_oracle():
    n, k = 1_000_000, DEFAULT_K
    pts = _wand(n, 11, 0.001).astype(F32)
    frame = frame_points(pts, _dev()).contiguous()
    rf = S.frame_map(pts)
    assert np.array_equal(frame.cpu().numpy().view(np.uint32), rf.view(np.uint32))
    out, st, nrm, flags, knn = _run(frame, k)
    r = S.smooth(rf, k)
    assert np.array_equal(knn, r["knn"])
    assert np.array_equal(nrm.view(np.uint32), r["normals"].view(np.uint32))
    assert np.array_equal(flags, r["flags"]) and st.tolist() == r["stats"].tolist()
    assert np.array_equal(out.view(np.uint32), r["points"].view(np.uint32))
    print(f"1M wand: {st.tolist()} (quadratic, singular, far)")


@gpu
def test_bad_input_raises_before_any_launch():
    dev = _dev()
    ok = torch.rand(100, 3, device=dev) - 0.5
    L = capi.lib()
    bad = [((ok.cpu(),), {}), ((ok.double(),), {}), ((ok[:, :2].contiguous(),), {}), ((ok.t().contiguous().t(),), {}),
           ((ok[:24].contiguous(),), {}), ((ok.cpu().numpy(),), {}),
           ((torch.full((100, 3), float("nan"), device=dev),), {}), ((torch.full((100, 3), float("inf"), device=dev),), {}),
           ((ok,), {"k": 4}), ((ok,), {"k": 0}), ((ok,), {"k": 65}), ((ok,), {"k": 2.5}), ((ok,), {"k": True}),
           ((ok,), {"k": "8"}), ((ok[:8].contiguous(),), {"k": 8})]
    torch.cuda.synchronize()
    before = L.ma_launch_count()
    for args, kw in bad:
        with pytest.raises(ValueError):
            capi.smooth_points(*args, **kw)
    assert L.ma_launch_count() == before
    out, st = capi.smooth_points(ok[:6].contiguous(), 5)          # the edges of every range are accepted
    assert int(st.sum()) == 6
    out, st = capi.smooth_points(ok, 64)
    assert int(st.sum()) == 100


OUT = {"k": 16, "std_ratio": 2.0, "min_component": 0.01}
SMOOTH = {"k": DEFAULT_K}


def _scene_file(tmp_path, kind, seed):
    """Two noisy wands 1.5 apart (two objects at --object_distance 0.02) and a few far strays."""
    a, b = _wand(12000, seed), _wand(12000, seed + 7)
    b[:, 0] += 1.5
    strays = np.random.default_rng(seed).normal(size=(30, 3)) * 4 + [0.7, 0, 3.0]
    pts = np.concatenate([a, b, strays]).astype(F32)
    data = pts if kind == "pc" else np.concatenate([pts, np.tile([[0.0, 0.0, 1.0]], (len(pts), 1))], axis=1)
    np.save(tmp_path / "scene.npy", data.astype(F32))
    return pts


@gpu
@pytest.mark.parametrize("objects", [False, True])
@pytest.mark.parametrize("outliers", [False, True])
@pytest.mark.parametrize("kind", ["pc", "pc_normal"])
def test_dataset_with_smoothing(tmp_path, monkeypatch, kind, outliers, objects):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    pts = _scene_file(tmp_path, kind, 3)
    kw = dict(outliers=OUT if outliers else None, objects={"distance": 0.02} if objects else None)
    np.random.seed(0)
    plain = cli.Dataset(kind, [str(tmp_path / "scene.npy")], **kw)
    np.random.seed(0)
    ds = cli.Dataset(kind, [str(tmp_path / "scene.npy")], smooth=SMOOTH, **kw)
    assert len(ds) == len(plain) == (2 if objects else 1)
    # the oracle chain: rows after outlier removal, smoothed, then the same subset draw as without smoothing
    rows = np.arange(len(pts))
    if outliers:
        rows = rows[OO.remove_outliers(OO.frame_map(pts), **OUT)["kept"]]
    smoothed, _ = S.smoothed_input(pts[rows], DEFAULT_K)
    if objects:
        r = JO.split_objects(JO.frame_map(smoothed), 0.02, 4096)
        parts = [r["indices"][r["offsets"][j]:r["offsets"][j + 1]] for j in range(2)]
    else:
        parts = [np.arange(len(rows))]
    for j, (it, base, part) in enumerate(zip(ds.data, plain.data, parts)):
        raw, ref_raw = it["pc_normal"], base["pc_normal"]
        # the same rows as without smoothing: each smoothed row maps back to its original row
        pick = np.array([np.flatnonzero((smoothed[part] == x).all(axis=1))[0] for x in raw[:, :3]])
        orig = pts[rows][part][pick]
        assert np.array_equal(orig, ref_raw[:, :3])
        assert not np.array_equal(raw[:, :3], ref_raw[:, :3])  # and they moved
        if kind == "pc_normal":
            assert np.array_equal(raw[:, 3:], ref_raw[:, 3:])  # the file's normals pass through
        pc = ds[j]["pc_normal"].astype(F64)
        assert np.all(np.abs(np.linalg.norm(pc[:, 3:], axis=1) - 1) < 2e-3)
        assert abs(np.abs(pc[:, :3]).max() - 0.9995) < 1e-3


@gpu
def test_main_cli_smooth(tmp_path):
    np.save(tmp_path / "scan.npy", _wand(20000, 8).astype(F32))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--out_dir", str(tmp_path / "out"), "--pretrained_weights",
           "synthetic", "--n_max_triangles", "6", "--input_path", str(tmp_path / "scan.npy"), "--smooth"]
    r = subprocess.run(cmd + ["--input_type", "pc"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "scan: smoothed 20000 points (k = 24): " in r.stdout and "(input units)" in r.stdout, r.stdout[-2000:]
    objs = sorted(f for _, _, fs in os.walk(tmp_path / "out") for f in fs if f.endswith(".obj"))
    assert objs == ["scan_gen.obj"]
    r = subprocess.run(cmd + ["--input_type", "mesh"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode != 0 and "point-cloud input" in r.stderr
