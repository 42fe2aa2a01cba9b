"""-m gpu: outlier removal (csrc/outliers.cu) against its numpy restatement (tests/outliers_oracle.py) bit for bit --
keep mask, kept indices, mean distances, mu, sigma, threshold, counts -- the exact kNN of its robust grid at 1M points
with far outliers, bad input refused before any launch, and the pipeline: `Dataset(..., outliers=...)` for `pc` and
`pc_normal`, `main.py --remove_outliers`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from meshanything_b200 import capi, metrics
from meshanything_b200.outliers import remove_outliers
from meshanything_b200.pointcloud import frame_points
from tests import outliers_oracle as O

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64


def _dev():
    return torch.device("cuda", 0)


def _sphere(n, rng, r=1.0):
    x = rng.normal(size=(n, 3))
    return x / np.linalg.norm(x, axis=1, keepdims=True) * r


def _cloud(n, k, seed, kind):
    """float64, offset by 1e4: a sphere of radius 10 with exact duplicates and (n >= 4096) a cluster of thousands of
    points inside one grid cell, whose last points are replaced by `kind`: far single outliers, 1 % scattered in a box
    10x the object, or floater clusters of more than k points.  Small n: uniform points."""
    rng = np.random.default_rng(seed)
    if n < 200:
        return rng.uniform(-10, 10, (n, 3)) + 1e4
    p = _sphere(n, rng, 10.0)
    p[n // 10:n // 10 + n // 20] = p[:n // 20]                                     # exact duplicates
    if n >= 4096:
        c = min(3000, n // 4)
        p[n // 2:n // 2 + c] = p[n // 2] + rng.uniform(-2e-3, 2e-3, (c, 3))         # cluster in one cell
    if kind == "far":
        m = max(1, n // 500)
        p[n - m:] = _sphere(m, rng) * rng.uniform(70, 100, (m, 1))
    elif kind == "scatter":
        m = max(1, n // 100)
        p[n - m:] = rng.uniform(-100, 100, (m, 3))
    else:
        size = max(k + 1, n // 200)
        for f in range(3):
            a = n - (f + 1) * size
            p[a:a + size] = _sphere(1, rng) * 30 + rng.uniform(-0.5, 0.5, (size, 3))
    return p + 1e4


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint8)


CASES = [(n, k, kind) for k in (1, 8, 16, 64) for n in (k + 1, 1000, 4096, 20000) for kind in ("far", "scatter", "floaters")
         if not (n == k + 1 and kind != "far")]


@gpu
@pytest.mark.parametrize("n,k,kind", CASES)
def test_kernel_matches_the_oracle_bit_for_bit(n, k, kind):
    pts = _cloud(n, k, n + 100 * k, kind)
    frame = frame_points(pts, _dev())
    rf = O.frame_map(pts)
    assert np.array_equal(frame.cpu().numpy().view(np.uint32), rf.view(np.uint32))
    mc = 0.01 if kind != "floaters" or n < 4096 else 0.02
    out = [t.cpu().numpy() if isinstance(t, torch.Tensor) else t for t in capi.remove_outliers(frame, k, 2.0, mc, True)]
    again = [t.cpu().numpy() if isinstance(t, torch.Tensor) else t for t in capi.remove_outliers(frame, k, 2.0, mc, True)]
    out[2], again[2] = out[2][:7], again[2][:7]                        # stats[7], the round count, is schedule's
    for x, y in zip(out, again):                                       # two calls: identical bits
        assert np.array_equal(_bits(x), _bits(y))
    idx, keep, st, mean, knn = out
    r = O.remove_outliers(rf, k, 2.0, mc)
    assert np.array_equal(knn, r["knn"]), np.argwhere(knn != r["knn"])[:5]
    assert np.array_equal(_bits(mean), _bits(r["mean_dist"])), np.argwhere(mean != r["mean_dist"])[:5]
    assert _bits(st[:3]).tobytes() == _bits(np.array([r["mu"], r["sigma"], r["threshold"]], F64)).tobytes()
    assert np.array_equal(keep, r["keep"]) and np.array_equal(idx, r["kept"])
    assert (int(st[3]), int(st[4]), int(st[5]), int(st[6])) == (r["inliers"], r["components"], r["dropped"], r["n_kept"])
    if kind == "far" and n >= 1000:
        assert not keep[n - max(1, n // 500):].any()                  # every far point goes
    pub, pst = remove_outliers(pts, k, 2.0, mc)                        # the public path
    assert np.array_equal(pub.cpu().numpy(), r["kept"]) and pst.kept == r["n_kept"]


@gpu
def test_identical_points_and_min_component_zero():
    z = torch.zeros((300, 3), device=_dev())
    idx, keep, st = capi.remove_outliers(z, 16, 2.0, 0.01)
    assert bool(keep.all()) and len(idx) == 300 and st[1] == 0 and st[4] == 1
    pts = _cloud(4096, 16, 7, "floaters")
    rf = O.frame_map(pts)
    idx, keep, st = capi.remove_outliers(frame_points(pts, _dev()), 16, 2.0, 0.0)
    r = O.remove_outliers(rf, 16, 2.0, 0.0)
    assert np.array_equal(idx.cpu().numpy(), r["kept"]) and st[4] == 0 and st[5] == 0


@gpu
def test_one_million_points_with_far_outliers_exact_knn():
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    v, f = torch.from_numpy(z["vertices"]).to(_dev()), torch.from_numpy(z["faces"]).to(_dev())
    n, k, m = 1_000_000, 16, 10_000
    xyz = capi.sample_surface(v, f, n - m, seed=11)[:, :3].float()
    lo, hi = xyz.amin(0), xyz.amax(0)
    g = torch.Generator(device=_dev()).manual_seed(5)
    far = (lo + hi) / 2 + (torch.rand(m, 3, device=_dev(), generator=g) - 0.5) * 10 * (hi - lo).max()
    frame = metrics.to_output_frame(torch.cat([xyz, far])[None])[0].contiguous()
    idx, keep, st, mean, knn = capi.remove_outliers(frame, k, 2.0, 0.01, want_terms=True)
    rng = np.random.default_rng(0)
    q = torch.from_numpy(np.concatenate([rng.choice(n - m, 1500, replace=False),
                                         n - m + rng.choice(m, 500, replace=False)])).to(_dev())
    for part in q.split(250):
        d = frame[part][:, None, :] - frame[None, :, :]
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        d2[torch.arange(len(part), device=d2.device), part] = float("inf")
        ref = torch.sort(d2, dim=1, stable=True).indices[:, :k]     # ties: lowest index first
        assert torch.equal(knn[part].long(), ref)
    assert int(keep[n - m:].sum()) < m // 100                           # nearly every far point goes
    assert int(keep[:n - m].sum()) > 0.97 * (n - m)
    print(f"1M + 1 % far: kept {int(st[6])}, {int(st[4])} components, {int(st[7])} rounds")


@gpu
def test_bad_input_raises_before_any_launch():
    dev = _dev()
    ok = torch.rand(100, 3, device=dev) - 0.5
    L = capi.lib()
    bad = [((ok.cpu(),), {}), ((ok.double(),), {}), ((ok[:, :2].contiguous(),), {}), ((ok.t().contiguous().t(),), {}),
           ((ok[:16].contiguous(),), {}), ((ok.cpu().numpy(),), {}),
           ((torch.full((100, 3), float("nan"), device=dev),), {}), ((torch.full((100, 3), float("inf"), device=dev),), {}),
           ((ok,), {"k": 0}), ((ok,), {"k": 65}), ((ok,), {"k": 2.5}), ((ok,), {"k": True}),
           ((ok,), {"std_ratio": float("inf")}), ((ok,), {"min_component": -0.1})]
    torch.cuda.synchronize()
    before = L.ma_launch_count()
    for args, kw in bad:
        with pytest.raises(ValueError):
            capi.remove_outliers(*args, **kw)
    assert L.ma_launch_count() == before
    capi.remove_outliers(ok[:65].contiguous(), k=64)  # the edges of every range are accepted


def _stray_sphere(seed, n=8000, strays=20):
    rng = np.random.default_rng(seed)
    s = _sphere(n, rng)
    far = _sphere(strays, rng) * rng.uniform(7, 10, (strays, 1))
    return np.concatenate([s, far]).astype(F32), s


OUT = {"k": 16, "std_ratio": 2.0, "min_component": 0.01}


@gpu
def test_dataset_pc_with_outliers(tmp_path, monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    pts, _ = _stray_sphere(1)
    np.save(tmp_path / "scan.npy", pts)
    idx, st = remove_outliers(pts, **OUT)
    assert int(idx.max()) < 8000 and st.removed_statistical + st.removed_components >= 20
    np.random.seed(0)
    pc = cli.Dataset("pc", [str(tmp_path / "scan.npy")], outliers=OUT)[0]["pc_normal"].astype(F64)
    xyz, nrm = pc[:, :3], pc[:, 3:]
    assert pc.shape == (4096, 6)
    assert np.all(np.abs(np.linalg.norm(nrm, axis=1) - 1) < 2e-3)
    assert ((nrm * xyz).sum(axis=1) > 0).mean() >= 0.99
    r = np.linalg.norm(xyz, axis=1)
    assert r.max() < 1.01 and r.min() > 0.95                            # surface points only: the strays are gone
    assert abs(np.abs(xyz).max() - 0.9995) < 1e-3                       # and the surface fills the frame
    np.random.seed(0)                                                   # without the flag: the unchanged path
    plain = cli.Dataset("pc", [str(tmp_path / "scan.npy")])[0]["pc_normal"]
    np.random.seed(0)
    assert np.array_equal(plain, cli.Dataset("pc", [str(tmp_path / "scan.npy")], outliers=None)[0]["pc_normal"])


@gpu
def test_dataset_pc_normal_with_outliers(tmp_path, monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    pts, s = _stray_sphere(2)
    rng = np.random.default_rng(3)
    nrm = np.concatenate([s, _sphere(len(pts) - len(s), rng)]).astype(F32)
    np.save(tmp_path / "scan.npy", np.concatenate([pts, nrm], axis=1))
    np.random.seed(0)
    pc = cli.Dataset("pc_normal", [str(tmp_path / "scan.npy")], outliers=OUT)[0]["pc_normal"].astype(F64)
    r = np.linalg.norm(pc[:, :3], axis=1)
    assert r.max() < 1.01 and r.min() > 0.95
    few = np.concatenate([pts[:5000], nrm[:5000]], axis=1)              # too few points left: a clear error
    few[:2000, :3] = _sphere(2000, rng) * 50
    np.save(tmp_path / "few.npy", few)
    with pytest.raises(ValueError, match="remain after outlier removal"):
        cli.Dataset("pc_normal", [str(tmp_path / "few.npy")], outliers=dict(OUT, min_component=0.5))


@gpu
def test_main_cli_remove_outliers(tmp_path):
    pts, _ = _stray_sphere(4)
    np.save(tmp_path / "scan.npy", pts)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--out_dir", str(tmp_path / "out"),
                        "--pretrained_weights", "synthetic", "--n_max_triangles", "6", "--input_type", "pc",
                        "--input_path", str(tmp_path / "scan.npy"), "--remove_outliers"], cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "scan: removed" in r.stdout and " kept" in r.stdout, r.stdout[-2000:]
    objs = sorted(f for _, _, fs in os.walk(tmp_path / "out") for f in fs if f.endswith(".obj"))
    assert objs == ["scan_gen.obj"]
