"""-m gpu: plane removal (csrc/plane.cu) against its numpy restatement (tests/plane_oracle.py) bit for bit -- every
hypothesis's plane and count, the refit plane, the keep mask, the kept indices and every stat -- every count at 1M
points against a chunked torch brute force, bad input refused before any launch, and the pipeline:
`Dataset(..., plane=...)` for `pc` and `pc_normal` with and without outlier removal, `main.py --remove_plane`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from meshanything_b200 import capi
from meshanything_b200.pointcloud import frame_points
from meshanything_b200.plane import remove_plane
from tests import outliers_oracle as OO
from tests import plane_oracle as P

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64
SEEDS = (0, (1 << 32) + 7, (1 << 64) - 1)


def _dev():
    return torch.device("cuda", 0)


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint8)


def _grid_cloud(n):
    """Points on a 1/64 grid in the planes z = 0, +-t, +-2t (t = 1/64): |s| = t exactly for a fifth of them."""
    rng = np.random.default_rng(n)
    xy = rng.integers(-32, 33, (n, 2)) / 64
    xy[:2] = [[-0.5, -0.5], [0.5, 0.5]]                          # the frame map stays the identity
    z = rng.choice([0, 0, 1, -1, 2, -2], n) / 64
    return np.concatenate([xy, z[:, None]], axis=1).astype(F32)


def _cloud(n, kind, seed):
    rng = np.random.default_rng(seed)
    if n == 3:
        return rng.uniform(-1, 1, (3, 3)) + 1e4
    if kind == "scene":                                          # float64 offset by 1e4, with exact duplicates
        p, _, _ = P.table_scene(seed, n=n)
        p[n // 7:n // 7 + n // 50] = p[:n // 50]
        return p + 1e4
    if kind == "collinear":
        return np.stack([rng.uniform(-1, 1, n), np.full(n, 0.25), np.full(n, 3.0)], axis=1).astype(F32)
    if kind == "identical":
        return np.tile([[0.5, -0.25, 2.0]], (n, 1)).astype(F32)
    return _grid_cloud(n)


CASES = ([(n, h, "scene") for n in (3, 1000, 4096, 20000, 100000) for h in (1, 64, 1000, 4097)]
         + [(n, h, kind) for kind in ("collinear", "identical", "grid") for n, h in ((1000, 64), (20000, 1000))])


@gpu
@pytest.mark.parametrize("n,h,kind", CASES)
def test_kernel_matches_the_oracle_bit_for_bit(n, h, kind):
    i = CASES.index((n, h, kind))
    seed = SEEDS[i % 3]
    pts = _cloud(n, kind, i)
    frame = frame_points(pts, _dev()).contiguous()
    rf = P.frame_map(pts)
    assert np.array_equal(frame.cpu().numpy().view(np.uint32), rf.view(np.uint32))
    t = 1 / 64 if kind == "grid" else 0.01
    out = [x.cpu().numpy() if isinstance(x, torch.Tensor) else x for x in capi.remove_plane(frame, t, h, seed, True)]
    again = [x.cpu().numpy() if isinstance(x, torch.Tensor) else x for x in capi.remove_plane(frame, t, h, seed, True)]
    for x, y in zip(out, again):                                 # two calls: identical bits
        assert np.array_equal(_bits(x), _bits(y))
    idx, keep, st, counts, planes = out
    r = P.remove_plane(rf, t, h, seed)
    assert np.array_equal(planes.view(np.uint32), r["planes"].view(np.uint32)), np.argwhere(planes != r["planes"])[:5]
    assert np.array_equal(counts, r["counts"]), np.argwhere(counts != r["counts"])[:5]
    assert np.array_equal(_bits(st), _bits(r["stats"])), (st, r["stats"])
    assert np.array_equal(keep, r["keep"]) and np.array_equal(idx, r["kept"])
    if kind in ("collinear", "identical"):
        assert not r["found"] and keep.all()
    if kind == "grid":
        assert r["found"] and abs(float(r["plane"][2])) > 0.999
    if kind == "scene" and n >= 4096 and h >= 64:
        assert r["found"] and r["plane"][2] > 0.999
    pub, pst = remove_plane(pts, t, h, seed)                     # the public path
    assert np.array_equal(pub.cpu().numpy(), r["kept"]) and pst.kept == r["n_kept"] and pst.found == r["found"]


@gpu
def test_one_million_points_every_count_against_torch():
    n, h, seed, t = 1_000_000, 1000, 77, 0.01
    pts, lab, _ = P.table_scene(3, n=n)
    frame = frame_points(pts, _dev()).contiguous()
    rf = P.frame_map(pts)
    assert np.array_equal(frame.cpu().numpy().view(np.uint32), rf.view(np.uint32))
    idx, keep, st, counts, planes = capi.remove_plane(frame, t, h, seed, want_terms=True)
    ref_planes, _ = P.hypotheses(rf, h, seed)
    assert np.array_equal(planes.cpu().numpy().view(np.uint32), ref_planes.view(np.uint32))
    px, py, pz = frame[:, 0], frame[:, 1], frame[:, 2]
    ref = torch.empty(h, dtype=torch.int64, device=_dev())
    for s in range(0, h, 16):                                    # separate elementwise ops: nothing is contracted
        pl = planes[s:s + 16]
        a = pl[:, 0:1] * px
        b = pl[:, 1:2] * py
        c = pl[:, 2:3] * pz
        d = ((a + b) + c) + pl[:, 3:4]
        ref[s:s + 16] = (d.abs() <= t).sum(dim=1)
    assert torch.equal(counts.long(), ref)
    r = P.remove_plane(rf, t, h, seed, planes=ref_planes, hyp_counts=ref.cpu().numpy())
    assert np.array_equal(_bits(st), _bits(r["stats"]))
    assert np.array_equal(keep.cpu().numpy(), r["keep"]) and np.array_equal(idx.cpu().numpy(), r["kept"])
    k = keep.cpu().numpy()
    assert not k[lab == 2].any() and k[lab == 1].mean() > 0.9 and not k[lab == 0].mean() > 0.001
    print(f"1M scene: winner {int(st[5])} with {int(st[6])} points, on {int(st[8])}, below {int(st[10])}, "
          f"kept {int(st[11])}")


@gpu
def test_bad_input_raises_before_any_launch():
    dev = _dev()
    ok = torch.rand(100, 3, device=dev) - 0.5
    L = capi.lib()
    bad = [((ok.cpu(),), {}), ((ok.double(),), {}), ((ok[:, :2].contiguous(),), {}), ((ok.t().contiguous().t(),), {}),
           ((ok[:2].contiguous(),), {}), ((ok.cpu().numpy(),), {}),
           ((torch.full((10, 3), float("nan"), device=dev),), {}), ((torch.full((10, 3), float("inf"), device=dev),), {}),
           ((ok,), {"distance": 0.0}), ((ok,), {"distance": -0.1}), ((ok,), {"distance": 1.5}),
           ((ok,), {"distance": float("nan")}), ((ok,), {"distance": 1e-50}), ((ok,), {"distance": "x"}),
           ((ok,), {"iterations": 0}), ((ok,), {"iterations": 65537}), ((ok,), {"iterations": 2.5}),
           ((ok,), {"iterations": True}), ((ok,), {"seed": -1}), ((ok,), {"seed": 1 << 64}), ((ok,), {"seed": 1.0})]
    torch.cuda.synchronize()
    before = L.ma_launch_count()
    for args, kw in bad:
        with pytest.raises(ValueError):
            capi.remove_plane(*args, **kw)
    assert L.ma_launch_count() == before
    idx, keep, st = capi.remove_plane(ok, 1.0, 1, (1 << 64) - 1)  # the edges of every range are accepted
    assert st[0] in (0.0, 1.0)


OUT = {"k": 16, "std_ratio": 2.0, "min_component": 0.01}
PLANE = {"distance": 0.01, "iterations": 1000}


def _scene_file(tmp_path, kind, outliers, seed):
    pts, lab, t = P.table_scene(seed, n=20000)
    above = (lab == 3) & (pts[:, 2] > -t)
    if outliers:                                                 # strays above the table: far from the object, as
        rng = np.random.default_rng(seed)                        # outlier removal defines them (a stray touching the
        d = rng.normal(size=(int(above.sum()), 3))               # sphere joins its component and is kept)
        d[:, 2] = np.abs(d[:, 2])
        pts[above] = [0, 0, 0.5] + d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(3, 4, (len(d), 1))
    else:                                                        # they would stretch the frame
        pts, lab = pts[~above], lab[~above]
    data = pts if kind == "pc" else np.concatenate([pts, np.tile([[0.0, 0.0, 1.0]], (len(pts), 1))], axis=1)
    np.save(tmp_path / "scene.npy", data.astype(F32))
    return pts.astype(F32).astype(F64), lab, t


@gpu
@pytest.mark.parametrize("outliers", [False, True])
@pytest.mark.parametrize("kind", ["pc", "pc_normal"])
def test_dataset_with_plane_removal(tmp_path, monkeypatch, kind, outliers):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    pts, lab, t = _scene_file(tmp_path, kind, outliers, 5 + outliers)
    np.random.seed(0)
    ds = cli.Dataset(kind, [str(tmp_path / "scene.npy")], plane=PLANE, outliers=OUT if outliers else None)
    raw = ds.data[0]["pc_normal"].astype(F64)
    np.random.seed(0)                                            # the oracle's rows under the same seed
    seed = int(np.random.randint(0, 2**62, dtype=np.int64))
    r = P.remove_plane(P.frame_map(pts.astype(F32)), seed=seed, **PLANE)
    rows = r["kept"]
    if outliers:
        rows = rows[OO.remove_outliers(OO.frame_map(pts[rows].astype(F32)), **OUT)["kept"]]
    rows = rows[np.random.choice(len(rows), 4096, replace=False)]
    assert np.array_equal(raw[:, :3], pts[rows].astype(F32))
    assert pts[rows, 2].min() >= -t                              # nothing below the table remains
    pc = ds[0]["pc_normal"].astype(F64)
    xyz, nrm = pc[:, :3], pc[:, 3:]
    assert np.all(np.abs(np.linalg.norm(nrm, axis=1) - 1) < 2e-3)
    assert abs(np.abs(xyz).max() - 0.9995) < 1e-3
    far = np.abs(xyz).max(axis=1) > 0.999
    assert np.all(lab[rows[far]] == 1), lab[rows[far]]           # the frame is the object's, not the table's
    print(f"{kind}, outliers={outliers}: kept {r['n_kept']} of {len(pts)}; rows from the object "
          f"{(lab[rows] == 1).mean():.3f}")


@gpu
def test_main_cli_remove_plane(tmp_path):
    pts, _, t = P.table_scene(8, n=20000)
    keep = ~((np.arange(len(pts)) >= len(pts) - 200) & (pts[:, 2] > -t))       # strays only below the table
    np.save(tmp_path / "scene.npy", pts[keep].astype(F32))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--out_dir", str(tmp_path / "out"), "--pretrained_weights",
           "synthetic", "--n_max_triangles", "6", "--input_path", str(tmp_path / "scene.npy"), "--remove_plane"]
    r = subprocess.run(cmd + ["--input_type", "pc"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "scene: plane n = (" in r.stdout and " kept" in r.stdout, r.stdout[-2000:]
    objs = sorted(f for _, _, fs in os.walk(tmp_path / "out") for f in fs if f.endswith(".obj"))
    assert objs == ["scene_gen.obj"]
    r = subprocess.run(cmd + ["--input_type", "mesh"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode != 0 and "point-cloud input" in r.stderr
