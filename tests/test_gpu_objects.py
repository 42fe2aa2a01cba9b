"""-m gpu: object splitting (csrc/objects.cu) against its numpy restatement (tests/objects_oracle.py) bit for bit --
labels, object indices, offsets and every stat, two calls identical -- at 1M points, bad input refused before any
launch, and the pipeline: `Dataset(..., plane=..., objects=...)` for `pc` and `pc_normal`, `--output_frame input`,
`main.py --remove_plane --split_objects --output_frame input`."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from meshanything_b200 import capi
from meshanything_b200.objects import split_objects
from meshanything_b200.pointcloud import frame_points
from tests import objects_oracle as O
from tests import outliers_oracle as OO
from tests import plane_oracle as P
from tests import subsample_oracle as SO

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64
CORNERS = np.array([[-0.5, -0.5, -0.5], [0.5, 0.5, 0.5]])


def _dev():
    return torch.device("cuda", 0)


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint8)


def _cloud(n, kind, eps, seed):
    """(points, labels the oracle may take instead of building the graph, or None)."""
    rng = np.random.default_rng(seed)
    if kind == "scene":                                          # float64 offset by 1e4, with exact duplicates
        p, _ = O.table_scene(seed, n=max(n, 1000))
        p = p[rng.permutation(len(p))[:n]]
        if n >= 50:
            p[n // 7:n // 7 + n // 50] = p[:n // 50]
        return p + 1e4, None
    if kind == "grid":                                           # the 1/64 grid: pairs at exactly d^2 = e2
        g = rng.integers(-32, 33, (n, 3)) / 64
        g[:2] = CORNERS
        return g.astype(F32), None
    if kind == "helix":                                          # one chain of points 0.9 e apart through many cells
        r, ds = 0.45, 0.9 * eps
        turns = n * ds / (2 * np.pi * r)
        th = np.arange(n) * ds / np.hypot(r, 1 / (2 * np.pi * turns))
        z = th / (2 * np.pi * turns) - 0.5
        return np.stack([r * np.cos(th), r * np.sin(th), z], axis=1).astype(F32), None
    if kind == "ball":                                           # every pair within 0.9 e, two far corners
        x = rng.normal(size=(n - 2, 3))
        b = x / np.linalg.norm(x, axis=1, keepdims=True) * (0.45 * eps * rng.random((n - 2, 1)) ** (1 / 3))
        p = np.concatenate([CORNERS, b]).astype(F32)
        lab = np.full(n, 2, np.int32)
        lab[:2] = [0, 1]
        return p, (lab if eps < 0.4 else np.zeros(n, np.int32))   # at e = 1 the ball reaches both corners
    if kind == "capped":                                         # a few e wide: cells capped at 2^-20, wider than e / 2
        u = (rng.random((n - 2, 3)) - 0.5) * 6 * eps             # spread points: cells that are not cliques
        clump = rng.random(n - 2) < 0.5                          # tight clumps: cells that are
        centre = (rng.random((40, 3)) - 0.5) * 6 * eps
        u[clump] = centre[rng.integers(40, size=int(clump.sum()))] + rng.normal(0, 0.05 * eps, (int(clump.sum()), 3))
        return np.concatenate([CORNERS, u]).astype(F32), None
    p = np.tile([[0.5, -0.25, 2.0]], (n, 1)).astype(F32)         # identical
    return p, np.zeros(n, np.int32)


CASES = ([(n, e, "scene") for n in (1, 2, 4096, 20000, 100000) for e in (1e-4, 0.005, 0.02)]
         + [(4096, 0.1, "scene"), (20000, 0.1, "scene"), (4096, 1.0, "scene"), (20000, 1e-6, "scene"),
            (20000, 1 / 64, "grid"), (20000, 0.005, "helix"), (100000, 1e-4, "helix"),
            (50000, 1e-4, "ball"), (50000, 0.02, "ball"), (50000, 0.1, "ball"), (50000, 1.0, "ball"),
            (20000, 1e-4, "identical"), (20000, 1.0, "identical"), (3000, 1e-6, "capped"), (8000, 1.5e-6, "capped")])


def cell_census(p, eps):
    """The cells of section 1.7's grid, restated (fp64 keys, the fp32 box test): (cells that are not cliques, clique
    cells holding two distinct points, clique cells with a non-clique cell in their 5^3 block)."""
    p = np.asarray(p, F32)
    e = F32(eps)
    e2 = F32(e * e)
    lo, hi = p.min(0).astype(F64), p.max(0).astype(F64)
    h = max(float(e) * (1.0 + 1e-5) / 2, float((hi - lo).max()) / (1 << 20))
    cell = np.clip(np.floor((p.astype(F64) - lo) * (1.0 / h)), 0, (1 << 21) - 1).astype(np.int64)
    keys, inv = np.unique(cell, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    bmin = np.full((len(keys), 3), np.inf, F32)
    bmax = np.full((len(keys), 3), -np.inf, F32)
    np.minimum.at(bmin, inv, p)
    np.maximum.at(bmax, inv, p)
    x = bmax - bmin
    clique = (x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2] <= e2
    distinct = (bmax > bmin).any(axis=1)
    bad = {tuple(k) for k in keys[~clique]}
    mixed = sum(any(tuple(k + d) in bad for d in np.stack(np.meshgrid(*[np.arange(-2, 3)] * 3, indexing="ij"),
                                                              -1).reshape(-1, 3)) for k in keys[clique])
    return int((~clique).sum()), int((clique & distinct).sum()), int(mixed)


@gpu
@pytest.mark.parametrize("min_points", [1, 4096])
@pytest.mark.parametrize("n,eps,kind", CASES)
def test_kernel_matches_the_oracle_bit_for_bit(n, eps, kind, min_points):
    mp = min(min_points, n)
    pts, lab = _cloud(n, kind, eps, CASES.index((n, eps, kind)))
    frame = frame_points(pts, _dev()).contiguous()
    rf = O.frame_map(pts)
    assert np.array_equal(frame.cpu().numpy().view(np.uint32), rf.view(np.uint32))
    if kind == "ball":
        assert np.abs(rf[2:]).max() < 0.45 * eps * 1.01
    out = [x.cpu().numpy() if isinstance(x, torch.Tensor) else x for x in capi.split_objects(frame, eps, mp)]
    again = [x.cpu().numpy() if isinstance(x, torch.Tensor) else x for x in capi.split_objects(frame, eps, mp)]
    for x, y in zip(out, again):                                 # two calls: identical bits
        assert np.array_equal(_bits(x), _bits(y))
    labels, idx, off, st = out
    r = O.split_objects(rf, eps, mp, labels=lab)
    assert np.array_equal(labels, r["labels"]), np.argwhere(labels != r["labels"])[:5]
    assert np.array_equal(st, r["stats"]), (st, r["stats"])
    assert np.array_equal(off, r["offsets"]) and np.array_equal(idx, r["indices"])
    if kind == "helix":
        assert r["stats"][0] == 1
    if kind == "capped":                                         # the per-point path: within cells and across
        assert all(c > 0 for c in cell_census(rf, eps)), cell_census(rf, eps)
    pub_idx, pub_off, pst = split_objects(pts, eps, mp)         # the public path
    assert np.array_equal(pub_idx.cpu().numpy(), r["indices"]) and np.array_equal(pub_off.cpu().numpy(), r["offsets"])
    assert pst.clusters == r["stats"][0] and pst.sizes == tuple(np.diff(r["offsets"]))


@gpu
def test_one_million_points_labels_equal_the_oracle():
    pts, _ = O.table_scene(9, n=1_000_000)
    eps = 0.003
    frame = frame_points(pts, _dev()).contiguous()
    labels, idx, off, st = capi.split_objects(frame, eps, 4096)
    r = O.split_objects(O.frame_map(pts), eps, 4096)
    assert np.array_equal(labels.cpu().numpy(), r["labels"])
    assert np.array_equal(st, r["stats"]) and np.array_equal(idx.cpu().numpy(), r["indices"])
    print(f"1M scene at e = {eps}: stats {st.tolist()}")


@gpu
def test_bad_input_raises_before_any_launch():
    dev = _dev()
    ok = torch.rand(100, 3, device=dev) - 0.5
    L = capi.lib()
    bad = [((ok.cpu(),), {}), ((ok.double(),), {}), ((ok[:, :2].contiguous(),), {}), ((ok.t().contiguous().t(),), {}),
           ((ok[:0].contiguous(),), {}), ((ok.cpu().numpy(),), {}),
           ((torch.full((10, 3), float("nan"), device=dev),), {}), ((torch.full((10, 3), float("inf"), device=dev),), {}),
           ((ok,), {"distance": 0.0}), ((ok,), {"distance": -0.1}), ((ok,), {"distance": 1.5}),
           ((ok,), {"distance": float("nan")}), ((ok,), {"distance": 1e-50}), ((ok,), {"distance": 1e-25}),
           ((ok,), {"distance": "x"}), ((ok,), {"distance": True}), ((ok,), {"min_points": 0}),
           ((ok,), {"min_points": 101}), ((ok,), {"min_points": 2.5}), ((ok,), {"min_points": True})]
    torch.cuda.synchronize()
    before = L.ma_launch_count()
    for args, kw in bad:
        with pytest.raises(ValueError):
            capi.split_objects(*args, **kw)
    assert L.ma_launch_count() == before
    labels, idx, off, st = capi.split_objects(ok, 1.0, 100)      # the edges of every range are accepted
    assert st[0] == 1 and np.array_equal(off.cpu().numpy(), [0, 100])


PLANE = {"distance": 0.01, "iterations": 1000}
OUT = {"k": 16, "std_ratio": 2.0, "min_component": 0.01}
OBJ = {"distance": 0.02}


def _scene_file(tmp_path, kind, seed):
    pts, lab = O.table_scene(seed)
    data = pts if kind == "pc" else np.concatenate([pts, np.tile([[0.0, 0.0, 1.0]], (len(pts), 1))], axis=1)
    np.save(tmp_path / "scene.npy", data.astype(F32))
    return pts.astype(F32).astype(F64), lab


@gpu
@pytest.mark.parametrize("subsample", ["random", "fps"])
@pytest.mark.parametrize("outliers", [False, True])
@pytest.mark.parametrize("kind", ["pc", "pc_normal"])
def test_dataset_with_object_split(tmp_path, monkeypatch, kind, outliers, subsample):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    pts, lab = _scene_file(tmp_path, kind, 11 + outliers)
    np.random.seed(0)
    ds = cli.Dataset(kind, [str(tmp_path / "scene.npy")], plane=PLANE, outliers=OUT if outliers else None,
                     subsample=subsample, objects=OBJ)
    assert [d["uid"] for d in ds.data] == ["scene_obj0", "scene_obj1", "scene_obj2"]
    np.random.seed(0)                                            # the oracle chain under the same seed
    seed = int(np.random.randint(0, 2**62, dtype=np.int64))
    rows = P.remove_plane(P.frame_map(pts.astype(F32)), seed=seed, **PLANE)["kept"]
    if outliers:
        rows = rows[OO.remove_outliers(OO.frame_map(pts[rows].astype(F32)), **OUT)["kept"]]
    r = O.split_objects(O.frame_map(pts[rows].astype(F32)), min_points=4096, **OBJ)
    assert r["stats"][1] == 3
    kinds = set()
    for k in range(3):
        obj = rows[r["indices"][r["offsets"][k]:r["offsets"][k + 1]]]
        if subsample == "fps":
            pick, _ = SO.farthest_point_sample(OO.frame_map(pts[obj].astype(F32)), 4096, np.random.randint(len(obj)))
        else:
            pick = np.random.choice(len(obj), 4096, replace=False)
        sel = obj[pick]
        raw = ds.data[k]["pc_normal"].astype(F64)
        assert np.array_equal(raw[:, :3], pts[sel].astype(F32)), k
        kinds |= set(np.unique(lab[sel]).tolist())
        item = ds[k]
        pc = item["pc_normal"].astype(F64)
        assert np.all(np.abs(np.linalg.norm(pc[:, 3:], axis=1) - 1) < 2e-3)
        assert abs(np.abs(pc[:, :3]).max() - 0.9995) < 1e-3
        centre, side = item["frame"]
        lo, hi = raw[:, :3].min(0), raw[:, :3].max(0)
        assert np.array_equal(centre.numpy(), (lo + hi) / 2) and side == (hi - lo).max()
    assert kinds == {1, 2, 3}                                    # one object each: the sphere, the wand, the cube


@gpu
def test_output_frame_input_places_every_vertex(tmp_path, monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    from MeshAnything.models.meshanything import MeshAnything
    from meshanything_b200 import checkpoint as ck
    from meshanything_b200 import metrics
    pts, _ = _scene_file(tmp_path, "pc", 13)
    np.random.seed(0)
    ds = cli.Dataset("pc", [str(tmp_path / "scene.npy")], plane=PLANE, objects=OBJ)
    args = argparse.Namespace(llm="facebook/opt-350m", codebook_size=8192, codebook_dim=1024, n_max_triangles=24,
                              seed=0)
    model = MeshAnything(args)
    model.load_state_dict(ck.synthetic_state_dict(0), strict=True, device=_dev())
    items = [ds[i] for i in range(len(ds))]
    out = model(torch.from_numpy(np.stack([it["pc_normal"] for it in items])))
    for it, mesh in zip(items, out):
        mesh = mesh[~torch.isnan(mesh[:, 0, 0])]
        placed = metrics.to_input_frame(mesh, it["frame"]).cpu().numpy()
        centre, side = it["frame"]
        c = centre.numpy()
        v = mesh.cpu().numpy().astype(F64)
        assert np.array_equal(placed, c + side * v)
        assert len(v) and np.all(np.abs(placed - c) <= side / 2 * (1 + 1e-12))


@gpu
@pytest.mark.parametrize("continuous", [False, True])
def test_main_cli_split_objects(tmp_path, continuous):
    pts, lab = O.table_scene(14)
    np.save(tmp_path / "scene.npy", pts.astype(F32))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--out_dir", str(tmp_path / "out"), "--pretrained_weights",
           "synthetic", "--n_max_triangles", "6", "--input_path", str(tmp_path / "scene.npy"), "--remove_plane",
           "--split_objects", "--output_frame", "input", "--batchsize_per_gpu", "2"]
    if continuous:
        cmd.append("--continuous_batching")
    r = subprocess.run(cmd + ["--input_type", "pc"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "scene: " in r.stdout and " 3 objects of " in r.stdout, r.stdout[-2000:]
    objs = sorted(os.path.join(d, f) for d, _, fs in os.walk(tmp_path / "out") for f in fs if f.endswith(".obj"))
    assert [os.path.basename(f) for f in objs] == [f"scene_obj{k}_gen.obj" for k in range(3)]
    boxes = []
    for k in (1, 2, 3):                                          # each object's cube in scan units, widened by 0.05
        p = pts[lab == k]                                        # for the shift of its 4096-point subset's cube
        boxes.append(((p.min(0) + p.max(0)) / 2, (p.max(0) - p.min(0)).max()))
    for f in objs:
        v = np.array([[float(x) for x in line.split()[1:4]] for line in open(f) if line.startswith("v ")])
        assert len(v)
        inside = [np.all(np.abs(v - c) <= L / 2 + 0.05) for c, L in boxes]
        assert sum(inside) == 1, f
    r = subprocess.run(cmd + ["--input_type", "mesh"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode != 0 and "point-cloud input" in r.stderr
