"""-m gpu: colour transfer (csrc/colors.cu) against its numpy restatement (tests/colors_oracle.py) bit for bit -- the
nearest faces, distances, weights, integer sums, colours, fallback flags and stats, two calls identical -- over a grid
of (N, F) with hard meshes and clouds and at 1M points, bad input refused before any launch, and the pipeline:
`Dataset(..., colors=True)` through plane, outlier removal, smoothing and splitting, and `main.py --transfer_colors`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from meshanything_b200 import capi
from meshanything_b200.colors import frame, transfer_colors
from tests import colors_oracle as CO

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64


def _dev():
    return torch.device("cuda", 0)


def sphere_mesh(F, seed):
    """F faces of a latitude-longitude sphere of radius 0.5 (float64), with a duplicate face, a face repeating a vertex
    index, a face of one vertex and a collinear face among them once F allows."""
    n = max(3, int(np.ceil(np.sqrt(F / 2))) + 1)
    th, ph = np.meshgrid(np.linspace(0.05, np.pi - 0.05, n), np.linspace(0, 2 * np.pi, n, endpoint=False),
                         indexing="ij")
    v = 0.5 * np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1).reshape(-1, 3)
    idx = np.arange(n * n).reshape(n, n)
    a, b = idx[:-1], np.roll(idx, -1, axis=1)[:-1]
    c, d = idx[1:], np.roll(idx, -1, axis=1)[1:]
    f = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([b, d, c], -1).reshape(-1, 3)])
    f = f[np.random.default_rng(seed).permutation(len(f))][:F].copy()
    v = np.concatenate([v, [[0.1, 0.1, 0.1], [0.2, 0.2, 0.2], [0.3, 0.3, 0.3]]])     # three collinear vertices
    m = len(v)
    hard = [f[0], [f[0][0], f[0][0], f[0][1]], [f[0][2]] * 3, [m - 3, m - 2, m - 1]]
    for k, h in enumerate(hard):
        if F > 4 * (k + 1):
            f[F // 5 * (k + 1)] = h
    return v, f


def scan(N, v, f, seed, offset=0.0):
    """N points: most near the mesh's surface with noise, some exactly on vertices and on edge midpoints, a few far;
    random colours in [0, 1]."""
    rng = np.random.default_rng(seed)
    t = v[f[rng.integers(0, len(f), N)]]
    r = rng.dirichlet([1, 1, 1], N)
    p = np.einsum("nk,nkd->nd", r, t) + rng.normal(0, 0.01, (N, 3))
    k = N // 10
    if k:
        p[:k] = v[f[rng.integers(0, len(f), k), 0]]
        p[k:2 * k] = 0.5 * (v[f[rng.integers(0, len(f), k), 0]] + v[f[rng.integers(0, len(f), k), 1]])
        p[2 * k:3 * k] += rng.normal(0, 0.3, (k, 3))
    c = rng.uniform(0, 1, (N, 3)).astype(F32)
    c[rng.random(N) < 0.05] = 1.0
    return p + offset, c


def _check(v, f, p, c, r=0.05):
    dev = _dev()
    fp, fv = frame(p, v, dev)
    rp, rv = CO.frame(p, v)
    assert np.array_equal(fp.cpu().numpy().view(np.uint32), rp.view(np.uint32))
    assert np.array_equal(fv.cpu().numpy().view(np.uint32), rv.view(np.uint32))
    ft = torch.as_tensor(np.asarray(f, np.int32), device=dev)
    ct = torch.as_tensor(c, device=dev)
    got = [x.cpu().numpy() if isinstance(x, torch.Tensor) else x
           for x in capi.transfer_colors(fv, ft, fp, ct, r, want_terms=True)]
    again = [x.cpu().numpy() if isinstance(x, torch.Tensor) else x
             for x in capi.transfer_colors(fv, ft, fp, ct, r, want_terms=True)]
    for x, y in zip(got, again):                                        # two calls: identical bits
        assert np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8))
    out, st, face, dist, w, sums, fb = got
    ref = CO.transfer(rv, f, rp, c, r)
    assert np.array_equal(face, ref["face"]), np.argwhere(face != ref["face"])[:5]
    assert np.array_equal(dist.view(np.uint32), ref["dist"].view(np.uint32))
    assert np.array_equal(w.view(np.uint32), ref["weights"].view(np.uint32)), np.argwhere(w != ref["weights"])[:5]
    assert np.array_equal(sums.view(np.uint64), ref["sums"])
    assert np.array_equal(fb.astype(bool), ref["fallback"])
    assert np.array_equal(out.view(np.uint32), ref["colors"].view(np.uint32)), np.argwhere(out != ref["colors"])[:5]
    assert st.tolist() == ref["stats"].tolist()
    pub, pst = transfer_colors(v, f, p, c, r)                           # the public path
    assert np.array_equal(pub.cpu().numpy().view(np.uint32), out.view(np.uint32))
    assert (pst.used, pst.beyond, pst.fallback_vertices) == tuple(st.tolist())
    return ref


CASES = [(n, F) for n in (1, 100, 4096, 100_000) for F in (1, 37, 800, 1600)]


@gpu
@pytest.mark.parametrize("n,F", CASES)
def test_kernel_matches_the_oracle_bit_for_bit(n, F):
    seed = CASES.index((n, F))
    v, f = sphere_mesh(F, seed)
    p, c = scan(n, v, f, seed + 100, offset=1e4 if seed % 2 else 0.0)
    ref = _check(v + (1e4 if seed % 2 else 0.0), f, p, c)
    if n >= 4096 and F >= 37:
        assert ref["stats"][0] > 0 and ref["stats"][1] > 0


@gpu
def test_one_million_points_against_the_oracle():
    v, f = sphere_mesh(800, 7)
    p, c = scan(1_000_000, v, f, 8)
    ref = _check(v, f, p, c)
    print(f"1M points, 800 faces: {ref['stats'].tolist()} (used, beyond r, fallback vertices)")


@gpu
def test_all_points_beyond_r():
    """Every point farther than r from a small mesh in the middle of the cloud: every vertex takes its nearest point."""
    v, f = sphere_mesh(800, 3)
    rng = np.random.default_rng(4)
    d = rng.normal(size=(20000, 3))
    p = d / np.linalg.norm(d, axis=1, keepdims=True) * 10.0
    c = rng.uniform(0, 1, (20000, 3)).astype(F32)
    ref = _check(v, f, p, c)
    assert ref["stats"].tolist() == [0, 20000, len(v)] and ref["fallback"].all()


@gpu
def test_bad_input_raises_before_any_launch():
    dev = _dev()
    v = torch.rand(10, 3, device=dev) - 0.5
    f = torch.tensor([[0, 1, 2], [3, 4, 5]], dtype=torch.int32, device=dev)
    p = torch.rand(100, 3, device=dev) - 0.5
    c = torch.rand(100, 3, device=dev)
    L = capi.lib()
    nan = torch.full_like(v, float("nan"))
    bad = [(v.cpu(), f, p, c, 0.05), (v.double(), f, p, c, 0.05), (v[:, :2].contiguous(), f, p, c, 0.05),
           (nan, f, p, c, 0.05), (v, f.long(), p, c, 0.05), (v, f.cpu(), p, c, 0.05), (v, f[:, :2].contiguous(), p, c, 0.05),
           (v, f + 8, p, c, 0.05), (v, f - 1, p, c, 0.05), (v, f[:0], p, c, 0.05), (v, f, p.cpu(), c, 0.05),
           (v, f, p.double(), c, 0.05), (v, f, p[:0], c[:0], 0.05), (v, f, p, c[:50], 0.05), (v, f, p, c.double(), 0.05),
           (v, f, p, c + 1, 0.05), (v, f, p, c - 1, 0.05), (v, f, p, torch.full_like(c, float("nan")), 0.05),
           (v, f, p, c, 0.0), (v, f, p, c, -1.0), (v, f, p, c, float("nan")), (v, f, p, c, float("inf")),
           (v, f, p, c, 1e-50), (v, f, p, c, True), (v, f, p, c, "0.1"), (v[:0], f[:0], p, c, 0.05),
           (v, f, p.t().contiguous().t(), c, 0.05), (v.t().contiguous().t(), f, p, c, 0.05)]
    torch.cuda.synchronize()
    before = L.ma_launch_count()
    for args in bad:
        with pytest.raises(ValueError):
            capi.transfer_colors(*args)
    assert L.ma_launch_count() == before
    out, st = capi.transfer_colors(v, f, p[:1].contiguous(), c[:1].contiguous(), 10.0)   # the edges are accepted
    assert st[:2].tolist() == [1, 0] and 7 <= st[2] <= 9 and bool(((out >= 0) & (out <= 1)).all())


def _colored_scene(tmp_path, kind, seed):
    """The tabletop scan of the object-splitting tests (three objects on a table disc with legs and strays), each row's
    colour encoding its index; saved with colours (scene.npy) and without them (plain.npy)."""
    from tests import objects_oracle as JO
    pts, _ = JO.table_scene(seed, n=40000)
    n = len(pts)
    idx = np.arange(n)
    rgb = np.stack([(idx % 256) / 255, ((idx // 256) % 256) / 255, (idx // 65536) / 255], 1)
    base = pts if kind == "pc" else np.concatenate([pts, np.tile([[0.0, 0.0, 1.0]], (n, 1))], 1)
    np.save(tmp_path / "scene.npy", np.concatenate([base, rgb], 1))
    np.save(tmp_path / "plain.npy", base)
    return pts, rgb


def _row_of(rgb):
    q = np.rint(np.asarray(rgb) * 255).astype(np.int64)
    return q[:, 0] + 256 * q[:, 1] + 65536 * q[:, 2]


@gpu
@pytest.mark.parametrize("objects", [False, True])
@pytest.mark.parametrize("kind", ["pc", "pc_normal"])
def test_dataset_colors_follow_their_rows(tmp_path, monkeypatch, kind, objects):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    pts, rgb = _colored_scene(tmp_path, kind, 2)
    kw = dict(plane={"distance": 0.01, "iterations": 1000}, outliers={"k": 16, "std_ratio": 2.0, "min_component": 0.01},
              smooth={"k": 24}, objects={"distance": 0.02} if objects else None)
    np.random.seed(0)
    ds = cli.Dataset(kind, [str(tmp_path / "scene.npy")], colors=True, **kw)
    np.random.seed(0)
    plain = cli.Dataset(kind, [str(tmp_path / "plain.npy")], **kw)
    assert len(ds) == len(plain) == (3 if objects else 1)
    for j in range(len(ds)):
        item, base = ds[j], plain[j]
        assert set(item) == {"pc_normal", "uid", "frame", "colors"} and set(base) == {"pc_normal", "uid", "frame"}
        assert np.array_equal(ds.data[j]["pc_normal"], plain.data[j]["pc_normal"])    # the flag changes no draw
        cloud = item["colors"]
        assert cloud.dtype == F64 and cloud.shape[1] == 6 and cloud.shape[0] >= 4096
        rows = _row_of(cloud[:, 3:])
        assert len(np.unique(rows)) == len(rows)
        assert np.array_equal(cloud[:, 3:], rgb[rows])                   # each row keeps its own colour
        moved = np.linalg.norm(cloud[:, :3] - pts[rows], axis=1)
        assert 0 < moved.max() < 0.05 and np.median(moved) < 0.01       # smoothing moved xyz, a little
        # the rows the model sees are rows of the full cloud, at the same coordinates
        sub = ds.data[j]["pc_normal"][:, :3]
        full = {tuple(x) for x in cloud[:, :3].astype(sub.dtype).tolist()}
        assert all(tuple(x) in full for x in sub.tolist())


def _read_obj(path):
    vs, fs = [], []
    for line in open(path):
        s = line.split()
        if s and s[0] == "v":
            vs.append([float(x) for x in s[1:7]])
        elif s and s[0] == "f":
            fs.append([int(x) - 1 for x in s[1:4]])
    return np.array(vs).reshape(-1, 6), np.array(fs, dtype=np.int64).reshape(-1, 3)


@gpu
def test_main_cli_transfer_colors(tmp_path):
    """The OBJ's vertex colours equal transfer_colors of the written mesh against the item's cloud, to the 8 decimals
    written, under --output_frame input, and per object under --split_objects; --output_frame model gives the same
    colours as input."""
    rng = np.random.default_rng(5)
    d = rng.normal(size=(12000, 3))
    a = d / np.linalg.norm(d, axis=1, keepdims=True) * [1.0, 0.7, 0.5] + [100.0, 50.0, 20.0]
    b = a + [4.0, 0.0, 0.0]
    rgb_a = (a - a.min(0)) / (a.max(0) - a.min(0))
    rgb_b = np.tile([[0.1, 0.8, 0.3]], (12000, 1))
    np.save(tmp_path / "scan.npy", np.concatenate([np.concatenate([a, rgb_a], 1), np.concatenate([b, rgb_b], 1)]))

    def run(*extra):
        out = tmp_path / ("out" + "_".join(extra))
        cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--out_dir", str(out), "--pretrained_weights",
               "synthetic", "--n_max_triangles", "24", "--input_type", "pc", "--input_path",
               str(tmp_path / "scan.npy"), "--transfer_colors", *extra]
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        assert "vertices from" in r.stdout and "nearest point's colour" in r.stdout, r.stdout[-2000:]
        return sorted(os.path.join(dp, x) for dp, _, fs in os.walk(out) for x in fs if x.endswith(".obj"))

    def check(path, xyz, rgb):
        vs, fs = _read_obj(path)
        assert len(fs) > 0
        want, _ = transfer_colors(vs[:, :3], fs, xyz, rgb, 0.05)
        assert np.abs(vs[:, 3:] - want.cpu().numpy()).max() <= 5e-9 + 1e-6
        assert not np.all(vs[:, 3:] == [1.0, 0.64705882, 0.0])
        return vs

    both = np.concatenate([np.concatenate([a, b]), np.concatenate([rgb_a, rgb_b])], 1)
    (inp,) = run("--output_frame", "input")
    vin = check(inp, both[:, :3], both[:, 3:])
    (mod,) = run("--output_frame", "model")
    vm, _ = _read_obj(mod)
    assert len(vm) == len(vin) and np.abs(vm[:, 3:] - vin[:, 3:]).max() <= 1e-6
    objs = run("--split_objects", "--output_frame", "input")
    assert len(objs) == 2
    for path in objs:
        vs, _ = _read_obj(path)
        near_a = np.linalg.norm(vs[:, :3].mean(0) - a.mean(0)) < np.linalg.norm(vs[:, :3].mean(0) - b.mean(0))
        check(path, a if near_a else b, rgb_a if near_a else rgb_b)
