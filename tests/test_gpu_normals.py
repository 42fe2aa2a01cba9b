"""-m gpu: the normal estimator of `--input_type pc` (csrc/normals.cu) against its numpy restatement
(tests/normals_oracle.py) -- kNN indices, unoriented and oriented normals bit for bit -- exact kNN at 1M points, bad
input refused before any launch, and the pipeline: `Dataset('pc')` and `main.py --input_type pc`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from meshanything_b200 import capi, metrics
from tests import normals_oracle as O

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _dev():
    return torch.device("cuda", 0)


def _sphere(n, rng, centre=(0.0, 0.0, 0.0), r=1.0):
    x = rng.normal(size=(n, 3))
    return x / np.linalg.norm(x, axis=1, keepdims=True) * r + np.asarray(centre)


def _cloud(n, seed):
    """A scan-like cloud offset by 1e4: a sphere of radius 10 with exact duplicates, a collinear and a coplanar subset,
    a cluster of thousands of points inside one grid cell, and a second component far away.  Small n: uniform."""
    rng = np.random.default_rng(seed)
    if n < 200:
        return (rng.uniform(-10, 10, (n, 3)) + 1e4).astype(F32)
    n2 = n // 5
    main = _sphere(n - n2, rng, r=10.0)
    m = len(main)
    main[m // 10:m // 10 + m // 20] = main[: m // 20]                              # exact duplicates
    t = np.linspace(0, 1, m // 20)[:, None]
    main[m // 5:m // 5 + m // 20] = main[0] + t * np.array([3.0, -2.0, 1.0])       # collinear
    uv = rng.uniform(0, 2, (m // 20, 2))
    main[m // 4:m // 4 + m // 20] = main[1] + uv[:, :1] * [1.0, 0.0, 0.5] + uv[:, 1:] * [0.0, 1.0, -0.5]   # coplanar
    if n >= 4096:
        c = min(3000, m // 4)
        main[m // 2:m // 2 + c] = main[m // 2] + rng.uniform(-2e-3, 2e-3, (c, 3))  # cluster in one cell
    other = _sphere(n2, rng, centre=(40.0, 5.0, -3.0), r=4.0)                     # second component
    return (np.concatenate([main, other]) + 1e4).astype(F32)


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


CASES = [(n, k) for k in (1, 8, 16, 64) for n in (k + 1, 1000, 4096, 20000)]


@gpu
@pytest.mark.parametrize("n,k", CASES)
def test_kernel_matches_the_oracle_bit_for_bit(n, k):
    pts = _cloud(n, seed=n + 100 * k)
    frame = metrics.to_output_frame(torch.from_numpy(pts)[None].to(_dev()))[0]
    rf = O.frame_map(pts)
    assert np.array_equal(_bits(frame.cpu().numpy()), _bits(rf))
    out = [t.cpu().numpy() for t in capi.estimate_normals(frame, k, want_terms=True)]
    again = [t.cpu().numpy() for t in capi.estimate_normals(frame, k, want_terms=True)]
    for x, y in zip(out, again):                                     # two calls: identical bits
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    normals, knn, uno = out
    r_normals, r_knn, r_uno = O.estimate_normals(rf, k)
    assert np.array_equal(knn, r_knn), np.argwhere(knn != r_knn)[:5]
    assert np.array_equal(_bits(uno), _bits(r_uno)), np.argwhere(_bits(uno) != _bits(r_uno))[:5]
    assert np.array_equal(_bits(normals), _bits(r_normals)), np.argwhere(_bits(normals) != _bits(r_normals))[:5]
    assert np.all(np.abs(np.linalg.norm(normals.astype(np.float64), axis=1) - 1) < 1e-6)
    from meshanything_b200.normals import estimate_normals
    assert np.array_equal(_bits(estimate_normals(pts, k).cpu().numpy()), _bits(normals))   # the public path


@gpu
def test_one_million_points_exact_knn_and_outward_sphere():
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    v, f = torch.from_numpy(z["vertices"]).to(_dev()), torch.from_numpy(z["faces"]).to(_dev())
    n, k = 1_000_000, 16
    xyz = capi.sample_surface(v, f, n, seed=11)[:, :3].float()
    frame = metrics.to_output_frame(xyz[None])[0]
    _, knn, _ = capi.estimate_normals(frame, k, want_terms=True)
    rounds = capi.lib().ma_estimate_normals_last_rounds()
    q = torch.from_numpy(np.random.default_rng(0).choice(n, 2000, replace=False)).to(_dev())
    for part in q.split(250):
        d = frame[part][:, None, :] - frame[None, :, :]
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        d2[torch.arange(len(part), device=d2.device), part] = float("inf")
        ref = torch.sort(d2, dim=1, stable=True).indices[:, :k]     # ties: lowest index first
        assert torch.equal(knn[part].long(), ref)
    g = torch.Generator(device=_dev()).manual_seed(3)
    s = torch.randn(n, 3, device=_dev(), generator=g)
    s = s / s.norm(dim=1, keepdim=True) * 2.0 + torch.tensor([1.0, -2.0, 0.5], device=_dev())
    sf = metrics.to_output_frame(s[None])[0]
    nrm = capi.estimate_normals(sf, k)
    out = (nrm * sf).sum(dim=1)
    assert bool((out > 0).all()), int((out <= 0).sum())
    print(f"1M wand points: {rounds} Boruvka rounds; 1M sphere: {capi.lib().ma_estimate_normals_last_rounds()} rounds")


@gpu
def test_bad_input_raises_before_any_launch():
    dev = _dev()
    ok = torch.rand(100, 3, device=dev) - 0.5
    L = capi.lib()
    bad = [((ok.cpu(),), {}), ((ok.double(),), {}), ((ok[:, :2].contiguous(),), {}), ((ok.t().contiguous().t(),), {}),
           ((ok[:16].contiguous(),), {}), ((ok.cpu().numpy(),), {}),
           ((torch.full((100, 3), float("nan"), device=dev),), {}), ((torch.full((100, 3), float("inf"), device=dev),), {}),
           ((ok,), {"k": 0}), ((ok,), {"k": 65}), ((ok,), {"k": 2.5}), ((ok,), {"k": True})]
    torch.cuda.synchronize()
    before = L.ma_launch_count()
    for args, kw in bad:
        with pytest.raises(ValueError):
            capi.estimate_normals(*args, **kw)
    assert L.ma_launch_count() == before
    capi.estimate_normals(ok[:65].contiguous(), k=64)  # the edges of every range are accepted


def _mouse():
    return np.load(os.path.join(ROOT, "tests", "golden", "config1_mouse.npz"))


@gpu
def test_dataset_pc_selects_the_points_pc_normal_selects(tmp_path, monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    fx = _mouse()
    np.save(tmp_path / "mouse.npy", fx["raw"][:, :3])
    np.random.seed(0)
    item = cli.Dataset("pc", [str(tmp_path / "mouse.npy")])[0]
    pc = item["pc_normal"]
    assert item["uid"] == "mouse" and pc.dtype == np.float16 and pc.shape == (4096, 6)
    assert np.array_equal(pc[:, :3].view(np.uint16), fx["pc_normal"][:, :3].view(np.uint16))
    assert np.all(np.abs(np.linalg.norm(pc[:, 3:].astype(np.float64), axis=1) - 1) < 2e-3)
    np.save(tmp_path / "with_normals.npy", fx["raw"])
    with pytest.raises(ValueError, match="--input_type pc_normal"):
        cli.Dataset("pc", [str(tmp_path / "with_normals.npy")])


def _main(args, tmp_path, timeout=900):
    return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--out_dir", str(tmp_path / "out"),
                           "--pretrained_weights", "synthetic", "--n_max_triangles", "6"] + args, cwd=ROOT,
                          capture_output=True, text=True, timeout=timeout)


def _objs(tmp_path):
    return sorted(f for _, _, fs in os.walk(tmp_path / "out") for f in fs if f.endswith(".obj"))


@gpu
def test_main_cli_pc_input_path(tmp_path):
    np.save(tmp_path / "mouse.npy", _mouse()["raw"][:, :3].astype(np.float32))
    r = _main(["--input_type", "pc", "--input_path", str(tmp_path / "mouse.npy")], tmp_path)
    assert r.returncode == 0, r.stderr[-2000:]
    assert _objs(tmp_path) == ["mouse_gen.obj"]


@gpu
def test_main_cli_default_input_type_reads_a_vertex_only_ply_directory(tmp_path):
    """No --input_type: the default is `pc`, a bare cloud; a binary vertex-only PLY in --input_dir goes through."""
    in_dir = tmp_path / "in"
    in_dir.mkdir()
    xyz = _mouse()["raw"][:, :3].astype(np.float32)
    rec = np.zeros(len(xyz), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4")])
    rec["x"], rec["y"], rec["z"] = xyz.T
    with open(in_dir / "scan.ply", "wb") as f:
        f.write(f"ply\nformat binary_little_endian 1.0\nelement vertex {len(xyz)}\nproperty float x\n"
                "property float y\nproperty float z\nend_header\n".encode())
        f.write(rec.tobytes())
    r = _main(["--input_dir", str(in_dir)], tmp_path)
    assert r.returncode == 0, r.stderr[-2000:]
    assert _objs(tmp_path) == ["scan_gen.obj"]
