"""-m gpu: farthest-point subsampling (csrc/subsample.cu) against its numpy restatement (tests/subsample_oracle.py) bit for
bit -- picks and covering radii on every kernel path, on both sides of the size that selects between them -- against a
brute-force loop of torch operations at 1M and 4M points, its input validation, and the pipeline: `Dataset(...,
subsample='fps')` for `pc` and `pc_normal`, with and without outlier removal, and `main.py --subsample fps`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from meshanything_b200 import capi
from meshanything_b200.outliers import remove_outliers
from meshanything_b200.pointcloud import frame_points
from meshanything_b200.subsample import farthest_point_sample
from tests import subsample_oracle as S

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64
SMALL_N = 8192                     # kFpsSmallN of subsample.cu: one CTA up to here, a cooperative grid above
PATHS = (capi.FPS_ONE_CTA, capi.FPS_GRID_SHARED, capi.FPS_GRID_GLOBAL)
ONE_CTA_MAX = 14_000               # a one-CTA forced run is tried up to here (the whole cloud in 227 KB of shared memory)


def _dev():
    return torch.device("cuda", 0)


def _sphere(n, rng):
    x = rng.normal(size=(n, 3))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _cloud(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "cube":
        return rng.uniform(-1, 1, (n, 3)).astype(F32)
    if kind == "dup_sphere":                                     # a sphere whose second half repeats the first exactly
        p = _sphere(n, rng)
        h = n // 2
        p[h:h + h] = p[:h]
        return p.astype(F32)
    if kind == "exp_sphere":                                     # density proportional to e^(3z)
        out = np.empty((0, 3))
        while len(out) < n:
            x = _sphere(4 * n + 64, rng)
            out = np.concatenate([out, x[rng.random(len(x)) < np.exp(3 * x[:, 2] - 3)]])
        return out[:n].astype(F32)
    if kind == "offset":                                         # float64 far from the origin
        return rng.uniform(-10, 10, (n, 3)) + 1e4
    if kind == "identical":
        return np.full((n, 3), 0.25, F32)
    raise ValueError(kind)


CLOUDS = ("cube", "dup_sphere", "exp_sphere", "offset", "identical")
SIZES = (1, 2, 4096, 5000, SMALL_N, SMALL_N + 1, 20000, 100_000)
CASES = []
for a, n in enumerate(SIZES):
    for b, m in enumerate(sorted({1, 64, 4096, n} if n <= 2 else (1, 64, 4096))):
        if m > n:
            continue
        for c, start in enumerate(("0", "last", "seeded")):
            CASES.append((n, m, start, CLOUDS[(a + b + c) % len(CLOUDS)]))


def _start(kind, n, seed):
    return {"0": 0, "last": n - 1, "seeded": int(np.random.default_rng(seed).integers(n))}[kind]


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


def _run_path(frame, m, start, path):
    L = capi.lib()
    prev = L.ma_farthest_point_sample_set_path(path)
    try:
        idx, r2 = capi.farthest_point_sample(frame, m, start)
        torch.cuda.synchronize()
        return idx.cpu().numpy(), r2.cpu().numpy(), L.ma_farthest_point_sample_last_path()
    finally:
        L.ma_farthest_point_sample_set_path(prev)


@gpu
@pytest.mark.parametrize("n,m,start,cloud", CASES)
def test_kernel_matches_the_oracle_bit_for_bit(n, m, start, cloud):
    pts = _cloud(cloud, n, n + m)
    s = _start(start, n, n * 7 + m)
    frame = frame_points(pts, _dev()).contiguous()
    rf = S.frame_map(pts)
    assert np.array_equal(frame.cpu().numpy().view(np.uint32), rf.view(np.uint32))
    ridx, rr2 = S.farthest_point_sample(rf, m, s)
    idx, r2, path = _run_path(frame, m, s, capi.FPS_AUTO)
    assert path == (capi.FPS_ONE_CTA if n <= SMALL_N else capi.FPS_GRID_SHARED)
    assert np.array_equal(idx, ridx), np.argwhere(idx != ridx)[:5]
    assert np.array_equal(_bits(r2), _bits(rr2)), np.argwhere(r2 != rr2)[:5]
    for forced in PATHS:                                         # every kernel path, same bits
        if forced == capi.FPS_ONE_CTA and n > ONE_CTA_MAX:
            continue
        fidx, fr2, fpath = _run_path(frame, m, s, forced)
        assert fpath == forced
        assert np.array_equal(fidx, ridx) and np.array_equal(_bits(fr2), _bits(rr2)), forced
    pidx, pr2 = farthest_point_sample(pts, m, s)                 # the public path
    assert np.array_equal(pidx.cpu().numpy(), ridx) and np.array_equal(_bits(pr2.cpu().numpy()), _bits(rr2))


def _wand(n, seed):
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    v, f = torch.from_numpy(z["vertices"]).to(_dev()), torch.from_numpy(z["faces"]).to(_dev())
    xyz = capi.sample_surface(v, f, n, seed=seed)[:, :3].float()
    return frame_points(xyz, _dev()).contiguous()


@gpu
@pytest.mark.parametrize("n,path", [(1_000_000, capi.FPS_GRID_SHARED), (4_000_000, capi.FPS_GRID_GLOBAL)])
def test_millions_of_points_match_torch_brute_force(n, path):
    """1M points fit the CTAs' shared memory on 132 SMs; 4M do not and run from global memory."""
    frame = _wand(n, seed=3)
    start = 12345
    idx, r2, got = _run_path(frame, 4096, start, capi.FPS_AUTO)
    assert got == path
    ridx, rr2 = S.torch_bruteforce(frame, 4096, start)
    assert np.array_equal(idx, ridx.cpu().numpy())
    assert np.array_equal(_bits(r2), _bits(rr2.cpu().numpy()))
    idx2, r22, _ = _run_path(frame, 4096, start, capi.FPS_AUTO)          # two calls: identical bits
    assert np.array_equal(idx, idx2) and np.array_equal(_bits(r2), _bits(r22))
    if path == capi.FPS_GRID_SHARED:                                     # the global-memory path on the same cloud
        oidx, or2, _ = _run_path(frame, 4096, start, capi.FPS_GRID_GLOBAL)
        assert np.array_equal(idx, oidx) and np.array_equal(_bits(r2), _bits(or2))
    print(f"{n} wand points: covering radius of 4096 picks {float(np.sqrt(r2[-1])):.5f} (output frame)")


@gpu
def test_bad_input_raises_value_error_and_launches_nothing():
    L = capi.lib()
    good = torch.rand((100, 3), device=_dev())
    nan = good.clone()
    nan[7, 1] = float("nan")
    inf = good.clone()
    inf[3, 0] = float("inf")
    bad = [
        (good.cpu().numpy(), 4, 0), (good[:, :2].contiguous(), 4, 0), (good.reshape(-1), 4, 0),
        (good[None], 4, 0), (good.double(), 4, 0), (good.half(), 4, 0), (good.t().contiguous().t(), 4, 0),
        (good.cpu(), 4, 0), (good[:0], 1, 0), (good, 0, 0), (good, 101, 0), (good, 4, -1), (good, 4, 100),
        (good, 4.0, 0), (good, 4, 1.5), (good, True, 0), (good, 4, None), (nan, 4, 0), (inf, 4, 0),
        (torch.empty((2 ** 24 + 1, 3), device=_dev()), 4, 0),
    ]
    torch.cuda.synchronize()
    before = L.ma_launch_count()
    for pts, m, start in bad:
        with pytest.raises(ValueError):
            capi.farthest_point_sample(pts, m, start)
    with pytest.raises(ValueError):
        farthest_point_sample(np.zeros((10, 2)), 4)
    with pytest.raises(ValueError):
        farthest_point_sample(np.zeros((10, 3)), 11)
    assert L.ma_launch_count() == before
    prev = L.ma_farthest_point_sample_set_path(capi.FPS_ONE_CTA)        # a forced path the device cannot hold
    try:
        with pytest.raises(RuntimeError, match="cannot hold"):
            capi.farthest_point_sample(torch.rand((100_000, 3), device=_dev()), 16, 0)
    finally:
        L.ma_farthest_point_sample_set_path(prev)
    idx, r2 = capi.farthest_point_sample(good, 4, 0)                    # and the library works on afterwards
    assert idx.tolist()[0] == 0 and len(set(idx.tolist())) == 4


def _uneven_scan(seed, n=9000, strays=20):
    """A sphere of density proportional to e^(3z) plus far stray points (the last `strays` rows), float64."""
    rng = np.random.default_rng(seed)
    s = _cloud("exp_sphere", n, seed).astype(F64)
    far = _sphere(strays, rng) * rng.uniform(7, 10, (strays, 1))
    return np.concatenate([s, far])


OUT = {"k": 16, "std_ratio": 2.0, "min_component": 0.01}


def _expected_picks(xyz, seed):
    """The oracle's picks from the start main.py draws: np.random.randint(N) right after np.random.seed(seed)."""
    np.random.seed(seed)
    s = np.random.randint(len(xyz))
    idx, _ = S.farthest_point_sample(S.frame_map(xyz), 4096, s)
    return idx


@gpu
@pytest.mark.parametrize("outliers", [None, OUT])
def test_dataset_pc_normal_fps(tmp_path, monkeypatch, outliers):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    xyz = _uneven_scan(1)
    nrm = np.concatenate([xyz[:-20], _sphere(20, np.random.default_rng(2))])
    cloud = np.concatenate([xyz, nrm], axis=1)
    np.save(tmp_path / "scan.npy", cloud)
    kept = np.arange(len(xyz)) if outliers is None else remove_outliers(xyz, **outliers)[0].cpu().numpy()
    want = cloud[kept][_expected_picks(xyz[kept], 5)]
    np.random.seed(5)
    got = cli.Dataset("pc_normal", [str(tmp_path / "scan.npy")], outliers=outliers, subsample="fps").data[0]["pc_normal"]
    assert np.array_equal(got, want)
    strays = np.isin(np.arange(len(xyz) - 20, len(xyz)), kept[_expected_picks(xyz[kept], 5)]).sum()
    assert strays == (20 if outliers is None else 0)               # FPS takes every stray unless they are removed


@gpu
@pytest.mark.parametrize("outliers", [None, OUT])
def test_dataset_pc_fps(tmp_path, monkeypatch, outliers):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    from meshanything_b200.normals import estimate_normals
    xyz = _uneven_scan(3)
    np.save(tmp_path / "scan.npy", xyz)
    kept = np.arange(len(xyz)) if outliers is None else remove_outliers(xyz, **outliers)[0].cpu().numpy()
    picks = _expected_picks(xyz[kept], 6)
    np.random.seed(6)
    got = cli.Dataset("pc", [str(tmp_path / "scan.npy")], outliers=outliers, subsample="fps").data[0]["pc_normal"]
    assert got.shape == (4096, 6)
    assert np.array_equal(got[:, :3], xyz[kept][picks])
    assert np.array_equal(got[:, 3:], estimate_normals(xyz[kept], 16).cpu().numpy()[picks].astype(F64))
    assert np.all(np.abs(np.linalg.norm(got[:, 3:], axis=1) - 1) < 1e-5)


@gpu
def test_main_cli_subsample_fps(tmp_path):
    xyz = _uneven_scan(4)
    np.save(tmp_path / "scan.npy", xyz)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--out_dir", str(tmp_path / "out"),
                        "--pretrained_weights", "synthetic", "--n_max_triangles", "6", "--input_type", "pc",
                        "--input_path", str(tmp_path / "scan.npy"), "--remove_outliers", "--subsample", "fps"],
                       cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "scan: 4096 of " in r.stdout and "points by farthest-point sampling; every point within" in r.stdout, \
        r.stdout[-2000:]
    objs = sorted(f for _, _, fs in os.walk(tmp_path / "out") for f in fs if f.endswith(".obj"))
    assert objs == ["scan_gen.obj"]
