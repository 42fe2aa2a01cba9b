"""-m gpu: the surface sampler (csrc/surface.cu) against its numpy restatement (tests/surface_oracle.py) bit for bit --
face indices and all six fp16 columns -- across one and many scan tiles, sample counts around the block size, both
Philox key words, degenerate, tiny and far-off faces, the committed wand and its marching-cubes remesh; its input
validation; and process_mesh_to_pc on a GPU box."""
import os

import numpy as np
import pytest
import torch

from meshanything_b200 import capi
from tests import surface_oracle as SO

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32

FACES = (1, 2, 1023, 1024, 1025, 2049, 100_000, 1_000_000)
SAMPLES = (1, 255, 256, 257, 4096, 200_000)
SEEDS = (0, 5, 2 ** 31 - 2, 2 ** 32 + 7, 2 ** 64 - 1)
MESHES = ("soup", "zero_runs", "tiny", "offset")
CASES = []
for a, F in enumerate(FACES):
    for b, n in enumerate(SAMPLES if F <= 1025 else (257, 4096, 200_000)):
        CASES.append((F, n, SEEDS[(a + b) % len(SEEDS)], MESHES[(a + 2 * b) % len(MESHES)]))


def _dev():
    return torch.device("cuda", 0)


def _mesh(kind, F, seed):
    """Vertices fp32 [V, 3] and faces int32 [F, 3] of a random soup of one of four kinds."""
    rng = np.random.default_rng(seed)
    V = max(3, F + 2)
    v = rng.normal(size=(V, 3))
    a, d1, d2 = rng.integers(0, V, F), rng.integers(1, V, F), rng.integers(1, V - 1, F)
    f = np.stack([a, (a + d1) % V, (a + d2 + (d2 >= d1)) % V], axis=1)          # three distinct vertices
    if kind == "tiny":                          # faces about 1e-4 across around random centres
        c = rng.normal(size=(F, 3))
        v = np.concatenate([c + rng.normal(size=(F, 3)) * 1e-4 for _ in range(3)])
        f = np.arange(3 * F).reshape(3, F).T
    elif kind == "offset":                      # far from the origin: fp32 differences lose low bits
        v = v + 1e4
    elif kind == "zero_runs":                   # zero-area faces at the start, at the end, in runs and scattered
        z = np.zeros(F, bool)
        z[:1 + F // 50] = True
        z[F - 1 - F // 100:] = True
        z[F // 3:F // 3 + F // 20] = True
        z[rng.random(F) < 0.05] = True
        if F > 1:
            z[F // 2] = False                   # at least one face of positive area
        f[z, 2] = f[z, 0]
    return v.astype(F32), f.astype(np.int32)


def _run(v, f, n, seed):
    out, idx = capi.sample_surface(torch.from_numpy(v).to(_dev()), torch.from_numpy(f).to(_dev()), n, seed=seed,
                                   want_index=True)
    return out.cpu().numpy(), idx.cpu().numpy()


def _check(v, f, n, seed):
    out, idx = _run(v, f, n, seed)
    rout, ridx = SO.sample_surface(v, f, n, seed)
    bad = np.argwhere(idx != ridx)
    assert not len(bad), (len(bad), bad[:5].ravel(), idx[bad[:5, 0]], ridx[bad[:5, 0]])
    ob, rb = out.view(np.uint16), rout.view(np.uint16)
    bad = np.argwhere(ob != rb)
    assert not len(bad), (len(bad), bad[:5], out[tuple(bad[:5].T)], rout[tuple(bad[:5].T)])
    return out, idx


@gpu
@pytest.mark.parametrize("F,n,seed,mesh", CASES)
def test_sampler_matches_the_oracle_bit_for_bit(F, n, seed, mesh):
    v, f = _mesh(mesh, F, F + n)
    out, idx = _check(v, f, n, seed)
    area = SO.face_areas(v, f)
    if area.sum() > 0:
        assert (area[idx] > 0).all()                     # zero-area faces are never drawn
    again = _run(v, f, n, seed)                          # two calls: identical bits
    assert np.array_equal(again[0].view(np.uint16), out.view(np.uint16)) and np.array_equal(again[1], idx)


@gpu
def test_all_degenerate_mesh_takes_the_last_face():
    v, f = _mesh("soup", 50, 1)
    f[:, 1] = f[:, 0]
    out, idx = _check(v, f, 1000, 5)
    assert (idx == 49).all() and (out[:, 3:] == 0).all()


def _wand():
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    return z["vertices"].astype(F32), z["faces"].astype(np.int32)


@gpu
@pytest.mark.parametrize("seed", [3, 2 ** 40 + 1])
def test_wand_and_its_remesh(seed):
    """The committed wand, and its marching-cubes remesh (many faces, a scan across many tiles)."""
    import mesh_to_pc
    v, f = _wand()
    _check(v, f, 200_000, seed)
    mc = mesh_to_pc.export_to_watertight(mesh_to_pc.SimpleMesh(v, f))
    mv, mf = np.asarray(mc.vertices, F32), np.asarray(mc.faces, np.int32)
    assert len(mf) > 20 * 1024
    _check(mv, mf, 200_000, seed)


@gpu
def test_process_mesh_to_pc_returns_the_oracle_cloud():
    """On a GPU box process_mesh_to_pc draws its seed from numpy's generator and returns the sampler's cloud."""
    import mesh_to_pc
    v, f = _wand()
    mesh = mesh_to_pc.SimpleMesh(v, f)
    np.random.seed(17)
    seed = int(np.random.randint(0, 2 ** 31 - 1))
    np.random.seed(17)
    clouds, used = mesh_to_pc.process_mesh_to_pc([mesh])
    want, _ = SO.sample_surface(v, f, 4096, seed)
    assert used[0] is mesh and clouds[0].dtype == np.float16
    assert np.array_equal(clouds[0].view(np.uint16), want.view(np.uint16))


@gpu
def test_bad_input_raises_value_error_and_launches_nothing(tmp_path):
    import mesh_to_pc
    L = capi.lib()
    v = torch.rand((10, 3), device=_dev())
    f = torch.tensor([[0, 1, 2], [3, 4, 5]], dtype=torch.int32, device=_dev())
    nan, inf = v.clone(), v.clone()
    nan[4, 1] = float("nan")
    inf[0, 2] = float("-inf")
    past, neg = f.clone(), f.clone()
    past[1, 2] = 10
    neg[0, 0] = -1
    bad = [
        (v[:, :2], f, 16, 0), (v.reshape(-1), f, 16, 0), (v, f[:, :2], 16, 0), (v, f.reshape(-1), 16, 0),
        (v, f[:0], 16, 0), (v, f, 0, 0), (v, f, -3, 0), (v, f, 2.0, 0), (v, f, 16, -1), (v, f, 16, 2 ** 64),
        (v, past, 16, 0), (v, neg, 16, 0), (v, f.float(), 16, 0), (nan, f, 16, 0), (inf, f, 16, 0),
    ]
    torch.cuda.synchronize()
    before = L.ma_launch_count()
    for vv, ff, n, seed in bad:
        with pytest.raises(ValueError):
            capi.sample_surface(vv, ff, n, seed=seed)
    with pytest.raises(ValueError, match="outside"):       # a malformed mesh through the drop-in entry point
        mesh_to_pc.process_mesh_to_pc([mesh_to_pc.SimpleMesh(v.cpu().numpy(), [[0, 1, 2], [7, 8, 10]])])
    p = tmp_path / "bad.obj"
    p.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 4\n")
    with pytest.raises(ValueError):
        mesh_to_pc.process_mesh_to_pc([mesh_to_pc.SimpleMesh.load_obj(str(p))])
    assert L.ma_launch_count() == before
    out = capi.sample_surface(v, f, 16, seed=0)           # and the library works on afterwards
    assert out.shape == (16, 6)
