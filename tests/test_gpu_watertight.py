"""-m gpu: the watertight remesh of `--mc` (csrc/watertight.cu): distance field and marching cubes bit-identical to the
numpy restatement (tests/watertight_oracle.py), surface properties on the reference's wand mesh, the drop-in
mesh_to_pc path and the `main.py --mc` command line."""
import os

import numpy as np
import pytest
import torch

import mesh_to_pc
from meshanything_b200 import capi
from tests import watertight_oracle as W

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wand_mesh.npz")


def _dev():
    return torch.device("cuda", 0)


def _wand():
    z = np.load(GOLDEN)
    return z["vertices"].astype(np.float64), z["faces"].astype(np.int64)


def _soup(n_tri, seed):
    rng = np.random.RandomState(seed)
    v = rng.uniform(-0.6, 0.6, (3 * n_tri, 3)).astype(np.float32)
    f = rng.randint(0, len(v), (n_tri, 3))
    f[0] = [1, 1, 2]                                     # repeated vertex: a segment
    f[1] = [5, 5, 5]                                     # a point
    v[f[2, 2]] = 0.5 * (v[f[2, 0]] + v[f[2, 1]])         # collinear: zero area
    return v, f


def _cube():
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)], np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))])
    return v, f


def _case(name):
    if name == "soup32":
        return (*_soup(40, 1), 32)
    if name == "soup64":
        return (*_soup(300, 2), 64)
    if name == "cube":
        return (*_cube(), 64)
    if name == "triangle":
        return np.array([[-0.4, -0.3, 0.1], [0.5, -0.2, -0.1], [0.0, 0.45, 0.2]], np.float32), np.array([[0, 1, 2]]), 32
    v, f = _wand()
    unit, _, _ = mesh_to_pc.normalize_vertices(v)
    return unit.astype(np.float32), f, 128


def _gpu_remesh(v, f, n):
    field = capi.udf_grid(torch.from_numpy(v).to(_dev()), torch.from_numpy(np.asarray(f, np.int32)).to(_dev()), n)
    verts, faces = capi.marching_cubes(field, 2.0 / n)
    torch.cuda.synchronize()
    return field.cpu().numpy(), verts.cpu().numpy(), faces.cpu().numpy()


@gpu
@pytest.mark.parametrize("name", ["soup32", "soup64", "cube", "triangle", "wand128"])
def test_field_and_mesh_bit_identical_to_the_oracle(name):
    v, f, n = _case(name)
    field, verts, faces = _gpu_remesh(v, f, n)
    ref = W.udf_grid(v, f, n)
    assert field.dtype == np.float32 and field.shape == (n, n, n)
    diff = int((field.view(np.uint32) != ref.view(np.uint32)).sum())
    assert diff == 0, f"{diff} grid points differ, max |d| {np.abs(field - ref).max()}"
    rv, rf = W.marching_cubes(ref, 2.0 / n)
    assert verts.shape == rv.shape and faces.shape == rf.shape, (verts.shape, rv.shape, faces.shape, rf.shape)
    assert np.array_equal(verts.view(np.uint32), rv.view(np.uint32))
    assert np.array_equal(faces, rf)
    assert len(faces) > 0 and W.is_watertight(faces)
    # a second run gives the same bits
    field2, verts2, faces2 = _gpu_remesh(v, f, n)
    assert np.array_equal(field2.view(np.uint32), field.view(np.uint32))
    assert np.array_equal(verts2.view(np.uint32), verts.view(np.uint32)) and np.array_equal(faces2, faces)


@gpu
def test_marching_cubes_of_an_analytic_shell_matches_the_oracle():
    n, R = 64, 0.5
    g = W.grid_coords(n).astype(np.float64)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    fld = np.abs(np.sqrt(X * X + Y * Y + Z * Z) - R).astype(np.float32)
    verts, faces = capi.marching_cubes(torch.from_numpy(fld).to(_dev()), 2.0 / n)
    rv, rf = W.marching_cubes(fld, 2.0 / n)
    assert np.array_equal(verts.cpu().numpy(), rv) and np.array_equal(faces.cpu().numpy(), rf)


@gpu
def test_wand_remesh_is_closed_oriented_and_at_distance_dx():
    v, f = _wand()
    unit, centre, factor = mesh_to_pc.normalize_vertices(v)
    n = 128
    dx = 2.0 / n
    field, verts, faces = _gpu_remesh(unit.astype(np.float32), f, n)
    assert W.is_watertight(faces)
    # orientation: along each face's normal the field grows (probed by trilinear interpolation half a cell away)
    from scipy.ndimage import map_coordinates
    nrm = W.face_normals(verts, faces)
    area = np.linalg.norm(nrm, axis=1)
    real = area > 0
    nh = nrm[real] / area[real, None]
    cen = verts[faces].astype(np.float64).mean(1)[real]
    up = map_coordinates(field.astype(np.float64), (cen + 0.5 * nh).T, order=1)
    down = map_coordinates(field.astype(np.float64), (cen - 0.5 * nh).T, order=1)
    good = up > down
    print("wand n=128: %d vertices, %d faces, normals along the field gradient for %.4f of the faces"
          % (len(verts), len(faces), good.mean()))
    assert good.mean() > 0.97
    # and per shell: a flipped component would fail here (shells of a few cells are too small for the half-cell probe)
    comp_of = np.empty(len(faces), dtype=np.int64)
    for ci, c in enumerate(W.components(faces, len(verts))):
        comp_of[c] = ci if len(c) >= 64 else -1
    for ci in np.unique(comp_of[comp_of >= 0]):
        sel = comp_of[real] == ci
        assert (area[real][sel] * good[sel]).sum() > 0.5 * area[real][sel].sum(), ci
    # every vertex, in the input frame, lies at distance dx (input units: dx / factor) from the input surface
    w = (verts.astype(np.float64) / n * 2 - 1) / factor + centre
    d = W.mesh_distance(w, v, f, 2 * dx / factor)
    err = np.abs(d - dx / factor) / (dx / factor)
    print("vertex distance to the input surface: |d - dx| / dx max %.3f, median %.4f" % (err.max(), np.median(err)))
    assert err.max() < 0.5


@gpu
def test_process_mesh_to_pc_with_marching_cubes(monkeypatch):
    v, f = _wand()
    mesh = mesh_to_pc.SimpleMesh(v, f)
    np.random.seed(0)
    clouds, used = mesh_to_pc.process_mesh_to_pc([mesh], marching_cubes=True)
    pc = clouds[0]
    assert pc.shape == (4096, 6) and pc.dtype == np.float16
    assert np.abs(np.linalg.norm(pc[:, 3:].astype(np.float32), axis=1) - 1).max() < 2e-3
    assert W.is_watertight(np.asarray(used[0].faces))
    _, _, factor = mesh_to_pc.normalize_vertices(v)
    level = (2.0 / 128) / factor                                   # iso level in input units
    d = W.mesh_distance(pc[:, :3].astype(np.float64), v, f, 4 * level)
    slack = 5e-4 * np.abs(v).max()                                 # fp16 rounding of the points
    print("sampled points: distance to the input surface / level max %.3f, median |d - level| / level %.4f"
          % (d.max() / level, np.median(np.abs(d - level)) / level))
    assert d.max() < 3.5 * level + slack
    assert np.median(np.abs(d - level)) < 0.25 * level
    # same seed -> same cloud
    np.random.seed(0)
    again, _ = mesh_to_pc.process_mesh_to_pc([mesh], marching_cubes=True)
    assert np.array_equal(again[0], pc)
    # MA_PC_SAMPLER=host keeps the mesh2sdf / scikit-image path
    monkeypatch.setenv("MA_PC_SAMPLER", "host")
    try:
        import mesh2sdf.core  # noqa: F401
        import skimage.measure  # noqa: F401
    except Exception:
        with pytest.raises(ImportError, match="mesh2sdf"):
            mesh_to_pc.process_mesh_to_pc([mesh], marching_cubes=True)


@gpu
def test_main_cli_mesh_with_mc_writes_obj(tmp_path):
    """`python main.py --input_type mesh --input_path wand.obj --mc` (the reference README's mesh command) runs
    offline and writes wand_gen.obj."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    v, f = _wand()
    obj = tmp_path / "wand.obj"
    with open(obj, "w") as fh:
        fh.writelines(f"v {x:.9g} {y:.9g} {z:.9g}\n" for x, y, z in v)
        fh.writelines(f"f {a + 1} {b + 1} {c + 1}\n" for a, b, c in f)
    out_dir = tmp_path / "out"
    r = subprocess.run([sys.executable, os.path.join(root, "main.py"), "--input_type", "mesh", "--input_path", str(obj),
                        "--mc", "--out_dir", str(out_dir), "--pretrained_weights", "synthetic", "--n_max_triangles", "6",
                        "--seed", "0"], cwd=root, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "MC over!" in r.stdout
    objs = [os.path.join(dp, x) for dp, _, fs in os.walk(out_dir) for x in fs if x.endswith("_gen.obj")]
    assert len(objs) == 1 and os.path.basename(objs[0]) == "wand_gen.obj"
