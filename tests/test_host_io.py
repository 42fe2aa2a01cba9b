"""not gpu: host-side pre/post-processing that main.py shares with the reference (main.py:15-58,156-175; mesh_to_pc.py)."""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUBE = """v 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nv 0 0 1\nv 1 0 1\nv 1 1 1\nv 0 1 1
f 1 2 3 4\nf 5 8 7 6\nf 1 5 6 2\nf 2 6 7 3\nf 3 7 8 4\nf 5 1 4 8\n"""


@pytest.mark.parametrize("face", ["f 1 2 9", "f 0 1 2", "f 1 2 -9"])
def test_obj_face_outside_the_vertex_list_raises(tmp_path, face):
    """A face index past the vertices read so far (or 0, or a relative index before the first) is refused at load time
    instead of reaching the surface sampler."""
    import mesh_to_pc
    p = tmp_path / "bad.obj"
    p.write_text(CUBE + face + "\n")
    with pytest.raises(ValueError, match="outside 1..8"):
        mesh_to_pc.SimpleMesh.load_obj(str(p))


def test_numpy_mesh_sampler(tmp_path):
    import mesh_to_pc
    p = tmp_path / "cube.obj"
    p.write_text(CUBE)
    mesh = mesh_to_pc.SimpleMesh.load_obj(str(p))
    assert mesh.faces.shape == (12, 3)                      # quads are fan-triangulated
    np.random.seed(0)
    clouds, used = mesh_to_pc.process_mesh_to_pc([mesh])
    pc = clouds[0]
    assert pc.shape == (4096, 6) and pc.dtype == np.float16 and used[0] is mesh
    xyz, nrm = pc[:, :3].astype(np.float32), pc[:, 3:].astype(np.float32)
    assert np.allclose(np.linalg.norm(nrm, axis=1), 1.0, atol=1e-3)
    on_face = np.isclose(xyz, 0, atol=2e-3) | np.isclose(xyz, 1, atol=2e-3)
    assert on_face.any(axis=1).all()                        # every sample lies on a cube face
    # area weighting: the six faces get ~1/6 of the samples each
    axis = np.argmax(np.abs(nrm), axis=1)
    side = (np.take_along_axis(nrm, axis[:, None], 1)[:, 0] > 0).astype(int)
    counts = np.bincount(axis * 2 + side, minlength=6)
    assert counts.min() > 4096 / 6 * 0.8


def test_dataset_normalisation(tmp_path, monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    from meshanything_b200.inputs import normalize_pc_normal, synthetic_pc_normal
    rng = np.random.default_rng(0)
    xyz = rng.uniform(-3, 5, size=(5000, 3))
    nrm = rng.normal(size=(5000, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    out = normalize_pc_normal(np.concatenate([xyz, nrm], axis=1))
    c = out[:, :3].astype(np.float64)
    assert out.dtype == np.float16 and abs(np.abs(c).max() - 0.9995) < 1e-3
    assert np.allclose(c.min(0) + c.max(0), 0, atol=2e-3) or np.abs(c).max() <= 1.0   # centred on the bounding box
    with pytest.raises(AssertionError):
        normalize_pc_normal(np.concatenate([xyz, nrm * 0.5], axis=1))            # main.py:54
    s = synthetic_pc_normal(2, first=0)
    assert s.shape == (2, 4096, 6) and s.dtype.is_floating_point


def test_dataset_matches_reference_dataset_on_mouse_example(tmp_path, monkeypatch):
    """BASELINE configs[0], host side: `Dataset('pc_normal', [mouse.npy])` under numpy seed 0 must hand the model exactly
    the array the reference's own Dataset class (main.py:15-58) produced from the same file -- fixture
    tests/golden/config1_mouse.npz, made by tests/golden/make_golden_inputs.py from the reference's class source."""
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    fx = np.load(os.path.join(ROOT, "tests", "golden", "config1_mouse.npz"))
    path = tmp_path / "mouse.npy"
    np.save(path, fx["raw"])
    np.random.seed(0)                       # what set_seed(args.seed) leaves in numpy (main.py:97)
    item = cli.Dataset("pc_normal", [str(path)])[0]
    assert item["uid"] == "mouse"
    assert item["pc_normal"].dtype == np.float16 and item["pc_normal"].shape == (4096, 6)
    assert np.array_equal(item["pc_normal"].view(np.uint16), fx["pc_normal"].view(np.uint16))


def test_obj_export_merges_vertices_and_faces(tmp_path, monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import importlib
    main = importlib.import_module("main")
    tri = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0]],
                    [[1, 0, 0], [0, 1, 0], [1, 1, 0]],
                    [[0, 0, 0], [1, 0, 0], [0, 1, 0]]], dtype=np.float32)      # third face duplicates the first
    path = tmp_path / "m.obj"
    n = main.export_obj(str(path), tri)
    txt = path.read_text().splitlines()
    assert n == 2 and sum(l.startswith("f ") for l in txt) == 2
    assert sum(l.startswith("v ") for l in txt) == 4                            # 9 corners -> 4 distinct vertices


def _cube():
    v = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], dtype=np.float32)
    quads = [[0, 1, 3, 2], [4, 6, 7, 5], [0, 4, 5, 1], [2, 3, 7, 6], [0, 2, 6, 4], [1, 5, 7, 3]]
    return v, quads


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian", "binary_big_endian"])
def test_numpy_ply_loader(tmp_path, fmt):
    """PLY without trimesh: ascii / binary, extra vertex properties, quads fan-triangulated, a skipped extra element."""
    import struct
    import mesh_to_pc
    v, quads = _cube()
    path = tmp_path / f"cube_{fmt}.ply"
    header = (f"ply\nformat {fmt} 1.0\ncomment made by a test\nelement vertex 8\nproperty float x\nproperty float y\n"
              "property float z\nproperty uchar red\nproperty double quality\nelement face 6\n"
              "property list uchar int vertex_indices\nelement edge 1\nproperty int vertex1\nproperty int vertex2\n"
              "end_header\n")
    with open(path, "wb") as f:
        f.write(header.encode())
        if fmt == "ascii":
            for p in v:
                f.write(f"{p[0]} {p[1]} {p[2]} 200 0.5\n".encode())
            for q in quads:
                f.write(("4 " + " ".join(map(str, q)) + "\n").encode())
            f.write(b"0 1\n")
        else:
            e = "<" if fmt == "binary_little_endian" else ">"
            for p in v:
                f.write(struct.pack(e + "fffBd", p[0], p[1], p[2], 200, 0.5))
            for q in quads:
                f.write(struct.pack(e + "Biiii", 4, *q))
            f.write(struct.pack(e + "ii", 0, 1))
    m = mesh_to_pc.SimpleMesh.load_ply(str(path))
    assert m.vertices.shape == (8, 3) and m.faces.shape == (12, 3)
    assert np.allclose(m.vertices, v)
    t = m.vertices[m.faces]
    area = 0.5 * np.linalg.norm(np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]), axis=1).sum()
    assert abs(area - 6.0) < 1e-9                      # the cube's surface, whatever the triangulation
    if mesh_to_pc.trimesh is None:
        pcs, _ = mesh_to_pc.process_mesh_to_pc([mesh_to_pc.load_mesh(str(path))])
        assert pcs[0].shape == (4096, 6)


def test_ply_errors(tmp_path):
    import mesh_to_pc
    bad = tmp_path / "x.ply"
    bad.write_bytes(b"plx\n")
    with pytest.raises(ValueError):
        mesh_to_pc.SimpleMesh.load_ply(str(bad))
    cloud = tmp_path / "cloud.ply"
    cloud.write_bytes(b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\nproperty float z\n"
                      b"end_header\n0 0 0\n")
    with pytest.raises(ValueError):
        mesh_to_pc.SimpleMesh.load_ply(str(cloud))
    if mesh_to_pc.trimesh is None:
        with pytest.raises(ImportError):
            mesh_to_pc.load_mesh(str(tmp_path / "m.stl"))


def test_fix_winding_orients_a_scrambled_cube_outwards():
    import main
    v, quads = _cube()
    tri = []
    for q in quads:
        tri += [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
    tri = np.array(tri)
    rng = np.random.default_rng(0)
    scrambled = tri.copy()
    flipped = rng.random(len(tri)) < 0.5
    scrambled[flipped] = scrambled[flipped][:, ::-1]
    # two cubes far apart = two components, the second one entirely inside-out
    v2 = np.concatenate([v, v + 10.0])
    tri2 = np.concatenate([scrambled, tri[:, ::-1] + 8])
    fixed = main.fix_winding(v2, tri2)
    assert sorted(map(tuple, np.sort(fixed, axis=1))) == sorted(map(tuple, np.sort(tri2, axis=1)))   # same faces
    t = v2[fixed].astype(np.float64)
    n = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
    centre = np.where((np.arange(len(fixed)) < len(tri))[:, None], v.mean(0), v.mean(0) + 10.0)
    assert (np.einsum("ij,ij->i", n, t.mean(1) - centre) > 0).all()          # every normal points away from its cube


def test_export_obj_merges_vertices_and_drops_duplicate_faces(tmp_path):
    import main
    tri = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0]],
                    [[1, 0, 0], [1, 1, 0], [0, 1, 0]],
                    [[0, 1, 0], [0, 0, 0], [1, 0, 0]]], dtype=np.float32)       # third = first, rotated
    path = tmp_path / "m.obj"
    n = main.export_obj(str(path), tri)
    txt = path.read_text().splitlines()
    vs = [l for l in txt if l.startswith("v ")]
    fs = [l for l in txt if l.startswith("f ")]
    assert n == 2 and len(fs) == 2 and len(vs) == 4


def test_dataset_from_mesh_files(tmp_path):
    """main.Dataset('mesh', [...]) on an OBJ and a PLY file (reference main.py:15-58): 4096 points, max |x| = 0.9995,
    unit normals, fp16."""
    import main
    import mesh_to_pc
    if mesh_to_pc.trimesh is not None:
        pytest.skip("exercises the numpy readers")
    v, quads = _cube()
    obj = tmp_path / "cube.obj"
    with open(obj, "w") as f:
        for p in v:
            f.write(f"v {p[0]} {p[1]} {p[2]}\n")
        for q in quads:
            f.write("f " + " ".join(str(i + 1) for i in q) + "\n")
    ply = tmp_path / "cube2.ply"
    with open(ply, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex 8\nproperty float x\nproperty float y\nproperty float z\n"
                "element face 6\nproperty list uchar int vertex_indices\nend_header\n")
        for p in v:
            f.write(f"{p[0] * 3} {p[1] * 3} {p[2] * 3}\n")
        for q in quads:
            f.write("4 " + " ".join(map(str, q)) + "\n")
    np.random.seed(0)
    ds = main.Dataset("mesh", [str(obj), str(ply)])
    assert len(ds) == 2 and [ds.data[i]["uid"] for i in range(2)] == ["cube", "cube2"]
    for i in range(2):
        pc = ds[i]["pc_normal"]
        assert pc.shape == (4096, 6) and pc.dtype == np.float16
        assert abs(np.abs(pc[:, :3].astype(np.float32)).max() - 0.9995) < 2e-3
        assert np.allclose(np.linalg.norm(pc[:, 3:].astype(np.float32), axis=1), 1.0, atol=5e-3)
