"""not gpu: the numpy restatement of colour transfer (tests/colors_oracle.py; DESIGN.md section 1.9) against float64
geometry and the mesh score's nearest faces, its colours on constant and two-colour scans, the cutoff and the fallback;
the coloured loaders and their refusals; `--transfer_colors` in check_args, export_obj and the Dataset draw."""
import argparse
import os

import numpy as np
import pytest

from tests import colors_oracle as CO
from tests import mesh_score_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64


def _closest64(p, a, b, c):
    """The point of triangle (a, b, c) nearest to p in float64 (Ericson, Real-Time Collision Detection 5.1.5); a
    degenerate triangle as the nearest point of its three segments."""
    ab, ac, ap = b - a, c - a, p - a
    if np.linalg.norm(np.cross(ab, ac)) == 0:
        best = None
        for s, e in ((a, b), (b, c), (c, a)):
            l = (e - s) @ (e - s)
            t = 0.0 if l == 0 else np.clip((p - s) @ (e - s) / l, 0, 1)
            q = s + t * (e - s)
            if best is None or np.linalg.norm(p - q) < np.linalg.norm(p - best):
                best = q
        return best
    d1, d2 = ab @ ap, ac @ ap
    if d1 <= 0 and d2 <= 0:
        return a
    bp = p - b
    d3, d4 = ab @ bp, ac @ bp
    if d3 >= 0 and d4 <= d3:
        return b
    vc = d1 * d4 - d3 * d2
    if vc <= 0 and d1 >= 0 and d3 <= 0:
        return a + d1 / (d1 - d3) * ab
    cp = p - c
    d5, d6 = ab @ cp, ac @ cp
    if d6 >= 0 and d5 <= d6:
        return c
    vb = d5 * d2 - d1 * d6
    if vb <= 0 and d2 >= 0 and d6 <= 0:
        return a + d2 / (d2 - d6) * ac
    va = d3 * d6 - d5 * d4
    if va <= 0 and (d4 - d3) >= 0 and (d5 - d6) >= 0:
        return b + (d4 - d3) / ((d4 - d3) + (d5 - d6)) * (c - b)
    den = 1 / (va + vb + vc)
    return a + ab * (vb * den) + ac * (vc * den)


def _bary(p, tri):
    t = tri.astype(F32)
    return CO.bary(CO._cols(p.astype(F32)), *(CO._cols(t[:, k]) for k in range(3)))


def test_weights_match_the_float64_closest_point_in_every_region():
    rng = np.random.default_rng(0)
    n = 4000
    tri = rng.uniform(-0.5, 0.5, (n, 3, 3))
    # interior (points just off the face), near each edge, beyond each vertex, and far
    r = rng.dirichlet([1, 1, 1], n)
    base = np.einsum("nk,nkd->nd", r, tri)
    nrm = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    p = base + nrm * rng.normal(0, 0.2, (n, 1))
    k = n // 4
    p[k:2 * k] = tri[k:2 * k, 0] + (tri[k:2 * k, 0] - tri[k:2 * k, 1]) * rng.uniform(0, 2, (k, 1))
    p[2 * k:3 * k] = base[2 * k:3 * k] + rng.normal(0, 1.0, (k, 3))
    tri[3 * k:3 * k + 100, 2] = tri[3 * k:3 * k + 100, 1]                   # two coincident vertices
    tri[3 * k + 100:3 * k + 200, 2] = 0.5 * (tri[3 * k + 100:3 * k + 200, 0] + tri[3 * k + 100:3 * k + 200, 1])
    tri[3 * k + 200:3 * k + 300] = tri[3 * k + 200:3 * k + 300, :1]         # one point
    w = _bary(p, tri)
    t32 = tri.astype(F32).astype(F64)
    p32 = p.astype(F32).astype(F64)
    assert np.all((w >= 0) & (w <= 1))
    assert np.all(np.abs(w.astype(F64).sum(1) - 1) < 1e-5)
    got = np.einsum("nk,nkd->nd", w.astype(F64), t32)
    want = np.array([_closest64(p32[i], *t32[i]) for i in range(n)])
    scale = 1 + np.linalg.norm(p32 - t32[:, 0], axis=1)
    err = np.linalg.norm(got - want, axis=1) / scale
    assert err.max() < 1e-5, (err.argmax(), err.max())
    # every region occurs: interior (three weights > 0), edges (one zero), vertices (two zeros)
    zeros = (w == 0).sum(1)
    assert (zeros == 0).sum() > 500 and (zeros == 1).sum() > 200 and (zeros == 2).sum() > 200


def test_weights_choose_the_region_of_the_distance():
    """The weights' point is at the fp32 distance tri_dist reports, up to rounding."""
    rng = np.random.default_rng(1)
    tri = rng.uniform(-0.5, 0.5, (3000, 3, 3)).astype(F32)
    p = rng.uniform(-1, 1, (3000, 3)).astype(F32)
    w = _bary(p, tri)
    q = np.einsum("nk,nkd->nd", w.astype(F64), tri.astype(F64))
    d = CO.tri_dist(CO._cols(p), *(CO._cols(tri[:, k]) for k in range(3))).astype(F64)
    assert np.abs(np.linalg.norm(p - q, axis=1) - d).max() < 1e-5


def test_nearest_faces_equal_the_mesh_score_oracle():
    rng = np.random.default_rng(2)
    v = rng.uniform(-0.5, 0.5, (60, 3)).astype(F32)
    f = rng.integers(0, 60, (90, 3))
    f[10] = f[3]                                                          # a duplicate: ties go to the lower index
    p = rng.uniform(-0.6, 0.6, (3000, 3)).astype(F32)
    face, dist = CO.nearest_faces(p, v, f)
    ref = MO.candidate(v[f], np.concatenate([p, np.zeros_like(p)], 1))
    assert np.array_equal(face, ref["point_face"]) and np.array_equal(dist, ref["point_dist"])
    assert not np.any(face == 10)


def _sphere(n_lat=12, n_lon=24):
    th, ph = np.meshgrid(np.linspace(0.1, np.pi - 0.1, n_lat), np.linspace(0, 2 * np.pi, n_lon, endpoint=False),
                         indexing="ij")
    v = 0.5 * np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1).reshape(-1, 3)
    idx = np.arange(n_lat * n_lon).reshape(n_lat, n_lon)
    a, b = idx[:-1], np.roll(idx, -1, axis=1)[:-1]
    c, d = idx[1:], np.roll(idx, -1, axis=1)[1:]
    return v, np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([b, d, c], -1).reshape(-1, 3)])


def test_a_constant_colour_scan_colours_every_vertex():
    v, f = _sphere()
    rng = np.random.default_rng(3)
    d = rng.normal(size=(20000, 3))
    p = d / np.linalg.norm(d, axis=1, keepdims=True) * 0.5 + 1e4               # offset: the float64 frame keeps it
    col = np.tile(np.array([[0.3, 0.6, 0.9]], F32), (len(p), 1))
    out, res = CO.transfer_colors(v + 1e4, f, p, col)
    assert res["stats"][0] > 19000 and res["stats"][2] == 0
    assert np.abs(out.astype(F64) - col[0].astype(F64)).max() <= 2.0 ** -20


def _banded_cube():
    """A cube [-0.5, 0.5]^3 with a ring of vertices at z = 0: top, upper band, lower band, bottom."""
    sq = np.array([[-0.5, -0.5], [0.5, -0.5], [0.5, 0.5], [-0.5, 0.5]])
    v = np.concatenate([np.c_[sq, np.full(4, z)] for z in (0.5, 0.0, -0.5)])
    f = [[0, 1, 2], [0, 2, 3], [8, 10, 9], [8, 11, 10]]
    for ring in (0, 4):
        for k in range(4):
            a, b = ring + k, ring + (k + 1) % 4
            f += [[a + 4, b + 4, b], [a + 4, b, a]]
    return v, np.array(f)


def test_a_two_colour_cube_gives_red_top_and_blue_bottom_vertices():
    v, f = _banded_cube()
    rng = np.random.default_rng(4)
    p = rng.uniform(-0.5, 0.5, (30000, 3))
    axis = rng.integers(0, 3, len(p))
    p[np.arange(len(p)), axis] = rng.choice([-0.5, 0.5], len(p))               # on the cube's surface
    p = p[np.abs(p[:, 2]) > 1e-3]
    col = np.where(p[:, 2:] > 0, [[1.0, 0.0, 0.0]], [[0.0, 0.0, 1.0]]).astype(F32)
    out, res = CO.transfer_colors(v, f, p, col)
    assert res["stats"][1] == 0 and res["stats"][2] == 0
    assert np.array_equal(out[:4], np.tile([[1, 0, 0]], (4, 1)).astype(F32))
    assert np.array_equal(out[8:], np.tile([[0, 0, 1]], (4, 1)).astype(F32))
    ring = out[4:8]
    assert np.all(ring[:, 1] == 0) and np.all(np.abs(ring[:, 0] - 0.5) < 0.1) and np.all(np.abs(ring[:, 2] - 0.5) < 0.1)


def test_points_beyond_r_are_ignored_and_the_fallback_is_taken():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 0]], F64)
    f = np.array([[0, 1, 2], [1, 3, 2]])
    rng = np.random.default_rng(5)
    r = rng.dirichlet([1, 1, 1], 500)
    near = r @ v[:3] * 0.9 + 0.03                                               # inside face 0
    far = near + [0.0, 0.0, 3.0]                                                # 3 above it: beyond r = 0.05 L
    p = np.concatenate([near, far, [[4.9, 4.9, 0.5]]])                          # and one point near vertex 3, 0.5 up
    col = np.concatenate([np.tile([[0.2, 0.4, 0.6]], (500, 1)), np.tile([[1.0, 1.0, 1.0]], (500, 1)),
                          [[0.0, 1.0, 0.0]]]).astype(F32)
    out, res = CO.transfer_colors(v, f, p, col, 0.05)
    assert res["stats"].tolist() == [500, 501, 1]
    assert np.abs(out[:3].astype(F64) - [0.2, 0.4, 0.6]).max() <= 2.0 ** -20   # the far white points are ignored
    assert res["fallback"].tolist() == [False, False, False, True]
    assert out[3].tolist() == [0.0, 1.0, 0.0]                                   # vertex 3: its nearest point
    _, res1 = CO.transfer_colors(v, f, p, col, 1.0)                             # everything within r = L
    assert res1["stats"].tolist()[:2] == [1001, 0]


def test_fixed_point_rounds_half_to_even():
    assert CO.fix(np.array([0.5 / 2 ** 24, 1.5 / 2 ** 24, 1.0], F32)).tolist() == [0, 2, 2 ** 24]


# ---------------------------------------------------------------- loaders

def _write_ply(path, xyz, rgb, fmt, types, alpha=False, faces=None):
    props = [("x", "f4"), ("y", "f4"), ("z", "f4")] + [(c, types) for c in ("red", "green", "blue")]
    if alpha:
        props.append(("alpha", types))
    names = {"f4": "float", "u1": "uchar", "u2": "ushort", "f8": "double"}
    head = [b"ply", f"format {fmt} 1.0".encode(), b"comment colours", f"element vertex {len(xyz)}".encode()]
    head += [f"property {names[t]} {n}".encode() for n, t in props]
    if faces is not None:
        head += [f"element face {len(faces)}".encode(), b"property list uchar int vertex_indices"]
    head.append(b"end_header")
    cols = [xyz[:, 0], xyz[:, 1], xyz[:, 2], rgb[:, 0], rgb[:, 1], rgb[:, 2]] + ([rgb[:, 0]] if alpha else [])
    with open(path, "wb") as fh:
        fh.write(b"\n".join(head) + b"\n")
        if fmt == "ascii":
            for i in range(len(xyz)):
                fh.write((" ".join(repr(float(c[i])) if t[0] == "f" else str(int(c[i]))
                                   for c, (_, t) in zip(cols, props)) + "\n").encode())
            for fc in (faces if faces is not None else []):
                fh.write(f"3 {fc[0]} {fc[1]} {fc[2]}\n".encode())
        else:
            dt = np.dtype([(n, "<" + t) for n, t in props])
            rec = np.zeros(len(xyz), dt)
            for (n, _), c in zip(props, cols):
                rec[n] = c
            fh.write(rec.tobytes())


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian"])
@pytest.mark.parametrize("types", ["u1", "u2", "f4"])
def test_ply_colours(tmp_path, fmt, types):
    from mesh_to_pc import load_points
    rng = np.random.default_rng(6)
    xyz = rng.normal(size=(50, 3)).astype(F32)
    top = {"u1": 255, "u2": 65535}.get(types)
    raw = rng.integers(0, top + 1, (50, 3)) if top else rng.uniform(0, 1, (50, 3)).astype(F32)
    path = str(tmp_path / "c.ply")
    _write_ply(path, xyz, raw, fmt, types, alpha=True)
    got_xyz, rgb = load_points(path, colors=True)
    assert np.array_equal(got_xyz, xyz.astype(F64))
    want = raw / top if top else raw.astype(F64)
    assert rgb.dtype == F64 and np.array_equal(rgb, want)
    assert np.array_equal(load_points(path), xyz.astype(F64))                  # without the flag: xyz as before


def test_npy_colour_layouts(tmp_path, monkeypatch):
    from mesh_to_pc import load_points
    rng = np.random.default_rng(7)
    xyz, rgb, nrm = rng.normal(size=(5000, 3)), rng.uniform(0, 1, (5000, 3)), rng.normal(size=(5000, 3))
    np.save(tmp_path / "pc.npy", np.concatenate([xyz, rgb], 1))
    got_xyz, got_rgb = load_points(str(tmp_path / "pc.npy"), colors=True)
    assert np.array_equal(got_xyz, xyz) and np.array_equal(got_rgb, rgb)
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    np.save(tmp_path / "pcn.npy", np.concatenate([xyz, nrm, rgb], 1))
    np.random.seed(0)
    entry = cli.Dataset("pc_normal", [str(tmp_path / "pcn.npy")], colors=True).data[0]
    assert entry["pc_normal"].shape == (4096, 6) and np.array_equal(entry["colors"], np.concatenate([xyz, rgb], 1))


def test_refusals(tmp_path, monkeypatch):
    from mesh_to_pc import load_cloud, load_points
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    rng = np.random.default_rng(8)
    xyz = rng.normal(size=(20, 3)).astype(F32)
    bare = tmp_path / "bare.ply"
    with open(bare, "wb") as fh:
        fh.write(b"ply\nformat ascii 1.0\nelement vertex 20\nproperty float x\nproperty float y\nproperty float z\n"
                 b"end_header\n" + "".join(f"{a} {b} {c}\n" for a, b, c in xyz).encode())
    with pytest.raises(ValueError, match="without red, green and blue"):
        load_points(str(bare), colors=True)
    assert load_points(str(bare)).shape == (20, 3)
    hot = str(tmp_path / "hot.ply")
    _write_ply(hot, xyz, rng.uniform(0, 2, (20, 3)), "binary_little_endian", "f4")
    with pytest.raises(ValueError, match=r"outside \[0, 1\]"):
        load_points(hot, colors=True)
    mesh = str(tmp_path / "mesh.ply")
    _write_ply(mesh, xyz, rng.integers(0, 256, (20, 3)), "ascii", "u1", faces=[[0, 1, 2]])
    with pytest.raises(ValueError, match="is a mesh"):
        load_points(mesh, colors=True)
    for shape in ((20, 3), (20, 4), (20, 9), (20,)):
        np.save(tmp_path / "w.npy", np.zeros(shape))
        with pytest.raises(ValueError, match=r"\(N, 6\), xyz \| rgb"):
            load_points(str(tmp_path / "w.npy"), colors=True)
    np.save(tmp_path / "neg.npy", np.concatenate([xyz, -np.ones((20, 3))], 1))
    with pytest.raises(ValueError, match=r"outside \[0, 1\]"):
        load_points(str(tmp_path / "neg.npy"), colors=True)
    np.save(tmp_path / "nan.npy", np.concatenate([xyz, np.full((20, 3), np.nan)], 1))
    with pytest.raises(ValueError, match=r"outside \[0, 1\]"):
        load_points(str(tmp_path / "nan.npy"), colors=True)
    for shape in ((5000, 6), (5000, 3)):
        np.save(tmp_path / "n9.npy", np.zeros(shape))
        with pytest.raises(ValueError, match=r"\(N, 9\), xyz \| normal \| rgb"):
            load_cloud(str(tmp_path / "n9.npy"), "pc_normal", colors=True)
    # without the flag the loaders' messages are unchanged
    np.save(tmp_path / "six.npy", np.zeros((20, 6)))
    with pytest.raises(ValueError, match="looks like points with normals"):
        load_points(str(tmp_path / "six.npy"))
    with pytest.raises(ValueError, match="colours of a mesh"):
        cli.Dataset("mesh", [], colors=True)


def _args(**kw):
    base = dict(num_samples=1, sampling=False, continuous_batching=False, remove_outliers=False, input_type="pc",
                transfer_colors=True, color_distance=0.05)
    base.update(kw)
    return argparse.Namespace(**base)


def test_check_args(monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    cli.check_args(_args())
    cli.check_args(_args(color_distance=1.0, input_type="pc_normal"))
    cli.check_args(_args(transfer_colors=False, input_type="mesh", color_distance=7.0))
    with pytest.raises(ValueError, match="--transfer_colors applies to point-cloud input"):
        cli.check_args(_args(input_type="mesh"))
    for bad in (0.0, -0.1, 1.5, float("nan"), float("inf"), 1e-50):
        with pytest.raises(ValueError, match="--color_distance"):
            cli.check_args(_args(color_distance=bad))


def test_export_obj_with_and_without_colours(tmp_path, monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    tri = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0]], [[1, 0, 0], [1, 1, 0], [0, 1, 0]],
                    [[0, 0, 0], [1, 0, 0], [0, 1, 0]]], F32)                   # a duplicate face
    cli.export_obj(str(tmp_path / "plain.obj"), tri)
    lines = open(tmp_path / "plain.obj").read().splitlines()
    assert [ln for ln in lines if ln.startswith("v ")] == [
        f"v {x:.8f} {y:.8f} 0.00000000 1.00000000 0.64705882 0.00000000" for x, y in ((0, 0), (0, 1), (1, 0), (1, 1))]
    seen = {}

    def paint(vertices, faces):
        seen["v"], seen["f"] = vertices, faces
        return np.asarray(vertices)[:, [0, 1, 2]] * [0.5, 0.25, 1.0]

    n = cli.export_obj(str(tmp_path / "col.obj"), tri, paint)
    assert n == 2 and seen["f"].shape == (2, 3) and seen["v"].shape == (4, 3)
    vs = [ln.split() for ln in open(tmp_path / "col.obj").read().splitlines() if ln.startswith("v ")]
    fs = [ln for ln in open(tmp_path / "col.obj").read().splitlines() if ln.startswith("f ")]
    assert len(fs) == 2
    for row, v in zip(vs, seen["v"]):
        assert [float(x) for x in row[4:]] == pytest.approx([v[0] * 0.5, v[1] * 0.25, 0.0], abs=1e-8)


def test_dataset_draw_unchanged_without_the_flag(tmp_path, monkeypatch):
    monkeypatch.syspath_prepend(ROOT)
    import main as cli
    rng = np.random.default_rng(9)
    nrm = rng.normal(size=(6000, 3))
    pcn = np.concatenate([rng.normal(size=(6000, 3)), nrm / np.linalg.norm(nrm, axis=1, keepdims=True)], 1)
    rgb = rng.uniform(0, 1, (6000, 3))
    np.save(tmp_path / "a.npy", pcn)
    np.save(tmp_path / "b.npy", np.concatenate([pcn, rgb], 1))
    np.random.seed(3)
    plain = cli.Dataset("pc_normal", [str(tmp_path / "a.npy")])
    after_plain = np.random.random()
    np.random.seed(3)
    col = cli.Dataset("pc_normal", [str(tmp_path / "b.npy")], colors=True)
    assert np.random.random() == after_plain
    assert set(plain.data[0]) == {"pc_normal", "uid"} and set(plain[0]) == {"pc_normal", "uid", "frame"}
    assert np.array_equal(plain.data[0]["pc_normal"], col.data[0]["pc_normal"])
    assert np.array_equal(col[0]["colors"], np.concatenate([pcn[:, :3], rgb], 1))
    assert np.array_equal(col[0]["pc_normal"], plain[0]["pc_normal"])
