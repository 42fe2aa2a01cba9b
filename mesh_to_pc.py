"""Drop-in for /root/reference/mesh_to_pc.py: mesh -> (4096, 6) fp16 point cloud with normals.

On a GPU box with the library, surface sampling (csrc/surface.cu) and the watertight remesh of `marching_cubes=True`
(distance field + marching cubes, csrc/watertight.cu) run in CUDA.  Otherwise, or with MA_PC_SAMPLER=host, trimesh /
mesh2sdf / skimage are used when they are installed (same calls as the reference); without them a small numpy
implementation of area-weighted surface sampling (what `trimesh.Trimesh.sample` does) is used (OBJ and ASCII/binary
PLY readers included) and `marching_cubes=True` raises (mesh2sdf is required for the host-side watertight conversion).
"""
import numpy as np

try:  # optional host-side dependencies of the reference
    import trimesh
except Exception:  # pragma: no cover
    trimesh = None


class SimpleMesh:
    """Minimal triangle mesh (vertices [V,3], faces [F,3]) with the two members the pipeline needs."""

    def __init__(self, vertices, faces):
        self.vertices = np.asarray(vertices, dtype=np.float64)
        self.faces = np.asarray(faces, dtype=np.int64)

    @property
    def face_normals(self):
        t = self.vertices[self.faces]
        n = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
        ln = np.linalg.norm(n, axis=1, keepdims=True)
        return n / np.where(ln > 0, ln, 1.0)

    def sample(self, count, return_index=False):
        t = self.vertices[self.faces]
        area = 0.5 * np.linalg.norm(np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]), axis=1)
        idx = np.searchsorted(np.cumsum(area), np.random.random(count) * area.sum())
        idx = np.minimum(idx, len(area) - 1)
        r = np.random.random((count, 2))
        flip = r.sum(axis=1) > 1.0
        r[flip] = 1.0 - r[flip]
        tri = t[idx]
        pts = tri[:, 0] + r[:, :1] * (tri[:, 1] - tri[:, 0]) + r[:, 1:] * (tri[:, 2] - tri[:, 0])
        return (pts, idx) if return_index else pts

    @staticmethod
    def load_obj(path):
        vs, fs = [], []
        with open(path) as f:
            for line in f:
                p = line.split()
                if not p:
                    continue
                if p[0] == "v":
                    vs.append([float(x) for x in p[1:4]])
                elif p[0] == "f":
                    ids = [int(x.split("/")[0]) for x in p[1:]]
                    ids = [i - 1 if i > 0 else len(vs) + i for i in ids]
                    if any(not 0 <= i < len(vs) for i in ids):   # vertices are declared before the faces using them
                        raise ValueError(f"{path}: face {line.strip()!r} refers to a vertex outside 1..{len(vs)}")
                    for k in range(1, len(ids) - 1):          # fan triangulation
                        fs.append([ids[0], ids[k], ids[k + 1]])
        return SimpleMesh(vs, fs)


    _PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
                  "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
                  "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}

    @staticmethod
    def load_ply(path):
        """ASCII and binary (little/big endian) PLY: `vertex` (x, y, z among any other scalar properties) and `face`
        (one list property of vertex indices, polygons fan-triangulated).  Other elements are skipped."""
        verts, faces = SimpleMesh._read_ply(path)
        if verts is None or not faces:
            raise ValueError(f"{path}: PLY without vertex/face elements (point clouds go through --input_type pc_normal)")
        return SimpleMesh(verts, np.asarray(faces, dtype=np.int64))

    @staticmethod
    def _read_ply(path, colors=False):
        """(vertices float64 [V, 3] or None, list of triangles) of a PLY file; with `colors` also the vertices' `red
        green blue` as float64 [V, 3] (integer types divided by their maximum, float types as stored; ValueError when
        they are missing or outside [0, 1])."""
        T = SimpleMesh._PLY_TYPES
        with open(path, "rb") as f:
            if f.readline().strip() != b"ply":
                raise ValueError(f"{path}: not a PLY file")
            fmt, elements = None, []
            while True:
                line = f.readline()
                if not line:
                    raise ValueError(f"{path}: truncated PLY header")
                p = line.decode("ascii", "replace").split()
                if not p or p[0] in ("comment", "obj_info"):
                    continue
                if p[0] == "format":
                    fmt = p[1]
                elif p[0] == "element":
                    elements.append({"name": p[1], "count": int(p[2]), "props": []})
                elif p[0] == "property":
                    if p[1] == "list":
                        elements[-1]["props"].append(("list", p[4], T[p[2]], T[p[3]]))
                    else:
                        elements[-1]["props"].append(("scalar", p[2], T[p[1]]))
                elif p[0] == "end_header":
                    break
            if fmt not in ("ascii", "binary_little_endian", "binary_big_endian"):
                raise ValueError(f"{path}: unsupported PLY format {fmt!r}")
            end = ">" if fmt == "binary_big_endian" else "<"
            verts, faces, rgb = None, [], None
            for el in elements:
                n, props = el["count"], el["props"]
                has_list = any(pr[0] == "list" for pr in props)
                if fmt == "ascii":
                    rows = [f.readline().split() for _ in range(n)]
                    if el["name"] == "vertex":
                        names = [pr[1] for pr in props]
                        ix = [names.index(c) for c in "xyz"]
                        verts = np.array([[float(r[i]) for i in ix] for r in rows], dtype=np.float64).reshape(-1, 3)
                        if colors:
                            ic = _rgb_columns(path, names)
                            rgb = np.array([[float(r[i]) for i in ic] for r in rows], dtype=np.float64).reshape(-1, 3)
                            rgb = _scale_rgb(path, rgb, [props[i][2] for i in ic])
                    elif el["name"] == "face":
                        for r in rows:   # list property first (the usual layout); scalar face properties follow it
                            k = int(r[0])
                            ids = [int(x) for x in r[1:1 + k]]
                            faces.extend([ids[0], ids[j], ids[j + 1]] for j in range(1, k - 1))
                    continue
                if not has_list:
                    dt = np.dtype([(pr[1], end + pr[2]) for pr in props])
                    block = np.frombuffer(f.read(dt.itemsize * n), dtype=dt, count=n)
                    if el["name"] == "vertex":
                        verts = np.stack([block[c].astype(np.float64) for c in "xyz"], axis=1)
                        if colors:
                            ic = _rgb_columns(path, [pr[1] for pr in props])
                            rgb = np.stack([block[props[i][1]].astype(np.float64) for i in ic], axis=1)
                            rgb = _scale_rgb(path, rgb, [props[i][2] for i in ic])
                    continue
                for _ in range(n):       # element with a list property: variable-length records
                    for pr in props:
                        if pr[0] == "scalar":
                            f.read(np.dtype(pr[2]).itemsize)
                            continue
                        k = int(np.frombuffer(f.read(np.dtype(pr[2]).itemsize), dtype=end + pr[2])[0])
                        ids = np.frombuffer(f.read(np.dtype(pr[3]).itemsize * k), dtype=end + pr[3]).astype(np.int64)
                        if el["name"] == "face":
                            faces.extend([ids[0], ids[j], ids[j + 1]] for j in range(1, k - 1))
        if colors:
            if verts is not None and rgb is None:
                raise ValueError(f"{path}: PLY vertices without red, green and blue properties (--transfer_colors "
                                 "needs the scan's colours)")
            return verts, faces, rgb
        return verts, faces


_RGB = ("red", "green", "blue")


def _rgb_columns(path, names):
    """Indices of red, green, blue among a vertex element's property names (alpha and the others are ignored)."""
    if not all(c in names for c in _RGB):
        raise ValueError(f"{path}: PLY vertices without red, green and blue properties (--transfer_colors needs the "
                         "scan's colours)")
    return [names.index(c) for c in _RGB]


def _scale_rgb(path, rgb, types):
    """PLY colour columns to [0, 1]: integer types divided by their maximum (255 for uchar), float types as stored."""
    for k, t in enumerate(types):
        if np.dtype(t).kind in "iu":
            rgb[:, k] /= np.iinfo(np.dtype(t)).max
    return check_rgb(path, rgb)


def check_rgb(path, rgb):
    """rgb [N, 3] float64, or ValueError unless every value is finite and in [0, 1]."""
    rgb = np.asarray(rgb, dtype=np.float64)
    if not np.all(np.isfinite(rgb) & (rgb >= 0) & (rgb <= 1)):
        raise ValueError(f"{path}: colours outside [0, 1] (integer colours are divided by their type's maximum, float "
                         "colours are taken as stored)")
    return rgb


def load_points(path, colors=False):
    """A bare point cloud for `--input_type pc`: an .npy of shape (N, 3), or a .ply with a `vertex` element (x, y, z
    among any other properties; ASCII or binary) and no faces.  Returns the xyz array ([N, 3]; the .npy's own dtype,
    float64 from a PLY).  An (N, 6) .npy is refused rather than having its normals dropped.

    With `colors` (`--transfer_colors`) returns (xyz, rgb float64 [N, 3] in [0, 1]) instead: an .npy of shape (N, 6),
    xyz | rgb, or a .ply whose vertices carry `red green blue` (see SimpleMesh._read_ply)."""
    low = path.lower()
    if colors and low.endswith(".npy"):
        cloud = np.load(path)
        if cloud.ndim != 2 or cloud.shape[1] != 6:
            raise ValueError(f"{path}: --transfer_colors reads a coloured point cloud as an array of shape (N, 6), "
                             f"xyz | rgb, got {cloud.shape}")
        return cloud[:, :3], check_rgb(path, cloud[:, 3:])
    if colors and low.endswith(".ply"):
        verts, faces, rgb = SimpleMesh._read_ply(path, colors=True)
        if verts is None:
            raise ValueError(f"{path}: PLY without a vertex element")
        if faces:
            raise ValueError(f"{path}: PLY with faces is a mesh; use --input_type mesh")
        return verts, rgb
    if low.endswith(".npy"):
        xyz = np.load(path)
        if xyz.ndim == 2 and xyz.shape[1] == 6:
            raise ValueError(f"{path}: shape {xyz.shape} looks like points with normals; use --input_type pc_normal, "
                             "which keeps them (--input_type pc estimates normals for bare (N, 3) clouds)")
        if xyz.ndim != 2 or xyz.shape[1] != 3:
            raise ValueError(f"{path}: a bare point cloud is an array of shape (N, 3), got {xyz.shape}")
        return xyz
    if low.endswith(".ply"):
        verts, faces = SimpleMesh._read_ply(path)
        if verts is None:
            raise ValueError(f"{path}: PLY without a vertex element")
        if faces:
            raise ValueError(f"{path}: PLY with faces is a mesh; use --input_type mesh")
        return verts
    raise ValueError(f"{path}: --input_type pc reads .npy (N, 3) and vertex-only .ply files")


def load_cloud(path, input_type, colors=False):
    """A point-cloud file as (xyz [N, 3], normals or None, rgb float64 [N, 3] in [0, 1] or None), rows aligned.

    `pc`: a bare cloud (load_points), integer xyz as float64; no normals.  `pc_normal`: an .npy of (xyz, normal) rows,
    both in the file's dtype.  With `colors` (`--transfer_colors`) also the colours: for pc as load_points reads them,
    for pc_normal from an (N, 9) .npy, xyz | normal | rgb."""
    if input_type == 'pc':
        xyz, rgb = load_points(path, colors=True) if colors else (load_points(path), None)
        if not np.issubdtype(xyz.dtype, np.floating):
            xyz = xyz.astype(np.float64)
        return xyz, None, rgb
    cloud, rgb = np.load(path), None
    if colors:
        if cloud.ndim != 2 or cloud.shape[1] != 9:
            raise ValueError(f"{path}: --transfer_colors reads a coloured pc_normal cloud as an array of shape (N, 9), "
                             f"xyz | normal | rgb, got {cloud.shape}")
        cloud, rgb = cloud[:, :6], check_rgb(path, cloud[:, 6:])
    return cloud[:, :3], cloud[:, 3:], rgb


def load_mesh(path):
    if trimesh is not None:
        return trimesh.load(path)
    low = path.lower()
    if low.endswith(".obj"):
        return SimpleMesh.load_obj(path)
    if low.endswith(".ply"):
        return SimpleMesh.load_ply(path)
    raise ImportError(f"{path}: trimesh is needed to load meshes other than .obj / .ply")


def normalize_vertices(vertices, scale=0.9):
    """Centre on the bounding box and scale its longest side to 2*scale; returns (vertices, centre, factor)."""
    lo, hi = vertices.min(0), vertices.max(0)
    centre = 0.5 * (lo + hi)
    factor = 2.0 * scale / (hi - lo).max()
    return (vertices - centre) * factor, centre, factor


def export_to_watertight(normalized_mesh, octree_depth: int = 7):
    """Watertight remesh used by `--mc` (reference mesh_to_pc.py:13-40): unsigned distance field on a 2^depth grid,
    marching cubes at iso level 2/size, mapped back to the input frame.  On a GPU box both stages run in CUDA
    (ma_udf_grid + ma_marching_cubes_*, csrc/watertight.cu); otherwise, or with MA_PC_SAMPLER=host, mesh2sdf and
    scikit-image do it as in the reference."""
    gpu = _gpu_sampler()
    if gpu is not None:
        return _watertight_gpu(normalized_mesh, octree_depth, *gpu)
    try:
        import mesh2sdf.core
        import skimage.measure
    except Exception as e:  # pragma: no cover
        raise ImportError("--mc needs mesh2sdf, scikit-image and trimesh") from e
    size = 2 ** octree_depth
    unit_vertices, centre, factor = normalize_vertices(normalized_mesh.vertices)
    field = np.abs(mesh2sdf.core.compute(unit_vertices, normalized_mesh.faces, size=size))
    verts, faces, normals, _ = skimage.measure.marching_cubes(field, 2 / size)
    verts = (verts / size * 2 - 1) / factor + centre
    return trimesh.Trimesh(verts, faces, normals=normals)


def _watertight_gpu(mesh, octree_depth, capi, torch):
    """Normalise in float64 on the host, narrow-band distance field (band 3 dx) and marching cubes at level dx = 2/size
    on the GPU, vertices mapped back with (v / size * 2 - 1) / factor + centre."""
    size = 2 ** octree_depth
    unit_vertices, centre, factor = normalize_vertices(np.asarray(mesh.vertices, dtype=np.float64))
    dev = torch.device("cuda", torch.cuda.current_device())
    v = torch.as_tensor(unit_vertices.astype(np.float32), device=dev)
    f = torch.as_tensor(np.asarray(mesh.faces, dtype=np.int32), device=dev)
    field = capi.udf_grid(v, f, size)
    verts, faces = capi.marching_cubes(field, 2.0 / size)
    verts = (verts.cpu().numpy().astype(np.float64) / size * 2 - 1) / factor + centre
    faces = faces.cpu().numpy().astype(np.int64)
    if trimesh is not None:
        return trimesh.Trimesh(verts, faces)
    return SimpleMesh(verts, faces)


def _gpu_sampler():
    """The CUDA surface sampler (ma_sample_surface) when a GPU and the library are there; MA_PC_SAMPLER=host keeps the
    trimesh / numpy sampler (same distribution, numpy's random stream: what the reference draws)."""
    import os
    if os.environ.get("MA_PC_SAMPLER", "gpu") != "gpu":
        return None
    try:
        import torch
        if not torch.cuda.is_available():
            return None
        from meshanything_b200 import capi
        capi.lib()
        return capi, torch
    except Exception:
        return None


def process_mesh_to_pc(mesh_list, marching_cubes=False, sample_num=4096):
    """[mesh] -> ([fp16 (sample_num, 6) points + face normals], [mesh actually sampled]).  On a GPU box the points are
    drawn by the CUDA sampler (seeded from numpy's generator, so `set_seed` still decides them)."""
    clouds, used = [], []
    gpu = _gpu_sampler()
    for mesh in mesh_list:
        if marching_cubes:
            mesh = export_to_watertight(mesh)
            print("MC over!")
        if gpu is not None:
            capi, torch = gpu
            dev = torch.device("cuda", torch.cuda.current_device())
            v = torch.as_tensor(np.asarray(mesh.vertices, dtype=np.float32), device=dev)
            f = torch.as_tensor(np.asarray(mesh.faces, dtype=np.int32), device=dev)
            seed = int(np.random.randint(0, 2 ** 31 - 1))
            clouds.append(capi.sample_surface(v, f, sample_num, seed=seed).cpu().numpy())
            used.append(mesh)
            print("process mesh success")
            continue
        pts, tri = mesh.sample(sample_num, return_index=True)
        clouds.append(np.concatenate([pts, mesh.face_normals[tri]], axis=-1, dtype=np.float16))
        used.append(mesh)
        print("process mesh success")
    return clouds, used
