"""Drop-in for /root/reference/main.py (same flags, same outputs) on top of the H100-native MeshAnything.

    python main.py --input_type pc_normal --input_path pc_examples/mouse.npy --out_dir out [--sampling]
    python main.py --input_type pc --input_path scan.npy       # bare (N, 3) cloud: normals estimated on the GPU
    python main.py --input_type pc --input_path scan.npy --remove_outliers   # drop stray points / floaters first
    python main.py --input_type pc --input_path scan.npy --subsample fps     # even coverage of uneven scan density
    python main.py --input_type pc --input_path scan.npy --remove_plane      # drop the table / floor under the object
    python main.py --input_type pc --input_path scan.npy --smooth            # pull scanner noise back onto the surface
    python main.py --input_type pc --input_path scan.npy --remove_plane --split_objects --output_frame input
                                                   # one mesh per object on the table, each where it stands in the scan
    python main.py --input_type pc --input_path scan.ply --remove_plane --transfer_colors
                                                   # vertex colours of the mesh from the scan's red green blue
    torchrun --nproc-per-node 8 main.py --input_type pc_normal --input_dir pcs --batchsize_per_gpu 64

Differences forced by the environment: no accelerate / hf_hub (there is no network) -- one process per
GPU is launched with torchrun, batches are dealt round-robin to the ranks as accelerate's prepared
DataLoader does (main.py:146), and weights come from `--pretrained_weights` (a local safetensors file
with the published keys) or, with `--pretrained_weights synthetic`, from the seeded random checkpoint.
"""
import argparse
import datetime
import os
import time

import numpy as np
import torch

from MeshAnything.models.meshanything import MeshAnything
from mesh_to_pc import load_mesh, process_mesh_to_pc


def _remove_outliers(xyz, path, outliers, n_points=4096):
    """`--remove_outliers`: the indices of the points of xyz [N, 3] that DESIGN.md section 1.3 keeps (on the GPU,
    meshanything_b200.outliers), with one line of counts per input."""
    from meshanything_b200.outliers import remove_outliers
    idx, st = remove_outliers(xyz, **outliers)
    print(f"{_uid_of(path)}: removed {st.removed_statistical} of {st.n_points} points by neighbour distance, "
          f"{st.removed_components} more in {st.components_dropped} of {st.components} components; {st.kept} kept")
    if st.kept < n_points:
        raise ValueError(f"{path}: {st.kept} points remain after outlier removal ({st.removed_statistical} removed by "
                         f"neighbour distance, {st.removed_components} in {st.components_dropped} small components), "
                         f"fewer than the {n_points} the model takes")
    return idx.cpu().numpy()


def _remove_plane(xyz, path, plane, n_points=4096):
    """`--remove_plane`: the indices of the points of xyz [N, 3] that DESIGN.md section 1.6 keeps (on the GPU,
    meshanything_b200.plane): the dominant plane and everything below it go.  The RANSAC seed is drawn from the global
    numpy RNG, so --seed selects it; one line per input with the plane and the counts."""
    from meshanything_b200.plane import remove_plane
    seed = int(np.random.randint(0, 2**62, dtype=np.int64))
    idx, st = remove_plane(xyz, seed=seed, **plane)
    if st.found:
        n = st.normal
        print(f"{_uid_of(path)}: plane n = ({n[0]:.4f}, {n[1]:.4f}, {n[2]:.4f}), d = {st.offset:.4f} (output frame), "
              f"t = {st.threshold:.4g} in input units; removed {st.on} on it and {st.below} below it; {st.kept} of "
              f"{xyz.shape[0]} kept")
    else:
        print(f"{_uid_of(path)}: no plane found ({st.valid_hypotheses} valid hypotheses); {st.kept} points kept")
    if st.kept < n_points:
        raise ValueError(f"{path}: {st.kept} points remain after plane removal ({st.on} on the plane, {st.below} below "
                         f"it), fewer than the {n_points} the model takes")
    return idx.cpu().numpy()


def _smooth(xyz, path, smooth):
    """`--smooth`: xyz [N, 3] projected onto the moving-least-squares surface of DESIGN.md section 1.8 (on the GPU,
    meshanything_b200.smooth), in xyz's dtype and units; every row is kept and nothing is drawn.  One line per input
    with the counts and the displacements in input units."""
    from meshanything_b200.smooth import smooth_points
    out, st = smooth_points(xyz, **smooth)
    print(f"{_uid_of(path)}: smoothed {st.n_points} points (k = {st.k}): {st.quadratic} on their quadratic, "
          f"{st.singular} singular and {st.far} far onto their plane; moved {st.mean_displacement:.4g} on average, "
          f"{st.max_displacement:.4g} at most (input units)")
    return out.cpu().numpy()


def _split_objects(xyz, path, objects, n_points=4096):
    """`--split_objects`: the point indices of every object of xyz [N, 3] that DESIGN.md section 1.7 defines (on the
    GPU, meshanything_b200.objects), objects in order, each ascending; one line per input with the clusters, the
    objects' sizes and the dropped points, e in the input's units."""
    from meshanything_b200.objects import split_objects
    idx, offsets, st = split_objects(xyz, min_points=n_points, **objects)
    print(f"{_uid_of(path)}: {st.clusters} clusters at e = {st.distance:.4g} in input units; {st.objects} objects of "
          f"{', '.join(str(s) for s in st.sizes) or 'no'} points; dropped {st.dropped_points} points in "
          f"{st.dropped_clusters} smaller clusters (the largest {st.largest_dropped})")
    if st.objects == 0:
        raise ValueError(f"{path}: no cluster of {n_points} points at e = {st.distance:.4g} ({st.clusters} clusters, "
                         f"the largest of {st.largest_dropped} points), fewer than the {n_points} the model takes")
    idx, offsets = idx.cpu().numpy(), offsets.cpu().numpy()
    return [idx[offsets[k]:offsets[k + 1]] for k in range(st.objects)]


def _farthest_points(xyz, path, n_points=4096):
    """`--subsample fps`: the picks of farthest-point sampling (DESIGN.md section 1.4, on the GPU,
    meshanything_b200.subsample) from a start drawn from the global numpy RNG, so --seed still selects the subset; one
    line per input with the covering radius."""
    from meshanything_b200.subsample import farthest_point_sample
    n = xyz.shape[0]
    idx, r2 = farthest_point_sample(xyz, n_points, np.random.randint(n))
    print(f"{_uid_of(path)}: {n_points} of {n} points by farthest-point sampling; every point within "
          f"{float(np.sqrt(r2[-1].item())):.4g} of one (output frame)")
    return idx.cpu().numpy()


def _rows(a, idx):
    """a[idx], or None for None: the colours of a cloud follow its rows through every stage that drops rows."""
    return None if a is None else a[idx]


def _colored(cloud, xyz, rgb):
    """cloud, or with rgb (`--transfer_colors`) (cloud, the full cleaned cloud float64 [M, 6]: xyz in the input's units |
    rgb), which the generated mesh takes its colours from."""
    if rgb is None:
        return cloud
    return cloud, np.concatenate([np.asarray(xyz, dtype=np.float64), np.asarray(rgb, dtype=np.float64)], axis=1)


def _subsample_points(path, n_points=4096, outliers=None, subsample='random', plane=None, objects=None, smooth=None,
                      colors=False):
    """`--input_type pc_normal`: an .npy of >= 4096 (xyz, normal) rows; a random 4096-subset without replacement
    (global numpy RNG, seeded by --seed as the reference does through accelerate.set_seed), or with
    subsample='fps' the farthest-point subset of the xyz columns.  With `outliers` (the keyword arguments of
    meshanything_b200.outliers.remove_outliers) the rows are first cleaned by their xyz; with `plane` (the keyword
    arguments of meshanything_b200.plane.remove_plane) the support plane goes before that.  With `smooth` ({'k': k})
    the xyz columns of the cleaned rows are smoothed; the normals pass through unchanged.  With `objects` ({'distance':
    e}) the cleaned cloud is split into objects and a list of one subset per object is returned, drawn in object
    order.  With `colors` the file is (N, 9), xyz | normal | rgb: the colours follow their rows, and every subset comes
    with its full cleaned cloud (see _colored)."""
    cloud, rgb = np.load(path), None
    if colors:
        if cloud.ndim != 2 or cloud.shape[1] != 9:
            raise ValueError(f"{path}: --transfer_colors reads a coloured pc_normal cloud as an array of shape (N, 9), "
                             f"xyz | normal | rgb, got {cloud.shape}")
        from mesh_to_pc import check_rgb
        cloud, rgb = cloud[:, :6], check_rgb(path, cloud[:, 6:])
    if plane is not None:
        keep = _remove_plane(cloud[:, :3], path, plane, n_points)
        cloud, rgb = cloud[keep], _rows(rgb, keep)
    if outliers is not None:
        keep = _remove_outliers(cloud[:, :3], path, outliers, n_points)
        cloud, rgb = cloud[keep], _rows(rgb, keep)
    if smooth is not None:
        cloud = cloud.copy()
        cloud[:, :3] = _smooth(cloud[:, :3], path, smooth)
    assert cloud.shape[0] >= n_points, "input pc_normal should have at least 4096 points"
    if objects is not None:
        return [_colored(_subset(cloud[part], path, n_points, subsample), cloud[part, :3], _rows(rgb, part))
                for part in _split_objects(cloud[:, :3], path, objects, n_points)]
    return _colored(_subset(cloud, path, n_points, subsample), cloud[:, :3], rgb)


def _subset(cloud, path, n_points, subsample):
    """The 4096 rows of a cloud the model sees: random without replacement (global numpy RNG) or farthest points."""
    if subsample == 'fps':
        return cloud[_farthest_points(cloud[:, :3], path, n_points)]
    keep = np.random.choice(cloud.shape[0], n_points, replace=False)
    return cloud[keep]


def _points_with_normals(path, n_points=4096, k=16, outliers=None, subsample='random', plane=None, objects=None,
                         smooth=None, colors=False):
    """`--input_type pc`: a bare cloud (.npy (N, 3) or vertex-only .ply) of >= 4096 points.  Normals are estimated on
    the GPU from all N points (meshanything_b200.normals), then the same 4096-subset as `pc_normal` is drawn: the
    xyz-only copy of a file selects the points the file with normals selects under the same seed.  With `outliers`
    the cloud is cleaned first, and normals and subset come from the kept points; `plane` removes the support plane
    before that; `smooth` smooths the cleaned points before their normals are estimated.  With `objects` the cleaned
    cloud is split into objects first, and every object gets its own normals (estimated on its points alone, so that
    their orientation is rooted at its own farthest point) and subset, in object order: a list of one cloud per object
    is returned.  With `colors` the file carries rgb (mesh_to_pc.load_points): the colours follow their rows, and every
    cloud comes with its full cleaned cloud (see _colored)."""
    from mesh_to_pc import load_points
    xyz, rgb = load_points(path, colors=True) if colors else (load_points(path), None)
    if not np.issubdtype(xyz.dtype, np.floating):
        xyz = xyz.astype(np.float64)
    assert xyz.shape[0] >= n_points, "input pc_normal should have at least 4096 points"
    if plane is not None:
        keep = _remove_plane(xyz, path, plane, n_points)
        xyz, rgb = xyz[keep], _rows(rgb, keep)
    if outliers is not None:
        keep = _remove_outliers(xyz, path, outliers, n_points)
        xyz, rgb = xyz[keep], _rows(rgb, keep)
    if smooth is not None:
        xyz = _smooth(xyz, path, smooth)
    if objects is not None:
        return [_colored(_with_normals(xyz[part], path, n_points, k, subsample), xyz[part], _rows(rgb, part))
                for part in _split_objects(xyz, path, objects, n_points)]
    return _colored(_with_normals(xyz, path, n_points, k, subsample), xyz, rgb)


def _with_normals(xyz, path, n_points, k, subsample):
    """Normals of every point of xyz on the GPU, then the subset: (4096, 6) rows."""
    from meshanything_b200.normals import estimate_normals
    normals = estimate_normals(xyz, k).cpu().numpy()
    if subsample == 'fps':
        keep = _farthest_points(xyz, path, n_points)
    else:
        keep = np.random.choice(xyz.shape[0], n_points, replace=False)
    return np.concatenate([xyz[keep], normals[keep].astype(xyz.dtype)], axis=1)


def _vertex_colors(item, vertices, faces, output_frame, distance):
    """`--transfer_colors`: rgb [V, 3] of the final mesh (vertices in the output frame) from the item's full cleaned
    cloud (DESIGN.md section 1.9, on the GPU, meshanything_b200.colors).  The mesh is first put in the input's units
    (metrics.to_input_frame), so that both output frames give the same colours; one line per item with the counts."""
    from meshanything_b200.colors import transfer_colors
    from meshanything_b200.metrics import to_input_frame
    if len(faces) == 0:
        return np.zeros((len(vertices), 3))
    v = torch.as_tensor(np.asarray(vertices, dtype=np.float64))
    if output_frame == 'model':
        v = to_input_frame(v, item['frame'])
    cloud = item['colors']
    rgb, st = transfer_colors(v, np.asarray(faces, dtype=np.int64), cloud[:, :3], cloud[:, 3:], distance)
    print(f"{item['uid']}: coloured {len(v)} vertices from {st.used} of {st.n_points} points ({st.beyond} farther than "
          f"{distance:g} of the cloud's longest side); {st.fallback_vertices} vertices took their nearest point's colour")
    return rgb.cpu().numpy()


def _uid_of(path):
    return path.split('/')[-1].split('.')[0]


_NO_MESH_OUTLIERS = ("--remove_outliers applies to point-cloud input (--input_type pc or pc_normal): the points of a "
                     "mesh are sampled from its surface and have no outliers")
_NO_MESH_FPS = ("--subsample fps applies to point-cloud input (--input_type pc or pc_normal): the points of a mesh are "
                "already sampled uniformly by area")
_NO_MESH_OBJECTS = ("--split_objects applies to point-cloud input (--input_type pc or pc_normal): splitting a mesh into "
                    "its connected parts is not supported")
_NO_MESH_SMOOTH = ("--smooth applies to point-cloud input (--input_type pc or pc_normal): the points of a mesh are "
                   "sampled exactly from its surface and carry no scanner noise")
_NO_MESH_COLORS = ("--transfer_colors applies to point-cloud input (--input_type pc or pc_normal): colours of a mesh's "
                   "own vertices or textures are not read")
_NO_MESH_PLANE = ("--remove_plane applies to point-cloud input (--input_type pc or pc_normal): the points of a mesh are "
                  "sampled from its own surface, which has no scanned support under it")
SUBSAMPLERS = ('random', 'fps')
OUTPUT_FRAMES = ('model', 'input')


def _check_subsample(input_type, subsample):
    if subsample not in SUBSAMPLERS:
        raise ValueError(f"--subsample must be one of {', '.join(SUBSAMPLERS)}, got {subsample!r}")
    if subsample == 'fps' and input_type not in ('pc', 'pc_normal'):
        raise ValueError(_NO_MESH_FPS)


class Dataset:
    """Same contract as the reference's Dataset (main.py:15-58): items are {'pc_normal': fp16 (4096, 6), 'uid': str},
    coordinates centred on the bounding box and scaled to max |x| = 0.9995, unit normals asserted.  `outliers` (point
    clouds only): None, or the keyword arguments of meshanything_b200.outliers.remove_outliers, to clean every cloud
    before normals and subset.  `subsample` (point clouds only): 'random' (the reference's np.random.choice) or 'fps'
    (farthest-point sampling on the GPU, DESIGN.md section 1.4).  `plane` (point clouds only): None, or the keyword
    arguments of meshanything_b200.plane.remove_plane, to remove the support plane (a table, the floor) first.
    `objects` (point clouds only): None, or {'distance': e}, to split every cloud after plane and outlier removal into
    objects (DESIGN.md section 1.7), each its own item with uid `{uid}_obj{k}`.  `smooth` (point clouds only): None, or
    {'k': k}, to smooth every cloud after plane and outlier removal (DESIGN.md section 1.8; for pc_normal only the xyz
    columns move).  Items also carry 'frame', the
    metrics.shape_frame of the rows before normalisation, which metrics.to_input_frame applies to put a mesh back in
    the input's coordinates.  `colors` (point clouds only, `--transfer_colors`): read the files' colours, and give every
    item a 'colors' entry, float64 [M, 6]: the full cleaned cloud it was drawn from (after plane and outlier removal,
    smoothing and splitting; not the 4096-point subset), xyz in the input's units | rgb in [0, 1]."""

    def __init__(self, input_type, input_list, mc=False, outliers=None, subsample='random', plane=None, objects=None,
                 smooth=None, colors=False):
        if outliers is not None and input_type not in ('pc', 'pc_normal'):
            raise ValueError(_NO_MESH_OUTLIERS)
        if plane is not None and input_type not in ('pc', 'pc_normal'):
            raise ValueError(_NO_MESH_PLANE)
        if objects is not None and input_type not in ('pc', 'pc_normal'):
            raise ValueError(_NO_MESH_OBJECTS)
        if smooth is not None and input_type not in ('pc', 'pc_normal'):
            raise ValueError(_NO_MESH_SMOOTH)
        if colors and input_type not in ('pc', 'pc_normal'):
            raise ValueError(_NO_MESH_COLORS)
        _check_subsample(input_type, subsample)
        kw = dict(outliers=outliers, subsample=subsample, plane=plane, objects=objects)
        if smooth is not None:
            kw['smooth'] = smooth
        if colors:
            kw['colors'] = True
        if input_type == 'pc_normal':
            clouds = [_subsample_points(p, **kw) for p in input_list]
        elif input_type == 'pc':
            clouds = [_points_with_normals(p, **kw) for p in input_list]
        elif input_type == 'mesh':
            if mc:
                print("First Marching Cubes and then sample point cloud, need several minutes...")
            clouds, _ = process_mesh_to_pc([load_mesh(p) for p in input_list], marching_cubes=mc)
        else:
            raise ValueError(f"unknown input_type {input_type!r}")
        if objects is None:
            self.data = [{'pc_normal': c, 'uid': _uid_of(p)} for c, p in zip(clouds, input_list)]
        else:
            self.data = [{'pc_normal': c, 'uid': f"{_uid_of(p)}_obj{k}"}
                         for cs, p in zip(clouds, input_list) for k, c in enumerate(cs)]
        if colors:
            for entry in self.data:
                entry['pc_normal'], entry['colors'] = entry['pc_normal']
        print(f"dataset total data samples: {len(self.data)}")

    def __len__(self):
        return len(self.data)

    def __getitem__(self, idx):
        from meshanything_b200.inputs import normalize_pc_normal
        from meshanything_b200.metrics import shape_frame
        entry = self.data[idx]
        item = {'pc_normal': normalize_pc_normal(entry['pc_normal']), 'uid': entry['uid'],
                'frame': shape_frame(entry['pc_normal'][:, :3])}
        if 'colors' in entry:
            item['colors'] = entry['colors']
        return item


_FLAGS = [  # (flag, default, type) -- the reference's command line (main.py:60-89)
    ('--llm', "facebook/opt-350m", str), ('--input_dir', None, str), ('--input_path', None, str),
    ('--out_dir', "inference_out", str), ('--pretrained_weights', "MeshAnything_350m.pth", str),
    ('--codebook_size', 8192, int), ('--codebook_dim', 1024, int), ('--n_max_triangles', 800, int),
    ('--batchsize_per_gpu', 1, int), ('--seed', 0, int),
]


def get_args():
    parser = argparse.ArgumentParser("MeshAnything", add_help=False)
    for flag, default, typ in _FLAGS:
        parser.add_argument(flag, default=default, type=typ)
    # 'pc' (the reference's default, which it does not implement): a bare (N, 3) cloud, normals estimated on the GPU
    parser.add_argument('--input_type', choices=['mesh', 'pc_normal', 'pc'], default='pc',
                        help="Type of the asset to process (default: pc)")
    for switch in ('--mc', '--sampling'):
        parser.add_argument(switch, default=False, action="store_true")
    # not in the reference: run this rank's shapes through `batchsize_per_gpu` decoder cache slots, refilling a slot as
    # soon as its mesh is complete, instead of padded batches (SURVEY.md section 8(f)2; MeshAnything.forward_queue)
    parser.add_argument('--continuous_batching', default=False, action="store_true")
    # not in the reference: sample N meshes of every shape in one batch and keep the one closest to the input cloud
    # (Chamfer distance on the GPU; MeshAnything.forward_candidates) instead of re-rolling --seed by hand
    parser.add_argument('--num_samples', default=1, type=int)
    # not in the reference: drop stray points and small floating clusters of a scan before normals and normalisation
    # (DESIGN.md section 1.3; meshanything_b200.outliers); the parameters follow Open3D's remove_statistical_outlier
    parser.add_argument('--remove_outliers', default=False, action="store_true")
    parser.add_argument('--outlier_neighbors', default=16, type=int)
    parser.add_argument('--outlier_std_ratio', default=2.0, type=float)
    parser.add_argument('--outlier_min_component', default=0.01, type=float)
    # not in the reference: how the 4096 points the model sees are picked from a point cloud -- 'random' (the
    # reference's np.random.choice) or 'fps', farthest-point sampling on the GPU, which covers a scan evenly whatever
    # its density (DESIGN.md section 1.4; meshanything_b200.subsample)
    parser.add_argument('--subsample', default='random', choices=SUBSAMPLERS)
    # not in the reference: remove the plane a scanned object stands on (a table, a turntable, the floor) and
    # everything below it, by RANSAC and a least-squares refit on the GPU (DESIGN.md section 1.6; meshanything_b200.plane)
    parser.add_argument('--remove_plane', default=False, action="store_true")
    parser.add_argument('--plane_distance', default=0.01, type=float)
    parser.add_argument('--plane_iterations', default=1000, type=int)
    # not in the reference: split every cloud into objects (connected components at --object_distance of the bounding
    # box's longest side; DESIGN.md section 1.7; meshanything_b200.objects) and mesh each one on its own
    parser.add_argument('--split_objects', default=False, action="store_true")
    parser.add_argument('--object_distance', default=0.02, type=float)
    # not in the reference: pull scanner noise back onto the surface by projecting every point onto the quadratic
    # fitted to its --smooth_neighbors nearest points (moving least squares on the GPU; DESIGN.md section 1.8;
    # meshanything_b200.smooth), after plane and outlier removal and before normals and the subset; for pc_normal input
    # only the xyz columns move, the file's normals pass through unchanged
    parser.add_argument('--smooth', default=False, action="store_true",
                        help="smooth scanner noise by moving-least-squares projection (point-cloud input; for "
                             "pc_normal only xyz moves, the normals pass through unchanged)")
    parser.add_argument('--smooth_neighbors', default=24, type=int,
                        help="neighbours of each point's local fit for --smooth, 5..64 (default 24)")
    # not in the reference: write meshes in the model's [-0.5, 0.5) frame (model, the reference's output) or back in
    # the input's coordinates (input: c + L v with the bounding box centre c and longest side L of the shape's points)
    parser.add_argument('--output_frame', default='model', choices=OUTPUT_FRAMES)
    # not in the reference: colour the mesh's vertices from the scan's per-point red green blue (a .ply with colour
    # properties, an (N, 6) xyz | rgb .npy for pc, an (N, 9) xyz | normal | rgb .npy for pc_normal) instead of the
    # constant orange; points farther than --color_distance of the cloud's longest side from the mesh are ignored
    # (DESIGN.md section 1.9; meshanything_b200.colors)
    parser.add_argument('--transfer_colors', default=False, action="store_true",
                        help="colour the mesh's vertices from the scan's per-point colours (point-cloud input)")
    parser.add_argument('--color_distance', default=0.05, type=float,
                        help="points farther than this share of the cloud's longest side from the mesh give no colour, "
                             "in (0, 1] (default 0.05)")
    return parser.parse_args()


def outlier_options(args):
    """The `outliers` argument of Dataset from the command line: None without --remove_outliers."""
    if not args.remove_outliers:
        return None
    return {'k': args.outlier_neighbors, 'std_ratio': args.outlier_std_ratio,
            'min_component': args.outlier_min_component}


def plane_options(args):
    """The `plane` argument of Dataset from the command line: None without --remove_plane."""
    if not getattr(args, 'remove_plane', False):
        return None
    return {'distance': getattr(args, 'plane_distance', 0.01), 'iterations': getattr(args, 'plane_iterations', 1000)}


def object_options(args):
    """The `objects` argument of Dataset from the command line: None without --split_objects."""
    if not getattr(args, 'split_objects', False):
        return None
    return {'distance': getattr(args, 'object_distance', 0.02)}


def smooth_options(args):
    """The `smooth` argument of Dataset from the command line: None without --smooth."""
    if not getattr(args, 'smooth', False):
        return None
    return {'k': getattr(args, 'smooth_neighbors', 24)}


def color_options(args):
    """The `colors` argument of Dataset from the command line."""
    return bool(getattr(args, 'transfer_colors', False))


def check_args(args):
    if args.num_samples < 1:
        raise ValueError(f"--num_samples must be >= 1, got {args.num_samples}")
    if args.num_samples > 1 and not args.sampling:
        raise ValueError("--num_samples > 1 needs --sampling: greedy decoding gives the same mesh every time")
    if args.num_samples > 1 and args.continuous_batching:
        raise ValueError("--num_samples > 1 does not run with --continuous_batching: best-of-N scores the candidates "
                         "of a padded batch together")
    if args.remove_outliers:
        if args.input_type == 'mesh':
            raise ValueError(_NO_MESH_OUTLIERS)
        if not 1 <= args.outlier_neighbors <= 64:
            raise ValueError(f"--outlier_neighbors must be in 1..64, got {args.outlier_neighbors}")
        if not (np.isfinite(args.outlier_std_ratio) and np.isfinite(args.outlier_min_component)
                and args.outlier_min_component >= 0):
            raise ValueError("--outlier_std_ratio must be finite and --outlier_min_component finite and >= 0")
    _check_subsample(args.input_type, getattr(args, 'subsample', 'random'))   # namespaces built without the flag
    if getattr(args, 'remove_plane', False):
        if args.input_type == 'mesh':
            raise ValueError(_NO_MESH_PLANE)
        distance = getattr(args, 'plane_distance', 0.01)
        iterations = getattr(args, 'plane_iterations', 1000)
        if not (np.isfinite(distance) and 0 < distance <= 1 and np.float32(distance) > 0):
            raise ValueError(f"--plane_distance must be in (0, 1] (a share of the bounding box's longest side), got "
                             f"{distance}")
        if not 1 <= iterations <= 65536:
            raise ValueError(f"--plane_iterations must be in 1..65536, got {iterations}")
    if getattr(args, 'split_objects', False):
        if args.input_type == 'mesh':
            raise ValueError(_NO_MESH_OBJECTS)
        distance = getattr(args, 'object_distance', 0.02)
        if not (np.isfinite(distance) and 0 < distance <= 1 and np.float32(distance) * np.float32(distance) > 0):
            raise ValueError(f"--object_distance must be in (0, 1] (a share of the bounding box's longest side, with a "
                             f"square above 0 in fp32), got {distance}")
    if getattr(args, 'smooth', False):
        if args.input_type == 'mesh':
            raise ValueError(_NO_MESH_SMOOTH)
        k = getattr(args, 'smooth_neighbors', 24)
        if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 5 <= k <= 64:
            raise ValueError(f"--smooth_neighbors must be in 5..64, got {k}")
    if getattr(args, 'transfer_colors', False):
        if args.input_type == 'mesh':
            raise ValueError(_NO_MESH_COLORS)
        distance = getattr(args, 'color_distance', 0.05)
        if not (np.isfinite(distance) and 0 < distance <= 1 and np.float32(distance) > 0):
            raise ValueError(f"--color_distance must be in (0, 1] (a share of the bounding box's longest side), got "
                             f"{distance}")
    if getattr(args, 'output_frame', 'model') not in OUTPUT_FRAMES:
        raise ValueError(f"--output_frame must be one of {', '.join(OUTPUT_FRAMES)}, got {args.output_frame!r}")


def load_model(args, device=None):
    model = MeshAnything(args)
    print("load model over!!!")
    if args.pretrained_weights == "synthetic":
        from meshanything_b200 import checkpoint
        tensors = checkpoint.synthetic_state_dict(0)
    else:
        from safetensors import safe_open
        if not os.path.exists(args.pretrained_weights):
            raise FileNotFoundError(f"{args.pretrained_weights}: put the published MeshAnything_350m.pth (safetensors) "
                                    "here, or pass --pretrained_weights synthetic")
        tensors = {}
        with safe_open(args.pretrained_weights, framework="pt", device="cpu") as f:
            for k in f.keys():
                tensors[k] = f.get_tensor(k)
    model.load_state_dict(tensors, strict=True, device=device)
    print("load weights over!!!")
    return model


def fix_winding(vertices, tri):
    """What `trimesh.Trimesh.fix_normals` does to the faces (main.py:166 of the reference), in numpy: make the winding
    consistent across every shared edge (breadth-first over face adjacency), then flip each connected component whose
    signed volume is negative so that normals point outwards."""
    tri = np.array(tri, dtype=np.int64, copy=True)
    nf = len(tri)
    if nf == 0:
        return tri
    # undirected edge -> faces that use it, with the direction each face traverses it in
    edges = {}
    for f in range(nf):
        for k in range(3):
            a, b = int(tri[f, k]), int(tri[f, (k + 1) % 3])
            if a != b:
                edges.setdefault((min(a, b), max(a, b)), []).append((f, a < b))
    adj = [[] for _ in range(nf)]
    for users in edges.values():
        if len(users) == 2:                       # manifold edge: consistent iff traversed in opposite directions
            (f0, d0), (f1, d1) = users
            adj[f0].append((f1, d0 == d1))
            adj[f1].append((f0, d0 == d1))
    comp = -np.ones(nf, dtype=np.int64)
    flip = np.zeros(nf, dtype=bool)
    ncomp = 0
    for seed in range(nf):
        if comp[seed] >= 0:
            continue
        comp[seed] = ncomp
        queue = [seed]
        while queue:
            f = queue.pop()
            for g, same_dir in adj[f]:
                if comp[g] < 0:
                    comp[g] = ncomp
                    flip[g] = flip[f] ^ same_dir     # same direction on the shared edge = opposite orientation
                    queue.append(g)
        ncomp += 1
    tri[flip] = tri[flip][:, ::-1]
    t = np.asarray(vertices, dtype=np.float64)[tri]
    vol6 = np.einsum("ij,ij->i", t[:, 0], np.cross(t[:, 1], t[:, 2]))
    for c in range(ncomp):
        sel = comp == c
        if vol6[sel].sum() < 0:
            tri[sel] = tri[sel][:, ::-1]
    return tri


def export_obj(path, faces_xyz, vertex_colors=None):
    """merge_vertices + unique_faces + fix_normals + orange face colour of main.py:161-174 (trimesh when available,
    the numpy equivalents otherwise).  With `vertex_colors`, a function of the final (vertices float64 [V, 3], faces
    int64 [F, 3]) returning rgb [V, 3] in [0, 1], the vertices get those colours instead of the orange."""
    vertices = faces_xyz.reshape(-1, 3)
    triangles = np.arange(len(vertices)).reshape(-1, 3)
    try:
        import trimesh
        mesh = trimesh.Trimesh(vertices=vertices, faces=triangles, force="mesh", merge_primitives=True)
        mesh.merge_vertices()
        mesh.update_faces(mesh.unique_faces())
        mesh.fix_normals()
        if vertex_colors is None:
            mesh.visual.face_colors = np.tile(np.array([255, 165, 0, 255], dtype=np.uint8), (len(mesh.faces), 1))
        else:
            rgb = np.asarray(vertex_colors(np.asarray(mesh.vertices, dtype=np.float64),
                                           np.asarray(mesh.faces, dtype=np.int64)), dtype=np.float64)
            mesh.visual.vertex_colors = np.concatenate(
                [np.round(rgb * 255).astype(np.uint8), np.full((len(rgb), 1), 255, np.uint8)], axis=1)
        mesh.export(path)
        return len(mesh.faces)
    except ImportError:
        uniq, inv = np.unique(np.round(vertices, 8), axis=0, return_inverse=True)
        tri = inv.reshape(-1)[triangles]
        _, keep = np.unique(np.sort(tri, axis=1), axis=0, return_index=True)
        tri = fix_winding(uniq, tri[np.sort(keep)])
        rgb = None if vertex_colors is None else np.asarray(vertex_colors(uniq, tri), dtype=np.float64)
        with open(path, "w") as f:
            for k, v in enumerate(uniq):
                if rgb is None:
                    f.write(f"v {v[0]:.8f} {v[1]:.8f} {v[2]:.8f} 1.00000000 0.64705882 0.00000000\n")
                else:
                    f.write(f"v {v[0]:.8f} {v[1]:.8f} {v[2]:.8f} {rgb[k, 0]:.8f} {rgb[k, 1]:.8f} {rgb[k, 2]:.8f}\n")
            for t in tri:
                f.write(f"f {t[0] + 1} {t[1] + 1} {t[2] + 1}\n")
        return len(tri)


if __name__ == "__main__":
    args = get_args()
    check_args(args)
    from meshanything_b200 import parallel
    rank, world, local = parallel.init_from_env()
    cur_time = datetime.datetime.now().strftime("%d_%H-%M-%S")
    checkpoint_dir = os.path.join(args.out_dir, cur_time)
    os.makedirs(checkpoint_dir, exist_ok=True)
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    model = load_model(args, device)

    if args.input_dir is not None:
        input_list = sorted(os.listdir(args.input_dir))
        if args.input_type == 'pc_normal':
            input_list = [os.path.join(args.input_dir, x) for x in input_list if x.endswith('.npy')]
        elif args.input_type == 'pc':
            input_list = [os.path.join(args.input_dir, x) for x in input_list if x.endswith('.npy') or x.endswith('.ply')]
        else:
            input_list = [os.path.join(args.input_dir, x) for x in input_list
                          if x.endswith('.ply') or x.endswith('.obj') or x.endswith('.npy')]
    elif args.input_path is not None:
        input_list = [args.input_path]
    else:
        raise ValueError("input_dir or input_path must be provided.")
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    dataset = Dataset(args.input_type, input_list, args.mc, outliers=outlier_options(args), subsample=args.subsample,
                      plane=plane_options(args), objects=object_options(args), smooth=smooth_options(args),
                      colors=color_options(args))

    bs = args.batchsize_per_gpu
    batches = [list(range(i, min(i + bs, len(dataset)))) for i in range(0, len(dataset), bs)]
    begin_time = time.time()
    print("Generation Start!!!")

    def save(item, recon_mesh):
        recon_mesh = recon_mesh[~torch.isnan(recon_mesh[:, 0, 0])]
        if args.output_frame == 'input':
            from meshanything_b200.metrics import to_input_frame
            recon_mesh = to_input_frame(recon_mesh, item['frame'])
        save_path = os.path.join(checkpoint_dir, f'{item["uid"]}_gen.obj')
        colors = None
        if 'colors' in item:
            def colors(vertices, faces):
                return _vertex_colors(item, vertices, faces, args.output_frame, args.color_distance)
        export_obj(save_path, recon_mesh.cpu().numpy(), colors)
        print(f"{save_path} Over!!")

    if args.continuous_batching:
        mine = [dataset[i] for i in range(rank, len(dataset), world)]   # shapes are independent: round-robin by rank
        outs = model.forward_queue((torch.from_numpy(it['pc_normal']) for it in mine), sampling=args.sampling,
                                   slots=max(1, bs))
        for it, recon_mesh in zip(mine, outs):
            save(it, recon_mesh)
        batches = []
    for bi, idxs in enumerate(batches):
        if bi % world != rank:
            continue
        items = [dataset[i] for i in idxs]
        pc = torch.from_numpy(np.stack([it['pc_normal'] for it in items]))
        if args.num_samples > 1:
            res = model.forward_candidates(pc, args.num_samples)
            chamfer, nc, index = res.chamfer.cpu().tolist(), res.normal_consistency.cpu().tolist(), res.index.tolist()
            for batch_id, it in enumerate(items):
                for k in range(args.num_samples):
                    kept = "  <- kept" if k == index[batch_id] else ""
                    print(f"{it['uid']} sample {k}: chamfer {chamfer[batch_id][k]:.6f} "
                          f"normal consistency {nc[batch_id][k]:.4f}{kept}")
                save(it, res.best[batch_id])
            continue
        outputs = model(pc, sampling=args.sampling)
        for batch_id, it in enumerate(items):
            save(it, outputs[batch_id])
    print(f"Total time: {time.time() - begin_time}")
