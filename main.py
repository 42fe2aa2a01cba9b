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
from typing import Callable, NamedTuple

import numpy as np
import torch

from MeshAnything.models.meshanything import MeshAnything
from mesh_to_pc import load_cloud, load_mesh, process_mesh_to_pc
from meshanything_b200 import capi


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


def _cloud_items(input_type, path, outliers=None, subsample='random', plane=None, objects=None, smooth=None,
                 colors=False, n_points=4096, k=16):
    """The Dataset entries of one point-cloud file (mesh_to_pc.load_cloud), its stages in this order: `plane` removes
    the support plane, `outliers` the stray points, `smooth` moves the xyz of the rest onto their surface (a pc_normal
    file's normals pass through unchanged), and `objects` splits it into objects, each its own entry with uid
    `{uid}_obj{k}`.  A stage that drops points drops the same rows of the file's normals and colours.  Then, object by
    object: a bare cloud (`pc`) gets normals estimated on the GPU from that object's points alone
    (meshanything_b200.normals), so that their orientation is rooted at its own farthest point, and the 4096 rows the
    model sees are drawn at random without replacement (global numpy RNG, seeded by --seed as the reference does
    through accelerate.set_seed), or with subsample='fps' by farthest-point sampling; the xyz-only copy of a file
    selects the points the file with normals selects under the same seed.  With `colors` every entry also gets
    'colors', float64 [M, 6]: the object's full cloud, xyz in the input's units | rgb, which the generated mesh takes
    its colours from."""
    from meshanything_b200.normals import estimate_normals
    xyz, normals, rgb = load_cloud(path, input_type, colors)
    if input_type == 'pc':   # a bare cloud is refused before its stages, one with normals after the ones that clean it
        assert xyz.shape[0] >= n_points, "input pc_normal should have at least 4096 points"
    for stage, options in ((_remove_plane, plane), (_remove_outliers, outliers)):
        if options is not None:
            keep = stage(xyz, path, options, n_points)
            xyz, normals, rgb = (None if a is None else a[keep] for a in (xyz, normals, rgb))
    if smooth is not None:
        xyz = _smooth(xyz, path, smooth)
    assert xyz.shape[0] >= n_points, "input pc_normal should have at least 4096 points"
    parts = [slice(None)] if objects is None else _split_objects(xyz, path, objects, n_points)
    uid = _uid_of(path)
    entries = []
    for j, part in enumerate(parts):
        obj = xyz[part]
        obj_normals = estimate_normals(obj, k).cpu().numpy() if normals is None else normals[part]
        keep = (_farthest_points(obj, path, n_points) if subsample == 'fps'
                else np.random.choice(obj.shape[0], n_points, replace=False))
        entry = {'pc_normal': np.concatenate([obj[keep], obj_normals[keep].astype(obj.dtype)], axis=1),
                 'uid': uid if objects is None else f"{uid}_obj{j}"}
        if rgb is not None:
            entry['colors'] = np.concatenate([np.asarray(obj, dtype=np.float64), rgb[part]], axis=1)
        entries.append(entry)
    return entries


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


SUBSAMPLERS = ('random', 'fps')
OUTPUT_FRAMES = ('model', 'input')


def _subsampler(subsample):
    if subsample not in SUBSAMPLERS:
        raise ValueError(f"--subsample must be one of {', '.join(SUBSAMPLERS)}, got {subsample!r}")
    return subsample


def _on(value):
    """Whether a Dataset argument of STAGES runs its stage: off is None, False or 'random'."""
    return value not in (None, False, 'random')


class Dataset:
    """Same contract as the reference's Dataset (main.py:15-58): items are {'pc_normal': fp16 (4096, 6), 'uid': str},
    coordinates centred on the bounding box and scaled to max |x| = 0.9995, unit normals asserted; they also carry
    'frame', the metrics.shape_frame of the rows before normalisation, which metrics.to_input_frame applies to put a
    mesh back in the input's coordinates.  The other arguments are the optional stages of point-cloud input (STAGES,
    refused for meshes; _cloud_items runs them): `outliers` None or the keyword arguments of
    meshanything_b200.outliers.remove_outliers (DESIGN.md section 1.3), `subsample` 'random' (the reference's
    np.random.choice) or 'fps' (section 1.4), `plane` None or those of meshanything_b200.plane.remove_plane (section
    1.6), `objects` None or {'distance': e} (section 1.7), `smooth` None or {'k': k} (section 1.8), and `colors`
    (section 1.9): give every item a 'colors' entry, float64 [M, 6], the full cleaned cloud it was drawn from (not the
    4096-point subset), xyz in the input's units | rgb in [0, 1]."""

    def __init__(self, input_type, input_list, mc=False, outliers=None, subsample='random', plane=None, objects=None,
                 smooth=None, colors=False):
        options = dict(outliers=outliers, subsample=_subsampler(subsample), plane=plane, objects=objects,
                       smooth=smooth, colors=colors)
        if input_type in ('pc', 'pc_normal'):
            self.data = [entry for p in input_list for entry in _cloud_items(input_type, p, **options)]
        else:
            for keyword, stage in STAGES.items():
                if _on(options[keyword]):
                    raise ValueError(stage.refusal)
            if input_type != 'mesh':
                raise ValueError(f"unknown input_type {input_type!r}")
            if mc:
                print("First Marching Cubes and then sample point cloud, need several minutes...")
            clouds, _ = process_mesh_to_pc([load_mesh(p) for p in input_list], marching_cubes=mc)
            self.data = [{'pc_normal': c, 'uid': _uid_of(p)} for c, p in zip(clouds, input_list)]
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


def _parser():
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
    return parser


def get_args():
    return _parser().parse_args()


_DEFAULTS = vars(_parser().parse_args([]))


def _arg(args, name):
    """args.<name>, or the command line's default for a namespace built without that flag."""
    return getattr(args, name, _DEFAULTS[name])


def _options(flag, **names):
    """args -> {key: args.<name>} of a stage turned on by --<flag>, or None when it is off."""
    return lambda args: {key: _arg(args, name) for key, name in names.items()} if _arg(args, flag) else None


def _check_share(args, name, square=False):
    """--<name> is a share of the bounding box's longest side: in (0, 1], and above 0 in fp32 (with `square` its
    square, which is what the kernel compares)."""
    d = _arg(args, name)
    if not (np.isfinite(d) and 0 < d <= 1 and (np.float32(d) * np.float32(d) if square else np.float32(d)) > 0):
        raise ValueError(f"--{name} must be in (0, 1] (a share of the bounding box's longest side"
                         f"{', with a square above 0 in fp32' if square else ''}), got {d}")


def _check_outliers(args):
    k, std_ratio, min_component = (_arg(args, 'outlier_' + s) for s in ('neighbors', 'std_ratio', 'min_component'))
    if not 1 <= k <= 64:
        raise ValueError(f"--outlier_neighbors must be in 1..64, got {k}")
    if not (np.isfinite(std_ratio) and np.isfinite(min_component) and min_component >= 0):
        raise ValueError("--outlier_std_ratio must be finite and --outlier_min_component finite and >= 0")


def _check_plane(args):
    _check_share(args, 'plane_distance')
    iterations = _arg(args, 'plane_iterations')
    if not 1 <= iterations <= capi.PLANE_MAX_H:
        raise ValueError(f"--plane_iterations must be in 1..{capi.PLANE_MAX_H}, got {iterations}")


def _check_smooth(args):
    k = _arg(args, 'smooth_neighbors')
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not capi.SMOOTH_MIN_K <= k <= 64:
        raise ValueError(f"--smooth_neighbors must be in {capi.SMOOTH_MIN_K}..64, got {k}")


class _Stage(NamedTuple):
    flag: str            # what turns the stage on, as the messages name it
    options: Callable    # args -> its Dataset argument; _on tells whether that runs the stage
    check: Callable      # args -> ValueError for options out of range (called when the stage runs)
    mesh: str            # why mesh input is refused

    @property
    def refusal(self):
        return f"{self.flag} applies to point-cloud input (--input_type pc or pc_normal): {self.mesh}"


# The optional stages of point-cloud input by their Dataset argument, in the order check_args checks them.
STAGES = {
    'outliers': _Stage('--remove_outliers', _options('remove_outliers', k='outlier_neighbors',
                                                      std_ratio='outlier_std_ratio',
                                                      min_component='outlier_min_component'), _check_outliers,
                       "the points of a mesh are sampled from its surface and have no outliers"),
    'subsample': _Stage('--subsample fps', lambda args: _subsampler(_arg(args, 'subsample')), lambda args: None,
                        "the points of a mesh are already sampled uniformly by area"),
    'plane': _Stage('--remove_plane', _options('remove_plane', distance='plane_distance',
                                                iterations='plane_iterations'), _check_plane,
                    "the points of a mesh are sampled from its own surface, which has no scanned support under it"),
    'objects': _Stage('--split_objects', _options('split_objects', distance='object_distance'),
                      lambda args: _check_share(args, 'object_distance', square=True),
                      "splitting a mesh into its connected parts is not supported"),
    'smooth': _Stage('--smooth', _options('smooth', k='smooth_neighbors'), _check_smooth,
                     "the points of a mesh are sampled exactly from its surface and carry no scanner noise"),
    'colors': _Stage('--transfer_colors', lambda args: bool(_arg(args, 'transfer_colors')),
                     lambda args: _check_share(args, 'color_distance'),
                     "colours of a mesh's own vertices or textures are not read"),
}
outlier_options = STAGES['outliers'].options
plane_options = STAGES['plane'].options
object_options = STAGES['objects'].options
smooth_options = STAGES['smooth'].options
color_options = STAGES['colors'].options


def check_args(args):
    if args.num_samples < 1:
        raise ValueError(f"--num_samples must be >= 1, got {args.num_samples}")
    if args.num_samples > 1 and not args.sampling:
        raise ValueError("--num_samples > 1 needs --sampling: greedy decoding gives the same mesh every time")
    if args.num_samples > 1 and args.continuous_batching:
        raise ValueError("--num_samples > 1 does not run with --continuous_batching: best-of-N scores the candidates "
                         "of a padded batch together")
    for stage in STAGES.values():
        if _on(stage.options(args)):
            if args.input_type == 'mesh':
                raise ValueError(stage.refusal)
            stage.check(args)
    if _arg(args, 'output_frame') not in OUTPUT_FRAMES:
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
    dataset = Dataset(args.input_type, input_list, args.mc, **{k: stage.options(args) for k, stage in STAGES.items()})

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
