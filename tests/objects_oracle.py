"""numpy restatement of csrc/objects.cu (test infrastructure only): splitting a point cloud into objects as DESIGN.md
section 1.7 defines it.

Candidate pairs come from scipy's cKDTree at radius e (1 + 1e-4) in float64 on the fp32 coordinates, a superset of the
pairs that pass the fp32 formula (those are within e (1 + ~4e-7)); the formula itself is one numpy float32 ufunc call
per operation (correctly rounded, never fused).  Components by scipy.sparse.csgraph, relabelled to their minima, then
the ordering rule: labels, object indices, offsets and stats agree with the GPU bit for bit.
"""
import numpy as np

from tests import outliers_oracle as OO

F32, F64 = np.float32, np.float64

frame_map = OO.frame_map


def e_and_e2(distance):
    """(e, e2) = (fp32(distance), fp32(e e))."""
    e = F32(distance)
    return e, F32(e * e)


def d2(p, q):
    """fp32 (dx dx + dy dy) + dz dz of rows p [M, 3] against rows q [M, 3]."""
    d = np.asarray(p, F32) - np.asarray(q, F32)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def edges(points_frame, distance):
    """int64 [M, 2] (i < j): every pair with fp32 d^2 <= e2."""
    from scipy.spatial import cKDTree
    p = np.asarray(points_frame, F32)
    e, e2 = e_and_e2(distance)
    if len(p) < 2:
        return np.zeros((0, 2), np.int64)
    pairs = cKDTree(p.astype(F64)).query_pairs(float(e) * (1 + 1e-4), output_type="ndarray").astype(np.int64)
    return pairs[d2(p[pairs[:, 0]], p[pairs[:, 1]]) <= e2]


def component_minima(n, pairs):
    """int32 [n]: the lowest index of every point's connected component in the graph of `pairs`."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    g = coo_matrix((np.ones(len(pairs), np.int8), (pairs[:, 0], pairs[:, 1])), shape=(n, n))
    _, comp = connected_components(g, directed=False)
    lo = np.full(comp.max() + 1, n, np.int64)
    np.minimum.at(lo, comp, np.arange(n))
    return lo[comp].astype(np.int32)


def order(labels, min_points):
    """(the cluster labels in order: size descending, the lowest label first on ties; their sizes; the objects)."""
    n = len(labels)
    sizes = np.bincount(labels, minlength=n)
    roots = np.nonzero(labels == np.arange(n))[0]
    ranked = roots[np.lexsort((roots, -sizes[roots]))]
    return ranked, sizes[ranked], ranked[sizes[ranked] >= min_points]


def split_objects(points_frame, distance=0.02, min_points=4096, labels=None):
    """Points already in the frame (fp32 [N, 3]) -> dict: labels int32 [N], clusters (labels in order), sizes,
    objects (labels), indices int64 (each object's points ascending, objects in order), offsets int64 [objects + 1],
    and stats int64 [6] as ma_split_objects writes them.  `labels` may be given to skip the graph."""
    p = np.asarray(points_frame, F32)
    n = len(p)
    assert 1 <= n <= 1 << 24 and 1 <= min_points <= n
    if labels is None:
        labels = component_minima(n, edges(p, distance))
    labels = np.asarray(labels, np.int32)
    ranked, sizes, objects = order(labels, min_points)
    rank_of = np.full(n, len(objects), np.int64)
    rank_of[objects] = np.arange(len(objects))
    key = rank_of[labels]
    sel = np.nonzero(key < len(objects))[0]
    indices = sel[np.argsort(key[sel], kind="stable")].astype(np.int64)
    obj_sizes = sizes[:len(objects)]
    offsets = np.concatenate([[0], np.cumsum(obj_sizes)]).astype(np.int64)
    dropped = sizes[len(objects):]
    stats = np.array([len(ranked), len(objects), int(obj_sizes.sum()), len(dropped), int(dropped.sum()),
                      int(dropped.max()) if len(dropped) else 0], np.int64)
    return {"labels": labels, "clusters": ranked, "sizes": sizes, "objects": objects, "indices": indices,
            "offsets": offsets, "stats": stats}


def union_find_labels(n, pairs):
    """An independent restatement: plain union-find with the larger root hooked under the smaller."""
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for a, b in pairs:
        ra, rb = find(int(a)), find(int(b))
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    return np.array([find(i) for i in range(n)], np.int32)


def _shape(kind, m, rng):
    """m points on an object of longest side about 0.3: "sphere", "cube" (surfaces) or "wand" (the golden mesh)."""
    import os
    if kind == "sphere":
        x = rng.normal(size=(m, 3))
        return x / np.linalg.norm(x, axis=1, keepdims=True) * 0.15 + [0, 0, 0.15]
    if kind == "cube":
        f = rng.integers(6, size=m)
        u = rng.random((m, 3))
        u[np.arange(m), f // 2] = f % 2
        return (u - [0.5, 0.5, 0]) * 0.25
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wand_mesh.npz"))
    tri = z["vertices"].astype(F64)[z["faces"]]
    a = rng.random((m, 2))
    a = np.where(a.sum(1, keepdims=True) > 1, 1 - a, a)
    f = rng.integers(len(tri), size=m)
    o = tri[f, 0] + a[:, :1] * (tri[f, 1] - tri[f, 0]) + a[:, 1:] * (tri[f, 2] - tri[f, 0])
    o = o[:, np.argsort(o.max(0) - o.min(0))]                       # standing: the longest axis up
    o = (o - o.min(0)) / (o.max(0) - o.min(0)).max() * 0.3
    o[:, :2] -= o[:, :2].mean(0)
    return o


def table_scene(seed, n=40000, table_share=0.4, stray_share=0.01):
    """A tabletop scan: a sphere, the wand and a cube (longest sides about 0.3) standing apart on a table disc 1.5
    across with four legs, and `stray_share` of the points scattered in the bounding box.  The table is z = 0 with
    Gaussian noise of 0.001 in z.  Returns (points float64 [n, 3], labels int8 [n]: 0 table, 1 sphere, 2 wand, 3 cube,
    4 leg, 5 stray).  A stray within e of an object would join it: strays are kept 0.05 from the objects."""
    rng = np.random.default_rng(seed)
    n_tab, n_str, n_leg = int(table_share * n), int(stray_share * n), n // 10
    n_obj = n - n_tab - n_str - n_leg
    m = [n_obj // 3, n_obj // 3, n_obj - 2 * (n_obj // 3)]
    places = np.array([[-0.4, -0.2, 0.002], [0.35, -0.25, 0.002], [0.0, 0.4, 0.002]])
    objs = [_shape(k, mm, rng) + c for k, mm, c in zip(("sphere", "wand", "cube"), m, places)]
    r = 0.75 * np.sqrt(rng.random(n_tab))
    ang = rng.random(n_tab) * 2 * np.pi
    tab = np.stack([r * np.cos(ang), r * np.sin(ang), rng.normal(0, 0.001, n_tab)], axis=1)
    corner = np.array([[1, 1], [1, -1], [-1, 1], [-1, -1]], F64) * 0.45
    leg = np.concatenate([corner[rng.integers(4, size=n_leg)] + rng.normal(0, 0.01, (n_leg, 2)),
                          -rng.uniform(0.03, 0.6, (n_leg, 1))], axis=1)
    lo, hi = np.array([-0.75, -0.75, -0.6]), np.array([0.75, 0.75, 0.6])
    allobj = np.concatenate(objs)
    stray = np.zeros((0, 3))
    from scipy.spatial import cKDTree
    tree = cKDTree(allobj)
    while len(stray) < n_str:
        s = lo + rng.random((n_str, 3)) * (hi - lo)
        s = s[tree.query(s)[0] > 0.05]
        stray = np.concatenate([stray, s])[:n_str]
    pts = np.concatenate([tab, *objs, leg, stray])
    lab = np.repeat(np.arange(6, dtype=np.int8), [n_tab, *m, n_leg, n_str])
    return pts, lab
