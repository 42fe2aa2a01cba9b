"""numpy restatement of csrc/plane.cu (test infrastructure only): removal of the dominant plane of a point cloud as
DESIGN.md section 1.6 defines it.

The hypothesis stream is surface_oracle's Philox4x32-10 with the plane tag, every fp32 operation is one numpy ufunc
call on float32 arrays (correctly rounded, never fused), every fp64 sum is outliers_oracle.fixed_sum (tiles of 256
indices in order, then the tile partials in order; off-plane points add +0), and the refit normal is
normals_oracle.jacobi with the smallest_vector rule: planes, counts, the refit plane, the mask and every stat agree
with the GPU bit for bit.
"""
import numpy as np

from tests import normals_oracle as NO
from tests import outliers_oracle as OO
from tests import surface_oracle as SO

F32, F64 = np.float32, np.float64
TAGS = (0x504c414e, 0x4d455348, 0x414e5954)      # "PLAN", "MESH", "ANYT": the hypotheses' stream tag
INVALID = np.array([0, 0, 0, np.inf], F32)      # the stored plane of an invalid hypothesis: no point is on it

frame_map = OO.frame_map


def hypothesis_indices(n, H, seed):
    """[H, 3] int64: i_j = (c_j n) >> 32 of Philox4x32-10 with counter (h, TAGS), key (seed mod 2^32, seed >> 32)."""
    seed = int(seed)
    assert 0 <= seed < 1 << 64 and 1 <= n <= 1 << 24
    c = SO.philox4x32_10((np.arange(H, dtype=np.uint64), *TAGS), (seed & 0xFFFFFFFF, seed >> 32))
    return np.stack([((w.astype(np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64) for w in c[:3]], axis=1)


def hypotheses(p, H, seed):
    """(planes fp32 [H, 4] = (nx, ny, nz, d), valid bool [H]) of the points already in the frame."""
    p = np.asarray(p, F32)
    idx = hypothesis_indices(len(p), H, seed)
    a, b, c = p[idx[:, 0]], p[idx[:, 1]], p[idx[:, 2]]
    u, w = b - a, c - a
    mx = u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1]
    my = u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2]
    mz = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
    with np.errstate(all="ignore"):
        ln = np.sqrt((mx * mx + my * my) + mz * mz)
        ok = (ln > 0) & (ln < np.inf)
        ls = np.where(ok, ln, F32(1))
        nx, ny, nz = mx / ls, my / ls, mz / ls
        d = -((nx * a[:, 0] + ny * a[:, 1]) + nz * a[:, 2])
    planes = np.stack([nx, ny, nz, d], axis=1).astype(F32)
    planes[~ok] = INVALID
    return planes, ok


def signed_distance(planes, p):
    """fp32 ((nx px + ny py) + nz pz) + d of planes [H, 4] against points [N, 3]: [H, N]."""
    pl, p = np.asarray(planes, F32), np.asarray(p, F32)
    with np.errstate(all="ignore"):
        return ((pl[:, 0:1] * p[None, :, 0] + pl[:, 1:2] * p[None, :, 1]) + pl[:, 2:3] * p[None, :, 2]) + pl[:, 3:4]


def counts(planes, p, t, budget=1 << 23):
    """On-plane points (|s| <= t) of every plane: int64 [H]."""
    planes = np.asarray(planes, F32)
    out = np.empty(len(planes), np.int64)
    step = max(1, budget // max(1, len(p)))
    for s in range(0, len(planes), step):
        out[s:s + step] = (np.abs(signed_distance(planes[s:s + step], p)) <= F32(t)).sum(axis=1)
    return out


def refit(p, on):
    """The least-squares plane of the points p[on]: (fp32 (nx, ny, nz, d), fp64 centroid [3], fp64 moments [6],
    fp64 unit normal [3])."""
    q = np.asarray(p, F32).astype(F64)
    cnt = F64(int(on.sum()))
    z = np.where(on[:, None], q, F64(0))
    cent = np.array([OO.fixed_sum(z[:, a]) for a in range(3)], F64) / cnt
    d = q - cent
    prods = [d[:, 0] * d[:, 0], d[:, 0] * d[:, 1], d[:, 0] * d[:, 2], d[:, 1] * d[:, 1], d[:, 1] * d[:, 2],
             d[:, 2] * d[:, 2]]
    mom = np.array([OO.fixed_sum(np.where(on, x, F64(0))) for x in prods], F64)
    diag, V = NO.jacobi(mom[None])
    m = 0                                                       # smallest_vector's rule, kept in fp64 for d
    if diag[0, 1] < diag[0, m]:
        m = 1
    if diag[0, 2] < diag[0, m]:
        m = 2
    v = V[0, :, m]
    n64 = v / np.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
    n32 = n64.astype(F32)
    assert np.array_equal(n32.view(np.uint32), NO.smallest_vector(diag, V)[0].view(np.uint32))
    off = F32(-((n64[0] * cent[0] + n64[1] * cent[1]) + n64[2] * cent[2]))
    return np.array([*n32, off], F32), cent, mom, n64


def remove_plane(points_frame, distance=0.01, iterations=1000, seed=0, planes=None, hyp_counts=None):
    """Points already in the frame (fp32 [N, 3]) -> dict: keep bool [N], kept int64 (ascending), planes fp32 [H, 4],
    valid bool [H], counts int64 [H], found, plane fp32 [4] (after the flip; zeros when nothing is found), winner,
    winner_count, valid_count, on, above, below, n_kept, flipped, and stats fp64 [12] as ma_remove_plane writes them.
    `planes` / `hyp_counts` may be given (e.g. counted by another implementation) to skip those steps."""
    p = np.asarray(points_frame, F32)
    n, t = len(p), F32(distance)
    if planes is None:
        planes, valid = hypotheses(p, iterations, seed)
    else:
        planes = np.asarray(planes, F32)
        valid = ~np.isinf(planes[:, 3])
    cnt = counts(planes, p, t) if hyp_counts is None else np.asarray(hyp_counts, np.int64)
    h = int(np.argmax(cnt))                                     # the first maximum: lowest h on ties
    r = {"planes": planes, "valid": valid, "counts": cnt, "winner": h, "winner_count": int(cnt[h]),
         "valid_count": int(valid.sum()), "found": bool(cnt[h] >= 3), "flipped": False}
    if not r["found"]:
        keep = np.ones(n, bool)
        plane = np.zeros(4, F32)
        on = above = below = 0
    else:
        on_w = np.abs(signed_distance(planes[h:h + 1], p)[0]) <= t
        assert int(on_w.sum()) == cnt[h]
        plane, r["centroid"], r["moments"], r["normal64"] = refit(p, on_w)
        s = signed_distance(plane[None], p)[0]
        is_on, is_above, is_below = np.abs(s) <= t, s > t, s < -t
        on, above, below = int(is_on.sum()), int(is_above.sum()), int(is_below.sum())
        keep = is_above
        r["refit"] = plane.copy()
        if below > above:
            plane, keep, above, below, r["flipped"] = -plane, is_below, below, above, True
    r.update(keep=keep, kept=np.nonzero(keep)[0], plane=plane, on=on, above=above, below=below,
             n_kept=int(keep.sum()))
    r["stats"] = np.array([float(r["found"]), *plane.astype(F64), h, cnt[h], r["valid_count"], on, above, below,
                           r["n_kept"]], F64)
    return r


def table_scene(seed, n=20000, distance=0.01, share=0.6, obj="sphere"):
    """A synthetic scan: an object standing on a table disc three object-lengths across that holds `share` of the
    points, four legs below it and 1 % stray points in the bounding box.  The table is the plane z = 0 with Gaussian
    noise of 0.2 t in z, t = distance times the scene's longest side (the disc's diameter).  obj: "sphere" (diameter 1,
    resting on the table) or "wand" (a few points per face of tests/golden/wand_mesh.npz, scaled to a longest side of 1,
    standing on it).  Returns (points float64 [n, 3], labels int8 [n]: 0 table, 1 object, 2 leg, 3 stray, t)."""
    import os
    rng = np.random.default_rng(seed)
    n_tab, n_str = int(share * n), n // 100
    n_leg = n // 10
    n_obj = n - n_tab - n_leg - n_str
    if obj == "sphere":
        x = rng.normal(size=(n_obj, 3))
        o = x / np.linalg.norm(x, axis=1, keepdims=True) * 0.5 + [0, 0, 0.5]
    else:
        z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wand_mesh.npz"))
        v = z["vertices"].astype(F64)
        tri = v[z["faces"]]
        a = rng.random((n_obj, 2))
        a = np.where(a.sum(1, keepdims=True) > 1, 1 - a, a)
        f = rng.integers(len(tri), size=n_obj)
        o = tri[f, 0] + a[:, :1] * (tri[f, 1] - tri[f, 0]) + a[:, 1:] * (tri[f, 2] - tri[f, 0])
        o = (o - o.min(0)) / (o.max(0) - o.min(0)).max()
        o[:, :2] -= o[:, :2].mean(0)
    size = 1.0
    L = 3 * size                                                  # the disc's diameter: the scene's longest side
    t = distance * L
    r = 1.5 * size * np.sqrt(rng.random(n_tab))
    ang = rng.random(n_tab) * 2 * np.pi
    tab = np.stack([r * np.cos(ang), r * np.sin(ang), rng.normal(0, 0.2 * t, n_tab)], axis=1)
    corner = np.array([[1, 1], [1, -1], [-1, 1], [-1, -1]], F64) * 0.9
    leg = np.concatenate([corner[rng.integers(4, size=n_leg)] + rng.normal(0, 0.01, (n_leg, 2)),
                          -rng.uniform(3 * t, 1.2 * size, (n_leg, 1))], axis=1)
    lo, hi = np.array([-1.5, -1.5, -1.2]), np.array([1.5, 1.5, 1.0])
    stray = lo + rng.random((n_str, 3)) * (hi - lo)
    pts = np.concatenate([tab, o, leg, stray])
    lab = np.repeat(np.arange(4, dtype=np.int8), [n_tab, n_obj, n_leg, n_str])
    return pts, lab, t
