"""numpy restatement of csrc/watertight.cu (test infrastructure only): the fp32 narrow-band distance field op for op,
marching cubes from the same generated table, and the mesh checks the watertight tests share.

Every fp32 operation of the kernel's distance formula is one numpy float32 ufunc call here (each rounds to nearest, none
is fused), so the field agrees bit for bit.  The oracle culls by bounding box only; the kernel's extra plane-slab test
is conservative, so both give min(band, distance) at every grid point.
"""
import numpy as np

from meshanything_b200 import mc_table

F32 = np.float32


def _sub(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _seg2(w, e):
    l = _dot(e, e)
    pos = l > 0
    t = np.where(pos, _dot(w, e) / np.where(pos, l, F32(1)), F32(0))
    t = np.minimum(np.maximum(t, F32(0)), F32(1))
    q = (w[0] - t * e[0], w[1] - t * e[1], w[2] - t * e[2])
    return _dot(q, q)


def tri_dist(p, a, b, c):
    """fp32 distance from points p to triangles (a, b, c); each argument is a tuple of three float32 arrays."""
    with np.errstate(all="ignore"):
        ab, bc, ca = _sub(b, a), _sub(c, b), _sub(a, c)
        ap, bp, cp = _sub(p, a), _sub(p, b), _sub(p, c)
        nrm = _cross(ab, _sub(c, a))
        nn = _dot(nrm, nrm)
        inside = ((nn > 0) & (_dot(_cross(ab, ap), nrm) >= 0) & (_dot(_cross(bc, bp), nrm) >= 0)
                  & (_dot(_cross(ca, cp), nrm) >= 0))
        h = _dot(ap, nrm)
        d_plane = np.sqrt((h * h) / np.where(inside, nn, F32(1)))
        d_edge = np.sqrt(np.minimum(np.minimum(_seg2(ap, ab), _seg2(bp, bc)), _seg2(cp, ca)))
        return np.where(inside, d_plane, d_edge)


def grid_coords(n):
    dx = F32(2) / F32(n)
    return F32(-1) + np.arange(n, dtype=F32) * dx


def udf_grid(vertices, faces, n, band=None, chunk=4_000_000):
    """fp32 [n, n, n]: min(band, distance from grid point (i, j, k) to the nearest face), band default 3 dx."""
    v = np.asarray(vertices, dtype=F32)
    f = np.asarray(faces, dtype=np.int64)
    dx = F32(2) / F32(n)
    band = F32(3 * 2.0 / n) if band is None else F32(band)
    g = grid_coords(n)
    field = np.full(n * n * n, band, dtype=F32)
    if len(f) == 0:
        return field.reshape(n, n, n)
    tri = v[f].astype(np.float64)                                   # [F, 3 vertices, 3 axes]
    reach = float(band) * 1.01 + 1e-4 * np.maximum(1.0, np.abs(tri).max(axis=(1, 2)))
    lo = np.clip(np.floor((tri.min(1) - reach[:, None] + 1.0) / float(dx)) - 1, 0, n - 1).astype(np.int64)
    hi = np.clip(np.ceil((tri.max(1) + reach[:, None] + 1.0) / float(dx)) + 1, 0, n - 1).astype(np.int64)
    ext = hi - lo + 1                                               # [F, 3]
    cnt = ext.prod(1)
    starts = np.concatenate([[0], np.cumsum(cnt)])
    fi_all = np.arange(len(f))
    pos = 0
    while pos < len(f):                                             # faces in chunks of about `chunk` pairs
        end = int(np.searchsorted(starts, starts[pos] + chunk, side="right")) - 1
        end = max(end, pos + 1)
        sel = fi_all[pos:end]
        rep = np.repeat(sel, cnt[sel])
        local = np.arange(len(rep)) - np.repeat(starts[sel] - starts[pos], cnt[sel])
        nk, nj = ext[rep, 2], ext[rep, 1]
        k = lo[rep, 2] + local % nk
        j = lo[rep, 1] + (local // nk) % nj
        i = lo[rep, 0] + local // (nk * nj)
        p = (g[i], g[j], g[k])
        t = v[f[rep]]
        d = tri_dist(p, (t[:, 0, 0], t[:, 0, 1], t[:, 0, 2]), (t[:, 1, 0], t[:, 1, 1], t[:, 1, 2]),
                     (t[:, 2, 0], t[:, 2, 1], t[:, 2, 2]))
        np.minimum.at(field, (i * n + j) * n + k, d)
        pos = end
    return field.reshape(n, n, n)


_TAB = mc_table.tables()
_TRI_COUNT = np.array([len(t) for t in _TAB], dtype=np.int64)
_TRI_EDGES = np.full((256, 15), -1, dtype=np.int64)
for _c, _t in enumerate(_TAB):
    _flat = [e for tri in _t for e in tri]
    _TRI_EDGES[_c, :len(_flat)] = _flat
_EDGE_C0 = np.array([e[0] for e in mc_table.EDGES], dtype=np.int64)
_EDGE_AXIS = np.array([e[2] for e in mc_table.EDGES], dtype=np.int64)


def marching_cubes(field, level):
    """(vertices fp32 [V, 3] in index space, faces int32 [T, 3]) in the kernel's order."""
    fld = np.asarray(field, dtype=F32)
    n = fld.shape[0]
    level = F32(level)
    inside = fld < level
    crossed = np.zeros((n, n, n, 3), dtype=bool)
    crossed[:-1, :, :, 0] = inside[:-1] != inside[1:]
    crossed[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    crossed[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = crossed.reshape(-1, 3)
    vid = (np.cumsum(flat.reshape(-1)) - 1).reshape(-1, 3)          # vertex id of each crossed (point, axis)
    p_idx, axis = np.nonzero(flat)
    i, j, k = np.unravel_index(p_idx, (n, n, n))
    step = np.array([n * n, n, 1])[axis]
    fa, fb = fld.reshape(-1)[p_idx], fld.reshape(-1)[p_idx + step]
    t = (level - fa) / (fb - fa)
    verts = np.stack([i, j, k], axis=1).astype(F32)
    verts[np.arange(len(axis)), axis] = verts[np.arange(len(axis)), axis] + t
    # cells
    case = np.zeros((n - 1, n - 1, n - 1), dtype=np.int64)
    for c in range(8):
        ox, oy, oz = mc_table.corner_offset(c)
        case |= inside[ox:n - 1 + ox, oy:n - 1 + oy, oz:n - 1 + oz].astype(np.int64) << c
    full_case = np.zeros((n, n, n), dtype=np.int64)
    full_case[:-1, :-1, :-1] = case
    full_case = full_case.reshape(-1)
    ntri = _TRI_COUNT[full_case]                                    # case 0 (no triangles) outside the cells
    cells = np.nonzero(ntri)[0]
    rep = np.repeat(cells, ntri[cells])
    tri_in_cell = np.arange(len(rep)) - np.repeat(np.cumsum(ntri[cells]) - ntri[cells], ntri[cells])
    faces = np.empty((len(rep), 3), dtype=np.int64)
    for s in range(3):
        e = _TRI_EDGES[full_case[rep], 3 * tri_in_cell + s]
        c0 = _EDGE_C0[e]
        q = rep + (c0 & 1) * n * n + ((c0 >> 1) & 1) * n + ((c0 >> 2) & 1)
        faces[:, s] = vid[q, _EDGE_AXIS[e]]
    return verts, faces.astype(np.int32)


# ---------------------------------------------------------------- mesh checks shared by the CPU and GPU tests

def directed_edges(faces):
    f = np.asarray(faces, dtype=np.int64)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def is_watertight(faces):
    """Every undirected edge is used by exactly two faces, once in each direction (closed, consistently oriented)."""
    e = directed_edges(faces)
    if len(e) == 0:
        return False
    d = np.unique(e, axis=0, return_counts=True)
    if (d[1] != 1).any():                                             # a directed edge used twice: orientation flip
        return False
    rev = set(map(tuple, e[:, ::-1].tolist()))
    return all(tuple(x) in rev for x in e.tolist())


def components(faces, n_vertices):
    """Connected components of the faces (by shared vertices): list of face-index arrays."""
    f = np.asarray(faces, dtype=np.int64)
    parent = np.arange(n_vertices)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for a, b in np.concatenate([f[:, [0, 1]], f[:, [1, 2]]]).tolist():
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
    roots = np.array([find(x) for x in f[:, 0].tolist()])
    return [np.nonzero(roots == r)[0] for r in np.unique(roots)]


def euler_characteristic(faces):
    f = np.asarray(faces, dtype=np.int64)
    V = len(np.unique(f))
    E = len(np.unique(np.sort(directed_edges(f), axis=1), axis=0))
    return V - E + len(f)


def mesh_distance(points, verts, faces, reach):
    """float64 distance from each point to the triangle mesh, exact where it is <= reach (inf where no face comes
    that close).  Candidate faces: the big ones always, the others from a KD-tree over their centroids."""
    from scipy.spatial import cKDTree
    pts = np.asarray(points, dtype=np.float64)
    tri = np.asarray(verts, dtype=np.float64)[np.asarray(faces, dtype=np.int64)]
    cen = tri.mean(1)
    rad = np.linalg.norm(tri - cen[:, None], axis=2).max(1)
    small = rad <= np.quantile(rad, 0.99)
    big_ids = np.nonzero(~small)[0]
    small_ids = np.nonzero(small)[0]
    hits = cKDTree(cen[small_ids]).query_ball_point(pts, reach + rad[small_ids].max() if len(small_ids) else 0.0)
    pi = np.concatenate([np.repeat(np.arange(len(pts)), [len(h) for h in hits])] +
                        [np.repeat(np.arange(len(pts)), len(big_ids))])
    fi = np.concatenate([small_ids[np.concatenate([np.asarray(h, dtype=np.int64) for h in hits])]] +
                        [np.tile(big_ids, len(pts))])
    out = np.full(len(pts), np.inf)
    for s in range(0, len(pi), 2_000_000):
        p, t = pts[pi[s:s + 2_000_000]], tri[fi[s:s + 2_000_000]]
        d = tri_dist((p[:, 0], p[:, 1], p[:, 2]), *[(t[:, v, 0], t[:, v, 1], t[:, v, 2]) for v in range(3)])
        np.minimum.at(out, pi[s:s + 2_000_000], d)
    return out


def face_normals(verts, faces):
    t = np.asarray(verts, dtype=np.float64)[np.asarray(faces, dtype=np.int64)]
    return np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
