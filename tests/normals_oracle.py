"""numpy restatement of csrc/normals.cu (test infrastructure only): oriented normals of a bare point cloud as DESIGN.md
section 1.2 defines them -- exact k nearest neighbours under the fp32 key, fp64 PCA with a fixed cyclic Jacobi, and
Hoppe-style orientation by propagation along the unique minimum spanning forest of the kNN graph.

Every fp32 / fp64 operation of the kernels is one numpy ufunc call here (each rounds to nearest, none is fused), so the
neighbour indices, the unoriented normals and the oriented normals agree with the GPU bit for bit.  The forest is
built by Kruskal over the strict edge order and the signs are propagated breadth-first from the root rule; the GPU gets
the same forest by Boruvka and the same signs by parity composition.
"""
import numpy as np

F32 = np.float32
F64 = np.float64
JACOBI_SWEEPS = 5            # cyclic sweeps over (0,1), (0,2), (1,2); DESIGN.md section 1.2 says why 5
_PAIRS = ((0, 1, 2), (0, 2, 1), (1, 2, 0))   # (p, q, the third index r)


def frame_map(points):
    """[N, 3] -> fp32 (p - c) / L, c the bounding-box centre, L its longest side (metrics.to_output_frame's rule)."""
    from tests.mesh_score_oracle import frame_map as fm
    return fm(np.asarray(points)[None].astype(F32))[0]


def _d2(q, p):
    """fp32 (dx dx + dy dy) + dz dz of q [..., 3] against p [..., 3] (broadcast)."""
    dx, dy, dz = q[..., 0] - p[..., 0], q[..., 1] - p[..., 1], q[..., 2] - p[..., 2]
    return (dx * dx + dy * dy) + dz * dz


def knn_bruteforce(p, k, rows=None, chunk=512):
    """Exact kNN by the definition: for each query i (all, or `rows`) the k other indices of smallest (d2, index)."""
    p = np.asarray(p, F32)
    n = len(p)
    rows = np.arange(n) if rows is None else np.asarray(rows)
    out = np.empty((len(rows), k), np.int64)
    for s in range(0, len(rows), chunk):
        r = rows[s:s + chunk]
        d2 = _d2(p[r][:, None, :], p[None, :, :])
        d2[np.arange(len(r)), r] = np.inf                      # not its own neighbour
        # every index whose d2 is at most the k-th smallest value (ties included), then the exact key order
        kth = np.partition(d2, k - 1, axis=1)[:, k - 1:k]
        for t in range(len(r)):
            cand = np.nonzero(d2[t] <= kth[t])[0]
            cand = cand[cand != r[t]]
            o = np.lexsort((cand, d2[t, cand]))
            out[s + t] = cand[o[:k]]
    return out


def knn(p, k, extra=16):
    """The same result as knn_bruteforce, fast: candidates from a KD-tree, ranked by the fp32 key, accepted only where no
    point outside the candidates can enter (the k-th fp32 key is clearly below the last candidate's distance); the
    other rows fall back to brute force."""
    from scipy.spatial import cKDTree
    p = np.asarray(p, F32)
    n = len(p)
    if n <= 4096:
        return knn_bruteforce(p, k)
    K = min(n, k + 1 + extra)
    dist, cand = cKDTree(p.astype(F64)).query(p.astype(F64), K)
    cand = cand.astype(np.int64)
    cand = np.where(cand == np.arange(n)[:, None], -1, cand)
    d2 = _d2(p[:, None, :], p[np.maximum(cand, 0)])
    d2 = np.where(cand < 0, np.inf, d2)
    order = np.lexsort((np.where(cand < 0, n, cand), d2), axis=-1)
    cand_s = np.take_along_axis(cand, order, axis=1)
    d2_s = np.take_along_axis(d2, order, axis=1)
    out = cand_s[:, :k].copy()
    ok = (d2_s[:, k - 1].astype(F64) < (dist[:, -1] ** 2) * (1 - 1e-5)) | (K == n)
    bad = np.nonzero(~ok)[0]
    if len(bad):
        out[bad] = knn_bruteforce(p, k, rows=bad)
    return out


def pca(p, nbr):
    """(fp64 covariance entries (xx, xy, xz, yy, yz, zz) [N, 6]) of each point with its neighbours: the point itself,
    then the neighbours in rank order, sequential fp64 sums; the centroid is the sum over k + 1."""
    p = np.asarray(p, F32).astype(F64)
    pts = [p] + [p[nbr[:, j]] for j in range(nbr.shape[1])]
    s = pts[0].copy()
    for q in pts[1:]:
        s = s + q
    m = s / F64(len(pts))
    cov = None
    for q in pts:
        d = q - m
        t = np.stack([d[:, 0] * d[:, 0], d[:, 0] * d[:, 1], d[:, 0] * d[:, 2],
                      d[:, 1] * d[:, 1], d[:, 1] * d[:, 2], d[:, 2] * d[:, 2]], axis=1)
        cov = t if cov is None else cov + t
    return cov


def jacobi(cov, sweeps=JACOBI_SWEEPS):
    """Cyclic Jacobi on symmetric 3x3 matrices given as (xx, xy, xz, yy, yz, zz) [N, 6] -> (diagonal [N, 3], V [N, 3, 3]
    with the eigenvectors in its columns), every operation fp64 and unfused, the kernel's order."""
    cov = np.asarray(cov, F64)
    n = len(cov)
    A = np.empty((n, 3, 3), F64)
    A[:, 0, 0], A[:, 0, 1], A[:, 0, 2], A[:, 1, 1], A[:, 1, 2], A[:, 2, 2] = cov.T
    A[:, 1, 0], A[:, 2, 0], A[:, 2, 1] = A[:, 0, 1], A[:, 0, 2], A[:, 1, 2]
    V = np.broadcast_to(np.eye(3), (n, 3, 3)).copy()
    with np.errstate(all="ignore"):
        for _ in range(sweeps):
            for p, q, r in _PAIRS:
                apq, app, aqq = A[:, p, q].copy(), A[:, p, p].copy(), A[:, q, q].copy()
                go = apq != 0
                theta = (aqq - app) / (F64(2) * apq)
                t = F64(1) / (np.abs(theta) + np.sqrt(theta * theta + F64(1)))
                t = np.where(theta < 0, -t, t)
                c = F64(1) / np.sqrt(t * t + F64(1))
                s = t * c
                tapq = t * apq
                arp, arq = A[:, r, p].copy(), A[:, r, q].copy()
                nrp, nrq = c * arp - s * arq, s * arp + c * arq
                upd = {(p, p): app - tapq, (q, q): aqq + tapq, (p, q): np.zeros(n), (r, p): nrp, (r, q): nrq}
                for (a, b), v in upd.items():
                    A[:, a, b] = np.where(go, v, A[:, a, b])
                    A[:, b, a] = A[:, a, b]
                vp, vq = V[:, :, p].copy(), V[:, :, q].copy()
                g = go[:, None]
                V[:, :, p] = np.where(g, c[:, None] * vp - s[:, None] * vq, vp)
                V[:, :, q] = np.where(g, s[:, None] * vp + c[:, None] * vq, vq)
    return np.stack([A[:, 0, 0], A[:, 1, 1], A[:, 2, 2]], axis=1), V


def smallest_vector(diag, V):
    """Column of the smallest diagonal entry (lowest column on ties), normalised in fp64, rounded to fp32."""
    m = np.zeros(len(diag), np.int64)
    m = np.where(diag[:, 1] < diag[np.arange(len(m)), m], 1, m)
    m = np.where(diag[:, 2] < diag[np.arange(len(m)), m], 2, m)
    v = V[np.arange(len(m)), :, m]
    ln = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    return (v / ln[:, None]).astype(F32)


def dot32(a, b):
    """fp32 (ax bx + ay by) + az bz."""
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def edges(nbr, u):
    """The undirected kNN graph: unique (a < b) pairs [E, 2] and their fp32 weights max(0, 1 - |u_a . u_b|)."""
    n, k = nbr.shape
    i = np.repeat(np.arange(n), k)
    j = nbr.reshape(-1)
    ab = np.unique(np.stack([np.minimum(i, j), np.maximum(i, j)], axis=1), axis=0)
    w = np.maximum(F32(0), F32(1) - np.abs(dot32(u[ab[:, 0]], u[ab[:, 1]])))
    return ab, w


def kruskal(n, ab, w):
    """The minimum spanning forest under the strict order (w, a, b): bool [E], True for the forest's edges."""
    order = np.lexsort((ab[:, 1], ab[:, 0], w))
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    keep = np.zeros(len(ab), bool)
    a_l, b_l = ab[:, 0].tolist(), ab[:, 1].tolist()
    for e in order.tolist():
        ra, rb = find(a_l[e]), find(b_l[e])
        if ra != rb:
            parent[ra] = rb
            keep[e] = True
    return keep


def orient(p, u, nbr, return_forest=False):
    """Oriented normals fp32 [N, 3]: per connected component the root is the point of largest fp32 |p|^2 (lowest index on
    ties), its sign is + iff u . p >= 0; along every forest edge from parent a to child b, s_b = s_a if u_a . u_b >= 0
    else -s_a."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import breadth_first_order, connected_components
    p, u = np.asarray(p, F32), np.asarray(u, F32)
    n = len(p)
    ab, w = edges(nbr, u)
    keep = kruskal(n, ab, w)
    t = ab[keep]
    tree = coo_matrix((np.ones(len(t)), (t[:, 0], t[:, 1])), shape=(n, n)).tocsr()
    ncomp, label = connected_components(tree, directed=False)
    r2 = dot32(p, p)
    order = np.lexsort((np.arange(n), -r2.astype(F64), label))       # per component: largest |p|^2, lowest index
    first = np.ones(n, bool)
    first[1:] = label[order[1:]] != label[order[:-1]]
    roots = order[first]
    sign = np.zeros(n, np.int8)
    for root in roots.tolist():
        sign[root] = 1 if dot32(u[root], p[root]) >= 0 else -1
        bfs, pred = breadth_first_order(tree, root, directed=False, return_predecessors=True)
        for b in bfs[1:].tolist():
            a = pred[b]
            sign[b] = sign[a] if dot32(u[a], u[b]) >= 0 else -sign[a]
    out = np.where((sign < 0)[:, None], -u, u)
    return (out, ab, w, keep, ncomp) if return_forest else out


def estimate_normals(points_frame, k):
    """Points already in the frame (fp32 [N, 3]) -> (oriented fp32 [N, 3], kNN int64 [N, k], unoriented fp32 [N, 3])."""
    p = np.asarray(points_frame, F32)
    nbr = knn(p, k)
    u = smallest_vector(*jacobi(pca(p, nbr)))
    return orient(p, u, nbr), nbr, u
