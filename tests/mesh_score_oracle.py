"""numpy restatement of csrc/mesh_score.cu and meshanything_b200/metrics.py (test infrastructure only): the frame map,
the per-point and per-quadrature-point nearest neighbours, the Chamfer / normal-consistency terms and the selection
rule of best-of-N sampling (DESIGN.md section 1, row f6).

Every fp32 operation of the kernels is one numpy float32 ufunc call here (each rounds to nearest, none is fused) and the
point-triangle distance is tests/watertight_oracle.py's tri_dist, so the per-point distances and argmins agree bit for
bit.  The fp64 sums run in numpy's order, not the kernels' tile order: the terms agree to about 1e-15 relative.
"""
import numpy as np

from tests.watertight_oracle import _cross, _dot, _sub, tri_dist

F32 = np.float32
S_SUB = 4                                    # each face is split into S_SUB^2 sub-triangles
# barycentric numerators over 3 S_SUB of the 16 sub-triangle centroids, in the kernel's order: the upward ones (i, j),
# i + j <= 3, at (3i+1, 3j+1), then the downward ones, i + j <= 2, at (3i+2, 3j+2); i outer, j inner
QUAD_NUM = np.array([(3 * i + 1, 3 * j + 1) for i in range(S_SUB) for j in range(S_SUB - i)]
                    + [(3 * i + 2, 3 * j + 2) for i in range(S_SUB - 1) for j in range(S_SUB - 1 - i)], dtype=np.int64)
QUAD_U = QUAD_NUM[:, 0].astype(F32) / F32(3 * S_SUB)
QUAD_V = QUAD_NUM[:, 1].astype(F32) / F32(3 * S_SUB)


def frame_map(pc_normal):
    """[..., P, 6] -> fp32: xyz to (p - c) / L (c the bounding-box centre, L its longest side; L = 0 -> 1), normals as
    given."""
    pc = np.asarray(pc_normal).astype(F32)
    xyz = pc[..., :3]
    lo, hi = xyz.min(axis=-2, keepdims=True), xyz.max(axis=-2, keepdims=True)
    centre = (lo + hi) / F32(2)
    side = (hi - lo).max(axis=-1, keepdims=True)
    side = np.where(side > 0, side, F32(1))
    return np.concatenate([(xyz - centre) / side, pc[..., 3:]], axis=-1)


def _cols(x):
    return (x[..., 0], x[..., 1], x[..., 2])


def unit_normal(a, b, c):
    """cross(b - a, c - a) / sqrt(its squared length) in fp32; zero where that length is zero."""
    with np.errstate(all="ignore"):
        n = _cross(_sub(b, a), _sub(c, a))
        nn = _dot(n, n)
        pos = nn > 0
        ln = np.sqrt(np.where(pos, nn, F32(1)))
        return tuple(np.where(pos, n[k] / ln, F32(0)) for k in range(3))


def face_area(tri):
    """float64 [F]: area from the fp32 vertex differences taken in float64 (no fused operations)."""
    t = np.asarray(tri, dtype=F32).astype(np.float64)
    ux, uy, uz = _cols(t[:, 1] - t[:, 0])
    wx, wy, wz = _cols(t[:, 2] - t[:, 0])
    nx, ny, nz = uy * wz - uz * wy, uz * wx - ux * wz, ux * wy - uy * wx
    return 0.5 * np.sqrt((nx * nx + ny * ny) + nz * nz)


def quadrature(tri):
    """(points fp32 [F, 16, 3], weights float64 [F, 16] = area / 16) of faces [F, 3, 3]."""
    t = np.asarray(tri, dtype=F32)
    a = t[:, None, 0]
    ab, ac = t[:, None, 1] - a, t[:, None, 2] - a
    pts = (a + QUAD_U[None, :, None] * ab) + QUAD_V[None, :, None] * ac
    w = np.repeat((face_area(t) * (1.0 / (S_SUB * S_SUB)))[:, None], S_SUB * S_SUB, axis=1)
    return pts, w


def candidate(tri, cloud, chunk=1_000_000):
    """One candidate mesh [F, 3, 3] (NaN first coordinate = absent face) against a cloud [P, 6] already in the output
    frame -> the kernel's per-point / per-quadrature-point outputs and its four fp64 terms."""
    tri = np.asarray(tri, dtype=F32)
    cloud = np.asarray(cloud, dtype=F32)
    F, P = len(tri), len(cloud)
    valid = ~np.isnan(tri[:, 0, 0])
    vi = np.nonzero(valid)[0]
    vt = tri[vi]
    p, npt = cloud[:, :3], cloud[:, 3:]
    out = {"faces": int(len(vi)),
           "point_dist": np.full(P, np.inf, F32), "point_face": np.full(P, -1, np.int32),
           "quad_dist": np.full((F, 16), np.inf, F32), "quad_point": np.full((F, 16), -1, np.int32)}
    if len(vi) == 0:
        out.update(p2m=np.inf, m2p=np.inf, nc_p=0.0, nc_m=0.0)
        return out
    fa, fb, fc = (_cols(vt[None, :, k]) for k in range(3))
    fn = unit_normal(_cols(vt[:, 0]), _cols(vt[:, 1]), _cols(vt[:, 2]))
    step = max(1, chunk // len(vi))
    nc_p = np.empty(P, F32)
    for s in range(0, P, step):                               # p2m: every point against every valid face
        q = p[s:s + step]
        d = tri_dist(_cols(q[:, None, :]), fa, fb, fc)
        j = np.argmin(d, axis=1)                              # first minimum: the lowest face index on ties
        out["point_dist"][s:s + step] = d[np.arange(len(q)), j]
        out["point_face"][s:s + step] = vi[j]
        nc_p[s:s + step] = np.abs(_dot(_cols(npt[s:s + step]), tuple(c[j] for c in fn)))
    qp, qw = quadrature(vt)
    qp, qw = qp.reshape(-1, 3), qw.reshape(-1)
    qn = tuple(np.repeat(c, 16) for c in fn)
    qd = np.empty(len(qp), F32)
    qj = np.empty(len(qp), np.int64)
    step = max(1, chunk // P)
    for s in range(0, len(qp), step):                         # m2p: every quadrature point against every cloud point
        x = qp[s:s + step, None, :]
        dx, dy, dz = x[..., 0] - p[None, :, 0], x[..., 1] - p[None, :, 1], x[..., 2] - p[None, :, 2]
        d2 = (dx * dx + dy * dy) + dz * dz
        j = np.argmin(d2, axis=1)
        qd[s:s + step] = np.sqrt(d2[np.arange(len(j)), j])
        qj[s:s + step] = j
    nc_m = np.abs(_dot(_cols(npt[qj]), qn))
    out["quad_dist"][vi] = qd.reshape(-1, 16)
    out["quad_point"][vi] = qj.reshape(-1, 16)
    wsum = qw.sum()
    out["p2m"] = float(out["point_dist"].astype(np.float64).mean())
    out["nc_p"] = float(nc_p.astype(np.float64).mean())
    out["m2p"] = float((qw * qd.astype(np.float64)).sum() / wsum) if wsum > 0 else np.inf
    out["nc_m"] = float((qw * nc_m.astype(np.float64)).sum() / wsum) if wsum > 0 else 0.0
    return out


def score(meshes, pc_normal):
    """meshes [S, N, F, 3, 3], clouds [S, P, 6] as given to the model -> (chamfer, normal consistency float64 [S, N],
    per-candidate outputs of `candidate` [S][N])."""
    meshes = np.asarray(meshes, dtype=F32)
    clouds = frame_map(pc_normal)
    S, N = meshes.shape[:2]
    res = [[candidate(meshes[s, n], clouds[s]) for n in range(N)] for s in range(S)]
    p2m = np.array([[r["p2m"] for r in row] for row in res])
    m2p = np.array([[r["m2p"] for r in row] for row in res])
    chamfer = p2m + m2p
    nc = np.array([[0.5 * (r["nc_p"] + r["nc_m"]) for r in row] for row in res])
    nc = np.where(np.isinf(chamfer), 0.0, nc)
    return chamfer, nc, res


def select(chamfer):
    """The argmin of chamfer along the last axis, lowest index on ties (candidate 0 when all are +inf)."""
    return np.argmin(np.asarray(chamfer), axis=-1)
