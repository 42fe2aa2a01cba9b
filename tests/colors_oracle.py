"""numpy restatement of csrc/colors.cu and meshanything_b200/colors.py (test infrastructure only): the frame map, the
nearest face of every point, the barycentric weights of tri_dist.cuh's wt_tri_bary, the fixed-point sums, the fallback
and the vertex colours (DESIGN.md section 1.9).

Every fp32 operation of the kernels is one numpy float32 ufunc call here (each rounds to nearest, none is fused), the
point-triangle distance is tests/watertight_oracle.py's tri_dist, and the sums are integer sums, so every output agrees
bit for bit.
"""
import numpy as np

from tests.watertight_oracle import _cross, _dot, _sub, tri_dist

F32, F64 = np.float32, np.float64
SCALE = F32(2 ** 24)


def frame(points, vertices=None):
    """(points, vertices) -> fp32 (x - c) / L, c and L the float64 bounding-box centre and longest side of the points
    (L = 0 counts as 1), computed in float64 and rounded once."""
    p = np.asarray(points, dtype=F64)
    lo, hi = p.min(axis=0), p.max(axis=0)
    c = (lo + hi) / 2
    side = float((hi - lo).max())
    side = side if side > 0 else 1.0
    out = ((p - c) / side).astype(F32)
    if vertices is None:
        return out
    return out, ((np.asarray(vertices, dtype=F64) - c) / side).astype(F32)


def _cols(x):
    return (x[..., 0], x[..., 1], x[..., 2])


def _seg_t(w, e):
    l = _dot(e, e)
    pos = l > 0
    t = np.where(pos, _dot(w, e) / np.where(pos, l, F32(1)), F32(0))
    return np.minimum(np.maximum(t, F32(0)), F32(1))


def _seg2_at(w, e, t):
    q = (w[0] - t * e[0], w[1] - t * e[1], w[2] - t * e[2])
    return _dot(q, q)


def bary(p, a, b, c):
    """fp32 weights [..., 3] of a, b, c at the point of triangle (a, b, c) nearest to p (wt_tri_bary); each argument a
    tuple of three float32 arrays."""
    with np.errstate(all="ignore"):
        ab, bc, ca = _sub(b, a), _sub(c, b), _sub(a, c)
        ap, bp, cp = _sub(p, a), _sub(p, b), _sub(p, c)
        nrm = _cross(ab, _sub(c, a))
        nn = _dot(nrm, nrm)
        eab, ebc, eca = _dot(_cross(ab, ap), nrm), _dot(_cross(bc, bp), nrm), _dot(_cross(ca, cp), nrm)
        s = (eab + ebc) + eca
        inside = (nn > 0) & (eab >= 0) & (ebc >= 0) & (eca >= 0) & (s > 0)
        sd = np.where(inside, s, F32(1))
        tab, tbc, tca = _seg_t(ap, ab), _seg_t(bp, bc), _seg_t(cp, ca)
        dab, dbc, dca = _seg2_at(ap, ab, tab), _seg2_at(bp, bc, tbc), _seg2_at(cp, ca, tca)
        on_ab = (dab <= dbc) & (dab <= dca)
        on_bc = ~on_ab & (dbc <= dca)
        z = np.zeros_like(tab)
        one = F32(1)
        w0 = np.where(on_ab, one - tab, np.where(on_bc, z, tca))
        w1 = np.where(on_ab, tab, np.where(on_bc, one - tbc, z))
        w2 = np.where(on_ab, z, np.where(on_bc, tbc, one - tca))
        w = np.stack([np.where(inside, ebc / sd, w0), np.where(inside, eca / sd, w1), np.where(inside, eab / sd, w2)],
                     axis=-1)
        return w.astype(F32)


def nearest_faces(p, verts, faces, chunk=2_000_000):
    """(face int32 [N], distance fp32 [N]) of fp32 points p [N, 3]: the first minimum of tri_dist over the faces."""
    tri = np.asarray(verts, dtype=F32)[np.asarray(faces, dtype=np.int64)]
    fa, fb, fc = (_cols(tri[None, :, k]) for k in range(3))
    N = len(p)
    face = np.empty(N, np.int32)
    dist = np.empty(N, F32)
    step = max(1, chunk // len(tri))
    for s in range(0, N, step):
        q = p[s:s + step]
        d = tri_dist(_cols(q[:, None, :]), fa, fb, fc)
        j = np.argmin(d, axis=1)
        face[s:s + step] = j
        dist[s:s + step] = d[np.arange(len(q)), j]
    return face, dist


def nearest_points(x, p, chunk=4_000_000):
    """index int64 [M] of the nearest of fp32 points p [N, 3] to every fp32 x [M, 3] by d^2 = (dx dx + dy dy) + dz dz,
    the lowest index on ties."""
    out = np.empty(len(x), np.int64)
    step = max(1, chunk // len(p))
    for s in range(0, len(x), step):
        y = x[s:s + step, None, :]
        dx, dy, dz = y[..., 0] - p[None, :, 0], y[..., 1] - p[None, :, 1], y[..., 2] - p[None, :, 2]
        out[s:s + step] = np.argmin((dx * dx + dy * dy) + dz * dz, axis=1)
    return out


def fix(x):
    """llrint(fl32(x 2^24)) as uint64 (x >= 0 fp32)."""
    return np.rint(np.asarray(x, F32) * SCALE).astype(np.uint64)


def transfer(verts, faces, points, colors, r):
    """The kernel on fp32 inputs already in the frame: a dict of face, dist, weights [N, 3], sums uint64 [V, 4],
    fallback bool [V], colors fp32 [V, 3], stats int64 [3] (used, beyond r, fallback vertices)."""
    v = np.asarray(verts, F32)
    f = np.asarray(faces, np.int64)
    p = np.asarray(points, F32)
    col = np.asarray(colors, F32)
    r = F32(r)
    face, dist = nearest_faces(p, v, f)
    corner = f[face]                                                   # [N, 3]
    w = bary(_cols(p), *(_cols(v[corner[:, k]]) for k in range(3)))
    used = dist <= r
    sums = np.zeros((len(v), 4), np.uint64)
    cu, wu, colu = corner[used], w[used], col[used]
    for k in range(3):
        np.add.at(sums[:, 0], cu[:, k], fix(wu[:, k]))
        for ch in range(3):
            np.add.at(sums[:, 1 + ch], cu[:, k], fix(wu[:, k] * colu[:, ch]))
    fallback = sums[:, 0] == 0
    out = np.empty((len(v), 3), F32)
    ok = ~fallback
    out[ok] = (sums[ok, 1:].astype(F64) / sums[ok, :1].astype(F64)).astype(F32)
    if fallback.any():
        out[fallback] = col[nearest_points(v[fallback], p)]
    stats = np.array([int(used.sum()), int((~used).sum()), int(fallback.sum())], np.int64)
    return {"face": face, "dist": dist, "weights": w, "sums": sums, "fallback": fallback, "colors": out,
            "stats": stats}


def transfer_colors(vertices, faces, points, colors, max_distance=0.05):
    """colors.transfer_colors restated: (vertex colours fp32 [V, 3], the dict of `transfer`)."""
    p, v = frame(points, vertices)
    res = transfer(v, faces, p, np.asarray(colors, F32), max_distance)
    return res["colors"], res
