"""numpy restatement of csrc/smooth.cu (test infrastructure only): moving-least-squares smoothing of a point cloud as
DESIGN.md section 1.8 defines it -- the exact kNN of section 1.2, weights (1 - d^2 / H)^2, the weighted local frame by
the fixed cyclic Jacobi, the weighted quadratic height field solved by Cholesky in fp64, and the plane fallback.

Every fp64 operation of the kernel is one numpy ufunc call here (each rounds to nearest, none is fused), and every
sum runs in the kernel's order, so the neighbours, the normals, the outcomes and the points agree with the GPU bit for
bit.  `python -m tests.smooth_oracle` prints the table of DESIGN.md section 1.8 the default k was chosen from.
"""
import numpy as np

from tests import normals_oracle as NO
from tests.outliers_oracle import frame_map  # noqa: F401  (float64 input shifted by its centre, as the product does)

F32, F64 = np.float32, np.float64
PIVOT = 1e-9                         # kSmPivot of csrc/smooth.cu: pivots at or below PIVOT M_00 are singular
QUADRATIC, SINGULAR, FAR = 0, 1, 2   # the outcome of a point (flag_out)
DEFAULT_K = 24                       # smooth.DEFAULT_K


def _dot(a, b):
    """fp64 (ax bx + ay by) + az bz over the last axis."""
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _unit(v):
    ln = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    return v / ln[:, None]


def _tri(a, b):
    return a * (a + 1) // 2 + b


def smooth(points_frame, k, nbr=None, plane_only=False, far_share=1.0):
    """Points already in the frame (fp32 [N, 3]) -> dict with "points" fp32 [N, 3], "normals" fp32 [N, 3], "flags"
    uint8 [N], "knn" int64 [N, k] and "stats" int64 [3] (quadratic, singular, far), and the fp64 terms "quadratic"
    (the projection onto the quadratic, where there is one), "plane" (onto the weighted plane) and "H".  Oracle options,
    not product options: plane_only projects every point onto its weighted plane (the comparison of section 1.8);
    far_share < 1 lowers the far limit to |q - p|^2 > far_share H, to exercise that branch."""
    p32 = np.asarray(points_frame, F32)
    n = len(p32)
    nbr = NO.knn(p32, k) if nbr is None else np.asarray(nbr, np.int64)
    p = p32.astype(F64)
    pts = [p] + [p[nbr[:, j]] for j in range(k)]
    last = pts[k] - p
    H = F64(2) * _dot(last, last)
    with np.errstate(all="ignore"):
        w = [np.ones(n)]
        for q in pts[1:]:
            d = q - p
            t = F64(1) - _dot(d, d) / H
            w.append(np.where(H == 0, F64(1), t * t))
        sw, s = np.zeros(n), np.zeros((n, 3))
        for wj, q in zip(w, pts):
            sw = sw + wj
            s = s + wj[:, None] * q
        m = s / sw[:, None]
        cov = np.zeros((n, 6))
        for wj, q in zip(w, pts):
            d = q - m
            cov = cov + np.stack([wj * (d[:, 0] * d[:, 0]), wj * (d[:, 0] * d[:, 1]), wj * (d[:, 0] * d[:, 2]),
                                  wj * (d[:, 1] * d[:, 1]), wj * (d[:, 1] * d[:, 2]), wj * (d[:, 2] * d[:, 2])], axis=1)
        diag, V = NO.jacobi(cov)
        ar = np.arange(n)
        cn = np.zeros(n, np.int64)
        cn = np.where(diag[:, 1] < diag[ar, cn], 1, cn)
        cn = np.where(diag[:, 2] < diag[ar, cn], 2, cn)
        c1, c2 = np.where(cn == 0, 1, 0), np.where(cn == 2, 1, 2)
        nv, t1, t2 = _unit(V[ar, :, cn]), _unit(V[ar, :, c1]), _unit(V[ar, :, c2])
        # normal equations, lower triangle row-major
        h = np.sqrt(H)
        M, b = [np.zeros(n) for _ in range(21)], [np.zeros(n) for _ in range(6)]
        for j, (wj, q) in enumerate(zip(w, pts)):
            r = q - m
            u, v, z = _dot(r, t1) / h, _dot(r, t2) / h, _dot(r, nv)
            if j == 0:
                up, vp = u, v
            phi = [np.ones(n), u, v, u * u, u * v, v * v]
            for a in range(6):
                wa = wj * phi[a]
                for c in range(a + 1):
                    M[_tri(a, c)] = M[_tri(a, c)] + wa * phi[c]
                b[a] = b[a] + wa * z
        ok = H != 0
        pivot_min = F64(PIVOT) * M[0]                          # the weight mass: u, v are O(1) in units of h
        for a in range(6):                                   # Cholesky in place, row by row
            for c in range(a + 1):
                s_ = M[_tri(a, c)]
                for t in range(c):
                    s_ = s_ - M[_tri(a, t)] * M[_tri(c, t)]
                if c == a:
                    ok = ok & (s_ > pivot_min)
                    M[_tri(a, a)] = np.sqrt(s_)
                else:
                    M[_tri(a, c)] = s_ / M[_tri(c, c)]
        for a in range(6):                                   # L y = b
            s_ = b[a]
            for t in range(a):
                s_ = s_ - M[_tri(a, t)] * b[t]
            b[a] = s_ / M[_tri(a, a)]
        for a in range(5, -1, -1):                           # L^T x = y
            s_ = b[a]
            for t in range(a + 1, 6):
                s_ = s_ - M[_tri(t, a)] * b[t]
            b[a] = s_ / M[_tri(a, a)]
        phi = [np.ones(n), up, vp, up * up, up * vp, vp * vp]
        zp = b[0] * phi[0]
        for a in range(1, 6):
            zp = zp + b[a] * phi[a]
        uh, vh = up * h, vp * h
        q = ((m + uh[:, None] * t1) + vh[:, None] * t2) + zp[:, None] * nv
        e = q - p
        far = ok & (_dot(e, e) > (H if far_share == 1.0 else F64(far_share) * H))
        quad = ok & ~far
        sp = _dot(p - m, nv)
        plane = p - sp[:, None] * nv
    if plane_only:
        quad = np.zeros(n, bool)
    flags = np.where(quad, QUADRATIC, np.where(ok, FAR, SINGULAR)).astype(np.uint8)
    out = np.where(quad[:, None], q, plane).astype(F32)
    stats = np.array([int(quad.sum()), int((~ok).sum()), int(far.sum())], np.int64)
    return {"points": out, "normals": nv.astype(F32), "flags": flags, "knn": nbr, "stats": stats, "quadratic": q,
            "plane": plane, "H": H}


def to_input_units(points, frame_before, frame_after):
    """x + L (q' - p') in float64 from the fp32 frame values, L the bounding box's longest side; fp32 input rounded once
    at the end, float64 input kept float64 (smooth.smooth_points)."""
    x = np.asarray(points)
    if not np.issubdtype(x.dtype, np.floating):
        x = x.astype(F64)
    side = float((x.astype(F64).max(axis=0) - x.astype(F64).min(axis=0)).max()) if len(x) else 0.0
    side = side if side > 0 else 1.0
    moved = x.astype(F64) + side * (frame_after.astype(F64) - frame_before.astype(F64))
    return moved.astype(x.dtype)


# ---------------------------------------------------------------- the evidence of DESIGN.md section 1.8

def surface_points(vertices, faces, n, seed):
    """n points on a mesh's surface in float64: the faces and barycentric draws of tests/surface_oracle.py (the sampler
    of ma_sample_surface), the points themselves without its fp16 rounding."""
    from tests import surface_oracle as SO
    v = np.ascontiguousarray(vertices, F32)
    f = np.asarray(faces, np.int64)
    u = SO.uniforms(seed, n)
    face = SO.pick_faces(SO.scan(SO.face_areas(v, f)), u[:, 0])
    t = v[f[face]].astype(F64)
    r1, r2 = u[:, 1].astype(F64), u[:, 2].astype(F64)
    flip = (r1 + r2) > 1
    r1[flip], r2[flip] = 1 - r1[flip], 1 - r2[flip]
    return t[:, 0] + r1[:, None] * (t[:, 1] - t[:, 0]) + r2[:, None] * (t[:, 2] - t[:, 0])


def add_noise(points, sigma, seed):
    """Gaussian noise of standard deviation sigma L (L the longest side) along a random direction per point."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=points.shape)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    side = float((points.max(axis=0) - points.min(axis=0)).max())
    return points + d * (rng.normal(size=(len(points), 1)) * sigma * side)


def point_to_mesh(points, vertices, faces, candidates=48):
    """Distance of every point to a mesh (float64 [N]): the fp32 point-to-triangle distance of the mesh score
    (tests/watertight_oracle.tri_dist) over the `candidates` faces with the nearest centroids.  On the wand's fine
    faces that set holds the nearest face for points this close to the surface."""
    from scipy.spatial import cKDTree
    from tests.watertight_oracle import tri_dist
    v = np.asarray(vertices, F32)
    tri = v[np.asarray(faces, np.int64)]
    cand = cKDTree(tri.mean(axis=1).astype(F64)).query(np.asarray(points, F64), candidates)[1]
    p = np.asarray(points, F32)
    out = np.empty(len(p))
    for s in range(0, len(p), 20000):
        c = cand[s:s + 20000]
        t = tri[c]
        q = p[s:s + 20000, None, :]
        d = tri_dist(tuple(np.broadcast_to(q[..., a], c.shape) for a in range(3)),
                     *(tuple(t[:, :, vtx, a] for a in range(3)) for vtx in range(3)))
        out[s:s + 20000] = d.min(axis=1)
    return out


def rms(x):
    return float(np.sqrt(np.mean(np.square(np.asarray(x, F64)))))


def smoothed_input(points, k, plane_only=False):
    """The public path on the CPU: frame, smoothing, back to the input's units."""
    before = frame_map(points)
    r = smooth(before, k, plane_only=plane_only)
    return to_input_units(points, before, r["points"]), r


def cube_points(n, seed):
    """n points uniform on the surface of the unit cube [-0.5, 0.5]^3 (float64)."""
    rng = np.random.default_rng(seed)
    p = rng.uniform(-0.5, 0.5, (n, 3))
    axis = rng.integers(0, 3, n)
    p[np.arange(n), axis] = np.where(rng.integers(0, 2, n) == 1, 0.5, -0.5)
    return p


def cube_distance(p):
    """Distance of points to the surface of the unit cube [-0.5, 0.5]^3."""
    a = np.abs(p) - 0.5
    outside = np.linalg.norm(np.maximum(a, 0), axis=1)
    return np.where(outside > 0, outside, -np.max(a, axis=1))


def sphere_points(n, seed, radius=0.5):
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1, keepdims=True) * radius


def k_table(n=100_000, ks=(8, 16, 24, 32, 48), sigmas=(0.0, 0.001, 0.003), seed=0):
    """The rows of DESIGN.md section 1.8: per cloud and noise level the RMS distance to the true surface before and
    after smoothing (quadratic, and the plane-only projection), in units of the longest side."""
    z = np.load(__file__.replace("smooth_oracle.py", "golden/wand_mesh.npz"))
    v, f = z["vertices"], z["faces"]
    wand = surface_points(v, f, n, seed)
    side = float((wand.max(axis=0) - wand.min(axis=0)).max())
    rows = []
    for sigma in sigmas:
        pts = add_noise(wand, sigma, seed + 1) if sigma else wand
        row = {"cloud": "wand", "sigma": sigma, "before": rms(point_to_mesh(pts, v, f)) / side}
        for kk in ks:
            for plane_only in (False, True):
                out, r = smoothed_input(pts, kk, plane_only)
                row[("plane" if plane_only else "quad", kk)] = rms(point_to_mesh(out, v, f)) / side
        rows.append(row)
    cube = cube_points(n, seed)
    edge = np.sort(np.abs(cube), axis=1)[:, 1] > 0.49      # within 0.01 of an edge
    for sigma in sigmas[:2]:
        pts = add_noise(cube, sigma, seed + 1) if sigma else cube
        row = {"cloud": "cube", "sigma": sigma, "before": rms(cube_distance(pts))}
        for kk in ks:
            out, _ = smoothed_input(pts, kk)
            row[("quad", kk)] = rms(cube_distance(out))
            row[("edge", kk)] = rms(cube_distance(out)[edge])
            row[("edge_max", kk)] = float(np.abs(cube_distance(out)[edge]).max())
        rows.append(row)
    sphere = sphere_points(n, seed)
    for sigma in sigmas[1:]:
        pts = add_noise(sphere, sigma, seed + 1)
        row = {"cloud": "sphere r=0.5", "sigma": sigma, "before": float(np.linalg.norm(pts, axis=1).mean()) - 0.5}
        for kk in ks:
            for plane_only in (False, True):
                out, _ = smoothed_input(pts, kk, plane_only)
                row[("plane" if plane_only else "quad", kk)] = float(np.linalg.norm(out, axis=1).mean()) - 0.5
        rows.append(row)
    return rows


if __name__ == "__main__":
    import sys
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000
    for row in k_table(n):
        print({str(key): (round(val, 7) if isinstance(val, float) else val) for key, val in row.items()})
