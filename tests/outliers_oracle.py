"""numpy restatement of csrc/outliers.cu (test infrastructure only): statistical and small-component outlier removal as
DESIGN.md section 1.3 defines it.

The neighbours are tests/normals_oracle.knn (the exact kNN of section 1.2), the fp32 sqrt is numpy's (correctly
rounded, like __fsqrt_rn), every fp64 sum is a sequential loop in the kernels' order (never numpy's pairwise
reduction), and the components come from scipy with their labels set to the lowest index: d_i, mu, sigma, the
threshold, the masks and the counts agree with the GPU bit for bit.
"""
import numpy as np

from tests import normals_oracle as NO

F32 = np.float32
F64 = np.float64
TILE = 256


def frame_map(points):
    """[N, 3] -> the fp32 output frame; float64 input is first shifted by its float64 bounding-box centre."""
    p = np.asarray(points)
    if p.dtype == F64:
        p = p - (p.min(axis=0) + p.max(axis=0)) / 2
    return NO.frame_map(p)


def d2_of(p, nbr):
    """fp32 (dx dx + dy dy) + dz dz of every point against its neighbours [N, k]."""
    p = np.asarray(p, F32)
    return NO._d2(p[:, None, :], p[nbr])


def mean_distance(p, nbr):
    """d_i = (sum over ranks, in rank order, of fp64(fp32 sqrt(d^2))) / k."""
    r = np.sqrt(d2_of(p, nbr)).astype(F64)
    s = np.zeros(len(r), F64)
    for e in range(r.shape[1]):
        s = s + r[:, e]
    return s / F64(r.shape[1])


def fixed_sum(x):
    """Sum of fp64 x [N]: tiles of 256 consecutive values, each summed in order from 0, then the partials in order."""
    x = np.asarray(x, F64)
    tiles = -(-len(x) // TILE)
    t = np.zeros(tiles * TILE, F64)
    t[:len(x)] = x
    t = t.reshape(tiles, TILE)
    part = np.zeros(tiles, F64)
    for j in range(TILE):
        part = part + t[:, j]        # zero padding adds exactly nothing to these non-negative sums
    s = 0.0
    for v in part.tolist():
        s = s + v
    return s


def moments(dbar, std_ratio):
    """(mu, sigma, threshold): mu = sum / N, sigma = sqrt(sum (d - mu)^2 / (N - 1)) (0 when N = 1)."""
    n = len(dbar)
    mu = F64(fixed_sum(dbar)) / F64(n)
    d = np.asarray(dbar, F64) - mu
    sigma = np.sqrt(F64(fixed_sum(d * d)) / F64(n - 1)) if n > 1 else F64(0)
    return mu, sigma, mu + F64(std_ratio) * sigma


def components(n, nbr, inl):
    """Labels [N] (lowest index of the component; -1 for non-inliers) of the graph of kNN edges between inliers."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    k = nbr.shape[1]
    i = np.repeat(np.arange(n), k)
    j = nbr.reshape(-1)
    ok = inl[i] & inl[j]
    g = coo_matrix((np.ones(int(ok.sum())), (i[ok], j[ok])), shape=(n, n)).tocsr()
    _, lab = connected_components(g, directed=False)
    low = np.full(lab.max() + 1, n, np.int64)
    np.minimum.at(low, lab, np.arange(n))
    return np.where(inl, low[lab], -1)


def remove_outliers(points_frame, k=16, std_ratio=2.0, min_component=0.01, nbr=None):
    """Points already in the frame (fp32 [N, 3]) -> dict: keep bool [N], kept int64 (ascending), mean_dist fp64 [N],
    knn int64 [N, k], mu, sigma, threshold, and the counts of stats_out (inliers, components, dropped, kept)."""
    p = np.asarray(points_frame, F32)
    n = len(p)
    nbr = NO.knn(p, k) if nbr is None else nbr
    dbar = mean_distance(p, nbr)
    mu, sigma, thr = moments(dbar, std_ratio)
    inl = dbar <= thr
    keep = inl.copy()
    ncomp = dropped = 0
    if min_component > 0:
        lab = components(n, nbr, inl)
        roots = np.nonzero(lab == np.arange(n))[0]
        size = np.bincount(lab[inl], minlength=n)
        ncomp = len(roots)
        largest = roots[np.argmax(size[roots])] if ncomp else -1      # argmax: the first (lowest) root on ties
        big = (size.astype(F64) >= F64(min_component) * F64(int(inl.sum()))) | (np.arange(n) == largest)
        keep = inl & big[np.maximum(lab, 0)]
        dropped = int((~big[roots]).sum())
    return {"keep": keep, "kept": np.nonzero(keep)[0], "mean_dist": dbar, "knn": nbr, "mu": mu, "sigma": sigma,
            "threshold": thr, "inliers": int(inl.sum()), "components": ncomp, "dropped": dropped,
            "n_kept": int(keep.sum())}
