"""Outlier removal of a point cloud on the GPU (ma_remove_outliers), for `--remove_outliers`.

    from meshanything_b200.outliers import remove_outliers
    idx, st = remove_outliers(xyz)          # xyz [N, 3] (numpy or torch) -> kept indices int64 (ascending, on the GPU)

The definition (DESIGN.md section 1.3): in the output frame of metrics.to_output_frame, a point's mean distance to its
k nearest other points is compared with the mean and standard deviation of that quantity over the cloud (a point is
kept iff d_i <= mu + std_ratio sigma, the rule of Open3D's remove_statistical_outlier), then the connected components of
the kNN graph among the kept points that hold less than min_component of them are dropped, the largest always
staying.  There is no CPU fallback.
"""
from __future__ import annotations

from typing import NamedTuple

from . import capi
from .pointcloud import frame_points, require_gpu


class OutlierStats(NamedTuple):
    n_points: int
    removed_statistical: int      # points over the distance threshold
    removed_components: int       # points of the dropped components
    components: int               # connected components among the statistical inliers (0: stage off)
    components_dropped: int
    mean_distance: float          # mu, sigma and mu + std_ratio sigma, in the output frame
    std_distance: float
    threshold: float
    kept: int


def remove_outliers(points, k: int = 16, std_ratio: float = 2.0, min_component: float = 0.01):
    """points [N, 3] -> (kept indices int64 [n_kept], ascending, on the GPU; OutlierStats).

    k neighbours (1..64, k < N), std_ratio the distance threshold in standard deviations above the mean,
    min_component the least share of the statistical inliers a connected component must hold (0: keep all)."""
    dev = require_gpu("removing outliers (--remove_outliers)")
    idx, keep, st = capi.remove_outliers(frame_points(points, dev, "remove_outliers"), k, std_ratio, min_component)
    n, inl, kept = keep.shape[0], int(st[3]), int(st[6])
    return idx, OutlierStats(n_points=n, removed_statistical=n - inl, removed_components=inl - kept,
                             components=int(st[4]), components_dropped=int(st[5]), mean_distance=float(st[0]),
                             std_distance=float(st[1]), threshold=float(st[2]), kept=kept)
