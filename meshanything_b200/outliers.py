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

import numpy as np
import torch

from . import capi, metrics


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


def _device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("removing outliers (--remove_outliers) needs a CUDA GPU and libmeshanything_b200.so; there is "
                           "no CPU fallback")
    try:
        capi.lib()
    except Exception as e:
        raise RuntimeError("removing outliers (--remove_outliers) needs libmeshanything_b200.so: " + str(e)) from e
    return torch.device("cuda", torch.cuda.current_device())


def frame_points(points, dev) -> torch.Tensor:
    """[N, 3] (numpy or torch, any float dtype) -> fp32 [N, 3] in the output frame on `dev`; float64 input is first
    shifted by its float64 bounding-box centre (as normals.estimate_normals does)."""
    pts = torch.as_tensor(np.asarray(points) if not isinstance(points, torch.Tensor) else points)
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise ValueError(f"remove_outliers: points [N, 3], got {tuple(pts.shape)}")
    if not pts.is_floating_point():
        pts = pts.to(torch.float64)
    pts = pts.to(dev)
    if pts.dtype == torch.float64 and pts.shape[0] > 0:
        pts = pts - (pts.amin(dim=0) + pts.amax(dim=0)) / 2
    return metrics.to_output_frame(pts[None])[0]


def remove_outliers(points, k: int = 16, std_ratio: float = 2.0, min_component: float = 0.01):
    """points [N, 3] -> (kept indices int64 [n_kept], ascending, on the GPU; OutlierStats).

    k neighbours (1..64, k < N), std_ratio the distance threshold in standard deviations above the mean,
    min_component the least share of the statistical inliers a connected component must hold (0: keep all)."""
    dev = _device()
    idx, keep, st = capi.remove_outliers(frame_points(points, dev), k, std_ratio, min_component)
    n, inl, kept = keep.shape[0], int(st[3]), int(st[6])
    return idx, OutlierStats(n_points=n, removed_statistical=n - inl, removed_components=inl - kept,
                             components=int(st[4]), components_dropped=int(st[5]), mean_distance=float(st[0]),
                             std_distance=float(st[1]), threshold=float(st[2]), kept=kept)
