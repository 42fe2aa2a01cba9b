"""Farthest-point subsampling of a point cloud on the GPU (ma_farthest_point_sample), for `--subsample fps`.

    from meshanything_b200.subsample import farthest_point_sample
    idx, r2 = farthest_point_sample(xyz, 4096, start)   # xyz [N, 3] (numpy or torch) -> picks int64 [4096], r2 fp32

The definition (DESIGN.md section 1.4): in the output frame of metrics.to_output_frame, pick 0 is `start` and every
next pick is the unpicked point farthest (fp32 d^2) from all picks so far, lowest index on ties; r2[t] is the squared
covering radius of the first t + 1 picks.  The subset covers the surface evenly whatever the density of the input.
FPS takes the extremes first, so a stray point is always among the first picks: clean scans with --remove_outliers
(outliers.remove_outliers) first.  There is no CPU fallback.
"""
from __future__ import annotations

from . import capi
from .pointcloud import frame_points, require_gpu


def farthest_point_sample(points, m: int = 4096, start: int = 0):
    """points [N, 3] (numpy or torch, any float dtype) -> (picks int64 [m] in pick order, r2 fp32 [m]), on the GPU.

    1 <= m <= N <= 2^24, 0 <= start < N.  r2[m - 1] is the squared covering radius of the whole subset in the output
    frame: every point lies within sqrt(r2[m - 1]) of a pick."""
    dev = require_gpu("farthest-point subsampling (--subsample fps)")
    return capi.farthest_point_sample(frame_points(points, dev, "farthest_point_sample"), m, start)
