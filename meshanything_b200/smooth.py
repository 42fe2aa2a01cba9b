"""Moving-least-squares smoothing of a point cloud on the GPU (ma_smooth_points), for `--smooth`.

    from meshanything_b200.smooth import smooth_points
    xyz2, st = smooth_points(xyz)          # xyz [N, 3] (numpy or torch) -> smoothed points, same dtype, on the GPU

The definition (DESIGN.md section 1.8): in the output frame of metrics.to_output_frame, each point is projected onto
the weighted least-squares quadratic height field fitted to it and its k nearest other points (weights
(1 - d^2 / H)^2, H twice the squared distance to the k-th neighbour), or onto their weighted plane where the quadratic
is singular or would move the point by more than sqrt(H).  Scanner noise a short way off the surface is pulled back
onto it; sharp edges are rounded.  Every row is kept and nothing random is drawn.  The move is added back in the input's
units in float64, so a point the stage does not move keeps its coordinates exactly.  There is no CPU fallback.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from . import capi
from .pointcloud import frame_points, longest_side, require_gpu

DEFAULT_K = 24   # DESIGN.md section 1.8: chosen from the k-table on the noisy wand


class SmoothStats(NamedTuple):
    n_points: int
    k: int
    quadratic: int                # points projected onto their quadratic
    singular: int                 # plane fallbacks: a Cholesky pivot at or below 1e-9 of the weight sum
    far: int                      # plane fallbacks: the quadratic would have moved the point by more than sqrt(H)
    mean_displacement: float      # how far the points moved, in the input's units
    max_displacement: float


def smooth_points(points, k: int = DEFAULT_K):
    """points [N, 3] -> (smoothed points [N, 3] in the input's dtype (float dtypes; float64 otherwise) and units, on the
    GPU; SmoothStats).  5 <= k <= 64, k < N <= 2^24."""
    dev = require_gpu("smoothing (--smooth)")
    frame = frame_points(points, dev, "smooth_points")
    q, st = capi.smooth_points(frame, k)
    x = points if isinstance(points, torch.Tensor) else torch.as_tensor(np.asarray(points))
    dtype = x.dtype if x.is_floating_point() else torch.float64
    x64 = x.to(dev, torch.float64)
    move = longest_side(points) * (q.to(torch.float64) - frame.to(torch.float64))
    dist = move.norm(dim=1)
    return (x64 + move).to(dtype), SmoothStats(
        n_points=int(frame.shape[0]), k=int(k), quadratic=int(st[0]), singular=int(st[1]), far=int(st[2]),
        mean_displacement=float(dist.mean()), max_displacement=float(dist.max()))
