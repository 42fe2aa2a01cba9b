"""Oriented normals of a bare point cloud on the GPU (ma_estimate_normals), for `--input_type pc`.

    from meshanything_b200.normals import estimate_normals
    n = estimate_normals(xyz, k=16)         # xyz [N, 3] (numpy or torch) -> fp32 [N, 3] unit normals on the GPU

The definition (DESIGN.md section 1.2): the cloud is mapped into the output frame by metrics.to_output_frame, each
point's normal is the smallest-eigenvalue direction of the covariance of the point and its k nearest neighbours, and
the signs are propagated along the minimum spanning forest of the kNN graph (Hoppe et al. 1992) from the point of each
connected component that lies farthest from the bounding-box centre, whose normal points away from that centre.
Estimate on the dense cloud: at the 4096 points the model sees, neighbourhoods are too wide for a usable plane fit.
There is no CPU fallback.
"""
from __future__ import annotations

import torch

from . import capi
from .pointcloud import frame_points, require_gpu


def estimate_normals(points, k: int = 16) -> torch.Tensor:
    """points [N, 3] (numpy or torch, any float dtype, any device) -> fp32 [N, 3] oriented unit normals on the GPU.

    float64 input is first shifted by its float64 bounding-box centre, so large offsets (scan or UTM coordinates) do not
    cost precision in the fp32 frame; fp32 / fp16 input goes through the frame map as it is."""
    dev = require_gpu("estimating normals (--input_type pc)",
                      " (clouds with normals go through --input_type pc_normal)")
    return capi.estimate_normals(frame_points(points, dev, "estimate_normals"), k)
