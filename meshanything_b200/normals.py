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

import numpy as np
import torch

from . import capi, metrics


def _device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("estimating normals (--input_type pc) needs a CUDA GPU and libmeshanything_b200.so; there is "
                           "no CPU fallback (clouds with normals go through --input_type pc_normal)")
    try:
        capi.lib()
    except Exception as e:
        raise RuntimeError("estimating normals (--input_type pc) needs libmeshanything_b200.so: " + str(e)) from e
    return torch.device("cuda", torch.cuda.current_device())


def estimate_normals(points, k: int = 16) -> torch.Tensor:
    """points [N, 3] (numpy or torch, any float dtype, any device) -> fp32 [N, 3] oriented unit normals on the GPU.

    float64 input is first shifted by its float64 bounding-box centre, so large offsets (scan or UTM coordinates) do not
    cost precision in the fp32 frame; fp32 / fp16 input goes through the frame map as it is."""
    dev = _device()
    pts = torch.as_tensor(np.asarray(points) if not isinstance(points, torch.Tensor) else points)
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise ValueError(f"estimate_normals: points [N, 3], got {tuple(pts.shape)}")
    if not pts.is_floating_point():
        pts = pts.to(torch.float64)
    pts = pts.to(dev)
    if pts.dtype == torch.float64 and pts.shape[0] > 0:
        pts = pts - (pts.amin(dim=0) + pts.amax(dim=0)) / 2
    frame = metrics.to_output_frame(pts[None])[0]
    return capi.estimate_normals(frame, k)
