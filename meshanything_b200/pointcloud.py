"""What the GPU point-cloud stages (normals, outliers, subsample, plane, objects) share: the device check and the
map of an input cloud into the fp32 output frame the kernels work in."""
from __future__ import annotations

import numpy as np
import torch

from . import capi, metrics


def require_gpu(what: str, hint: str = "") -> torch.device:
    """The current CUDA device; RuntimeError naming `what` (e.g. "removing outliers (--remove_outliers)") when there is
    no GPU or no libmeshanything_b200.so.  `hint` follows the no-GPU message."""
    if not torch.cuda.is_available():
        raise RuntimeError(f"{what} needs a CUDA GPU and libmeshanything_b200.so; there is no CPU fallback{hint}")
    try:
        capi.lib()
    except Exception as e:
        raise RuntimeError(f"{what} needs libmeshanything_b200.so: " + str(e)) from e
    return torch.device("cuda", torch.cuda.current_device())


def frame_points(points, dev, what: str = "frame_points") -> torch.Tensor:
    """[N, 3] (numpy or torch, any float dtype) -> contiguous fp32 [N, 3] in the output frame on `dev`; float64 input
    is first shifted by its float64 bounding-box centre, so large offsets (scan or UTM coordinates) do not cost
    precision in the fp32 frame.  ValueError prefixed by `what` for any other shape."""
    pts = torch.as_tensor(np.asarray(points) if not isinstance(points, torch.Tensor) else points)
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise ValueError(f"{what}: points [N, 3], got {tuple(pts.shape)}")
    if not pts.is_floating_point():
        pts = pts.to(torch.float64)
    pts = pts.to(dev)
    if pts.dtype == torch.float64 and pts.shape[0] > 0:
        pts = pts - (pts.amin(dim=0) + pts.amax(dim=0)) / 2
    return metrics.to_output_frame(pts[None])[0]


def longest_side(points) -> float:
    """The longest side of the bounding box in the input's units (the length the frame divides by; 0 counts as 1)."""
    pts = points if isinstance(points, torch.Tensor) else torch.as_tensor(np.asarray(points))
    pts = pts.to(torch.float64)
    side = float((pts.amax(dim=0) - pts.amin(dim=0)).max()) if pts.shape[0] else 0.0
    return side if side > 0 else 1.0
