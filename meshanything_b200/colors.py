"""The colours of a scan carried onto the mesh made from it, on the GPU (ma_transfer_colors), for `--transfer_colors`.

    from meshanything_b200.colors import transfer_colors
    rgb, st = transfer_colors(vertices, faces, points, colors)   # numpy or torch -> fp32 [V, 3] in [0, 1], on the GPU

The definition (DESIGN.md section 1.9): the vertices and the points are mapped into one fp32 frame (x - c) / L, c and L
the float64 bounding-box centre and longest side of the points.  Every point within max_distance L of the mesh adds its
colour to the corners of its nearest face, weighted by the barycentric coordinates of its nearest point on that face,
in exact fixed-point sums; a vertex no point reaches takes the colour of its nearest point.  Colours are averaged as
stored (no gamma conversion).  There is no CPU fallback.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from . import capi
from .pointcloud import require_gpu

DEFAULT_DISTANCE = 0.05   # DESIGN.md section 1.9: a share of the scan's longest side; not tuned on real scans


class ColorStats(NamedTuple):
    n_points: int
    used: int                 # points within max_distance of the mesh, whose colours were averaged
    beyond: int               # points farther away (on something the mesh does not cover)
    fallback_vertices: int    # vertices no used point reached, coloured by their nearest point


def _f64(x, dev) -> torch.Tensor:
    t = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))
    return t.to(dev, torch.float64)


def frame(points, vertices, dev):
    """(points, vertices) -> contiguous fp32 (x - c) / L on `dev`, c and L the float64 bounding-box centre and longest
    side of the points (0 counts as 1), computed in float64 and rounded once, so large offsets (scan or UTM
    coordinates) cost no precision."""
    p, v = _f64(points, dev), _f64(vertices, dev)
    if p.dim() != 2 or p.shape[1] != 3 or v.dim() != 2 or v.shape[1] != 3:
        raise ValueError(f"transfer_colors: points [N, 3] and vertices [V, 3], got {tuple(p.shape)} and "
                         f"{tuple(v.shape)}")
    if p.shape[0] == 0:
        raise ValueError("transfer_colors: no points")
    lo, hi = p.amin(dim=0), p.amax(dim=0)
    c = (lo + hi) / 2
    side = float((hi - lo).max())
    side = side if side > 0 else 1.0
    return ((p - c) / side).float().contiguous(), ((v - c) / side).float().contiguous()


def transfer_colors(vertices, faces, points, colors, max_distance: float = DEFAULT_DISTANCE):
    """vertices [V, 3] and faces [F, 3] of a mesh, points [N, 3] and colors [N, 3] (in [0, 1]) of the scan it was made
    from, in the same units (numpy or torch) -> (vertex colours fp32 [V, 3] on the GPU, ColorStats).  max_distance is a
    share of the points' longest side, in (0, 1]."""
    dev = require_gpu("colour transfer (--transfer_colors)")
    if isinstance(max_distance, bool) or not isinstance(max_distance, (int, float, np.floating, np.integer)):
        raise ValueError(f"transfer_colors: max_distance must be a real number, got {max_distance!r}")
    if not (np.isfinite(max_distance) and 0 < max_distance <= 1):
        raise ValueError(f"transfer_colors: max_distance must be in (0, 1] (a share of the points' longest side), got "
                         f"{max_distance}")
    p, v = frame(points, vertices, dev)
    f = faces if isinstance(faces, torch.Tensor) else torch.as_tensor(np.asarray(faces))
    if f.dtype.is_floating_point or f.dtype.is_complex or f.dtype == torch.bool:
        raise ValueError(f"transfer_colors: integer face indices, got {f.dtype}")
    if f.numel() and (int(f.min()) < 0 or int(f.max()) >= v.shape[0]):
        raise ValueError(f"transfer_colors: face indices outside [0, {v.shape[0]})")
    f = f.to(dev, torch.int32).contiguous()
    c = colors if isinstance(colors, torch.Tensor) else torch.as_tensor(np.asarray(colors))
    c = c.to(dev, torch.float32).contiguous()
    out, st = capi.transfer_colors(v, f, p, c, float(max_distance))
    return out, ColorStats(n_points=int(p.shape[0]), used=int(st[0]), beyond=int(st[1]), fallback_vertices=int(st[2]))
