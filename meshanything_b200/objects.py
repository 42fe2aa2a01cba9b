"""Splitting a point cloud into objects on the GPU (ma_split_objects), for `--split_objects`.

    from meshanything_b200.objects import split_objects
    idx, offsets, st = split_objects(xyz)   # xyz [N, 3] (numpy or torch) -> object k: idx[offsets[k]:offsets[k + 1]]

The definition (DESIGN.md section 1.7): in the output frame of metrics.to_output_frame, two points are neighbours when
their fp32 squared distance is at most fp32(e e), e = `distance` of the bounding box's longest side; the clusters are
the connected components of that graph, ordered by size (descending, lowest point index first on ties), and the
objects are the clusters of at least `min_points` points.  Objects that touch, or come closer than e, stay together:
run it after `--remove_plane`, or the table joins everything into one object.  There is no CPU fallback.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from . import capi
from .outliers import frame_points
from .plane import _longest_side


class ObjectStats(NamedTuple):
    clusters: int                 # connected components
    objects: int                  # clusters of at least min_points points
    object_points: int
    dropped_clusters: int
    dropped_points: int
    largest_dropped: int          # points in the largest dropped cluster (0: none dropped)
    sizes: tuple                  # points per object, in order
    distance: float               # e in the input's own units


def _device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("splitting a cloud into objects (--split_objects) needs a CUDA GPU and "
                           "libmeshanything_b200.so; there is no CPU fallback")
    try:
        capi.lib()
    except Exception as e:
        raise RuntimeError("splitting a cloud into objects (--split_objects) needs libmeshanything_b200.so: " + str(e)) from e
    return torch.device("cuda", torch.cuda.current_device())


def split_objects(points, distance: float = 0.02, min_points: int = 4096):
    """points [N, 3] -> (object indices int64 on the GPU, offsets int64 [objects + 1] on the GPU, ObjectStats).

    Object k holds indices[offsets[k]:offsets[k + 1]], ascending.  distance the neighbour distance as a share of the
    bounding box's longest side (0 < distance <= 1), 1 <= min_points <= N, 1 <= N <= 2^24."""
    dev = _device()
    shape = tuple(points.shape) if hasattr(points, "shape") else np.shape(points)
    if len(shape) != 2 or shape[1] != 3:
        raise ValueError(f"split_objects: points [N, 3], got {shape}")
    frame = frame_points(points, dev).contiguous()
    _, idx, offsets, st = capi.split_objects(frame, distance, min_points)
    off = offsets.cpu().numpy()
    return idx, offsets, ObjectStats(clusters=int(st[0]), objects=int(st[1]), object_points=int(st[2]),
                                     dropped_clusters=int(st[3]), dropped_points=int(st[4]),
                                     largest_dropped=int(st[5]), sizes=tuple(int(x) for x in np.diff(off)),
                                     distance=float(np.float32(distance)) * _longest_side(points))
