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

from . import capi
from .pointcloud import frame_points, longest_side, require_gpu


class ObjectStats(NamedTuple):
    clusters: int                 # connected components
    objects: int                  # clusters of at least min_points points
    object_points: int
    dropped_clusters: int
    dropped_points: int
    largest_dropped: int          # points in the largest dropped cluster (0: none dropped)
    sizes: tuple                  # points per object, in order
    distance: float               # e in the input's own units


def split_objects(points, distance: float = 0.02, min_points: int = 4096):
    """points [N, 3] -> (object indices int64 on the GPU, offsets int64 [objects + 1] on the GPU, ObjectStats).

    Object k holds indices[offsets[k]:offsets[k + 1]], ascending.  distance the neighbour distance as a share of the
    bounding box's longest side (0 < distance <= 1), 1 <= min_points <= N, 1 <= N <= 2^24."""
    dev = require_gpu("splitting a cloud into objects (--split_objects)")
    _, idx, offsets, st = capi.split_objects(frame_points(points, dev, "split_objects"), distance, min_points)
    off = offsets.cpu().numpy()
    return idx, offsets, ObjectStats(clusters=int(st[0]), objects=int(st[1]), object_points=int(st[2]),
                                     dropped_clusters=int(st[3]), dropped_points=int(st[4]),
                                     largest_dropped=int(st[5]), sizes=tuple(int(x) for x in np.diff(off)),
                                     distance=float(np.float32(distance)) * longest_side(points))
