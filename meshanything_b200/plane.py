"""Removal of the dominant plane of a point cloud on the GPU (ma_remove_plane), for `--remove_plane`.

    from meshanything_b200.plane import remove_plane
    idx, st = remove_plane(xyz)            # xyz [N, 3] (numpy or torch) -> kept indices int64 (ascending, on the GPU)

The definition (DESIGN.md section 1.6): in the output frame of metrics.to_output_frame, RANSAC draws `iterations`
planes through three seeded random points and keeps the one with the most points within `distance` (lowest hypothesis
on ties); its points are refitted by least squares, and the points on the refit plane and below it (the side holding
fewer points: the table, its legs, the floor) are removed.  A scanned object stands on something, and that support is
often most of the scan.  The step removes the largest plane whatever it is: a box with no support under it loses its
largest face.  There is no CPU fallback.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

from . import capi
from .pointcloud import frame_points, longest_side, require_gpu


class PlaneStats(NamedTuple):
    found: bool                   # False: no hypothesis had 3 points on it, nothing was removed
    normal: tuple                 # unit normal of the refit plane in the output frame, from the support to the object
    offset: float                 # d of n . p + d = 0 in the output frame
    threshold: float              # the distance threshold in the input's own units
    hypothesis: int               # the winning hypothesis and its on-plane count
    hypothesis_count: int
    valid_hypotheses: int         # hypotheses whose three points span a plane
    on: int                       # points on the refit plane, above it (kept) and below it
    above: int
    below: int
    kept: int


def remove_plane(points, distance: float = 0.01, iterations: int = 1000, seed: int = 0):
    """points [N, 3] -> (kept indices int64 [n_kept], ascending, on the GPU; PlaneStats).

    distance the on-plane threshold as a share of the bounding box's longest side (0 < distance <= 1), iterations the
    number of RANSAC hypotheses (1..65536), seed any integer in [0, 2^64).  3 <= N <= 2^24."""
    dev = require_gpu("removing the support plane (--remove_plane)")
    idx, keep, st = capi.remove_plane(frame_points(points, dev, "remove_plane"), distance, iterations, seed)
    t32 = float(np.float32(distance))
    return idx, PlaneStats(found=bool(st[0]), normal=(float(st[1]), float(st[2]), float(st[3])), offset=float(st[4]),
                           threshold=t32 * longest_side(points), hypothesis=int(st[5]), hypothesis_count=int(st[6]),
                           valid_hypotheses=int(st[7]), on=int(st[8]), above=int(st[9]), below=int(st[10]),
                           kept=int(st[11]))
