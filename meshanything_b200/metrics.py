"""Quality of generated meshes against the point cloud they were made from, scored on the GPU (ma_mesh_score).

    from meshanything_b200 import metrics
    s = metrics.score(model(pc), pc)        # any output of MeshAnything.forward with its input cloud
    s["chamfer"], s["normal_consistency"]   # [S] per shape (or [S, N] for meshes [S, N, F, 3, 3])

The metric (DESIGN.md section 1, row f6): the cloud is mapped into the output frame, p' = (p - c) / L with c the centre
and L the longest side of its bounding box (the rule the reference's app uses to show the input beside the output);
chamfer = p2m + m2p, where p2m is the mean distance from the cloud points to the nearest valid face and m2p the
area-weighted mean distance from 16 fixed quadrature points per face to the nearest cloud point; normal consistency is
the mean of the two matching |n . n_face| means.  Lower chamfer is better.  A candidate without a valid face, or whose
faces have zero total area, scores chamfer = +inf and normal consistency 0.
"""
from __future__ import annotations

import torch

from . import capi


def to_output_frame(pc_normal: torch.Tensor) -> torch.Tensor:
    """[S, P, 6] (xyz | normal, any float dtype) -> fp32 [S, P, 6] with xyz mapped to (p - c) / L in fp32 (L = 0, a
    single point, maps by p - c); the normals are passed through, converted but not renormalised."""
    pc = torch.as_tensor(pc_normal).to(torch.float32)
    xyz = pc[..., :3]
    lo, hi = xyz.amin(dim=-2, keepdim=True), xyz.amax(dim=-2, keepdim=True)
    centre = (lo + hi) / 2
    side = (hi - lo).amax(dim=-1, keepdim=True)
    side = torch.where(side > 0, side, torch.ones_like(side))
    return torch.cat([(xyz - centre) / side, pc[..., 3:]], dim=-1)


def shape_frame(xyz) -> tuple:
    """The map to_output_frame applies to rows [P, 3] (any float dtype), in float64: (centre [3], longest side), the
    bounding box's centre and longest side, 0 counting as 1."""
    p = torch.as_tensor(xyz).to(torch.float64)
    lo, hi = p.amin(dim=0), p.amax(dim=0)
    side = float((hi - lo).max())
    return (lo + hi) / 2, side if side > 0 else 1.0


def to_input_frame(faces: torch.Tensor, frame: tuple) -> torch.Tensor:
    """The inverse of to_output_frame in float64: every coordinate v of `faces` (any shape [..., 3]) becomes
    centre + side v, with frame = shape_frame of the cloud the faces were generated from."""
    centre, side = frame
    v = torch.as_tensor(faces).to(torch.float64)
    return centre.to(v.device) + side * v


def score(meshes: torch.Tensor, pc_normal: torch.Tensor) -> dict:
    """Score candidate meshes against the clouds they were generated from.

    meshes fp32 [S, N, F, 3, 3] (or [S, F, 3, 3]: one candidate per shape) on a CUDA device, NaN rows = absent faces,
    coordinates in the detokenizer frame; pc_normal [S, P, 6], the cloud as given to the model (any device).  Returns
    fp64 chamfer, p2m, m2p, normal_consistency and int32 faces (valid faces), each [S, N] (or [S]), on the meshes'
    device."""
    m = torch.as_tensor(meshes)
    single = m.dim() == 4
    if single:
        m = m.unsqueeze(1)
    cloud = to_output_frame(torch.as_tensor(pc_normal).to(m.device))
    terms, faces = capi.mesh_score(m, cloud)
    p2m, m2p, nc_p, nc_m = terms.unbind(-1)
    chamfer = p2m + m2p
    nc = torch.where(torch.isinf(chamfer), torch.zeros_like(chamfer), 0.5 * (nc_p + nc_m))
    out = {"chamfer": chamfer, "p2m": p2m, "m2p": m2p, "normal_consistency": nc, "faces": faces}
    return {k: v[:, 0] for k, v in out.items()} if single else out


def select(chamfer: torch.Tensor) -> torch.Tensor:
    """Index of the best candidate along the last axis: the lowest chamfer, the lowest index on ties (so candidate 0
    when every candidate scores +inf)."""
    return torch.argmin(chamfer, dim=-1)
