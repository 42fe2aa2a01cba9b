"""Drop-in for /root/reference/MeshAnything/miche/encode.py: `load_model(ckpt_path=None)` returns the point
encoder object `MeshAnything` holds as `self.point_encoder`.

The reference builds a Lightning-era module tree from `shapevae-256.yaml` with OmegaConf and runs it with
PyTorch ops.  Here the module is a thin handle: its weights arrive through
`MeshAnything.load_state_dict` (keys `point_encoder.model.shape_model.*`) and its two entry points
call the sm_90a kernels through the C ABI (`ma_encoder_forward`).  The yaml values are constants of
`meshanything_b200.config.ENC`.
"""
from __future__ import annotations

from typing import Optional

import torch

from meshanything_b200.config import ENC


class PointEncoder(torch.nn.Module):
    """`encode_latents` / `to_shape_latents` of AlignedShapeAsLatentPLModule (asl_pl_module.py:145-157,182-185)."""

    def __init__(self):
        super().__init__()
        self.arena = None          # meshanything_b200.encoder.EncoderArena, set by MeshAnything.load_state_dict
        self._last = None          # (point_feature, prefix) of the last encode: the C entry point produces both

    def _need(self):
        if self.arena is None:
            raise RuntimeError("point encoder has no weights: call MeshAnything.load_state_dict first")

    def encode_latents(self, surface: torch.Tensor) -> torch.Tensor:
        self._need()
        pf, prefix = self.arena.forward(surface)
        self._last = (pf, prefix)
        assert pf.shape[1] == ENC.num_latents
        return pf

    def encode_with_prefix(self, surface: torch.Tensor):
        """point_feature and the decoder prefix (process_point_feature, meshanything.py:125-132) in one call."""
        self._need()
        self._last = self.arena.forward(surface)
        return self._last


def load_model(ckpt_path: Optional[str] = None) -> PointEncoder:
    if ckpt_path is not None:
        raise ValueError("MeshAnything loads the encoder weights through load_state_dict (ckpt_path must be None, "
                         "as at meshanything.py:86)")
    return PointEncoder().eval()
