"""Shared helpers of the test-suite (synthetic checkpoint, inputs)."""
import functools

import torch

from meshanything_b200.checkpoint import synthetic_decoder_state_dict


@functools.lru_cache(maxsize=4)
def decoder_sd(n_layers: int, seed: int = 0):
    return synthetic_decoder_state_dict(seed, n_layers=n_layers)


def random_prefix(batch: int, seed: int = 1) -> torch.Tensor:
    """Stand-in for processed_point_feature (meshanything.py:138): fp32 [B,257,1024]."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(batch, 257, 1024, generator=g) * 0.7
