"""Shared helpers of the test-suite (synthetic checkpoint, inputs)."""
import functools

import torch

from meshanything_b200.checkpoint import synthetic_decoder_state_dict


@functools.lru_cache(maxsize=4)
def decoder_sd(n_layers: int, seed: int = 0):
    return synthetic_decoder_state_dict(seed, n_layers=n_layers)


def skip_unless_persistent(flags: int) -> None:
    """flags = 0 selects the persistent decode kernel for batch-1 greedy decoding; on a device that cannot host it
    (ma_decode_persistent_supported: SM count and shared memory, e.g. an H100 with 132 SMs) the same call would run
    the per-phase kernels, which the flags = 16 cases already check, so the case is skipped and shows as such."""
    import pytest
    from meshanything_b200 import capi
    if flags == 0 and capi.lib().ma_decode_persistent_supported() != 1:
        pytest.skip("persistent decode kernel not supported on this device (needs every CTA to own fc1 and lm_head rows, "
                    "at most 64 each, no out_proj rows in the last 16 CTAs, and its rows within the shared memory of "
                    "an SM: 147 SMs); batch-1 greedy decoding runs on the per-phase kernels here")


def random_prefix(batch: int, seed: int = 1) -> torch.Tensor:
    """Stand-in for processed_point_feature (meshanything.py:138): fp32 [B,257,1024]."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(batch, 257, 1024, generator=g) * 0.7
