"""Host side of the ShapeOPT-350M decoder: weight arena + `generate()`.

Mirrors what `MeshAnything.forward` asks of `self.transformer.generate(...)`
(/root/reference/MeshAnything/models/meshanything.py:144-162) with the state-dict keys of
/root/reference/MeshAnything/models/shape_opt.py:188-235.  All arithmetic runs in
libmeshanything_b200.so; PyTorch only owns the memory.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import capi
from .config import DEC

_P = "transformer.model.decoder"


class DecoderArena:
    """fp16 (Linear) / fp32 (LayerNorm, embeddings) device copies of the decoder weights + the C struct."""

    def __init__(self, sd: Dict[str, torch.Tensor], device: torch.device, n_layers: Optional[int] = None):
        if device.type != "cuda":
            raise RuntimeError("DecoderArena needs a CUDA device (no CPU fallback)")
        if n_layers is None:
            n_layers = 0
            while f"{_P}.layers.{n_layers}.fc1.weight" in sd:
                n_layers += 1
        self.n_layers = n_layers
        self.device = device
        self.keep = []   # tensors referenced by raw pointers
        w = capi.DecoderWeights()
        w.n_layers = n_layers
        w.vocab = sd["transformer.lm_head.weight"].shape[0]

        def h16(t):
            t = t.detach().to(device=device, dtype=torch.float16).contiguous()
            self.keep.append(t)
            return t

        def f32(t):
            t = t.detach().to(device=device, dtype=torch.float32).contiguous()
            if t.data_ptr() % 256:      # a view into a packed buffer (e.g. the broadcast arena): kernels use 16-byte loads
                t = t.clone()
            self.keep.append(t)
            return t

        for i in range(n_layers):
            q = f"{_P}.layers.{i}"
            wqkv = torch.cat([sd[f"{q}.self_attn.{n}_proj.weight"] for n in "qkv"], dim=0)
            bqkv = torch.cat([sd[f"{q}.self_attn.{n}_proj.bias"] for n in "qkv"], dim=0)
            w.wqkv[i] = h16(wqkv).data_ptr()
            w.bqkv[i] = h16(bqkv).data_ptr()
            w.wo[i] = h16(sd[f"{q}.self_attn.out_proj.weight"]).data_ptr()
            w.bo[i] = h16(sd[f"{q}.self_attn.out_proj.bias"]).data_ptr()
            w.w1[i] = h16(sd[f"{q}.fc1.weight"]).data_ptr()
            w.b1[i] = h16(sd[f"{q}.fc1.bias"]).data_ptr()
            w.w2[i] = h16(sd[f"{q}.fc2.weight"]).data_ptr()
            w.b2[i] = h16(sd[f"{q}.fc2.bias"]).data_ptr()
            w.ln1g[i] = f32(sd[f"{q}.self_attn_layer_norm.weight"]).data_ptr()
            w.ln1b[i] = f32(sd[f"{q}.self_attn_layer_norm.bias"]).data_ptr()
            w.ln2g[i] = f32(sd[f"{q}.final_layer_norm.weight"]).data_ptr()
            w.ln2b[i] = f32(sd[f"{q}.final_layer_norm.bias"]).data_ptr()
        w.lm_head = h16(sd["transformer.lm_head.weight"]).data_ptr()
        # embed_with_vae (shape_opt.py:237-245): input_layer(quantize_codebooks[0][id-3]) does not depend
        # on the step -> fold it once into a [codebook,1024] fp16 table with the same canonical Linear.
        cb = h16(sd[f"{_P}.quantize_codebooks"][0])
        in_w = h16(sd[f"{_P}.input_layer.weight"])
        in_b = h16(sd[f"{_P}.input_layer.bias"])
        self.tok_table = capi.linear_f16(in_w, in_b, cb)
        torch.cuda.synchronize(device)
        self.keep = [t for t in self.keep if t is not cb and t is not in_w and t is not in_b]
        w.codebook = cb.shape[0]
        w.tok_table = self.tok_table.data_ptr()
        w.extra = f32(sd[f"{_P}.extra_embeds.weight"]).data_ptr()
        w.tok_pos = f32(sd[f"{_P}.token_embed_positions.weight"]).data_ptr()
        w.cond = f32(sd[f"{_P}.cond_embed.weight"]).data_ptr()
        pos = f32(sd[f"{_P}.embed_positions.weight"])
        w.pos = pos.data_ptr()
        w.npos = pos.shape[0]
        self.c = w

    def weight_bytes_per_step(self) -> int:
        """fp16 bytes of weights one decode step reads (SURVEY.md 8d, minus the folded input_layer)."""
        per_layer = (3 * 1024 * 1024 + 3 * 1024) + (1024 * 1024 + 1024) + (4096 * 1024 + 4096) + (1024 * 4096 + 1024)
        return 2 * (self.n_layers * per_layer + self.c.vocab * 1024)


class Generator:
    """Preallocated KV cache + workspace for `batch` sequences of at most `tmax` positions."""

    def __init__(self, arena: DecoderArena, batch: int, tmax: int):
        self.arena, self.batch, self.tmax = arena, batch, tmax
        L = capi.lib()
        dev = arena.device
        self.kv = torch.empty(L.ma_kv_cache_bytes(arena.n_layers, batch, tmax), dtype=torch.uint8, device=dev)
        self.ws = torch.empty(L.ma_decoder_workspace_bytes(batch, tmax), dtype=torch.uint8, device=dev)

    def generate(self, prefix: torch.Tensor, max_new_tokens: int, do_sample: bool = False, top_k: int = 50,
                 top_p: float = 0.95, seed: int = 0, eos_id: int = DEC.eos_id, pad_id: int = DEC.pad_id,
                 forced_ids: Optional[torch.Tensor] = None, want_logits: bool = False, flags: int = 0):
        """prefix fp32 [B,257,1024] on the device -> (ids int32 [B,max_new], lens int32 [B][, logits])."""
        B = prefix.shape[0]
        assert B == self.batch and prefix.shape[1:] == (DEC.cond_length, DEC.hidden)
        assert prefix.is_cuda and prefix.dtype == torch.float32
        prefix = prefix.contiguous()
        dev = prefix.device
        # persistent output buffers: stable pointers keep the per-step CUDA graphs of the library reusable across calls
        if getattr(self, "_ids_buf", None) is None or self._ids_buf.shape != (B, max_new_tokens):
            self._ids_buf = torch.empty((B, max_new_tokens), dtype=torch.int32, device=dev)
            self._lens_buf = torch.empty((B,), dtype=torch.int32, device=dev)
        ids, lens = self._ids_buf, self._lens_buf
        logits = None
        if want_logits:
            logits = torch.zeros((max_new_tokens, B, self.arena.c.vocab), dtype=torch.float16, device=dev)
        if forced_ids is not None:
            forced_ids = forced_ids.to(device=dev, dtype=torch.int32).contiguous()
        samp = capi.Sampling(int(do_sample), int(top_k), float(top_p), int(seed))
        rc = capi.lib().ma_decode_generate(C.byref(self.arena.c), capi.ptr(prefix), B, self.tmax, max_new_tokens,
                                           C.byref(samp), eos_id, pad_id, capi.ptr(self.kv), capi.ptr(self.ws),
                                           capi.ptr(ids), capi.ptr(lens), capi.ptr(forced_ids), capi.ptr(logits),
                                           flags, capi.stream_ptr())
        capi.check(rc, "ma_decode_generate")
        ids, lens = ids.clone(), lens.clone()          # the caller owns what it gets; the buffers are reused
        return (ids, lens, logits) if want_logits else (ids, lens)
