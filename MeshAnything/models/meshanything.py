"""Drop-in for /root/reference/MeshAnything/models/meshanything.py: same import path, constructor,
`load_state_dict(strict=True)` key set and `forward(pc_normal, sampling=False)` contract
(SURVEY.md 8b), with every arithmetic stage running in libmeshanything_b200.so (sm_90a):

    forward (meshanything.py:134-176)
      point_encoder.encode_latents + process_point_feature  -> ma_encoder_forward
      transformer.generate(inputs_embeds=..., greedy | top-k 50 / top-p 0.95)  -> ma_decode_generate
      ids post-processing + get_codes + tokenizer(...)       -> ma_detokenize

There is no PyTorch / CPU fallback: without a CUDA device or without the shared library this raises.
"""
from __future__ import annotations

from typing import Dict, NamedTuple

import torch
from torch import nn

from MeshAnything.miche.encode import load_model
from meshanything_b200 import checkpoint as _ck
from meshanything_b200.config import DEC


class Candidates(NamedTuple):
    """What MeshAnything.forward_candidates returns."""
    best: torch.Tensor                # [B, F, 3, 3] the kept candidate of every shape
    meshes: torch.Tensor              # [B, N, F, 3, 3] every candidate
    chamfer: torch.Tensor             # [B, N] fp64, lower is better (+inf: no face with an area)
    normal_consistency: torch.Tensor  # [B, N] fp64 in [0, 1]
    index: torch.Tensor               # [B] int64, the kept candidate


class MeshAnything(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        self.point_encoder = load_model(ckpt_path=None)
        self.num_quantizers = 3
        self.face_per_token = self.num_quantizers * 3
        self.cond_length = 257
        self.cond_dim = 768
        self.n_max_triangles = int(args.n_max_triangles)
        self.max_length = self.n_max_triangles * self.face_per_token + 2 + self.cond_length
        if int(getattr(args, "codebook_size", 8192)) != DEC.codebook_size or \
                int(getattr(args, "codebook_dim", 1024)) != DEC.codebook_dim:
            raise ValueError("only the published 8192 x 1024 codebook geometry is supported")
        if self.max_length > DEC.n_positions:
            raise ValueError(f"n_max_triangles={self.n_max_triangles} exceeds the {DEC.n_positions} learned positions")
        self.bos_token_id, self.eos_token_id, self.pad_token_id = DEC.bos_id, DEC.eos_id, DEC.pad_id
        self.seed = int(getattr(args, "seed", 0))
        self._dec = self._tok = None
        self._gens = {}
        self._device = None
        self._calls = 0
        self.eval()

    # ------------------------------------------------------------------ weights
    def expected_keys(self):
        return list(_ck.all_specs(DEC.n_layers).keys())

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True, device=None):
        """Same keys as the reference checkpoint (main.py:99-104).  Tensors may live on any device; they are
        converted to the fp16 / fp32 arenas on `device` (default: the tensors' CUDA device, else cuda:0)."""
        from meshanything_b200.decoder import DecoderArena
        from meshanything_b200.encoder import EncoderArena, TokenizerArena
        exp = set(self.expected_keys())
        got = set(state_dict.keys())
        # the BERT layers may come in either spelling; compare modulo that family
        bert = lambda ks: {k for k in ks if not k.startswith("tokenizer.decoder.layer.")}
        missing, unexpected = sorted(bert(exp) - bert(got)), sorted(bert(got) - bert(exp))
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict for MeshAnything: missing {missing[:5]} "
                               f"unexpected {unexpected[:5]}")
        if device is None:
            any_t = next(iter(state_dict.values()))
            device = any_t.device if any_t.is_cuda else torch.device("cuda", torch.cuda.current_device()) \
                if torch.cuda.is_available() else None
        if device is None:
            raise RuntimeError("MeshAnything needs a CUDA device (no CPU fallback)")
        device = torch.device(device)
        self._device = device
        self.point_encoder.arena = EncoderArena(state_dict, device)
        self._dec = DecoderArena(state_dict, device)
        self._tok = TokenizerArena(state_dict, device)
        self._gens = {}
        self._engines = {}
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def _generator(self, batch: int):
        from meshanything_b200.decoder import Generator
        g = self._gens.get(batch)
        if g is None:
            g = self._gens[batch] = Generator(self._dec, batch, self.max_length)
        return g

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, pc_normal, sampling: bool = False) -> torch.Tensor:
        """pc_normal [B,4096,6] (fp16, any device; host tensors are copied) -> [B, n_max_triangles, 3, 3] fp32 on
        the GPU, coordinates in [-0.5, 0.5), NaN rows where no face was generated."""
        if self._dec is None:
            raise RuntimeError("MeshAnything has no weights: call load_state_dict first")
        pc = torch.as_tensor(pc_normal)
        if not pc.is_cuda:
            pc = pc.to(self._device, non_blocking=True)
        point_feature, prefix = self.point_encoder.encode_with_prefix(pc)
        generate_length = self.max_length - self.cond_length
        gen = self._generator(pc.shape[0])
        ids, _lens = gen.generate(prefix, generate_length, do_sample=bool(sampling), top_k=50, top_p=0.95,
                                  seed=self.seed + self._calls, eos_id=self.eos_token_id, pad_id=self.pad_token_id)
        self._calls += 1
        self.last_ids = ids
        return self._tok.detokenize(ids, point_feature, self.n_max_triangles)

    # ------------------------------------------------------------------ best of N samples
    @torch.no_grad()
    def forward_candidates(self, pc_normal, num_samples: int) -> Candidates:
        """Not in the reference (whose app tells users to re-roll the seed when a result is unsatisfying): samples
        `num_samples` meshes of every shape as one batch and keeps the one closest to the input cloud.

        One sampled `forward` of pc_normal.repeat_interleave(num_samples, 0) -- candidate k of shape b is row
        b * num_samples + k of that call, bit for bit, and draws from its Philox stream -- then `metrics.score` against
        the shape's cloud and the lowest chamfer (lowest index on ties).  Returns Candidates(best [B, F, 3, 3],
        meshes [B, N, F, 3, 3], chamfer [B, N], normal_consistency [B, N], index [B])."""
        from meshanything_b200 import metrics
        n = int(num_samples)
        if n < 1:
            raise ValueError(f"num_samples must be >= 1, got {num_samples}")
        if self._dec is None:
            raise RuntimeError("MeshAnything has no weights: call load_state_dict first")
        pc = torch.as_tensor(pc_normal)
        if not pc.is_cuda:
            pc = pc.to(self._device)
        B = pc.shape[0]
        out = self.forward(pc.repeat_interleave(n, 0), sampling=True)
        meshes = out.reshape(B, n, *out.shape[1:])
        s = metrics.score(meshes, pc)
        index = metrics.select(s["chamfer"])
        best = meshes[torch.arange(B, device=meshes.device), index]
        return Candidates(best, meshes, s["chamfer"], s["normal_consistency"], index)

    # ------------------------------------------------------------------ queue of shapes (continuous batching)
    @torch.no_grad()
    def forward_queue(self, pc_normals, sampling: bool = False, slots: int = 8, poll_every: int = 32):
        """Not in the reference (SURVEY.md section 8(f)2): runs any number of point clouds ([4096,6] each) through
        `slots` decoder cache slots, refilling a slot as soon as its mesh has hit EOS instead of padding it until the
        longest mesh of a batch ends (`main.py:137-152` + HF generate).  Returns a list of [n_max_triangles,3,3]
        tensors in input order; under greedy decoding each equals `forward` on that shape alone."""
        from meshanything_b200.scheduler import SlotEngine, SlotScheduler
        if self._dec is None:
            raise RuntimeError("MeshAnything has no weights: call load_state_dict first")
        generate_length = self.max_length - self.cond_length
        key = (int(slots), bool(sampling))
        feats = {}

        def to_prefix(item):
            idx, pc = item
            pc = torch.as_tensor(pc)
            if not pc.is_cuda:
                pc = pc.to(self._device, non_blocking=True)
            point_feature, prefix = self.point_encoder.encode_with_prefix(pc.reshape(1, *pc.shape[-2:]))
            feats[idx] = point_feature
            return prefix[0]

        eng = self._engines.get(key)
        if eng is None:
            eng = self._engines[key] = SlotEngine(self._dec, int(slots), self.max_length, generate_length,
                                                  do_sample=bool(sampling), top_k=50, top_p=0.95, seed=self.seed,
                                                  eos_id=self.eos_token_id, pad_id=self.pad_token_id)
        eng.to_prefix = to_prefix
        eng.samp.seed = self.seed + self._calls
        eng.reset()
        self._calls += 1
        sched = SlotScheduler(eng, int(slots), generate_length, prefix_len=self.cond_length, poll_every=poll_every)
        out = {}
        for idx, ids in sched.run(enumerate(pc_normals)):
            row = torch.full((1, generate_length), self.pad_token_id, dtype=torch.int32, device=self._device)
            row[0, :ids.numel()] = ids
            out[idx] = self._tok.detokenize(row, feats.pop(idx), self.n_max_triangles)[0]
        self.last_queue_stats = sched.stats
        return [out[i] for i in range(len(out))]
