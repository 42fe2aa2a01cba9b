"""ctypes front end of the CPU decoder oracle (oracle/decoder_oracle.c) -- TEST INFRASTRUCTURE ONLY.

`OracleDecoder.generate` restates what `MeshAnything.forward` asks of HF `generate()`
(/root/reference/MeshAnything/models/meshanything.py:144-162) for transformers==4.39.3
`GenerationMixin._greedy_search`: step 0 feeds `inputs_embeds`, later steps feed only the last id;
greedy = argmax of the fp16 logits (lowest index on ties), or any other pick the caller passes (the sampler
restatement of tests/sampler_oracle.py); a finished row emits pad; stop when every row has produced eos or after
`max_new_tokens`.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libma_oracle.so")
_lib = None

u16p = C.POINTER(C.c_uint16)
f32p = C.POINTER(C.c_float)
i32p = C.POINTER(C.c_int)


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (recipe: oracle/Makefile)."""
    src = os.path.join(_HERE, "decoder_oracle.c")
    hdr = os.path.join(_HERE, "..", "include", "ma_canon_constants.h")
    stale = (not os.path.exists(_LIB_PATH)
             or os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(src), os.path.getmtime(hdr)))
    if force or stale:
        env = dict(os.environ)
        env.pop("CC", None)
        subprocess.run(["make", "-C", _HERE, "-B"], check=True, env=env, capture_output=True)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.orc_linear.argtypes = [u16p, u16p, u16p, C.c_int, C.c_int, C.c_int, C.c_int, u16p]
        L.orc_layernorm.argtypes = [f32p, u16p, f32p, f32p, C.c_float, C.c_int, C.c_int, f32p, u16p]
        L.orc_attention.argtypes = [u16p, u16p, u16p, i32p, C.c_int, C.c_int, C.c_long, u16p]
        L.orc_exp.argtypes = [C.c_float]
        L.orc_exp.restype = C.c_float
        L.orc_exp_n.argtypes = [f32p, C.c_int, f32p]
        L.orc_exp_n.restype = None
        L.orc_set_threads.argtypes = [C.c_int]
        L.orc_set_threads.restype = None
        L.orc_max_threads.restype = C.c_int
        L.orc_dec_create.argtypes = [C.c_int, C.c_int, C.c_int]
        L.orc_dec_create.restype = C.c_void_p
        L.orc_dec_set_layer.argtypes = [C.c_void_p, C.c_int] + [u16p] * 12 + [f32p] * 4
        L.orc_dec_set_globals.argtypes = [C.c_void_p, u16p, u16p, C.c_int, u16p, u16p, f32p, f32p, f32p, f32p, C.c_int]
        L.orc_dec_tok_table.argtypes = [C.c_void_p]
        L.orc_dec_tok_table.restype = u16p
        L.orc_dec_len.argtypes = [C.c_void_p]
        L.orc_dec_reset.argtypes = [C.c_void_p]
        L.orc_dec_destroy.argtypes = [C.c_void_p]
        L.orc_dec_prefill.argtypes = [C.c_void_p, f32p, C.c_int, u16p, f32p]
        L.orc_dec_step.argtypes = [C.c_void_p, C.c_int, C.c_int, u16p, f32p]
        L.orc_dec_get_kv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, u16p]
        _lib = L
    return _lib


def _h(t: torch.Tensor) -> np.ndarray:
    """fp32/fp16 tensor -> contiguous uint16 view of its fp16 (RNE) rounding, as autocast does."""
    return np.ascontiguousarray(t.detach().to(torch.float16).cpu().numpy()).view(np.uint16)


def _f(t: torch.Tensor) -> np.ndarray:
    return np.ascontiguousarray(t.detach().to(torch.float32).cpu().numpy())


def _p16(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(u16p)


def _p32(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(f32p)


# ---------------------------------------------------------------- unit-level canonical ops

def linear(w: torch.Tensor, b: Optional[torch.Tensor], x: torch.Tensor, relu: bool = False) -> torch.Tensor:
    """fp16(x @ w.T + b) in the canonical order. w [N,K], x [M,K] -> fp16 [M,N]."""
    W, X = _h(w), _h(x)
    B = _h(b) if b is not None else None
    M, K = X.shape
    N = W.shape[0]
    y = np.empty((M, N), dtype=np.uint16)
    lib().orc_linear(_p16(W), _p16(B), _p16(X), M, N, K, int(relu), _p16(y))
    return torch.from_numpy(y.view(np.float16).copy())


def layernorm(x: torch.Tensor, res16: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor,
              eps: float = 1e-5) -> Tuple[torch.Tensor, torch.Tensor]:
    X = _f(x)
    R = _h(res16) if res16 is not None else None
    M, W = X.shape
    y = np.empty((M, W), dtype=np.float32)
    y16 = np.empty((M, W), dtype=np.uint16)
    lib().orc_layernorm(_p32(X), _p16(R), _p32(_f(gamma)), _p32(_f(beta)), eps, M, W, _p32(y), _p16(y16))
    return torch.from_numpy(y), torch.from_numpy(y16.view(np.float16).copy())


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, nkeys: List[int]) -> torch.Tensor:
    """q [M,H,64]; k,v [H,T,64]; row m attends keys [0,nkeys[m]). -> fp16 [M,H,64]."""
    Q, K, V = _h(q), _h(k), _h(v)
    M, H, _ = Q.shape
    T = K.shape[1]
    nk = np.asarray(nkeys, dtype=np.int32)
    out = np.empty((M, H, 64), dtype=np.uint16)
    lib().orc_attention(_p16(Q), _p16(K), _p16(V), nk.ctypes.data_as(i32p), M, H, T, _p16(out))
    return torch.from_numpy(out.view(np.float16).copy())


def set_threads(n: int) -> None:
    """OpenMP team size of the oracle's loops (results do not depend on it: every reduction is within one thread)."""
    lib().orc_set_threads(int(n))


def max_threads() -> int:
    return int(lib().orc_max_threads())


# ---------------------------------------------------------------- the decoder

class OracleDecoder:
    """One sequence at a time (sequences of a batch are independent: SURVEY.md section 8e)."""

    def __init__(self, sd: Dict[str, torch.Tensor], n_layers: int, tmax: int, vocab: int = 8195):
        L = lib()
        self.L = L
        self.n_layers, self.tmax, self.vocab = n_layers, tmax, vocab
        self.h = L.orc_dec_create(n_layers, vocab, tmax)
        p = "transformer.model.decoder"
        for i in range(n_layers):
            q = f"{p}.layers.{i}"
            arrs = []
            for name in ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.out_proj", "fc1", "fc2"):
                arrs += [_h(sd[f"{q}.{name}.weight"]), _h(sd[f"{q}.{name}.bias"])]
            lns = [_f(sd[f"{q}.self_attn_layer_norm.weight"]), _f(sd[f"{q}.self_attn_layer_norm.bias"]),
                   _f(sd[f"{q}.final_layer_norm.weight"]), _f(sd[f"{q}.final_layer_norm.bias"])]
            L.orc_dec_set_layer(self.h, i, *[_p16(a) for a in arrs], *[_p32(a) for a in lns])
        cb = sd[f"{p}.quantize_codebooks"][0]
        pos = _f(sd[f"{p}.embed_positions.weight"])
        L.orc_dec_set_globals(
            self.h, _p16(_h(sd["transformer.lm_head.weight"])), _p16(_h(cb)), cb.shape[0],
            _p16(_h(sd[f"{p}.input_layer.weight"])), _p16(_h(sd[f"{p}.input_layer.bias"])),
            _p32(_f(sd[f"{p}.extra_embeds.weight"])), _p32(_f(sd[f"{p}.token_embed_positions.weight"])),
            _p32(_f(sd[f"{p}.cond_embed.weight"])), _p32(pos), pos.shape[0])
        self.codebook = cb.shape[0]

    def __del__(self):
        try:
            self.L.orc_dec_destroy(self.h)
        except Exception:
            pass

    def tok_table(self) -> torch.Tensor:
        ptr = self.L.orc_dec_tok_table(self.h)
        a = np.ctypeslib.as_array(ptr, shape=(self.codebook, 1024)).view(np.float16).copy()
        return torch.from_numpy(a)

    def reset(self):
        self.L.orc_dec_reset(self.h)

    def prefill(self, prefix: torch.Tensor, want_hidden: bool = False):
        """prefix fp32 [n,1024] -> fp16 logits [vocab] of the last row (and fp32 hidden [n,1024])."""
        P = _f(prefix)
        n = P.shape[0]
        logits = np.empty(self.vocab, dtype=np.uint16)
        hid = np.empty((n, 1024), dtype=np.float32) if want_hidden else None
        self.L.orc_dec_prefill(self.h, _p32(P), n, _p16(logits), _p32(hid))
        lg = torch.from_numpy(logits.view(np.float16).copy())
        return (lg, torch.from_numpy(hid)) if want_hidden else lg

    def step(self, tok: int, gen_count: int, want_hidden: bool = False):
        logits = np.empty(self.vocab, dtype=np.uint16)
        hid = np.empty(1024, dtype=np.float32) if want_hidden else None
        self.L.orc_dec_step(self.h, int(tok), int(gen_count), _p16(logits), _p32(hid))
        lg = torch.from_numpy(logits.view(np.float16).copy())
        return (lg, torch.from_numpy(hid)) if want_hidden else lg

    def get_kv(self, layer: int, kv: int, pos: int) -> torch.Tensor:
        out = np.empty(1024, dtype=np.uint16)
        self.L.orc_dec_get_kv(self.h, layer, kv, pos, _p16(out))
        return torch.from_numpy(out.view(np.float16).copy())

    def generate(self, prefix: torch.Tensor, max_new_tokens: int, eos_id: int = 1, pad_id: int = 2,
                 forced: Optional[List[int]] = None, keep_logits: bool = False,
                 pick: Optional[Callable[[torch.Tensor, int], int]] = None):
        """Greedy generate() for ONE sequence.  Returns (ids list, logits list).

        `forced`: teacher forcing -- feed these ids instead of the argmax (logits are still returned),
        used to compare logits along a sequence produced elsewhere.
        `pick(logits, step) -> id`: replaces the argmax, e.g. the sampler restatement of tests/sampler_oracle.py.
        """
        self.reset()
        ids: List[int] = []
        all_logits: List[torch.Tensor] = []
        logits = self.prefill(prefix)
        finished = False
        for i in range(max_new_tokens):
            if keep_logits:
                all_logits.append(logits)
            if pick is not None:
                nxt = int(pick(logits, i))
            else:
                nxt = greedy_pick(logits)   # lowest index among exact fp16 ties (float() is exact)
            if forced is not None:
                nxt = forced[i]
            if finished:
                nxt = pad_id
            ids.append(nxt)
            if nxt == eos_id:
                finished = True
            if finished and forced is None:
                break  # batch of one: HF stops when all rows are finished
            if i + 1 < max_new_tokens:
                logits = self.step(nxt, i + 1)
        return ids, all_logits


def greedy_pick(logits: torch.Tensor) -> int:
    lf = logits.float()
    return int((lf == lf.max()).nonzero()[0].item())
