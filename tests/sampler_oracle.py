"""Numpy restatement of `sample_kernel` (csrc/elementwise.cu), operation for operation -- TEST INFRASTRUCTURE ONLY.

DESIGN.md section 5 defines the pick.  Every fp32 operation below is a numpy float32 operation (correctly rounded, as
the kernel's __fadd_rn / __fmul_rn / __fdiv_rn are); `ma_exp` is the C oracle's own (`orc_exp_n`).  The draw is
Philox4x32-10 with counter (step, stream, 0x4d455348, 0x414e5954) and key (seed_lo, seed_hi).
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np

KEEP_MAX = 256           # capacity of the kernel's kept set
F32 = np.float32
_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key) -> np.ndarray:
    """Philox4x32-10 of Random123.  ctr: 4 uint32 arrays (or ints), key: 2 -> uint32 [4, n]."""
    c = [np.atleast_1d(np.asarray(x, dtype=np.uint64)) for x in ctr]
    k0, k1 = (np.atleast_1d(np.asarray(x, dtype=np.uint64)) for x in key)
    n = max(len(x) for x in c + [k0, k1])
    c = [np.broadcast_to(x, (n,)).copy() for x in c]
    k0, k1 = np.broadcast_to(k0, (n,)).copy(), np.broadcast_to(k1, (n,)).copy()
    for _ in range(10):
        p0, p1 = c[0] * np.uint64(_M0), c[2] * np.uint64(_M1)
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(_MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(_MASK)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + np.uint64(_W0)) & np.uint64(_MASK), (k1 + np.uint64(_W1)) & np.uint64(_MASK)
    return np.stack(c).astype(np.uint32)


def uniform(seed: int, stream, step) -> np.ndarray:
    """The kernel's r = (c0 >> 8) * 2^-24 in [0, 1), float32, for every (stream, step) pair given."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    out = philox4x32_10((step, stream, 0x4d455348, 0x414e5954), (seed & _MASK, seed >> 32))
    return (out[0] >> np.uint32(8)).astype(F32) * F32(1.0 / 16777216.0)


def key16(h: np.ndarray) -> np.ndarray:
    """Order-preserving 16-bit key of fp16 values; -0 takes +0's key."""
    u = np.ascontiguousarray(h, dtype=np.float16).view(np.uint16).astype(np.uint32)
    u = np.where(u == 0x8000, 0, u)
    return np.where(u & 0x8000, ~u & 0xFFFF, u | 0x8000)


def kept_set(row: np.ndarray, top_k: int) -> Tuple[np.ndarray, np.ndarray]:
    """Top-k stage: (ids, float32 values) sorted by descending value, ties by descending id; at most KEEP_MAX."""
    row = np.asarray(row, dtype=np.float16)
    k = min(int(top_k), row.size)
    keys = key16(row)
    kth = np.sort(keys)[::-1][k - 1]
    # compaction: key > kth in ascending id order, then key == kth in ascending id order, cut to KEEP_MAX
    ids = np.concatenate([np.nonzero(keys > kth)[0], np.nonzero(keys == kth)[0]])[:KEEP_MAX]
    vals = row[ids].astype(F32)
    order = np.lexsort((-ids, -vals))    # descending value (-0 == +0), then descending id
    return ids[order], vals[order]


def _exp(x: np.ndarray) -> np.ndarray:
    import ctypes as C
    from oracle.decoder import lib
    x = np.ascontiguousarray(x, dtype=F32)
    y = np.empty_like(x)
    lib().orc_exp_n(x.ctypes.data_as(C.POINTER(C.c_float)), x.size, y.ctypes.data_as(C.POINTER(C.c_float)))
    return y


def _seq_sum(a: np.ndarray) -> F32:
    s = F32(0.0)
    for v in a:
        s = F32(s + v)
    return s


def distribution(row: np.ndarray, top_k: int, top_p: float):
    """Top-k then top-p of one fp16 row: (kept ids, their fp32 probabilities, their running sums acc, ksum)."""
    ids, vals = kept_set(row, top_k)
    with np.errstate(invalid="ignore"):
        e = _exp(vals - vals[0])
    p = e / _seq_sum(e)                       # each divided by the fp32 sum taken in order
    keep, cum, thr = len(p), F32(0.0), F32(F32(1.0) - F32(top_p))
    for j in range(len(p) - 1, 0, -1):        # ascending probability; index 0 is always kept
        cum = F32(cum + p[j])
        if cum <= thr:
            keep = j
        else:
            break
    p = p[:keep]
    acc = np.empty(keep, dtype=F32)
    s = F32(0.0)
    for j in range(keep):
        s = F32(s + p[j])
        acc[j] = s
    return ids[:keep], p, acc, s               # ksum == acc[-1]: the same sum in the same order


def sample_row(row: np.ndarray, top_k: int, top_p: float, seed: int, stream: int, step: int) -> Tuple[int, np.ndarray]:
    """One sampled pick: (token, kept ids after top-k / top-p)."""
    ids, _, acc, ksum = distribution(row, top_k, top_p)
    u = F32(uniform(seed, stream, step)[0] * ksum)
    hit = np.nonzero(u < acc)[0]
    return int(ids[hit[0]] if len(hit) else ids[-1]), ids


def greedy_row(row: np.ndarray) -> int:
    """Lowest index of the maximum."""
    v = np.asarray(row, dtype=np.float16).astype(F32)
    return int(np.nonzero(v == v.max())[0][0])


def pick(row, seed: int, stream: int, step: int, do_sample: bool = True, top_k: int = 50, top_p: float = 0.95) -> int:
    """The token `sample_kernel` picks from fp16 logits `row` (numpy or torch) for (seed, stream, step)."""
    row = _np16(row)
    if not do_sample:
        return greedy_row(row)
    return sample_row(row, top_k, top_p, seed, stream, step)[0]


def sample_tokens(logits, top_k: int, top_p: float, seed: int) -> Tuple[np.ndarray, np.ndarray]:
    """What `ma_sample_tokens` returns for [B, vocab] fp16 logits: tokens [B] and the kept set [B, 256] (-1 padded);
    row b draws from stream b at step 0."""
    lg = _np16(logits)
    B = lg.shape[0]
    tok = np.empty(B, dtype=np.int32)
    sup = np.full((B, KEEP_MAX), -1, dtype=np.int32)
    for b in range(B):
        t, ids = sample_row(lg[b], top_k, top_p, seed, b, 0)
        tok[b] = t
        sup[b, :len(ids)] = ids
    return tok, sup


def draw_law(row: np.ndarray, top_k: int, top_p: float) -> Tuple[np.ndarray, np.ndarray]:
    """Exact probability of every kept token under the kernel's draw: u(m) = fl32(m 2^-24 ksum) is monotone in the
    2^24 grid values m, so counting the m that land on each token is exact.  Returns (kept ids, probabilities)."""
    ids, _, acc, ksum = distribution(row, top_k, top_p)
    u = np.arange(1 << 24, dtype=np.uint32).astype(F32) * F32(1.0 / 16777216.0) * ksum
    j = np.minimum(np.searchsorted(acc, u, side="right"), len(ids) - 1)   # first j with u < acc_j, else the last
    return ids, np.bincount(j, minlength=len(ids)) / float(1 << 24)


def generate_pick(seed: int, stream: int, do_sample: bool = True, top_k: int = 50, top_p: float = 0.95):
    """`pick` argument of OracleDecoder.generate: the sampler for one sequence's Philox stream."""
    return lambda logits, step: pick(logits, seed, stream, step, do_sample, top_k, top_p)


def _np16(x) -> np.ndarray:
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    return np.asarray(x, dtype=np.float16)


def oracle_generate(oracle, prefix, max_new: int, seed: int, stream: int = 0, top_k: int = 50, top_p: float = 0.95,
                    eos_id: int = 1, pad_id: int = 2, keep_logits: bool = False,
                    forced: Optional[List[int]] = None):
    """Sampled generate() of one sequence on the C oracle's decoder (OracleDecoder.generate with the sampler)."""
    return oracle.generate(prefix, max_new, eos_id=eos_id, pad_id=pad_id, forced=forced, keep_logits=keep_logits,
                           pick=generate_pick(seed, stream, True, top_k, top_p))
