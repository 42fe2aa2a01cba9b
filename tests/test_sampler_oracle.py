"""The sampler restatement (tests/sampler_oracle.py) on the CPU: Philox against Random123's known answers, the order
keys, the kept set against transformers' TopKLogitsWarper -> TopPLogitsWarper, the exact law of the draw against the
float64 renormalised softmax, and the oracle decoder driven by a picker."""
import numpy as np
import pytest
import torch

from tests import sampler_oracle as S


def _row(seed, scale, V=8195):
    return (np.random.default_rng(seed).standard_normal(V) * scale).astype(np.float16)


def _hf_support(row16, top_k, top_p, dtype=torch.float32):
    """ids kept by transformers' own warpers (the chain HF _sample builds for meshanything.py:150-158)."""
    from transformers.generation.logits_process import TopKLogitsWarper, TopPLogitsWarper
    s = torch.from_numpy(row16).to(dtype)[None]
    s = TopKLogitsWarper(top_k)(None, s)
    if top_p < 1.0:          # generation/utils.py adds the top-p warper only below 1.0
        s = TopPLogitsWarper(top_p)(None, s)
    return np.nonzero(np.isfinite(s[0].float().numpy()))[0]


def _near_top_p_edge(row16, top_k, top_p):
    """Does the ascending cumulative probability (fp64) pass within 1e-5 of 1 - top_p?"""
    ids, vals = S.kept_set(row16, top_k)
    p = np.exp(vals.astype(np.float64) - float(vals[0]))
    cum = np.cumsum((p / p.sum())[::-1])
    return top_p < 1.0 and bool((np.abs(cum - (1 - top_p)) < 1e-5).any())


# ---------------------------------------------------------------- Philox and the order keys

@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    """Random123's kat_vectors for philox4x32 with 10 rounds."""
    assert S.philox4x32_10(ctr, key)[:, 0].tolist() == list(want)


def test_uniform_is_the_top_24_bits_of_word_0():
    seed = (0x12345678 << 32) | 0x9abcdef0
    steps, streams = np.arange(50), np.arange(50)[::-1]
    c0 = S.philox4x32_10((steps, streams, 0x4d455348, 0x414e5954), (0x9abcdef0, 0x12345678))[0]
    r = S.uniform(seed, streams, steps)
    assert r.dtype == np.float32 and np.array_equal(r.astype(np.float64), (c0 >> 8) / 2.0 ** 24)
    assert not np.array_equal(r, S.uniform(seed, steps, streams))             # (step, stream) is ordered
    assert not np.array_equal(r, S.uniform(seed & 0xffffffff, streams, steps))  # the high seed word counts


def test_key16_orders_every_fp16_value():
    """larger value <=> larger key; equal values (only +0 and -0 among the non-NaN) <=> equal keys."""
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
    h = h[~np.isnan(h)]
    k = S.key16(h)
    v = h.astype(np.float64)
    o = np.argsort(v, kind="stable")
    assert (np.diff(k[o].astype(np.int64)) >= 0).all()
    assert np.array_equal(np.diff(k[o].astype(np.int64)) == 0, np.diff(v[o]) == 0)
    assert S.key16(np.array([-0.0], np.float16))[0] == S.key16(np.array([0.0], np.float16))[0]


# ---------------------------------------------------------------- the kept set against HF

def _crafted_rows():
    V = 8195
    rows = {f"normal_{s}": _row(10 + i, s) for i, s in enumerate((0.5, 1.6, 6.0, 30.0))}
    rows["integers"] = np.round(np.random.default_rng(3).standard_normal(V) * 2).astype(np.float16)
    for n in (255, 256):
        r = np.full(V, -3.0, np.float16)
        r[np.random.default_rng(n).choice(V, n, replace=False)] = 2.5
        rows[f"ties_{n}"] = r
    z = np.full(V, -1.0, np.float16)                         # the k-th largest (k = 50) is +0, and -0 ties with it
    z[100:145] = np.linspace(0.5, 3.0, 45).astype(np.float16)
    z[[7, 300, 301, 5000, 8000]] = 0.0
    z[[9, 4000]] = -0.0
    rows["signed_zeros"] = z
    f = _row(4, 2.0)
    f[np.random.default_rng(5).random(V) < 0.5] = -np.inf
    rows["minus_inf"] = f
    return rows


@pytest.mark.parametrize("top_k", [1, 2, 50, 128])
@pytest.mark.parametrize("top_p", [0.5, 0.9, 0.95, 1.0])
def test_kept_set_matches_hf_warpers_fp32(top_k, top_p):
    for name, row in _crafted_rows().items():
        got = S.distribution(row, top_k, top_p)[0]
        want = _hf_support(row, top_k, top_p)
        after_k = _hf_support(row, top_k, 1.0)
        if len(after_k) > S.KEEP_MAX:                  # the kernel's capacity rule (next tests): 256 of HF's ids
            kth = np.sort(row.astype(np.float32))[::-1][top_k - 1]
            gt, eq = np.nonzero(row > kth)[0], np.nonzero(row == kth)[0]
            rule = set(gt) | set(eq[:S.KEEP_MAX - len(gt)])
            assert set(S.kept_set(row, top_k)[0]) == rule and rule <= set(after_k), name
            assert set(got) <= rule, name
            continue
        # which of several EQUAL logits the cut keeps is undefined in HF (unstable torch.sort): compare values
        gv, wv = sorted(row[got].astype(np.float32))[::-1], sorted(row[want].astype(np.float32))[::-1]
        if _near_top_p_edge(row, top_k, top_p):       # summation order may move one boundary token
            short, long_ = sorted((gv, wv), key=len)
            assert len(long_) - len(short) <= 1 and long_[:len(short)] == short, name
            continue
        assert gv == wv, (name, len(got), len(want))     # the same values kept
        if len(set(row[want]) & set(row[np.setdiff1d(np.arange(row.size), want)])) == 0:
            assert set(got) == set(want), name           # no value is split by the cut: the same ids


def test_signed_zeros_at_the_threshold_are_all_kept():
    """The k-th largest logit is +0 and two -0 logits tie with it: `scores < kth` keeps all 52, in fp32 and fp16."""
    row = _crafted_rows()["signed_zeros"]
    got = S.distribution(row, 50, 1.0)[0]
    assert len(got) == 52 and {9, 4000} <= set(got.tolist())
    assert set(got) == set(_hf_support(row, 50, 1.0)) == set(_hf_support(row, 50, 1.0, torch.float16))


@pytest.mark.parametrize("n_gt,n_eq", [(0, 300), (10, 300), (0, 8195)])
def test_more_ties_than_the_kept_set_keep_the_lowest_ids(n_gt, n_eq):
    """The kernel's rule where it departs from HF: with more than 256 logits at or above the threshold, the kept set
    is every id above the threshold, then the ties at the threshold in ascending id order, cut to 256.  HF keeps every
    tie; the ids the kernel drops are exactly the highest tied ids."""
    V = 8195
    rng = np.random.default_rng(n_gt + n_eq)
    row = np.full(V, -3.0, np.float16)
    eq = np.sort(rng.choice(V, n_eq, replace=False))
    row[eq] = 2.5
    gt = np.sort(rng.choice(np.setdiff1d(np.arange(V), eq), n_gt, replace=False)) if n_gt else np.zeros(0, np.int64)
    row[gt] = 4.0
    ids, vals = S.kept_set(row, 50)
    assert len(ids) == S.KEEP_MAX
    assert np.array_equal(ids[:n_gt], gt[::-1]) and np.array_equal(ids[n_gt:], eq[:S.KEEP_MAX - n_gt][::-1])
    hf = _hf_support(row, 50, 1.0)
    assert len(hf) == n_gt + n_eq and set(ids) <= set(hf)
    assert np.array_equal(np.setdiff1d(hf, ids), eq[S.KEEP_MAX - n_gt:])
    assert np.array_equal(S.distribution(row, 50, 1.0)[0], ids)       # equal probabilities: no top-p cut at 1.0


def test_vocab_smaller_than_top_k_keeps_the_whole_row():
    row = _row(8, 1.0, V=40)
    ids, p, acc, ksum = S.distribution(row, 50, 1.0)
    assert sorted(ids.tolist()) == list(range(40)) and ksum == acc[-1]


# ---------------------------------------------------------------- the law of the draw

@pytest.mark.parametrize("scale", [0.5, 1.6, 6.0])
@pytest.mark.parametrize("top_k,top_p", [(50, 0.95), (128, 0.5), (2, 1.0), (50, 1.0)])
def test_draw_law_is_the_renormalised_softmax(scale, top_k, top_p):
    """Exact probability of every kept token (all 2^24 uniforms counted) against the fp64 softmax over the kept set:
    the fp32 exponentials and sums and the 2^-24 grid move each probability by less than 1e-6."""
    row = _row(int(scale * 10) + top_k, scale)
    ids, law = S.draw_law(row, top_k, top_p)
    v = row[ids].astype(np.float64)
    p = np.exp(v - v.max())
    p /= p.sum()
    assert abs(law.sum() - 1.0) < 1e-12
    err = np.abs(law - p).max()
    assert err < 1e-6, err


def test_draws_follow_the_law():
    """1000 streams of one row: the sampler's picks stay inside the kept set and their counts follow the law (5 sigma)."""
    row = _row(77, 1.6)
    ids, law = S.draw_law(row, 50, 0.95)
    toks = [S.sample_row(row, 50, 0.95, 5, b, 3)[0] for b in range(1000)]
    assert set(toks) <= set(ids.tolist())
    counts = np.array([toks.count(i) for i in ids]) / 1000.0
    assert (np.abs(counts - law) < 5 * np.sqrt(law * (1 - law) / 1000) + 1e-3).all()


def test_greedy_is_the_lowest_index_of_the_maximum():
    row = np.zeros(100, np.float16)
    row[[3, 50, 99]] = 2.0
    assert S.greedy_row(row) == 3 and S.pick(row, 0, 0, 0, do_sample=False) == 3


# ---------------------------------------------------------------- the oracle decoder with a picker

def test_oracle_generate_with_a_picker():
    """pick=None is the greedy argmax; a sampled picker draws step by step from the same logits; eos stops a batch of
    one; forced ids still override the picker."""
    from oracle.decoder import OracleDecoder, greedy_pick
    from tests.util import decoder_sd, random_prefix
    n = 12
    oracle = OracleDecoder(decoder_sd(1), 1, 257 + n)
    prefix = random_prefix(1, seed=2)[0]
    greedy, lg = oracle.generate(prefix, n, eos_id=-1, keep_logits=True)
    assert oracle.generate(prefix, n, eos_id=-1, pick=lambda logits, step: greedy_pick(logits))[0] == greedy
    ids, lgs = S.oracle_generate(oracle, prefix, n, seed=9, stream=4, eos_id=-1, keep_logits=True)
    assert ids == [S.pick(lgs[i], 9, 4, i) for i in range(n)] and ids != greedy
    eos = ids[5]
    first = ids.index(eos)
    short, _ = S.oracle_generate(oracle, prefix, n, seed=9, stream=4, eos_id=eos)
    assert short == ids[:first + 1]
    forced = list(range(3, 3 + n))
    assert S.oracle_generate(oracle, prefix, n, seed=9, stream=4, eos_id=-1, forced=forced)[0] == forced
