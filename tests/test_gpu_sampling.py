"""-m gpu: sampled decoding token for token against the sampler restatement (tests/sampler_oracle.py).

At batch 1 (and in a single cache slot) sampling runs on the canonical CUDA-core kernels, so the C oracle's logits
followed by the restated sampler predict every sampled id bit for bit.  On the tensor-core batched path the logits are
not the oracle's, but the pick is a deterministic function of (the fp16 logits it read, seed, stream, step), and
`want_logits` returns those logits: every (row, step) is still checked exactly.
"""
import argparse

import numpy as np
import pytest
import torch

from tests import sampler_oracle as S
from tests.util import decoder_sd, random_prefix

gpu = pytest.mark.gpu
NL = 3
LONG = 600       # 257 + 600 keys: the context crosses three 256-key attention chunks
PAD = 2


def _dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def small():
    from meshanything_b200.decoder import DecoderArena
    from oracle.decoder import OracleDecoder
    sd = decoder_sd(NL)
    return sd, DecoderArena(sd, _dev()), OracleDecoder(sd, NL, 257 + LONG)


@pytest.fixture(scope="module")
def long_run(small):
    """The oracle's 600-token sampled sequence (seed 2^32 + 5, stream 0) and its logits."""
    _, _, oracle = small
    prefix = random_prefix(1, seed=13)
    ids, logits = S.oracle_generate(oracle, prefix[0], LONG, seed=(1 << 32) + 5, eos_id=-1, keep_logits=True)
    return prefix, ids, logits


def _check_sampled_row(ids, lens, logits, b, seed, top_k, top_p, eos):
    """Row b of a batched sampled generate: every id before eos is the restated pick from the returned logits (stream
    b), pad after it, and lens counts up to and including eos."""
    ids, n = ids[b].tolist(), len(ids[b])
    end = n
    for i in range(n):
        assert ids[i] == S.pick(logits[i, b], seed, b, i, True, top_k, top_p), (b, i)
        if ids[i] == eos:
            end = i + 1
            break
    assert all(t == PAD for t in ids[end:]), b
    assert int(lens[b]) == end, (b, int(lens[b]), end)
    return end


# ---------------------------------------------------------------- A: ma_sample_tokens on crafted rows

def _signed_zero_row(V):
    """+0 is the 50th largest value and two -0 tie with it."""
    z = np.full(V, -1.0, np.float16)
    z[100:145] = np.linspace(0.5, 3.0, 45).astype(np.float16)
    z[[7, 300, 301, 500, 800]] = 0.0
    z[[9, 400]] = -0.0
    return z


def _rows(V, n_random=6):
    g = np.random.default_rng(V)
    rows = [(g.standard_normal(V) * s).astype(np.float16) for s in (0.5, 1.6, 6.0, 30.0)]
    rows += [(g.standard_normal(V) * 1.6).astype(np.float16) for _ in range(n_random)]
    rows.append(np.round(g.standard_normal(V) * 2).astype(np.float16))            # integer ties
    for n in (255, 256, 300):                                                     # n ties at the threshold
        r = np.full(V, -3.0, np.float16)
        r[g.choice(V, min(n, V), replace=False)] = 2.5
        rows.append(r)
    r = np.full(V, -3.0, np.float16)                                              # 10 above, 300 tied
    r[g.choice(V, min(310, V), replace=False)] = 2.5
    r[g.choice(V, 10, replace=False)] = 4.0
    rows.append(r)
    if V >= 1000:
        rows.append(_signed_zero_row(V))
    f = (g.standard_normal(V) * 2).astype(np.float16)                          # -inf entries
    f[g.random(V) < 0.5] = -np.inf
    rows.append(f)
    f = np.full(V, -np.inf, np.float16)                                           # only 20 finite: -inf ties kept
    f[g.choice(V, 20, replace=False)] = (g.standard_normal(20) * 2).astype(np.float16)
    rows.append(f)
    rows.append(np.zeros(V, np.float16))                                          # all equal
    rows.append(np.full(V, 1.5, np.float16))
    return np.stack(rows)


def _sample_and_compare(lg, top_k, top_p, seed):
    from meshanything_b200 import capi
    tok, sup = capi.sample_tokens(torch.from_numpy(lg).to(_dev()), True, top_k, top_p, seed=seed, want_support=True)
    want_tok, want_sup = S.sample_tokens(lg, top_k, top_p, seed)
    tok, sup = tok.cpu().numpy(), sup.cpu().numpy()
    bad = np.nonzero((tok != want_tok) | (sup != want_sup).any(1))[0]
    assert len(bad) == 0, f"rows {bad.tolist()} differ (of {len(lg)})"


@gpu
@pytest.mark.parametrize("top_k", [1, 2, 50, 128])
@pytest.mark.parametrize("top_p", [0.5, 0.9, 0.95, 1.0])
@pytest.mark.parametrize("seed", [3, (7 << 32) | 3])
def test_sample_tokens_bit_exact(top_k, top_p, seed):
    _sample_and_compare(_rows(8195), top_k, top_p, seed)


@gpu
def test_sample_tokens_signed_zero_threshold_keeps_every_zero():
    """+0 is the 50th largest logit and two -0 tie with it: all 52 are kept, as TopKLogitsWarper keeps them."""
    from meshanything_b200 import capi
    z = _signed_zero_row(8195)
    _, sup = capi.sample_tokens(torch.from_numpy(z[None].copy()).to(_dev()), True, 50, 1.0, seed=1, want_support=True)
    kept = [int(v) for v in sup[0].cpu() if v >= 0]
    assert len(kept) == 52 and {9, 400} <= set(kept)
    _sample_and_compare(z[None].copy(), 50, 1.0, 1)


@gpu
@pytest.mark.parametrize("V", [1000, 40, 16384])
def test_sample_tokens_vocab_sizes(V):
    """vocab 1000, a vocab smaller than top_k, and the largest vocab whose keys fit in shared memory."""
    lg = _rows(V)
    for top_k, top_p in ((50, 0.95), (128, 1.0), (2, 0.5)):
        _sample_and_compare(lg, top_k, top_p, 11)


@gpu
def test_sample_tokens_1000_rows():
    g = np.random.default_rng(5)
    lg = (g.standard_normal((1000, 8195)) * g.uniform(0.5, 6.0, (1000, 1))).astype(np.float16)
    _sample_and_compare(lg, 50, 0.95, (1 << 40) + 17)


@gpu
def test_sample_tokens_argument_errors():
    from meshanything_b200 import capi
    lg = torch.zeros((2, 8195), dtype=torch.float16, device=_dev())
    with pytest.raises(RuntimeError, match="top_k"):
        capi.sample_tokens(lg, True, 129, 0.95)
    with pytest.raises(RuntimeError, match="vocab"):
        capi.sample_tokens(torch.zeros((2, 16385), dtype=torch.float16, device=_dev()), True, 50, 0.95)


# ---------------------------------------------------------------- B: batch-1 sampled generate, every kernel variant

@gpu
@pytest.mark.parametrize("flags", [0, 4, 1, 2, 2 | 1])
def test_batch1_sampled_generate_bit_exact(small, long_run, flags):
    """600 sampled tokens at batch 1: ids and every step's fp16 logits equal the oracle's.  flags: 0 per-phase kernels
    with PDL and CUDA graphs, 4 without PDL, 1 without graphs, 2 the general batched kernels (canonical at B = 1)."""
    from meshanything_b200.decoder import Generator
    _, arena, _ = small
    prefix, ref_ids, ref_logits = long_run
    gen = Generator(arena, 1, 257 + LONG)
    ids, lens, logits = gen.generate(prefix.to(_dev()), LONG, do_sample=True, seed=(1 << 32) + 5, eos_id=-1,
                                     want_logits=True, flags=flags)
    got = ids[0].cpu().tolist()
    first = next((i for i, (a, b) in enumerate(zip(got, ref_ids)) if a != b), None)
    assert first is None, f"flags={flags}: first different id at step {first}"
    lg = logits[:, 0].cpu()
    for i, rl in enumerate(ref_logits):
        assert torch.equal(lg[i].view(torch.int16), rl.view(torch.int16)), f"flags={flags}: logits differ at step {i}"
    assert int(lens[0]) == LONG


@gpu
def test_batch1_sampled_generate_stops_at_eos(small, long_run):
    """eos re-declared as a token the sampled sequence emits: the ids stop there, pad after, lens = its step + 1."""
    from meshanything_b200.decoder import Generator
    _, arena, oracle = small
    prefix, free, _ = long_run
    eos = free[100]
    ref, _ = S.oracle_generate(oracle, prefix[0], LONG, seed=(1 << 32) + 5, eos_id=eos)
    assert ref == free[:free.index(eos) + 1]
    for flags in (0, 2):
        ids, lens = Generator(arena, 1, 257 + LONG).generate(prefix.to(_dev()), LONG, do_sample=True,
                                                              seed=(1 << 32) + 5, eos_id=eos, flags=flags)
        got = ids[0].cpu().tolist()
        assert got[:len(ref)] == ref and all(t == PAD for t in got[len(ref):]), flags
        assert int(lens[0]) == len(ref), flags


@gpu
@pytest.mark.slow
def test_batch1_sampled_generate_full_depth():
    """24 layers, F = 64 (578 sampled tokens) at batch 1: ids equal the oracle's."""
    from meshanything_b200.decoder import DecoderArena, Generator
    from oracle.decoder import OracleDecoder
    sd = decoder_sd(24)
    n = 64 * 9 + 2
    prefix = random_prefix(1, seed=1)
    ids, _ = Generator(DecoderArena(sd, _dev()), 1, 257 + n).generate(prefix.to(_dev()), n, do_sample=True, seed=21,
                                                                      eos_id=-1)
    ref, _ = S.oracle_generate(OracleDecoder(sd, 24, 257 + n), prefix[0], n, seed=21, eos_id=-1)
    assert ids[0].cpu().tolist() == ref


# ---------------------------------------------------------------- C: tensor-core batches

@gpu
@pytest.mark.parametrize("B", [2, 17, 64])
def test_tensor_core_sampled_batches_pick_exactly(small, B):
    """Every (row, step) id is the restated pick from the logits the kernel read (stream = row), or pad after the row's
    eos; lens match.  eos is re-declared so that rows finish at different steps."""
    from meshanything_b200.decoder import Generator
    _, arena, _ = small
    n = 40
    prefix = random_prefix(B, seed=40 + B).to(_dev())
    gen = Generator(arena, B, 257 + n)
    free, _ = gen.generate(prefix, n, do_sample=True, seed=9, eos_id=-1)
    free = free.cpu()
    firsts = {}
    for t in free[0, 5:30].tolist():        # a token of row 0 that first shows up at different steps across rows
        pos = [(free[b] == t).nonzero()[0, 0].item() if (free[b] == t).any() else n for b in range(B)]
        firsts[t] = len(set(pos))
    eos = max(firsts, key=firsts.get)
    ids, lens, logits = gen.generate(prefix, n, do_sample=True, seed=9, eos_id=eos, want_logits=True)
    ids, lens, logits = ids.cpu(), lens.cpu(), logits.cpu()
    ends = [_check_sampled_row(ids, lens, logits, b, 9, 50, 0.95, eos) for b in range(B)]
    assert B == 2 or len(set(ends)) >= 2, ends


# ---------------------------------------------------------------- D: the per-step graph cache

_CALLS = [dict(seed=5), dict(seed=6), dict(seed=6 + (1 << 32)), dict(seed=6 + (1 << 32), top_p=0.5),
          dict(seed=6 + (1 << 32), top_p=0.5, top_k=7), dict(seed=6 + (1 << 32), top_p=0.5, top_k=7, eos_id=None)]


def _settings(c, eos):
    s = dict(seed=c["seed"], top_k=c.get("top_k", 50), top_p=c.get("top_p", 0.95), eos_id=-1)
    if "eos_id" in c:
        s["eos_id"] = eos
    return s


@gpu
def test_graph_cache_batch1_follows_every_sampling_argument(small):
    """One Generator, calls that change only the seed (then only its high 32 bits), only top_p, only top_k, only eos:
    each call's ids are its own oracle prediction, never a replay of a graph captured for another call."""
    from meshanything_b200.decoder import Generator
    _, arena, oracle = small
    n = 24
    prefix = random_prefix(1, seed=50)
    gen = Generator(arena, 1, 257 + n)
    eos = None
    for c in _CALLS:
        if eos is None and "eos_id" in c:
            eos = prev[8]
        s = _settings(c, eos)
        ref, _ = S.oracle_generate(oracle, prefix[0], n, seed=s["seed"], top_k=s["top_k"], top_p=s["top_p"],
                                   eos_id=s["eos_id"])
        ids, lens = gen.generate(prefix.to(_dev()), n, do_sample=True, **s)
        got = ids[0].cpu().tolist()
        assert got[:len(ref)] == ref and all(t == PAD for t in got[len(ref):]), c
        assert int(lens[0]) == len(ref), c
        prev = ref


@gpu
def test_graph_cache_batch17_follows_every_sampling_argument(small):
    """The same at B = 17 (tensor-core graphs): each graph replay gives the ids of an eager run of the same call, and
    the eager run's ids are the restated picks from its logits."""
    from meshanything_b200 import capi
    from meshanything_b200.decoder import Generator
    _, arena, _ = small
    B, n = 17, 24
    prefix = random_prefix(B, seed=51).to(_dev())
    gen = Generator(arena, B, 257 + n)
    eager = Generator(arena, B, 257 + n)
    eos, prev = None, None
    for c in _CALLS:
        if eos is None and "eos_id" in c:
            eos = int(prev[0, 8])
        s = _settings(c, eos)
        ids, lens = gen.generate(prefix, n, do_sample=True, **s)
        ref, ref_lens, logits = eager.generate(prefix, n, do_sample=True, want_logits=True,
                                               flags=capi.GEN_NO_GRAPH, **s)
        ref, ref_lens, logits = ref.cpu(), ref_lens.cpu(), logits.cpu()
        for b in range(B):
            _check_sampled_row(ref, ref_lens, logits, b, s["seed"], s["top_k"], s["top_p"], s["eos_id"])
        assert torch.equal(ids.cpu(), ref) and torch.equal(lens.cpu(), ref_lens), c
        prev = ref


# ---------------------------------------------------------------- E: one cache slot, sampling

@gpu
def test_single_slot_sampling_streams_are_queue_indices(small):
    """A queue of 3 prefixes (the first repeated last) through ONE slot with sampling and a re-declared eos: sequence
    k equals the oracle's sampled sequence from Philox stream k."""
    from meshanything_b200.scheduler import SlotEngine, SlotScheduler
    _, arena, oracle = small
    n = 40
    p = random_prefix(2, seed=60)
    queue = [p[0], p[1], p[0]]
    free = [S.oracle_generate(oracle, q, n, seed=11, stream=k, eos_id=-1)[0] for k, q in enumerate(queue)]
    eos = free[0][12]
    refs = [S.oracle_generate(oracle, q, n, seed=11, stream=k, eos_id=eos)[0] for k, q in enumerate(queue)]
    assert len(refs[0]) == free[0].index(eos) + 1
    eng = SlotEngine(arena, 1, 257 + n, n, do_sample=True, seed=11, eos_id=eos)
    got = {k: ids.cpu().tolist() for k, ids in SlotScheduler(eng, 1, n, poll_every=7).run([q.to(_dev()) for q in queue])}
    for k in range(3):
        assert got[k] == refs[k], (k, len(got[k]), len(refs[k]))


# ---------------------------------------------------------------- F: MeshAnything.forward(sampling=True)

@gpu
def test_forward_sampling_draws_from_seed_plus_call_index(small, monkeypatch):
    """Two sampled forward calls of one shape: the ids are the oracle's from the recorded prefix with seeds
    args.seed + 0 and args.seed + 1 (stream 0)."""
    from MeshAnything.models.meshanything import MeshAnything
    from meshanything_b200 import checkpoint as ck
    from meshanything_b200.decoder import Generator
    from meshanything_b200.inputs import synthetic_pc_normal
    _, _, oracle = small
    F = 8
    args = argparse.Namespace(llm="facebook/opt-350m", codebook_size=8192, codebook_dim=1024, n_max_triangles=F,
                              seed=123)
    model = MeshAnything(args)
    model.load_state_dict(ck.synthetic_state_dict(0, n_dec_layers=NL), strict=False, device=_dev())
    seen = []
    real = Generator.generate

    def record(self, prefix, *a, **kw):
        out = real(self, prefix, *a, **kw)
        seen.append((prefix.cpu().clone(), out[0].cpu().clone(), kw))
        return out

    monkeypatch.setattr(Generator, "generate", record)
    pc = synthetic_pc_normal(2, first=3)
    for _ in range(2):
        model(pc[:1], sampling=True)
    assert len(seen) == 2
    n = F * 9 + 2
    for call, (prefix, ids, kw) in enumerate(seen):
        assert kw["seed"] == 123 + call
        ref, _ = S.oracle_generate(oracle, prefix[0], n, seed=123 + call, eos_id=1, pad_id=PAD)
        got = ids[0].tolist()
        assert got[:len(ref)] == ref and all(t == PAD for t in got[len(ref):]), call
    assert seen[0][1].tolist() != seen[1][1].tolist()


# ---------------------------------------------------------------- G: HF's warpers on CUDA fp16 scores

@gpu
def test_hf_warpers_on_fp16_scores_differ_by_at_most_one_boundary_token():
    """HF's TopK -> TopP run on CUDA fp16 scores, the dtype the reference's autocast lm_head gives.  Its softmax and
    cumulative sum round to fp16, the sampler's to fp32: where they disagree, the two kept sets differ by one token at
    the top-p boundary.  Prints the share of such rows."""
    from transformers.generation.logits_process import TopKLogitsWarper, TopPLogitsWarper
    g = np.random.default_rng(8)
    total, differ = 0, 0
    for scale in (0.5, 1.6, 6.0, 30.0):
        lg = (g.standard_normal((375, 8195)) * scale).astype(np.float16)
        s = torch.from_numpy(lg).to(_dev())
        s = TopPLogitsWarper(0.95)(None, TopKLogitsWarper(50)(None, s))
        keep = torch.isfinite(s).cpu().numpy()
        n_scale = 0
        for r in range(len(lg)):
            mine = S.distribution(lg[r], 50, 0.95)[0]
            theirs = np.nonzero(keep[r])[0]
            a = sorted(lg[r, mine].astype(np.float32))[::-1]     # equal logits are interchangeable in HF's sort
            b = sorted(lg[r, theirs].astype(np.float32))[::-1]
            if a != b:
                short, long_ = sorted((a, b), key=len)
                assert len(long_) == len(short) + 1 and long_[:len(short)] == short, (scale, r, len(a), len(b))
                n_scale += 1
        print(f"scale {scale}: {n_scale} of {len(lg)} rows keep a different set under HF fp16")
        total += len(lg)
        differ += n_scale
    print(f"HF fp16 warpers vs the sampler: {differ} of {total} rows ({100.0 * differ / total:.2f} %) differ by one "
          f"boundary token")
