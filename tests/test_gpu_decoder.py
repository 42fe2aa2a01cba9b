"""-m gpu: ShapeOPT decoder generate() on the GPU against the CPU oracle (bit-exact ids AND fp16 logits)."""
import pytest
import torch

from tests.util import decoder_sd, random_prefix

gpu = pytest.mark.gpu
NL = 3          # layers of the small synthetic decoder used by most cases
NEW = 40        # new tokens of the short cases


def _dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def small():
    from meshanything_b200.decoder import DecoderArena
    from oracle.decoder import OracleDecoder
    sd = decoder_sd(NL)
    arena = DecoderArena(sd, _dev())
    oracle = OracleDecoder(sd, NL, 257 + 600)
    return sd, arena, oracle


@gpu
def test_tok_table_matches_oracle(small):
    _, arena, oracle = small
    assert torch.equal(arena.tok_table.cpu().view(torch.int16), oracle.tok_table().view(torch.int16))


@gpu
@pytest.mark.parametrize("flags", [0, 16, 4, 1, 2, 2 | 1])
def test_greedy_bit_exact_vs_oracle(small, flags):
    """free-running greedy decode: token ids and every step's fp16 logits equal the oracle's.
    flags: 0 per-phase kernels + PDL, 16 the same (MA_GEN_NO_MEGA is accepted and ignored), 4 without PDL, |1 without
    CUDA graph, 2 batched kernels."""
    from meshanything_b200.decoder import Generator
    _, arena, oracle = small
    prefix = random_prefix(1, seed=3)
    gen = Generator(arena, 1, 257 + NEW)
    ids, lens, logits = gen.generate(prefix.to(_dev()), NEW, want_logits=True, flags=flags)
    torch.cuda.synchronize()
    ref_ids, ref_logits = oracle.generate(prefix[0], NEW, keep_logits=True)
    assert ids[0].cpu().tolist() == ref_ids
    for i, rl in enumerate(ref_logits):
        assert torch.equal(logits[i, 0].cpu().view(torch.int16), rl.view(torch.int16)), f"logits differ at step {i}"
    assert int(lens[0]) == NEW


@gpu
def test_batch_invariance_and_batched_parity(small):
    """a batch of 5 gives, row by row, what each sequence gives alone (and what the oracle gives)."""
    from meshanything_b200.decoder import Generator
    _, arena, oracle = small
    B = 5
    prefix = random_prefix(B, seed=11)
    gen = Generator(arena, B, 257 + NEW)
    ids, lens = gen.generate(prefix.to(_dev()), NEW)
    torch.cuda.synchronize()
    single = Generator(arena, 1, 257 + NEW)
    for b in range(B):
        one, _ = single.generate(prefix[b:b + 1].to(_dev()), NEW)
        assert ids[b].cpu().tolist() == one[0].cpu().tolist()
    for b in (0, B - 1):
        ref_ids, _ = oracle.generate(prefix[b], NEW)
        assert ids[b].cpu().tolist() == ref_ids


@gpu
def test_prefill_larger_than_one_pass(small):
    """more sequences than one prefill pass (8) takes."""
    from meshanything_b200.decoder import Generator
    _, arena, oracle = small
    B = 10
    prefix = random_prefix(B, seed=21)
    gen = Generator(arena, B, 257 + 6)
    ids, _ = gen.generate(prefix.to(_dev()), 6)
    ref_ids, _ = oracle.generate(prefix[9], 6)
    assert ids[9].cpu().tolist() == ref_ids


@gpu
def test_eos_and_padding(small):
    """HF semantics: a row that emitted eos is padded; generation stops early when all rows finished."""
    from meshanything_b200.decoder import Generator
    _, arena, oracle = small
    prefix = random_prefix(2, seed=5)
    gen = Generator(arena, 2, 257 + NEW)
    free, _ = gen.generate(prefix.to(_dev()), NEW)
    free = free.cpu()
    eos = int(free[0, 7])                     # pretend the 8th token of row 0 is eos
    first0 = free[0].tolist().index(eos)
    ids, lens = gen.generate(prefix.to(_dev()), NEW, eos_id=eos, pad_id=2)
    ids, lens = ids.cpu(), lens.cpu()
    assert ids[0, :first0 + 1].tolist() == free[0, :first0 + 1].tolist()
    assert all(t == 2 for t in ids[0, first0 + 1:].tolist())
    assert int(lens[0]) == first0 + 1
    row1 = free[1].tolist()
    if eos in row1:
        j = row1.index(eos)
        assert ids[1, :j + 1].tolist() == row1[:j + 1] and int(lens[1]) == j + 1
    else:
        assert ids[1].tolist() == row1 and int(lens[1]) == NEW
    # batch of one (fast path): stops at eos, remaining ids are pad, oracle agrees
    g1 = Generator(arena, 1, 257 + NEW)
    ids1, lens1 = g1.generate(prefix[:1].to(_dev()), NEW, eos_id=eos)
    ref_ids, _ = oracle.generate(prefix[0], NEW, eos_id=eos)
    got = ids1[0].cpu().tolist()
    assert got[:len(ref_ids)] == ref_ids and all(t == 2 for t in got[len(ref_ids):])
    assert int(lens1[0]) == len(ref_ids)


@gpu
def test_teacher_forced_logits(small):
    """forced ids (incl. specials 0/1/2, which take the extra_embeds path) give the oracle's logits, on the per-phase
    kernels (flags 0) and the batched kernels (flags 2)."""
    from meshanything_b200.decoder import Generator
    _, arena, oracle = small
    prefix = random_prefix(1, seed=8)
    forced = [0, 5, 8194, 1, 2, 3, 77, 4000, 2, 9, 10, 11, 12]
    n = len(forced)
    gen = Generator(arena, 1, 257 + n)
    f = torch.tensor([forced], dtype=torch.int32)
    _, ref_logits = oracle.generate(prefix[0], n, eos_id=-1, forced=forced, keep_logits=True)
    for flags in (0, 2):
        ids, lens, logits = gen.generate(prefix.to(_dev()), n, forced_ids=f, want_logits=True, eos_id=-1, flags=flags)
        assert ids[0].cpu().tolist() == forced
        for i in range(n):
            assert torch.equal(logits[i, 0].cpu().view(torch.int16), ref_logits[i].view(torch.int16)), (flags, i)


@gpu
def test_tensor_core_decoder_logits_within_tolerance(small):
    """MA_GEN_TC (implied by sampling for batches): prefill GEMMs on gemm_tc_kernel, decode-step GEMMs on the
    weight-streaming gemm_ws_kernel.  Teacher-forced logits of a batch of 4 stay within a stated tolerance of the CPU
    oracle's (the tensor core sums K in its own order: fp32 rounding differences, amplified by the fp16 rounding points
    of 3 layers), the argmax agrees wherever the oracle's top-2 margin exceeds the tolerance, and two runs are
    bit-identical (deterministic K-slice reduction)."""
    from meshanything_b200 import capi
    from meshanything_b200.decoder import Generator
    _, arena, oracle = small
    B, n = 4, 20
    prefix = random_prefix(B, seed=31)
    forced = torch.randint(3, 8195, (B, n), generator=torch.Generator().manual_seed(5), dtype=torch.int32)
    forced[0, 4], forced[1, 7], forced[2, 2] = 0, 1, 2
    gen = Generator(arena, B, 257 + n)
    ids, lens, logits = gen.generate(prefix.to(_dev()), n, forced_ids=forced, want_logits=True, eos_id=-1,
                                     flags=capi.GEN_TC)
    _, _, logits2 = gen.generate(prefix.to(_dev()), n, forced_ids=forced, want_logits=True, eos_id=-1,
                                 flags=capi.GEN_TC)
    assert torch.equal(logits.view(torch.int16), logits2.view(torch.int16))
    worst = 0.0
    for b in range(B):
        _, ref = oracle.generate(prefix[b], n, eos_id=-1, forced=forced[b].tolist(), keep_logits=True)
        ref = torch.stack(ref).float()
        got = logits[:, b].cpu().float()
        diff = (got - ref).abs()
        worst = max(worst, float(diff.max()))
        assert diff.max() < 3e-2 and diff.mean() < 3e-3, (b, float(diff.max()), float(diff.mean()))
        top2 = torch.topk(ref, 2, dim=1).values
        clear = (top2[:, 0] - top2[:, 1]) > 6e-2
        assert torch.equal(got.argmax(1)[clear], ref.argmax(1)[clear])
    print("tensor-core decoder: max |logit diff| vs oracle", worst)


@gpu
def test_long_context_crosses_chunks(small):
    """600 new tokens: the context crosses three 256-key attention chunks (257 -> 857); per-phase kernels."""
    from meshanything_b200.decoder import Generator
    _, arena, oracle = small
    prefix = random_prefix(1, seed=13)
    n = 600
    ref_ids, _ = oracle.generate(prefix[0], n)
    gen = Generator(arena, 1, 257 + n)
    ids, _ = gen.generate(prefix.to(_dev()), n)
    assert ids[0].cpu().tolist() == ref_ids


@gpu
def test_sampling_is_deterministic_and_in_support(small):
    from meshanything_b200.decoder import Generator
    _, arena, _ = small
    prefix = random_prefix(2, seed=17)
    gen = Generator(arena, 2, 257 + 24)
    a, _, lg = gen.generate(prefix.to(_dev()), 24, do_sample=True, seed=7, want_logits=True)
    b, _ = gen.generate(prefix.to(_dev()), 24, do_sample=True, seed=7)
    c, _ = gen.generate(prefix.to(_dev()), 24, do_sample=True, seed=8)
    assert torch.equal(a, b)
    assert not torch.equal(a, c)
    # every sampled token is inside the reference's top-k(50) support of that step's logits
    for i in range(24):
        for r in range(2):
            top = torch.topk(lg[i, r].float(), 50).values[-1]
            assert lg[i, r, int(a[r, i])].float() >= top


@gpu
@pytest.mark.slow
def test_full_depth_config1_golden():
    """24 layers, F=64 (578 new tokens): ids equal the oracle's; cross-checked with the committed golden."""
    import json, os
    from meshanything_b200.decoder import DecoderArena, Generator
    from oracle.decoder import OracleDecoder
    sd = decoder_sd(24)
    arena = DecoderArena(sd, _dev())
    prefix = random_prefix(1, seed=1)
    n = 64 * 9 + 2
    gen = Generator(arena, 1, 257 + n)
    ids, _ = gen.generate(prefix.to(_dev()), n)
    got = ids[0].cpu().tolist()
    gold = os.path.join(os.path.dirname(__file__), "golden", "decoder_greedy_seed0_F64.json")
    if os.path.exists(gold):
        assert got == json.load(open(gold))["ids"]
    else:
        oracle = OracleDecoder(sd, 24, 257 + n)
        ref, _ = oracle.generate(prefix[0], n)
        assert got == ref


@gpu
@pytest.mark.slow
def test_full_depth_config2_golden():
    """BASELINE.json configs[1] parity: 24 layers, 800-face cap (7202 new tokens, contexts up to 7458), batch 1, greedy.
    The free-running token ids on the per-phase kernels equal the CPU oracle's (tests/golden/decoder_greedy_seed0_F800.json,
    generated by tests/golden/make_golden.py greedy800)."""
    import json, os
    from meshanything_b200.decoder import DecoderArena, Generator
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "decoder_greedy_seed0_F800.json")))["ids"]
    arena = DecoderArena(decoder_sd(24), _dev())
    prefix = random_prefix(1, seed=1).to(_dev())
    n = 800 * 9 + 2
    gen = Generator(arena, 1, 257 + n)
    ids, lens = gen.generate(prefix, n)
    got = ids[0].cpu().tolist()
    first_bad = next((i for i, (a, b) in enumerate(zip(got, gold)) if a != b), None)
    assert first_bad is None, f"first divergence at step {first_bad}"
    assert int(lens[0]) == n


@gpu
@pytest.mark.slow
def test_long_context_config5_golden():
    """BASELINE.json configs[4] length (V1 architecture, 1600-face cap: 14402 new tokens, contexts up to 14658 = 58
    attention chunks).  First 4 layers of the synthetic decoder; ids equal the CPU oracle's
    (tests/golden/decoder_greedy_seed0_F1600.json, make_golden.py greedy1600) for the per-phase kernels and for a batch
    of 2 on the batched kernels (row 0 = the golden prefix, row 1 another prefix: rows are independent)."""
    import json, os
    from meshanything_b200.decoder import DecoderArena, Generator
    g = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "decoder_greedy_seed0_F1600.json")))
    gold, NL, eos = g["ids"], g["n_layers"], g.get("eos_id", 1)
    assert len(gold) == 1600 * 9 + 2
    arena = DecoderArena(decoder_sd(NL), _dev())
    prefix = random_prefix(1, seed=1).to(_dev())
    n = 1600 * 9 + 2
    gen = Generator(arena, 1, 257 + n)
    ids, lens = gen.generate(prefix, n, eos_id=eos)
    got = ids[0].cpu().tolist()
    first_bad = next((i for i, (a, b) in enumerate(zip(got, gold)) if a != b), None)
    assert first_bad is None, f"first divergence at step {first_bad}"
    assert int(lens[0]) == n
    two = torch.cat([prefix, random_prefix(1, seed=5).to(_dev())], dim=0)
    gen2 = Generator(arena, 2, 257 + n)
    ids2, _ = gen2.generate(two, n, eos_id=eos)
    assert ids2[0].cpu().tolist() == gold


@gpu
@pytest.mark.parametrize("slots,poll_every,flags", [(2, 4, 0), (3, 7, 1), (1, 5, 0)])
def test_continuous_batching_equals_solo_generation(small, slots, poll_every, flags):
    """SURVEY 8(f)2: a queue of 6 prefixes through `slots` cache slots with refill on EOS.  EOS is re-declared as a
    token each sequence emits at a different step, so lengths differ; every sequence must come back with exactly the
    ids (and length) a solo `Generator.generate` gives it."""
    from meshanything_b200.decoder import Generator
    from meshanything_b200.scheduler import SlotEngine, SlotScheduler
    _, arena, _ = small
    n, NP = 40, 6
    prefixes = random_prefix(NP, seed=23).to(_dev())
    solo_gen = Generator(arena, 1, 257 + n)
    free = [solo_gen.generate(prefixes[i:i + 1], n)[0][0].cpu().tolist() for i in range(NP)]
    # an eos that shows up at different steps in different sequences (and not at all in some)
    cand = {}
    for t in set(free[0][3:]) | set(free[1][10:]) | set(free[2][20:]):
        firsts = [seq.index(t) if t in seq else None for seq in free]
        cand[t] = firsts
    eos = max(cand, key=lambda t: len({f for f in cand[t] if f is not None}))
    solo = []
    for i in range(NP):
        ids, lens = solo_gen.generate(prefixes[i:i + 1], n, eos_id=eos)
        solo.append(ids[0, :int(lens[0])].cpu().tolist())
    assert len({len(s) for s in solo}) >= 2, "test needs sequences of different lengths"
    eng = SlotEngine(arena, slots, 257 + n, n, eos_id=eos, flags=flags)
    sched = SlotScheduler(eng, slots, n, poll_every=poll_every)
    got = {idx: ids.cpu().tolist() for idx, ids in sched.run([prefixes[i] for i in range(NP)])}
    assert sorted(got) == list(range(NP))
    for i in range(NP):
        assert got[i] == solo[i], (i, len(got[i]), len(solo[i]))
    assert sched.stats.prefills == NP


@gpu
def test_continuous_batching_sampling_streams_follow_the_queue(small):
    """Sampling under continuous batching: draws are keyed by (seed, index of the shape in the queue, token index), not
    by the cache slot.  The same prefix queued three times through ONE slot must give three different samples (a
    slot-keyed stream would repeat the first), and a queue's results must not depend on how many slots it ran through
    (2 vs 3 slots: same kernels, same per-row arithmetic, different slot assignment)."""
    from meshanything_b200.scheduler import SlotEngine, SlotScheduler
    _, arena, _ = small
    n = 24
    p = random_prefix(2, seed=31).to(_dev())

    def run(queue, slots):
        eng = SlotEngine(arena, slots, 257 + n, n, do_sample=True, seed=11, eos_id=-1)
        sched = SlotScheduler(eng, slots, n, poll_every=5)
        got = {idx: ids.cpu().tolist() for idx, ids in sched.run(queue)}
        return [got[i] for i in range(len(queue))]

    one = run([p[0], p[0], p[0]], 1)
    assert one[0] != one[1] and one[1] != one[2] and one[0] != one[2]
    assert run([p[0], p[0], p[0]], 1) == one
    q = [p[0], p[1], p[0], p[1], p[0]]
    assert run(q, 2) == run(q, 3)
