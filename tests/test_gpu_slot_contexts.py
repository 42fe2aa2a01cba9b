"""-m gpu: decode attention launched the way a decode step launches it, with a grid sized apart from each row's context.

A decode step sizes its attention grid by a 1024-key bucket, max_keys = min(tmax, bucket * 1024), and reuses one
scratch area for every launch.  Under continuous batching a finished slot stays frozen at its last position while the
bucket follows the live slots, so a frozen row can hold more keys than the launch has chunks for; both kernels then
attend over the first cap = ceil(max_keys / 256) * 256 keys of that row (its output is discarded).

  A  ma_attention_decode_f16 (attention_stream_kernel, KV append folded in) and ma_attention_f16 (attention_kernel,
     slot = row) with an explicit max_keys and a caller-owned scratch: a grid larger than the rows need, frozen rows
     above the capacity next to live rows, one scratch across buckets;
  B  the slot engine (3-layer synthetic decoder) with a slot frozen at 2557 keys while the other runs through the
     1024 / 2048 boundaries: greedy, through SlotScheduler, on attention_kernel (MA_B200_NO_STREAM_ATTN=1), sampled;
  C  ma_decode_slots_seek against the state of a real run.

Every comparison is bit for bit (DESIGN.md section 6).
"""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

from tests.util import decoder_sd, random_prefix

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, CHUNK, PREFIX = 16, 256, 257
LDQ, LDO = 3072, 1024 + 64             # qkv rows; the output buffer is padded to catch writes past column 1024
SENTINEL = 0x7E5A                      # an fp16 quiet-NaN bit pattern no kernel produces
POISON = 0.5                           # cache rows a call must not write (finite: a later launch may read them)
NAN = float("nan")


def _dev():
    return torch.device("cuda:0")


def _cap(max_keys: int) -> int:
    """Keys a launch sized by max_keys has chunks for."""
    return -(-max_keys // CHUNK) * CHUNK


def _bucket_max_keys(ctx: int, tmax: int) -> int:
    """The grid size of a decode step whose live rows see at most ctx keys (ma_decode_slots_step)."""
    return min(tmax, -(-ctx // 1024) * 1024)


# ------------------------------------------------------------------------------------------------------------------ A
class _Cache:
    """M cache slots (K and V, [M, 16, T, 64] fp16) on the device, and on the host what they must hold."""

    def __init__(self, M: int, T: int, seed: int):
        self.M, self.T = M, T
        self.g = torch.Generator(device=_dev()).manual_seed(seed)
        self.kd = torch.randn(M, H, T, 64, generator=self.g, device=_dev()).half()
        self.vd = torch.randn(M, H, T, 64, generator=self.g, device=_dev()).half()
        self.k, self.v = self.kd.cpu(), self.vd.cpu()


def _scratch(M: int, max_keys: int) -> torch.Tensor:
    from meshanything_b200 import capi
    return torch.zeros(capi.lib().ma_attention_scratch_bytes(M, H, max_keys), dtype=torch.uint8, device=_dev())


def _launch(kernel: str, cache: _Cache, qkv: torch.Tensor, nk, max_keys: int, scratch: torch.Tensor) -> torch.Tensor:
    """One decode attention over the cache with this max_keys and scratch.  Returns the whole output buffer
    [M + 3, LDO] (int16), filled with the sentinel before the call."""
    from meshanything_b200 import capi
    L, M = capi.lib(), cache.M
    nkeys = torch.tensor(nk, dtype=torch.int32, device=_dev())
    buf = torch.full((M + 3, LDO), SENTINEL, dtype=torch.int16, device=_dev())
    if kernel == "stream":
        rc = L.ma_attention_decode_f16(capi.ptr(qkv), LDQ, capi.ptr(cache.kd), capi.ptr(cache.vd), cache.T,
                                       capi.ptr(nkeys), max_keys, M, 0.125, capi.ptr(buf), LDO, capi.ptr(scratch),
                                       capi.stream_ptr())
    else:
        rc = L.ma_attention_f16(capi.ptr(qkv), LDQ, capi.ptr(cache.kd), capi.ptr(cache.vd), cache.T, H, None,
                                capi.ptr(nkeys), max_keys, M, 0.125, capi.ptr(buf), LDO, capi.ptr(scratch),
                                capi.stream_ptr())
    capi.check(rc, kernel)
    torch.cuda.synchronize()
    return buf


def _step(kernel: str, cache: _Cache, nk, max_keys: int, scratch: torch.Tensor, what):
    """One decode step's attention over a fresh qkv.  Rows with nkeys <= cap are live: their current k / v go to the
    cache at nkeys - 1 (by the kernel for "stream", which must not read that row from the cache, so it is NaN
    beforehand; for "chunked" beforehand, as kv_append_kernel does).  The others are frozen: their row nkeys - 1 is
    poisoned and must keep its bits.  Checks every row against the oracle over min(nkeys, cap) keys, the whole cache,
    the output buffer outside [0, M) x [0, 1024) and the scratch's counters.  Returns (qkv, output [M, 1024] int16)."""
    from oracle import decoder as orc
    M, cap = cache.M, _cap(max_keys)
    assert len(nk) == M and max(nk) <= cache.T
    qkv = torch.randn(M, LDQ, generator=cache.g, device=_dev()).half()
    qh = qkv.cpu()
    for m, n in enumerate(nk):
        if n <= cap:
            cache.k[m, :, n - 1] = qh[m, 1024:2048].view(H, 64)
            cache.v[m, :, n - 1] = qh[m, 2048:].view(H, 64)
            if kernel == "stream":
                cache.kd[m, :, n - 1] = NAN
                cache.vd[m, :, n - 1] = NAN
            else:
                cache.kd[m, :, n - 1] = qkv[m, 1024:2048].view(H, 64)
                cache.vd[m, :, n - 1] = qkv[m, 2048:].view(H, 64)
        else:
            for t in (cache.k, cache.v, cache.kd, cache.vd):
                t[m, :, n - 1] = POISON
    buf = _launch(kernel, cache, qkv, nk, max_keys, scratch)
    out = buf[:M, :1024].cpu()
    assert bool((buf[M:] == SENTINEL).all()) and bool((buf[:M, 1024:] == SENTINEL).all()), (what, "wrote outside")
    assert torch.equal(cache.kd.cpu().view(torch.int16), cache.k.view(torch.int16)), (what, "K cache")
    assert torch.equal(cache.vd.cpu().view(torch.int16), cache.v.view(torch.int16)), (what, "V cache")
    assert int(scratch[:M * H * 4].view(torch.int32).count_nonzero()) == 0, (what, "counters not re-armed")
    for m, n in enumerate(nk):
        ref = orc.attention(qh[m:m + 1, :1024].view(1, H, 64), cache.k[m], cache.v[m], [min(n, cap)])
        assert torch.equal(out[m], ref.view(-1).view(torch.int16)), (what, m, n, cap)
    return qkv, out


KERNELS = ["stream", "chunked"]
# (max_keys, nkeys of the rows): bucket sizes of production (a multiple of 1024, or tmax = 2557, whose 10 chunks hold
# 2560 keys), with max_keys equal to, above and below max(nkeys)
A1_CASES = [(1024, [1, 255, 256, 257, 1023, 1024]), (2048, [1025, 1500, 2048, 300]), (2048, [1, 257, 700, 1023]),
            (2557, [2557, 2558, 2560, 2300, 1, 2049]), (2557, [300, 1024, 1025])]


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("max_keys,nk", A1_CASES)
def test_grid_larger_than_the_rows_need(kernel, max_keys, nk):
    """Every row live, the grid sized by max_keys: bit-exact to the oracle (and the streaming kernel's appended cache
    rows equal to the qkv buffer's k / v), and bit-identical to the same call with max_keys = max(nkeys)."""
    M = len(nk)
    cache = _Cache(M, 2600, seed=max_keys * 10 + M)
    assert max(nk) <= _cap(max_keys)
    qkv, out = _step(kernel, cache, nk, max_keys, _scratch(M, max_keys), (kernel, max_keys))
    # the appended rows are in place now, so the streaming kernel rewrites the same bits
    buf = _launch(kernel, cache, qkv, nk, max(nk), _scratch(M, max(nk)))
    assert torch.equal(buf[:M, :1024].cpu(), out)


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("max_keys", [1024, 2048, 2557])
def test_frozen_rows_above_the_capacity(kernel, max_keys):
    """Frozen rows (nkeys = cap + 1, cap + 256, T) directly before live rows and at the last row, so that chunk partials
    or an output spilled past a frozen row's region would land on a live row's: live rows bit-exact to the oracle,
    frozen rows the oracle over their first cap keys, nothing appended to a frozen row's cache, nothing written outside
    the output rows."""
    T = 3000
    cap = _cap(max_keys)
    nk = [700, cap + 1, cap, cap + 256, T, 257, 1, cap + 1]
    frozen = [m for m, n in enumerate(nk) if n > cap]
    assert frozen == [1, 3, 4, 7] and all(m + 1 == len(nk) or nk[m + 1] <= cap for m in (1, 4))
    _step(kernel, _Cache(len(nk), T, seed=max_keys), nk, max_keys, _scratch(len(nk), max_keys), (kernel, max_keys))


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
def test_one_scratch_across_buckets(kernel):
    """One scratch area sized for the largest bucket and never re-zeroed, M = 40 rows (10 chunks x 16 heads x 40 rows is
    more work than one wave of the streaming kernel's CTAs), launches at max_keys 1024 -> 2557 -> 1024 -> 2048 -> 1024.
    Rows change between live and frozen from one launch to the next; row 7 is frozen in the first launch and live over
    8 chunks in the second, reusing the counters the clamp went through.  Every launch as in the tests above."""
    M, T = 40, 2600
    seq = [1024, 2557, 1024, 2048, 1024]
    cache = _Cache(M, T, seed=40)
    scratch = _scratch(M, max(seq))
    g = torch.Generator().manual_seed(41)
    history = []
    for i, max_keys in enumerate(seq):
        cap = _cap(max_keys)
        nk = []
        for m in range(M):
            if torch.rand(1, generator=g).item() < 0.35:
                nk.append(int(torch.randint(cap + 1, T + 1, (1,), generator=g)))
            else:
                nk.append(int(torch.randint(1, cap + 1, (1,), generator=g)))
        nk[0], nk[M - 1] = cap, T              # a full live row first, a frozen row last
        nk[7] = 2000                           # frozen in the first launch, 8 chunks live in the second
        history.append([n > cap for n in nk])
        _step(kernel, cache, nk, max_keys, scratch, (kernel, i, max_keys))
    assert history[0][7] and not history[1][7]
    assert all(sum(f) >= 5 and sum(f) <= M - 5 for f in history)


# ------------------------------------------------------------------------------------------------------------------ B
NL = 3
MAX_NEW = 2300
TMAX = PREFIX + MAX_NEW                # 2557: three buckets, the last one 2557 keys
POLL = 37
SEED = 19
# C's (and D's) steps at which the other slot, frozen at 2557 keys, holds more keys than the launch's chunks
ABOVE = sum(TMAX > _cap(_bucket_max_keys(PREFIX + 1 + j, TMAX)) for j in range(MAX_NEW - 1))


def _frozen_nkeys(lens: int) -> int:
    """Keys a finished slot's row attends at every later step: pos + 1, pos = 256 + lens (257 for a free slot)."""
    return PREFIX + 1 if lens == 0 else PREFIX + lens


class _Tracked:
    """A SlotScheduler engine over a SlotEngine that counts the decode steps in which a finished slot (as of the last
    poll) held more keys than that step's attention launch has chunks for, and the kernel launches per step."""

    def __init__(self, eng):
        self.eng = eng
        self.fin, self.lens = [1] * eng.B, [0] * eng.B      # ma_decode_slots_init: every slot free
        self.above = self.steps = self.launches = 0

    def prefill(self, slot, payload, stream_id=None):
        if stream_id is None:
            self.eng.prefill(slot, payload)
        else:
            _prefill_on_stream(self.eng, slot, payload, stream_id)
        self.fin[slot] = 0

    def step(self, n, max_ctx):
        from meshanything_b200 import capi
        frozen = [_frozen_nkeys(ln) for f, ln in zip(self.fin, self.lens) if f]
        for i in range(n):
            cap = _cap(_bucket_max_keys(min(self.eng.tmax, max_ctx + i), self.eng.tmax))
            self.above += any(nk > cap for nk in frozen)
        before = capi.lib().ma_launch_count()
        self.eng.step(n, max_ctx)
        self.launches += capi.lib().ma_launch_count() - before
        self.steps += n

    def poll(self):
        self.fin, self.lens = self.eng.poll()
        return self.fin, self.lens

    def fetch(self, slot, n):
        return self.eng.fetch(slot, n)


def _prefill_on_stream(eng, slot, prefix, stream_id):
    """SlotEngine.prefill with a chosen Philox stream (the engine numbers the streams by its own prefills)."""
    from meshanything_b200 import capi
    L = capi.lib()
    capi.check(L.ma_decode_slot_stream(slot, eng.B, eng.tmax, stream_id, capi.ptr(eng.ws), capi.stream_ptr()),
               "ma_decode_slot_stream")
    capi.check(L.ma_decode_slot_prefill(C.byref(eng.arena.c), capi.ptr(prefix.contiguous()), slot, eng.B, eng.tmax,
                                        eng.max_new, C.byref(eng.samp), eng.eos_id, eng.pad_id, capi.ptr(eng.kv),
                                        capi.ptr(eng.ws), capi.ptr(eng.ids), capi.stream_ptr()),
               "ma_decode_slot_prefill")


def _drive(tr: _Tracked, slot: int, prefix, stream_id=None):
    """Prefill `slot` and step it to its token cap in calls of POLL steps with SlotScheduler's max_ctx (prefix + 1 +
    steps since the prefill), polling after each call.  Returns the slot's ids."""
    tr.prefill(slot, prefix, stream_id)
    done = 0
    while done < MAX_NEW - 1:
        n = min(POLL, MAX_NEW - 1 - done)
        tr.step(n, PREFIX + 1 + done)
        done += n
        fin, lens = tr.poll()
        assert lens[slot] == 1 + done and bool(fin[slot]) == (done == MAX_NEW - 1), (slot, done, fin, lens)
    return tr.eng.ids[slot].cpu().tolist()


def _three_phases(arena, prefixes, do_sample=False):
    """Slot 0 <- A, run to its cap (frozen at 2557 keys from then on); slot 1 <- C, run to its cap; slot 0 <- D, run to
    its cap.  Returns the ids of A, C, D, the steps of C's and of D's phase with the other slot above the capacity, and
    the kernel launches per decode step."""
    from meshanything_b200.scheduler import SlotEngine
    tr = _Tracked(SlotEngine(arena, 2, TMAX, MAX_NEW, do_sample=do_sample, seed=SEED, eos_id=-1))
    a = _drive(tr, 0, prefixes[0])
    tr.above = 0
    c = _drive(tr, 1, prefixes[1])
    above_c, tr.above = tr.above, 0
    d = _drive(tr, 0, prefixes[2])
    return {"ids": [a, c, d], "above": [above_c, tr.above], "launches_per_step": tr.launches / tr.steps}


def _prefixes():
    return random_prefix(3, seed=57).to(_dev())


@pytest.fixture(scope="module")
def dec():
    """(arena, prefixes A / C / D, their ids from a solo Generator.generate of MAX_NEW tokens)."""
    from meshanything_b200.decoder import DecoderArena, Generator
    arena = DecoderArena(decoder_sd(NL), _dev())
    prefixes = _prefixes()
    solo = Generator(arena, 1, TMAX)
    ids = [solo.generate(prefixes[i:i + 1], MAX_NEW, eos_id=-1)[0][0].cpu().tolist() for i in range(3)]
    return arena, prefixes, ids


@gpu
def test_slot_frozen_above_the_bucket_greedy(dec):
    """A runs to its cap in slot 0, then C in slot 1 through the 1024 and 2048 boundaries while row 0 stays frozen at
    2557 keys (above the capacity of the first two buckets), then D in slot 0 on the counters row 0 used under the
    clamp: A, C and D each equal solo generation."""
    arena, prefixes, solo = dec
    got = _three_phases(arena, prefixes)
    print(f"[slot contexts] greedy: steps with a frozen row above the bucket's capacity: {got['above']}")
    assert got["above"] == [ABOVE, ABOVE] and ABOVE > 1000
    for name, a, b in zip("ACD", got["ids"], solo):
        assert a == b, (name, next(i for i, (x, y) in enumerate(zip(a, b)) if x != y))


@gpu
@pytest.mark.parametrize("poll_every", [37, 1])
def test_scheduler_with_a_slot_frozen_above_the_bucket(dec, poll_every):
    """A, C, D through SlotScheduler with 2 slots: A and C end together, D runs in slot 0 while slot 1 is frozen at
    2557 keys; every sequence equals solo generation."""
    from meshanything_b200.scheduler import SlotEngine, SlotScheduler
    arena, prefixes, solo = dec
    tr = _Tracked(SlotEngine(arena, 2, TMAX, MAX_NEW, eos_id=-1))
    sched = SlotScheduler(tr, 2, MAX_NEW, poll_every=poll_every)
    got = {i: ids.cpu().tolist() for i, ids in sched.run(list(prefixes))}
    print(f"[slot contexts] scheduler, poll_every {poll_every}: steps with a frozen row above the bucket's capacity: "
          f"{tr.above}")
    assert [got[i] for i in range(3)] == solo
    assert sched.stats.steps == 2 * (MAX_NEW - 1)          # A and C side by side, then D alone
    assert tr.above == ABOVE


def _phases_in_child():
    """Run in a fresh process (see the test below): prints the result of the greedy three phases as JSON."""
    from meshanything_b200.decoder import DecoderArena
    arena = DecoderArena(decoder_sd(NL), _dev())
    print(json.dumps(_three_phases(arena, _prefixes())))


@gpu
def test_slot_frozen_above_the_bucket_on_attention_kernel(dec):
    """The greedy three phases with MA_B200_NO_STREAM_ATTN=1 (kv_append_kernel + attention_kernel in each decode step;
    the library reads the variable once when it loads, so in a child process): A, C and D equal solo generation, and
    each step launches one kernel more per layer than on the streaming path."""
    from meshanything_b200.scheduler import SlotEngine
    arena, prefixes, solo = dec
    env = dict(os.environ, MA_B200_NO_STREAM_ATTN="1", MA_B200_NO_AUTOBUILD="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "from tests.test_gpu_slot_contexts import _phases_in_child; _phases_in_child()"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    child = json.loads(r.stdout.strip().splitlines()[-1])
    print(f"[slot contexts] attention_kernel: steps with a frozen row above the bucket's capacity: {child['above']}")
    assert child["above"] == [ABOVE, ABOVE]
    for name, a, b in zip("ACD", child["ids"], solo):
        assert a == b, name
    tr = _Tracked(SlotEngine(arena, 2, TMAX, MAX_NEW, eos_id=-1))
    tr.prefill(0, prefixes[0])
    tr.step(3, PREFIX + 1)
    assert child["launches_per_step"] == tr.launches / tr.steps + NL


@gpu
def test_slot_frozen_above_the_bucket_sampled(dec):
    """The three phases with top-k / top-p sampling (tensor-core GEMMs at B = 2; A, C, D draw from Philox streams 0, 1,
    2).  C equals C alone in slot 1 of a fresh engine on stream 1, D equals D alone in slot 0 on stream 2: a row frozen
    above the bucket does not leak into the live one."""
    from meshanything_b200.scheduler import SlotEngine
    arena, prefixes, solo = dec
    got = _three_phases(arena, prefixes, do_sample=True)
    print(f"[slot contexts] sampled: steps with a frozen row above the bucket's capacity: {got['above']}")
    assert got["above"] == [ABOVE, ABOVE]
    for slot, i in ((1, 1), (0, 2)):
        tr = _Tracked(SlotEngine(arena, 2, TMAX, MAX_NEW, do_sample=True, seed=SEED, eos_id=-1))
        alone = _drive(tr, slot, prefixes[i], stream_id=i)
        assert got["ids"][i] == alone, "CD"[i - 1]
    assert got["ids"][1] != solo[1] and got["ids"][2] != solo[2]      # sampled, not greedy


# ------------------------------------------------------------------------------------------------------------------ C
@gpu
def test_slots_seek_reproduces_a_real_run(dec):
    """Two slots run the same prefix greedily for 1400 tokens.  Seeking both to g0 generated tokens (pos = 256 + g0,
    gen = g0, tok = ids[g0 - 1], as bench.py does) and stepping 100 times with max_ctx = pos + 1 gives the run's ids
    g0 .. g0 + 99, lens g0 + 100 unfinished, and a KV cache bit-identical to the run's.  g0 = 767 crosses the 1024-key
    bucket boundary.  Out-of-range arguments are refused before anything is launched."""
    from meshanything_b200 import capi
    from meshanything_b200.scheduler import SlotEngine
    arena, prefixes, _ = dec
    L = capi.lib()
    max_new = 1400
    tmax = PREFIX + max_new
    eng = SlotEngine(arena, 2, tmax, max_new, eos_id=-1)
    eng.prefill(0, prefixes[0])
    eng.prefill(1, prefixes[0])
    done = 0
    while done < max_new - 1:
        n = min(POLL, max_new - 1 - done)
        eng.step(n, PREFIX + 1 + done)
        done += n
    assert eng.poll() == ([1, 1], [max_new, max_new])
    ids, kv = eng.ids.clone(), eng.kv.clone()
    assert torch.equal(ids[0], ids[1])
    buckets = {}
    for g0 in (767, 900):
        pos = PREFIX - 1 + g0
        buckets[g0] = {_bucket_max_keys(pos + 1 + i, tmax) for i in range(100)}
        eng.ids.fill_(eng.pad_id)
        capi.check(L.ma_decode_slots_seek(2, tmax, pos, g0, int(ids[0, g0 - 1]), capi.ptr(eng.ws), capi.stream_ptr()),
                   "ma_decode_slots_seek")
        eng.step(100, pos + 1)
        assert eng.poll() == ([0, 0], [g0 + 100, g0 + 100]), g0
        assert torch.equal(eng.ids[:, g0:g0 + 100], ids[:, g0:g0 + 100]), g0
        assert bool((eng.ids[:, :g0] == eng.pad_id).all()) and bool((eng.ids[:, g0 + 100:] == eng.pad_id).all())
        assert torch.equal(eng.kv, kv), g0
    assert buckets == {767: {1024, tmax}, 900: {tmax}}
    before = L.ma_launch_count()
    for pos, gen in ((PREFIX - 1, 5), (tmax, 5), (PREFIX + 10, 0)):
        assert L.ma_decode_slots_seek(2, tmax, pos, gen, 5, capi.ptr(eng.ws), capi.stream_ptr()) != 0, (pos, gen)
        assert "ma_decode_slots_seek" in L.ma_last_error().decode()
    assert L.ma_launch_count() == before
    assert eng.poll() == ([0, 0], [1000, 1000])              # the state of the last seek's run, untouched
