"""Continuous batching of the decode loop over a fixed number of cache slots (SURVEY.md section 8(f)2).

The reference pads every finished row of a batch until the longest sequence ends (HF `generate`, a10) and `main.py:137-152`
walks the dataset one padded batch at a time.  Here a slot is refilled from the queue of pending shapes as soon as its
sequence has hit EOS (or the token cap), so real-weight runs with EOS at varied lengths keep every slot busy.

Two layers:
  * `SlotScheduler` -- pure host logic over an engine interface (`prefill`, `step`, `poll`, `fetch`); tested on the CPU
    with a scripted engine (tests/test_scheduler.py);
  * `SlotEngine` -- that interface on the GPU over the C ABI (`ma_decode_slots_*`, include/meshanything_b200.h).

Rows never interact and the kernels are batch-invariant, so every sequence gets the ids a solo
`Generator.generate` gives it (greedy; with sampling the Philox stream is keyed by the shape's index in the queue,
whatever slot it lands in).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Callable, Iterable, Iterator, List, Optional, Tuple

import torch

from . import capi
from .config import DEC


@dataclass
class _Slot:
    item: Optional[int] = None     # index of the queued item that owns the slot (None: free)
    steps: int = 0                 # decode steps run since its prefill (upper bound of tokens generated - 1)


@dataclass
class SchedulerStats:
    steps: int = 0                 # batched decode steps enqueued
    polls: int = 0                 # synchronising polls
    prefills: int = 0
    slot_steps_live: int = 0       # sum over steps of slots that held an unfinished sequence at the last poll
    finished_order: List[int] = field(default_factory=list)


class SlotScheduler:
    """Runs a queue of items through `slots` cache slots of `engine`.

    engine.prefill(slot, payload)      -- start `payload` in `slot` (enqueue only)
    engine.step(n_steps, max_ctx)      -- n decode steps of every slot (enqueue only)
    engine.poll() -> (finished, lens)  -- per-slot lists (synchronises)
    engine.fetch(slot, n) -> result    -- the first n ids of the slot's output row
    """

    def __init__(self, engine, slots: int, max_new: int, prefix_len: int = DEC.cond_length, poll_every: int = 32):
        assert slots >= 1 and max_new >= 1 and poll_every >= 1
        self.engine, self.n_slots, self.max_new, self.prefix_len = engine, slots, max_new, prefix_len
        self.poll_every = poll_every
        self.stats = SchedulerStats()

    def run(self, items: Iterable) -> Iterator[Tuple[int, object]]:
        """Yields (index of the item in `items`, result) in completion order."""
        it = enumerate(items)
        slots = [_Slot() for _ in range(self.n_slots)]
        exhausted = False

        def refill() -> None:
            nonlocal exhausted
            for s, sl in enumerate(slots):
                if sl.item is None and not exhausted:
                    try:
                        idx, payload = next(it)
                    except StopIteration:
                        exhausted = True
                        return
                    self.engine.prefill(s, payload)
                    self.stats.prefills += 1
                    sl.item, sl.steps = idx, 0

        refill()
        while any(sl.item is not None for sl in slots):
            live = [sl for sl in slots if sl.item is not None]
            # a live slot has generated 1 + steps tokens: its next step attends to prefix + 1 + steps keys
            max_ctx = self.prefix_len + 1 + max(sl.steps for sl in live)
            # a sequence needs at most max_new - 1 decode steps after its prefill (which picks token 0)
            remaining = max(self.max_new - 1 - sl.steps for sl in live)
            if remaining > 0:
                n = min(self.poll_every, remaining)
                self.engine.step(n, max_ctx)
                self.stats.steps += n
                self.stats.slot_steps_live += n * len(live)
                for sl in live:
                    sl.steps = min(sl.steps + n, self.max_new - 1)
            finished, lens = self.engine.poll()
            self.stats.polls += 1
            for s, sl in enumerate(slots):
                if sl.item is not None and finished[s]:
                    result = self.engine.fetch(s, int(lens[s]))
                    self.stats.finished_order.append(sl.item)
                    yield sl.item, result
                    sl.item = None
                elif sl.item is not None and sl.steps >= self.max_new - 1:
                    raise RuntimeError(f"slot {s} ran {sl.steps} steps past its prefill and did not finish")
            refill()


class SlotEngine:
    """The scheduler's engine on the GPU: B cache slots of one `DecoderArena` over `ma_decode_slots_*`."""

    def __init__(self, arena, slots: int, tmax: int, max_new: int, do_sample: bool = False, top_k: int = 50,
                 top_p: float = 0.95, seed: int = 0, eos_id: int = DEC.eos_id, pad_id: int = DEC.pad_id,
                 flags: int = 0, to_prefix: Optional[Callable] = None):
        self.arena, self.B, self.tmax, self.max_new = arena, slots, tmax, max_new
        self.eos_id, self.pad_id, self.flags = eos_id, pad_id, flags
        self.to_prefix = to_prefix          # payload -> fp32 [257,1024] device tensor (e.g. the point-cloud encoder)
        L = capi.lib()
        dev = arena.device
        self.kv = torch.empty(L.ma_kv_cache_bytes(arena.n_layers, slots, tmax), dtype=torch.uint8, device=dev)
        self.ws = torch.empty(L.ma_decoder_workspace_bytes(slots, tmax), dtype=torch.uint8, device=dev)
        self.ids = torch.full((slots, max_new), pad_id, dtype=torch.int32, device=dev)
        self.samp = capi.Sampling(int(do_sample), int(top_k), float(top_p), int(seed))
        self._fin = (C.c_int32 * slots)()
        self._len = (C.c_int32 * slots)()
        self.reset()

    def reset(self) -> None:
        """Every slot free again (call between queues; sequences still in flight are dropped)."""
        self._n_prefills = 0
        capi.check(capi.lib().ma_decode_slots_init(self.B, self.tmax, self.pad_id, capi.ptr(self.ws),
                                                   capi.stream_ptr()), "ma_decode_slots_init")

    def prefill(self, slot: int, payload) -> None:
        prefix = self.to_prefix(payload) if self.to_prefix is not None else payload
        assert prefix.is_cuda and prefix.dtype == torch.float32
        prefix = prefix.reshape(DEC.cond_length, DEC.hidden).contiguous()
        if self.samp.do_sample:      # the k-th shape of this run draws from Philox stream k, whatever slot it lands in
            capi.check(capi.lib().ma_decode_slot_stream(slot, self.B, self.tmax, self._n_prefills, capi.ptr(self.ws),
                                                        capi.stream_ptr()), "ma_decode_slot_stream")
        self._n_prefills += 1
        capi.check(capi.lib().ma_decode_slot_prefill(C.byref(self.arena.c), capi.ptr(prefix), slot, self.B, self.tmax,
                                                     self.max_new, C.byref(self.samp), self.eos_id, self.pad_id,
                                                     capi.ptr(self.kv), capi.ptr(self.ws), capi.ptr(self.ids),
                                                     capi.stream_ptr()), "ma_decode_slot_prefill")
        # `prefix` may be dropped right away: the library reads it on its own stream, and the current stream waits for
        # that stream's event before the call returns, so a later reuse of the block (same stream) is ordered after it

    def step(self, n_steps: int, max_ctx: int) -> None:
        capi.check(capi.lib().ma_decode_slots_step(C.byref(self.arena.c), self.B, self.tmax, self.max_new, n_steps,
                                                   min(max_ctx, self.tmax), C.byref(self.samp), self.eos_id,
                                                   self.pad_id, capi.ptr(self.kv), capi.ptr(self.ws),
                                                   capi.ptr(self.ids), self.flags, capi.stream_ptr()),
                   "ma_decode_slots_step")

    def poll(self):
        capi.check(capi.lib().ma_decode_slots_poll(self.B, self.tmax, capi.ptr(self.ws), self._fin, self._len,
                                                   capi.stream_ptr()), "ma_decode_slots_poll")
        return list(self._fin), list(self._len)

    def fetch(self, slot: int, n: int) -> torch.Tensor:
        return self.ids[slot, :n].clone()


def generate_queue(arena, prefixes: Iterable[torch.Tensor], slots: int, max_new: int, poll_every: int = 32,
                   **engine_kw) -> List[torch.Tensor]:
    """ids (int32, up to and including eos) of every prefix, in input order."""
    tmax = DEC.cond_length + max_new
    eng = SlotEngine(arena, slots, tmax, max_new, **engine_kw)
    out = {}
    for idx, ids in SlotScheduler(eng, slots, max_new, poll_every=poll_every).run(prefixes):
        out[idx] = ids
    return [out[i] for i in range(len(out))]
