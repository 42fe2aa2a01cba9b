"""Where the time of a batch-1 greedy decode step goes (bench.py config 2: batch 1, 800-face cap, per-phase kernels).

    python tools/bench_decode_b1.py [--faces 800] [--layers 24] [--reps 3] [--no-profile] [--json FILE]

Runs Generator.generate on the synthetic checkpoint (seed 0) at batch 1, greedy, early exit off, and reports:
  * end to end, CUDA events, profiler off: us per decode step over the whole generate, and over the short-context
    slice (T(300 tokens) - T(100 tokens)) / 200 as bench.py computes it;
  * per kernel, torch.profiler (CUDA activities) over one generate of its own: for three context bands (~300, ~3900,
    ~7400 keys) and each phase of the step (qkv, attention, out_proj, fc1, fc2, lm_head), the mean kernel duration and
    the mean increment of the chain -- this kernel's end minus the previous kernel's end, i.e. what the phase adds to
    the step.  With programmatic dependent launch a kernel starts long before its inputs exist, so its duration includes
    the wait for the previous kernel; the increments add up to the step.
Prints the card name and power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from meshanything_b200 import capi  # noqa: E402
from meshanything_b200.checkpoint import synthetic_decoder_state_dict  # noqa: E402
from meshanything_b200.config import DEC  # noqa: E402
from meshanything_b200.decoder import DecoderArena, Generator  # noqa: E402

OPS = ("qkv", "attention", "out_proj", "fc1", "fc2", "lm_head")
BANDS = (300, 3900, 7400)   # keys seen by the step
BAND_STEPS = 64             # steps per band


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_max_clock"] = [s.strip() for s in out.split(",")]
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"unknown ({e})"
    return info


def op_of(name):
    # attention_stream_kernel: the decode steps; attention_kernel: the prefill, and the decode steps under
    # MA_B200_NO_STREAM_ATTN=1 (whose kv_append_kernel is not matched: its time falls into the attention increment)
    if "attention_stream_kernel" in name or "attention_kernel" in name:
        return "attention"
    if "fast_gemv_kernel" in name:
        mode = name.split("fast_gemv_kernel<", 1)[1].split(">", 1)[0].split(",")[1].strip()
        return {"0": "qkv", "1": "out_proj", "2": "fc1", "3": "fc2", "4": "lm_head"}[mode]
    return None


def profile(gen, prefix, max_new, n_layers):
    from torch.profiler import ProfilerActivity, profile as tprofile
    per_step = 5 * n_layers + 1
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        gen.generate(prefix, max_new, flags=capi.GEN_NO_EARLY_EXIT)
        torch.cuda.synchronize()
    evs = []
    for e in prof.profiler.kineto_results.events():
        if e.device_type() != torch.autograd.DeviceType.CUDA:
            continue
        op = op_of(e.name())
        if op is not None:
            evs.append((e.start_ns(), e.end_ns(), op))
    evs.sort()
    # the decode steps start at the first fast_gemv_kernel (the prefill also runs attention_kernel); a step ends with
    # lm_head; a step whose kernel count is off (an event the profiler dropped) is skipped
    first = next(i for i, e in enumerate(evs) if e[2] != "attention")
    evs = evs[first:]
    steps, cur = [], []
    for e in evs:
        cur.append(e)
        if e[2] == "lm_head":
            steps.append(cur if len(cur) == per_step else None)
            cur = []
    rows = {}
    for c in BANDS:
        s0 = max(0, min(len(steps) - BAND_STEPS, c - DEC.cond_length - 1 - BAND_STEPS // 2))
        dur = {o: [] for o in OPS}
        inc = {o: [] for o in OPS}
        walls = []
        for s in range(max(1, s0), s0 + BAND_STEPS):
            st, prev = steps[s], steps[s - 1]
            if st is None or prev is None:
                continue
            last_end = prev[-1][1]
            walls.append((st[-1][1] - last_end) / 1e3)
            for (b, e, o) in st:
                dur[o].append((e - b) / 1e3)
                inc[o].append((e - last_end) / 1e3)
                last_end = e
        n = len(walls)
        if n == 0:
            continue
        rows[c] = {"keys": [DEC.cond_length + 1 + s0, DEC.cond_length + s0 + BAND_STEPS], "steps": n,
                   "us_per_step": sum(walls) / n,
                   "ops": {o: {"launches_per_step": len(dur[o]) // n,
                               "mean_duration_us": sum(dur[o]) / max(1, len(dur[o])),
                               "chain_us_per_step": sum(inc[o]) / n} for o in OPS}}
    return {"steps_parsed": sum(s is not None for s in steps), "steps_total": len(steps), "bands": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, default=800)
    ap.add_argument("--layers", type=int, default=24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode_b1.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    arena = DecoderArena(synthetic_decoder_state_dict(0, args.layers), dev)
    max_new = DEC.max_new_tokens(args.faces)
    gen = Generator(arena, 1, DEC.cond_length + max_new)
    prefix = (torch.randn(1, DEC.cond_length, DEC.hidden, generator=torch.Generator().manual_seed(1000)) * 0.7).to(dev)
    fl = capi.GEN_NO_EARLY_EXIT

    def timed(n, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        gen.generate(prefix, n, flags=fl)       # warm-up: graph capture of every shape this length uses
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            gen.generate(prefix, n, flags=fl)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps      # ms

    res = {"card": card(), "workload": f"batch 1, greedy, {args.layers} layers, {args.faces}-face cap "
                                       f"({max_new} new tokens), synthetic checkpoint seed 0"}
    t_full = timed(max_new, args.reps)
    t100, t300 = timed(100, 5), timed(300, 5)
    short = (t300 - t100) / 200 * 1e3
    prefill = t100 - 99 * short / 1e3
    res["e2e"] = {"generate_ms": t_full, "us_per_step_avg": (t_full - prefill) * 1e3 / (max_new - 1),
                  "us_per_step_short_context": short, "prefill_ms": prefill}
    if not args.no_profile:
        res["profile"] = profile(gen, prefix, max_new, args.layers)

    c = res["card"]
    print(f"# {c['name']}, power limit {c.get('power_limit')}, max SM clock {c.get('sm_max_clock')}")
    print(f"# {res['workload']}")
    e = res["e2e"]
    print(f"e2e (CUDA events, profiler off): generate {e['generate_ms']:.1f} ms, {e['us_per_step_avg']:.1f} us/step "
          f"averaged over the run, {e['us_per_step_short_context']:.1f} us/step at context 357..557")
    if "profile" in res:
        p = res["profile"]
        print(f"profile (torch.profiler, CUDA activities): {p['steps_parsed']} of {p['steps_total']} steps parsed")
        for band, r in p["bands"].items():
            print(f"\nkeys {r['keys'][0]}..{r['keys'][1]} ({r['steps']} steps): {r['us_per_step']:.1f} us/step")
            print(f"  {'phase':<10} {'launches':>8} {'mean dur us':>12} {'chain us/step':>14} {'share':>6}")
            for o in OPS:
                q = r["ops"][o]
                print(f"  {o:<10} {q['launches_per_step']:>8} {q['mean_duration_us']:>12.2f} "
                      f"{q['chain_us_per_step']:>14.1f} {q['chain_us_per_step'] / r['us_per_step']:>6.1%}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
