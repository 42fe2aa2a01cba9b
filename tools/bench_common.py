"""What the tools/bench_*.py scripts share: summary statistics, the device a run was measured on, and timing of a
library call stage by stage through its ma_*_set_events hook."""
import ctypes as C
import subprocess

import torch


def stats(xs):
    xs = sorted(xs)
    return {"median": round(xs[len(xs) // 2], 4), "min": round(xs[0], 4), "max": round(xs[-1], 4), "n": len(xs)}


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")[:2]]
    except Exception as e:  # pragma: no cover
        info["power_limit"] = f"unavailable ({type(e).__name__})"
    return info


def stage_times(set_events, stages, call, warmup, repeats):
    """Runs call() warmup + repeats times with the library's stage-timing hook set_events (a ma_*_set_events, which
    takes len(stages) + 1 event handles) on, and the whole call under a second pair of events.  Returns {"total_ms":
    stats, "<stage>_ms": stats per stage} over the repeats."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(stages) + 1)]
    for e in ev:                                               # torch creates the CUDA event at its first record
        e.record()
    handles = (C.c_void_p * len(ev))(*[e.cuda_event for e in ev])
    total, times = [], {s: [] for s in stages}
    for it in range(warmup + repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        set_events(handles)
        a.record()
        call()
        b.record()
        set_events(None)
        b.synchronize()
        if it >= warmup:
            total.append(a.elapsed_time(b))
            for i, s in enumerate(stages):
                times[s].append(ev[i].elapsed_time(ev[i + 1]))
    return {"total_ms": stats(total), **{f"{s}_ms": stats(v) for s, v in times.items()}}
