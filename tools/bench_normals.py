"""Times the normal estimator of `--input_type pc` (ma_estimate_normals, csrc/normals.cu) stage by stage; prints one
JSON line.

    python tools/bench_normals.py [--repeats 10] [--warmup 2] [--out r.json]

Workloads: N = 4096, 100 000 and 1 000 000 points, k = 16, drawn on the wand surface (tests/golden/wand_mesh.npz,
ma_sample_surface) and on a sphere, mapped into the output frame.  Per workload and stage -- grid build (count, scan,
scatter), kNN, PCA + Jacobi, orientation (weights, Boruvka rounds with their read-backs, root rule) -- CUDA events
recorded by the library between the stages, median / min / max over the repeats after warm-up; the whole call under a
second pair of events; the number of Boruvka rounds.  The device name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from meshanything_b200 import capi, metrics  # noqa: E402

STAGES = ("grid", "knn", "pca", "orient")


def _stats(xs):
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


def cloud(kind, n):
    dev = torch.device("cuda", 0)
    if kind == "wand":
        z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
        v, f = torch.from_numpy(z["vertices"]).to(dev), torch.from_numpy(z["faces"]).to(dev)
        xyz = capi.sample_surface(v, f, n, seed=5)[:, :3].float()
    else:
        x = torch.randn(n, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
        xyz = x / x.norm(dim=1, keepdim=True)
    return metrics.to_output_frame(xyz[None])[0].contiguous()


def workload(kind, n, k, warmup, repeats):
    dev = torch.device("cuda", 0)
    pts = cloud(kind, n)
    ref = capi.estimate_normals(pts, k)                        # checked call once; the timed calls skip the checks
    L = capi.lib()
    ws = torch.empty(L.ma_estimate_normals_workspace_bytes(n, k), dtype=torch.uint8, device=dev)
    out = torch.empty_like(ref)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    for e in ev:                                               # torch creates the CUDA event at its first record
        e.record()
    handles = (C.c_void_p * 5)(*[e.cuda_event for e in ev])
    stages = {s: [] for s in STAGES}
    total, rounds = [], set()
    for it in range(warmup + repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        L.ma_estimate_normals_set_events(handles)
        a.record()
        capi.check(L.ma_estimate_normals(capi.ptr(pts), n, k, capi.ptr(out), None, None, capi.ptr(ws),
                                         capi.stream_ptr()), "ma_estimate_normals")
        b.record()
        L.ma_estimate_normals_set_events(None)
        b.synchronize()
        rounds.add(L.ma_estimate_normals_last_rounds())
        if it >= warmup:
            total.append(a.elapsed_time(b))
            for i, s in enumerate(STAGES):
                stages[s].append(ev[i].elapsed_time(ev[i + 1]))
    assert torch.equal(out, ref)
    return {"cloud": kind, "N": n, "k": k, "total_ms": _stats(total), **{f"{s}_ms": _stats(v) for s, v in stages.items()},
            "boruvka_rounds": sorted(rounds)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_normals: needs a CUDA device")
    result = {"bench": "normals", **device_info(),
              "runs": [workload(kind, n, 16, args.warmup, args.repeats)
                       for kind in ("wand", "sphere") for n in (4096, 100_000, 1_000_000)]}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
