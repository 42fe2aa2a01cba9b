"""Times farthest-point subsampling (ma_farthest_point_sample, csrc/subsample.cu); prints one JSON line.

    python tools/bench_subsample.py [--repeats 10] [--warmup 2] [--out r.json]

Workloads: M = 4096 picks from the wand surface (tests/golden/wand_mesh.npz, ma_sample_surface) mapped into the output
frame, at N = 8192 and 12 288 (one CTA below kFpsSmallN = 8192 points, a grid above), 100 000, 1 000 000 (the slices in
shared memory on 132 SMs) and 4 000 000 points (beyond shared memory: the slices in global memory).  Per workload: the
call as the library chooses its path, then every path forced where the device can hold it (1 one CTA, 2 grid with
shared-memory slices, 3 grid with global-memory slices), and the torch brute-force loop of tests/subsample_oracle.py
on the same device; CUDA events around each call, median / min / max over the repeats after warm-up.  Every timed
result is checked against the first call, and that against the brute force, bit for bit.  The device name and power
limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_common import device_info, stats  # noqa: E402
from meshanything_b200 import capi, metrics  # noqa: E402
from tests.subsample_oracle import torch_bruteforce  # noqa: E402

M = 4096
PATHS = {1: "one_cta", 2: "grid_shared", 3: "grid_global"}


def wand(n):
    dev = torch.device("cuda", 0)
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    v, f = torch.from_numpy(z["vertices"]).to(dev), torch.from_numpy(z["faces"]).to(dev)
    xyz = capi.sample_surface(v, f, n, seed=5)[:, :3].float()
    return metrics.to_output_frame(xyz[None])[0].contiguous()


def _time(fn, warmup, repeats):
    out, times = None, []
    for it in range(warmup + repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        if it >= warmup:
            times.append(a.elapsed_time(b))
    return out, stats(times)


def workload(n, warmup, repeats):
    dev = torch.device("cuda", 0)
    pts = wand(n)
    start = n // 3
    ref_idx, ref_r2 = capi.farthest_point_sample(pts, M, start)   # checked call once; the timed calls skip the checks
    L = capi.lib()
    ws = torch.empty(L.ma_farthest_point_sample_workspace_bytes(n, M), dtype=torch.uint8, device=dev)
    idx = torch.empty((M,), dtype=torch.int64, device=dev)
    r2 = torch.empty((M,), dtype=torch.float32, device=dev)

    def call():
        capi.check(L.ma_farthest_point_sample(capi.ptr(pts), n, M, start, capi.ptr(idx), capi.ptr(r2), capi.ptr(ws),
                                              capi.stream_ptr()), "ma_farthest_point_sample")

    def same():
        return torch.equal(idx, ref_idx) and torch.equal(r2.view(torch.int32), ref_r2.view(torch.int32))

    _, auto = _time(call, warmup, repeats)
    assert same()
    run = {"N": n, "M": M, "path": PATHS[L.ma_farthest_point_sample_last_path()], "fps_ms": auto}
    for p, name in PATHS.items():
        prev = L.ma_farthest_point_sample_set_path(p)
        try:
            if L.ma_farthest_point_sample(capi.ptr(pts), n, M, start, capi.ptr(idx), capi.ptr(r2), capi.ptr(ws),
                                          capi.stream_ptr()) != 0:
                run[f"{name}_ms"] = "cannot run: " + L.ma_last_error().decode()
                continue
            _, run[f"{name}_ms"] = _time(call, warmup, repeats)
            assert same(), name
        finally:
            L.ma_farthest_point_sample_set_path(prev)
    (bidx, br2), run["torch_bruteforce_ms"] = _time(lambda: torch_bruteforce(pts, M, start), 1, repeats)
    assert torch.equal(bidx, ref_idx) and torch.equal(br2.view(torch.int32), ref_r2.view(torch.int32))
    run["speedup_over_torch"] = round(run["torch_bruteforce_ms"]["median"] / auto["median"], 1)
    run["per_pick_us"] = round(1000 * auto["median"] / M, 3)
    run["covering_radius"] = round(float(ref_r2[-1].sqrt()), 5)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_subsample: needs a CUDA device")
    runs = [workload(n, args.warmup, args.repeats) for n in (8192, 12_288, 100_000, 1_000_000, 4_000_000)]
    result = {"bench": "subsample", **device_info(), "sms": torch.cuda.get_device_properties(0).multi_processor_count,
              "runs": runs}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
