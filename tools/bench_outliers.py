"""Times outlier removal (ma_remove_outliers, csrc/outliers.cu) stage by stage; prints one JSON line.

    python tools/bench_outliers.py [--repeats 10] [--warmup 2] [--out r.json]

Workloads, k = 16, std_ratio 2, min_component 0.01, mapped into the output frame: the wand surface
(tests/golden/wand_mesh.npz, ma_sample_surface) clean at 4096, 100 000 and 1 000 000 points; 1M points of which 1 % are
far outliers drawn uniformly in a box 10x the wand's longest side around it; 1M points of which 20 floater clusters of
500 points each sit 1.5 to 3 wand sizes from its centre.  Per workload and stage -- grid (two histogram passes, the
extent read-back, counting sort, occupied-cell boxes), kNN, statistics (mean distances, mu, sigma, inlier mask),
components (connectivity rounds with their read-backs, sizes, keep mask, compaction) -- CUDA events recorded by the
library between the stages, median / min / max over the repeats after warm-up; the whole call under a second pair of
events; kept points and connectivity rounds.  The ratio of the 1 % outlier cloud's median to the clean 1M cloud's is
the `outlier_over_clean_1M` field.  The device name and power limit are read in the same run.
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

from bench_common import device_info, stage_times  # noqa: E402
from meshanything_b200 import capi, metrics  # noqa: E402

STAGES = ("grid", "knn", "stats", "components")


def cloud(kind, n):
    dev = torch.device("cuda", 0)
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    v, f = torch.from_numpy(z["vertices"]).to(dev), torch.from_numpy(z["faces"]).to(dev)
    g = torch.Generator(device=dev).manual_seed(7)
    m = {"clean": 0, "far": n // 100, "floaters": 20 * 500}[kind]
    xyz = capi.sample_surface(v, f, n - m, seed=5)[:, :3].float()
    lo, hi = xyz.amin(0), xyz.amax(0)
    c, size = (lo + hi) / 2, (hi - lo).max()
    if kind == "far":
        extra = c + (torch.rand(m, 3, device=dev, generator=g) - 0.5) * 10 * size
    elif kind == "floaters":
        d = torch.randn(20, 3, device=dev, generator=g)
        centres = c + d / d.norm(dim=1, keepdim=True) * size * (1.5 + 1.5 * torch.rand(20, 1, device=dev, generator=g))
        extra = (centres[:, None, :] + (torch.rand(20, 500, 3, device=dev, generator=g) - 0.5) * 0.02 * size).reshape(-1, 3)
    else:
        extra = xyz[:0]
    return metrics.to_output_frame(torch.cat([xyz, extra])[None])[0].contiguous()


def workload(kind, n, k, warmup, repeats):
    dev = torch.device("cuda", 0)
    pts = cloud(kind, n)
    ref_idx, ref_keep, ref_st = capi.remove_outliers(pts, k)   # checked call once; the timed calls skip the checks
    L = capi.lib()
    ws = torch.empty(L.ma_remove_outliers_workspace_bytes(n, k), dtype=torch.uint8, device=dev)
    keep = torch.empty((n,), dtype=torch.uint8, device=dev)
    idx = torch.empty((n,), dtype=torch.int64, device=dev)
    nk = torch.empty((1,), dtype=torch.int64, device=dev)
    st = torch.empty((8,), dtype=torch.float64, device=dev)

    def call():
        capi.check(L.ma_remove_outliers(capi.ptr(pts), n, k, C.c_double(2.0), C.c_double(0.01), capi.ptr(keep),
                                        capi.ptr(idx), capi.ptr(nk), None, None, capi.ptr(st), capi.ptr(ws),
                                        capi.stream_ptr()), "ma_remove_outliers")

    times = stage_times(L.ma_remove_outliers_set_events, STAGES, call, warmup, repeats)
    # every stat but the last: the number of connectivity rounds depends on the schedule of the hooking atomics
    assert torch.equal(keep.bool(), ref_keep) and torch.equal(st.cpu()[:7], torch.from_numpy(ref_st[:7]))
    return {"cloud": kind, "N": n, "k": k, **times,
            "kept": int(ref_st[6]), "components": int(ref_st[4]), "components_dropped": int(ref_st[5]),
            "rounds": int(ref_st[7])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_outliers: needs a CUDA device")
    runs = [workload(kind, n, 16, args.warmup, args.repeats)
            for kind, n in (("clean", 4096), ("clean", 100_000), ("clean", 1_000_000), ("far", 1_000_000),
                            ("floaters", 1_000_000))]
    ratio = runs[3]["total_ms"]["median"] / runs[2]["total_ms"]["median"]
    result = {"bench": "outliers", **device_info(), "outlier_over_clean_1M": round(ratio, 3), "runs": runs}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
