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
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_common import device_info, stage_times  # noqa: E402
from meshanything_b200 import capi, metrics  # noqa: E402

STAGES = ("grid", "knn", "pca", "orient")


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
    rounds = set()

    def call():
        capi.check(L.ma_estimate_normals(capi.ptr(pts), n, k, capi.ptr(out), None, None, capi.ptr(ws),
                                         capi.stream_ptr()), "ma_estimate_normals")
        rounds.add(L.ma_estimate_normals_last_rounds())

    times = stage_times(L.ma_estimate_normals_set_events, STAGES, call, warmup, repeats)
    assert torch.equal(out, ref)
    return {"cloud": kind, "N": n, "k": k, **times, "boruvka_rounds": sorted(rounds)}


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
