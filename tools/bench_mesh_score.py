"""Times the best-of-N mesh score (ma_mesh_score, csrc/mesh_score.cu) and, for scale, the sampled generation it ranks;
prints one JSON line.

    python tools/bench_mesh_score.py [--repeats 20] [--warmup 3] [--forward-faces 800] [--no-forward] [--out r.json]

Workloads: S x N = 64 candidates of F = 800 faces against P = 4096-point clouds, as S = 1, N = 64 and as S = 8, N = 8
(random soups in the output frame, every face present).  Per workload: ma_mesh_score under CUDA events, median / min /
max over the repeats after warm-up; the pair evaluations it does (S N P F point-triangle + S N 16 F P point-point) and
their rate; and the kernels' share of the H100 SXM data-sheet FP32 rate (67 TFLOP/s), counting 59 flops per
point-triangle pair (the cheaper, plane branch of the formula) and 8 per point-point pair -- a lower bound on the work,
so the share is one too.  Then one sampled MeshAnything.forward of 64 rows at F = 800 faces (synthetic checkpoint: random
weights never emit EOS, so every row runs the cap) by host clock around a device synchronise.  The device name and power
limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_common import device_info, stats  # noqa: E402
from meshanything_b200 import capi, metrics  # noqa: E402
from meshanything_b200.inputs import synthetic_pc_normal  # noqa: E402

FP32_PEAK = 67e12          # H100 SXM data sheet, dense FP32 (a card allowed up to 700 W)
FLOP_TRI, FLOP_PT = 59, 8


def score_workload(S, N, F, P, warmup, repeats):
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(S * 1000 + N)
    meshes = (torch.rand(S, N, F, 3, 3, generator=g) - 0.5).to(dev)
    cloud = metrics.to_output_frame(synthetic_pc_normal(S, first=0, n_points=P).to(dev))
    terms, faces = capi.mesh_score(meshes, cloud)             # checked call once; the timed calls skip the checks
    L = capi.lib()
    ws = torch.empty(L.ma_mesh_score_workspace_bytes(S, N, F, P), dtype=torch.uint8, device=dev)
    out = torch.empty_like(terms)

    def call():
        capi.check(L.ma_mesh_score(capi.ptr(meshes), capi.ptr(cloud), S, N, F, P, capi.ptr(out), capi.ptr(faces),
                                   None, None, None, None, capi.ptr(ws), capi.stream_ptr()), "ma_mesh_score")

    for _ in range(warmup):
        call()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    assert torch.equal(out, terms)
    tri_pairs, pt_pairs = S * N * P * F, S * N * 16 * F * P
    med = stats(ms)["median"] * 1e-3
    return {"S": S, "N": N, "F": F, "P": P, "mesh_score_ms": stats(ms),
            "point_triangle_pairs": tri_pairs, "point_point_pairs": pt_pairs,
            "pair_evaluations_per_s": round((tri_pairs + pt_pairs) / med, -6),
            "kernel_share_of_fp32_datasheet_rate": round((tri_pairs * FLOP_TRI + pt_pairs * FLOP_PT) / med / FP32_PEAK, 4)}


def forward_workload(B, F):
    from MeshAnything.models.meshanything import MeshAnything
    from meshanything_b200 import checkpoint as ck
    dev = torch.device("cuda", 0)
    sd = ck.synthetic_state_dict(0)
    pc = synthetic_pc_normal(B, first=0).to(dev)
    warm = MeshAnything(argparse.Namespace(codebook_size=8192, codebook_dim=1024, n_max_triangles=4, seed=0))
    warm.load_state_dict(sd, strict=True, device=dev)
    warm(pc, sampling=True)                                  # loads the modules and the encoder / detokenizer paths
    del warm
    model = MeshAnything(argparse.Namespace(codebook_size=8192, codebook_dim=1024, n_max_triangles=F, seed=0))
    model.load_state_dict(sd, strict=True, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = model(pc, sampling=True)
    torch.cuda.synchronize()
    return {"rows": B, "F": F, "sampled_forward_s": round(time.perf_counter() - t0, 3),
            "valid_faces": int((~torch.isnan(out[:, :, 0, 0])).sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--forward-faces", type=int, default=800)
    ap.add_argument("--no-forward", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh_score: needs a CUDA device")
    result = {"bench": "mesh_score", **device_info(),
              "score": [score_workload(1, 64, 800, 4096, args.warmup, args.repeats),
                        score_workload(8, 8, 800, 4096, args.warmup, args.repeats)]}
    if not args.no_forward:
        result["forward"] = forward_workload(64, args.forward_faces)
        result["score_over_forward"] = round(result["score"][0]["mesh_score_ms"]["median"] * 1e-3
                                             / result["forward"]["sampled_forward_s"], 6)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
