"""Times support-plane removal (ma_remove_plane, csrc/plane.cu) stage by stage; prints one JSON line.

    python tools/bench_plane.py [--repeats 10] [--warmup 2] [--out r.json]

Workload: the wand surface (tests/golden/wand_mesh.npz, ma_sample_surface) scaled to a longest side of 1 and standing
on a table disc three wand-lengths across that holds 60 % of the points (Gaussian noise 0.2 t in its normal, t = 0.01 of
the scene's longest side), with 10 % of the points on four legs below it; mapped into the output frame.  Sizes 100k,
1M and 4M points at H = 1000 hypotheses, and 1M at H = 4096; t = 0.01.  Per workload and stage -- hypotheses, scoring
(with the winner), refit (centroid, moments, Jacobi), classification with the compaction -- CUDA events recorded by the
library between the stages, median / min / max over the repeats after warm-up; the whole call under a second pair of
events; point-plane tests per second of the scoring stage (N H over its median); the chunked torch restatement of the
scoring (separate elementwise ops, 16 planes per chunk) timed the same way on the same GPU, with its counts checked
equal.  The device name and power limit are read in the same run.
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

from bench_common import device_info, stage_times, stats  # noqa: E402
from meshanything_b200 import capi, metrics  # noqa: E402

STAGES = ("hypotheses", "scoring", "refit", "classify")


def scene(n):
    """The wand on a noisy table disc with legs, in the output frame: fp32 [n, 3] on the GPU."""
    dev = torch.device("cuda", 0)
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    v, f = torch.from_numpy(z["vertices"]).to(dev), torch.from_numpy(z["faces"]).to(dev)
    g = torch.Generator(device=dev).manual_seed(7)
    n_tab, n_leg = int(0.6 * n), n // 10
    wand = capi.sample_surface(v, f, n - n_tab - n_leg, seed=5)[:, :3].float()
    lo, hi = wand.amin(0), wand.amax(0)
    wand = (wand - lo) / (hi - lo).max()
    wand[:, :2] -= wand[:, :2].mean(0)
    t = 0.01 * 3.0
    r = 1.5 * torch.rand(n_tab, device=dev, generator=g).sqrt()
    a = torch.rand(n_tab, device=dev, generator=g) * 2 * np.pi
    tab = torch.stack([r * a.cos(), r * a.sin(), torch.randn(n_tab, device=dev, generator=g) * 0.2 * t], dim=1)
    corner = torch.tensor([[1, 1], [1, -1], [-1, 1], [-1, -1]], dtype=torch.float32, device=dev) * 0.9
    leg = torch.cat([corner[torch.randint(4, (n_leg,), device=dev, generator=g)],
                     -3 * t - torch.rand(n_leg, 1, device=dev, generator=g) * 1.1], dim=1)
    return metrics.to_output_frame(torch.cat([tab, wand, leg])[None])[0].contiguous()


def torch_counts(pts, planes, t):
    px, py, pz = pts[:, 0], pts[:, 1], pts[:, 2]
    out = torch.empty(len(planes), dtype=torch.int64, device=pts.device)
    for s in range(0, len(planes), 16):
        pl = planes[s:s + 16]
        a = pl[:, 0:1] * px
        b = pl[:, 1:2] * py
        c = pl[:, 2:3] * pz
        out[s:s + 16] = ((((a + b) + c) + pl[:, 3:4]).abs() <= t).sum(dim=1)
    return out


def workload(n, h, warmup, repeats, torch_repeats):
    dev = torch.device("cuda", 0)
    pts = scene(n)
    t, seed = 0.01, 12345
    ref_idx, ref_keep, ref_st, ref_counts, ref_planes = capi.remove_plane(pts, t, h, seed, want_terms=True)
    L = capi.lib()
    ws = torch.empty(L.ma_remove_plane_workspace_bytes(n, h), dtype=torch.uint8, device=dev)
    keep = torch.empty((n,), dtype=torch.uint8, device=dev)
    idx = torch.empty((n,), dtype=torch.int64, device=dev)
    nk = torch.empty((1,), dtype=torch.int64, device=dev)
    st = torch.empty((12,), dtype=torch.float64, device=dev)

    def call():
        capi.check(L.ma_remove_plane(capi.ptr(pts), n, h, C.c_float(t), seed, capi.ptr(keep), capi.ptr(idx),
                                     capi.ptr(nk), None, None, capi.ptr(st), capi.ptr(ws), capi.stream_ptr()),
                   "ma_remove_plane")

    times = stage_times(L.ma_remove_plane_set_events, STAGES, call, warmup, repeats)
    assert torch.equal(keep.bool(), ref_keep) and torch.equal(st.cpu(), torch.from_numpy(ref_st))
    tt = []
    for it in range(1 + torch_repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        tc = torch_counts(pts, ref_planes, t)
        b.record()
        b.synchronize()
        if it:
            tt.append(a.elapsed_time(b))
    assert torch.equal(tc, ref_counts.long())
    score = times["scoring_ms"]
    return {"N": n, "H": h, **times,
            "tests_per_s": float(f"{n * h / (score['median'] * 1e-3):.4g}"), "torch_scoring_ms": stats(tt),
            "torch_over_kernel_scoring": round(stats(tt)["median"] / score["median"], 1),
            "found": bool(ref_st[0]), "winner_count": int(ref_st[6]), "on": int(ref_st[8]), "above": int(ref_st[9]),
            "below": int(ref_st[10]), "kept": int(ref_st[11])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--torch_repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_plane: needs a CUDA device")
    runs = [workload(n, h, args.warmup, args.repeats, args.torch_repeats)
            for n, h in ((100_000, 1000), (1_000_000, 1000), (1_000_000, 4096), (4_000_000, 1000))]
    result = {"bench": "plane", **device_info(), "t": 0.01, "runs": runs}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
