"""Times object splitting (ma_split_objects, csrc/objects.cu) stage by stage; prints one JSON line.

    python tools/bench_objects.py [--repeats 10] [--warmup 2] [--out r.json]

Workloads, all mapped into the output frame:
  scene  eight objects -- four copies of the wand surface (tests/golden/wand_mesh.npz, ma_sample_surface) and four
         sphere surfaces, each of longest side 0.3 -- on a 4 x 2 layout 0.6 apart, with 1 % of the points as strays
         scattered in a cube as wide as the layout, none within 0.1 of an object (so they never bridge two objects,
         and they are sparse enough not to chain into a cluster of 4096); 100k, 1M and 4M points at e = 0.02 and
         0.005 of the longest side.
  dense  full cells: 1M points uniform in five balls of radius e = 0.1 whose centres lie 0.4 apart, so that
         neighbouring cells hold thousands of points each.
  sheets the slow case of the pair tests: 1M points on two parallel square sheets tilted to the normal (1, 1, 1) / sqrt 3,
         1.5 e apart at e = 0.1.  The cell boxes across the gap overlap in every axis, so the box tests cannot rule a
         pair of cells out, and with no pair within e every point pair of those cells is tested.
Per workload and stage -- grid (box, cell keys, sort, occupied cells), connectivity (clique cells, pair tests, labels
and sizes), order and selection -- CUDA events recorded by the library between the stages, median / min / max over
the repeats after warm-up; the whole call under a second pair of events.  At 100k points a chunked torch brute force
on the same GPU (every pair's fp32 d^2 in separate elementwise ops, then min-label propagation with pointer jumping
over the edges) is timed once after a warm-up, and its component count is checked equal.  The device name and power
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

from bench_common import device_info, stage_times  # noqa: E402
from meshanything_b200 import capi, metrics  # noqa: E402

STAGES = ("grid", "connectivity", "order")


def scene(n):
    """Eight objects and 1 % strays in the output frame: fp32 [n, 3] on the GPU."""
    dev = torch.device("cuda", 0)
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    v, f = torch.from_numpy(z["vertices"]).to(dev), torch.from_numpy(z["faces"]).to(dev)
    g = torch.Generator(device=dev).manual_seed(7)
    n_str = n // 100
    per = (n - n_str) // 8
    parts = []
    for k in range(8):
        m = per if k < 7 else n - n_str - 7 * per
        if k % 2 == 0:
            o = capi.sample_surface(v, f, m, seed=5 + k)[:, :3].float()
            lo, hi = o.amin(0), o.amax(0)
            o = (o - (lo + hi) / 2) / (hi - lo).max() * 0.3
        else:
            o = torch.randn(m, 3, device=dev, generator=g)
            o = o / o.norm(dim=1, keepdim=True) * 0.15
        parts.append(o + torch.tensor([0.6 * (k % 4), 0.6 * (k // 4), 0.0], device=dev))
    pts = torch.cat(parts)
    lo, hi = pts.amin(0), pts.amax(0)
    side = float((hi - lo).max())
    centres = torch.tensor([[0.6 * (k % 4), 0.6 * (k // 4), 0.0] for k in range(8)], device=dev)
    strays = torch.zeros(0, 3, device=dev)
    while len(strays) < n_str:                                 # every object lies within 0.26 of its centre
        s = (lo + hi) / 2 + (torch.rand(n_str, 3, device=dev, generator=g) - 0.5) * side
        strays = torch.cat([strays, s[torch.cdist(s, centres).amin(1) > 0.36]])[:n_str]
    parts.append(strays)
    return metrics.to_output_frame(torch.cat(parts)[None])[0].contiguous()


def dense(n, e):
    """n points uniform in five balls of radius e, centres 0.4 apart, plus the frame's corners."""
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(11)
    x = torch.randn(n - 2, 3, device=dev, generator=g)
    r = e * torch.rand(n - 2, 1, device=dev, generator=g) ** (1 / 3)
    c = torch.tensor([[-0.4, 0, 0], [0, 0, 0], [0.4, 0, 0], [0, 0.4, 0], [0, -0.4, 0]], device=dev)
    pts = x / x.norm(dim=1, keepdim=True) * r + c[torch.arange(n - 2, device=dev) % 5]
    corners = torch.tensor([[-0.5, -0.5, -0.5], [0.5, 0.5, 0.5]], device=dev)
    return torch.cat([corners, pts]).contiguous()


def sheets(n, e):
    """n points on two parallel unit squares with normal (1, 1, 1) / sqrt 3, 1.5 e apart, in the output frame."""
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(13)
    nrm = torch.tensor([1.0, 1.0, 1.0], device=dev) / 3 ** 0.5
    u = torch.tensor([1.0, -1.0, 0.0], device=dev) / 2 ** 0.5
    v = torch.linalg.cross(nrm, u)
    ab = torch.rand(n, 2, device=dev, generator=g) - 0.5
    side = (torch.arange(n, device=dev) % 2).float()[:, None] * 1.5 * e
    pts = ab[:, :1] * u + ab[:, 1:] * v + side * nrm
    return metrics.to_output_frame(pts[None])[0].contiguous()


def torch_components(pts, e, chunk=2048):
    """Components of the graph d^2 <= fp32(e e) by brute force: every pair's fp32 d^2 (separate elementwise ops), the
    edges, then min-label propagation with pointer jumping until nothing changes."""
    n = len(pts)
    e2 = float(np.float32(np.float32(e) * np.float32(e)))
    src, dst = [], []
    for s in range(0, n, chunk):
        q = pts[s:s + chunk]
        dx = q[:, None, 0] - pts[None, :, 0]
        dy = q[:, None, 1] - pts[None, :, 1]
        dz = q[:, None, 2] - pts[None, :, 2]
        a = dx * dx
        b = dy * dy
        c = dz * dz
        i, j = ((a + b) + c <= e2).nonzero(as_tuple=True)
        src.append(i + s)
        dst.append(j)
    src, dst = torch.cat(src), torch.cat(dst)
    lab = torch.arange(n, device=pts.device)
    while True:
        new = lab.scatter_reduce(0, src, lab[dst], reduce="amin")
        new = new[new]
        if torch.equal(new, lab):
            break
        lab = new
    return int((lab == torch.arange(n, device=pts.device)).sum())


def workload(name, pts, e, warmup, repeats, brute):
    dev = torch.device("cuda", 0)
    n, mp = len(pts), 4096
    ref_lab, ref_idx, ref_off, ref_st = capi.split_objects(pts, e, mp)
    L = capi.lib()
    ws = torch.empty(L.ma_split_objects_workspace_bytes(n, mp), dtype=torch.uint8, device=dev)
    lab = torch.empty((n,), dtype=torch.int32, device=dev)
    idx = torch.empty((n,), dtype=torch.int64, device=dev)
    off = torch.empty((n // mp + 1,), dtype=torch.int64, device=dev)
    st = torch.empty((6,), dtype=torch.int64, device=dev)

    def call():
        capi.check(L.ma_split_objects(capi.ptr(pts), n, C.c_float(np.float32(e)), mp, capi.ptr(lab), capi.ptr(idx),
                                      capi.ptr(off), capi.ptr(st), capi.ptr(ws), capi.stream_ptr()), "ma_split_objects")

    times = stage_times(L.ma_split_objects_set_events, STAGES, call, warmup, repeats)
    assert torch.equal(lab, ref_lab) and torch.equal(st.cpu(), torch.from_numpy(ref_st))
    out = {"workload": name, "N": n, "e": e, **times, "clusters": int(ref_st[0]), "objects": int(ref_st[1]),
           "object_sizes": np.diff(ref_off.cpu().numpy()).tolist(), "dropped_points": int(ref_st[4])}
    if brute:
        torch_components(pts[:4096], e)                        # warm-up
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        comps = torch_components(pts, e)
        b.record()
        b.synchronize()
        assert comps == int(ref_st[0]), (comps, int(ref_st[0]))
        out["torch_brute_force_ms"] = round(a.elapsed_time(b), 2)
        out["torch_over_kernel"] = round(out["torch_brute_force_ms"] / out["total_ms"]["median"], 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_objects: needs a CUDA device")
    runs = []
    for n in (100_000, 1_000_000, 4_000_000):
        pts = scene(n)
        for e in (0.02, 0.005):
            runs.append(workload("scene", pts, e, args.warmup, args.repeats, brute=n == 100_000))
    runs.append(workload("dense", dense(1_000_000, 0.1), 0.1, args.warmup, args.repeats, brute=False))
    runs.append(workload("sheets", sheets(1_000_000, 0.1), 0.1, args.warmup, args.repeats, brute=False))
    result = {"bench": "objects", **device_info(), "min_points": 4096, "runs": runs}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
