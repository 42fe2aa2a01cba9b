"""Times the colour transfer of `--transfer_colors` (ma_transfer_colors, csrc/colors.cu) stage by stage; prints one JSON
line.

    python tools/bench_colors.py [--repeats 10] [--warmup 2] [--out r.json]

Workloads: a latitude-longitude sphere mesh of F = 800 and 1600 faces (the sizes MeshAnything generates) and a scan of
100 000, 1 000 000 and 4 000 000 points on its surface with Gaussian noise of 0.002 of the longest side and random
colours, in the points' frame; and the worst case of the fallback, 1 000 000 points on a sphere ten times the mesh's
size, so that every point is beyond r and every vertex takes its nearest point.  Per workload and stage -- assignment,
accumulation, fallback with the colours -- CUDA events recorded by the library between the stages, median / min / max
over the repeats after warm-up; the whole call under a second pair of events.  Alongside, in the same run: the normal
estimator (ma_estimate_normals, k = 16) on the same points, and a chunked torch restatement of the assignment and the
accumulation (fp32 distances, int64 sums) with its agreement with the kernel.  The device name and power limit are read
in the same run.
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_common import device_info, stage_times, stats  # noqa: E402
from meshanything_b200 import capi  # noqa: E402
from meshanything_b200.colors import DEFAULT_DISTANCE  # noqa: E402

STAGES = ("assign", "accumulate", "fallback")


def sphere_mesh(F, dev):
    """F faces of a latitude-longitude sphere of radius 0.5: (vertices fp32 [V, 3], faces int32 [F, 3])."""
    n = max(3, math.ceil(math.sqrt(F / 2)) + 1)
    th = torch.linspace(0.05, math.pi - 0.05, n, dtype=torch.float64)
    ph = torch.arange(n, dtype=torch.float64) * (2 * math.pi / n)
    th, ph = torch.meshgrid(th, ph, indexing="ij")
    v = 0.5 * torch.stack([th.sin() * ph.cos(), th.sin() * ph.sin(), th.cos()], -1).reshape(-1, 3)
    idx = torch.arange(n * n).reshape(n, n)
    a, b = idx[:-1], torch.roll(idx, -1, 1)[:-1]
    c, d = idx[1:], torch.roll(idx, -1, 1)[1:]
    f = torch.cat([torch.stack([a, b, c], -1).reshape(-1, 3), torch.stack([b, d, c], -1).reshape(-1, 3)])[:F]
    return v.float().to(dev), f.int().to(dev)


def scan(n, radius, dev, sigma=0.002):
    g = torch.Generator(device=dev).manual_seed(7)
    d = torch.randn(n, 3, device=dev, generator=g)
    p = d / d.norm(dim=1, keepdim=True) * radius
    p = p + torch.randn(n, 3, device=dev, generator=g) * (sigma * 2 * radius)
    return p.contiguous(), torch.rand(n, 3, device=dev, generator=g)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _seg2(w, e):
    ll = _dot(e, e)
    t = torch.where(ll > 0, _dot(w, e) / torch.where(ll > 0, ll, torch.ones_like(ll)), torch.zeros_like(ll))
    t = t.clamp(0, 1)
    q = w - t[..., None] * e
    return _dot(q, q)


def torch_transfer(v, f, p, c, r, chunk=1 << 24):
    """The assignment (every point against every face, fp32 distances in separate elementwise ops) and the fixed-point
    sums in int64, chunked over the points; the weights are the kernel's formula's interior case and its nearest
    segment, enough for timing."""
    a, b, cc = v[f[:, 0].long()], v[f[:, 1].long()], v[f[:, 2].long()]
    ab, bc, ca = b - a, cc - b, a - cc
    nrm = torch.cross(ab, cc - a, dim=1)
    nn = _dot(nrm, nrm)
    V = v.shape[0]
    sums = torch.zeros(V * 4, dtype=torch.int64, device=v.device)
    face_all = torch.empty(p.shape[0], dtype=torch.int64, device=v.device)
    step = max(1, chunk // f.shape[0])
    for s in range(0, p.shape[0], step):
        q = p[s:s + step, None, :]
        ap, bp, cp = q - a, q - b, q - cc
        inside = ((nn > 0) & (_dot(torch.cross(ab.expand_as(ap), ap, dim=2), nrm) >= 0)
                  & (_dot(torch.cross(bc.expand_as(bp), bp, dim=2), nrm) >= 0)
                  & (_dot(torch.cross(ca.expand_as(cp), cp, dim=2), nrm) >= 0))
        h = _dot(ap, nrm)
        d2 = torch.where(inside, h * h / torch.where(inside, nn, torch.ones_like(nn)),
                         torch.minimum(torch.minimum(_seg2(ap, ab), _seg2(bp, bc)), _seg2(cp, ca)))
        dist, face = d2.sqrt().min(dim=1)
        face_all[s:s + step] = face
        used = dist <= r
        fq = f[face].long()
        x, y, z = (v[fq[:, k]] for k in range(3))
        nrm_q = nrm[face]
        e = torch.stack([_dot(torch.cross(z - y, p[s:s + step] - y, dim=1), nrm_q),
                         _dot(torch.cross(x - z, p[s:s + step] - z, dim=1), nrm_q),
                         _dot(torch.cross(y - x, p[s:s + step] - x, dim=1), nrm_q)], 1).clamp(min=0)
        w = e / e.sum(1, keepdim=True).clamp(min=1e-30)
        for k in range(3):
            idx = fq[used, k] * 4
            sums.index_add_(0, idx, torch.round(w[used, k] * 2 ** 24).long())
            for ch in range(3):
                sums.index_add_(0, idx + 1 + ch, torch.round(w[used, k] * c[s:s + step][used, ch] * 2 ** 24).long())
    return face_all, sums.view(V, 4)


def timed(fn, warmup, repeats):
    ts = []
    for it in range(warmup + repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        if it >= warmup:
            ts.append(a.elapsed_time(b))
    return stats(ts)


def workload(n, F, warmup, repeats, worst=False):
    dev = torch.device("cuda", 0)
    v, f = sphere_mesh(F, dev)
    p, c = scan(n, 5.0 if worst else 0.5, dev)
    r = DEFAULT_DISTANCE * (10.0 if worst else 1.0)   # r in units of the points' side: the frame is the caller's here
    ref, st, face, _, _, _, _ = capi.transfer_colors(v, f, p, c, r, want_terms=True)   # checked once
    L = capi.lib()
    V = v.shape[0]
    ws = torch.empty(L.ma_transfer_colors_workspace_bytes(V, F, n), dtype=torch.uint8, device=dev)
    out = torch.empty_like(ref)
    stats_dev = torch.empty(3, dtype=torch.int64, device=dev)

    def call():
        capi.check(L.ma_transfer_colors(capi.ptr(v), V, capi.ptr(f), F, capi.ptr(p), capi.ptr(c), n,
                                        capi.C.c_float(r), capi.ptr(out), capi.ptr(stats_dev), None, None, None, None,
                                        None, capi.ptr(ws), capi.stream_ptr()), "ma_transfer_colors")

    times = stage_times(L.ma_transfer_colors_set_events, STAGES, call, warmup, repeats)
    assert torch.equal(out, ref) and stats_dev.cpu().tolist() == st.tolist()
    row = {"mesh": "sphere", "scan": "shell x10" if worst else "surface+noise", "N": n, "F": F, "V": V, **times,
           "stats": st.tolist(), "pairs_per_s": round(n * F / (times["assign_ms"]["median"] * 1e-3), -9)}
    if not worst:
        row["estimate_normals_k16_ms"] = timed(lambda: capi.estimate_normals(p, 16), warmup, repeats)
        if n <= 1_000_000:
            tf, _ = torch_transfer(v, f, p, c, r)
            row["torch_ms"] = timed(lambda: torch_transfer(v, f, p, c, r), 1, 3)
            row["torch_face_agreement"] = float((tf == face.long()).float().mean())
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_colors: needs a CUDA device")
    runs = [workload(n, F, args.warmup, args.repeats) for n in (100_000, 1_000_000, 4_000_000) for F in (800, 1600)]
    runs.append(workload(1_000_000, 800, args.warmup, args.repeats, worst=True))
    result = {"bench": "colors", **device_info(), "runs": runs}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
