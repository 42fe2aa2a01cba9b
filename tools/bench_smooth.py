"""Times the moving-least-squares smoothing of `--smooth` (ma_smooth_points, csrc/smooth.cu) stage by stage; prints one
JSON line.

    python tools/bench_smooth.py [--repeats 10] [--warmup 2] [--out r.json]

Workloads: the wand surface (tests/golden/wand_mesh.npz, ma_sample_surface) with Gaussian noise of 0.002 of the
longest side along random directions, at 100 000, 1 000 000 and 4 000 000 points, at the default k and at k = 64, in
the output frame.  Per workload and stage -- grid build (count, scan, scatter), kNN, fit -- CUDA events recorded by the
library between the stages, median / min / max over the repeats after warm-up; the whole call under a second pair of
events.  Alongside, in the same run: the fit with its threads in index order instead of cell order, the normal
estimator (ma_estimate_normals, k = 16) on the same points, and a chunked torch restatement of the fit (fp64, eigh and
the cyclic Jacobi and torch.linalg's Cholesky) on the same kNN with its largest difference to the kernel.  The device name and power limit
are read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_common import device_info, stage_times, stats  # noqa: E402
from meshanything_b200 import capi, metrics  # noqa: E402
from meshanything_b200.smooth import DEFAULT_K  # noqa: E402

STAGES = ("grid", "knn", "fit")


def cloud(n, sigma=0.002):
    dev = torch.device("cuda", 0)
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    v, f = torch.from_numpy(z["vertices"]).to(dev), torch.from_numpy(z["faces"]).to(dev)
    xyz = capi.sample_surface(v, f, n, seed=5)[:, :3].float()
    g = torch.Generator(device=dev).manual_seed(7)
    d = torch.randn(n, 3, device=dev, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    side = float((xyz.amax(0) - xyz.amin(0)).max())
    xyz = xyz + d * torch.randn(n, 1, device=dev, generator=g) * (sigma * side)
    return metrics.to_output_frame(xyz[None])[0].contiguous()


def torch_jacobi(A, sweeps=5):
    """Eigenvectors (columns of V) of symmetric [C, 3, 3] by the cyclic Jacobi of jacobi3.cuh, batched in torch."""
    A = A.clone()
    V = torch.eye(3, dtype=A.dtype, device=A.device).expand_as(A).clone()
    for _ in range(sweeps):
        for p, q, r in ((0, 1, 2), (0, 2, 1), (1, 2, 0)):
            apq, app, aqq = A[:, p, q], A[:, p, p], A[:, q, q]
            go = apq != 0
            theta = (aqq - app) / torch.where(go, 2 * apq, torch.ones_like(apq))
            t = torch.sign(theta) / (theta.abs() + torch.sqrt(theta * theta + 1))
            t = torch.where(theta == 0, torch.ones_like(t), t)
            t = torch.where(go, t, torch.zeros_like(t))
            c = 1 / torch.sqrt(t * t + 1)
            s = t * c
            arp, arq = A[:, r, p].clone(), A[:, r, q].clone()
            A[:, p, p], A[:, q, q] = app - t * apq, aqq + t * apq
            A[:, p, q] = A[:, q, p] = 0
            A[:, r, p] = A[:, p, r] = c * arp - s * arq
            A[:, r, q] = A[:, q, r] = s * arp + c * arq
            vp, vq = V[:, :, p].clone(), V[:, :, q].clone()
            V[:, :, p], V[:, :, q] = c[:, None] * vp - s[:, None] * vq, s[:, None] * vp + c[:, None] * vq
    return torch.diagonal(A, dim1=1, dim2=2), V


def torch_fit(p, knn, chunk=1 << 18):
    """The fit of DESIGN.md section 1.8 in torch fp64, chunk by chunk (not bit-exact: batched sums, fused ops)."""
    out = torch.empty_like(p)
    P64 = p.double()
    for s in range(0, p.shape[0], chunk):
        i = torch.arange(s, min(s + chunk, p.shape[0]), device=p.device)
        pts = torch.cat([P64[i, None, :], P64[knn[i].long()]], dim=1)                # [C, k+1, 3]
        d2 = ((pts - pts[:, :1]) ** 2).sum(-1)
        H = 2 * d2[:, -1:]
        w = torch.where(H > 0, (1 - d2 / H.clamp_min(1e-300)) ** 2, torch.ones_like(d2))
        w[:, 0] = 1
        m = (w[..., None] * pts).sum(1) / w.sum(1, keepdim=True)
        r = pts - m[:, None]
        cov = torch.einsum("cj,cja,cjb->cab", w, r, r)
        d, V = torch_jacobi(cov)
        order = torch.argsort(d, dim=1, stable=True)                                 # smallest first, lowest on ties
        V = torch.gather(V, 2, order[:, None, :].expand(-1, 3, -1))
        V = V / V.norm(dim=1, keepdim=True)
        n = V[..., 0]
        t1 = torch.where((order[:, 1] < order[:, 2])[:, None], V[..., 1], V[..., 2])
        t2 = torch.where((order[:, 1] < order[:, 2])[:, None], V[..., 2], V[..., 1])
        h = H.sqrt().clamp_min(1e-300)
        u, v, z = (r * t1[:, None]).sum(-1) / h, (r * t2[:, None]).sum(-1) / h, (r * n[:, None]).sum(-1)
        phi = torch.stack([torch.ones_like(u), u, v, u * u, u * v, v * v], -1)      # [C, k+1, 6]
        M = torch.einsum("cj,cja,cjb->cab", w, phi, phi)
        b = torch.einsum("cj,cja,cj->ca", w, phi, z)
        L, info = torch.linalg.cholesky_ex(M)
        a = torch.cholesky_solve(b[..., None], L)[..., 0]
        q = m + (u[:, :1] * h) * t1 + (v[:, :1] * h) * t2 + (phi[:, 0] * a).sum(-1, keepdim=True) * n
        plane = pts[:, 0] - (r[:, 0] * n).sum(-1, keepdim=True) * n
        bad = (info != 0) | (((q - pts[:, 0]) ** 2).sum(-1) > H[:, 0])
        out[i] = torch.where(bad[:, None], plane, q).float()
    return out


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


def workload(n, k, warmup, repeats):
    dev = torch.device("cuda", 0)
    pts = cloud(n)
    ref, st, _, _, knn = capi.smooth_points(pts, k, want_terms=True)   # checked call once; the timed calls skip checks
    L = capi.lib()
    ws = torch.empty(L.ma_smooth_points_workspace_bytes(n, k), dtype=torch.uint8, device=dev)
    out = torch.empty_like(ref)
    stats_dev = torch.empty(3, dtype=torch.int64, device=dev)

    def call():
        capi.check(L.ma_smooth_points(capi.ptr(pts), n, k, capi.ptr(out), None, None, None, capi.ptr(stats_dev),
                                      capi.ptr(ws), capi.stream_ptr()), "ma_smooth_points")

    times = stage_times(L.ma_smooth_points_set_events, STAGES, call, warmup, repeats)
    assert torch.equal(out, ref) and stats_dev.cpu().tolist() == st.tolist()
    L.ma_smooth_points_set_order(0)
    index_order = stage_times(L.ma_smooth_points_set_events, STAGES, call, warmup, repeats)["fit_ms"]
    L.ma_smooth_points_set_order(1)
    assert torch.equal(out, ref)
    row = {"cloud": "wand+noise", "N": n, "k": k, **times, "fit_index_order_ms": index_order,
           "stats": st.tolist()}
    if k == DEFAULT_K:
        row["estimate_normals_k16_ms"] = timed(lambda: capi.estimate_normals(pts, 16), warmup, repeats)
    if n <= 1_000_000:
        tq = torch_fit(pts, knn)
        row["torch_fit_ms"] = timed(lambda: torch_fit(pts, knn), 1, 3)
        row["torch_fit_max_diff"] = float((tq - ref).abs().max())
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_smooth: needs a CUDA device")
    result = {"bench": "smooth", **device_info(),
              "runs": [workload(n, k, args.warmup, args.repeats)
                       for n in (100_000, 1_000_000, 4_000_000) for k in (DEFAULT_K, 64)]}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
