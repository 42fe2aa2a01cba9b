"""Times the watertight remesh of `--mc` (csrc/watertight.cu) and prints one JSON line.

    python tools/bench_watertight.py [--repeats 10] [--warmup 2] [--out result.json]

Workloads: the reference's wand mesh (tests/golden/wand_mesh.npz) at n = 128, and a seeded synthetic sphere of about
1M faces (an icosahedron, each face split into 224^2 triangles, pushed onto a sphere with smooth seeded noise) at n = 128
and n = 256.  Per workload: the distance field (ma_udf_grid) and marching cubes (count + read-back + emit) under CUDA
events, median / min / max over the repeats after warm-up; the end-to-end mesh_to_pc.export_to_watertight (host
normalisation, upload, both stages, read-back, back-mapping) by host clock; vertex and face counts.  Also the numpy
oracle's host time on the wand at n = 128, for context, and the device name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_common import device_info, stats  # noqa: E402
import mesh_to_pc  # noqa: E402
from meshanything_b200 import capi  # noqa: E402


def icosphere_soup(m=224, seed=0):
    t = (1 + 5 ** 0.5) / 2
    V = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=np.float64)
    F = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11],
                  [6, 2, 10], [8, 6, 7], [9, 8, 1]])
    ii, jj = [a.ravel() for a in np.meshgrid(np.arange(m + 1), np.arange(m + 1), indexing="ij")]
    keep = ii + jj <= m
    ii, jj = ii[keep], jj[keep]
    index = -np.ones((m + 1, m + 1), dtype=np.int64)
    index[ii, jj] = np.arange(len(ii))
    up = [(index[i, j], index[i + 1, j], index[i, j + 1]) for i in range(m) for j in range(m - i)]
    down = [(index[i + 1, j], index[i + 1, j + 1], index[i, j + 1]) for i in range(m) for j in range(m - i - 1)]
    local = np.array(up + down, dtype=np.int64)                      # m^2 triangles per icosahedron face
    verts, faces = [], []
    for f in F:
        a, b, c = V[f]
        p = a + np.outer(ii / m, b - a) + np.outer(jj / m, c - a)
        verts.append(p / np.linalg.norm(p, axis=1, keepdims=True))
        faces.append(local + len(ii) * len(faces))
    v = np.concatenate(verts)
    rng = np.random.RandomState(seed)
    k, ph = rng.uniform(3, 9, (3, 3)), rng.uniform(0, 2 * np.pi, (3, 3))
    noise = sum(np.sin(k[q, 0] * v[:, 0] + ph[q, 0]) * np.sin(k[q, 1] * v[:, 1] + ph[q, 1])
                * np.sin(k[q, 2] * v[:, 2] + ph[q, 2]) for q in range(3))
    return v * (0.8 * (1 + 0.03 * noise))[:, None], np.concatenate(faces)


def _events(fn, warmup, repeats):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def run(name, vertices, faces, n, warmup, repeats):
    dev = torch.device("cuda", 0)
    unit, _, _ = mesh_to_pc.normalize_vertices(vertices)
    v = torch.as_tensor(unit.astype(np.float32), device=dev)
    f = torch.as_tensor(faces.astype(np.int32), device=dev)
    field = capi.udf_grid(v, f, n)
    udf_ms = _events(lambda: capi.udf_grid(v, f, n), warmup, repeats)
    res = {}
    mc_ms = _events(lambda: res.update(out=capi.marching_cubes(field, 2.0 / n)), warmup, repeats)
    mv, mf = res["out"]
    mesh = mesh_to_pc.SimpleMesh(vertices, faces)
    e2e = []
    for i in range(warmup + max(3, repeats // 3)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mesh_to_pc.export_to_watertight(mesh, octree_depth=int(round(np.log2(n))))
        torch.cuda.synchronize()
        if i >= warmup:
            e2e.append((time.perf_counter() - t0) * 1e3)
    return {"workload": name, "n": n, "input_faces": int(len(faces)), "udf_ms": stats(udf_ms),
            "marching_cubes_ms": stats(mc_ms), "export_to_watertight_ms": stats(e2e),
            "out_vertices": int(mv.shape[0]), "out_faces": int(mf.shape[0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_watertight: needs a CUDA device")
    z = np.load(os.path.join(ROOT, "tests", "golden", "wand_mesh.npz"))
    wand_v, wand_f = z["vertices"].astype(np.float64), z["faces"].astype(np.int64)
    sph_v, sph_f = icosphere_soup()
    result = {"bench": "watertight", **device_info(), "results": [
        run("wand", wand_v, wand_f, 128, args.warmup, args.repeats),
        run("sphere_1m", sph_v, sph_f, 128, args.warmup, args.repeats),
        run("sphere_1m", sph_v, sph_f, 256, args.warmup, args.repeats),
    ]}
    if not args.no_oracle:
        from tests import watertight_oracle as W
        unit, _, _ = mesh_to_pc.normalize_vertices(wand_v)
        t0 = time.perf_counter()
        W.marching_cubes(W.udf_grid(unit.astype(np.float32), wand_f, 128), 2.0 / 128)
        result["numpy_oracle_wand_n128_s"] = round(time.perf_counter() - t0, 2)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
