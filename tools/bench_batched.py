"""Per-kernel timings of the BATCHED decode step (configs 3-5: batch 64 per GPU, long context).

    python tools/bench_batched.py [--batch 64]

Times, with CUDA events on the launching stream (20 launches after 5 warm-ups, inputs larger than L2 or rotated):
  * attention_kernel (ma_attention_f16) for B rows x 16 heads at several context lengths -> achieved KV GB/s;
  * the canonical fp32-FMA GEMM (ma_linear_f16), the tiled wgmma GEMM (ma_linear_tc_f16) and the weight-streaming
    wgmma GEMM (ma_linear_ws_f16) at M = B for the five decoder shapes -> us per call, weight GB/s, TFLOP/s.
Prints one JSON object."""
import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from meshanything_b200 import capi  # noqa: E402


def timed(fn, n=20, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n  # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--skip-linear", action="store_true")
    ap.add_argument("--only-keys", type=int, default=0, help="a single context length for the attention part")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    B, H, D = args.batch, 16, 64
    L = capi.lib()
    out = {"batch": B, "attention": [], "linear": []}

    for nk in (() if args.skip_attention else ((args.only_keys,) if args.only_keys else (512, 2048, 4096, 7459))):
        T = nk
        k = torch.randn(B, H, T, D, device=dev, dtype=torch.float16)
        v = torch.randn(B, H, T, D, device=dev, dtype=torch.float16)
        q = torch.randn(B, H, D, device=dev, dtype=torch.float16)
        nkeys = torch.full((B,), nk, dtype=torch.int32, device=dev)
        scratch = torch.zeros(L.ma_attention_scratch_bytes(B, H, nk), dtype=torch.uint8, device=dev)
        o = torch.empty((B, H, D), dtype=torch.float16, device=dev)

        def run():
            capi.check(L.ma_attention_f16(capi.ptr(q), H * D, capi.ptr(k), capi.ptr(v), T, H, None, capi.ptr(nkeys),
                                          nk, B, C.c_float(0.125), capi.ptr(o), H * D, capi.ptr(scratch),
                                          capi.stream_ptr()), "attn")
        us = timed(run)
        nbytes = 2 * B * H * nk * D * 2
        qkv = torch.randn(B, 3072, device=dev, dtype=torch.float16)
        o2 = torch.empty((B, 1024), dtype=torch.float16, device=dev)

        def run_stream():     # attention_stream_kernel: persistent + pipelined, kv append folded in
            capi.check(L.ma_attention_decode_f16(capi.ptr(qkv), 3072, capi.ptr(k), capi.ptr(v), T, capi.ptr(nkeys), nk, B,
                                                 C.c_float(0.125), capi.ptr(o2), 1024, capi.ptr(scratch),
                                                 capi.stream_ptr()), "attn stream")
        us2 = timed(run_stream)
        out["attention"].append({"nkeys": nk, "us": round(us, 2), "kv_MB": round(nbytes / 1e6, 1),
                                 "GBps": round(nbytes / us / 1e3, 1),
                                 "stream": {"us": round(us2, 2), "GBps": round(nbytes / us2 / 1e3, 1)}})
        del k, v

    shapes = [("qkv", 3072, 1024), ("out_proj", 1024, 1024), ("fc1", 4096, 1024), ("fc2", 1024, 4096),
              ("lm_head", 8195, 1024)]
    for name, N, K in (() if args.skip_linear else shapes):
        # 24 distinct weight matrices rotated so that weights come from HBM, as in the layer loop
        ws = [torch.randn(N, K, device=dev, dtype=torch.float16) * 0.02 for _ in range(24)]
        b = torch.zeros(N, device=dev, dtype=torch.float16)
        x = torch.randn(B, K, device=dev, dtype=torch.float16)

        def graph_of(f):  # 24 back-to-back launches in one CUDA graph: no host launch overhead in the timing
            f(ws[0], b, x)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for w in ws:
                    f(w, b, x)
            return g
        rec = {"name": name, "N": N, "K": K}
        for tag, f in (("canon", capi.linear_f16), ("wgmma", capi.linear_tc_f16), ("wgmma_ws", capi.linear_ws_f16),
                       ("wgmma_ws_ticket", capi.linear_ws_f16)):
            L.ma_linear_ws_set_mode(0 if tag == "wgmma_ws_ticket" else 1)
            try:
                g = graph_of(f)
                us = timed(g.replay, n=10, warm=2) / 24
                rec[tag] = {"us": round(us, 2), "weight_GBps": round(N * K * 2 / us / 1e3, 1),
                            "TFLOPs": round(2.0 * B * N * K / us / 1e6, 2)}
            except Exception as e:  # noqa: BLE001
                rec[tag] = {"error": str(e)[:200]}
        out["linear"].append(rec)
    L.ma_linear_ws_set_mode(1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
