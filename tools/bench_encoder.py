"""Encoder / detokenizer stage timings under the three kernel selections of ma_set_tensor_cores (0: canonical CUDA-core
kernels, 1: wgmma GEMMs, 2: wgmma GEMMs + wgmma attention).  CUDA events, 5 timed runs after 2 warm-ups.

    python tools/bench_encoder.py [--batch 8] [--faces 800]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from meshanything_b200 import capi, checkpoint as ck  # noqa: E402
from meshanything_b200.encoder import EncoderArena, TokenizerArena  # noqa: E402
from meshanything_b200.inputs import synthetic_pc_normal  # noqa: E402


def timed(fn, n=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--faces", type=int, default=800)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    sd = ck.make_state_dict(ck.all_specs(1), 0)          # decoder depth is irrelevant here
    enc, tok = EncoderArena(sd, dev), TokenizerArena(sd, dev)
    pc = synthetic_pc_normal(args.batch, first=0).to(dev)
    F = args.faces
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(3, 8195, (args.batch, 9 * F + 2), generator=g, dtype=torch.int32).to(dev)
    pf, _ = enc.forward(pc)
    out = {"batch": args.batch, "faces": F, "modes": {}}
    # useful flops per shape (SURVEY.md section 8(d)): encoder ~108 GFLOP, detokenizer 6 BERT layers over 257+F tokens
    S = 257 + F
    det_flop = 6 * (2 * S * 768 * (3 * 768 + 768 + 2 * 3072) + 4 * S * S * 768) + 2 * F * 3072 * 768 + 2 * F * 768 * 1152
    for mode in (0, 1, 2):
        old = capi.lib().ma_set_tensor_cores(mode)
        try:
            t_enc = timed(lambda: enc.forward(pc))
            t_det = timed(lambda: tok.detokenize(ids, pf, F))
        finally:
            capi.lib().ma_set_tensor_cores(old)
        out["modes"][str(mode)] = {"encoder_ms": round(t_enc, 3), "detokenizer_ms": round(t_det, 3),
                                   "encoder_TFLOPs": round(108e9 * args.batch / t_enc / 1e9, 1),
                                   "detokenizer_TFLOPs": round(det_flop * args.batch / t_det / 1e9, 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
