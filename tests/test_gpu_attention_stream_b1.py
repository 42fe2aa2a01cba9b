"""-m gpu: the batch-1 decode attention on attention_stream_kernel.

A batch-1 decode step runs the streaming kernel with M = 1, which the launcher gives its own geometry (one CTA per SM,
a CTA alone on its SM).  Checked bit for bit: the kernel at that geometry against the oracle (output and the appended
cache row), and the whole batch-1 greedy decode on the streaming kernel against the same decode on
kv_append_kernel + attention_kernel (MA_B200_NO_STREAM_ATTN=1), ids and every step's logits.
"""
import ctypes
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

from tests.util import decoder_sd, random_prefix

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = 16


@gpu
@pytest.mark.parametrize("bucket", [False, True])
def test_attention_stream_one_row_bit_exact(bucket):
    """One launch per row with M = 1, as decode_fast.cu launches it, on one cache and one scratch area: rows of 1,
    255-257, 1024 / 1025, 3900 and 7459 keys.  bucket: the launch is sized by the decode loop's 1024-key bucket (3900
    keys -> 16 chunks, 2 per segment; 7459 -> 32 chunks, 4 per segment: several segments per head, merged by the one
    that arrives last), else by the row's own keys.  The cache row of the current token is poisoned before each call and
    must hold the qkv buffer's k / v afterwards; a second launch gives the same bits."""
    from meshanything_b200 import capi
    from oracle import decoder as orc
    L = capi.lib()
    T = 8192
    d = torch.device("cuda:0")
    g = torch.Generator().manual_seed(7459 + int(bucket))
    k = torch.randn(1, H, T, 64, generator=g).half()
    v = torch.randn(1, H, T, 64, generator=g).half()
    kd, vd = k.to(d), v.to(d)
    scratch = torch.zeros(L.ma_attention_scratch_bytes(1, H, T), dtype=torch.uint8, device=d)
    for n in (1, 255, 256, 257, 1024, 1025, 3900, 7459):
        qkv = torch.randn(1, 3072, generator=g).half()
        k[0, :, n - 1] = qkv[0, 1024:2048].view(H, 64)
        v[0, :, n - 1] = qkv[0, 2048:].view(H, 64)
        kd[0, :, n - 1] = float("nan")
        vd[0, :, n - 1] = float("nan")
        max_keys = min(T, (n + 1023) // 1024 * 1024) if bucket else n
        qd = qkv.to(d)
        nkeys = torch.tensor([n], dtype=torch.int32, device=d)
        outs = []
        for _ in range(2):
            out = torch.empty((1, 1024), dtype=torch.float16, device=d)
            capi.check(L.ma_attention_decode_f16(capi.ptr(qd), 3072, capi.ptr(kd), capi.ptr(vd), T, capi.ptr(nkeys),
                                                 max_keys, 1, ctypes.c_float(0.125), capi.ptr(out), 1024,
                                                 capi.ptr(scratch), capi.stream_ptr()), "ma_attention_decode_f16")
            outs.append(out.cpu())
        assert torch.equal(kd[0, :, n - 1].cpu().view(torch.int16), k[0, :, n - 1].view(torch.int16)), n
        assert torch.equal(vd[0, :, n - 1].cpu().view(torch.int16), v[0, :, n - 1].view(torch.int16)), n
        ref = orc.attention(qkv[:, :1024].view(1, H, 64), k[0], v[0], [n])
        assert torch.equal(outs[0].view(torch.int16), ref.view(1, -1).view(torch.int16)), (n, max_keys)
        assert torch.equal(outs[1].view(torch.int16), outs[0].view(torch.int16)), (n, max_keys)
    assert torch.equal(kd.cpu().view(torch.int16), k.view(torch.int16))
    assert torch.equal(vd.cpu().view(torch.int16), v.view(torch.int16))


NL, MAX_NEW = 3, 1100     # 1100 steps: contexts 258..1357 cross the 1024-key bucket boundary


def _b1_greedy():
    from meshanything_b200.decoder import DecoderArena, Generator
    dev = torch.device("cuda:0")
    arena = DecoderArena(decoder_sd(NL), dev)
    ids, lens, logits = Generator(arena, 1, 257 + MAX_NEW).generate(random_prefix(1, seed=11).to(dev), MAX_NEW,
                                                                    eos_id=-1, want_logits=True)
    torch.cuda.synchronize()
    return {"ids": ids[0].cpu().tolist(), "lens": lens.cpu().tolist(),
            "logits_sha256": hashlib.sha256(logits.cpu().view(torch.int16).numpy().tobytes()).hexdigest()}


def _b1_greedy_in_child():
    """Run in a fresh process (see the test below): prints the batch-1 greedy result as JSON."""
    print(json.dumps(_b1_greedy()))


@gpu
def test_b1_greedy_streaming_equals_attention_kernel():
    """Batch-1 greedy decode (3-layer synthetic decoder, 1100 tokens) on attention_stream_kernel equals the same decode
    with MA_B200_NO_STREAM_ATTN=1 (the library reads the variable once when it loads, so in a child process): same
    ids, same fp16 logits at every step."""
    got = _b1_greedy()
    env = dict(os.environ, MA_B200_NO_STREAM_ATTN="1", MA_B200_NO_AUTOBUILD="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "from tests.test_gpu_attention_stream_b1 import _b1_greedy_in_child; _b1_greedy_in_child()"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    child = json.loads(r.stdout.strip().splitlines()[-1])
    assert child["ids"] == got["ids"]
    assert child["lens"] == got["lens"]
    assert child["logits_sha256"] == got["logits_sha256"]
