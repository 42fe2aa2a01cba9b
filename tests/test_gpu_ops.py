"""-m gpu: the canonical CUDA building blocks against the CPU oracle, bit for bit (through the C ABI)."""
import pytest
import torch

gpu = pytest.mark.gpu


def _dev():
    return torch.device("cuda:0")


@gpu
@pytest.mark.parametrize("M,N,K,epi", [(1, 1024, 1024, 0), (3, 100, 256, 0), (9, 515, 768, 1), (64, 1024, 4096, 0),
                                        (257, 200, 1024, 1), (5, 8195, 1024, 0), (8, 64, 1536, 0)])
def test_linear_bit_exact(M, N, K, epi):
    from meshanything_b200 import capi
    from oracle import decoder as orc
    g = torch.Generator().manual_seed(M * 1000 + N)
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    b = (torch.randn(N, generator=g) * 0.1).half()
    x = torch.randn(M, K, generator=g).half()
    ref = orc.linear(w, b, x, relu=bool(epi))
    got = capi.linear_f16(w.to(_dev()), b.to(_dev()), x.to(_dev()), epilogue=epi).cpu()
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
    ref_nb = orc.linear(w, None, x, relu=False)
    got_nb = capi.linear_f16(w.to(_dev()), None, x.to(_dev())).cpu()
    assert torch.equal(got_nb.view(torch.int16), ref_nb.view(torch.int16))
    # an epilogue outside MA_EPI_NONE / RELU / GELU is refused, not run as a plain Linear
    with pytest.raises(RuntimeError, match="epilogue"):
        capi.linear_f16(w.to(_dev()), b.to(_dev()), x.to(_dev()), epilogue=0x10)


@gpu
def test_linear_gelu_tolerance():
    from meshanything_b200 import capi
    g = torch.Generator().manual_seed(5)
    w = (torch.randn(300, 768, generator=g) * 0.05).half()
    b = (torch.randn(300, generator=g) * 0.1).half()
    x = torch.randn(17, 768, generator=g).half()
    got = capi.linear_f16(w.to(_dev()), b.to(_dev()), x.to(_dev()), epilogue=capi.EPI_GELU).cpu().float()
    pre = (x.double() @ w.double().T + b.double()).half().float()
    ref = torch.nn.functional.gelu(pre)
    assert (got - ref).abs().max() < 4e-3  # fp16 output rounding (1 ulp at |y| < 4)


@gpu
@pytest.mark.parametrize("W", [768, 1024])
def test_layernorm_bit_exact(W):
    from meshanything_b200 import capi
    from oracle import decoder as orc
    g = torch.Generator().manual_seed(W)
    x = torch.randn(11, W, generator=g) * 2
    r = torch.randn(11, W, generator=g).half()
    gamma = 1 + 0.1 * torch.randn(W, generator=g)
    beta = 0.1 * torch.randn(W, generator=g)
    for eps in (1e-5, 1e-12):
        ref32, ref16 = orc.layernorm(x, r, gamma, beta, eps)
        o32, o16 = capi.layernorm(x.to(_dev()), r.to(_dev()), gamma.to(_dev()), beta.to(_dev()), eps)
        assert torch.equal(o32.cpu().view(torch.int32), ref32.view(torch.int32))
        assert torch.equal(o16.cpu().view(torch.int16), ref16.view(torch.int16))
    ref32, _ = orc.layernorm(x, None, gamma, beta, 1e-5)
    o32, _ = capi.layernorm(x.to(_dev()), None, gamma.to(_dev()), beta.to(_dev()), 1e-5)
    assert torch.equal(o32.cpu().view(torch.int32), ref32.view(torch.int32))
    torch_ref = torch.nn.functional.layer_norm(x, (W,), gamma, beta, 1e-5)
    assert (o32.cpu() - torch_ref).abs().max() < 1e-5


@gpu
@pytest.mark.parametrize("H,T,nk", [(16, 300, [1, 2, 31, 32, 33, 255, 256, 257, 300]), (12, 1100, [1100, 513, 1024]),
                                     (2, 4096, [4096])])
def test_attention_bit_exact(H, T, nk):
    from meshanything_b200 import capi
    from oracle import decoder as orc
    g = torch.Generator().manual_seed(T)
    M = len(nk)
    q = torch.randn(M, H, 64, generator=g).half()
    k = torch.randn(H, T, 64, generator=g).half()
    v = torch.randn(H, T, 64, generator=g).half()
    ref = orc.attention(q, k, v, nk)
    d = _dev()
    slots = torch.zeros(M, dtype=torch.int32, device=d)
    nkeys = torch.tensor(nk, dtype=torch.int32, device=d)
    got = capi.attention_f16(q.to(d), k.unsqueeze(0).contiguous().to(d), v.unsqueeze(0).contiguous().to(d), nkeys,
                             slots).cpu()
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
    # and against plain fp32 softmax attention (tolerance: fp16 P and output rounding)
    for m, n in enumerate(nk):
        s = torch.einsum("hd,htd->ht", q[m].float(), k[:, :n].float()) * 0.125
        o = torch.einsum("ht,htd->hd", torch.softmax(s, -1), v[:, :n].float())
        assert (got[m].float() - o).abs().max() < 3e-3


@gpu
def test_attention_at_the_encoder_layout_on_one_scratch():
    """The encoder's use of the canonical attention: 8 shapes x 257 latent rows, 12 heads, slot = row // 257, first over
    the 4096 point keys (16 chunks) and then over 257 keys (2 chunks), both launches on ONE scratch area zeroed once --
    the kernel re-arms its per-(row, head) counters itself.  Sampled rows bit for bit against the oracle."""
    import ctypes
    from meshanything_b200 import capi
    from oracle import decoder as orc
    d = _dev()
    L = capi.lib()
    S, R, H = 8, 257, 12
    M = S * R
    scratch = torch.zeros(L.ma_attention_scratch_bytes(M, H, 4096), dtype=torch.uint8, device=d)
    slots = (torch.arange(M, dtype=torch.int32) // R).to(d)
    g = torch.Generator().manual_seed(257)
    rows = sorted(set([s * R for s in range(S)] + [s * R + R - 1 for s in range(S)]
                      + torch.randperm(M, generator=g)[:64].tolist()))
    for T in (4096, 257):
        q = torch.randn(M, H, 64, generator=g).half()
        k = torch.randn(S, H, T, 64, generator=g).half()
        v = torch.randn(S, H, T, 64, generator=g).half()
        qd, kd, vd = q.to(d), k.to(d), v.to(d)
        nkeys = torch.full((M,), T, dtype=torch.int32, device=d)
        out = torch.empty((M, H, 64), dtype=torch.float16, device=d)
        capi.check(L.ma_attention_f16(capi.ptr(qd), H * 64, capi.ptr(kd), capi.ptr(vd), T, H,
                                      capi.ptr(slots), capi.ptr(nkeys), T, M, ctypes.c_float(0.125), capi.ptr(out),
                                      H * 64, capi.ptr(scratch), capi.stream_ptr()), "ma_attention_f16")
        torch.cuda.synchronize()
        out = out.cpu()
        for s in range(S):
            mine = [m for m in rows if m // R == s]
            ref = orc.attention(q[mine], k[s], v[s], [T] * len(mine))
            assert torch.equal(out[mine].view(torch.int16), ref.view(torch.int16)), (T, s)


@gpu
@pytest.mark.parametrize("T,nk", [(300, [1, 2, 33, 256, 257, 258, 300]), (1100, [1100, 513, 1024, 1025, 7]),
                                  (7500, [7459, 7425, 258, 4096] * 6)])
def test_attention_decode_stream_bit_exact(T, nk):
    """attention_stream_kernel (persistent, pipelined, kv append folded in) against the oracle's canonical attention:
    every cache slot has its own length; the cache row of the current token is poisoned before the call and must hold
    the k / v of the qkv buffer afterwards.  Chunk boundaries (256, 257, 1024, 1025), single-key rows, >= 29 chunks
    (two merge rounds) and more (row, head, chunk) items than one wave of CTAs are all in the cases."""
    from meshanything_b200 import capi
    from oracle import decoder as orc
    g = torch.Generator().manual_seed(T)
    M, H = len(nk), 16
    qkv = torch.randn(M, 3072, generator=g).half()
    k = torch.randn(M, H, T, 64, generator=g).half()
    v = torch.randn(M, H, T, 64, generator=g).half()
    d = _dev()
    kd, vd = k.clone(), v.clone()
    for m, n in enumerate(nk):
        kd[m, :, n - 1] = float("nan")
        vd[m, :, n - 1] = float("nan")
        k[m, :, n - 1] = qkv[m, 1024:2048].view(H, 64)
        v[m, :, n - 1] = qkv[m, 2048:].view(H, 64)
    kd, vd = kd.to(d), vd.to(d)
    nkeys = torch.tensor(nk, dtype=torch.int32, device=d)
    got = capi.attention_decode_f16(qkv.to(d), kd, vd, nkeys).cpu()
    assert torch.equal(kd.cpu().view(torch.int16), k.view(torch.int16))
    assert torch.equal(vd.cpu().view(torch.int16), v.view(torch.int16))
    distinct = {}
    for m, n in enumerate(nk):
        if (n, m % 4) in distinct and M > 8:      # the long case repeats lengths: check each length on a few rows only
            continue
        distinct[(n, m % 4)] = 1
        ref = orc.attention(qkv[m:m + 1, :1024].view(1, H, 64), k[m], v[m], [n])
        assert torch.equal(got[m].view(torch.int16), ref.view(-1).view(torch.int16)), (m, n)
    # a second launch on the same scratch (tickets re-armed) gives the same bits
    again = capi.attention_decode_f16(qkv.to(d), kd, vd, nkeys).cpu()
    assert torch.equal(again.view(torch.int16), got.view(torch.int16))


@gpu
@pytest.mark.parametrize("M,N,K,epi", [(128, 128, 256, 0), (257, 768, 768, 0), (4096, 1536, 768, 0), (130, 128, 256, 1),
                                        (1057, 3072, 768, 2), (300, 768, 3072, 0), (64, 1152, 768, 0)])
def test_linear_tensor_core(M, N, K, epi):
    """wgmma/TMA GEMM (encoder / detokenizer): fp16 in, fp32 accumulate in the hardware's order -> compared with an
    fp64 product rounded once to fp16 (tolerance: one fp16 ulp + fp32 accumulation noise) and with the canonical kernel."""
    from meshanything_b200 import capi
    g = torch.Generator().manual_seed(M + N + K)
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    b = (torch.randn(N, generator=g) * 0.1).half()
    x = torch.randn(M, K, generator=g).half()
    d = _dev()
    got = capi.linear_tc_f16(w.to(d), b.to(d), x.to(d), epilogue=epi).cpu()
    canon = capi.linear_f16(w.to(d), b.to(d), x.to(d), epilogue=epi).cpu()
    pre = x.double() @ w.double().T + b.double()
    if epi == 1:
        pre = torch.relu(pre)
    elif epi == 2:
        pre = torch.nn.functional.gelu(pre.half().double())
    tol = 2.0 ** -10 * pre.abs() + 2e-3
    assert ((got.double() - pre).abs() <= tol).all(), (got.double() - pre).abs().max()
    # same values as the canonical kernel up to the last fp16 bit in a small fraction of the entries
    diff = (got.float() - canon.float()).abs()
    assert (diff <= 2.0 ** -9 * canon.float().abs() + 1e-3).all()
    assert (diff == 0).float().mean() > 0.98


@gpu
@pytest.mark.parametrize("M,N,K,epi", [(1, 1024, 1024, 0), (5, 3072, 1024, 0), (16, 1024, 4096, 0), (33, 4096, 1024, 1),
                                        (64, 1024, 1024, 0), (64, 8195, 1024, 0), (128, 4096, 1024, 1), (100, 768, 3072, 2),
                                        (2, 200, 64, 0)])
@pytest.mark.parametrize("cluster", [1, 0])
def test_linear_weight_streaming_tensor_core(M, N, K, epi, cluster):
    """gemm_ws_kernel (swap-AB wgmma GEMM for M <= 128 rows, K split across CTAs): K slices added over distributed
    shared memory inside a thread-block cluster (cluster = 1, the default) or through L2 with an atomic ticket
    (cluster = 0).  fp16 in, fp32 accumulate in the hardware's order -> compared with an fp64 product rounded once to
    fp16 and with the canonical kernel; two runs give identical bits (the K-slice sum is taken in slice order)."""
    from meshanything_b200 import capi
    capi.lib().ma_linear_ws_set_mode(cluster)
    g = torch.Generator().manual_seed(M * 31 + N + K)
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    b = (torch.randn(N, generator=g) * 0.1).half() if N != 8195 else None       # lm_head has no bias
    x = torch.randn(M, K, generator=g).half()
    d = _dev()
    wd, bd, xd = w.to(d), (b.to(d) if b is not None else None), x.to(d)
    got = capi.linear_ws_f16(wd, bd, xd, epilogue=epi).cpu()
    again = capi.linear_ws_f16(wd, bd, xd, epilogue=epi).cpu()
    assert torch.equal(got.view(torch.int16), again.view(torch.int16))
    pre = x.double() @ w.double().T + (b.double() if b is not None else 0.0)
    if epi == 1:
        pre = torch.relu(pre)
    elif epi == 2:
        pre = torch.nn.functional.gelu(pre.half().double())
    tol = 2.0 ** -10 * pre.abs() + 2e-3
    assert ((got.double() - pre).abs() <= tol).all(), (got.double() - pre).abs().max()
    if K % 256 == 0:
        canon = capi.linear_f16(wd, bd, xd, epilogue=epi).cpu()
        diff = (got.float() - canon.float()).abs()
        assert (diff <= 2.0 ** -9 * canon.float().abs() + 1e-3).all()
        assert (diff == 0).float().mean() > 0.97
    capi.lib().ma_linear_ws_set_mode(1)


def _hf_support(row: torch.Tensor, top_k: int, top_p: float):
    """Support after transformers' own TopKLogitsWarper -> TopPLogitsWarper (the chain HF _sample builds for
    meshanything.py:150-158), evaluated in fp32 on the CPU.  Returns (ids by descending logit, near_boundary)."""
    from transformers.generation.logits_process import TopKLogitsWarper, TopPLogitsWarper
    s = row.float()[None]
    s = TopKLogitsWarper(top_k)(None, s)
    after_k = s.clone()
    if top_p < 1.0:  # generation/utils.py adds the top-p warper only below 1.0
        s = TopPLogitsWarper(top_p)(None, s)
    keep = torch.nonzero(torch.isfinite(s[0]))[:, 0]
    order = sorted(keep.tolist(), key=lambda i: (-float(row[i]), -i))  # reverse of torch's stable ascending sort
    # rows whose ascending cumulative probability passes within 1e-5 of 1 - top_p can flip with summation order
    cum = torch.sort(after_k[0].double()).values.softmax(-1).cumsum(-1)
    near = top_p < 1.0 and bool(((cum - (1 - top_p)).abs() < 1e-5).any())
    return order, near


@gpu
@pytest.mark.parametrize("top_k,top_p", [(50, 0.95), (50, 1.0), (1, 0.95), (128, 0.5), (7, 0.9)])
def test_sampler_support_matches_hf_warpers(top_k, top_p):
    """ma_sample_tokens keeps exactly the tokens HF's warpers keep — including every tie at the k-th value
    (fp16 logits over 8195 ids tie often) — and draws inside that set."""
    from meshanything_b200 import capi
    g = torch.Generator().manual_seed(top_k)
    B, V = 48, 8195
    lg = (torch.randn(B, V, generator=g) * 2.0).half()
    lg[1] = (torch.randn(V, generator=g) * 0.01).half()                  # nearly flat: top-p removes nothing much
    lg[2] = torch.round(torch.randn(V, generator=g) * 2).half()          # heavy ties (integers)
    lg[3] = 0                                                            # everything ties
    lg[3, 77] = 1.0
    lg[4, :] = -3.0
    lg[4, 5:60] = 2.5                                                    # 55 ties at the threshold for k = 50
    lg[5] = (torch.randn(V, generator=g) * 30).half()                    # peaked: one token takes the mass
    lg[6] = -lg[0].abs()                                                 # all non-positive
    tok, sup = capi.sample_tokens(lg.to(_dev()), True, top_k, top_p, seed=3, want_support=True)
    tok, sup = tok.cpu(), sup.cpu()
    checked = 0
    for r in range(B):
        got = [int(v) for v in sup[r] if v >= 0]
        if lg[r].float().ge(torch.topk(lg[r].float(), top_k).values[-1]).sum() > 256:
            continue  # more ties than the kernel's kept-set capacity (row 3): covered below
        want, near = _hf_support(lg[r], top_k, top_p)
        if near:
            continue
        # torch.sort inside TopPLogitsWarper is unstable: which of several EQUAL logits at the top-p boundary
        # survive is undefined in the reference.  Everything else must be identical: the count, the kept
        # values, and every member above the boundary value.
        assert len(got) == len(want), r
        assert [float(lg[r, i]) for i in got] == [float(lg[r, i]) for i in want], r
        edge = float(lg[r, want[-1]])
        assert [i for i in got if float(lg[r, i]) > edge] == [i for i in want if float(lg[r, i]) > edge], r
        n_edge_all = int((lg[r].float() == edge).sum())
        if n_edge_all == sum(1 for i in want if float(lg[r, i]) == edge):
            assert got == want, r                      # no tie was cut: full identity
        assert int(tok[r]) in got
        checked += 1
    assert checked >= B - 6
    # same seed -> same draw; another seed -> another draw somewhere
    tok2 = capi.sample_tokens(lg.to(_dev()), True, top_k, top_p, seed=3).cpu()
    assert torch.equal(tok, tok2)
    if top_k > 1:
        tok3 = capi.sample_tokens(lg.to(_dev()), True, top_k, top_p, seed=4).cpu()
        assert not torch.equal(tok, tok3)
    # greedy = lowest index among the maxima
    am = capi.sample_tokens(lg.to(_dev()), False).cpu()
    for r in range(B):
        m = lg[r].float().max()
        assert int(am[r]) == int(torch.nonzero(lg[r].float() == m)[0, 0])


@gpu
def test_sampler_draw_frequencies():
    """Every row has the same logits and its own Philox stream: empirical frequencies follow the renormalised
    top-k/top-p softmax (5-sigma binomial band)."""
    from meshanything_b200 import capi
    g = torch.Generator().manual_seed(9)
    V, B = 8195, 20000
    row = (torch.randn(V, generator=g) * 1.5).half()
    hf, _ = _hf_support(row, 50, 0.95)
    tok, sup = capi.sample_tokens(row[None].repeat(B, 1).contiguous().to(_dev()), True, 50, 0.95, seed=11,
                                  want_support=True)
    tok = tok.cpu()
    want = [int(v) for v in sup[0].cpu() if v >= 0]
    assert row[want].tolist() == row[hf].tolist()   # same kept values as HF (equal logits at the edge are interchangeable)
    p = torch.softmax(row[want].double(), -1)
    counts = torch.bincount(tok.long(), minlength=V)
    assert int(counts.sum()) == B and int(counts[want].sum()) == B
    f = counts[want].double() / B
    sigma = (p * (1 - p) / B).sqrt()
    assert bool(((f - p).abs() < 5 * sigma + 1e-4).all())


@gpu
@pytest.mark.parametrize("S,rows,n,H", [(2, 257, 4096, 12), (3, 257, 257, 12), (2, 256, 256, 12), (1, 311, 311, 12),
                                        (1, 128, 128, 2), (1, 5, 70, 1)])
def test_attention_tc_vs_fp64(S, rows, n, H):
    """wgmma flash attention (ma_attention_tc_f16) against softmax attention in float64 on the same fp16 inputs.
    Stated tolerance: 2e-3 absolute on outputs of magnitude <= ~1 (P is rounded to fp16 before P.V, as in the canonical
    kernel; accumulation is fp32 in registers).  Also checks the V^T layout kernel bit for bit."""
    from meshanything_b200 import capi
    g = torch.Generator().manual_seed(S * 1000 + n)
    q = (torch.randn(S * rows, H * 64, generator=g) * 1.0).half()
    kv_src = (torch.randn(S * n, 3 * H * 64, generator=g) * 1.0).half()      # [token][q|k|v blocks of H*64]
    k = kv_src[:, H * 64:2 * H * 64].reshape(S, n, H, 64).permute(0, 2, 1, 3).contiguous()   # [S,H,n,64]
    v = kv_src[:, 2 * H * 64:].reshape(S, n, H, 64).permute(0, 2, 1, 3).contiguous()
    vt = capi.transpose_heads_f16(kv_src.to(_dev()), 2 * H * 64, 64, H, n, S)
    Tpad = (n + 127) // 128 * 128
    want_vt = torch.zeros(S, H, 64, Tpad, dtype=torch.float16)
    want_vt[..., :n] = v.transpose(2, 3)
    assert torch.equal(vt.cpu().view(torch.int16), want_vt.view(torch.int16))
    out = capi.attention_tc_f16(q.to(_dev()), k.to(_dev()), vt, n, rows).cpu()
    qd = q.double().reshape(S, rows, H, 64).permute(0, 2, 1, 3)
    att = torch.softmax(qd @ k.double().transpose(2, 3) * 0.125, dim=-1) @ v.double()      # [S,H,rows,64]
    ref = att.permute(0, 2, 1, 3).reshape(S * rows, H * 64)
    err = (out.double() - ref).abs()
    print("attention_tc err max %.3g mean %.3g" % (err.max(), err.mean()))
    assert err.max() < 2e-3
