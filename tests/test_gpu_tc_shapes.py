"""-m gpu: the tensor-core kernels and the stages built on them, at the shapes the batched and best-of-N runs use.

  A  gemm_ws_kernel (ma_linear_ws_f16): every tile width MP = 16 / 32 / 64 / 128 on both sides of its boundary, every
     K-slice count the cluster reduction selects (1, 2, 4, 8) and the ticket reduction with more than one slice, the
     five decoder matrices, strided x and y, and nothing written outside [0, M) x [0, N);
  B  gemm_tc_kernel (ma_linear_tc_f16): fewer k-blocks than pipeline stages, ragged row tiles, no bias, the encoder's
     strided pre_kl call and its 32768-row input_proj / c_kv calls; the canonical kernel on cond_head_proj's gathered rows;
  C  attention_tc_kernel at the detokenizer's 1057 and 1857 tokens, and keys beyond nkeys masked by selection;
  D  the decoder with tensor-core GEMMs at batch 17 / 32 / 64 / 100 in both reduction modes, graph runs against eager
     runs, and the slot engine after the weights behind its DecoderWeights struct changed;
  E  the encoder and the detokenizer across their 8-shape chunks.

GEMM and attention references are float64 computations on the same fp16 inputs; they run on the device so that every
row of the large shapes is checked.  Tolerances are those of DESIGN.md section 6.
"""
import ctypes as C
import zlib

import pytest
import torch

from tests.util import decoder_sd, random_prefix

gpu = pytest.mark.gpu

SENTINEL = 0x7E5A          # an fp16 quiet-NaN bit pattern that no kernel produces: marks memory a call must not write
NAN16 = float("nan")


def _dev():
    return torch.device("cuda:0")


def _seed(*parts) -> int:
    return zlib.crc32(repr(parts).encode())


def _sentinel_out(M: int, N: int, ldy: int, extra_rows: int = 3):
    """(whole buffer [M + extra_rows, ldy] filled with SENTINEL, the [M, N] view a GEMM writes with ldy)."""
    buf = torch.full((M + extra_rows, ldy), SENTINEL, dtype=torch.int16, device=_dev()).view(torch.float16)
    return buf, buf[:M, :N]


def _assert_outside_untouched(buf: torch.Tensor, M: int, N: int, what):
    b = buf.view(torch.int16)
    assert bool((b[M:] == SENTINEL).all()) and bool((b[:M, N:] == SENTINEL).all()), f"{what}: wrote outside [0,M)x[0,N)"


def _strided_x(x: torch.Tensor, ldx: int) -> torch.Tensor:
    """x [M, K] as the first K columns of a [M, ldx] buffer whose other columns are NaN."""
    M, K = x.shape
    if ldx == K:
        return x.contiguous()
    buf = torch.full((M, ldx), NAN16, dtype=torch.float16, device=x.device)
    buf[:, :K] = x
    return buf[:, :K]


def _ref_linear(x: torch.Tensor, w: torch.Tensor, b, epi: int = 0) -> torch.Tensor:
    """float64 x @ w.T + b (ReLU for epi 1), on the device of x."""
    ref = x.double() @ w.double().T
    if b is not None:
        ref += b.double()
    if epi == 1:
        ref = torch.relu(ref)
    return ref


def _same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _check_tol(got: torch.Tensor, ref: torch.Tensor, what):
    """|y - ref| <= 2^-10 |ref| + 2e-3 (one fp16 rounding + fp32 accumulation noise).
    Returns (largest |y - ref|, largest |y - ref| / tolerance)."""
    err = (got.double() - ref).abs()
    tol = 2.0 ** -10 * ref.abs() + 2e-3
    ok = err <= tol
    assert bool(ok.all()), (what, float(err.max()), int((~ok).sum()))
    return float(err.max()), float((err / tol).max())


def _report(group: str, what, value, tol):
    """One line per case (pytest -s): the largest error and the tolerance it is held to."""
    if isinstance(value, tuple):
        value = "%.4g (%.2f of the tolerance)" % value
    else:
        value = "%.4g" % value
    print(f"[tc-shapes {group}] {what}: max err {value}; tolerance {tol}")


def _worst(a, b):
    return (max(a[0], b[0]), max(a[1], b[1]))


# ------------------------------------------------------------------------------------------------------------------ A
# name: (N, K, epilogue, bias).  K slices (cluster mode / ticket mode) from launch_linear_ws's selection:
WS_SHAPES = {
    "qkv": (3072, 1024, 0, True),         # 24 row tiles: cluster 4, ticket 1
    "out_proj": (1024, 1024, 0, True),    # 8 row tiles: cluster 8, ticket 4
    "fc1": (4096, 1024, 1, True),         # 32 row tiles: cluster 2, ticket 1
    "fc2": (1024, 4096, 0, True),         # 8 row tiles: cluster 8, ticket 4
    "lm_head": (8195, 1024, 0, False),    # 65 row tiles, no bias: cluster 2, ticket 1
    "k128": (1024, 128, 0, True),         # 2 k-blocks: cluster 1, ticket 2
    "n8449": (8449, 1024, 0, True),       # 67 row tiles: cluster 1, ticket 1
}
M_ALL = [1, 15, 16, 17, 24, 31, 32, 33, 63, 64, 65, 100, 127, 128]
M_EDGE = [1, 16, 17, 32, 33, 64, 65, 128]    # both sides of every MP boundary (16 / 32 / 64 / 128)
WS_CASES = [(s, m) for s in WS_SHAPES for m in (M_ALL if s in ("out_proj", "lm_head") else M_EDGE)]


@pytest.fixture(scope="module")
def ws_operands():
    """Per shape: w, bias, 128 rows of x on the device and the float64 reference of all 128 rows (M rows = a prefix)."""
    cache = {}

    def get(name):
        if name not in cache:
            N, K, epi, has_bias = WS_SHAPES[name]
            g = torch.Generator().manual_seed(_seed("ws", name))
            w = (torch.randn(N, K, generator=g) * 0.05).half().to(_dev())
            b = (torch.randn(N, generator=g) * 0.1).half().to(_dev()) if has_bias else None
            x = torch.randn(128, K, generator=g).half().to(_dev())
            cache[name] = (w, b, x, _ref_linear(x, w, b, epi))
        return cache[name]

    yield get
    cache.clear()


@gpu
@pytest.mark.parametrize("shape,M", WS_CASES)
def test_gemm_ws_tile_widths_and_k_slices(ws_operands, shape, M):
    """gemm_ws_kernel in both reduction modes against the float64 product: dense, padded (ldx = K + 64, ldy = N + 8) and
    odd-ldy (scalar store) layouts give identical bits and leave every element outside [0, M) x [0, N) alone; two calls
    give identical bits; where K % 256 == 0, >= 97 % of the values equal the canonical kernel's bit for bit."""
    from meshanything_b200 import capi
    N, K, epi, _ = WS_SHAPES[shape]
    w, b, x_all, ref_all = ws_operands(shape)
    x, ref = x_all[:M], ref_all[:M]
    layouts = [(K, N), (K + 64, N + 8), (K + 64, 8195 if N < 8195 else N + 2)]
    worst = (0.0, 0.0)
    try:
        for cluster in (1, 0):
            capi.lib().ma_linear_ws_set_mode(cluster)
            first = None
            for ldx, ldy in layouts:
                buf, out = _sentinel_out(M, N, ldy)
                capi.linear_ws_f16(w, b, _strided_x(x, ldx), epilogue=epi, out=out)
                _assert_outside_untouched(buf, M, N, (shape, M, cluster, ldx, ldy))
                worst = _worst(worst, _check_tol(out, ref, (shape, M, cluster, ldx, ldy)))
                if first is None:
                    first = out.clone()
                else:
                    assert _same_bits(out, first), (shape, M, cluster, ldx, ldy)
            again = capi.linear_ws_f16(w, b, x, epilogue=epi)
            assert _same_bits(again, first), (shape, M, cluster, "second call")
            if K % 256 == 0:
                canon = capi.linear_f16(w, b, x, epilogue=epi).float()
                diff = (first.float() - canon).abs()
                assert bool((diff <= 2.0 ** -9 * canon.abs() + 1e-3).all()), (shape, M, cluster)
                assert float((diff == 0).float().mean()) > 0.97, (shape, M, cluster)
    finally:
        capi.lib().ma_linear_ws_set_mode(1)
    _report("A", (shape, M), worst, "2^-10|y| + 2e-3")


# ------------------------------------------------------------------------------------------------------------------ B
def _tc_operands(M, N, K, has_bias, tag):
    g = torch.Generator().manual_seed(_seed("tc", tag, M, N, K))
    w = (torch.randn(N, K, generator=g) * 0.05).half().to(_dev())
    b = (torch.randn(N, generator=g) * 0.1).half().to(_dev()) if has_bias else None
    x = torch.randn(M, K, generator=g).half().to(_dev())
    return w, b, x


@gpu
@pytest.mark.parametrize("K", [64, 128, 192, 256])
@pytest.mark.parametrize("M", [64, 127, 128, 129, 255, 256])
def test_gemm_tc_pipeline_edges(M, K):
    """gemm_tc_kernel with 1 to 4 k-blocks (its pipeline has 4 stages) and ragged 128-row tiles, with and without bias,
    dense and strided (ldx = K + 64, ldy = N + 8) operands: within tolerance of float64, identical bits in both layouts,
    nothing written outside [0, M) x [0, N)."""
    from meshanything_b200 import capi
    N = 256
    worst = (0.0, 0.0)
    for has_bias in (True, False):
        w, b, x = _tc_operands(M, N, K, has_bias, "edges")
        ref = _ref_linear(x, w, b)
        first = None
        for ldx, ldy in ((K, N), (K + 64, N + 8)):
            buf, out = _sentinel_out(M, N, ldy)
            capi.linear_tc_f16(w, b, _strided_x(x, ldx), out=out)
            _assert_outside_untouched(buf, M, N, (M, K, has_bias, ldx, ldy))
            worst = _worst(worst, _check_tol(out, ref, (M, K, has_bias, ldx, ldy)))
            if first is None:
                first = out.clone()
            else:
                assert _same_bits(out, first), (M, K, has_bias)
    _report("B", ("edges", M, K), worst, "2^-10|y| + 2e-3")


@gpu
@pytest.mark.parametrize("has_bias", [False, True])
def test_gemm_tc_pre_kl_strided_input(has_bias):
    """The encoder's pre_kl call (api_encoder.cu): 8 shapes x 256 latents = 2048 rows, N = 128, K = 768, x = the first 768
    columns of the 1536-wide cat16 buffer (ldx = 1536; the other half is NaN here), with and without bias."""
    from meshanything_b200 import capi
    M, N, K = 2048, 128, 768
    w, b, x = _tc_operands(M, N, K, has_bias, "pre_kl")
    buf, out = _sentinel_out(M, N, N)
    capi.linear_tc_f16(w, b, _strided_x(x, 2 * K), out=out)
    _assert_outside_untouched(buf, M, N, "pre_kl")
    _report("B", ("pre_kl", has_bias), _check_tol(out, _ref_linear(x, w, b), "pre_kl"), "2^-10|y| + 2e-3")


@gpu
@pytest.mark.parametrize("name,N,K,has_bias", [("input_proj", 768, 256, True), ("c_kv", 1536, 768, False)])
def test_gemm_tc_encoder_point_rows(name, N, K, has_bias):
    """input_proj and c_kv of an 8-shape encoder chunk: 8 x 4096 = 32768 rows (256 row tiles); every row against float64,
    and >= 98 % of the values equal the canonical kernel's bit for bit."""
    from meshanything_b200 import capi
    M = 8 * 4096
    w, b, x = _tc_operands(M, N, K, has_bias, name)
    buf, out = _sentinel_out(M, N, N)
    capi.linear_tc_f16(w, b, x, out=out)
    _assert_outside_untouched(buf, M, N, name)
    err = _check_tol(out, _ref_linear(x, w, b), name)
    canon = capi.linear_f16(w, b, x).float()
    diff = (out.float() - canon).abs()
    assert bool((diff <= 2.0 ** -9 * canon.abs() + 1e-3).all())
    assert float((diff == 0).float().mean()) > 0.98
    _report("B", name, err, "2^-10|y| + 2e-3")


@gpu
@pytest.mark.parametrize("M", [1, 8])
@pytest.mark.parametrize("N", [1024, 768])
def test_canonical_linear_cond_head_gathered_rows(M, N):
    """cond_head_proj of the encoder (N = 1024) and of the detokenizer (N = 768): row 0 of every shape, read straight
    from the [shapes x 257, 768] feature buffer with ldx = 257 * 768, bit for bit against the oracle on those rows."""
    from meshanything_b200 import capi
    from oracle import decoder as orc
    K = 768
    g = torch.Generator().manual_seed(_seed("cond_head", M, N))
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    b = (torch.randn(N, generator=g) * 0.1).half()
    feats = torch.randn(M * 257, K, generator=g).half()
    x = feats.to(_dev())[::257]
    assert x.stride(0) == 257 * K
    got = capi.linear_f16(w.to(_dev()), b.to(_dev()), x).cpu()
    ref = orc.linear(w, b, feats[::257].contiguous())
    assert _same_bits(got, ref)


# ------------------------------------------------------------------------------------------------------------------ C
def _attention_inputs(S, n, H, seed):
    """q [S*n, H*64]; k [S, H, n, 64]; v [S, H, n, 64] (fp16, device) from one [S*n, 3*H*64] qkv-like source."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(S * n, H * 64, generator=g).half().to(_dev())
    src = torch.randn(S * n, 3 * H * 64, generator=g).half().to(_dev())
    k = src[:, H * 64:2 * H * 64].reshape(S, n, H, 64).permute(0, 2, 1, 3).contiguous()
    v = src[:, 2 * H * 64:].reshape(S, n, H, 64).permute(0, 2, 1, 3).contiguous()
    return q, src, k, v


@gpu
@pytest.mark.parametrize("S,n", [(8, 1057), (1, 1857)])
def test_attention_tc_detokenizer_shapes(S, n):
    """A detokenizer chunk: S shapes x (257 + F) tokens x 12 heads, every token attending to all tokens of its shape
    (F = 800: 9 query / key tiles, the last with 33 rows; F = 1600: 1857), against float64 softmax attention."""
    from meshanything_b200 import capi
    H = 12
    q, src, k, v = _attention_inputs(S, n, H, _seed("attn", S, n))
    vt = capi.transpose_heads_f16(src, 2 * H * 64, 64, H, n, S)
    out = capi.attention_tc_f16(q, k, vt, n, n)
    qd = q.double().reshape(S, n, H, 64).permute(0, 2, 1, 3)
    ref = torch.softmax(qd @ k.double().transpose(2, 3) * 0.125, dim=-1) @ v.double()
    ref = ref.permute(0, 2, 1, 3).reshape(S * n, H * 64)
    err = float((out.double() - ref).abs().max())
    assert err < 2e-3, err
    _report("C", (S, n), err, 2e-3)


@gpu
def test_attention_tc_keys_beyond_nkeys_are_masked():
    """K rows nkeys .. T-1 of a slot's cache (T = Tpad = 1152 > nkeys = 1057) are loaded with the last key tile but must
    not take part: NaN there gives the same bits as zeros there, and as a cache of exactly nkeys rows."""
    from meshanything_b200 import capi
    S, n, H, T = 2, 1057, 12, 1152
    q, src, k, _ = _attention_inputs(S, n, H, _seed("attn-mask"))
    vt = capi.transpose_heads_f16(src, 2 * H * 64, 64, H, n, S)
    assert vt.shape[3] == T
    k_zero = torch.zeros((S, H, T, 64), dtype=torch.float16, device=_dev())
    k_zero[:, :, :n] = k
    k_nan = k_zero.clone()
    k_nan[:, :, n:] = NAN16
    exact = capi.attention_tc_f16(q, k, vt, n, n)
    zero = capi.attention_tc_f16(q, k_zero, vt, n, n)
    nan = capi.attention_tc_f16(q, k_nan, vt, n, n)
    assert bool(torch.isfinite(nan).all())
    assert _same_bits(nan, zero)
    assert _same_bits(zero, exact)


# ------------------------------------------------------------------------------------------------------------------ D
NL = 3


@pytest.fixture(scope="module")
def dec3():
    from meshanything_b200.decoder import DecoderArena
    sd = decoder_sd(NL)
    return sd, DecoderArena(sd, _dev())


class _FixedRun:
    """ma_decode_generate on one Generator with output, forced-id and logits buffers that stay put: every run keys the
    per-step graph cache with the same pointers, so a replay is found whenever the rest of the key matches."""

    def __init__(self, gen, prefix, forced):
        self.gen, self.prefix, self.forced = gen, prefix.contiguous(), forced.to(_dev(), torch.int32).contiguous()
        B, n = self.forced.shape
        self.ids = torch.empty((B, n), dtype=torch.int32, device=_dev())
        self.lens = torch.empty((B,), dtype=torch.int32, device=_dev())
        self.logits = torch.empty((n, B, gen.arena.c.vocab), dtype=torch.float16, device=_dev())

    def __call__(self, flags):
        from meshanything_b200 import capi
        g = self.gen
        B, n = self.forced.shape
        samp = capi.Sampling(0, 50, 0.95, 0)
        capi.check(capi.lib().ma_decode_generate(C.byref(g.arena.c), capi.ptr(self.prefix), B, g.tmax, n, C.byref(samp),
                                                 -1, 2, capi.ptr(g.kv), capi.ptr(g.ws), capi.ptr(self.ids),
                                                 capi.ptr(self.lens), capi.ptr(self.forced), capi.ptr(self.logits), flags,
                                                 capi.stream_ptr()), "ma_decode_generate")
        assert self.ids.cpu().tolist() == self.forced.cpu().tolist()
        return self.logits.cpu()


@gpu
@pytest.mark.parametrize("B", [17, 32, 64, 100])
def test_tensor_core_decoder_production_batches(dec3, B):
    """Teacher-forced decode (16 tokens, specials 0 / 1 / 2 among them) with MA_GEN_TC at batch B: decode-step GEMMs on
    gemm_ws_kernel<32> (B = 17, 32), <64>, <128>, or in ticket mode gemm_tc_kernel (B >= 64, K <= 1024); prefill in
    ceil(B / 8) passes on gemm_tc_kernel.  Reference: the canonical batched run of the same batch (the oracle's logits,
    anchored on rows 0 and 31 of B = 32).  Cluster mode, then ticket mode on the same Generator and buffers: in each
    mode the graph run equals an eager run bit for bit, and every row is within the decoder's tensor-core tolerance."""
    from meshanything_b200 import capi
    from meshanything_b200.decoder import Generator
    sd, arena = dec3
    n = 16
    prefix = random_prefix(B, seed=50 + B).to(_dev())
    forced = torch.randint(3, 8195, (B, n), generator=torch.Generator().manual_seed(B), dtype=torch.int32)
    for r in range(B):
        forced[r, 1 + r % (n - 1)] = r % 3
    run = _FixedRun(Generator(arena, B, 257 + n), prefix, forced)
    canon = run(0).float()
    if B == 32:
        from oracle.decoder import OracleDecoder
        oracle = OracleDecoder(sd, NL, 257 + n)
        for r in (0, 31):
            _, ref = oracle.generate(prefix[r].cpu(), n, eos_id=-1, forced=forced[r].tolist(), keep_logits=True)
            assert _same_bits(canon[:, r].half(), torch.stack(ref)), r
    top2 = torch.topk(canon, 2, dim=2).values
    clear = (top2[..., 0] - top2[..., 1]) > 6e-2              # [n, B]
    got = {}
    worst = (0.0, 0.0)
    try:
        for cluster in (1, 0):
            capi.lib().ma_linear_ws_set_mode(cluster)
            tc = run(capi.GEN_TC)
            eager = run(capi.GEN_TC | capi.GEN_NO_GRAPH)
            assert _same_bits(tc, eager), f"graph replay != eager run (cluster={cluster})"
            diff = (tc.float() - canon).abs()
            for r in range(B):
                d = diff[:, r]
                assert float(d.max()) < 3e-2 and float(d.mean()) < 3e-3, (cluster, r, float(d.max()), float(d.mean()))
                am = tc[:, r].float().argmax(1)
                assert torch.equal(am[clear[:, r]], canon[:, r].argmax(1)[clear[:, r]]), (cluster, r)
            worst = (max(worst[0], float(diff.max())), max(worst[1], float(diff.mean(0).max())))
            got[cluster] = tc
    finally:
        capi.lib().ma_linear_ws_set_mode(1)
    # the two reductions round differently: a stale graph of the other mode would have shown above
    assert not _same_bits(got[1], got[0])
    _report("D", ("batch", B), worst[0], "max 3e-2, per-row mean 3e-3 (worst row mean %.3g)" % worst[1])


@gpu
def test_tensor_core_sampling_batch_32(dec3):
    """Sampled decode at batch 32 (tensor-core GEMMs): the same seed gives the same ids, and every id lies inside the
    top-k(50) support of its step's logits."""
    from meshanything_b200.decoder import Generator
    _, arena = dec3
    B, n = 32, 24
    prefix = random_prefix(B, seed=77).to(_dev())
    gen = Generator(arena, B, 257 + n)
    a, _, lg = gen.generate(prefix, n, do_sample=True, seed=7, want_logits=True, eos_id=-1)
    b, _ = gen.generate(prefix, n, do_sample=True, seed=7, eos_id=-1)
    assert torch.equal(a, b)
    lg, a = lg.float().cpu(), a.cpu().long()
    kth = torch.topk(lg, 50, dim=2).values[..., -1]                    # [n, B]
    picked = lg.gather(2, a.T[..., None])[..., 0]                      # [n, B]
    assert bool((picked >= kth).all())


@gpu
def test_slot_engine_sees_weights_replaced_at_the_same_address():
    """Continuous batching after the weights behind a DecoderWeights struct changed: the struct keeps its address, its
    pointers name another arena's tensors (a reloaded checkpoint).  The slot engine's cached step graphs must not be
    replayed with the old pointers: every sequence of the second queue equals solo generation with the new weights.
    Both arenas stay allocated, so a stale graph would give wrong ids, not touch freed memory."""
    from meshanything_b200 import capi
    from meshanything_b200.decoder import DecoderArena, Generator
    from meshanything_b200.scheduler import SlotEngine, SlotScheduler
    arena_a = DecoderArena(decoder_sd(NL, 0), _dev())          # private: its struct is overwritten below
    arena_b = DecoderArena(decoder_sd(NL, 1), _dev())
    n, NP, slots = 24, 3, 2
    prefixes = random_prefix(NP, seed=91).to(_dev())

    def solo(arena):
        g = Generator(arena, 1, 257 + n)
        return [g.generate(prefixes[i:i + 1], n, eos_id=-1)[0][0].cpu().tolist() for i in range(NP)]

    solo_a, solo_b = solo(arena_a), solo(arena_b)
    assert solo_a != solo_b
    eng = SlotEngine(arena_a, slots, 257 + n, n, eos_id=-1)

    def queue():
        got = {i: ids.cpu().tolist() for i, ids in SlotScheduler(eng, slots, n, poll_every=8).run(list(prefixes))}
        return [got[i] for i in range(NP)]

    assert queue() == solo_a
    C.memmove(C.addressof(arena_a.c), C.addressof(arena_b.c), C.sizeof(capi.DecoderWeights))
    eng.reset()
    assert queue() == solo_b


# ------------------------------------------------------------------------------------------------------------------ E
TOL_PF_MAX, TOL_PF_MEAN = 1.5e-2, 2.5e-3          # DESIGN.md section 6 (as tests/test_gpu_pipeline.py)
TOL_PREFIX_MAX, TOL_PREFIX_MEAN = 4e-2, 6e-3


@pytest.fixture(scope="module")
def enc_sd():
    """Encoder + tokenizer weights of the synthetic checkpoint (the same values as with 24 decoder layers)."""
    from meshanything_b200 import checkpoint as ck
    return ck.make_state_dict(ck.all_specs(1), 0)


def _nan_bits(t: torch.Tensor) -> torch.Tensor:
    return torch.nan_to_num(t, nan=7.0).view(torch.int32)


@gpu
def test_encoder_across_chunks(enc_sd):
    """ma_encoder_forward at B = 17 (chunks of 8 + 8 + 1): every shape's point_feature and prefix equal a forward of that
    shape alone bit for bit, and shapes 0, 8 and 16 are within the encoder tolerances of the fp32 restatement."""
    from meshanything_b200.encoder import EncoderArena
    from meshanything_b200.inputs import synthetic_pc_normal
    from oracle import torch_ref
    B = 17
    pc = synthetic_pc_normal(B, first=40)
    enc = EncoderArena(enc_sd, _dev())
    pf, prefix = enc.forward(pc.to(_dev()))
    for b in range(B):
        pf1, prefix1 = enc.forward(pc[b:b + 1].to(_dev()))
        assert torch.equal(pf1[0].view(torch.int32), pf[b].view(torch.int32)), b
        assert torch.equal(prefix1[0].view(torch.int32), prefix[b].view(torch.int32)), b
    rows = [0, 8, 16]
    with torch.no_grad():
        rpf, rprefix = torch_ref.encoder_forward(enc_sd, pc[rows])
    d1, d2 = (pf[rows].cpu() - rpf).abs(), (prefix[rows].cpu() - rprefix).abs()
    for i, r in enumerate(rows):
        assert d1[i].max() < TOL_PF_MAX and d1[i].mean() < TOL_PF_MEAN, (r, float(d1[i].max()), float(d1[i].mean()))
        assert d2[i].max() < TOL_PREFIX_MAX and d2[i].mean() < TOL_PREFIX_MEAN, (r, float(d2[i].max()))
    _report("E", "encoder point_feature", float(d1.max()), f"max {TOL_PF_MAX}, mean {TOL_PF_MEAN} (mean {float(d1.mean()):.3g})")
    _report("E", "encoder prefix", float(d2.max()), f"max {TOL_PREFIX_MAX}, mean {TOL_PREFIX_MEAN} (mean {float(d2.mean()):.3g})")


@gpu
def test_detokenizer_across_chunks(enc_sd):
    """ma_detokenize at B = 9, F = 800 (chunks of 8 + 1; 1057 tokens per shape): an eos inside a face, padding after it,
    a special id inside the last face and an all-padding row.  ids equal postprocess_ids; every shape's coordinates equal
    a call with that shape alone bit for bit; shapes 0 and 8 pass the bins rule against the fp32 restatement."""
    from meshanything_b200.encoder import EncoderArena, TokenizerArena
    from meshanything_b200.inputs import synthetic_pc_normal
    from oracle import torch_ref
    B, F = 9, 800
    g = torch.Generator().manual_seed(_seed("detok", B, F))
    gen_ids = torch.randint(3, 8195, (B, 9 * F + 2), generator=g, dtype=torch.int64)
    gen_ids[0, 1 + 9 * 300 + 4] = 1          # eos inside face 300 -> face 300 absent
    gen_ids[0, 1 + 9 * 600:] = 2             # padding after face 599
    gen_ids[4, 1:] = 2                       # nothing generated
    gen_ids[8, 1 + 9 * 799 + 8] = 0          # a special id inside the last face
    pf, _ = EncoderArena(enc_sd, _dev()).forward(synthetic_pc_normal(B, first=70).to(_dev()))
    tok = TokenizerArena(enc_sd, _dev())
    ids_d = gen_ids.to(torch.int32).to(_dev())
    coords, ids = tok.detokenize(ids_d, pf, F, want_ids=True)
    ref_ids = torch_ref.postprocess_ids(gen_ids, F)
    assert torch.equal(ids.cpu().long(), ref_ids)
    assert bool(torch.isnan(coords[4]).all())
    for b in range(B):
        one = tok.detokenize(ids_d[b:b + 1], pf[b:b + 1], F)
        assert torch.equal(_nan_bits(one[0]), _nan_bits(coords[b])), b
    rows = [0, 8]
    with torch.no_grad():
        rcoords, rlogits = torch_ref.detokenize(enc_sd, ref_ids[rows], pf[rows].cpu(), return_logits=True)
    c = coords[rows].cpu()
    assert torch.equal(torch.isnan(c), torch.isnan(rcoords))
    top2 = torch.topk(rlogits, 2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1]).view(len(rows), F, 3, 3)
    for i, r in enumerate(rows):
        valid = ~torch.isnan(rcoords[i])
        same = c[i][valid] == rcoords[i][valid]
        m = margin[i][valid]
        assert float(same.float().mean()) > 0.97, (r, float(same.float().mean()))
        assert bool((m[~same] < 0.08).all()), (r, float(m[~same].max()))
        _report("E", ("detokenizer bins", r), 1.0 - float(same.float().mean()),
                "<= 3 %% unequal, only where the margin < 0.08 (largest margin at a mismatch %.3g)"
                % (float(m[~same].max()) if bool((~same).any()) else 0.0))
