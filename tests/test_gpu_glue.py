"""-m gpu: the glue kernels of the encoder and the detokenizer (csrc/glue.cu) through their test entry points, each
against a torch-on-CPU (or numpy) restatement at the arguments its call sites in api_encoder.cu use.  Every destination
starts filled with a NaN sentinel, and every element outside the region a call writes must still hold it."""
import numpy as np
import pytest
import torch

from meshanything_b200 import capi

gpu = pytest.mark.gpu
NLAT, EW, NPTS = 257, 768, 4096


def _dev():
    return torch.device("cuda", 0)


def _filled(shape, dtype):
    """A destination filled with the sentinel: all-ones bits (a NaN no kernel writes) for floats, -12345 for ints."""
    t = torch.empty(shape, dtype=dtype, device=_dev())
    if dtype == torch.float16:
        t.view(torch.int16).fill_(-1)
    elif dtype == torch.float32:
        t.view(torch.int32).fill_(-1)
    else:
        t.fill_(-12345)
    return t


def _bits(t):
    t = t.detach().cpu()
    if t.dtype == torch.float16:
        return t.view(torch.int16)
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _untouched(t):
    b = _bits(t)
    return bool((b == (-1 if t.dtype in (torch.float16, torch.float32) else -12345)).all())


def _assert_bits(got, want):
    g, w = _bits(got), _bits(want)
    bad = (g != w).nonzero()
    assert not len(bad), (len(bad), bad[:5].tolist(), got.cpu()[tuple(bad[:5].T)], want.cpu()[tuple(bad[:5].T)])


# ---------------------------------------------------------------------------------------------------- fourier_embed

def _pc(rows, seed):
    g = torch.Generator().manual_seed(seed)
    pc = torch.randn(rows, 6, generator=g).half()
    special = torch.tensor([1.0, -1.0, 0.0, -0.0, 2.0 ** -24, -(2.0 ** -24), 2.0 ** -15, -3 * 2.0 ** -20, 65504.0,
                            -65504.0, 3.140625, 1000.0], dtype=torch.float16)
    flat = pc.view(-1)
    k = min(len(special), flat.numel())
    flat[:k] = special[:k]                                    # the first rows carry the edge values
    if rows > 8:
        flat[-k:] = special[:k].flip(0)                       # and the last
    return pc


def _fp16_window(x):
    """fp16 values of float64 x and of x +- 2 fp32 ulps: where they differ, a 2-ulp sinf / cosf may round either way."""
    ulp = 2.0 * np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)
    lo, hi = (x - ulp).astype(np.float16), (x + ulp).astype(np.float16)
    exact = x.astype(np.float16)
    zero = x == 0
    lo[zero], hi[zero] = exact[zero], exact[zero]
    return exact, lo, hi


@gpu
@pytest.mark.parametrize("rows", [32768, 1, 3, 4097])
def test_fourier_embed(rows):
    pc = _pc(rows, rows)
    out = _filled((rows + 1, 256), torch.float16)
    capi.fourier_embed_f16(pc.to(_dev()), out=out)
    assert _untouched(out[rows:])
    got = out[:rows].cpu()
    _assert_bits(got[:, 0:3], pc[:, 0:3])
    _assert_bits(got[:, 51:54], pc[:, 3:6])
    assert (got[:, 54:].view(torch.int16) == 0).all()        # +0 padding
    x = pc[:, :3].double().numpy()
    arg = (x[:, :, None] * (2.0 ** np.arange(8))).reshape(rows, 24)   # coordinate-major; x 2^j is exact in fp32
    loose = 0
    for col0, fn in ((3, np.sin), (27, np.cos)):
        g = got[:, col0:col0 + 24].numpy()
        exact, lo, hi = _fp16_window(fn(arg))
        tight = lo.view(np.uint16) == hi.view(np.uint16)
        ok = np.where(tight, g.view(np.uint16) == exact.view(np.uint16),
                      (g.view(np.uint16) == lo.view(np.uint16)) | (g.view(np.uint16) == hi.view(np.uint16)))
        bad = np.argwhere(~ok)
        assert not len(bad), (fn.__name__, len(bad), bad[:5].tolist(), g[tuple(bad[:5].T)], exact[tuple(bad[:5].T)])
        loose += int((~tight).sum())
    print(f"fourier_embed rows={rows}: {loose} of {rows * 48} sin/cos values within 2 fp32 ulps of an fp16 midpoint")


# ---------------------------------------------------------------------------------------------------- scatter_heads

def _scatter_ref(src, rows, col0, stride, H, rps, T):
    idx = col0 + stride * torch.arange(H)[:, None] + torch.arange(64)
    sub = src[:rows][:, idx]                                   # [rows, H, 64]
    slots = rows // rps
    out = torch.full((slots, H, T, 64), float("nan"), dtype=torch.float16)
    out.view(torch.int16).fill_(-1)
    out[:, :, :rps] = sub.view(slots, rps, H, 64).permute(0, 2, 1, 3)
    return out


SCATTER = [  # (ld, col0, head_stride, H, rows_per_slot, T, rows)
    (3 * EW, 0, 192, 12, 1, 1, 8 * NLAT),                      # self-attention q
    (3 * EW, 64, 192, 12, NLAT, NLAT, 8 * NLAT),               # self-attention k
    (3 * EW, 128, 192, 12, 256, 256, 3 * 256),                 # self-attention v, the fp16-stream blocks
    (2 * EW, 0, 128, 12, NPTS, NPTS, 8 * NPTS),                # cross-attention k
    (2 * EW, 64, 128, 12, NPTS, NPTS, 2 * NPTS),               # cross-attention v
    (3 * EW, 0, 64, 12, 1, 1, 2 * (NLAT + 800)),               # detokenizer q
    (3 * EW, EW, 64, 12, NLAT + 800, NLAT + 800, 2 * (NLAT + 800)),      # detokenizer k
    (3 * EW, 2 * EW, 64, 12, NLAT + 13, NLAT + 16, 3 * (NLAT + 13)),    # detokenizer v, T > rows per slot
]


@gpu
@pytest.mark.parametrize("ld,col0,stride,H,rps,T,rows", SCATTER)
def test_scatter_heads(ld, col0, stride, H, rps, T, rows):
    g = torch.Generator().manual_seed(rows + col0)
    src = torch.randn(rows, ld, generator=g).half()
    n = rows // rps * H * T * 64
    dst = _filled((n + 4096,), torch.float16)
    capi.scatter_heads_f16(src.to(_dev()), col0, stride, H, rps, T, dst)
    assert _untouched(dst[n:])
    _assert_bits(dst[:n].view(rows // rps, H, T, 64), _scatter_ref(src, rows, col0, stride, H, rps, T))


# ---------------------------------------------------------------------------------------------------- residual_add

def _residual_operands(n, x_dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, generator=g) * 100).to(x_dtype)
    y = (torch.randn(n, generator=g) * 100).half()
    inf = float("inf")
    pairs = [(-0.0, 0.0), (0.0, -0.0), (-0.0, -0.0), (inf, 1.0), (-inf, 2.0), (1.0, inf), (3.0, -inf), (-inf, -inf),
             (65504.0, 65504.0), (65504.0, 16.0), (65504.0, 15.0), (-65504.0, -32.0), (3.0e38, 65504.0),
             (2.0 ** -24, 2.0 ** -25), (1.0, -1.0)]
    for i, (a, b) in enumerate(pairs):
        x[7 * i] = a
        y[7 * i] = b
    return x, y


@gpu
@pytest.mark.parametrize("x_dtype", [torch.float32, torch.float16])
def test_residual_add(x_dtype):
    n = 8 * NLAT * EW
    x, y = _residual_operands(n, x_dtype, 3)
    buf = _filled((n + 8,), x_dtype)
    buf[:n] = x.to(_dev())
    capi.residual_add(buf[:n], y.to(_dev()))
    assert _untouched(buf[n:])
    want = x + y.float() if x_dtype == torch.float32 else (x.float() + y.float()).half()
    _assert_bits(buf[:n], want)
    if x_dtype == torch.float16:
        assert torch.isinf(buf[9 * 7]).item() and buf[10 * 7].item() == 65504.0   # 65520 ties up to inf; 65519 does not


@gpu
def test_glue_entry_points_refuse_bad_arguments():
    L = capi.lib()
    d = _dev()
    h = torch.zeros(4096, dtype=torch.float16, device=d)
    f = torch.zeros(4096, dtype=torch.float32, device=d)
    i = torch.zeros(64, dtype=torch.int32, device=d)
    p = lambda t: capi.ptr(t)                                        # noqa: E731
    st = capi.stream_ptr()
    torch.cuda.synchronize()
    before = L.ma_launch_count()
    calls = [
        lambda: L.ma_fourier_embed_f16(None, 1, p(h), st),
        lambda: L.ma_fourier_embed_f16(p(h), 0, p(h), st),
        lambda: L.ma_scatter_heads_f16(p(h), 64, 0, 64, 1, 1, 1, None, 1, st),
        lambda: L.ma_scatter_heads_f16(p(h), 64, 4, 64, 1, 1, 1, p(h), 1, st),
        lambda: L.ma_scatter_heads_f16(p(h), 64, 0, 64, 0, 1, 1, p(h), 1, st),
        lambda: L.ma_scatter_heads_f16(p(h), 64, 0, 64, 1, 0, 1, p(h), 1, st),
        lambda: L.ma_scatter_heads_f16(p(h[1:]), 64, 0, 64, 1, 1, 1, p(h), 1, st),
        lambda: L.ma_residual_add(p(f), None, p(h), 6, st),           # n % 4 != 0: used to skip the tail silently
        lambda: L.ma_residual_add(p(f), None, p(h), 0, st),
        lambda: L.ma_residual_add(p(f), p(h), p(h), 8, st),           # both streams
        lambda: L.ma_residual_add(None, None, p(h), 8, st),
        lambda: L.ma_residual_add(p(f), None, None, 8, st),
        lambda: L.ma_convert_rows(p(f), 0, 8, p(h), 1, 8, 1, 6, 0, st),  # cols % 4 != 0
        lambda: L.ma_convert_rows(p(f), 0, 8, p(h), 1, 8, 0, 8, 0, st),
        lambda: L.ma_convert_rows(None, 0, 8, p(h), 1, 8, 1, 8, 0, st),
        lambda: L.ma_convert_rows(p(f), 0, 8, p(h), 1, 8, 1, 8, -1, st),
        lambda: L.ma_add_table(p(h), None, p(f), 0, p(f), 1, st),
        lambda: L.ma_add_table(p(h), None, None, 1, p(f), 1, st),
        lambda: L.ma_add_table(p(h), None, p(f), 1, p(f), 0, st),
        lambda: L.ma_gather_codes(p(i), 11, 1, 0, p(f), p(h), p(i), None, st),
        lambda: L.ma_gather_codes(p(i), 11, 1, 1, p(f), p(h), None, None, st),
        lambda: L.ma_gather_codes(None, 11, 1, 1, p(f), p(h), p(i), None, st),
        lambda: L.ma_coords(p(h), p(i), p(f), 0, st),
        lambda: L.ma_coords(p(h), None, p(f), 1, st),
    ]
    for k, call in enumerate(calls):
        assert call() != 0, k
        assert b"bad arguments" in L.ma_last_error(), (k, L.ma_last_error())
    assert L.ma_launch_count() == before


# ---------------------------------------------------------------------------------------------------- convert_rows

def _convert_src(rows, cols, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, cols, generator=g, dtype=torch.float64) * 300
    flat = x.view(-1)
    edge = [1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -(1 + 2.0 ** -11), 65504.0, 65519.0, 65520.0, -65520.0, 1e6, -1e30,
            2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -26, -(2.0 ** -25), 2.0 ** -14 - 2.0 ** -25, 1e-30, -0.0, 0.0,
            float("inf"), float("-inf"), 2049.0, 2051.0]
    flat[:len(edge)] = torch.tensor(edge, dtype=torch.float64)
    return x.to(dtype)


CONVERT = [  # (src dtype, dst dtype, rows, cols, lds, ldd, src_rows_mod, src rows, dst col0)
    (torch.float32, torch.float32, 8 * NLAT, EW, EW, EW, NLAT, NLAT, 0),          # x = query, broadcast to 8 shapes
    (torch.float16, torch.float32, 8, 1024, 1024, NLAT * 1024, 0, 8, 0),          # prefix row 0 of every shape
    (torch.float16, torch.float16, 256, EW, EW, 2 * EW, 0, 256, 0),               # latents into the cat16 left half
    (torch.float16, torch.float16, 8 * 256, EW, EW, 2 * EW, 0, 8 * 256, EW),      # shape latents into the right half
    (torch.float16, torch.float16, 8 * 256, 64, 128, 256, 0, 8 * 256, 0),         # pre_kl mean -> lat16
    (torch.float16, torch.float32, 256, 1024, 1024, 1024, 0, 256, 0),             # prefix rows 1..256
    (torch.float32, torch.float16, 8 * NLAT, EW, EW, EW, 0, 8 * NLAT, 0),         # point_feature -> fp16
    (torch.float32, torch.float16, 5, 1024, 1028, 1024, 0, 5, 0),                 # the edge values, fp32 -> fp16
    (torch.float32, torch.float16, 2 * NLAT + 3, 8, 8, 8, NLAT, NLAT, 0),         # a row modulus that wraps unevenly
]


@gpu
@pytest.mark.parametrize("sd,dd,rows,cols,lds,ldd,mod,srows,dcol0", CONVERT)
def test_convert_rows(sd, dd, rows, cols, lds, ldd, mod, srows, dcol0):
    src_full = _convert_src(srows, lds, sd, rows + cols)
    dst_full = _filled((rows * ldd + ldd,), dd)                  # rows * ldd elements and one spare row
    dst = dst_full[:rows * ldd].view(rows, ldd)[:, dcol0:dcol0 + cols]
    capi.convert_rows(src_full.to(_dev())[:, :cols], dst, rows, cols, mod)
    r = torch.arange(rows) % mod if mod else torch.arange(rows)
    want_rows = src_full[:, :cols][r]
    if dd == torch.float16 and sd == torch.float32:
        with np.errstate(over="ignore"):                             # the overflow cases round to +-inf
            want = torch.from_numpy(want_rows.numpy().astype(np.float16))  # numpy: round to nearest even
    else:
        want = want_rows.to(dd)
    _assert_bits(dst, want)
    written = torch.zeros(rows * ldd + ldd, dtype=torch.bool)
    written[:rows * ldd].view(rows, ldd)[:, dcol0:dcol0 + cols] = True
    assert _untouched(dst_full[~written.to(_dev())])
    if dd == torch.float16 and sd == torch.float32 and rows == 5:
        e = dst[0, :21].cpu().float().tolist()
        assert e[:3] == [1.0, 1 + 2 * 2.0 ** -10, -1.0]                  # ties to even
        assert e[3:9] == [65504.0, 65504.0, float("inf"), float("-inf"), float("inf"), float("-inf")]
        assert e[9:14] == [0.0, 2 * 2.0 ** -24, 0.0, -0.0, 2.0 ** -14]     # subnormals
        assert e[19:21] == [2048.0, 2052.0]


# ---------------------------------------------------------------------------------------------------- add_table

@gpu
@pytest.mark.parametrize("rows,table_rows,masked", [(8 * NLAT, NLAT, False), (8 * 800, 800, True),
                                                     (3 * 50, 50, False)])
def test_add_table(rows, table_rows, masked):
    g = torch.Generator().manual_seed(rows)
    y = (torch.randn(rows, EW, generator=g) * 3).half()
    table = torch.randn(table_rows, EW, generator=g)
    table[0, :4] = torch.tensor([-0.0, 0.0, float("inf"), -1e38])
    y[0, :4] = torch.tensor([0.0, -0.0, 1.0, -65504.0]).half()
    mask = (torch.rand(rows, generator=g) > 0.3).int() if masked else None
    if masked:
        mask[table_rows] = 0                                    # a masked row over table row 0 (+0 + -0 = +0)
    out = _filled((rows + 2, EW), torch.float32)
    capi.add_table(y.to(_dev()), table.to(_dev()), None if mask is None else mask.to(_dev()), out=out[:rows])
    assert _untouched(out[rows:])
    yf = y.float() if mask is None else torch.where(mask[:, None].bool(), y.float(), torch.zeros(()))
    _assert_bits(out[:rows], yf + table[torch.arange(rows) % table_rows])
    if masked:
        assert (_bits(out[table_rows, :1]) == 0).all()


# ---------------------------------------------------------------------------------------------------- gather_codes

@gpu
def test_gather_codes():
    from oracle import torch_ref
    B, F = 8, 800
    max_new = 9 * F + 2
    g = torch.Generator().manual_seed(9)
    gi = torch.randint(3, 8195, (B, max_new), generator=g, dtype=torch.int64)
    gi[0, 1 + 9 * 3] = 0                                        # specials at the first token of a face
    gi[0, 1 + 9 * 4] = 1
    gi[0, 1 + 9 * 5] = 2
    gi[1, 1 + 9 * 3 + 8] = 0                                    # and at the last
    gi[1, 1 + 9 * 4 + 8] = 2
    gi[1, 1 + 9 * (F - 1) + 8] = 1                              # the very last kept token
    gi[2, 1 + 9 * 10 + 4:] = 1                                  # eos mid-face, then eos to the end
    gi[3, 1 + 9 * 500:] = 2                                     # padding after face 500
    gi[4, :] = 2                                                # a row of padding only
    gi[5, 0] = 1                                                # position 0 (the predicted bos) is dropped
    gi[6, -1] = 0                                               # and so is the last position
    codebook = torch.randn(8192, 1024, generator=g)
    dev = _dev()
    code16 = _filled((B * F + 1, 3072), torch.float16)
    mask = _filled((B * F + 1,), torch.int32)
    ids = _filled((B * F + 1, 9), torch.int32)
    capi.gather_codes(gi.int().to(dev), F, codebook.to(dev), out=(code16[:-1], mask[:-1], ids[:-1]))
    assert _untouched(code16[-1:]) and _untouched(mask[-1:]) and _untouched(ids[-1:])
    want_ids = torch_ref.postprocess_ids(gi, F).view(B * F, 9)
    assert torch.equal(ids[:-1].cpu().long(), want_ids)
    assert torch.equal(mask[:-1].cpu(), (want_ids >= 0).all(1).int())
    c = torch.where(want_ids[..., None] >= 0, codebook[want_ids.clamp(min=0)], torch.zeros(()))    # [BF, 9, 1024]
    c = c.view(B * F, 3, 3, 1024)
    want = ((c[:, :, 0] + c[:, :, 1]) + c[:, :, 2]).half().view(B * F, 3072)
    _assert_bits(code16[:-1], want)
    assert int(mask[:-1].sum()) < B * F - 600                   # the cases above did mask faces


# ---------------------------------------------------------------------------------------------------- coords

@gpu
def test_coords():
    faces = 2 * 800 + 3
    g = torch.Generator().manual_seed(4)
    lg = (torch.randn(faces, 9, 128, generator=g) * 4).half()
    inf = float("inf")
    lg[0, 0] = 7.0                                              # ties: the lowest index of the maxima
    lg[0, 0, 5] = lg[0, 0, 77] = 9.0
    lg[0, 1] = -1.0
    lg[0, 1, 3], lg[0, 1, 64] = -0.0, 0.0                       # -0 and +0 tie
    lg[0, 2] = -1.0
    lg[0, 2, 96], lg[0, 2, 31] = 0.0, -0.0
    lg[0, 3] = 2.5                                              # all equal
    lg[0, 4] = -inf                                             # all -inf
    lg[0, 5] = -inf
    lg[0, 5, 127] = -65504.0
    lg[0, 6, 100] = inf                                         # +inf wins
    lg[0, 6, 33] = inf                                          # two +inf: the lower index
    lg[0, 7, 0] = -inf
    lg[0, 8, 31], lg[0, 8, 32] = 60000.0, 60000.0               # a tie across the lanes' stride of 32
    lg[1] = lg[1, :, :1]                                        # every coordinate of face 1: all equal
    mask = (torch.rand(faces, generator=g) > 0.2).int()
    mask[0] = mask[1] = 1
    out = _filled((faces + 1, 9), torch.float32)
    capi.coords(lg.view(faces, 1152).to(_dev()), mask.to(_dev()), out=out[:faces])
    assert _untouched(out[faces:])
    v = lg.float()
    lowest = (v == v.max(-1, keepdim=True).values).int().argmax(-1)     # first index among the maxima
    assert torch.equal(lowest, torch.argmax(v, dim=-1))
    assert lowest[0].tolist() == [5, 3, 31, 0, 0, 127, 33, lowest[0, 7].item(), 31] and (lowest[1] == 0).all()
    want = lowest.float() / 128 - 0.5
    want.view(torch.int32)[mask == 0] = 0x7fc00000
    _assert_bits(out[:faces], want)
