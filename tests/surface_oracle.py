"""numpy restatement of csrc/surface.cu (test infrastructure only): the area-weighted surface sampler as DESIGN.md
section 1.5 defines it, operation for operation.

- Philox4x32-10 with counter (i, 0x53555246, 0x4d455348, 0x414e5954) and key (seed low word, seed high word); the three
  uniforms are (c_j >> 8) 2^-24, j = 0, 1, 2.
- float64 face areas 0.5 sqrt((nx nx + ny ny) + nz nz) of the cross product of (b - a, c - a) taken in float64.
- Their inclusive scan in the kernel's order: 1024-element tiles; inside a tile a Hillis-Steele shfl_up scan of each warp
  of 32, a scan of the 32 warp totals in the same way, then the tile's carry (the previous tile's last sum, padding
  included) added as carry + warp offset.  Then the running maximum over the faces of positive area (0 before the
  first): cum never decreases and a face of zero area repeats the previous value.
- Face = the first face whose cumulative area exceeds float64(u0) cum[F - 1], by the kernel's binary search (F - 1 when
  none does: a mesh of zero total area gets its last face).
- float32 point (a + r1 u) + r2 w after reflecting (r1, r2) when r1 + r2 > 1, and float32 unit normal n / sqrt(n.n)
  (n / 1 when the length is 0), each operation rounded on its own (numpy never fuses a multiply-add); fp16 output
  rounded to nearest even.
"""
import numpy as np

F32, F64 = np.float32, np.float64
M32 = np.uint64(0xFFFFFFFF)
PHILOX_M0, PHILOX_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85
COUNTER_WORDS = (0x53555246, 0x4d455348, 0x414e5954)     # "FRUS", "HSEM", "YTNA": the sampler's stream tag
TILE, WARP = 1024, 32


def philox4x32_10(counter, key):
    """Philox4x32-10 of Random123: counter = 4 arrays (or ints) of uint32 words, key = 2 ints -> 4 uint32 arrays."""
    c = [np.asarray(w, dtype=np.uint64) & M32 for w in counter]
    c = [np.broadcast_to(w, np.broadcast(*c).shape).copy() for w in c]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = PHILOX_M0 * c[0], PHILOX_M1 * c[2]          # < 2^64: exact in uint64
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & M32, p1 >> np.uint64(32), p1 & M32
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + PHILOX_W0) & 0xFFFFFFFF, (k1 + PHILOX_W1) & 0xFFFFFFFF
    return [w.astype(np.uint32) for w in c]


def uniforms(seed, n):
    """The three fp32 uniforms in [0, 1) of samples 0..n-1: [n, 3]."""
    seed = int(seed)
    assert 0 <= seed < 1 << 64
    i = np.arange(n, dtype=np.uint64)
    c = philox4x32_10((i, *COUNTER_WORDS), (seed & 0xFFFFFFFF, seed >> 32))
    return np.stack([(w[:] >> np.uint32(8)).astype(F32) * F32(2.0 ** -24) for w in c[:3]], axis=1)


def face_areas(vertices, faces):
    v = np.ascontiguousarray(vertices, F32).astype(F64)
    t = v[np.asarray(faces, np.int64)]
    u, w = t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]
    nx = u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1]
    ny = u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2]
    nz = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
    return F64(0.5) * np.sqrt((nx * nx + ny * ny) + nz * nz)


def _hillis_steele(x):
    """Inclusive scan along the last axis (32 lanes) as the kernel's shfl_up loop computes it."""
    x = x.copy()
    o = 1
    while o < WARP:
        y = x.copy()
        x[..., o:] = y[..., o:] + y[..., :-o]
        o <<= 1
    return x


def tile_sums(area):
    """The Hillis-Steele sums of surface_scan_kernel (one CTA of 1024 threads walking the array in tiles)."""
    a = np.asarray(area, F64)
    F = len(a)
    T = (F + TILE - 1) // TILE
    x = np.zeros(T * TILE, F64)
    x[:F] = a
    x = _hillis_steele(x.reshape(T, WARP, WARP))              # [tile][warp][lane]
    ws = _hillis_steele(x[:, :, WARP - 1])                    # scanned warp totals [tile][warp]
    prev = np.concatenate([np.zeros((T, 1), F64), ws[:, :-1]], axis=1)
    carry = np.zeros(T, F64)
    for t in range(1, T):                                     # carry = the previous tile's sum at element 1023
        carry[t] = x[t - 1, WARP - 1, WARP - 1] + (carry[t - 1] + prev[t - 1, WARP - 1])
    return (x + (carry[:, None] + prev)[:, :, None]).reshape(-1)[:F]


def scan(area):
    """The cumulative areas surface_scan_kernel leaves: the running maximum of the tile sums over positive faces."""
    a = np.asarray(area, F64)
    return np.maximum.accumulate(np.where(a > 0, tile_sums(a), F64(0)))


def pick_faces(cum, u0):
    """The kernel's binary search: the first face with cum > float64(u0) cum[F - 1], else F - 1."""
    cum = np.asarray(cum, F64)
    F = len(cum)
    target = u0.astype(F64) * cum[F - 1]
    lo = np.zeros(len(u0), np.int64)
    hi = np.full(len(u0), F - 1, np.int64)
    while True:
        act = lo < hi
        if not act.any():
            return lo
        mid = (lo + hi) >> 1
        right = cum[mid] > target
        hi = np.where(act & right, mid, hi)
        lo = np.where(act & ~right, mid + 1, lo)


def sample_surface(vertices, faces, n, seed):
    """-> (out fp16 [n, 6] = point | unit face normal, face int32 [n]), the bits ma_sample_surface writes."""
    v = np.ascontiguousarray(vertices, F32)
    f = np.asarray(faces, np.int64)
    assert v.ndim == 2 and v.shape[1] == 3 and f.ndim == 2 and f.shape[1] == 3 and len(f) >= 1 and n >= 1
    u = uniforms(seed, n)
    face = pick_faces(scan(face_areas(v, f)), u[:, 0])
    t = v[f[face]]                                            # [n, 3 vertices, 3] fp32
    a, b, c = t[:, 0], t[:, 1], t[:, 2]
    r1, r2 = u[:, 1].copy(), u[:, 2].copy()
    flip = (r1 + r2) > F32(1)
    r1[flip], r2[flip] = F32(1) - r1[flip], F32(1) - r2[flip]
    uu, ww = b - a, c - a
    p = (a + r1[:, None] * uu) + r2[:, None] * ww
    nx = uu[:, 1] * ww[:, 2] - uu[:, 2] * ww[:, 1]
    ny = uu[:, 2] * ww[:, 0] - uu[:, 0] * ww[:, 2]
    nz = uu[:, 0] * ww[:, 1] - uu[:, 1] * ww[:, 0]
    ln = np.sqrt((nx * nx + ny * ny) + nz * nz)
    inv = np.where(ln > F32(0), F32(1) / np.where(ln > F32(0), ln, F32(1)), F32(1)).astype(F32)
    nrm = np.stack([nx * inv, ny * inv, nz * inv], axis=1)
    assert p.dtype == F32 and nrm.dtype == F32
    return np.concatenate([p, nrm], axis=1).astype(np.float16), face.astype(np.int32)
