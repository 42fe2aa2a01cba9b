"""not gpu: the numpy restatement of the surface sampler (tests/surface_oracle.py) -- Philox known-answer vectors, the
tiled scan against np.cumsum, the face pick's treatment of zero-area faces and the rule for a mesh of zero area."""
import numpy as np
import pytest

from tests import surface_oracle as SO

F64 = np.float64


@pytest.mark.parametrize("counter,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(counter, key, want):
    """Random123's known-answer vectors for Philox4x32-10."""
    got = SO.philox4x32_10(counter, key)
    assert tuple(int(w) for w in got) == want


def test_uniforms_use_both_key_words():
    """The key is (seed low word, seed high word): seeds that differ only in the high word give other draws."""
    lo, hi, both = SO.uniforms(7, 64), SO.uniforms(7 + (1 << 32), 64), SO.uniforms((1 << 64) - 1, 64)
    assert not np.array_equal(lo, hi) and not np.array_equal(lo, both)
    u = SO.uniforms(5, 100_000)
    assert u.dtype == np.float32 and u.min() >= 0 and u.max() < 1
    assert np.all((u * 2 ** 24) == np.floor(u * 2 ** 24))           # multiples of 2^-24
    assert np.abs(u.mean(0) - 0.5).max() < 5e-3


@pytest.mark.parametrize("F", [1, 1023, 1024, 1025, 3000, 1_000_000])
def test_scan_equals_cumsum_and_is_monotone(F):
    rng = np.random.default_rng(F)
    a = rng.exponential(size=F) * rng.choice([1e-6, 1.0, 1e3], size=F)
    a[rng.random(F) < 0.05] = 0.0
    ref = np.cumsum(a)
    for s in (SO.tile_sums(a), SO.scan(a)):
        assert s.dtype == F64 and s.shape == (F,)
        assert np.all(np.abs(s - ref) <= 1e-12 * ref[-1])
        assert s[0] == a[0]
    s = SO.scan(a)
    assert np.all(np.diff(s) >= 0)
    assert np.all(s[1:][a[1:] == 0] == s[:-1][a[1:] == 0])            # zero-area faces add exactly nothing
    if F == 1_000_000:
        # why the kernel takes the running maximum: the tile sums alone step down, and step up across zero-area faces
        d = np.diff(SO.tile_sums(a))
        assert (d < 0).any() and (d[a[1:] == 0] > 0).any()


def test_scan_carries_across_tiles():
    """Ones: every tile adds exactly 1024 to the carry (integers stay exact in float64)."""
    s = SO.scan(np.ones(5000))
    assert np.array_equal(s, np.arange(1, 5001, dtype=F64))


def _soup(F, rng):
    v = rng.normal(size=(3 * F, 3)).astype(np.float32)
    return v, np.arange(3 * F, dtype=np.int32).reshape(F, 3)


def test_zero_area_faces_are_never_picked():
    rng = np.random.default_rng(1)
    v, f = _soup(3000, rng)
    zero = np.zeros(3000, bool)
    zero[:40] = True                                                  # a leading run
    zero[1000:1100] = True                                            # a run across no tile boundary
    zero[2040:2060] = True                                            # a run across the tile boundary at 2048
    zero[-5:] = True                                                  # a trailing run
    zero[rng.choice(3000, 200, replace=False)] = True                 # scattered
    f[zero, 1] = f[zero, 0]                                           # repeated vertex: area exactly 0
    out, face = SO.sample_surface(v, f, 200_000, seed=3)
    assert not zero[face].any()
    assert face.min() == np.argmin(zero)                            # the leading run is skipped
    hits = np.bincount(face, minlength=3000)
    area = SO.face_areas(v, f)
    assert (hits[area > 4 * area.sum() / 200_000] > 0).all()        # every face of more than 4 expected hits is hit


def test_all_degenerate_mesh_gives_the_last_face_and_a_zero_normal():
    """Zero total area: the search finds no cumulative area above the target 0, so every sample takes the last face,
    and its normal is 0 (length 0 divides by 1).  The point is that face's (collapsed) vertex position."""
    v = np.array([[0, 0, 0], [1, 2, 3], [4, 5, 6], [7, 8, 9]], np.float32)
    f = np.array([[0, 0, 0], [1, 1, 2], [3, 3, 3]], np.int32)
    out, face = SO.sample_surface(v, f, 1000, seed=11)
    assert np.all(face == 2)
    assert np.all(out[:, 3:] == 0) and np.all(out[:, :3] == np.float16([7, 8, 9]))


def test_sampled_points_and_normals_agree_with_float64_geometry():
    """A sanity check of the restatement itself: every point lies in its triangle, every normal is the face normal."""
    rng = np.random.default_rng(2)
    v, f = _soup(500, rng)
    out, face = SO.sample_surface(v, f, 20_000, seed=9)
    t = v[f[face]].astype(F64)
    a, b, c = t[:, 0], t[:, 1], t[:, 2]
    n = np.cross(b - a, c - a)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    p = out[:, :3].astype(F64)
    assert np.abs(((p - a) * n).sum(1)).max() < 4e-3 * np.abs(t).max()
    assert np.abs(out[:, 3:].astype(F64) - n).max() < 2e-3
    area = SO.face_areas(v, f)
    counts = np.bincount(face, minlength=500)
    pr = area / area.sum()
    assert np.all(np.abs(counts - 20_000 * pr) < 5 * np.sqrt(20_000 * pr * (1 - pr)) + 1)
