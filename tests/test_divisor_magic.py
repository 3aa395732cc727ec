"""The kernels decode a sample index with a multiply and a shift instead of dividing by the launch's samples per
frame and tile columns (kernels.cu: divisor_magic, decode_sample).  The host's multipliers, applied the way the
device applies them, must give plain division's quotient for every 32-bit index: checked here for every tile
column count up to 2^16 and a sample of larger ones up to what tb200_init accepts, and for a wide sample of
samples-per-frame values, at edge and random indices."""
import ctypes as C

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import build

U32_MAX = (1 << 32) - 1
MAX_TILES_X = ((1 << 31) - 1 + 7) >> 3   # tb200_init takes any positive int width


@pytest.fixture(scope="module")
def lib():
    if build.needs_build():
        build.build_native()
    return tb.load_library()


def magic(lib, d):
    mul, shift = C.c_uint(), C.c_uint()
    lib.tb200_divisor_magic(d, C.byref(mul), C.byref(shift))
    return mul.value, shift.value


def device_div(n, mul, shift):
    """(__umulhi(n, mul) + n) >> shift, the sum in 64 bits (kernels.cu: div_magic)."""
    n = n.astype(np.uint64)
    return (((n * np.uint64(mul)) >> np.uint64(32)) + n) >> np.uint64(shift)


def indices(d, rng, randoms=64):
    """0, 1, multiples of d and their neighbours (near 0, near 2^31 and near 2^32), 2^32 - 1, random indices."""
    d = int(d)
    edge = {0, 1, 2, U32_MAX, U32_MAX - 1, 1 << 31, (1 << 31) - 1}
    for k in (1, 2, 3, 7, (1 << 31) // d, U32_MAX // d - 1, U32_MAX // d):
        for e in (-1, 0, 1):
            edge.add(k * d + e)
    edge = [v for v in edge if 0 <= v <= U32_MAX]
    return np.concatenate([np.array(edge, np.uint64), rng.integers(0, 1 << 32, randoms, dtype=np.uint64)])


def check(lib, divisors, rng, randoms=64):
    for d in divisors:
        mul, shift = magic(lib, int(d))
        n = indices(d, rng, randoms)
        q = device_div(n, mul, shift)
        bad = np.nonzero(q != n // np.uint64(d))[0]
        assert bad.size == 0, "d=%d mul=%d shift=%d: n=%d gives %d" % (d, mul, shift, n[bad[0]], q[bad[0]])


def test_zero_divisor_gives_zero(lib):
    assert magic(lib, 0) == (0, 0)


def test_every_tile_column_count_up_to_2_16(lib):
    check(lib, range(1, (1 << 16) + 1), np.random.default_rng(1), randoms=16)


def test_large_tile_column_counts(lib):
    rng = np.random.default_rng(2)
    ds = {MAX_TILES_X, MAX_TILES_X - 1}
    for k in range(16, 29):
        ds.update({(1 << k) - 1, 1 << k, (1 << k) + 1})
    ds.update(int(v) for v in rng.integers(1 << 16, MAX_TILES_X + 1, 2000))
    check(lib, sorted(d for d in ds if 1 <= d <= MAX_TILES_X), rng)


def test_samples_per_frame(lib):
    """tilesX * tileRows * 32: multiples of 32 in practice, but every divisor is checked the same way."""
    rng = np.random.default_rng(3)
    ds = set()
    for k in range(0, 32):
        ds.update({(1 << k) - 1, 1 << k, (1 << k) + 1})
    ds.update({U32_MAX, U32_MAX - 1, 1024 * 1024, 1920 * 1088, 3840 * 2160 // 32 * 32})
    ds.update(32 * int(v) for v in rng.integers(1, 1 << 26, 2000))
    ds.update(int(v) for v in rng.integers(1, 1 << 32, 2000, dtype=np.uint64))
    check(lib, sorted(d for d in ds if 1 <= d <= U32_MAX), rng)
