"""The film's splat on the device (tb_film.cuh: add_sample, add_sample_small) against the CPU restatement's AddSample
(render.cpp:401-445), one term per pixel, bit for bit; and the filter options the renderer refuses.

tests/splat_harness.cu runs one case per thread, each into its own film between zeroed guard zones, so every pixel
receives at most one term and the device's value is that term itself.  For every case:
  1. add_sample_small gives add_sample's bits (NaN compared as NaN);
  2. add_sample gives the restatement's bits per pixel, except that a denormal term reads as zero on the device (the
     L2 adder flushes it, tb_film.cuh: accum_add), +0 and -0 are equal and NaN payloads are not compared; rows
     outside the case's slab [rowLo, rowHi) stay zero;
  3. the filterArgZero shortcut (film_filter_arg_zero, the rule fill_params applies) gives the bits of no shortcut.
The cases are drawn from the edges where the splat can go wrong: raster positions on and one ulp beside the integers
where int(raster +- width) flips, widths on and beside 1, steep and degenerate falloffs, offsets outside (0, 1),
clamps of 0 and NaN, samples whose length or weighted value overflows, non-finite channels, tiny films and slabs."""
import ctypes as C

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import cuda_harness
import refdrv

# struct SplatCase in splat_harness.cu
CASE_DTYPE = np.dtype([("width", "<i4"), ("height", "<i4"), ("filterType", "<i4"), ("rowLo", "<i4"), ("rowHi", "<i4"),
                       ("filterWidth", "<f4"), ("filterFalloff", "<f4"), ("filterOffset", "<f4"), ("clamp", "<f4"),
                       ("filterArgZero", "<f4"), ("rasterX", "<f4"), ("rasterY", "<f4"), ("r", "<f4"), ("g", "<f4"),
                       ("b", "<f4"), ("pad", "<f4")])
ADD_SAMPLE, ADD_SAMPLE_SMALL, ADD_SAMPLE_NO_SHORTCUT = 0, 1, 2

FILM_SIZES = [(1, 1), (1, 5), (5, 1), (3, 3), (4, 4), (9, 7)]
BATCH = 1 << 16
BATCHES = 16   # 2^20 cases
F32 = np.float32
INF = F32(np.inf)

# ---- the harness ----


def harness_path():
    return cuda_harness.harness_path("splat_harness")


_harness = None


def harness():
    global _harness
    if _harness is None:
        lib = C.CDLL(harness_path())
        lib.splat_filter_arg_zero.restype = None
        lib.splat_filter_arg_zero.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int]
        lib.splat_run.restype = C.c_int
        lib.splat_run.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.c_longlong, C.c_int]
        _harness = lib
    return _harness


def arg_zero(offsets):
    offsets = np.ascontiguousarray(offsets, F32)
    out = np.empty_like(offsets)
    harness().splat_filter_arg_zero(offsets.ctypes.data_as(C.POINTER(C.c_float)), out.ctypes.data_as(C.POINTER(C.c_float)),
                                    offsets.size)
    return out


# ---- the cases ----


def _pick(rng, n, edges, uniform, p_edge=0.8):
    """n values: from `edges` with probability p_edge, else from uniform(rng, n)."""
    edges = np.asarray(edges, F32)
    v = edges[rng.integers(0, edges.size, n)]
    u = uniform(n).astype(F32)
    return np.where(rng.random(n) < p_edge, v, u).astype(F32)


def _raster(rng, n, size, w):
    """Positions along one axis of `size` pixels: integers, one ulp either side, half-integers, k +- width exactly
    and one ulp beside it (where int(r +- w) flips), 0, the far border exactly, and uniform draws."""
    k = rng.integers(0, size + 1, n).astype(F32)
    up, down = np.nextafter(k, INF), np.nextafter(k, -INF)
    kpw, kmw = (k + w).astype(F32), (k - w).astype(F32)
    kinds = [k, up, down, k + F32(0.5), kpw, np.nextafter(kpw, INF), np.nextafter(kpw, -INF), kmw,
             np.nextafter(kmw, INF), np.nextafter(kmw, -INF), np.zeros(n, F32), np.full(n, size, F32),
             (rng.random(n) * size).astype(F32)]
    pick = rng.integers(0, len(kinds), n)
    return np.choose(pick, kinds).astype(F32)


def make_cases(seed, size):
    """BATCH cases on films of `size` (W, H), from numpy's generator seeded with `seed`."""
    W, H = size
    n = BATCH
    rng = np.random.default_rng(seed)
    c = np.zeros(n, CASE_DTYPE)
    c["width"], c["height"] = W, H
    c["filterType"] = np.where(rng.random(n) < 0.25, abi.FILTER_BOX, abi.FILTER_GAUSSIAN)
    one = F32(1.0)
    w = _pick(rng, n, [0.0, 0.25, 0.5, 0.75, np.nextafter(one, F32(0)), 1.0, np.nextafter(one, INF), 1.5, 2.0, 3.5,
                       -1e-7, -0.25, -1.0], lambda m: rng.random(m) * 3.5)
    c["filterWidth"] = w
    c["filterFalloff"] = _pick(rng, n, [1.0, 1.0, 3.0, 9.0, 0.0, -1.0, 1e30, np.nan], lambda m: rng.random(m) * 10.0)
    offset = _pick(rng, n, [0.569782853, 0.569782853, 0.0, 0.1, 0.999, 1.0, 1.5, -0.5, 1e-40, np.nan],
                   lambda m: rng.random(m))
    c["clamp"] = _pick(rng, n, [np.inf, np.inf, 0.75, 0.0, 1e-30, np.nan], lambda m: rng.random(m) * 4.0)
    c["rasterX"] = _raster(rng, n, W, w)
    c["rasterY"] = _raster(rng, n, H, w)
    # samples: ordinary, zero, negative, denormal, 1e30 (the length overflows), 3e38 (with a negative offset the
    # weights exceed 1 and the terms overflow), and +-inf or NaN in one channel
    s = rng.normal(0.0, 2.0, (n, 3)).astype(F32)
    kind = rng.integers(0, 9, n)
    s[kind == 1] = 0.0
    s[kind == 2] = -np.abs(s[kind == 2])
    s[kind == 3] = (s[kind == 3] * F32(1e-39)).astype(F32)
    s[kind == 4] = (np.sign(s[kind == 4]) * F32(1e30)).astype(F32)
    s[kind == 5] = F32(3e38)
    offset[(kind == 5) & (rng.random(n) < 0.5)] = -0.5
    ch = rng.integers(0, 3, n)
    rows = np.arange(n)
    for kk, val in ((6, np.inf), (7, -np.inf), (8, np.nan)):
        m = kind == kk
        s[rows[m], ch[m]] = val
    c["r"], c["g"], c["b"] = s[:, 0], s[:, 1], s[:, 2]
    c["filterOffset"] = offset
    # slabs: the whole image, the first, last or middle row, an empty one, and one far from the footprint
    slab = rng.integers(0, 6, n)
    ry = c["rasterY"]
    mid = H // 2
    far = np.where(ry < H / 2.0, H - 1, 0)
    lo = np.choose(slab, [np.zeros(n, int), np.zeros(n, int), np.full(n, H - 1), np.full(n, mid), np.full(n, mid), far])
    hi = np.choose(slab, [np.full(n, H), np.ones(n, int), np.full(n, H), np.full(n, mid + 1), np.full(n, mid), far + 1])
    c["rowLo"], c["rowHi"] = lo, hi
    c["filterArgZero"] = arg_zero(c["filterOffset"])
    return c


def all_batches():
    """The 2^20 cases, as (film size, cases) batches."""
    for b in range(BATCHES):
        size = FILM_SIZES[b % len(FILM_SIZES)]
        yield size, make_cases(20261016 + b, size)


def _trunc(x):
    return np.trunc(x).astype(np.int64)


def classify(c):
    """The case classes, from the kernel's own predicates (tb_film.cuh), as boolean masks."""
    with np.errstate(all="ignore"):
        W, H = c["width"].astype(np.int64), c["height"].astype(np.int64)
        rx, ry, w = c["rasterX"], c["rasterY"], c["filterWidth"]
        lo_x, hi_x, lo_y, hi_y = _trunc(rx - w), _trunc(rx + w), _trunc(ry - w), _trunc(ry + w)
        sx, sy = np.maximum(0, lo_x), np.maximum(c["rowLo"], lo_y)
        ex, ey = np.minimum(hi_x, W - 1), np.minimum(hi_y, c["rowHi"] - 1)
        s = np.stack([c["r"], c["g"], c["b"]], 1)
        l = np.sqrt((s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2])
        clamped = np.where((l > c["clamp"])[:, None], s * (c["clamp"] / l)[:, None], s)
        finite = np.isfinite(clamped).all(1)
        gauss = c["filterType"] == abi.FILTER_GAUSSIAN
        empty = (sx > ex) | (sy > ey)
        # some column or row of the footprint has an argument below filterArgZero
        cut = np.zeros(c.size, bool)
        for start, end, r in ((sx, ex, rx), (sy, ey, ry)):
            for k in range(12):
                d = (start + k).astype(F32) - r
                a = -c["filterFalloff"] * d * d
                cut |= (start + k <= end) & (a < c["filterArgZero"])
        return {
            "fast path": gauss & finite & (ex - sx <= 2) & (ey - sy <= 2),
            "wider than 3": gauss & finite & ((ex - sx > 2) | (ey - sy > 2)),
            "box": ~gauss,
            "non-finite": gauss & ~finite,
            "clipped left": lo_x < 0,
            "clipped right": hi_x > W - 1,
            "clipped top": lo_y < 0,
            "clipped bottom": hi_y > H - 1,
            "empty footprint": empty,
            "slab-clipped": ~empty & (((lo_y < c["rowLo"]) & (c["rowLo"] > 0)) | ((hi_y > c["rowHi"] - 1) & (c["rowHi"] < H))),
            "shortcut active": gauss & ~empty & cut,
        }


MIN_PER_CLASS = 5000


def test_harness_compiles_for_sm90a():
    """The harness against the headers as they are (no GPU needed): a header change that breaks it fails here."""
    harness_path()
    z = arg_zero([0.569782853, 0.0, 1.0, np.nan, 0.5])
    assert np.isneginf(z[1:4]).all() and z[0] < 0 and z[4] < 0


def test_case_coverage():
    """Every class of case occurs often enough, so that an edit to the generator cannot quietly drop one."""
    counts = None
    for _, c in all_batches():
        k = {name: int(m.sum()) for name, m in classify(c).items()}
        counts = k if counts is None else {name: counts[name] + k[name] for name in counts}
    print("splat cases per class: %s" % counts)
    low = {name: v for name, v in counts.items() if v < MIN_PER_CLASS}
    assert not low, low


def test_oracle_add_samples_export():
    """oracle_add_samples against AddSample written out here for a few plain cases."""
    t = np.array([abi.FILTER_BOX, abi.FILTER_GAUSSIAN, abi.FILTER_GAUSSIAN], np.int32)
    p = np.array([[1.0, 1.0, 0.5, np.inf], [1.0, 1.0, 0.1, np.inf], [0.5, 2.0, 0.0, 1.0]], F32)
    s = np.array([[2.5, 1.25, 1.0, 2.0, 3.0], [0.0, 0.0, 1.0, 1.0, 1.0], [3.9, 3.5, 3.0, 4.0, 0.0]], F32)
    films = refdrv.port_add_samples(4, 4, t, p, s)
    assert (films[0, 0:3, 1:4] == [1, 2, 3, 1]).all() and films[0].sum() == 9 * 7
    gx = np.maximum(F32(0), np.exp(-np.array([0.0, 1.0], np.float64)) - 0.1)
    w = np.outer(gx, gx)
    assert np.allclose(films[1, 0:2, 0:2, 3], w, rtol=1e-6) and films[1, 2:].sum() == 0
    assert (films[2, :, :, :3].max() <= 0.8) and np.count_nonzero(films[2, ..., 3]) == 1


# ---- the GPU side ----


def _bits_equal(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _run(cases_t, n, size, mode):
    import torch
    W, H = size
    guard = W * (H + 4)   # two rows of overrun from a 3x3 loop fit inside
    stride = 2 * guard + W * H
    films = torch.zeros((n, stride, 4), dtype=torch.float32, device="cuda")
    rc = harness().splat_run(cases_t.data_ptr(), n, films.data_ptr(), stride, guard, mode)
    assert rc == 0, "splat_run: cudaError %d" % rc
    return films, guard


@pytest.mark.gpu
def test_splat_matches_restatement():
    import torch
    counts = {}
    flushed = 0
    for size, c in all_batches():
        W, H = size
        n = c.size
        cases_t = torch.from_numpy(c.view(np.uint8)).cuda()
        films = {}
        for mode in (ADD_SAMPLE, ADD_SAMPLE_SMALL, ADD_SAMPLE_NO_SHORTCUT):
            f, guard = _run(cases_t, n, size, mode)
            gz = torch.cat([f[:, :guard], f[:, guard + W * H:]], 1)
            bad = (gz.view(torch.int32) != 0).any(2).any(1)
            assert not bool(bad.any()), "mode %d: %d cases of %dx%d wrote outside their film, first %s" % (
                mode, int(bad.sum()), W, H, c[int(torch.nonzero(bad)[0])])
            films[mode] = f[:, guard:guard + W * H].cpu().numpy().reshape(n, H, W, 4)
        dev = films[ADD_SAMPLE]
        for mode, what in ((ADD_SAMPLE_SMALL, "add_sample_small"), (ADD_SAMPLE_NO_SHORTCUT, "add_sample without the shortcut")):
            same = _bits_equal(films[mode], dev).reshape(n, -1).all(1)
            assert same.all(), "%s differs from add_sample in %d cases of %dx%d, first %s" % (
                what, int((~same).sum()), W, H, c[int(np.argmax(~same))])
        params = np.stack([c["filterWidth"], c["filterFalloff"], c["filterOffset"], c["clamp"]], 1)
        samples = np.stack([c["rasterX"], c["rasterY"], c["r"], c["g"], c["b"]], 1)
        ref = refdrv.port_add_samples(W, H, c["filterType"], params, samples)
        y = np.arange(H)[None, :]
        ref[~((y >= c["rowLo"][:, None]) & (y < c["rowHi"][:, None]))] = 0.0
        denormal = (ref != 0) & (np.abs(ref) < np.finfo(F32).tiny)
        same = _bits_equal(dev, ref) | ((dev == 0) & (ref == 0)) | ((dev == 0) & denormal)
        flushed += int(((dev == 0) & denormal).sum())
        ok = same.reshape(n, -1).all(1)
        if not ok.all():
            k = int(np.argmax(~ok))
            yy, xx, ch = [int(v[0]) for v in np.nonzero(~same[k])]
            pytest.fail("add_sample differs from the restatement in %d cases of %dx%d; first %s: pixel (%d, %d) channel %d: "
                        "device %r, restatement %r" % (int((~ok).sum()), W, H, c[k], xx, yy, ch, dev[k, yy, xx, ch],
                                                       ref[k, yy, xx, ch]))
        for name, m in classify(c).items():
            counts[name] = counts.get(name, 0) + int(m.sum())
    print("splat: %d cases bit-exact; per class %s; %d denormal terms flushed to zero" % (BATCH * BATCHES, counts, flushed))


# ---- options the renderer refuses ----

BAD_OPTIONS = [("filterType", 2), ("filterType", -1), ("filterWidth", float("nan")), ("filterWidth", float("inf")),
               ("filterWidth", float("-inf")), ("filterWidth", 2.0 ** 30), ("filterWidth", -2.0 ** 30), ("filterWidth", 1e30)]


@pytest.mark.gpu
def test_filter_options_that_would_read_differently_are_refused():
    """A filter type other than box or Gaussian, or a width that is not finite or reaches 2^30: every call that takes
    options raises, launches nothing and leaves the accumulator as it was.  A width just below 2^30 is accepted (a
    box that covers the whole image from every sample), and valid options render afterwards."""
    size = (24, 16)
    snap = tb.Snapshot(tb.scene_path("cornell"))
    cam, good = snap.camera, snap.options
    good.width, good.height = size
    r = tb.Renderer(snap.scene)
    r.Init(*size)
    r.render_device(cam, good, 1)
    out = np.zeros((size[1], size[0], 4), np.float32)
    for field, value in BAD_OPTIONS:
        bad = abi.copy_struct(good)
        setattr(bad, field, value)
        calls = [("Render", lambda: r.Render(cam, bad, out)), ("render_device", lambda: r.render_device(cam, bad, 1)),
                 ("render_n", lambda: r.render_n(cam, bad, 2, out)), ("trace_frame", lambda: r.trace_frame(cam, bad, 0))]
        for name, call in calls:
            before, st = r.read_accumulator(), r.stats()
            with pytest.raises(tb.TinselB200Error, match="filter"):
                call()
            after, st2 = r.read_accumulator(), r.stats()
            what = "%s with %s = %r" % (name, field, value)
            assert (st2.kernelLaunches, st2.frames) == (st.kernelLaunches, st.frames), what
            assert (after.view(np.uint32) == before.view(np.uint32)).all(), what
    f0 = r.stats().frames
    r.render_device(cam, good, 1)
    assert r.stats().frames == f0 + 1 and np.isfinite(r.read_accumulator()).all()
    # the largest width below the bound: every sample's box covers the whole image
    wide = abi.copy_struct(good)
    wide.filterType, wide.filterWidth = abi.FILTER_BOX, float(np.nextafter(F32(2.0 ** 30), F32(0)))
    r.Init(*size)
    r.render_device(cam, wide, 1)
    assert (r.read_accumulator()[..., 3] == size[0] * size[1]).all()
    r.close()
    snap.close()
