"""A float64 reference of the framebuffer: CpuRenderer::AddSample (render.cpp:401-445) with Filter::Eval
(render.h:13-39), vectorised with numpy, and the comparison a GPU accumulator must pass against it.

Every splat term is evaluated in float32 in the kernel's order of operations (tb_film.cuh: add_sample), so
the terms are the reference's own; only their sum is taken in float64.  The one freedom a GPU film has is
the order of its fp32 additions (plus the flush to zero of the L2 vector adder), and both are bounded:

    |gpu - ref| <= (n + 4) * 2^-24 * sum|term| + 2 n * 2^-126

per pixel and channel, with n the number of terms the pixel received.  (n - 1) * 2^-24 * sum|term| bounds
any order of an fp32 sum of n terms; the 5 extra units cover expf, which the reference here takes as
float32(exp(float64(x))) where tbm_expf is correctly rounded except for about 1e-7 of its arguments.  Each
flushed denormal loses less than 2^-126, at most two per addition.

The reference follows the reference renderer, not the kernel's shortcuts: it skips no zero-weight term and
has no zero-band cut-off, so a non-finite sample poisons every pixel of its footprint, as in render.cpp.

TEST INFRASTRUCTURE: only tests/ import this."""
import numpy as np

from tinsel_b200 import abi

U = 2.0 ** -24        # unit roundoff of fp32
TINY = 2.0 ** -126    # smallest normal fp32


class Film64:
    """Running float64 sums of a film: sums (H,W,4), abs (H,W,4) = per-channel sum of |term|, n (H,W) =
    terms per pixel, samples = samples splatted (lost ones included, see add)."""

    def __init__(self, width, height, options):
        self.width, self.height = int(width), int(height)
        self.filter_type = int(options.filterType)
        self.fw = np.float32(options.filterWidth)
        self.falloff = np.float32(options.filterFalloff)
        self.offset = np.float32(options.filterOffset)
        self.clamp = np.float32(options.clamp)
        npix = self.width * self.height
        self._sums = np.zeros((4, npix))
        self._abs = np.zeros((4, npix))
        self._n = np.zeros(npix, np.int64)
        self.samples = 0

    @property
    def sums(self):
        return self._sums.T.reshape(self.height, self.width, 4)

    @property
    def abs(self):
        return self._abs.T.reshape(self.height, self.width, 4)

    @property
    def n(self):
        return self._n.reshape(self.height, self.width)

    def copy(self):
        c = Film64.__new__(Film64)
        c.__dict__.update(self.__dict__)
        c._sums, c._abs, c._n = self._sums.copy(), self._abs.copy(), self._n.copy()
        return c

    def _weights(self, pos, start, k):
        """Per-axis Gaussian weight of footprint offset k (render.h:29-32): max(0, expf((-falloff*d)*d) - offset)."""
        d = (start + k).astype(np.float32) - pos
        arg = (-self.falloff * d) * d
        e = np.exp(arg.astype(np.float64)).astype(np.float32)
        return np.maximum(np.float32(0.0), e - self.offset)

    def add(self, raster, radiance, sample_mask=None):
        """Splats samples: raster (..., 2) and radiance (..., 3) float32, one sample per row; sample_mask
        (...) bool keeps a subset.  A sample whose footprint is empty (raster position rounded onto the
        right or bottom border) counts in `samples` and adds nothing, as in render.cpp."""
        raster = np.asarray(raster, np.float32).reshape(-1, 2)
        radiance = np.asarray(radiance, np.float32).reshape(-1, 3)
        if sample_mask is not None:
            m = np.asarray(sample_mask, bool).reshape(-1)
            raster, radiance = raster[m], radiance[m]
        self.samples += raster.shape[0]
        W, H = self.width, self.height
        rx, ry = raster[:, 0], raster[:, 1]
        with np.errstate(all="ignore"):
            # footprint: int() truncates toward zero (render.cpp:404-407)
            sx = np.maximum(0, (rx - self.fw).astype(np.int64))
            sy = np.maximum(0, (ry - self.fw).astype(np.int64))
            ex = np.minimum((rx + self.fw).astype(np.int64), W - 1)
            ey = np.minimum((ry + self.fw).astype(np.int64), H - 1)
            # ClampLength (maths.h:1577-1589): length = sqrt((x*x + y*y) + z*z), then sample * (clamp / l)
            x, y, z = radiance[:, 0], radiance[:, 1], radiance[:, 2]
            l = np.sqrt((x * x + y * y) + z * z)
            big = l > self.clamp
            c = np.where(big[:, None], radiance * (self.clamp / l)[:, None], radiance)
            kx = int((ex - sx).max(initial=-1)) + 1
            ky = int((ey - sy).max(initial=-1)) + 1
            box = self.filter_type == abi.FILTER_BOX
            gxs = [None if box else self._weights(rx, sx, i) for i in range(kx)]
            gys = [None if box else self._weights(ry, sy, j) for j in range(ky)]
            for i in range(kx):
                for j in range(ky):
                    m = (sx + i <= ex) & (sy + j <= ey)
                    if not m.any():
                        continue
                    idx = (sy[m] + j) * W + (sx[m] + i)
                    cm = c[m]
                    if box:
                        w = np.ones(cm.shape[0], np.float32)
                        terms = [cm[:, 0], cm[:, 1], cm[:, 2], w]
                    else:
                        w = gxs[i][m] * gys[j][m]
                        terms = [cm[:, 0] * w, cm[:, 1] * w, cm[:, 2] * w, w]
                    for ch, t in enumerate(terms):
                        t = t.astype(np.float64)
                        self._sums[ch] += np.bincount(idx, weights=t, minlength=W * H)
                        if ch < 3:
                            self._abs[ch] += np.bincount(idx, weights=np.abs(t), minlength=W * H)
                    self._n += np.bincount(idx, minlength=W * H)
            self._abs[3] = self._sums[3]   # weights are never negative
        return self

    def __iadd__(self, other):
        assert (other.width, other.height) == (self.width, self.height)
        self._sums += other._sums
        self._abs += other._abs
        self._n += other._n
        self.samples += other.samples
        return self


def films_of_frames(width, height, options_list, trace, frames, threads=None, sample_mask=None):
    """One Film64 per entry of options_list, of the samples trace(frame) -> (radiance, raster) returns for
    every frame in `frames`.  `threads` workers trace and splat frames side by side (the tracer and
    numpy's bincount release the GIL); trace(frame) must be safe to call from several threads."""
    import os
    from concurrent.futures import ThreadPoolExecutor
    frames = list(frames)
    threads = max(1, min(threads or min(os.cpu_count() or 8, 32), len(frames)))

    def work(k):
        films = [Film64(width, height, o) for o in options_list]
        for f in frames[k::threads]:
            rad, ras = trace(f)
            for film in films:
                film.add(ras, rad, sample_mask)
        return films

    with ThreadPoolExecutor(threads) as ex:
        parts = list(ex.map(work, range(threads)))
    out = parts[0]
    for p in parts[1:]:
        for a, b in zip(out, p):
            a += b
    return out


def splat64(width, height, raster, radiance, options, sample_mask=None):
    """float64 sums (H,W,4), per-channel sum of |term| (H,W,4) and term count n (H,W) of the samples."""
    f = Film64(width, height, options).add(raster, radiance, sample_mask)
    return f.sums, f.abs, f.n


def film_error(gpu, ref):
    """(worst error / bound over every finite value, description of the first violation or None).
    `ref` is a Film64 or the (sums, abs, n) triple of splat64."""
    sums, absum, n = (ref.sums, ref.abs, ref.n) if isinstance(ref, Film64) else ref
    gpu = np.asarray(gpu, np.float32).astype(np.float64)
    assert gpu.shape == sums.shape, (gpu.shape, sums.shape)
    for name, cls in (("NaN", np.isnan), ("+inf", np.isposinf), ("-inf", np.isneginf)):
        a, b = cls(gpu), cls(sums)
        if not np.array_equal(a, b):
            yx = np.argwhere(a != b)[0]
            return np.inf, "%s mask differs at %d values, first (y, x, channel) %s: gpu %r, reference %r" % (
                name, int((a != b).sum()), tuple(int(v) for v in yx), gpu[tuple(yx)], sums[tuple(yx)])
    fin = np.isfinite(sums)
    nn = np.broadcast_to(n[..., None], sums.shape).astype(np.float64)
    bound = np.where(fin, (nn + 4.0) * U * np.where(fin, absum, 0.0) + 2.0 * nn * TINY, 0.0)
    err = np.where(fin, np.abs(gpu - np.where(fin, sums, 0.0)), 0.0)
    over = err > bound
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))
    worst = float(ratio.max(initial=0.0))
    if over.any():
        yx = tuple(int(v) for v in np.unravel_index(int(np.argmax(ratio)), ratio.shape))
        return worst, "%d values off by more than the bound; worst at (y, x, channel) %s: gpu %r, reference %r, bound %.3g (n=%d)" % (
            int(over.sum()), yx, gpu[yx], sums[yx], bound[yx], int(nn[yx]))
    return worst, None


def assert_film_close(gpu, ref, what=""):
    """Same NaN / +inf / -inf masks per channel, every finite value within the summation-order bound.
    Prints and returns the worst error-to-bound ratio, so that a loss of headroom is visible."""
    worst, bad = film_error(gpu, ref)
    print("film %-48s worst error/bound %.3f" % (what, worst))
    assert bad is None, "%s: %s" % (what, bad)
    return worst


def assert_counts(gpu, ref, what=""):
    """Counting mode (box filter of width 0: every sample adds exactly 1.0 to one pixel's weight): the
    weight channel must equal the reference's term counts bit for bit."""
    n = ref.n if isinstance(ref, Film64) else np.asarray(ref)
    w = np.asarray(gpu)[..., 3]
    bad = w != n.astype(np.float32)
    assert not bad.any(), "%s: %d pixels hold another sample count, first (y, x) %s: %r instead of %d" % (
        what, int(bad.sum()), tuple(int(v) for v in np.argwhere(bad)[0]), float(w[bad][0]), int(n[bad][0]))


def counting_options(options):
    """A copy of `options` in counting mode: box filter of width 0."""
    o = abi.copy_struct(options)
    o.filterType = abi.FILTER_BOX
    o.filterWidth = 0.0
    return o
