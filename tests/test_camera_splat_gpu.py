"""The camera-sample and splat queries on the device (tb200_camera_rays / tb200_splat, Renderer.camera_rays / splat).

Camera rays are compared bit for bit with the CPU restatement's camera samples (tests/camera_oracle.cpp: trace_sample's draws) and
with the raster positions of the renderer's trace_frame, so the query returns the samples the image is made of.
The splat is compared term by term with the restatement's AddSample (oracle_add_samples) on test_splat_gpu's edge
cases, each sample alone in its own film, under the excuses that file allows (a denormal term flushed, +0 == -0, NaN
payloads); summed, against filmref.Film64's summation-order bound.  Then the two are composed with trace_frame,
trace_rays and finish, and the refusals, streams, variants and side effects are those of the other queries."""
import ctypes as C

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import cameraoracle
import filmref
import queryscenes
import refdrv
import test_camera_splat as cpu
import test_splat_gpu as splat_cases

pytestmark = pytest.mark.gpu

F32 = np.float32
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1
TWO30 = F32(2.0 ** 30)


def _torch():
    import torch
    return torch


def _bits_equal(a, b):
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _options(W, H, filter_type=abi.FILTER_GAUSSIAN, width=1.0, falloff=2.0, offset=0.0, clamp=np.inf):
    o = abi.Options()
    o.mode, o.width, o.height = abi.MODE_PATHTRACE, W, H
    o.filterType, o.filterWidth, o.filterFalloff, o.filterOffset = int(filter_type), float(width), float(falloff), float(offset)
    o.clamp, o.maxDepth, o.exposure, o.limit = float(clamp), 4, 1.0, 1.5
    return o


_CAMERAS = []


def _snapshot_cameras():
    """Every snapshot's camera, then test_camera_splat's rotated wide and narrow ones."""
    if _CAMERAS:
        return _CAMERAS
    out = []
    for name in ("cornell", "veach", "motionblur", "meshlight", "glass", "gloss", "many", "mini", "simple", "emitter",
                 "envmini", "furnace", "conservation"):
        snap = tb.Snapshot(tb.scene_path(name))
        out.append((name, snap.camera))
        snap.close()
    _CAMERAS.extend(out + cpu._cameras()[2:])
    return _CAMERAS


def _device_camera_rays(r, cam, W, H, samples):
    torch = _torch()
    s = torch.from_numpy(np.ascontiguousarray(samples, np.int32)).cuda(r.device)
    opt = _options(W, H)
    rays, raster = r.camera_rays(cam, opt, s)
    return rays.cpu().numpy(), raster.cpu().numpy()


def _check_camera_rays(rays, raster, expected, what):
    o, d, t, ras = expected
    want = np.concatenate([o, t[:, None], d, np.where(np.isnan(ras[:, :1]), F32(0), F32(np.inf))], 1).astype(F32)
    bad = ~(_bits_equal(rays, want).all(1) & _bits_equal(raster, ras).all(1))
    if bad.any():
        k = int(np.argmax(bad))
        pytest.fail("%s: %d of %d camera samples differ; first %d: device %r %r, restatement %r %r" % (
            what, int(bad.sum()), bad.size, k, rays[k], raster[k], want[k], ras[k]))


# ---- 1. camera rays, bit for bit ----


@pytest.mark.parametrize("size", [(1, 1), (7, 5), (640, 480), (1024, 1024)])
def test_camera_rays_match_restatement(size):
    W, H = size
    rng = np.random.default_rng(W * 7 + H)
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    npix = W * H
    pixels = np.arange(npix) if npix <= 4096 else rng.integers(0, npix, 1 << 14)
    odd = np.array([-1, npix, INT_MIN, INT_MAX, 0, npix - 1], np.int64)
    for frame in (0, 1, INT_MAX, -1, int(rng.integers(INT_MIN, INT_MAX))):
        px = np.concatenate([pixels, odd])
        s = np.stack([px, np.full(px.size, frame)], 1).astype(np.int32)
        for name, cam in _snapshot_cameras():
            rays, raster = _device_camera_rays(r, cam, W, H, s)
            _check_camera_rays(rays, raster, cameraoracle.camera_samples(cam, W, H, s), "%s %dx%d frame %d" % (name, W, H, frame))
            assert (rays[-6:-2] == 0).all() and np.isnan(raster[-6:-2]).all()
    # random frames per record
    s = np.stack([rng.integers(-2, npix + 2, 4096), rng.integers(INT_MIN, INT_MAX, 4096)], 1).astype(np.int32)
    for name, cam in _snapshot_cameras()[:3]:
        rays, raster = _device_camera_rays(r, cam, W, H, s)
        _check_camera_rays(rays, raster, cameraoracle.camera_samples(cam, W, H, s), "%s random frames" % name)
    r.close()
    snap.close()


# ---- 2. the renderer's own samples ----


@pytest.mark.parametrize("name", ["cornell", "veach", "motionblur"])
def test_camera_rays_are_the_samples_the_image_is_made_of(name):
    snap = tb.Snapshot(tb.scene_path(name))
    cam, opt = snap.camera, snap.options
    W, H = opt.width, opt.height
    r = tb.Renderer(snap.scene)
    r.Init(W, H)
    for frame in (0, 5):
        _, ras = r.trace_frame(cam, opt, frame)
        rays, raster = r.camera_rays(cam, opt, tb.frame_samples(W, H, frame, device="cuda"))
        raster = raster.cpu().numpy()
        assert (raster.view(np.uint32) == ras.reshape(-1, 2).view(np.uint32)).all(), (name, frame)
        assert (rays[:, 7] == float("inf")).all()
    # two frames in one call are the two frames one after the other
    _, r7 = r.trace_frame(cam, opt, 7)
    _, raster = r.camera_rays(cam, opt, tb.frame_samples(W, H, 6, 2, device="cuda"))
    assert (raster[W * H:].cpu().numpy().view(np.uint32) == r7.reshape(-1, 2).view(np.uint32)).all()
    r.close()
    snap.close()


# ---- 3. the splat, term by term ----

CASES_PER_SIZE = 1024


def test_splat_terms_match_restatement():
    """test_splat_gpu's edge cases, each sample alone in its own zeroed film through tb200_splat (whole rows: the
    cases' slabs do not apply), between guard zones that must stay zero."""
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    flushed = cases = 0
    for b, size in enumerate(splat_cases.FILM_SIZES):
        W, H = size
        c = splat_cases.make_cases(20261016 + b, size)[:CASES_PER_SIZE]
        n = c.size
        guard = W * (H + 4)
        films = torch.zeros((n, 2 * guard + W * H, 4), dtype=torch.float32, device="cuda")
        raster = torch.from_numpy(np.stack([c["rasterX"], c["rasterY"]], 1).astype(F32)).cuda()
        radiance = torch.from_numpy(np.stack([c["r"], c["g"], c["b"]], 1).astype(F32)).cuda()
        for k in range(n):
            o = _options(W, H, int(c["filterType"][k]), c["filterWidth"][k], c["filterFalloff"][k], c["filterOffset"][k],
                         c["clamp"][k])
            r.splat(o, raster[k:k + 1], radiance[k:k + 1], films[k, guard:guard + W * H].view(H, W, 4))
        f = films.cpu().numpy()
        assert not f[:, :guard].view(np.uint32).any() and not f[:, guard + W * H:].view(np.uint32).any(), size
        dev = f[:, guard:guard + W * H].reshape(n, H, W, 4)
        params = np.stack([c["filterWidth"], c["filterFalloff"], c["filterOffset"], c["clamp"]], 1)
        samples = np.stack([c["rasterX"], c["rasterY"], c["r"], c["g"], c["b"]], 1)
        ref = refdrv.port_add_samples(W, H, c["filterType"], params, samples)
        denormal = (ref != 0) & (np.abs(ref) < np.finfo(F32).tiny)
        same = _bits_equal(dev, ref) | ((dev == 0) & (ref == 0)) | ((dev == 0) & denormal)
        flushed += int(((dev == 0) & denormal).sum())
        ok = same.reshape(n, -1).all(1)
        if not ok.all():
            k = int(np.argmax(~ok))
            yy, xx, ch = [int(v[0]) for v in np.nonzero(~same[k])]
            pytest.fail("tb200_splat differs from the restatement in %d cases of %dx%d; first %s: pixel (%d, %d) channel "
                        "%d: device %r, restatement %r" % (int((~ok).sum()), W, H, c[k], xx, yy, ch, dev[k, yy, xx, ch],
                                                           ref[k, yy, xx, ch]))
        cases += n
    print("tb200_splat: %d edge cases bit-exact, %d denormal terms flushed" % (cases, flushed))
    r.close()
    snap.close()


# ---- 4. the splat, summed ----

SUM_W, SUM_H = 48, 32


def _summed_samples(rng, n):
    """n samples over the image and a 4-pixel margin around it, an eighth of them on one pixel, with ordinary radiance."""
    ras = np.stack([rng.uniform(-4, SUM_W + 4, n), rng.uniform(-4, SUM_H + 4, n)], 1).astype(F32)
    ras[: n // 8] = (F32(17.25), F32(9.5))   # many samples on one pixel
    rad = np.abs(rng.normal(0.0, 1.5, (n, 3))).astype(F32)
    return ras, rad


@pytest.mark.parametrize("count", [1, 31, 33, 10 ** 6 + 7])
@pytest.mark.parametrize("filter_type", [abi.FILTER_BOX, abi.FILTER_GAUSSIAN])
def test_splat_sums_within_bound(filter_type, count):
    torch = _torch()
    rng = np.random.default_rng(count * 3 + filter_type)
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    ras, rad = _summed_samples(rng, count)
    tras, trad = torch.from_numpy(ras).cuda(), torch.from_numpy(rad).cuda()
    for width in (0.0, 0.5, 1.0, 1.5, 3.0):
        for clamp in (2.0, np.inf):
            o = _options(SUM_W, SUM_H, filter_type, width, 2.25, 0.0 if filter_type == abi.FILTER_BOX else 0.05, clamp)
            acc = torch.zeros((SUM_H, SUM_W, 4), dtype=torch.float32, device="cuda")
            assert r.splat(o, tras, trad, acc) is acc
            ref = filmref.Film64(SUM_W, SUM_H, o).add(ras, rad)
            filmref.assert_film_close(acc.cpu().numpy(), ref, "type %d width %g clamp %g n %d" % (filter_type, width, clamp, count))
            if filter_type == abi.FILTER_BOX and width == 0.0:
                filmref.assert_counts(acc.cpu().numpy(), ref, "counts, n %d" % count)
    r.close()
    snap.close()


def test_splat_skips_unusable_rasters_and_poisons_with_non_finite_radiance():
    """NaN, infinite and 2^30-or-larger raster coordinates are skipped (a NaN one would otherwise land on pixel 0 as
    int(NaN) does on the device); just inside the bound they are splatted, and add nothing because their footprint
    misses the image.  A non-finite radiance poisons its whole footprint, zero-weight pixels included."""
    torch = _torch()
    rng = np.random.default_rng(5)
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    near = np.nextafter(TWO30, F32(0))
    bad = [np.nan, np.inf, -np.inf, TWO30, -TWO30, F32(3e38)]
    ras = [(x, F32(3.5)) for x in bad] + [(F32(3.5), y) for y in bad] + [(near, F32(2.0)), (-near, F32(2.0)), (F32(1.0), near)]
    ras = np.asarray(ras, F32)
    keep = (np.abs(ras) < TWO30).all(1)
    base_ras, base_rad = _summed_samples(rng, 4096)
    for filter_type in (abi.FILTER_BOX, abi.FILTER_GAUSSIAN):
        for width in (0.0, 1.5):
            o = _options(SUM_W, SUM_H, filter_type, width, 3.0, 0.2)
            rad = np.ones((ras.shape[0], 3), F32)
            all_ras, all_rad = np.concatenate([base_ras, ras]), np.concatenate([base_rad, rad])
            acc = torch.zeros((SUM_H, SUM_W, 4), dtype=torch.float32, device="cuda")
            r.splat(o, torch.from_numpy(all_ras).cuda(), torch.from_numpy(all_rad).cuda(), acc)
            mask = np.concatenate([np.ones(base_ras.shape[0], bool), keep])
            ref = filmref.Film64(SUM_W, SUM_H, o).add(all_ras, all_rad, mask)
            filmref.assert_film_close(acc.cpu().numpy(), ref, "unusable rasters, type %d width %g" % (filter_type, width))
            # non-finite radiance: its footprint becomes NaN or inf exactly where the reference's does
            for val in (np.nan, np.inf, -np.inf):
                pr = np.array([[10.7, 6.2], [0.3, 0.9]], F32)
                pv = np.array([[val, 0.0, 1.0], [1.0, val, 0.0]], F32)
                acc.zero_()
                r.splat(o, torch.from_numpy(np.concatenate([base_ras, pr])).cuda(),
                        torch.from_numpy(np.concatenate([base_rad, pv])).cuda(), acc)
                ref = filmref.Film64(SUM_W, SUM_H, o).add(np.concatenate([base_ras, pr]), np.concatenate([base_rad, pv]))
                got = acc.cpu().numpy()
                filmref.assert_film_close(got, ref, "radiance %r, type %d width %g" % (val, filter_type, width))
                assert not np.isfinite(got).all()
    r.close()
    snap.close()


# ---- 5. composition ----


def _small(name, W, H):
    snap = tb.Snapshot(tb.scene_path(name))
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = W, H
    return snap, cam, opt


def test_trace_frame_splatted_matches_the_restatements_film():
    torch = _torch()
    W, H = 64, 48
    snap, cam, opt = _small("cornell", W, H)
    r = tb.Renderer(snap.scene)
    r.Init(W, H)
    port = refdrv.PortScene.from_snapshot(tb.scene_path("cornell"))
    port.set_size(W, H)
    for k in (0, 3):
        rad, ras = r.trace_frame(cam, opt, k)
        acc = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
        r.splat(opt, torch.from_numpy(ras.reshape(-1, 2)).cuda(), torch.from_numpy(rad.reshape(-1, 3)).cuda(), acc)
        prad, pras = port.trace_frame(k, 4)
        ref = filmref.Film64(W, H, opt).add(pras, prad)
        filmref.assert_film_close(acc.cpu().numpy(), ref, "trace_frame(%d) splatted" % k)
        # and what render_device of frame k leaves
        r.Init(W, H)
        r.set_frame(k)
        r.render_device(cam, opt, 1)
        filmref.assert_film_close(r.read_accumulator(), ref, "render_device frame %d" % k)
    port.close()
    r.close()
    snap.close()


def test_camera_rays_trace_rays_splat_of_normals():
    """The documented AOV use: a normal map filtered exactly like the image, from the image's own camera samples."""
    torch = _torch()
    W, H = 40, 30
    for name in ("cornell", "motionblur"):
        snap, cam, opt = _small(name, W, H)
        r = tb.Renderer(snap.scene)
        samples = tb.frame_samples(W, H, 2, device="cuda")
        rays, raster = r.camera_rays(cam, opt, samples)
        hits, prims = r.trace_rays(rays)
        acc = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
        r.splat(opt, raster, hits[:, 1:4].contiguous(), acc)
        port = refdrv.PortScene.from_snapshot(tb.scene_path(name))
        o, d, t, ras = cameraoracle.camera_samples(cam, W, H, samples.cpu().numpy())
        normals = np.zeros((W * H, 3), F32)
        for k in range(W * H):
            _, _, normals[k] = port.trace(o[k], d[k], float(t[k]))
        ref = filmref.Film64(W, H, opt).add(ras, normals)
        filmref.assert_film_close(acc.cpu().numpy(), ref, "%s normals" % name)
        assert (hits[:, 1:4].cpu().numpy().view(np.uint32) == normals.view(np.uint32)).all()
        port.close()
        r.close()
        snap.close()


def test_splat_into_the_renderers_film_then_finish():
    """With a box filter of width 0 a frame gives every pixel at most two terms (its own sample and a neighbour's that
    rounded onto it), whose sum is the same in either order: splatting trace_frame's samples into the renderer's own
    film (accum=None) must leave the accumulator, and finish()'s and nlm()'s outputs, bit for bit as rendering the
    frame does."""
    W, H = 64, 48
    snap, cam, opt = _small("cornell", W, H)
    opt = filmref.counting_options(opt)
    rendered = tb.Renderer(snap.scene)
    rendered.Init(W, H)
    rendered.render_device(cam, opt, 1)
    splatted = tb.Renderer(snap.scene)
    splatted.Init(W, H)
    torch = _torch()
    for k in (0,):
        rad, ras = splatted.trace_frame(cam, opt, k)
        assert splatted.splat(opt, torch.from_numpy(ras.reshape(-1, 2)).cuda(), torch.from_numpy(rad.reshape(-1, 3)).cuda()) is None
    a, b = rendered.read_accumulator(), splatted.read_accumulator()
    assert (a.view(np.uint32) == b.view(np.uint32)).all()
    fa, ba = rendered.finish(1.0, 1.5)
    fb, bb = splatted.finish(1.0, 1.5)
    assert _bits_equal(fa, fb).all() and np.array_equal(ba, bb)
    assert _bits_equal(rendered.nlm(200.0, 1), splatted.nlm(200.0, 1)).all()
    # accum=None needs the size of the last Init
    wrong = abi.copy_struct(opt)
    wrong.width = W + 1
    with pytest.raises(ValueError):
        splatted.splat(wrong, torch.zeros((1, 2), device="cuda"), torch.zeros((1, 3), device="cuda"))
    rendered.close()
    splatted.close()
    snap.close()


# ---- 6. refusals and behaviour ----


@pytest.mark.parametrize("variant", ["cached", "group"])
def test_variants_give_the_same_bits(variant, tmp_path):
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("motionblur"))
    cam, opt = snap.camera, snap.options
    W, H = 96, 64
    opt.width, opt.height = W, H
    plain = tb.Renderer(snap.scene)
    r = queryscenes.variant_renderer(variant, snap, tmp_path)
    s = tb.frame_samples(W, H, 3, device="cuda")
    rad = torch.rand((W * H, 3), device="cuda")
    out = []
    for x in (plain, r):
        rays, raster = x.camera_rays(cam, opt, s)
        acc = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
        o = filmref.counting_options(opt)
        x.splat(o, raster, rad, acc)
        out.append((rays.cpu().numpy(), raster.cpu().numpy(), acc.cpu().numpy()))
    for a, b in zip(*out):
        assert (a.view(np.uint32) == b.view(np.uint32)).all(), variant
    r.close()
    plain.close()
    snap.close()


@pytest.mark.parametrize("count", [0, 1, 31, 33, 10 ** 6 + 7])
def test_counts(count):
    torch = _torch()
    snap, cam, opt = _small("cornell", 1024, 1024)
    r = tb.Renderer(snap.scene)
    rng = np.random.default_rng(count)
    s = np.stack([rng.integers(0, 1 << 20, count), rng.integers(0, 8, count)], 1).astype(np.int32)
    launches = r.stats().kernelLaunches
    rays, raster = r.camera_rays(cam, opt, torch.from_numpy(s).cuda())
    assert tuple(rays.shape) == (count, 8) and tuple(raster.shape) == (count, 2)
    k = np.unique(np.linspace(0, max(count - 1, 0), min(count, 4096)).astype(np.int64)) if count else np.zeros(0, np.int64)
    _check_camera_rays(rays.cpu().numpy()[k], raster.cpu().numpy()[k], cameraoracle.camera_samples(cam, 1024, 1024, s[k]),
                       "count %d" % count)
    acc = torch.zeros((1024, 1024, 4), dtype=torch.float32, device="cuda")
    r.splat(filmref.counting_options(opt), raster, torch.ones((count, 3), device="cuda"), acc)
    # a raster position that rounds onto the right or bottom border has an empty footprint, as in render.cpp
    inside = int((raster[:, 0] < 1024).logical_and(raster[:, 1] < 1024).sum())
    assert float(acc[..., 3].sum()) == inside
    assert r.stats().kernelLaunches == launches + 2 * (count > 0)
    r.close()
    snap.close()


def test_queries_on_the_callers_stream_and_before_init():
    torch = _torch()
    W, H = 128, 96
    snap, cam, opt = _small("veach", W, H)
    r = tb.Renderer(snap.scene)   # never Init
    s = tb.frame_samples(W, H, 0, device="cuda")
    want_rays, want_raster = r.camera_rays(cam, opt, s)
    rad = torch.rand((W * H, 3), device="cuda")
    want = torch.zeros((H, W, 4), device="cuda")
    r.splat(opt, want_raster, rad, want)
    ref = filmref.Film64(W, H, opt).add(want_raster.cpu().numpy(), rad.cpu().numpy())
    filmref.assert_film_close(want.cpu().numpy(), ref, "before Init")
    torch.cuda.synchronize()
    dst = torch.zeros_like(s)
    st = torch.cuda.Stream()
    r.set_stream(st.cuda_stream)
    with torch.cuda.stream(st):
        torch.cuda._sleep(20_000_000)   # the copy lands well after the calls have been queued
        dst.copy_(s)
        rays, raster = r.camera_rays(cam, opt, dst)
        acc = torch.zeros((H, W, 4), device="cuda")
        r.splat(opt, raster, rad, acc)
    st.synchronize()
    r.set_stream(None)
    assert torch.equal(rays.view(torch.int32), want_rays.view(torch.int32))
    assert torch.equal(raster.view(torch.int32), want_raster.view(torch.int32))
    filmref.assert_film_close(acc.cpu().numpy(), ref, "caller's stream")
    r.close()
    snap.close()


def test_no_side_effects():
    torch = _torch()
    W, H = 64, 48
    snap, cam, opt = _small("cornell", W, H)
    r = tb.Renderer(snap.scene)
    r.Init(W, H)
    out = np.zeros((H, W, 4), np.float32)
    r.Render(cam, opt, out)
    acc0, st0, kernel0 = r.read_accumulator(), r.stats(), r.last_kernel()
    rays, raster = r.camera_rays(cam, opt, tb.frame_samples(W, H, 9, device="cuda"))
    st1 = r.stats()
    assert st1.kernelLaunches == st0.kernelLaunches + 1 and st1.gpuMs > 0.0
    r.splat(opt, raster, torch.ones((W * H, 3), device="cuda"), torch.zeros((H, W, 4), device="cuda"))
    st2 = r.stats()
    assert st2.kernelLaunches == st0.kernelLaunches + 2 and st2.gpuMs > 0.0
    assert (st2.frames, st2.samples) == (st0.frames, st0.samples) and r.last_kernel() == kernel0
    assert (r.read_accumulator().view(np.uint32) == acc0.view(np.uint32)).all()
    # the frame counter did not move: the next Render adds frame 1, as a second Render of a fresh renderer does
    r.Render(cam, opt, out)
    other = tb.Renderer(snap.scene)
    other.Init(W, H)
    out2 = np.zeros((H, W, 4), np.float32)
    other.Render(cam, opt, out2)
    other.Render(cam, opt, out2)
    rel = np.linalg.norm((out - out2).astype(np.float64)) / np.linalg.norm(out2.astype(np.float64))
    assert rel < 1e-5, rel
    other.close()
    r.close()
    snap.close()


def test_bad_arguments_are_refused_before_any_launch():
    torch = _torch()
    W, H = 16, 8
    snap, cam, opt = _small("cornell", W, H)
    r = tb.Renderer(snap.scene)
    lib = r.lib
    n = 64
    s = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    rays = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    ras = torch.zeros((n, 2), dtype=torch.float32, device="cuda")
    rad = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
    acc = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
    host = np.zeros((n, 8), np.float32)
    launches = r.stats().kernelLaunches
    cam_p, opt_p = C.byref(cam), C.byref(opt)

    def refused(entry, head, args, count, words):
        assert getattr(lib, entry)(r.h, *head, *args, count) != 0
        msg = tb.last_error()
        assert msg.startswith(entry + ":") and any(w in msg for w in words), msg

    calls = (("tb200_camera_rays", [cam_p, opt_p], [s.data_ptr(), rays.data_ptr(), ras.data_ptr()], [4, 8, 4]),
             ("tb200_splat", [opt_p], [ras.data_ptr(), rad.data_ptr(), acc.data_ptr()], [4, 2, 8]))
    for entry, head, args, skew in calls:
        for k in range(len(args)):
            bad = list(args)
            bad[k] = None
            refused(entry, head, bad, n, ["null"])
            bad[k] = host.ctypes.data
            refused(entry, head, bad, n, ["not device memory"])
            bad[k] = args[k] + skew[k]
            refused(entry, head, bad, n - 1 if k < 2 else n, ["aligned"])
        refused(entry, head, args, -1, ["out of range"])
        assert getattr(lib, entry)(r.h, *head, *[None] * len(args), 0) == 0   # nothing to do: nothing launched
        for w, h in ((0, 8), (16, 0), (-3, 8), (65536, 65536)):
            o = abi.copy_struct(opt)
            o.width, o.height = w, h
            head2 = [cam_p, C.byref(o)] if entry == "tb200_camera_rays" else [C.byref(o)]
            refused(entry, head2, args, n, ["width/height"])
        head2 = [cam_p, None] if entry == "tb200_camera_rays" else [None]
        refused(entry, head2, args, n, ["options is null"])
    refused("tb200_camera_rays", [None, opt_p], calls[0][2], n, ["camera is null"])
    for field, value in splat_cases.BAD_OPTIONS:
        o = abi.copy_struct(opt)
        setattr(o, field, value)
        refused("tb200_splat", [C.byref(o)], calls[1][2], n, ["filter"])
        # the camera rays read the image size only
        assert lib.tb200_camera_rays(r.h, cam_p, C.byref(o), *calls[0][2], n) == 0
        launches += 1
    assert lib.tb200_splat(None, opt_p, *calls[1][2], n) != 0 and "null renderer" in tb.last_error()
    assert lib.tb200_camera_rays(None, cam_p, opt_p, *calls[0][2], n) != 0 and "null renderer" in tb.last_error()
    # spans past the end: tensors that own their segments (a fresh 24 MiB tensor gets a segment of its own)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    big_n = (24 << 20) // 8
    big_s = torch.zeros((big_n, 2), dtype=torch.int32, device="cuda")
    big_rays = torch.empty((big_n + 1, 8), dtype=torch.float32, device="cuda")
    big_ras = torch.empty((big_n + 1, 2), dtype=torch.float32, device="cuda")
    refused("tb200_camera_rays", [cam_p, opt_p], [big_s.data_ptr(), big_rays.data_ptr(), big_ras.data_ptr()], big_n + 1,
            ["past the end"])
    big_acc = torch.zeros((1024 * 1536 * 4,), dtype=torch.float32, device="cuda")   # 24 MiB: a 1024 x 1536 film
    o = abi.copy_struct(opt)
    o.width, o.height = 1025, 1536
    refused("tb200_splat", [C.byref(o)], [ras.data_ptr(), rad.data_ptr(), big_acc.data_ptr()], n, ["accum", "past the end"])
    assert "accum" in tb.last_error() and "past the end" in tb.last_error()
    assert r.stats().kernelLaunches == launches
    # a foreign device's memory
    if torch.cuda.device_count() > 1:
        other = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda:1")
        refused("tb200_splat", [opt_p], [ras.data_ptr(), rad.data_ptr(), other.data_ptr()], n, ["lies on device"])
    # the Python interface checks shapes, dtypes, contiguity and the device itself
    with pytest.raises(TypeError):
        r.camera_rays(cam, opt, s.long())
    with pytest.raises(ValueError):
        r.camera_rays(cam, opt, s.cpu())
    with pytest.raises(ValueError):
        r.splat(opt, ras, rad[:n - 1])
    with pytest.raises(ValueError):
        r.splat(opt, ras, rad, torch.zeros((H, W + 1, 4), device="cuda"))
    with pytest.raises(ValueError):
        r.splat(opt, ras, rad, torch.zeros((W, H, 4), device="cuda").transpose(0, 1))
    with pytest.raises(ValueError):   # never Init: no film of this size
        r.splat(opt, ras, rad)
    r.close()
    snap.close()
