"""Display/finish step (SURVEY 8f rank 1; src/main.cpp:262-271, util.h:25-42, maths.h:1545-1555,
src/png.cpp:324-343).  CPU part: the restatement oracle/tinsel_oracle.cpp against the golden
vectors produced by the reference's own ToneMap / LinearToSrgb / WritePng (tools/make_golden.py,
detmath flavour) and, when oracle/_ref is present, against the reference directly -- bit for bit.
GPU part: tb200_finish / tb200_render_n through the C ABI against the same."""
import os
import subprocess

import numpy as np
import pytest

import tinsel_b200 as tb
import refdrv
import schedenv

GOLD = os.path.join(refdrv.ROOT, "tests", "golden", "finish.npz")


@pytest.fixture(autouse=True)
def default_knobs():
    with schedenv.knobs():
        yield


@pytest.fixture(scope="module", autouse=True)
def port_built():
    subprocess.check_call(["make", "-s", "-C", os.path.join(refdrv.ROOT, "oracle"), "port"])


def _same(a, b):
    return bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


def test_port_finish_matches_golden():
    g = np.load(GOLD)
    for k, e in enumerate(g["exposures"]):
        f = refdrv.port_finish(g["pixels"], float(e))
        assert _same(f, g["filtered_%d" % k]), "exposure %g" % e
        assert np.array_equal(refdrv.port_quantize(f), g["rgb8_%d" % k])
    # the alpha channel comes out 0 (ToneMap rebuilds Color(retColor, 0.0f)); zero-weight pixels are black
    f = g["filtered_0"]
    assert (f[..., 3] == 0.0).all()
    assert (f[64, :8, :3] == 0.0).all()          # 0 * inf = NaN -> Max(0, NaN) = 0
    assert np.isnan(f[64, 8:16, :3]).all()       # inf / inf
    assert (g["rgb8_0"][64, 8:16] == 255).all()  # Clamp(NaN) -> 255


def test_port_finish_matches_reference_directly(tmp_path):
    if not refdrv.have_ref("detmath"):
        pytest.skip("oracle/_ref not built")
    rng = np.random.RandomState(3)
    px = np.empty((33, 47, 4), np.float32)
    px[..., 3] = rng.uniform(0.2, 40.0, px.shape[:2])
    px[..., :3] = rng.gamma(0.6, 1.5, px.shape[:2] + (3,)) * px[..., 3:4]
    for e in (1.0, 0.6):
        f_ref = refdrv.ref_finish(px, e)
        assert _same(refdrv.port_finish(px, e), f_ref)
        assert np.array_equal(refdrv.port_quantize(f_ref), refdrv.ref_png_bytes(f_ref, tmp_path / "a.png"))


def test_literal_libm_agrees_to_one_ulp():
    """glibc powf vs include/tb200_detmath.h powf: the finished image differs by at most a few ulp."""
    if not refdrv.have_ref("literal"):
        pytest.skip("oracle/_ref not built")
    g = np.load(GOLD)
    px = g["pixels"][:64]
    a = refdrv.ref_finish(px, 1.0, flavour="literal")
    b = g["filtered_0"][:64]
    assert np.allclose(a, b, rtol=4e-7, atol=1e-7)


def test_port_nlm_matches_golden_and_reference():
    """NonLocalMeansFilter (src/nlm.cpp:36-73): restatement vs golden vectors from the reference's own
    compiled filter (radius 0, 1 = what main.cpp uses, 3), and vs the reference directly on a ragged image."""
    g = np.load(GOLD)
    img = g["filtered_0"][:64]
    assert _same(refdrv.port_nlm(img, 200.0, 1), g["nlm_r1"])
    assert _same(refdrv.port_nlm(img, 35.0, 3), g["nlm_r3"])
    assert _same(refdrv.port_nlm(img, 200.0, 0), g["nlm_r0"])
    assert _same(g["nlm_r0"][..., :3], img[..., :3])          # a 1x1 window returns the pixel itself (x*1/1)
    if refdrv.have_ref("detmath"):
        rng = np.random.RandomState(5)
        im = rng.uniform(0.0, 1.0, (19, 7, 4)).astype(np.float32)
        for radius, falloff in ((1, 200.0), (2, 10.0), (9, 1.0)):   # radius 9 > the image width: fully clamped windows
            assert _same(refdrv.port_nlm(im, falloff, radius), refdrv.ref_nlm(im, falloff, radius))


# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_nlm_bit_exact():
    import torch
    g = np.load(GOLD)
    px = g["pixels"][:64]
    h, w = px.shape[:2]
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    r.Init(w, h)
    with pytest.raises(tb.TinselB200Error):
        r.nlm(200.0, 1)                                         # nothing finished yet
    acc = torch.from_numpy(px.copy()).cuda()
    r.bind_accumulator(acc.data_ptr())
    f, _ = r.finish(1.0, 1.5, filtered=True, rgb8=False)
    assert _same(f, g["filtered_0"][:64])
    assert _same(r.nlm(200.0, 1), g["nlm_r1"])
    assert _same(r.nlm(35.0, 3), g["nlm_r3"])
    assert _same(r.nlm(200.0, 0), g["nlm_r0"])
    r.close()
    snap.close()
    # a rendered, ragged-size image with the 8-bit-only finish in front (the float image stays on the device)
    snap = tb.Snapshot(tb.scene_path("veach"))
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = 203, 77
    r = tb.Renderer(snap.scene)
    r.Init(opt.width, opt.height)
    out = np.zeros((opt.height, opt.width, 4), np.float32)
    r.render_n(cam, opt, 4, out)
    r.finish(float(opt.exposure), float(opt.limit), filtered=False, rgb8=True)
    want = refdrv.port_nlm(refdrv.port_finish(out, float(opt.exposure)), 200.0, 2)
    assert _same(r.nlm(200.0, 2), want)
    r.close()
    snap.close()


@pytest.mark.gpu
def test_gpu_finish_bit_exact_on_golden_accumulators():
    import torch
    g = np.load(GOLD)
    px = g["pixels"]
    h, w = px.shape[:2]
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    r.Init(w, h)
    acc = torch.from_numpy(px.copy()).cuda()
    r.bind_accumulator(acc.data_ptr())
    for k, e in enumerate(g["exposures"]):
        f, b = r.finish(float(e), 1.5)
        assert _same(f, g["filtered_%d" % k]), "exposure %g" % e
        assert np.array_equal(b, g["rgb8_%d" % k])
    # either output alone
    f, b = r.finish(1.0, 1.5, filtered=True, rgb8=False)
    assert b is None and _same(f, g["filtered_0"])
    f, b = r.finish(1.0, 1.5, filtered=False, rgb8=True)
    assert f is None and np.array_equal(b, g["rgb8_0"])
    r.close()
    snap.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,size", [("cornell", (256, 256)), ("veach", (321, 123)), ("envmini", (127, 95)), ("mini", (1, 1))])
def test_gpu_render_n_then_finish_matches_oracle(name, size):
    """n x Render with one read-back, then the finish step on the device, against the oracle chain
    (seeded accumulation -> finish -> quantise) on the GPU's own accumulator (bit-exact) and on the
    oracle's accumulator (8-bit values within 1)."""
    snap = tb.Snapshot(tb.scene_path(name))
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = size
    r = tb.Renderer(snap.scene)
    r.Init(opt.width, opt.height)
    out = np.zeros((opt.height, opt.width, 4), np.float32)
    r.render_n(cam, opt, 5, out)
    assert r.stats().frames == 5
    one = tb.Renderer(snap.scene)
    one.Init(opt.width, opt.height)
    ref = np.zeros_like(out)
    for _ in range(5):
        one.Render(cam, opt, ref)
    assert np.allclose(out, ref, rtol=2e-5, atol=1e-6)          # same samples, different summation order
    r.render_n(cam, opt, 1, out)                                 # n = 1 degenerates to Render
    assert r.stats().frames == 6
    assert (out.view(np.uint32) == r.read_accumulator().view(np.uint32)).all()
    exposure = float(opt.exposure)
    f, b = r.finish(exposure, float(opt.limit))
    fo = refdrv.port_finish(out, exposure)
    assert _same(f, fo)
    assert np.array_equal(b, refdrv.port_quantize(fo))
    port = refdrv.PortScene.from_snapshot(tb.scene_path(name))
    port.set_size(opt.width, opt.height)
    bo = refdrv.port_quantize(refdrv.port_finish(port.render_seeded(0, 6, 1), exposure))
    assert int(np.abs(b.astype(np.int32) - bo.astype(np.int32)).max()) <= 1
    port.close()
    one.close()
    r.close()
    snap.close()
