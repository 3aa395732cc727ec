"""The reference-facing C++ adapter (tinsel_b200/plugin): a reference `Scene` (rebuilt from a
snapshot by oracle/_ref) goes through the Itanium-mangled CreateGpuWavefrontRenderer(const Scene*),
Renderer::Init and Renderer::Render exactly as tinsel's main.cpp would call them."""
import ctypes as C
import os

import numpy as np
import pytest

import tinsel_b200 as tb
import refdrv
import schedenv

PLUGIN = os.path.join(tb.ROOT, "tinsel_b200", "plugin", "libtinsel_b200_plugin.so")


@pytest.fixture(autouse=True)
def default_knobs():
    with schedenv.knobs():
        yield


def test_plugin_exports_reference_factory_symbol():
    if not os.path.exists(PLUGIN):
        pytest.skip("plugin not built (needs the reference headers; build container only)")
    lib = C.CDLL(PLUGIN)
    assert hasattr(lib, "_Z26CreateGpuWavefrontRendererPK5Scene")   # Renderer* CreateGpuWavefrontRenderer(const Scene*)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cornell", "veach"])
def test_plugin_render_matches_seeded_oracle(name):
    if not os.path.exists(PLUGIN) or not refdrv.have_ref("detmath"):
        pytest.skip("plugin or oracle/_ref not built")
    ref = refdrv.RefScene.from_snapshot(tb.scene_path(name), "detmath")
    ref.set_size(96, 80)
    lib = C.CDLL(PLUGIN)
    lib.tb200_plugin_render.restype = C.c_int
    lib.tb200_plugin_render.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_float)]
    out = np.zeros((80, 96, 4), np.float32)
    rc = lib.tb200_plugin_render(ref.lib.ref_native_scene(ref.h), ref.lib.ref_native_camera(ref.h),
                                 ref.lib.ref_native_options(ref.h), 4, out.ctypes.data_as(C.POINTER(C.c_float)))
    assert rc == 0
    oracle = ref.render_seeded(0, 4, 4)
    rel = np.linalg.norm((out - oracle).astype(np.float64)) / np.linalg.norm(oracle.astype(np.float64))
    assert rel <= 1e-4, rel
    ref.close()


@pytest.mark.gpu
def test_plugin_multi_gpu_factory(monkeypatch):
    """TINSEL_GPUS=N: CreateGpuWavefrontRenderer builds the multi-device renderer (row slabs, every member
    delivers its own rows into the caller's Color buffer); Init / Render through the reference vtable as
    before.  On a one-GPU box the members share device 0 (test hook)."""
    import torch
    if not os.path.exists(PLUGIN) or not refdrv.have_ref("detmath"):
        pytest.skip("plugin or oracle/_ref not built")
    n, dup = min(torch.cuda.device_count(), 4), None
    if n < 2:
        n, dup = 3, "1"
    monkeypatch.setenv("TINSEL_GPUS", str(n))
    ref = refdrv.RefScene.from_snapshot(tb.scene_path("cornell"), "detmath")
    ref.set_size(128, 100)
    lib = C.CDLL(PLUGIN)
    lib.tb200_plugin_render.restype = C.c_int
    lib.tb200_plugin_render.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_float)]
    out = np.full((100, 128, 4), -3.0, np.float32)
    with schedenv.knobs(TEST_DUP_DEVICES=dup):
        rc = lib.tb200_plugin_render(ref.lib.ref_native_scene(ref.h), ref.lib.ref_native_camera(ref.h),
                                     ref.lib.ref_native_options(ref.h), 5, out.ctypes.data_as(C.POINTER(C.c_float)))
    assert rc == 0
    oracle = ref.render_seeded(0, 5, 4)
    rel = np.linalg.norm((out - oracle).astype(np.float64)) / np.linalg.norm(oracle.astype(np.float64))
    assert rel <= 1e-4, rel
    assert np.allclose(out[..., 3], oracle[..., 3], rtol=1e-5, atol=1e-6)   # every row was delivered by its owner
    ref.close()


@pytest.mark.gpu
def test_plugin_fast_paths_render_n_and_finish(tmp_path):
    """TinselB200RenderN + TinselB200Finish (tinsel_b200_plugin.h) on a reference Scene, against the
    reference's own finish loop and PNG writer applied to the sums the call returned."""
    if not os.path.exists(PLUGIN) or not refdrv.have_ref("detmath"):
        pytest.skip("plugin or oracle/_ref not built")
    ref = refdrv.RefScene.from_snapshot(tb.scene_path("veach"), "detmath")
    ref.set_size(96, 80)
    lib = C.CDLL(PLUGIN)
    f32p = C.POINTER(C.c_float)
    lib.tb200_plugin_present.restype = C.c_int
    lib.tb200_plugin_present.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, f32p, f32p, C.POINTER(C.c_ubyte)]
    out = np.zeros((80, 96, 4), np.float32)
    filtered = np.zeros((80, 96, 4), np.float32)
    rgb8 = np.zeros((80, 96, 3), np.uint8)
    rc = lib.tb200_plugin_present(ref.lib.ref_native_scene(ref.h), ref.lib.ref_native_camera(ref.h), ref.lib.ref_native_options(ref.h),
                                  6, out.ctypes.data_as(f32p), filtered.ctypes.data_as(f32p), rgb8.ctypes.data_as(C.POINTER(C.c_ubyte)))
    assert rc == 0
    oracle = ref.render_seeded(0, 6, 4)
    rel = np.linalg.norm((out - oracle).astype(np.float64)) / np.linalg.norm(oracle.astype(np.float64))
    assert rel <= 1e-4, rel
    exposure = float(ref.options.exposure)
    want = refdrv.ref_finish(out, exposure)
    assert ((filtered.view(np.uint32) == want.view(np.uint32)) | (np.isnan(filtered) & np.isnan(want))).all()
    assert np.array_equal(rgb8, refdrv.ref_png_bytes(want, tmp_path / "v.png"))
    ref.close()


HEADLESS = os.path.join(tb.ROOT, "tinsel_b200", "plugin", "tinsel_headless")
HEADLESS_CPU = os.path.join(tb.ROOT, "tinsel_b200", "plugin", "tinsel_headless_cpu")


def _png(path):
    from PIL import Image
    return np.asarray(Image.open(path).convert("RGB"), dtype=np.float64)


@pytest.mark.gpu
def test_unmodified_tinsel_app_renders_through_the_plugin(tmp_path):
    """tinsel's OWN application -- src/main.cpp + loader + PNG writer compiled unmodified (only a
    force-included GL/GLUT shim and -DCreateCpuRenderer=CreateGpuWavefrontRenderer on main.cpp's
    compile line) -- loads tests/data/mini0.tin in batch mode, renders 64 spp through this repo's
    renderer and writes the PNG; the same app with tinsel's CpuRenderer is the comparison."""
    import shutil
    import subprocess
    if not (os.path.exists(HEADLESS) and os.path.exists(HEADLESS_CPU)):
        pytest.skip("headless tinsel app not built (build container only)")
    imgs = {}
    for name, exe in (("gpu", HEADLESS), ("cpu", HEADLESS_CPU)):
        d = tmp_path / name
        d.mkdir()
        shutil.copy(os.path.join(tb.ROOT, "tests", "data", "mini0.tin"), d / "mini0.tin")
        # batch mode: renders mini0.tin, writes mini0.tin.png, exits(-1) when mini1.tin is missing (main.cpp:128-132)
        subprocess.run([exe, "-spp=64", "mini%d.tin"], cwd=d, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, timeout=300)
        assert (d / "mini0.tin.png").exists(), "%s app wrote no image" % name
        imgs[name] = _png(str(d / "mini0.tin.png"))
    g, c = imgs["gpu"], imgs["cpu"]
    assert g.shape == c.shape == (64, 96, 3)
    # different RNG streams (the CPU renderer has one sequential stream): compare statistically
    assert abs(g.mean() - c.mean()) / c.mean() < 0.02
    blur = lambda a: a.reshape(16, 4, 24, 4, 3).mean(axis=(1, 3))
    assert np.abs(blur(g) - blur(c)).mean() < 6.0   # 8-bit sRGB units on 4x4 block means
