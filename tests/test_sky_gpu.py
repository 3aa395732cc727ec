"""A new sky for a live renderer (tb200_set_sky) and the probe's sampling tables built on the device
(tb200_probe_tables).

The tables must be Probe::BuildCDF's bit for bit (NaN where NaN): against bigscene.build_cdf and the tables a snapshot
load builds, on envmini's probe, env's 4000 x 2000 stand-in and edge probes.  A renderer that swaps its sky must be
indistinguishable from one created with that sky: the same per-sample radiance under every route, the same kernel (the
one test_route_gpu's rule predicts for the new sky), and the same answers from the sky and light queries."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import tinsel_b200 as tb
from tinsel_b200 import abi
import bigscene
import refdrv
import schedenv
from test_route_gpu import facts, kernel, route

pytestmark = pytest.mark.gpu

SIZE = (48, 32)
F32 = np.float32


@pytest.fixture(autouse=True)
def default_knobs():
    with schedenv.knobs():
        yield


def same_bits(a, b):
    """Bit-identical float32 arrays, any NaN matching any NaN."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return a.shape == b.shape and bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


def make_probe(height, width, seed, alpha=False):
    """A probe of random texels in [0, 2) with a hot texel and a black row (when there are rows to spare)."""
    rng = np.random.RandomState(seed)
    img = rng.uniform(0.0, 2.0, (height, width, 4)).astype(F32)
    if not alpha:
        img[..., 3] = 0.0
    img[rng.randint(height), rng.randint(width), :3] = 5.0e3
    if height > 2:
        img[height // 2, :, :3] = 0.0
    return img


def snapshot_probe(snap):
    k = snap.scene.contents.sky
    n = k.probeWidth * k.probeHeight
    return np.ctypeslib.as_array(k.probeData, (n * 4,)).reshape(k.probeHeight, k.probeWidth, 4).copy()


class Sky:
    """A sky: the gradient colours and, unless None, an (H, W, 4) float32 probe."""

    def __init__(self, horizon, zenith, probe=None):
        self.horizon, self.zenith, self.probe = list(horizon), list(zenith), probe

    def scene(self, base):
        """A copy of tb200_scene `base` with this sky, its tables from bigscene.build_cdf; returns (scene, arrays it
        points into)."""
        sc = abi.copy_struct(base)
        sc.sky.horizon[:] = self.horizon
        sc.sky.zenith[:] = self.zenith
        keep = []
        if self.probe is None:
            sc.sky.probeValid = sc.sky.probeWidth = sc.sky.probeHeight = 0
            for f in ("probeData", "pdfValuesX", "cdfValuesX", "pdfValuesY", "cdfValuesY"):
                setattr(sc.sky, f, None)
        else:
            keep = [np.ascontiguousarray(self.probe)] + [np.ascontiguousarray(t, F32) for t in bigscene.build_cdf(self.probe)]
            sc.sky.probeValid = 1
            sc.sky.probeHeight, sc.sky.probeWidth = self.probe.shape[:2]
            for f, a in zip(("probeData", "pdfValuesX", "cdfValuesX", "pdfValuesY", "cdfValuesY"), keep):
                setattr(sc.sky, f, a.ctypes.data_as(abi.c_float_p))
        return sc, keep

    def set_on(self, r, on_device=False):
        probe = self.probe
        if probe is not None and on_device:
            probe = torch.from_numpy(probe).to(torch.device("cuda", r.device))
        r.set_sky(self.horizon, self.zenith, probe)


GRADIENT = Sky([0.0, 0.0, 0.0], [0.0, 0.0, 0.0])
COLOURS = Sky([0.7, 0.5, 0.25], [0.1, 0.3, 1.5])
PROBE_A = Sky([0.2, 0.2, 0.2], [0.0, 0.1, 0.4], make_probe(48, 96, 1))
PROBE_B = Sky([0.0, 0.0, 0.0], [0.0, 0.0, 0.0], make_probe(32, 64, 2))


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    """Scene name -> snapshot path; ajax_like is written by bigscene."""
    paths = {n: tb.scene_path(n) for n in ("envmini", "cornell", "veach", "motionblur")}
    paths["ajax_like"] = str(tmp_path_factory.mktemp("sky") / "ajax_like.tsnap")
    bigscene.ajax_like(paths["ajax_like"])
    return paths


def sky_of(snap):
    k = snap.scene.contents.sky
    return Sky(list(k.horizon), list(k.zenith), snapshot_probe(snap) if k.probeValid else None)


class Setup:
    """A snapshot, a small image of it, and renderers made from its scene with a given sky."""

    def __init__(self, path):
        self.snap = tb.Snapshot(path)
        self.cam, self.opt = self.snap.camera, self.snap.options
        self.opt.width, self.opt.height = SIZE
        self.keep = []

    def renderer(self, sky, **kw):
        sc, keep = sky.scene(self.snap.scene.contents)
        self.keep += [sc, keep]
        r = tb.Renderer(C.pointer(sc), **kw)
        r.Init(*SIZE)
        return r

    def save(self, sky, path):
        """Writes the snapshot of this scene with `sky` (for facts() and the CPU restatement)."""
        sc, keep = sky.scene(self.snap.scene.contents)
        assert tb.load_library().tb200_snapshot_save(str(path).encode(), C.byref(sc), C.byref(self.cam), C.byref(self.opt)) == 0
        return str(path)

    def inputs(self, r):
        """Inputs of the sky and light queries: random rays, seeds, and the light queries of the image's first hits."""
        dev = torch.device("cuda", r.device)
        g = torch.Generator().manual_seed(7)
        rays = torch.zeros((4096, 8), dtype=torch.float32)
        rays[:, 4:7] = torch.randn((4096, 3), generator=g)
        rays = rays.to(dev)
        seeds = torch.arange(4096, dtype=torch.int32, device=dev) * 7919
        cam_rays, _ = r.camera_rays(self.cam, self.opt, tb.frame_samples(SIZE[0], SIZE[1], 3, device=dev))
        hits, prims = r.trace_rays(cam_rays)
        d = cam_rays[:, 4:7]
        p = cam_rays[:, :3] + hits[:, :1] * d
        q = tb.light_queries(prims, p, hits[:, 1:4].contiguous(), (-d).contiguous(), 1.0, 1.5, cam_rays[:, 3].contiguous())
        return rays, seeds, q, seeds[:q.shape[0]].contiguous()

    def answers(self, r, inputs):
        rays, seeds, q, qseeds = inputs
        probe = torch.empty((seeds.shape[0], 8), dtype=torch.float32, device=seeds.device)
        r.sample_probe(seeds, out=probe)
        return [r.sky(rays).cpu().numpy(), probe.cpu().numpy(), r.sample_lights(q, qseeds).cpu().numpy()]

    def frames(self, r):
        out = []
        for frame in (0, 3):
            rad, ras = r.trace_frame(self.cam, self.opt, frame)
            out += [rad, ras]
        return out

    def close(self):
        self.snap.close()


def assert_same(a, b, what):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert same_bits(x, y), "%s: output %d differs (%d values)" % (what, k, int((~((np.asarray(x).view(np.uint32) == np.asarray(y).view(np.uint32)) | (np.isnan(x) & np.isnan(y)))).sum()))


# ---- the tables ----------------------------------------------------------------------------------------------------

def edge_probes():
    rng = np.random.RandomState(11)
    out = {}
    # widths around a tile of k_probe_rows (128 texels) and of a warp; heights past k_probe_cols' chunks of 4096 rows
    for shape in [(1, 1), (1, 50), (50, 1), (5, 31), (5, 32), (5, 33), (3, 127), (3, 128), (3, 129), (3, 4097),
                  (40, 70), (8193, 1), (4097, 3)]:
        out["%dx%d" % shape] = rng.uniform(0.0, 2.0, shape + (4,)).astype(F32)
    base = lambda: rng.uniform(0.0, 2.0, (6, 37, 4)).astype(F32)
    p = base(); p[2, :, :3] = 0.0; out["black-row"] = p
    out["all-black"] = np.zeros((4, 9, 4), F32)
    p = np.zeros((7, 13, 4), F32); p[3, 5, :3] = 1.0e4; out["one-hot-texel"] = p
    p = base(); p[1, 4, 0] = np.inf; out["inf"] = p
    p = base(); p[4, 10, 1] = np.nan; out["nan"] = p
    p = base(); p[0, :5, 2] = -3.0; p[5, 7, :3] = -1.0; out["negative"] = p
    p = base(); p[3, :, :3] = np.float32(1.0e-39); p[2, 3, :3] = np.float32(1.4e-45); out["subnormal"] = p
    p = base(); p[2, :, :3] = np.float32(3.0e38); out["row-overflow"] = p
    p = base(); p[..., 3] = np.float32(np.nan); out["alpha-ignored"] = p
    return out


EDGES = edge_probes()


@pytest.fixture(scope="module")
def renderer():
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    yield r
    r.close()
    snap.close()


def own_segment():
    """A (768, 2048, 4) float32 probe of 24 MiB in a segment of its own, so that a span one row longer runs past
    the end of its allocation."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.zeros((768, 2048, 4), dtype=torch.float32, device="cuda")


def tables_on_device(r, probe):
    out = r.probe_tables(torch.from_numpy(probe).cuda())
    return [t.cpu().numpy() for t in out]


def snapshot_tables(probe, tmp_path):
    """The tables tb200_snapshot_load builds for `probe` (a cornell snapshot with this probe, saved and loaded)."""
    setup = Setup(tb.scene_path("cornell"))
    path = setup.save(Sky([0.0] * 3, [0.0] * 3, probe), tmp_path / "probe.tsnap")
    setup.close()
    snap = tb.Snapshot(path)
    t = bigscene.probe_tables(snap.scene.contents.sky)
    snap.close()
    return t


@pytest.mark.parametrize("name", ["envmini", "env_like"] + sorted(EDGES))
def test_tables_bit_exact(name, renderer, tmp_path):
    if name == "envmini":
        snap = tb.Snapshot(tb.scene_path("envmini"))
        probe, loaded = snapshot_probe(snap), bigscene.probe_tables(snap.scene.contents.sky)
        snap.close()
    else:
        probe = bigscene.probe_image() if name == "env_like" else EDGES[name]
        loaded = snapshot_tables(probe, tmp_path)
    got = tables_on_device(renderer, probe)
    want = bigscene.build_cdf(probe)
    for k, what in enumerate(("pdfX", "cdfX", "pdfY", "cdfY")):
        assert same_bits(got[k], want[k]), "%s: %s differs from build_cdf" % (name, what)
        assert same_bits(got[k], loaded[k]), "%s: %s differs from the snapshot's tables" % (name, what)
    if name == "all-black":
        assert np.isnan(got[0]).all() and np.isnan(got[2]).all()


def test_tables_stats_and_refusals(renderer):
    st = renderer.stats()
    probe = torch.from_numpy(EDGES["40x70"]).cuda()
    renderer.probe_tables(probe)
    after = renderer.stats()
    assert after.kernelLaunches == st.kernelLaunches + 3 and after.gpuMs > 0.0
    assert (after.frames, after.samples, after.h2dBytes, after.d2hBytes) == (st.frames, st.samples, st.h2dBytes, st.d2hBytes)
    lib, h = renderer.lib, renderer.h
    out = [torch.empty(40 * 70, device="cuda") for _ in range(4)]
    ptrs = [o.data_ptr() for o in out]
    ok = lambda w, hh, p=probe.data_ptr(), q=ptrs: lib.tb200_probe_tables(h, p, w, hh, *q)
    assert ok(70, 40) == 0
    assert ok(0, 40) == -1 and ok(70, -1) == -1 and ok(65536, 32768) == -1
    assert ok(70, 40, p=probe.data_ptr() + 4) == -1 and "aligned" in tb.last_error()
    host = np.zeros((40, 70, 4), F32)
    assert ok(70, 40, p=host.ctypes.data) == -1 and "not device memory" in tb.last_error()
    assert ok(70, 40, q=[None] + ptrs[1:]) == -1 and "null" in tb.last_error()
    # a span past the end: a probe that owns its segment (a fresh 24 MiB tensor gets one of its own)
    big = own_segment()
    big_out = [torch.empty(769 * 2048, device="cuda") for _ in range(4)]
    assert ok(2048, 769, p=big.data_ptr(), q=[o.data_ptr() for o in big_out]) == -1 and "past the end" in tb.last_error()
    assert renderer.stats().kernelLaunches == after.kernelLaunches + 3
    with pytest.raises(ValueError):
        renderer.probe_tables(probe.cpu())
    with pytest.raises(TypeError):
        renderer.probe_tables(EDGES["40x70"])
    with pytest.raises(TypeError):
        renderer.probe_tables(probe.double())
    with pytest.raises(ValueError):
        renderer.probe_tables(probe[..., :3])


# ---- swap equals create --------------------------------------------------------------------------------------------

CASES = [("envmini", "own", PROBE_A), ("envmini", "own", GRADIENT), ("cornell", GRADIENT, PROBE_B),
         ("cornell", GRADIENT, COLOURS), ("veach", GRADIENT, PROBE_B), ("veach", GRADIENT, COLOURS),
         ("motionblur", GRADIENT, PROBE_B), ("ajax_like", GRADIENT, PROBE_B)]
ROUTES = ["default"] + sorted(schedenv.ROUTES)


def large_spp(num_sms):
    return math.ceil(6 * num_sms * 1024 / (SIZE[0] * SIZE[1]))


@pytest.mark.parametrize("route_name", ROUTES)
@pytest.mark.parametrize("case", range(len(CASES)), ids=["%s-%d" % (c[0], i) for i, c in enumerate(CASES)])
def test_swap_equals_create(case, route_name, scenes, tmp_path):
    name, s1, s2 = CASES[case]
    setup = Setup(scenes[name])
    s1 = sky_of(setup.snap) if s1 == "own" else s1
    settings = {} if route_name == "default" else schedenv.ROUTES[route_name]
    with schedenv.knobs(**settings) as applied:
        a = setup.renderer(s1)
        b = setup.renderer(s2)
    before = a.stats()
    s2.set_on(a)
    after = a.stats()
    assert (after.frames, after.samples) == (before.frames, before.samples)
    assert after.kernelLaunches == before.kernelLaunches + (3 if s2.probe is not None else 0)
    assert_same(setup.frames(a), setup.frames(b), "%s %s trace_frame" % (name, route_name))
    inputs = setup.inputs(b)
    assert_same(setup.answers(a, inputs), setup.answers(b, inputs), "%s %s queries" % (name, route_name))
    spp = large_spp(torch.cuda.get_device_properties(0).multi_processor_count)
    a.render_device(setup.cam, setup.opt, spp)
    b.render_device(setup.cam, setup.opt, spp)
    assert a.last_kernel() == b.last_kernel()
    if route_name != "mega":
        want = kernel(route(facts(setup.save(s2, tmp_path / "s2.tsnap")), applied), SIZE[0] * SIZE[1] * spp,
                      torch.cuda.get_device_properties(0).multi_processor_count)
        assert a.last_kernel() == want, (name, route_name, a.last_kernel(), want)
    if name == "cornell" and route_name == "default":
        assert (b.last_kernel() == "wf2_lq.specialized") == (s2.probe is None), b.last_kernel()
    a.close()
    b.close()
    setup.close()


def test_swap_matches_cpu_restatement(tmp_path):
    """envmini after a swap to another probe, per sample against the CPU restatement of that scene."""
    setup = Setup(tb.scene_path("envmini"))
    a = setup.renderer(sky_of(setup.snap))
    PROBE_A.set_on(a, on_device=True)
    subprocess.check_call(["make", "-s", "-C", os.path.join(refdrv.ROOT, "oracle"), "port"])
    port = refdrv.PortScene.from_snapshot(setup.save(PROBE_A, tmp_path / "a.tsnap"))
    port.set_size(*SIZE)
    for frame in (0, 5):
        rad, ras = a.trace_frame(setup.cam, setup.opt, frame)
        prad, pras = port.trace_frame(frame, nthreads=8)
        assert np.array_equal(ras, pras)
        same = (rad.view(np.uint32) == prad.view(np.uint32)).all(-1) | (np.isnan(rad).any(-1) & np.isnan(prad).any(-1))
        assert same.all(), "frame %d: %d samples differ" % (frame, int((~same).sum()))
    port.close()
    a.close()
    setup.close()


def test_round_trip_and_host_equals_device():
    setup = Setup(tb.scene_path("envmini"))
    s1 = sky_of(setup.snap)
    ref = setup.renderer(s1)
    inputs = setup.inputs(ref)
    want = setup.frames(ref) + setup.answers(ref, inputs)
    host, dev = setup.renderer(s1), setup.renderer(s1)
    for sky in (PROBE_A, GRADIENT, COLOURS, s1):
        sky.set_on(host)
        sky.set_on(dev, on_device=True)
        assert_same(setup.frames(host) + setup.answers(host, inputs), setup.frames(dev) + setup.answers(dev, inputs),
                    "host vs device probe")
    assert_same(setup.frames(host) + setup.answers(host, inputs), want, "S1 -> S2 -> S1")
    for r in (ref, host, dev):
        r.close()
    setup.close()


def test_side_effects_and_external_stream():
    """The accumulator and the frame counter carry on through a swap: rendering 2 frames, setting the same sky
    again and rendering 2 more gives the image of 4 frames (frames 0 and 1 again would be far off).  The copies count in h2dBytes only from the host."""
    setup = Setup(tb.scene_path("envmini"))
    s1 = sky_of(setup.snap)
    ref, a = setup.renderer(s1), setup.renderer(s1)
    want = np.zeros((SIZE[1], SIZE[0], 4), F32)
    got = np.zeros_like(want)
    for _ in range(4):
        ref.Render(setup.cam, setup.opt, want)
    for _ in range(2):
        a.Render(setup.cam, setup.opt, got)
    st = a.stats()
    s1.set_on(a)
    mid = a.stats()
    assert np.array_equal(a.read_accumulator().view(np.uint32), got.view(np.uint32))
    assert (mid.frames, mid.samples, mid.d2hBytes) == (st.frames, st.samples, st.d2hBytes)
    assert mid.kernelLaunches == st.kernelLaunches + 3 and mid.h2dBytes == st.h2dBytes + s1.probe.nbytes
    assert mid.gpuMs > 0.0
    last = a.last_kernel()
    s1.set_on(a, on_device=True)
    assert a.stats().h2dBytes == mid.h2dBytes and a.last_kernel() == last
    for _ in range(2):
        a.Render(setup.cam, setup.opt, got)
    # the splat's sums form in the order its reductions reach memory: equal up to that order (test_multi_gpu's bound)
    assert np.allclose(got, want, rtol=2e-6, atol=1e-6), float(np.abs(got - want).max())
    # the caller's stream: the copy and the build are ordered there
    b = setup.renderer(PROBE_A)
    s = torch.cuda.Stream()
    a.set_stream(s.cuda_stream)
    with torch.cuda.stream(s):
        probe = torch.from_numpy(PROBE_A.probe).cuda()
        a.set_sky(PROBE_A.horizon, PROBE_A.zenith, probe)
    a.set_stream(None)
    assert_same(setup.frames(a), setup.frames(b), "set_sky on the caller's stream")
    for r in (ref, a, b):
        r.close()
    setup.close()


def test_refusals_leave_the_renderer_unchanged():
    setup = Setup(tb.scene_path("envmini"))
    a = setup.renderer(sky_of(setup.snap))
    inputs = setup.inputs(a)
    want = setup.frames(a) + setup.answers(a, inputs)
    lib, h = a.lib, a.h
    col = (C.c_float * 3)(0.5, 0.5, 0.5)
    small = torch.from_numpy(PROBE_B.probe).cuda()
    host = PROBE_B.probe
    calls = [
        (col, col, host.ctypes.data, 0, 32), (col, col, host.ctypes.data, 64, -1), (col, col, None, 64, 32),
        (col, col, None, 0, 1), (col, col, host.ctypes.data, 65536, 32768), (col, col, small.data_ptr(), 65536, 32768),
        (None, col, None, 0, 0), (col, None, host.ctypes.data, 64, 32),
        (col, col, small.data_ptr() + 4, 64, 32), (col, col, own_segment().data_ptr(), 2048, 769),
    ]
    for args in calls:
        assert lib.tb200_set_sky(h, *args) == -1, args
        assert "tb200_set_sky" in tb.last_error()
    with pytest.raises(ValueError):
        a.set_sky([0.5, 0.5], [0.0] * 3)
    with pytest.raises(ValueError):
        a.set_sky([0.0] * 3, [0.0] * 4, host)
    with pytest.raises(TypeError):
        a.set_sky([0.0] * 3, [0.0] * 3, host.astype(np.float64))
    with pytest.raises(ValueError):
        a.set_sky([0.0] * 3, [0.0] * 3, np.zeros((4, 4, 3), F32))
    with pytest.raises(ValueError):
        a.set_sky([0.0] * 3, [0.0] * 3, np.zeros((4, 8, 4), F32)[:, ::2])
    with pytest.raises(TypeError):
        a.set_sky([0.0] * 3, [0.0] * 3, small.double())
    with pytest.raises(ValueError):
        a.set_sky([0.0] * 3, [0.0] * 3, small[:, ::2])
    if torch.cuda.device_count() > 1:
        other = small.to("cuda:1")
        assert lib.tb200_set_sky(h, col, col, other.data_ptr(), 64, 32) == -1 and "device 1" in tb.last_error()
        with pytest.raises(ValueError):
            a.set_sky([0.0] * 3, [0.0] * 3, other)
    assert_same(setup.frames(a) + setup.answers(a, inputs), want, "after refused calls")
    a.close()
    setup.close()


def test_group_and_cache(tmp_path):
    setup = Setup(tb.scene_path("cornell"))
    b = setup.renderer(PROBE_B)
    want = np.zeros((SIZE[1], SIZE[0], 4), F32)
    for _ in range(4):
        b.Render(setup.cam, setup.opt, want)
    for on_device in (False, True):
        with schedenv.knobs(TEST_DUP_DEVICES="1"):
            m = setup.renderer(GRADIENT, devices=[0, 0, 0])
        launches = [m.member_stats(k)[0].kernelLaunches for k in range(3)]
        PROBE_B.set_on(m, on_device=on_device)
        assert [m.member_stats(k)[0].kernelLaunches for k in range(3)] == [n + 3 for n in launches]
        out = np.zeros_like(want)
        for _ in range(4):
            m.Render(setup.cam, setup.opt, out)
        assert np.allclose(out, want, rtol=2e-6, atol=1e-6), float(np.abs(out - want).max())
        assert_same(setup.frames(m), setup.frames(b), "group trace_frame")
        m.close()
    sc, keep = GRADIENT.scene(setup.snap.scene.contents)
    path = str(tmp_path / "cornell.tcache")
    tb.scene_cache_save(C.pointer(sc), path)
    c = tb.Renderer(None, cache=path)
    c.Init(*SIZE)
    PROBE_B.set_on(c)
    inputs = setup.inputs(b)
    assert_same(setup.frames(c) + setup.answers(c, inputs), setup.frames(b) + setup.answers(b, inputs), "cached renderer")
    c.close()
    b.close()
    setup.close()


def test_swaps_free_the_previous_probe():
    setup = Setup(tb.scene_path("envmini"))
    a = setup.renderer(sky_of(setup.snap))
    big = torch.from_numpy(bigscene.probe_image()).cuda()
    a.set_sky([0.0] * 3, [0.0] * 3, big)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(10):
        a.set_sky([0.0] * 3, [0.0] * 3, big)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 < 192e6, "free memory fell by %.0f MB over 10 swaps" % ((free0 - free1) / 1e6)
    a.close()
    setup.close()
