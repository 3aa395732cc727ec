"""The renderer at the limits tb200_create accepts (tests/fuzzscene.py make_limit_scene): 40, 41 and 42 primitives
(where the wavefront stops staging the primitive records and the scene BVH on chip), 600 and 4095 primitives, and
255-4095 shadow rays per surface hit (the wavefront's NEE cursor keeps 12-bit primitive and sample indices and a
probe flag).  CPU: the generator makes what it claims, the limits are accepted and one past them refused, and the
port matches the reference's own code.  GPU: per sample and bit for bit against the port in every kernel variant,
the 4-spp image, the normals image and the closest-hit query."""
import ctypes as C
import os

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import fuzzscene
import rayoracle
import raysets
import refdrv
import schedenv

CASES = list(fuzzscene.LIMIT_CASES)
PRIMS_CASES = [c for c in CASES if c.startswith("prims")]
SMALL_CASES = [c for c in CASES if not c.startswith("prims")]      # 8 primitives: the flat scene program
NTHREADS = os.cpu_count() or 8


@pytest.fixture(autouse=True)
def default_knobs():
    with schedenv.knobs():
        yield


def _size(case):
    return (24, 16) if case == "prims4095" else (48, 32)


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    """case -> (snapshot path, info); each scene is written once per module."""
    root = tmp_path_factory.mktemp("limits")
    made = {}

    def get(case):
        if case not in made:
            path = str(root / ("%s.tsnap" % case))
            made[case] = (path, fuzzscene.make_limit_scene(case, path, *_size(case)))
        return made[case]
    return get


@pytest.fixture(scope="module")
def port_frames(scenes):
    """(case, frame) -> the port's (radiance, raster) for that frame, computed once per module."""
    done = {}

    def get(case, frame):
        if (case, frame) not in done:
            port = refdrv.PortScene.from_snapshot(scenes(case)[0])
            done[(case, frame)] = port.trace_frame(frame, NTHREADS)
            port.close()
        return done[(case, frame)]
    return get


def _bad_samples(rad, ras, prad, pras):
    assert np.array_equal(ras, pras)
    return int((~((rad.view(np.uint32) == prad.view(np.uint32)) | (np.isnan(rad) & np.isnan(prad))).all(-1)).sum())


def _same(a, b):
    return bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


def _scene_pairs(path, tmp_path):
    """The number of scene-level BVH pair records in the device image (from the scene cache file's header)."""
    snap = tb.Snapshot(path)
    cache = str(tmp_path / "pairs.tcache")
    tb.scene_cache_save(snap.scene, cache)
    snap.close()
    data = open(cache, "rb").read()
    u64 = lambda o: int.from_bytes(data[o:o + 8], "little")
    size_prim = int.from_bytes(data[12:16], "little")
    return u64(24 + 8 + u64(24) * size_prim)


# ---- CPU ---------------------------------------------------------------------------------------------

def test_limit_generator_makes_what_it_claims(scenes, tmp_path):
    """Primitive and pair counts, shadow rays per hit, where the lights sit; camera rays of the many-shadow-ray
    scenes hit non-emissive surfaces (each such hit draws every shadow ray); the port renders every scene lit."""
    for case in CASES:
        path, info = scenes(case)
        snap = tb.Snapshot(path)
        sc = snap.scene.contents
        samples = [sc.primitives[i].lightSamples for i in range(sc.numPrimitives)]
        assert sc.numPrimitives == info["prims"] and bool(sc.sky.probeValid) == info["probe"], info
        assert info["numNee"] == sum(samples) + int(info["probe"]), info
        assert info["lights"] == [i for i, s in enumerate(samples) if s > 0], info
        rays = raysets.camera_rays(snap.camera, 2000, np.random.RandomState(1), *_size(case))
        oracle = rayoracle.RayOracle.from_snapshot(path)
        _, prims = oracle.trace_rays(rays)
        oracle.close()
        surface = float(((prims >= 0) & (np.array(samples)[np.maximum(prims, 0)] == 0)).mean())
        assert surface > 0.9, (case, surface)
        port = refdrv.PortScene.from_snapshot(path)
        rad, _ = port.trace_frame(0, NTHREADS)
        assert float(np.nan_to_num(rad).sum()) > 0.0, info
        assert not np.isnan(rad).any(), info
        port.close()
        if case.startswith("nee") or case in ("probe255", "meshlight300"):
            n = int("".join(ch for ch in case if ch.isdigit()))
            at = 3 if case in ("nee300_odd", "probe255") else 2
            assert info["prims"] == 8 and info["light_samples"] == {at: n}, info
            assert info["numNee"] == n + int(case == "probe255"), info
            assert sc.primitives[at].type == (abi.MESH if case == "meshlight300" else abi.SPHERE), info
        if case == "meshlight300":
            assert info["tris"][0] < 4096, info
        snap.close()
    # the shared-memory boundary: 40 primitives and 39 pairs, 41 and 40, 42 and 41 (TB_WF2_MAX_PRIMS/PAIRS = 40)
    for case, n in (("prims40", 40), ("prims41", 41), ("prims42", 42)):
        path, info = scenes(case)
        assert info["prims"] == n and _scene_pairs(path, tmp_path) == n - 1, info
        assert all(s <= 2 for s in info["light_samples"].values()) and len(info["lights"]) >= 5, info
    # the 256th shadow ray: inside (not last of) an even-index light, with lights at odd indices and after it
    info = scenes("prims600")[1]
    prim, k = info["ray256"]
    assert info["prims"] == 600 and info["numNee"] > 256 and prim % 2 == 0 and k + 1 < info["light_samples"][prim], info
    assert any(i % 2 for i in info["lights"]) and info["lightEnd"] > prim + 1 and info["lightBegin"] > 2, info
    info = scenes("prims4095")[1]
    assert info["prims"] == fuzzscene.MAX_PRIMS and info["light_samples"] == {fuzzscene.MAX_PRIMS - 1: fuzzscene.MAX_LIGHT_SAMPLES}
    for case in ("nee256", "nee257", "nee300", "meshlight300"):
        assert scenes(case)[1]["ray256"] == (2, 255)
    assert scenes("nee300_odd")[1]["ray256"] == (3, 255)
    assert scenes("probe255")[1]["ray256"] == (3, 254) and "ray256" not in scenes("nee255")[1]


def _refusals(scene_ptr, tmp_path):
    """(tb200_create's error, tb200_scene_cache_save's error); None where the call accepted the scene."""
    lib = tb.load_library()
    h = lib.tb200_create(scene_ptr, 0)
    if h:
        lib.tb200_destroy(h)
    create = tb.last_error() if not h else ""
    create = create if "invalid scene" in create else None
    rc = lib.tb200_scene_cache_save(scene_ptr, str(tmp_path / "x.tcache").encode())
    save = tb.last_error() if rc != 0 else None
    return create, save


def _spheres(n, light_samples):
    prims = (abi.Primitive * n)()
    rng = np.random.RandomState(n)
    bounds = [fuzzscene._sphere(prims[k], rng.uniform(-2.0, 2.0, 3), 0.01, abi.Material.default()) for k in range(n)]
    prims[n - 1].lightSamples = light_samples
    return fuzzscene.make_scene_struct(prims, fuzzscene._build_bvh(bounds), [])


def test_limits_are_accepted_and_one_past_them_refused(scenes, tmp_path):
    """4095 primitives and 4095 lightSamples pass tb200_create's and tb200_scene_cache_save's validation, 4096 of
    either are refused, and so is a cache file holding 4096 primitives.  All of it runs before a device is opened."""
    snap = tb.Snapshot(scenes("prims4095")[0])
    assert _refusals(snap.scene, tmp_path) == (None, None)
    snap.close()
    for n, samples, expect in ((fuzzscene.MAX_PRIMS, fuzzscene.MAX_LIGHT_SAMPLES, None),
                               (fuzzscene.MAX_PRIMS + 1, 1, "more than 4095 primitives"),
                               (8, fuzzscene.MAX_LIGHT_SAMPLES + 1, "primitive 7: lightSamples out of range")):
        sc, keep = _spheres(n, samples)
        for err in _refusals(C.pointer(sc), tmp_path):
            if expect is None:
                assert err is None, err
            else:
                assert err and "invalid scene" in err and expect in err, err
    # a cache file: the 4095-primitive image with its last primitive record repeated
    sc, keep = _spheres(fuzzscene.MAX_PRIMS, fuzzscene.MAX_LIGHT_SAMPLES)
    good = str(tmp_path / "good.tcache")
    tb.scene_cache_save(C.pointer(sc), good)
    data = open(good, "rb").read()
    size_prim = int.from_bytes(data[12:16], "little")
    n = int.from_bytes(data[24:32], "little")
    assert n == fuzzscene.MAX_PRIMS
    end = 32 + n * size_prim
    big = data[:24] + (n + 1).to_bytes(8, "little") + data[32:end] + data[end - size_prim:end] + data[end:]
    lib = tb.load_library()
    for blob, bad in ((data, False), (big, True)):
        p = str(tmp_path / "x.tcache")
        open(p, "wb").write(blob)
        h = lib.tb200_create_cached(p.encode(), 0)
        if h:
            lib.tb200_destroy(h)
            err = ""
        else:
            err = tb.last_error()
        assert ("invalid cache file" in err and "bad primitive count" in err) == bad, err


@pytest.mark.skipif(not refdrv.have_ref("detmath"), reason="oracle/_ref not built")
@pytest.mark.parametrize("case", CASES)
def test_port_matches_reference_on_limit_scenes(case, scenes, port_frames):
    path, info = scenes(case)
    ref = refdrv.RefScene.from_snapshot(path, "detmath")
    for frame in (0, 3):
        a, ar = ref.trace_frame(frame, NTHREADS)
        b, br = port_frames(case, frame)
        assert np.array_equal(ar, br), info
        assert _same(a, b), info
    ref.close()


# ---- GPU ---------------------------------------------------------------------------------------------

def _gpu_vs_port(path, port_frames, case, routes, frames=(0, 3)):
    """{(route, frame): samples that differ from the port}; routes: {route: its knob settings}."""
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    bad = {}
    try:
        for route, settings in routes.items():
            with schedenv.knobs(**settings):
                r = tb.Renderer(snap.scene)
            r.Init(opt.width, opt.height)
            for frame in frames:
                rad, ras = r.trace_frame(cam, opt, frame)
                n = _bad_samples(rad, ras, *port_frames(case, frame))
                if n:
                    bad[(route, frame)] = n
            r.close()
    finally:
        snap.close()
    return bad


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_gpu_matches_port_at_the_limits(case, scenes, port_frames):
    """Both pipelines as the default routing picks their kernels (for the many-shadow-ray scenes: hard phases and
    the ring queues, which store the NEE cursor between the shade and shadow stages)."""
    path, info = scenes(case)
    bad = _gpu_vs_port(path, port_frames, case, {p: schedenv.ROUTES[p] for p in ("mega", "wavefront")})
    assert not bad, "%s: samples differ %s" % (info["case"], bad)


@pytest.mark.gpu
@pytest.mark.parametrize("sched,cta", [(s, c) for s in schedenv.SCHEDS for c in schedenv.CTAS])
@pytest.mark.parametrize("case", CASES)
def test_limit_scenes_under_every_scheduler_variant(case, sched, cta, scenes, port_frames):
    path, info = scenes(case)
    bad = _gpu_vs_port(path, port_frames, case, {sched: schedenv.sched_knobs(sched, cta)})
    assert not bad, "%s %s/%s: samples differ %s" % (case, sched, cta, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SMALL_CASES)
def test_small_limit_scenes_without_the_flat_program(case, scenes, port_frames):
    """The scene level runs the reference-order walk instead of the flat program (default routing otherwise)."""
    path, info = scenes(case)
    bad = _gpu_vs_port(path, port_frames, case, {"no-flat": schedenv.ROUTES["no-flat"]})
    assert not bad, "%s: samples differ %s" % (case, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_limit_scene_images_match_port(case, scenes):
    """The 4-spp image against the port's seeded render (rel-L2 <= 1e-4: the framebuffer sums run in another
    order, NaN on the same pixels), and for the prims* scenes the normals image bit for bit."""
    path, info = scenes(case)
    port = refdrv.PortScene.from_snapshot(path)
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    r = tb.Renderer(snap.scene)
    r.Init(opt.width, opt.height)
    out = np.zeros((opt.height, opt.width, 4), np.float32)
    for _ in range(4):
        r.Render(cam, opt, out)
    expect = port.render_seeded(0, 4, nthreads=NTHREADS)
    nan = np.isnan(out).any(-1)
    assert np.array_equal(nan, np.isnan(expect).any(-1)), info
    rel = np.linalg.norm((out[~nan] - expect[~nan]).astype(np.float64)) / np.linalg.norm(expect[~nan].astype(np.float64))
    assert rel <= 1e-4, "%s: rel L2 %g" % (case, rel)
    if case in PRIMS_CASES:
        opt.mode = abi.MODE_NORMALS
        port.set_mode(abi.MODE_NORMALS)
        r.Init(opt.width, opt.height)
        out = np.zeros_like(out)
        r.Render(cam, opt, out)
        expect = port.render_normals()
        assert np.array_equal(out.view(np.uint32), expect.view(np.uint32)), "%s: %d normals differ" % (
            case, int((out != expect).any(-1).sum()))
    r.close()
    port.close()
    snap.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", PRIMS_CASES)
def test_limit_scene_rays_match_port(case, scenes):
    """Renderer.trace_rays on camera, random and secondary rays against the port's Trace, per ray and bit for bit."""
    import torch
    path, info = scenes(case)
    snap = tb.Snapshot(path)
    oracle = rayoracle.RayOracle.from_snapshot(path)
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(info["prims"])
    n = 1 << 14
    cam = raysets.camera_rays(snap.camera, n, rng)
    h, p = oracle.trace_rays(cam)
    for what, rays in (("camera", cam), ("random", raysets.random_rays(snap.scene.contents, n, rng)),
                       ("secondary", raysets.secondary_rays(cam, h, p, rng))):
        hits, prims = r.trace_rays(torch.from_numpy(np.ascontiguousarray(rays)).cuda(r.device))
        hits, prims = hits.cpu().numpy(), prims.cpu().numpy()
        want_h, want_p = oracle.trace_rays(rays)
        bad = raysets.mismatches(hits, prims, want_h, want_p)
        assert len(bad) == 0, "%s/%s: %d of %d rays differ" % (case, what, len(bad), len(rays))
        if what == "camera":
            assert (prims >= 0).mean() > 0.9
    r.close()
    oracle.close()
    snap.close()
