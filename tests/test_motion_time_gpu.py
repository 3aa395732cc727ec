"""Every entry point that takes a ray time, at the times its contract allows, against the CPU restatement per ray, sample
or query, bit for bit (a NaN matching any NaN).  The scenes are fuzzscene's `rotating` family (every sphere and mesh
rotates, with random, antipodal, nearly antipodal, tiny-lerp and one-ulp rotation pairs) and `signed_zero` family
(static primitives written with -0 beside twins written with +0), motionblur and many; the times are
queryscenes.TIMES, zeros of both signs to +-FLT_MAX.  Then: a static sphere at (-0, 0, 0) traced at t = -0.5, camera
samples under reversed, empty, signed-zero and huge shutters, the renderer's own samples under every scheduler variant
and an accumulated image, and non-finite times (exact where every sphere and mesh moves; written and fault-free on
static primitives, the documented exception)."""
import ctypes as C

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import cameraoracle
import emitteroracle
import fuzzscene
import lightoracle
import occlusionsets
import queryscenes
import rayoracle
import raysets
import refdrv
import schedenv
from queryscenes import NONFINITE_TIMES, TIMES

pytestmark = pytest.mark.gpu

F32 = np.float32
PER_SET = 2048          # rays of each ray set, each crossed with every time
FAMILY_SCENES = [("rotating", 0), ("rotating", 1), ("signed_zero", 0), ("signed_zero", 1)]
SCENES = ["fuzz_%s_%d" % fs for fs in FAMILY_SCENES] + ["motionblur", "many"]


def _torch():
    import torch
    return torch


def _same(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _path(name, tmp_path):
    if not name.startswith("fuzz_"):
        return tb.scene_path(name)
    family, seed = name[5:].rsplit("_", 1)
    path = str(tmp_path / "s.tsnap")
    fuzzscene.make_mesh_scene(int(seed), path, family)
    return path


def _cross(rays, times):
    """Every ray of `rays` at every time of `times`."""
    out = np.repeat(rays, len(times), axis=0)
    out[:, 3] = np.tile(np.asarray(times, F32), len(rays))
    return out


def _zero_plane_rays(scene, rng, n=PER_SET):
    """Rays that stay on the x = -0 or the z = -0 plane, where the signed_zero family's primitives sit: origin and
    direction have -0 in that component, so every hit point has it too."""
    lo, hi = raysets.scene_bounds(scene)
    o = rng.uniform(lo - 1.0, hi + 1.0, (n, 3))
    d = rng.normal(size=(n, 3))
    k = np.where(np.arange(n) % 2 == 0, 0, 2)
    o[np.arange(n), k] = -0.0
    d[np.arange(n), k] = -0.0
    return raysets.pack(o, d, 0.0)


def _ray_sets(snap, oracle, rng):
    scene = snap.scene.contents
    sets = queryscenes.ray_sets(scene, snap.camera, oracle, rng)
    out = {k: sets[k][rng.choice(len(sets[k]), min(PER_SET, len(sets[k])), replace=False)] for k in ("camera", "random", "secondary")}
    out["zero_plane"] = _zero_plane_rays(scene, rng)
    return out


def check_ray_queries(r, oracle, rays, what):
    """trace_rays, trace_rays_tri and occluded (tmax +inf, t and the float above t) on `rays`, against the restatement."""
    torch = _torch()
    dev = torch.from_numpy(np.ascontiguousarray(rays)).cuda()
    hits, prims = (x.cpu().numpy() for x in r.trace_rays(dev))
    want_h, want_p, want_tri, want_uvw = oracle.trace_rays_tri(rays)
    bad = raysets.mismatches(hits, prims, want_h, want_p)
    assert len(bad) == 0, "%s trace_rays: %d of %d rays differ; first ray %s: device %s %s, restatement %s %s" % (
        what, len(bad), len(rays), rays[bad[0]], prims[bad[0]], hits[bad[0]], want_p[bad[0]], want_h[bad[0]])
    th, tp, tri, uvw = (x.cpu().numpy() for x in r.trace_rays_tri(dev))
    bad = np.union1d(raysets.mismatches(th, tp, want_h, want_p),
                     np.nonzero((tri != want_tri) | (uvw.view(np.uint32) != want_uvw.view(np.uint32)).any(axis=1))[0])
    assert len(bad) == 0, "%s trace_rays_tri: %d of %d rays differ; first ray %s: device %s %s %s, restatement %s %s %s" % (
        what, len(bad), len(rays), rays[bad[0]], tp[bad[0]], tri[bad[0]], uvw[bad[0]], want_p[bad[0]], want_tri[bad[0]], want_uvw[bad[0]])
    t = want_h[:, 0]
    with np.errstate(over="ignore"):   # a miss's t is FLT_MAX: the float above it is +inf
        t_up = np.nextafter(t, F32(np.inf))
    for name, tmax in (("inf", np.full(len(t), np.inf, F32)), ("t", t), ("t_up", t_up)):
        q = occlusionsets.with_tmax(rays, tmax)
        got = r.occluded(torch.from_numpy(q).cuda()).cpu().numpy()
        bad = np.nonzero(got != occlusionsets.occluded(want_h, want_p, tmax))[0]
        assert len(bad) == 0, "%s occluded (tmax %s): %d of %d rays differ; first ray %s" % (what, name, len(bad), len(rays), q[bad[0]])
    return want_p


# ---- 1. the three ray queries at every time ----


@pytest.mark.parametrize("name", SCENES)
def test_ray_queries_at_every_time(name, tmp_path):
    path = _path(name, tmp_path)
    snap = tb.Snapshot(path)
    oracle = rayoracle.RayOracle.from_snapshot(path)
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(23)
    for what, rays in _ray_sets(snap, oracle, rng).items():
        prims = check_ray_queries(r, oracle, _cross(rays, TIMES), "%s/%s" % (name, what))
        if what == "camera":
            assert (prims >= 0).any(), name
    r.close()
    oracle.close()
    snap.close()


def _worked_example():
    """A static sphere of radius 1 at (-0, 0, 0) and nothing else; (scene, keepalive)."""
    prims = (abi.Primitive * 1)()
    bounds = [fuzzscene._sphere(prims[0], (-0.0, 0.0, 0.0), 1.0, abi.Material.default())]
    return fuzzscene.make_scene_struct(prims, fuzzscene._build_bvh(bounds), [])


def test_static_sphere_at_negative_zero():
    """The ray from (-0, 5, 0) along (-0, -1, 0) at t = -0.5 hits (-0, 1, 0).  The reference's centre x is
    -0 + (+0 * -0.5) = -0, so the normal's x is -0 - (-0) = +0; at t >= +0 the centre x is +0 and the normal's x -0.  A
    device that took the sphere's transform at t = 0 for every time would return -0 at t = -0.5."""
    torch = _torch()
    scene, keep = _worked_example()
    oracle = rayoracle.RayOracle(C.byref(scene), keepalive=keep)
    r = tb.Renderer(C.byref(scene))
    rays = _cross(raysets.pack([(-0.0, 5.0, 0.0)], [(-0.0, -1.0, 0.0)], 0.0), TIMES)
    check_ray_queries(r, oracle, rays, "sphere at -0")
    one = raysets.pack([(-0.0, 5.0, 0.0)], [(-0.0, -1.0, 0.0)], -0.5)
    hits, prims = (x.cpu().numpy() for x in r.trace_rays(torch.from_numpy(one).cuda()))
    assert prims[0] == 0 and hits[0, 0] == 4.0 and hits[0, 1:4].view(np.uint32).tolist() == [0, 0x3f800000, 0], hits[0]
    r.close()
    oracle.close()


# ---- 2. light and emitter queries at every time ----


def _seeds(rng, n):
    return rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(np.int32)


def _lights(scene):
    return [i for i in range(scene.numPrimitives) if scene.primitives[i].lightSamples > 0]


@pytest.mark.parametrize("family,seed", FAMILY_SCENES)
def test_light_queries_at_every_time(family, seed, tmp_path):
    path = _path("fuzz_%s_%d" % (family, seed), tmp_path)
    snap = tb.Snapshot(path)
    oracle = rayoracle.RayOracle.from_snapshot(path)
    r = tb.Renderer(snap.scene)
    check_lights_and_emitters(r, snap, oracle, np.random.default_rng(29), TIMES, "%s/%d" % (family, seed))
    r.close()
    oracle.close()
    snap.close()


def _hit_records(r, snap, oracle, rng, times):
    """Light queries at the hits of camera and zero-plane rays, crossed with `times`."""
    torch = _torch()
    scene = snap.scene.contents
    rays = np.concatenate([raysets.camera_rays(snap.camera, 1024, np.random.RandomState(int(rng.integers(1 << 30)))),
                           _zero_plane_rays(scene, np.random.RandomState(int(rng.integers(1 << 30))), 512)])
    h, p = oracle.trace_rays(rays)
    keep = p >= 0
    rays, h, p = rays[keep], h[keep], p[keep]
    rays = _cross(rays, times)
    h, p = np.repeat(h, len(times), axis=0), np.repeat(p, len(times))
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    o, d = cuda(rays[:, 0:3]), cuda(rays[:, 4:7])
    return tb.light_queries(cuda(p), o + d * cuda(h[:, 0:1]), cuda(h[:, 1:4]), -d, 1.0, 1.5, cuda(rays[:, 3]))


def check_lights_and_emitters(r, snap, oracle, rng, times, what):
    """sample_lights over hit records and sample_emitters of every light, each crossed with `times`."""
    torch = _torch()
    q = _hit_records(r, snap, oracle, rng, times)
    seeds = _seeds(rng, q.shape[0])
    got = r.sample_lights(q, torch.from_numpy(seeds).cuda()).cpu().numpy()
    want = lightoracle.sample_lights(snap.scene, q.cpu().numpy(), seeds)
    bad = ~_same(got, want).all(1)
    assert not bad.any(), "%s sample_lights: %d of %d differ; first record %s" % (what, bad.sum(), len(bad), q[int(np.argmax(bad))].cpu().numpy())
    lights = _lights(snap.scene.contents)
    assert lights
    n = 512 * len(times)
    for light in lights:
        t = np.tile(np.asarray(times, F32), n // len(times))
        seeds = _seeds(rng, n)
        eq = tb.emitter_queries(torch.full((n,), light, dtype=torch.int32, device="cuda"), torch.from_numpy(t).cuda())
        out = torch.full((n, 8), float("nan"), device="cuda")
        r.sample_emitters(eq, torch.from_numpy(seeds).cuda(), out)
        got = out.cpu().numpy()
        want = emitteroracle.sample_emitters(snap.scene, eq.cpu().numpy(), seeds)
        bad = ~_same(got, want).all(1)
        assert not bad.any(), "%s sample_emitters light %d: %d of %d differ; first time %r device %s restatement %s" % (
            what, light, bad.sum(), n, t[int(np.argmax(bad))], got[int(np.argmax(bad))], want[int(np.argmax(bad))])


# ---- 3. camera samples under any shutter ----


@pytest.mark.parametrize("shutter", [(-0.5, 0.5), (1.0, 0.0), (0.3, 0.3), (-0.0, -0.0), (-1e30, 1e30)])
def test_camera_rays_under_any_shutter(shutter):
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("motionblur"))
    cam = abi.copy_struct(snap.camera)
    cam.shutterStart, cam.shutterEnd = shutter
    r = tb.Renderer(snap.scene)
    W, H = 64, 48
    opt = abi.copy_struct(snap.options)
    opt.width, opt.height = W, H
    rng = np.random.default_rng(31)
    s = np.stack([rng.integers(0, W * H, 1 << 14), rng.integers(-2 ** 31, 2 ** 31, 1 << 14)], 1).astype(np.int32)
    rays, raster = (x.cpu().numpy() for x in r.camera_rays(cam, opt, torch.from_numpy(s).cuda()))
    o, d, t, ras = cameraoracle.camera_samples(cam, W, H, s)
    want = np.concatenate([o, t[:, None], d, np.full((len(t), 1), np.inf, F32)], 1).astype(F32)
    bad = ~(_same(rays, want).all(1) & _same(raster, ras).all(1))
    assert not bad.any(), "shutter %r: %d of %d samples differ; first device %s restatement %s" % (
        shutter, bad.sum(), len(bad), rays[int(np.argmax(bad))], want[int(np.argmax(bad))])
    if shutter[0] == shutter[1]:    # Lerp(a, a, t) = a + 0 t: a itself, but +0 for a = -0
        assert (rays[:, 3].view(np.uint32) == (F32(shutter[0]) + F32(0.0)).view(np.uint32)).all()
    r.close()
    snap.close()


# ---- 4. the renderer's own samples ----

VARIANTS = [("default", None, None, False)] + [("sched", s, c, False) for s in schedenv.SCHEDS for c in schedenv.CTAS] + \
           [("sched", "free", "768", True)]


@pytest.mark.parametrize("family,seed", FAMILY_SCENES)
def test_renderer_samples_under_every_scheduler_variant(family, seed, tmp_path):
    path = str(tmp_path / "s.tsnap")
    fuzzscene.make_mesh_scene(seed, path, family, width=96, height=64)
    port = refdrv.PortScene.from_snapshot(path)
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    want = {frame: port.trace_frame(frame, 8) for frame in (0, 3)}
    bad = {}
    for kind, sched, cta, no_flat in VARIANTS:
        with schedenv.knobs(**(schedenv.sched_knobs(sched, cta, no_flat) if sched else {})):
            r = tb.Renderer(snap.scene)
        r.Init(opt.width, opt.height)
        for frame, (prad, pras) in want.items():
            rad, ras = r.trace_frame(cam, opt, frame)
            assert np.array_equal(ras, pras)
            n = int((~_same(rad, prad).all(-1)).sum())
            if n:
                bad[(sched or kind, cta, no_flat, frame)] = n
        r.close()
    assert not bad, "%s/%d: samples differ %s" % (family, seed, bad)
    # the accumulated image against the seeded restatement (the framebuffer sums run in another order)
    with schedenv.knobs():
        r = tb.Renderer(snap.scene)
    r.Init(opt.width, opt.height)
    out = np.zeros((opt.height, opt.width, 4), F32)
    for _ in range(4):
        r.Render(cam, opt, out)
    expect = port.render_seeded(0, 4, nthreads=8)
    nan = np.isnan(out).any(-1)
    assert np.array_equal(nan, np.isnan(expect).any(-1))
    rel = np.linalg.norm((out[~nan] - expect[~nan]).astype(np.float64)) / np.linalg.norm(expect[~nan].astype(np.float64))
    assert rel <= 1e-4, rel
    r.close()
    port.close()
    snap.close()


# ---- 5. non-finite times ----


@pytest.mark.parametrize("seed", [0, 1])
def test_nonfinite_times_are_exact_where_everything_moves(seed, tmp_path):
    """The rotating family interpolates every sphere and mesh at the ray's time (its planes ignore transforms), so even
    an infinite or NaN time is exact: the exception for static primitives is no wider than the contracts say."""
    path = _path("fuzz_rotating_%d" % seed, tmp_path)
    snap = tb.Snapshot(path)
    oracle = rayoracle.RayOracle.from_snapshot(path)
    r = tb.Renderer(snap.scene)
    scene = snap.scene.contents
    assert all(not fuzzscene.is_static(scene.primitives[i]) for i in range(scene.numPrimitives) if scene.primitives[i].type != abi.PLANE)
    rng = np.random.RandomState(37)
    for what, rays in _ray_sets(snap, oracle, rng).items():
        check_ray_queries(r, oracle, _cross(rays, NONFINITE_TIMES), "rotating %d/%s" % (seed, what))
    check_lights_and_emitters(r, snap, oracle, np.random.default_rng(38), NONFINITE_TIMES, "rotating %d" % seed)
    r.close()
    oracle.close()
    snap.close()


@pytest.mark.parametrize("seed", [0, 1])
def test_nonfinite_times_on_static_primitives_write_every_output(seed, tmp_path):
    """The documented exception: a static primitive keeps its transform at a NaN or infinite time, where the reference
    gets NaN.  Every output is still written, and every primitive index is a primitive or -1."""
    torch = _torch()
    path = _path("fuzz_signed_zero_%d" % seed, tmp_path)
    snap = tb.Snapshot(path)
    oracle = rayoracle.RayOracle.from_snapshot(path)
    r = tb.Renderer(snap.scene)
    scene = snap.scene.contents
    rays = np.concatenate(list(_ray_sets(snap, oracle, np.random.RandomState(41)).values()))
    rays = torch.from_numpy(_cross(rays, NONFINITE_TIMES)).cuda()
    n = rays.shape[0]
    sentinel = 0x7fbadbad
    filled = lambda shape: torch.full(shape, sentinel, dtype=torch.int32, device="cuda")
    hits, prims, tris = filled((n, 4)), filled((n,)), filled((n, 4))
    r.trace_rays_tri(rays, hits.view(torch.float32), prims, tris)
    for x in (hits, prims, tris):
        assert (x != sentinel).all()
    assert ((prims >= -1) & (prims < scene.numPrimitives)).all()
    occ = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    r.occluded(rays, occ.view(torch.bool))
    assert (occ <= 1).all()
    q = _hit_records(r, snap, oracle, np.random.default_rng(42), NONFINITE_TIMES)
    rad = torch.full((q.shape[0], 3), sentinel, dtype=torch.int32, device="cuda")
    r.sample_lights(q, torch.zeros(q.shape[0], dtype=torch.int32, device="cuda"), rad.view(torch.float32))
    assert (rad != sentinel).all()
    for light in _lights(scene):
        t = torch.from_numpy(np.tile(NONFINITE_TIMES, 64)).cuda()
        eq = tb.emitter_queries(torch.full((t.shape[0],), light, dtype=torch.int32, device="cuda"), t)
        out = torch.full((t.shape[0], 8), sentinel, dtype=torch.int32, device="cuda")
        r.sample_emitters(eq, torch.zeros(t.shape[0], dtype=torch.int32, device="cuda"), out.view(torch.float32))
        assert (out != sentinel).all()
    torch.cuda.synchronize()
    r.close()
    oracle.close()
    snap.close()
