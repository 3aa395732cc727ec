"""The batched occlusion query on the device (tb200_occluded_rays / Renderer.occluded) against the CPU restatement's
Trace (render.cpp:17-62, batched by tests/rayoracle.py), per ray and exactly: a ray is occluded iff Trace hits a
primitive and its t < tmax (column 7 of the ray).  Every snapshot with camera, random, secondary and fallback rays,
each crossed with tmax = +inf, uniform below twice the closest t, and the edge values around each ray's own t;
point-to-point segment rays; motion blur; every fuzzscene family; a mesh BVH from tb200_bvh_build; the scheduling and
upload variants; ray counts; streams; side effects; and the refusals of bad arguments."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import tinsel_b200 as tb
from queryscenes import FUZZ, N, SNAPSHOTS
import occlusionsets
import queryscenes
import rayoracle
import raysets
import refdrv

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def port_built():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "port"])


def _torch():
    import torch
    return torch


def _query(r, rays):
    torch = _torch()
    return r.occluded(torch.from_numpy(np.ascontiguousarray(rays)).cuda(r.device)).cpu().numpy()


def _check_set(r, rays, hits, prims, what):
    """The device's verdicts on `rays` (tmax in column 7) against those derived from the closest hits hits / prims."""
    got = _query(r, rays)
    want = occlusionsets.occluded(hits, prims, rays[:, 7])
    assert got.dtype == np.bool_ and got.shape == (len(rays),)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, "%s: %d of %d rays differ; first ray %s: device %s, port %s (prim %d, t %r)" % (
        what, len(bad), len(rays), rays[bad[0]], got[bad[0]], want[bad[0]], prims[bad[0]], float(hits[bad[0], 0]))
    return got


def _check(r, port, rays, rng, what=""):
    """`rays` crossed with every tmax set of occlusionsets.tmax_sets; returns the closest hits the sets were built from."""
    hits, prims = port.trace_rays(rays)
    for name, tmax in occlusionsets.tmax_sets(hits, prims, rng).items():
        _check_set(r, occlusionsets.with_tmax(rays, tmax), hits, prims, "%s/tmax=%s" % (what, name))
    return hits, prims


def _check_point_to_point(r, port, camera, rng, what):
    """Segments between the hit points of two camera batches (the shadow-ray use), with tmax 1 - 1e-4 and 1."""
    a = raysets.camera_rays(camera, N, rng)
    b = raysets.camera_rays(camera, N, rng)
    ha, pa = port.trace_rays(a)
    hb, pb = port.trace_rays(b)
    seen = 0
    for tmax in (np.float32(1.0) - np.float32(1e-4), np.float32(1.0)):
        rays = occlusionsets.point_to_point_rays(a, ha, pa, b, hb, pb, np.random.RandomState(1), tmax)
        if len(rays) == 0:
            continue
        hits, prims = port.trace_rays(rays)
        seen += int(_check_set(r, rays, hits, prims, "%s/point_to_point/tmax=%r" % (what, float(tmax))).sum())
    return seen


@pytest.mark.parametrize("name", SNAPSHOTS)
def test_snapshot_occlusion_matches_port(name):
    snap = tb.Snapshot(tb.scene_path(name))
    port = rayoracle.RayOracle.from_snapshot(tb.scene_path(name))
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(zlib.crc32(name.encode()) & 0xffff)
    sets = queryscenes.ray_sets(snap.scene.contents, snap.camera, port, rng)
    if name == "motionblur":   # times outside the shutter too
        sets["motion"] = raysets.camera_rays(snap.camera, N, rng, time=rng.uniform(-0.5, 1.5, N))
        sets["motion_random"] = raysets.random_rays(snap.scene.contents, N, rng, (-0.5, 1.5))
    for what, rays in sets.items():
        _check(r, port, rays, rng, "%s/%s" % (name, what))
    _check_point_to_point(r, port, snap.camera, rng, name)
    if refdrv.have_ref("detmath"):
        # the reference's own Trace on a subset, with tmax on both sides of its t
        ref = refdrv.RefScene.from_snapshot(tb.scene_path(name), "detmath")
        rays = np.concatenate(list(sets.values()))
        sub = rays[rng.choice(len(rays), 300, replace=False)]
        want_t = np.zeros(len(sub), np.float32)
        want_hit = np.zeros(len(sub), bool)
        for i, ray in enumerate(sub):
            prim, t, _ = ref.trace(ray[0:3], ray[4:7], float(ray[3]))
            want_t[i], want_hit[i] = t, prim >= 0
        for tmax in (want_t, np.nextafter(want_t, np.float32(np.inf)), np.full(len(sub), np.inf, np.float32)):
            got = _query(r, occlusionsets.with_tmax(sub, tmax))
            assert (got == (want_hit & (want_t < tmax))).all()
        ref.close()
    r.close()
    port.close()
    snap.close()


@pytest.mark.parametrize("family,seed,swap", FUZZ)
def test_fuzz_scenes_occlusion_matches_port(family, seed, swap, tmp_path):
    path = str(tmp_path / "s.tsnap")
    queryscenes.fuzz_scene(family, seed, swap, path)
    snap = tb.Snapshot(path)
    port = rayoracle.RayOracle.from_snapshot(path)
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(seed + 17)
    sets = queryscenes.ray_sets(snap.scene.contents, snap.camera, port, rng)
    sets["times"] = raysets.random_rays(snap.scene.contents, N, rng, (-0.5, 1.5))
    for what, rays in sets.items():
        _check(r, port, rays, rng, "%s/%d/%s" % (family, seed, what))
    _check_point_to_point(r, port, snap.camera, rng, family)
    r.close()
    port.close()
    snap.close()


def test_mesh_with_device_built_bvh_occlusion_matches_port():
    scene, keep, cam, rng = queryscenes.bvh_build_scene()
    port = rayoracle.RayOracle(C.byref(scene), keepalive=keep)
    r = tb.Renderer(C.byref(scene))
    for what, rays in queryscenes.ray_sets(scene, cam, port, rng).items():
        _check(r, port, rays, rng, "bvh_build/" + what)
    assert _check_point_to_point(r, port, cam, rng, "bvh_build") > 0
    r.close()
    port.close()


@pytest.mark.parametrize("variant", ["no_flat", "cached", "group"])
@pytest.mark.parametrize("name", ["cornell", "meshlight", "fuzz_instanced"])
def test_occlusion_variants_give_the_same_answers(variant, name, tmp_path):
    path = queryscenes.variant_path(name, tmp_path)
    snap = tb.Snapshot(path)
    port = rayoracle.RayOracle.from_snapshot(path)
    rng = np.random.RandomState(5)
    rays = np.concatenate(list(queryscenes.ray_sets(snap.scene.contents, snap.camera, port, rng).values()))
    r = queryscenes.variant_renderer(variant, snap, tmp_path)
    _check(r, port, rays, rng, "%s/%s" % (name, variant))
    _check_point_to_point(r, port, snap.camera, rng, "%s/%s" % (name, variant))
    r.close()
    port.close()
    snap.close()


def test_edge_tmax_pins_the_boundary():
    """tmax equal to the closest hit's t is not occluded, the next float above it is; misses never are."""
    snap = tb.Snapshot(tb.scene_path("veach"))
    port = rayoracle.RayOracle.from_snapshot(tb.scene_path("veach"))
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(21)
    rays = np.concatenate([raysets.camera_rays(snap.camera, N, rng), raysets.random_rays(snap.scene.contents, N, rng)])
    hits, prims = port.trace_rays(rays)
    hit = prims >= 0
    assert hit.any() and (~hit).any()
    sets = occlusionsets.tmax_sets(hits, prims, rng)
    assert not _query(r, occlusionsets.with_tmax(rays, sets["t"])).any()
    assert (_query(r, occlusionsets.with_tmax(rays, sets["t_up"])) == hit).all()
    assert (_query(r, occlusionsets.with_tmax(rays, sets["inf"])) == hit).all()
    for name in ("zero", "minus_zero", "negative", "nan"):
        assert not _query(r, occlusionsets.with_tmax(rays, sets[name])).any(), name
    r.close()
    port.close()
    snap.close()


@pytest.mark.parametrize("count", [1, 31, 33, 10 ** 6 + 7])
def test_occlusion_ray_counts(count):
    snap = tb.Snapshot(tb.scene_path("cornell"))
    port = rayoracle.RayOracle.from_snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(count % 1000)
    rays = raysets.random_rays(snap.scene.contents, count, rng)
    hits, prims = port.trace_rays(rays)
    rays = occlusionsets.with_tmax(rays, rng.uniform(0.0, 2.0, count))
    got = _check_set(r, rays, hits, prims, "count %d" % count)
    assert got.shape == (count,)
    r.close()
    port.close()
    snap.close()


def test_occlusion_on_the_callers_stream():
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("meshlight"))
    port = rayoracle.RayOracle.from_snapshot(tb.scene_path("meshlight"))
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(9)
    rays = raysets.random_rays(snap.scene.contents, N, rng)
    rays[:, 7] = rng.uniform(0.0, 3.0, N)
    src = torch.from_numpy(rays).cuda()
    dst = torch.zeros_like(src)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    r.set_stream(s.cuda_stream)
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)   # the copy below lands well after the call has been queued
        dst.copy_(src)
        got = r.occluded(dst)
    hits, prims = port.trace_rays(rays)
    assert (got.cpu().numpy() == occlusionsets.occluded(hits, prims, rays[:, 7])).all()
    r.set_stream(None)
    r.close()
    port.close()
    snap.close()


def test_occlusion_has_no_side_effects():
    snap = tb.Snapshot(tb.scene_path("cornell"))
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = 64, 48
    port = rayoracle.RayOracle.from_snapshot(tb.scene_path("cornell"))
    rng = np.random.RandomState(11)
    rays = raysets.random_rays(snap.scene.contents, 4096, rng)
    hits, prims = port.trace_rays(rays)
    rays = occlusionsets.with_tmax(rays, rng.uniform(0.0, 2.0, len(rays)))
    fresh = tb.Renderer(snap.scene)
    _check_set(fresh, rays, hits, prims, "before Init")   # no film needed
    fresh.close()

    # as in test_query_has_no_side_effects: a frame counter moved by the query would seed other samples
    out = [np.zeros((48, 64, 4), np.float32) for _ in range(2)]
    for k, query in enumerate((False, True)):
        r = tb.Renderer(snap.scene)
        r.Init(64, 48)
        r.Render(cam, opt, out[k])
        rad0, _ = r.trace_frame(cam, opt, 0)
        if query:
            acc0, st0, kernel0 = r.read_accumulator(), r.stats(), r.last_kernel()
            _check_set(r, rays, hits, prims, "after Render")
            st1 = r.stats()
            assert (st1.frames, st1.samples) == (st0.frames, st0.samples)
            assert st1.kernelLaunches == st0.kernelLaunches + 1
            assert st1.gpuMs > 0.0
            assert r.last_kernel() == kernel0
            assert (r.read_accumulator().view(np.uint32) == acc0.view(np.uint32)).all()
            rad1, _ = r.trace_frame(cam, opt, 0)
            assert (rad0.view(np.uint32) == rad1.view(np.uint32)).all()
        r.Render(cam, opt, out[k])   # the second frame
        r.close()
    rel = np.linalg.norm((out[0] - out[1]).astype(np.float64)) / np.linalg.norm(out[0].astype(np.float64))
    assert rel < 1e-5, rel
    port.close()
    snap.close()


def test_occlusion_bad_arguments_are_refused_before_any_launch():
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    lib = r.lib
    n = 64
    rays = torch.from_numpy(raysets.random_rays(snap.scene.contents, n, np.random.RandomState(1))).cuda()
    occ = torch.empty((n,), dtype=torch.bool, device="cuda")
    host = np.zeros((n, 8), np.float32)
    host_occ = np.zeros(n, np.uint8)
    launches = r.stats().kernelLaunches

    def refused(a, b, count, words):
        assert lib.tb200_occluded_rays(r.h, a, b, count) != 0
        msg = tb.last_error()
        assert msg.startswith("tb200_occluded_rays: ") and any(w in msg for w in words), msg

    refused(host.ctypes.data, occ.data_ptr(), n, ["not device memory"])
    refused(rays.data_ptr(), host_occ.ctypes.data, n, ["not device memory"])
    refused(rays.data_ptr() + 4, occ.data_ptr(), n - 1, ["aligned"])
    refused(rays.data_ptr(), occ.data_ptr(), -1, ["out of range"])
    refused(None, occ.data_ptr(), n, ["null"])
    refused(rays.data_ptr(), None, n, ["null"])
    assert lib.tb200_occluded_rays(None, rays.data_ptr(), occ.data_ptr(), n) != 0
    assert "null renderer" in tb.last_error()
    # a tensor that owns its whole segment: the caching allocator gives a fresh 20 MiB tensor a segment of its own
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    big_n = (20 << 20) // 32
    big = torch.zeros((big_n, 8), dtype=torch.float32, device="cuda")
    big_occ = torch.empty((big_n + 1,), dtype=torch.bool, device="cuda")
    refused(big.data_ptr(), big_occ.data_ptr(), big_n + 1, ["past the end"])
    assert r.stats().kernelLaunches == launches
    assert lib.tb200_occluded_rays(r.h, None, None, 0) == 0   # nothing to do: nothing launched
    assert lib.tb200_occluded_rays(r.h, big.data_ptr(), big_occ.data_ptr(), big_n) == 0
    assert r.stats().kernelLaunches == launches + 1
    assert not big_occ[:big_n].any()   # tmax 0: never occluded
    # the Python interface checks shapes, dtypes, contiguity and the device itself
    with pytest.raises(TypeError):
        r.occluded(rays.double())
    with pytest.raises(TypeError):
        r.occluded(rays, out=torch.empty((n,), dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        r.occluded(rays[:, :4].contiguous())
    with pytest.raises(ValueError):
        r.occluded(torch.zeros((8, n), dtype=torch.float32, device="cuda").t())
    with pytest.raises(ValueError):
        r.occluded(rays.cpu())
    with pytest.raises(ValueError):
        r.occluded(rays, out=occ[:-1])
    with pytest.raises(ValueError):
        r.occluded(rays, out=torch.empty((2 * n,), dtype=torch.bool, device="cuda")[::2])
    assert r.occluded(rays[:0]).shape == (0,)
    r.close()
    snap.close()
