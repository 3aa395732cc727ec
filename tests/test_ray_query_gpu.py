"""The batched closest-hit query on the device (tb200_trace_rays / Renderer.trace_rays) against the CPU restatement's
Trace (render.cpp:17-62, batched by tests/rayoracle.py), per ray and bit for bit: the primitive, and the bits of t and of the face-forwarded normal.
Every snapshot with camera, random and secondary rays; rays that reach the ordered fallback; motion blur; every
fuzzscene family; a mesh BVH from tb200_bvh_build; the scheduling and upload variants; consistency with eNormals;
streams; side effects; and the refusals of bad arguments."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import fuzzscene
import rayoracle
import raysets
import refdrv
import schedenv

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SNAPSHOTS = sorted(f[:-6] for f in os.listdir(os.path.join(ROOT, "scenes")) if f.endswith(".tsnap"))
N = 1 << 15


@pytest.fixture(scope="module", autouse=True)
def port_built():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "port"])


def _torch():
    import torch
    return torch


def _query(r, rays):
    torch = _torch()
    hits, prims = r.trace_rays(torch.from_numpy(np.ascontiguousarray(rays)).cuda(r.device))
    return hits.cpu().numpy(), prims.cpu().numpy()


def _check(r, port, rays, what=""):
    hits, prims = _query(r, rays)
    want_h, want_p = port.trace_rays(rays)
    bad = raysets.mismatches(hits, prims, want_h, want_p)
    assert len(bad) == 0, "%s: %d of %d rays differ; first ray %s: device %s %s, port %s %s" % (
        what, len(bad), len(rays), rays[bad[0]], prims[bad[0]], hits[bad[0]], want_p[bad[0]], want_h[bad[0]])
    return hits, prims


def _ray_sets(scene, camera, port, rng):
    """Camera rays through jittered raster positions, random rays in and around the scene, secondary rays from the
    camera rays' hit points, and rays that reach the ordered fallback."""
    cam = raysets.camera_rays(camera, N, rng)
    h, p = port.trace_rays(cam)
    return {"camera": cam, "random": raysets.random_rays(scene, N, rng), "secondary": raysets.secondary_rays(cam, h, p, rng),
            "fallback": raysets.fallback_rays(scene, rng)}


@pytest.mark.parametrize("name", SNAPSHOTS)
def test_snapshot_rays_match_port(name):
    snap = tb.Snapshot(tb.scene_path(name))
    port = rayoracle.RayOracle.from_snapshot(tb.scene_path(name))
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(zlib.crc32(name.encode()) & 0xffff)
    time = (-0.5, 1.5) if name == "motionblur" else None
    sets = _ray_sets(snap.scene.contents, snap.camera, port, rng)
    if time:
        sets["motion"] = raysets.camera_rays(snap.camera, N, rng, time=rng.uniform(time[0], time[1], N))
        sets["motion_random"] = raysets.random_rays(snap.scene.contents, N, rng, time)
    for what, rays in sets.items():
        hits, prims = _check(r, port, rays, "%s/%s" % (name, what))
        if what == "camera":
            assert (prims >= 0).any()
    if refdrv.have_ref("detmath"):
        ref = refdrv.RefScene.from_snapshot(tb.scene_path(name), "detmath")
        rays = np.concatenate(list(sets.values()))
        sub = rays[rng.choice(len(rays), 300, replace=False)]
        hits, prims = _query(r, sub)
        for i, ray in enumerate(sub):
            prim, t, n = ref.trace(ray[0:3], ray[4:7], float(ray[3]))
            want = np.array([t, n[0], n[1], n[2]], np.float32)
            assert prim == prims[i] and len(raysets.mismatches(hits[i:i + 1], prims[i:i + 1], want[None], np.array([prim]))) == 0, ray
        ref.close()
    r.close()
    port.close()
    snap.close()


FUZZ = [("ties", 0, False), ("ties", 0, True), ("ties", 3, True), ("many", 1, False), ("big", 0, False),
        ("caterpillar", 0, False), ("instanced", 0, False), ("instanced", 1, False), ("instanced", 2, False), ("probe", 0, False)]


@pytest.mark.parametrize("family,seed,swap", FUZZ)
def test_fuzz_scenes_match_port(family, seed, swap, tmp_path):
    path = str(tmp_path / "s.tsnap")
    info = fuzzscene.make_mesh_scene(seed, path, family, swap_ties=swap, levels=30 if family == "caterpillar" else None)
    if family == "caterpillar":
        assert info["levels"] == 30
    if family == "big":
        assert max(info["tris"]) > 4096
    snap = tb.Snapshot(path)
    port = rayoracle.RayOracle.from_snapshot(path)
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(seed + 17)
    sets = _ray_sets(snap.scene.contents, snap.camera, port, rng)
    sets["times"] = raysets.random_rays(snap.scene.contents, N, rng, (-0.5, 1.5))
    for what, rays in sets.items():
        _check(r, port, rays, "%s/%d/%s" % (family, seed, what))
    r.close()
    port.close()
    snap.close()


def test_mesh_with_device_built_bvh_matches_port():
    p, n, f = fuzzscene._icosphere(4, np.random.RandomState(3), bump=0.05)
    mesh = fuzzscene.MeshData(p, n, f)
    nodes = np.zeros((2 * len(mesh.idx) - 1) * 8, np.float32)
    tb.bvh_build(mesh.pos, mesh.idx, nodes)
    rng = np.random.RandomState(4)
    prims = (abi.Primitive * 3)()
    bounds = [fuzzscene._floor(prims[0], rng)]
    prims[1].material = fuzzscene._material(rng, False)
    bounds.append(fuzzscene._instance(prims[1], 0, mesh, (0.0, 1.0, 0.0), fuzzscene._quat(rng), 0.8, (0.2, 1.1, 0.0)))
    bounds.append(fuzzscene._sphere(prims[2], (0.0, 3.0, 1.0), 0.3, fuzzscene._material(rng, True), 1))
    scene, keep = fuzzscene.make_scene_struct(prims, fuzzscene._build_bvh(bounds), [mesh])
    scene.meshes[0].nodes = nodes.ctypes.data_as(C.POINTER(abi.BvhNode))
    scene.meshes[0].numNodes = 2 * len(mesh.idx) - 1
    base = tb.Snapshot(tb.scene_path("cornell"))
    cam = abi.copy_struct(base.camera)
    cam.position[:] = [0.0, 1.2, 6.0]
    cam.rotation[:] = [0.0, 0.0, 0.0, 1.0]
    port = rayoracle.RayOracle(C.byref(scene), keepalive=(keep, nodes))
    r = tb.Renderer(C.byref(scene))
    for what, rays in _ray_sets(scene, cam, port, rng).items():
        _check(r, port, rays, "bvh_build/" + what)
    r.close()
    port.close()
    base.close()


@pytest.mark.parametrize("variant", ["no_flat", "cached", "group"])
@pytest.mark.parametrize("name", ["cornell", "meshlight", "fuzz_instanced"])
def test_variants_give_the_same_bits(variant, name, tmp_path):
    if name.startswith("fuzz_"):
        path = str(tmp_path / "s.tsnap")
        fuzzscene.make_mesh_scene(2, path, name[5:])
    else:
        path = tb.scene_path(name)
    snap = tb.Snapshot(path)
    port = rayoracle.RayOracle.from_snapshot(path)
    rng = np.random.RandomState(5)
    rays = np.concatenate(list(_ray_sets(snap.scene.contents, snap.camera, port, rng).values()))
    if variant == "no_flat":
        with schedenv.knobs(**schedenv.ROUTES["no-flat"]):
            r = tb.Renderer(snap.scene)
    elif variant == "cached":
        cache = str(tmp_path / "s.tcache")
        tb.scene_cache_save(snap.scene, cache)
        r = tb.Renderer(None, cache=cache)
    else:
        with schedenv.knobs(TEST_DUP_DEVICES="1"):
            r = tb.Renderer(snap.scene, devices=[0, 0])
        assert r.num_devices() == 2
    _check(r, port, rays, "%s/%s" % (name, variant))
    r.close()
    port.close()
    snap.close()


def test_normals_image_equals_the_query():
    """eNormals (render.cpp:494-515) is Trace of the integer-raster camera rays at time 1.0: n*0.5+0.5, alpha 1."""
    snap = tb.Snapshot(tb.scene_path("veach"))
    cam, opt = snap.camera, snap.options
    W, H = 96, 72
    opt.width, opt.height, opt.mode = W, H, abi.MODE_NORMALS
    r = tb.Renderer(snap.scene)
    r.Init(W, H)
    img = np.zeros((H, W, 4), np.float32)
    r.Render(cam, opt, img)
    lib = refdrv.load_port()
    rays = np.zeros((H * W, 8), np.float32)
    o, d = np.zeros(3, np.float32), np.zeros(3, np.float32)
    for j in range(H):
        for i in range(W):
            lib.oracle_generate_ray(C.byref(cam), W, H, float(i), float(j), refdrv._fp(o), refdrv._fp(d))
            rays[j * W + i] = [o[0], o[1], o[2], 1.0, d[0], d[1], d[2], 0.0]
    hits, prims = _query(r, rays)
    want = np.zeros((H * W, 4), np.float32)
    hit = prims >= 0
    want[hit, 0:3] = hits[hit, 1:4] * np.float32(0.5) + np.float32(0.5)
    want[hit, 3] = 1.0
    assert hit.any() and (img.reshape(-1, 4).view(np.uint32) == want.view(np.uint32)).all()
    r.close()
    snap.close()


@pytest.mark.parametrize("count", [1, 31, 33, 10 ** 6 + 7])
def test_ray_counts(count):
    snap = tb.Snapshot(tb.scene_path("cornell"))
    port = rayoracle.RayOracle.from_snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(count % 1000)
    rays = raysets.random_rays(snap.scene.contents, count, rng)
    hits, prims = _check(r, port, rays, "count %d" % count)
    assert hits.shape == (count, 4) and prims.shape == (count,)
    r.close()
    port.close()
    snap.close()


def test_rays_written_on_the_callers_stream():
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("meshlight"))
    port = rayoracle.RayOracle.from_snapshot(tb.scene_path("meshlight"))
    r = tb.Renderer(snap.scene)
    rays = raysets.random_rays(snap.scene.contents, N, np.random.RandomState(9))
    src = torch.from_numpy(rays).cuda()
    dst = torch.zeros_like(src)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    r.set_stream(s.cuda_stream)
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)   # the copy below lands well after the call has been queued
        dst.copy_(src)
        hits, prims = r.trace_rays(dst)
    want_h, want_p = port.trace_rays(rays)
    assert len(raysets.mismatches(hits.cpu().numpy(), prims.cpu().numpy(), want_h, want_p)) == 0
    r.set_stream(None)
    r.close()
    port.close()
    snap.close()


def test_query_has_no_side_effects():
    snap = tb.Snapshot(tb.scene_path("cornell"))
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = 64, 48
    port = rayoracle.RayOracle.from_snapshot(tb.scene_path("cornell"))
    rays = raysets.random_rays(snap.scene.contents, 4096, np.random.RandomState(11))
    fresh = tb.Renderer(snap.scene)
    _check(fresh, port, rays, "before Init")   # no film needed
    fresh.close()

    # the accumulator sums splats in whatever order the device retires them, so two renderers are compared with a
    # tolerance: a frame counter moved by the query would seed other samples and miss it by orders of magnitude
    out = [np.zeros((48, 64, 4), np.float32) for _ in range(2)]
    for k, query in enumerate((False, True)):
        r = tb.Renderer(snap.scene)
        r.Init(64, 48)
        r.Render(cam, opt, out[k])
        rad0, _ = r.trace_frame(cam, opt, 0)
        if query:
            acc0, st0, kernel0 = r.read_accumulator(), r.stats(), r.last_kernel()
            _check(r, port, rays, "after Render")
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


def test_bad_arguments_are_refused_before_any_launch():
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    lib = r.lib
    n = 64
    rays = torch.from_numpy(raysets.random_rays(snap.scene.contents, n, np.random.RandomState(1))).cuda()
    hits = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    prims = torch.empty((n,), dtype=torch.int32, device="cuda")
    host = np.zeros((n, 8), np.float32)
    launches = r.stats().kernelLaunches

    def refused(a, b, c, count, words):
        assert lib.tb200_trace_rays(r.h, a, b, c, count) != 0
        msg = tb.last_error()
        assert any(w in msg for w in words), msg

    refused(host.ctypes.data, hits.data_ptr(), prims.data_ptr(), n, ["not device memory"])
    refused(rays.data_ptr(), host.ctypes.data, prims.data_ptr(), n, ["not device memory"])
    refused(rays.data_ptr() + 4, hits.data_ptr(), prims.data_ptr(), n - 1, ["aligned"])
    refused(rays.data_ptr(), hits.data_ptr() + 8, prims.data_ptr(), n - 1, ["aligned"])
    refused(rays.data_ptr(), hits.data_ptr(), prims.data_ptr(), -1, ["out of range"])
    refused(None, hits.data_ptr(), prims.data_ptr(), n, ["null"])
    refused(rays.data_ptr(), None, prims.data_ptr(), n, ["null"])
    refused(rays.data_ptr(), hits.data_ptr(), None, n, ["null"])
    # a tensor that owns its whole segment: the caching allocator gives a fresh 20 MiB tensor a segment of its own
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    big_n = (20 << 20) // 32
    big = torch.zeros((big_n, 8), dtype=torch.float32, device="cuda")
    big_hits = torch.empty((big_n + 1, 4), dtype=torch.float32, device="cuda")
    big_prims = torch.empty((big_n + 1,), dtype=torch.int32, device="cuda")
    refused(big.data_ptr(), big_hits.data_ptr(), big_prims.data_ptr(), big_n + 1, ["past the end"])
    assert r.stats().kernelLaunches == launches
    assert lib.tb200_trace_rays(r.h, None, None, None, 0) == 0   # nothing to do: nothing launched
    assert lib.tb200_trace_rays(r.h, big.data_ptr(), big_hits.data_ptr(), big_prims.data_ptr(), big_n) == 0
    assert r.stats().kernelLaunches == launches + 1
    # the Python interface checks shapes, dtypes, contiguity and the device itself
    with pytest.raises(TypeError):
        r.trace_rays(rays.double())
    with pytest.raises(ValueError):
        r.trace_rays(rays[:, :4].contiguous())
    with pytest.raises(ValueError):
        r.trace_rays(torch.zeros((8, n), dtype=torch.float32, device="cuda").t())
    with pytest.raises(ValueError):
        r.trace_rays(rays.cpu())
    with pytest.raises(ValueError):
        r.trace_rays(rays, hits=hits[:-1])
    h0, p0 = r.trace_rays(rays[:0])
    assert h0.shape == (0, 4) and p0.shape == (0,)
    r.close()
    snap.close()
