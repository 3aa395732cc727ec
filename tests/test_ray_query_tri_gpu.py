"""The closest-hit query with the hit triangle on the device (tb200_trace_rays_tri / Renderer.trace_rays_tri) against
the CPU restatement (tests/trioracle.py), per ray and bit for bit: the primitive, the bits of t and of the normal, the
triangle and the bits of u, v, w.  Its hits and primitives are also tb200_trace_rays' own, bit for bit, and its
triangle records pass trioracle.check_semantics.  Every snapshot with camera, random, secondary and fallback rays;
motion blur; every fuzzscene family; a mesh BVH from tb200_bvh_build; the upload and multi-device variants; ray
counts; streams; side effects; and the refusals of bad arguments."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import fuzzscene
import raysets
import schedenv
import trioracle

pytestmark = pytest.mark.gpu

SNAPSHOTS = sorted(f[:-6] for f in os.listdir(tb.SCENE_DIR) if f.endswith(".tsnap"))
N = 1 << 15


def _torch():
    import torch
    return torch


def _query(r, rays):
    """trace_rays_tri and trace_rays of the same rays on the device: (hits, prims, tri, uvw) of the first, as numpy,
    after checking that its hits and prims are the second's, bit for bit."""
    torch = _torch()
    dev = torch.from_numpy(np.ascontiguousarray(rays)).cuda(r.device)
    hits, prims, tri, uvw = r.trace_rays_tri(dev)
    assert tri.dtype == torch.int32 and tri.shape == (len(rays),) and uvw.dtype == torch.float32 and uvw.shape == (len(rays), 3)
    hits, prims, tri, uvw = hits.cpu().numpy(), prims.cpu().numpy(), tri.cpu().numpy(), uvw.cpu().numpy()
    plain_h, plain_p = r.trace_rays(dev)
    assert (plain_h.cpu().numpy().view(np.uint32) == hits.view(np.uint32)).all() and (plain_p.cpu().numpy() == prims).all(), \
        "trace_rays_tri's hits or prims differ from trace_rays'"
    return hits, prims, tri, uvw


def _check(r, oracle, scene, rays, what=""):
    hits, prims, tri, uvw = _query(r, rays)
    want_h, want_p, want_tri, want_uvw = oracle.trace_rays_tri(rays)
    bad = raysets.mismatches(hits, prims, want_h, want_p)
    bad = np.union1d(bad, np.nonzero((tri != want_tri) | (uvw.view(np.uint32) != want_uvw.view(np.uint32)).any(axis=1))[0])
    assert len(bad) == 0, "%s: %d of %d rays differ; first ray %s: device %s %s %s %s, port %s %s %s %s" % (
        what, len(bad), len(rays), rays[bad[0]], prims[bad[0]], hits[bad[0]], tri[bad[0]], uvw[bad[0]],
        want_p[bad[0]], want_h[bad[0]], want_tri[bad[0]], want_uvw[bad[0]])
    return trioracle.check_semantics(scene, rays, hits, prims, tri, uvw, what)


def _ray_sets(scene, camera, oracle, rng):
    """test_ray_query_gpu's sets: camera rays through jittered raster positions, random rays in and around the scene,
    secondary rays from the camera rays' hit points, and rays that reach the ordered fallback."""
    cam = raysets.camera_rays(camera, N, rng)
    h, p = oracle.trace_rays(cam)
    return {"camera": cam, "random": raysets.random_rays(scene, N, rng), "secondary": raysets.secondary_rays(cam, h, p, rng),
            "fallback": raysets.fallback_rays(scene, rng)}


def test_snapshots_hit_meshes_and_other_primitives():
    """The snapshot test below must see both kinds of hit: it checks that records are set on one and cleared on the other."""
    seen = np.zeros(2, np.int64)
    for name in SNAPSHOTS:
        snap = tb.Snapshot(tb.scene_path(name))
        oracle = trioracle.TriOracle.from_snapshot(tb.scene_path(name))
        r = tb.Renderer(snap.scene)
        seen += _check(r, oracle, snap.scene.contents, raysets.camera_rays(snap.camera, 4096, np.random.RandomState(2)), name)
        r.close()
        oracle.close()
        snap.close()
    assert seen[0] > 0 and seen[1] > 0, seen


@pytest.mark.parametrize("name", SNAPSHOTS)
def test_snapshot_rays_match_port(name):
    snap = tb.Snapshot(tb.scene_path(name))
    oracle = trioracle.TriOracle.from_snapshot(tb.scene_path(name))
    r = tb.Renderer(snap.scene)
    scene = snap.scene.contents
    rng = np.random.RandomState(zlib.crc32(name.encode()) & 0xffff)
    sets = _ray_sets(scene, snap.camera, oracle, rng)
    if name == "motionblur":   # times in and outside the shutter
        sets["motion"] = raysets.camera_rays(snap.camera, N, rng, time=rng.uniform(-0.5, 1.5, N))
        sets["motion_random"] = raysets.random_rays(scene, N, rng, (-0.5, 1.5))
    for what, rays in sets.items():
        _check(r, oracle, scene, rays, "%s/%s" % (name, what))
    r.close()
    oracle.close()
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
    oracle = trioracle.TriOracle.from_snapshot(path)
    r = tb.Renderer(snap.scene)
    scene = snap.scene.contents
    rng = np.random.RandomState(seed + 17)
    sets = _ray_sets(scene, snap.camera, oracle, rng)
    sets["times"] = raysets.random_rays(scene, N, rng, (-0.5, 1.5))
    mesh_hits = 0
    for what, rays in sets.items():
        mesh_hits += _check(r, oracle, scene, rays, "%s/%d/%s" % (family, seed, what))[0]
    assert mesh_hits > 0
    r.close()
    oracle.close()
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
    oracle = trioracle.TriOracle(C.byref(scene), keepalive=(keep, nodes))
    r = tb.Renderer(C.byref(scene))
    mesh_hits = 0
    for what, rays in _ray_sets(scene, cam, oracle, rng).items():
        mesh_hits += _check(r, oracle, scene, rays, "bvh_build/" + what)[0]
    assert mesh_hits > 0
    r.close()
    oracle.close()
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
    oracle = trioracle.TriOracle.from_snapshot(path)
    rng = np.random.RandomState(5)
    rays = np.concatenate(list(_ray_sets(snap.scene.contents, snap.camera, oracle, rng).values()))
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
    _check(r, oracle, snap.scene.contents, rays, "%s/%s" % (name, variant))
    r.close()
    oracle.close()
    snap.close()


@pytest.mark.parametrize("count", [1, 31, 33, 10 ** 6 + 7])
def test_ray_counts(count):
    snap = tb.Snapshot(tb.scene_path("meshlight"))
    oracle = trioracle.TriOracle.from_snapshot(tb.scene_path("meshlight"))
    r = tb.Renderer(snap.scene)
    rays = raysets.random_rays(snap.scene.contents, count, np.random.RandomState(count % 1000))
    _check(r, oracle, snap.scene.contents, rays, "count %d" % count)
    r.close()
    oracle.close()
    snap.close()


def test_rays_written_on_the_callers_stream():
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("meshlight"))
    oracle = trioracle.TriOracle.from_snapshot(tb.scene_path("meshlight"))
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
        hits, prims, tri, uvw = r.trace_rays_tri(dst)
    want_h, want_p, want_tri, want_uvw = oracle.trace_rays_tri(rays)
    assert len(raysets.mismatches(hits.cpu().numpy(), prims.cpu().numpy(), want_h, want_p)) == 0
    assert (tri.cpu().numpy() == want_tri).all() and (uvw.cpu().numpy().view(np.uint32) == want_uvw.view(np.uint32)).all()
    assert (want_tri >= 0).any()
    r.set_stream(None)
    r.close()
    oracle.close()
    snap.close()


def test_query_has_no_side_effects():
    snap = tb.Snapshot(tb.scene_path("meshlight"))
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = 64, 48
    oracle = trioracle.TriOracle.from_snapshot(tb.scene_path("meshlight"))
    scene = snap.scene.contents
    rays = raysets.random_rays(scene, 4096, np.random.RandomState(11))
    fresh = tb.Renderer(snap.scene)
    _check(fresh, oracle, scene, rays, "before Init")   # no film needed
    fresh.close()

    r = tb.Renderer(snap.scene)
    r.Init(64, 48)
    out = np.zeros((48, 64, 4), np.float32)
    r.Render(cam, opt, out)
    rad0, _ = r.trace_frame(cam, opt, 0)
    acc0, st0, kernel0 = r.read_accumulator(), r.stats(), r.last_kernel()
    torch = _torch()
    r.trace_rays_tri(torch.from_numpy(rays).cuda())
    st1 = r.stats()
    assert (st1.frames, st1.samples) == (st0.frames, st0.samples)
    assert st1.kernelLaunches == st0.kernelLaunches + 1
    assert st1.gpuMs > 0.0
    assert r.last_kernel() == kernel0
    assert (r.read_accumulator().view(np.uint32) == acc0.view(np.uint32)).all()
    rad1, _ = r.trace_frame(cam, opt, 0)   # the frame counter did not move
    assert (rad0.view(np.uint32) == rad1.view(np.uint32)).all()
    r.close()
    oracle.close()
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
    tris = torch.empty((n, 4), dtype=torch.int32, device="cuda")
    host = np.zeros((n, 8), np.float32)
    launches = r.stats().kernelLaunches

    def refused(a, b, c, d, count, words):
        assert lib.tb200_trace_rays_tri(r.h, a, b, c, d, count) != 0
        msg = tb.last_error()
        assert "tb200_trace_rays_tri" in msg and any(w in msg for w in words), msg

    ok = [rays.data_ptr(), hits.data_ptr(), prims.data_ptr(), tris.data_ptr()]
    for k, name in enumerate(("rays", "hits", "prims", "tris")):
        args = list(ok)
        args[k] = host.ctypes.data
        refused(*args, n, [name + " is not device memory"])
        args[k] = None
        refused(*args, n, [name + " is null"])
        if name != "prims":   # prims needs 4 bytes, the others 16
            args[k] = ok[k] + 4
            refused(*args, n - 1, [name + " is not aligned"])
    refused(*ok, -1, ["out of range"])
    # a tensor that owns its whole segment: the caching allocator gives a fresh 20 MiB tensor a segment of its own
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    big_n = (20 << 20) // 16
    big_tris = torch.empty((big_n, 4), dtype=torch.int32, device="cuda")
    big_rays = torch.zeros((big_n + 1, 8), dtype=torch.float32, device="cuda")
    big_hits = torch.empty((big_n + 1, 4), dtype=torch.float32, device="cuda")
    big_prims = torch.empty((big_n + 1,), dtype=torch.int32, device="cuda")
    big = [big_rays.data_ptr(), big_hits.data_ptr(), big_prims.data_ptr(), big_tris.data_ptr()]
    refused(*big, big_n + 1, ["tris: %d bytes from this address run past the end" % ((big_n + 1) * 16)])
    assert r.stats().kernelLaunches == launches
    assert lib.tb200_trace_rays_tri(r.h, None, None, None, None, 0) == 0   # nothing to do: nothing launched
    assert r.stats().kernelLaunches == launches
    assert lib.tb200_trace_rays_tri(r.h, *big, big_n) == 0
    assert r.stats().kernelLaunches == launches + 1
    # the Python interface checks types, shapes, dtypes, contiguity and the device itself
    with pytest.raises(TypeError):
        r.trace_rays_tri(rays.double())
    with pytest.raises(ValueError):
        r.trace_rays_tri(rays[:, :4].contiguous())
    with pytest.raises(ValueError):
        r.trace_rays_tri(torch.zeros((8, n), dtype=torch.float32, device="cuda").t())
    with pytest.raises(ValueError):
        r.trace_rays_tri(rays.cpu())
    with pytest.raises(ValueError):
        r.trace_rays_tri(rays, hits=hits[:-1])
    with pytest.raises(TypeError):
        r.trace_rays_tri(rays, tris=tris.float())
    with pytest.raises(TypeError):
        r.trace_rays_tri(rays, tris=np.zeros((n, 4), np.int32))
    with pytest.raises(ValueError):
        r.trace_rays_tri(rays, tris=tris[:, :3].contiguous())
    with pytest.raises(ValueError):
        r.trace_rays_tri(rays, tris=tris.cpu())
    with pytest.raises(ValueError):
        r.trace_rays_tri(rays, tris=torch.empty((4, n), dtype=torch.int32, device="cuda").t())
    assert r.stats().kernelLaunches == launches + 1
    h0, p0, t0, w0 = r.trace_rays_tri(rays[:0])
    assert h0.shape == (0, 4) and p0.shape == (0,) and t0.shape == (0,) and w0.shape == (0, 3)
    # results land in the tensors the caller passes
    h1, p1, t1, w1 = r.trace_rays_tri(rays, hits, prims, tris)
    assert h1.data_ptr() == hits.data_ptr() and p1.data_ptr() == prims.data_ptr() and t1.data_ptr() == tris.data_ptr()
    assert w1.data_ptr() == tris.data_ptr() + 4
    r.close()
    snap.close()
