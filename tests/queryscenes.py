"""TEST INFRASTRUCTURE: the scenes, ray sets and renderer variants that the device's ray query tests share
(test_ray_query_gpu.py, test_ray_query_tri_gpu.py, test_occlusion_gpu.py)."""
import ctypes as C
import os

import numpy as np

import tinsel_b200 as tb
from tinsel_b200 import abi
import fuzzscene
import raysets
import schedenv

SNAPSHOTS = sorted(f[:-6] for f in os.listdir(tb.SCENE_DIR) if f.endswith(".tsnap"))
N = 1 << 15   # rays per set
_FMAX = np.finfo(np.float32).max
_DENORM = np.nextafter(np.float32(0.0), np.float32(1.0))
# ray times, inside the shutter and outside: zeros of both signs, the smallest denormals, times near 0 and 1, and
# times where the lerp of a moving primitive overflows
TIMES = np.array([0.0, -0.0, _DENORM, -_DENORM, 1e-30, -1e-30, 0.25, 0.5, 1.0, np.nextafter(np.float32(1.0), np.float32(0.0)), -0.5,
                  -1.0, 1.5, 10.0, 1e6, -1e6, 1e30, -1e30, _FMAX, -_FMAX], np.float32)
NONFINITE_TIMES = np.array([np.inf, -np.inf, np.nan], np.float32)
# fuzzscene families as (family, seed, swap_ties)
FUZZ = [("ties", 0, False), ("ties", 0, True), ("ties", 3, True), ("many", 1, False), ("big", 0, False),
        ("caterpillar", 0, False), ("instanced", 0, False), ("instanced", 1, False), ("instanced", 2, False), ("probe", 0, False)]


def ray_sets(scene, camera, oracle, rng):
    """Camera rays through jittered raster positions, random rays in and around the scene, secondary rays from the
    camera rays' hit points, and rays that reach the ordered fallback."""
    cam = raysets.camera_rays(camera, N, rng)
    h, p = oracle.trace_rays(cam)
    return {"camera": cam, "random": raysets.random_rays(scene, N, rng), "secondary": raysets.secondary_rays(cam, h, p, rng),
            "fallback": raysets.fallback_rays(scene, rng)}


def fuzz_scene(family, seed, swap, path):
    """Writes the snapshot of one FUZZ entry to `path`, checking that caterpillar has its 30 BVH levels and big a mesh
    of more than 4096 triangles."""
    info = fuzzscene.make_mesh_scene(seed, path, family, swap_ties=swap, levels=30 if family == "caterpillar" else None)
    if family == "caterpillar":
        assert info["levels"] == 30
    if family == "big":
        assert max(info["tris"]) > 4096


def bvh_build_scene():
    """A floor, a sphere and an instance of a bumpy icosphere whose BVH tb200_bvh_build made, and a camera
    facing them: (scene, keepalive for the scene's arrays, camera, the generator the scene was drawn from)."""
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
    base.close()
    cam.position[:] = [0.0, 1.2, 6.0]
    cam.rotation[:] = [0.0, 0.0, 0.0, 1.0]
    return scene, (keep, nodes), cam, rng


def variant_path(name, tmp_path):
    """The snapshot of a variant test's scene: a snapshot's name, or fuzz_<family> for that family's seed-2 scene,
    written under tmp_path."""
    if not name.startswith("fuzz_"):
        return tb.scene_path(name)
    path = str(tmp_path / "s.tsnap")
    fuzzscene.make_mesh_scene(2, path, name[5:])
    return path


def variant_renderer(variant, snap, tmp_path):
    """A renderer of snap's scene made the variant's way: without the flat scene program (no_flat), from a scene cache
    file written under tmp_path (cached), or as a group of two renderers on device 0 (group)."""
    if variant == "no_flat":
        with schedenv.knobs(**schedenv.ROUTES["no-flat"]):
            return tb.Renderer(snap.scene)
    if variant == "cached":
        cache = str(tmp_path / "s.tcache")
        tb.scene_cache_save(snap.scene, cache)
        return tb.Renderer(None, cache=cache)
    with schedenv.knobs(TEST_DUP_DEVICES="1"):
        r = tb.Renderer(snap.scene, devices=[0, 0])
    assert r.num_devices() == 2
    return r
