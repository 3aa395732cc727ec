"""Fuzz parity over random scenes (tests/fuzzscene.py): the whole Disney parameter space, moving and
scaled spheres, sphere lights with 1-2 samples, gradient skies.  CPU: the restatement against the
reference's own compiled PathTrace, per sample, bit for bit.  GPU: the CUDA path against the same."""
import ctypes as C
import os

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import refdrv
import fuzzscene
import schedenv

SEEDS = list(range(12))            # GPU part
CPU_SEEDS = list(range(48))        # restatement vs the reference's compiled code


def _same(a, b):
    return bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


@pytest.mark.skipif(not refdrv.have_ref("detmath"), reason="oracle/_ref not built")
@pytest.mark.parametrize("seed", CPU_SEEDS)
def test_port_matches_reference_on_random_scenes(seed, tmp_path):
    path = str(tmp_path / "fuzz.tsnap")
    what = fuzzscene.make_scene(seed, path)
    ref = refdrv.RefScene.from_snapshot(path, "detmath")
    port = refdrv.PortScene.from_snapshot(path)
    for frame in (0, 3):
        a, ar = ref.trace_frame(frame, 4)
        b, br = port.trace_frame(frame, 4)
        assert np.array_equal(ar, br), what
        assert _same(a, b), what
    assert float(np.nan_to_num(a).sum()) > 0.0, what      # the scene is lit
    ref.close()
    port.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_gpu_matches_oracle_on_random_scenes(seed, tmp_path):
    os.environ.pop("TINSEL_B200_PIPELINE", None)
    path = str(tmp_path / "fuzz.tsnap")
    what = fuzzscene.make_scene(seed, path, width=96, height=64)
    port = refdrv.PortScene.from_snapshot(path)
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    r = tb.Renderer(snap.scene)
    r.Init(opt.width, opt.height)
    for frame in (0, 3):
        rad, ras = r.trace_frame(cam, opt, frame)
        prad, pras = port.trace_frame(frame, 8)
        assert np.array_equal(ras, pras), what
        bad = int((~((rad.view(np.uint32) == prad.view(np.uint32)) | (np.isnan(rad) & np.isnan(prad))).all(-1)).sum())
        assert bad == 0, "%s: %d of %d samples differ" % (what, bad, rad.shape[0] * rad.shape[1])
    r.close()
    port.close()
    snap.close()


# ---- triangle meshes (fuzzscene.make_mesh_scene) ------------------------------------------------------

MESH_CASES = ([("instanced", s) for s in range(8)] + [("ties", s) for s in range(5)] + [("many", s) for s in range(6)] +
              [("big", s) for s in range(4)] + [("probe", s) for s in range(6)] + [("caterpillar", s) for s in range(3)])
MATRIX_CASES = [("instanced", 1), ("ties", 0), ("many", 1), ("big", 0), ("probe", 1), ("caterpillar", 0)]
CPU_MESH_CASES = [(f, s) for f in fuzzscene.FAMILIES for s in range(4)]
LIMIT = 31    # TB200_MAX_BVH_LEVELS


def _bad_samples(rad, ras, prad, pras):
    assert np.array_equal(ras, pras)
    return int((~((rad.view(np.uint32) == prad.view(np.uint32)) | (np.isnan(rad) & np.isnan(prad))).all(-1)).sum())


def _gpu_vs_port(path, pipelines=("mega", "wavefront"), frames=(0, 3)):
    port = refdrv.PortScene.from_snapshot(path)
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    bad = {}
    try:
        for pipeline in pipelines:
            if pipeline:
                os.environ["TINSEL_B200_PIPELINE"] = pipeline
            r = tb.Renderer(snap.scene)
            r.Init(opt.width, opt.height)
            for frame in frames:
                rad, ras = r.trace_frame(cam, opt, frame)
                prad, pras = port.trace_frame(frame, 8)
                n = _bad_samples(rad, ras, prad, pras)
                if n:
                    bad[(pipeline, frame)] = n
            r.close()
    finally:
        os.environ.pop("TINSEL_B200_PIPELINE", None)
    return bad, port, snap


@pytest.mark.gpu
@pytest.mark.parametrize("family,seed", MESH_CASES)
def test_gpu_matches_port_on_mesh_scenes(family, seed, tmp_path):
    """Per sample and bit for bit in both pipelines, then the 4-spp image (rel-L2 <= 1e-4: the framebuffer
    sums run in another order) and the normals image bit for bit."""
    path = str(tmp_path / "mesh.tsnap")
    what = fuzzscene.make_mesh_scene(seed, path, family, width=96, height=64)
    bad, port, snap = _gpu_vs_port(path)
    assert not bad, "%s: samples differ %s" % (what, bad)
    cam, opt = snap.camera, snap.options
    r = tb.Renderer(snap.scene)
    r.Init(opt.width, opt.height)
    out = np.zeros((opt.height, opt.width, 4), np.float32)
    for _ in range(4):
        r.Render(cam, opt, out)
    expect = port.render_seeded(0, 4, nthreads=8)
    # a probe with black rows gives NaN samples (its sampling tables divide by a zero row sum, as the
    # reference's BuildCDF does): they must land on the same pixels, the rest agrees to rel-L2 <= 1e-4
    nan = np.isnan(out).any(-1)
    assert np.array_equal(nan, np.isnan(expect).any(-1)), what
    rel = np.linalg.norm((out[~nan] - expect[~nan]).astype(np.float64)) / np.linalg.norm(expect[~nan].astype(np.float64))
    assert rel <= 1e-4, "%s: rel L2 %g" % (what, rel)
    opt.mode = abi.MODE_NORMALS
    port.set_mode(abi.MODE_NORMALS)
    r.Init(opt.width, opt.height)
    out = np.zeros_like(out)
    r.Render(cam, opt, out)
    expect = port.render_normals()
    assert np.array_equal(out.view(np.uint32), expect.view(np.uint32)), "%s: %d normals differ" % (what, int((out != expect).any(-1).sum()))
    r.close()
    port.close()
    snap.close()


@pytest.mark.gpu
@pytest.mark.parametrize("sched,cta,no_flat", [(s, c, False) for s in schedenv.SCHEDS for c in schedenv.CTAS] + [("free", "768", True)])
def test_mesh_scenes_under_every_scheduler_variant(sched, cta, no_flat, tmp_path):
    with schedenv.sched_env(sched, cta, no_flat=no_flat):
        for family, seed in MATRIX_CASES:
            path = str(tmp_path / ("%s%d.tsnap" % (family, seed)))
            what = fuzzscene.make_mesh_scene(seed, path, family, width=96, height=64)
            bad, port, snap = _gpu_vs_port(path, pipelines=("wavefront",), frames=(3, 4))
            assert not bad, "%s: samples differ %s" % (what, bad)
            port.close()
            snap.close()


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [LIMIT - 1, LIMIT])
def test_deepest_accepted_bvh_is_bit_exact(levels, tmp_path):
    """A caterpillar BVH fills the traversal stack to levels + 1 entries: at the bound (31 interior levels,
    32 entries) the inline walk, the megakernel and the offloaded walker CTAs still match the port."""
    path = str(tmp_path / "deep.tsnap")
    what = fuzzscene.make_mesh_scene(0, path, "caterpillar", width=96, height=64, levels=levels)
    assert what["levels"] == levels
    bad, port, snap = _gpu_vs_port(path)
    assert not bad, "%s: samples differ %s" % (what, bad)
    port.close()
    snap.close()
    with schedenv.sched_env("offload", "512"):
        bad, port, snap = _gpu_vs_port(path, pipelines=("wavefront",))
        assert not bad, "%s offload: samples differ %s" % (what, bad)
        port.close()
        snap.close()


@pytest.mark.skipif(not refdrv.have_ref("detmath"), reason="oracle/_ref not built")
@pytest.mark.parametrize("family,seed", CPU_MESH_CASES)
def test_port_matches_reference_on_mesh_scenes(family, seed, tmp_path):
    path = str(tmp_path / "mesh.tsnap")
    what = fuzzscene.make_mesh_scene(seed, path, family)
    ref = refdrv.RefScene.from_snapshot(path, "detmath")
    port = refdrv.PortScene.from_snapshot(path)
    for frame in (0, 3):
        a, ar = ref.trace_frame(frame, 4)
        b, br = port.trace_frame(frame, 4)
        assert np.array_equal(ar, br), what
        assert _same(a, b), what
    ref.close()
    port.close()


def test_mesh_generator_makes_what_it_claims(tmp_path):
    """Each family holds what it is there to test, the scenes pass validation, and the port renders them lit."""
    seen = {f: [] for f in fuzzscene.FAMILIES}
    for family, seed in MESH_CASES + CPU_MESH_CASES:
        path = str(tmp_path / "m.tsnap")
        info = fuzzscene.make_mesh_scene(seed, path, family)
        seen[family].append(info)
        snap = tb.Snapshot(path)
        sc = snap.scene.contents
        assert sc.numMeshes == info["meshes"] >= 1 and sc.numPrimitives == info["prims"], info
        assert bool(sc.sky.probeValid) == (family == "probe"), info
        tb.scene_cache_save(snap.scene, str(tmp_path / "m.tcache"))      # validate_scene accepts it
        port = refdrv.PortScene.from_snapshot(path)
        rad, _ = port.trace_frame(0, 4)
        assert float(np.nan_to_num(rad).sum()) > 0.0, info
        port.close()
        snap.close()
    inst = seen["instanced"] + seen["probe"]
    assert all(1 <= i["meshes"] <= 4 for i in inst)
    assert all(i["zero_area"] > 0 for f in ("ties", "many", "big") for i in seen[f])
    assert any(i["moving_scale"] > 0 and i["mesh_lights"] > 0 and i["zero_area"] > 0 for i in inst)
    assert all(17 <= i["prims"] <= 40 for i in seen["many"])
    assert all(i["prims"] <= 16 for f in ("instanced", "ties", "big", "probe", "caterpillar") for i in seen[f])
    assert all(max(i["tris"]) > 4096 for i in seen["big"])
    assert all(i["levels"] == LIMIT - 1 for i in seen["caterpillar"])


@pytest.mark.parametrize("seed", range(5))
def test_exact_ties_decide_the_result(seed, tmp_path):
    """The port's samples change when the materials of the exact duplicates are swapped: the tie-break
    (first found along the reference's visit order wins) decides what the GPU tests compare."""
    a, b = str(tmp_path / "a.tsnap"), str(tmp_path / "b.tsnap")
    fuzzscene.make_mesh_scene(seed, a, "ties")
    fuzzscene.make_mesh_scene(seed, b, "ties", swap_ties=True)
    pa, pb = refdrv.PortScene.from_snapshot(a), refdrv.PortScene.from_snapshot(b)
    ra, _ = pa.trace_frame(0, 4)
    rb, _ = pb.trace_frame(0, 4)
    assert not _same(ra, rb)
    pa.close()
    pb.close()


# ---- BVHs the traversal stack cannot hold are refused ----------------------------------------------

def _refusals(scene_ptr, tmp_path):
    """(tb200_create's error, tb200_scene_cache_save's error); None where the call did not reject the scene."""
    lib = tb.load_library()
    h = lib.tb200_create(scene_ptr, 0)
    if h:
        lib.tb200_destroy(h)
    create = tb.last_error()
    create = create if "invalid scene" in create else None
    rc = lib.tb200_scene_cache_save(scene_ptr, str(tmp_path / "x.tcache").encode())
    save = tb.last_error() if rc != 0 else None
    return create, save


def _caterpillar(tmp_path, levels):
    path = str(tmp_path / ("cat%d.tsnap" % levels))
    fuzzscene.make_mesh_scene(0, path, "caterpillar", levels=levels)
    return path


def _scene_with_mesh_nodes(snap, mutate):
    base = snap.scene.contents
    sc = abi.copy_struct(base)
    meshes = (abi.Mesh * base.numMeshes)()
    C.memmove(meshes, base.meshes, C.sizeof(meshes))
    nodes = (abi.BvhNode * meshes[0].numNodes)()
    C.memmove(nodes, meshes[0].nodes, C.sizeof(nodes))
    mutate(nodes)
    meshes[0].nodes = C.cast(nodes, C.POINTER(abi.BvhNode))
    sc.meshes = C.cast(meshes, C.POINTER(abi.Mesh))
    return sc, (meshes, nodes)


def test_bvh_depth_bound_is_tight(tmp_path):
    """31 interior levels are accepted everywhere; 32 are refused by tb200_create, tb200_scene_cache_save
    and the port, for a mesh BVH and for the scene BVH."""
    ok = tb.Snapshot(_caterpillar(tmp_path, LIMIT))
    create, save = _refusals(ok.scene, tmp_path)
    assert create is None and save is None, (create, save)
    refdrv.PortScene.from_snapshot(_caterpillar(tmp_path, LIMIT)).close()
    deep = tb.Snapshot(_caterpillar(tmp_path, LIMIT + 1))
    for err in _refusals(deep.scene, tmp_path):
        assert err and "invalid scene" in err and "mesh 0" in err and "32 levels" in err, err
    with pytest.raises(RuntimeError, match="refused"):
        refdrv.PortScene.from_snapshot(_caterpillar(tmp_path, LIMIT + 1))
    ok.close()
    deep.close()
    # scene level: a chain of spheres along the view axis, nearer ones deeper
    for levels in (LIMIT, LIMIT + 1):
        n = levels + 1
        prims = (abi.Primitive * n)()
        bounds = [fuzzscene._sphere(prims[k], (0.0, 1.0, -1.0 - 0.1 * (n - k)), 0.04, abi.Material.default()) for k in range(n)]
        tree = fuzzscene._chain_bvh(bounds)
        assert fuzzscene.tree_levels(tree) == levels
        sc, keep = fuzzscene.make_scene_struct(prims, tree, [])
        create, save = _refusals(C.pointer(sc), tmp_path)
        if levels == LIMIT:
            assert create is None and save is None, (create, save)
        else:
            for err in (create, save):
                assert err and "scene: BVH has 32 levels" in err, err
        port = refdrv.load_port().oracle_create(C.pointer(sc))
        assert bool(port) == (levels == LIMIT)
        if port:
            refdrv.load_port().oracle_destroy(port)


def test_bvh_that_is_not_a_tree_is_refused(tmp_path):
    snap = tb.Snapshot(_caterpillar(tmp_path, 4))

    def shared(nodes):      # node 2 (interior) also points at node 1, node 0's leaf
        nodes[2].right_leaf = 1

    def cycle(nodes):       # the deepest interior node points back at the root
        last = max(i for i in range(len(nodes)) if not nodes[i].right_leaf >> 31)
        nodes[last].left = 0

    for mutate in (shared, cycle):
        sc, keep = _scene_with_mesh_nodes(snap, mutate)
        for err in _refusals(C.pointer(sc), tmp_path):
            assert err and "invalid scene" in err and "reached twice" in err, (mutate.__name__, err)
        assert not refdrv.load_port().oracle_create(C.pointer(sc)), mutate.__name__
    snap.close()


def _mesh_pairs_offsets(data):
    """Byte offsets in a scene cache file (api.cu image_save) of mesh 0's pair count and of its stored depth."""
    u64 = lambda o: int.from_bytes(data[o:o + 8], "little")
    u32 = lambda o: int.from_bytes(data[o:o + 4], "little")
    size_prim, size_pair, size_op = u32(12), u32(16), u32(20)
    o = 24
    o += 8 + u64(o) * size_prim          # prims
    o += 8 + u64(o) * size_pair          # scene pairs
    o += 4                               # scene root
    o += 8 + u64(o) * size_op            # flat program
    o += 8                               # mesh count
    pairs = o
    o += 8 + u64(o) * size_pair
    o += 8 + u64(o) * 16                 # verts
    o += 8 + u64(o) * 16                 # normals
    o += 8 + u64(o) * 4                  # cdf
    return pairs, o + 8                  # numTris, rootRef, depth


def test_cache_file_with_too_deep_a_mesh_bvh_is_refused(tmp_path):
    """tb200_create_cached checks the pair records it loads: a stored depth over the bound, and a tree that is
    deeper than its stored depth says, are both refused before anything reaches the device."""
    path = _caterpillar(tmp_path, LIMIT)
    snap = tb.Snapshot(path)
    # one spare triangle that the tree does not reference, to hang a 32nd level on in the cache file
    base = snap.scene.contents
    sc = abi.copy_struct(base)
    g = base.meshes[0]
    pos = np.ctypeslib.as_array(g.positions, shape=(g.numVertices * 3,)).copy()
    nrm = np.ctypeslib.as_array(g.normals, shape=(g.numVertices * 3,)).copy()
    pos = np.concatenate([pos, pos[-9:]])
    nrm = np.concatenate([nrm, nrm[-9:]])
    idx = np.arange(g.numIndices + 3, dtype=np.int32)
    cdf = np.concatenate([np.ctypeslib.as_array(g.cdf, shape=(g.numIndices // 3,)), [1.0]]).astype(np.float32)
    meshes = (abi.Mesh * 1)()
    meshes[0] = g
    meshes[0].positions, meshes[0].normals = pos.ctypes.data_as(abi.c_float_p), nrm.ctypes.data_as(abi.c_float_p)
    meshes[0].indices, meshes[0].cdf = idx.ctypes.data_as(abi.c_int_p), cdf.ctypes.data_as(abi.c_float_p)
    meshes[0].numVertices, meshes[0].numIndices = g.numVertices + 3, g.numIndices + 3
    sc.meshes = C.cast(meshes, C.POINTER(abi.Mesh))
    good = str(tmp_path / "good.tcache")
    tb.scene_cache_save(C.pointer(sc), good)
    data = bytearray(open(good, "rb").read())
    pairs_at, depth_at = _mesh_pairs_offsets(data)
    assert int.from_bytes(data[depth_at:depth_at + 4], "little", signed=True) == LIMIT
    lib = tb.load_library()

    def attempt(blob):
        p = str(tmp_path / "bad.tcache")
        open(p, "wb").write(bytes(blob))
        h = lib.tb200_create_cached(p.encode(), 0)
        if h:
            lib.tb200_destroy(h)
        return tb.last_error()

    err = attempt(data)
    assert "invalid cache file" not in err, err
    stored = bytearray(data)
    stored[depth_at:depth_at + 4] = (LIMIT + 1).to_bytes(4, "little")
    err = attempt(stored)
    assert "invalid cache file" in err and "stored BVH depth 32" in err, err
    # a 32nd pair below the deepest one, the depth field left at 31
    n = int.from_bytes(data[pairs_at:pairs_at + 8], "little")
    recs = np.frombuffer(bytes(data[pairs_at + 8:pairs_at + 8 + 64 * n]), np.uint32).reshape(n, 16).copy()
    leaf = 0x80000000
    deepest = [k for k in range(n) if recs[k, 12] & leaf and recs[k, 13] & leaf]
    assert len(deepest) == 1
    k = deepest[0]
    slot = 12 if recs[k, 12] == leaf | LIMIT else 13
    assert recs[k, slot] == leaf | LIMIT
    extra = recs[k].copy()
    extra[12], extra[13] = leaf | LIMIT, leaf | (LIMIT + 1)
    recs[k, slot] = n
    deep = data[:pairs_at] + (n + 1).to_bytes(8, "little") + recs.tobytes() + extra.tobytes() + data[pairs_at + 8 + 64 * n:]
    err = attempt(deep)
    assert "invalid cache file" in err and "32 levels" in err, err
    snap.close()
