"""The batched BSDF queries on the device (tb200_bsdf_eval / tb200_bsdf_sample, Renderer.bsdf_eval / bsdf_sample)
against the CPU restatement (oracle_bsdf_eval / oracle_bsdf_sample, batched by oracle_bsdf_cases), per query and bit
for bit; a NaN matches any NaN and nothing else is excused, not even the sign of a zero.  The materials are the
scene's own: a query names a primitive, and the restatement gets that primitive's tb200_material.

The inputs: hits of camera and random rays on every snapshot, with the light direction uniform on the sphere, along
the normal, mirrored and along -V, in both of PathTrace's eta conventions; test_bsdf_gpu's edge materials and
directions and test_bsdf_view_gpu's edges (dot(N, V) <= 0, L == -V, an underflowing |L + V|^2, NaN and infinite
components); etas outside the range where the renderer's skip flags are exact, with non-unit vectors, on materials
that carry those flags; primitives outside the scene; seeds at the edges of their range and the renderer's own."""
import ctypes as C

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import fuzzscene
import queryscenes
import raysets
import refdrv
import test_bsdf_gpu as bsdf
import test_bsdf_view_gpu as view

pytestmark = pytest.mark.gpu

F32 = np.float32
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1


def _torch():
    import torch
    return torch


# ---- scenes whose primitives carry given materials ----


def materials_of(scene):
    """The scene's tb200_material per primitive, as a MAT_DTYPE array."""
    n = scene.numPrimitives
    out = np.zeros(n, bsdf.MAT_DTYPE)
    for i in range(n):
        C.memmove(out[i:i + 1].ctypes.data, C.byref(scene.primitives[i].material), bsdf.MAT_DTYPE.itemsize)
    return out


def material_scene(mats):
    """A scene of one sphere per material of `mats` (MAT_DTYPE, at most 4095): primitive i carries mats[i].
    Returns (scene, keepalive)."""
    prims = (abi.Primitive * len(mats))()
    bounds = []
    for i in range(len(mats)):
        m = abi.Material()
        C.memmove(C.byref(m), mats[i:i + 1].ctypes.data, bsdf.MAT_DTYPE.itemsize)
        bounds.append(fuzzscene._sphere(prims[i], (3.0 * (i % 64), 3.0 * (i // 64), 0.0), 1.0, m))
    return fuzzscene.make_scene_struct(prims, fuzzscene._build_bvh(bounds), [])


# ---- running and comparing ----


def _queries(c):
    """The (N, 12) query records of CASE_DTYPE cases, c["mat"] being the primitive."""
    q = np.zeros((c.size, 12), F32)
    q[:, 0:3], q[:, 4:7], q[:, 8:11] = c["n"], c["v"], c["l"]
    q[:, 3] = c["mat"].astype(np.int32).view(F32)
    q[:, 7], q[:, 11] = c["etaI"], c["etaO"]
    return q


def device(r, c):
    """(eval (N, 4), sample (N, 8) with the type's bits in column 7) of the cases on renderer r."""
    torch = _torch()
    q = torch.from_numpy(_queries(c)).cuda(r.device)
    seeds = torch.from_numpy(np.ascontiguousarray(c["seed"]).astype(np.int32)).cuda(r.device)
    ev = r.bsdf_eval(q)
    l, pdf, f, t = r.bsdf_sample(q, seeds)
    s = torch.cat([l, pdf[:, None], f, t.view(torch.float32)[:, None]], 1)
    return ev.cpu().numpy(), s.cpu().numpy()


def expected(mats, c):
    """What the queries must return, from the restatement: (eval (N, 4), sample (N, 8)).  Cases whose primitive lies
    outside `mats` get zeros and type -1."""
    inside = (c["mat"] >= 0) & (c["mat"] < len(mats))
    ci = np.ascontiguousarray(c[inside])
    ref = bsdf._oracle(mats, ci)
    # f of the sampled direction: oracle_bsdf_eval at it, where its pdf > 0
    c2 = ci.copy()
    c2["l"] = ref["light"]
    at = bsdf._oracle(mats, c2)
    ev = np.zeros((c.size, 4), F32)
    s = np.zeros((c.size, 8), F32)
    s[:, 7] = np.int32(-1).view(F32)
    ev[inside, 0:3], ev[inside, 3] = ref["f"], ref["pdf"]
    fs = np.where((ref["spdf"] > 0)[:, None], at["f"], F32(0))
    s[inside, 0:3], s[inside, 3], s[inside, 4:7] = ref["light"], ref["spdf"], fs
    s[inside, 7] = ref["type"].astype(np.int32).view(F32)
    return ev, s


def mismatches(got, want):
    """Per query, whether any output differs: bits, except that a NaN matches any NaN."""
    return ~((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all(1)


def check(r, mats, c, what):
    ev, s = device(r, c)
    wev, ws = expected(mats, c)
    for name, got, want in (("eval", ev, wev), ("sample", s, ws)):
        bad = mismatches(got, want)
        if bad.any():
            k = int(np.argmax(bad))
            mat = mats[c["mat"][k]] if 0 <= c["mat"][k] < len(mats) else None
            raise AssertionError("%s, %s: %d of %d queries differ; first: case %s material %s device %s restatement %s" % (
                what, name, int(bad.sum()), c.size, c[k], mat, got[k], want[k]))
    return ev, s


# ---- the directions and etas of real hits ----


def hit_cases(r, scene, camera, mats, rng, n):
    """Cases from camera and random rays' hits on the device: prim, n, v = -dir, l in four kinds, both eta
    conventions, seeds of every kind.  Misses keep their prim -1."""
    torch = _torch()
    rays = np.concatenate([raysets.camera_rays(camera, n // 2, rng), raysets.random_rays(scene, n - n // 2, rng)])
    hits, prims = r.trace_rays(torch.from_numpy(rays).cuda(r.device))
    hits, prims = hits.cpu().numpy(), prims.cpu().numpy()
    c = np.zeros(n, bsdf.CASE_DTYPE)
    c["mat"] = prims
    N = hits[:, 1:4]
    V = -rays[:, 4:7]
    kind = rng.integers(0, 4, n)
    U = rng.normal(size=(n, 3))
    U = (U / np.linalg.norm(U, axis=1, keepdims=True)).astype(F32)
    mirror = (F32(2) * bsdf._dot(N, V))[:, None] * N - V
    L = np.choose(kind[:, None], [U, N, mirror, -V]).astype(F32)
    c["n"], c["v"], c["l"] = N, V, L
    ior = tb.material_ior(mats["eta"], mats["specular"])
    p = np.clip(prims, 0, len(mats) - 1)
    inside = rng.random(n) < 0.5
    c["etaI"] = np.where(inside, ior[p], F32(1))
    c["etaO"] = np.where(inside, F32(1), ior[p])
    c["seed"] = seeds(rng, n)
    return c


def seeds(rng, n):
    """int32 bits of uint32 seeds: 0, 0xffffffff, tb200_sample_seed of random pixels and frames, and random ones."""
    s = rng.integers(INT_MIN, INT_MAX + 1, n, dtype=np.int64)
    k = rng.integers(0, 4, n)
    s[k == 0] = 0
    s[k == 1] = -1
    idx = np.flatnonzero(k == 2)
    for i in idx:
        s[i] = int(tb.sample_seed(int(rng.integers(0, 1 << 20)), int(rng.integers(0, 1 << 12))))
    return (s & 0xffffffff).astype(np.uint32).view(np.int32)


@pytest.mark.parametrize("name", queryscenes.SNAPSHOTS)
def test_real_hits_match_restatement(name):
    snap = tb.Snapshot(tb.scene_path(name))
    scene = snap.scene.contents
    mats = materials_of(scene)
    r = tb.Renderer(snap.scene)
    rng = np.random.default_rng(sum(map(ord, name)))
    c = hit_cases(r, scene, snap.camera, mats, rng, 1 << 14)
    assert (c["mat"] >= 0).sum() > 1000, name
    check(r, mats, c, name)
    r.close()
    snap.close()


# ---- edge materials and edge directions ----


def _edge_cases(seed, count=4000):
    """test_bsdf_gpu's materials (the first `count`) and the cases that use them, with test_bsdf_view_gpu's edges."""
    mats, c, _ = bsdf.make_cases(seed)
    c, kind = view.with_edges(c, seed)
    mats = np.ascontiguousarray(mats[:count])
    c = np.ascontiguousarray(c[c["mat"] < count])
    return mats, c, kind


@pytest.mark.parametrize("seed", [20261016, 20261017])
def test_edge_materials_and_directions_match_restatement(seed):
    mats, c, _ = _edge_cases(seed)
    scene, keep = material_scene(mats)
    r = tb.Renderer(scene)
    assert c.size > 6000
    check(r, mats, c, "edge materials, seed %d" % seed)
    r.close()


@pytest.mark.parametrize("unsafe", [False, True])
def test_edge_scenes_match_restatement(unsafe, tmp_path):
    """test_bsdf_gpu's edge-material scenes (skips exact, and skips that would be NaN), with its case directions."""
    path = str(tmp_path / "edge.tsnap")
    bsdf.make_edge_scene(1, path, unsafe)
    snap = tb.Snapshot(path)
    mats = materials_of(snap.scene.contents)
    r = tb.Renderer(snap.scene)
    _, c, _ = bsdf.make_cases(7 + int(unsafe))
    c, _ = view.with_edges(c, 3)
    rng = np.random.default_rng(5)
    c["mat"] = rng.integers(0, len(mats), c.size)
    ior = tb.material_ior(mats["eta"], mats["specular"])
    inside = rng.random(c.size) < 0.5
    c["etaI"] = np.where(inside, ior[c["mat"]], F32(1))
    c["etaO"] = np.where(inside, F32(1), ior[c["mat"]])
    check(r, mats, c, "edge scene unsafe=%s" % unsafe)
    r.close()
    snap.close()


# ---- etas and vectors outside what a path produces ----

ODD_ETAS = np.array([0.0, -0.0, -1.0, 1.0 / 512, 300.0, 1e30, np.inf, -np.inf, np.nan, 1e-40, 1.0, 1.5], F32)


def odd_cases(rng, mats, n):
    c = np.zeros(n, bsdf.CASE_DTYPE)
    c["mat"] = rng.integers(0, len(mats), n)
    c["etaI"] = ODD_ETAS[rng.integers(0, ODD_ETAS.size, n)]
    c["etaO"] = ODD_ETAS[rng.integers(0, ODD_ETAS.size, n)]
    scale = np.array([1.0, 0.5, 3.0, 1e-3, 1e3], F32)
    for k in ("n", "v", "l"):
        d = rng.normal(size=(n, 3))
        d = d / np.linalg.norm(d, axis=1, keepdims=True) * scale[rng.integers(0, scale.size, n)][:, None]
        c[k] = d.astype(F32)
    # a share front-facing with unit vectors, where only the etas are odd
    unit = rng.random(n) < 0.3
    N = bsdf._unit(c["n"].astype(np.float64))
    V = bsdf._unit(c["v"].astype(np.float64))
    V[bsdf._dot(N, V) < 0] *= F32(-1)
    c["n"][unit], c["v"][unit] = N[unit], V[unit]
    c["seed"] = seeds(rng, n)
    return c


def flagged_materials(rng, n):
    """Materials with transmission 0 and clearcoat 0, on which the renderer sets TB_MAT_NO_FRESNEL and
    TB_MAT_NO_CLEARCOAT."""
    m = bsdf.edge_materials(rng, n)
    m["transmission"] = 0.0
    m["clearcoat"] = 0.0
    m["eta"] = rng.choice(np.array([0.0, 1.0, 1.5, 0.5], F32), n)
    m["specular"] = rng.random(n)
    m["clearcoatGloss"] = rng.random(n)
    m["subsurface"] = rng.choice(np.array([0.0, 0.5], F32), n)
    return m


def test_flags_are_set_on_these_materials():
    """The materials of the next test carry both skip flags in the renderer, so the test sees the skips if the kernel
    keeps them (no GPU needed)."""
    mats = flagged_materials(np.random.default_rng(8), 256)
    _, flags, _, _ = bsdf.make_materials(mats, len(mats))
    assert ((flags & bsdf.NO_FRESNEL) != 0).all() and ((flags & bsdf.NO_CLEARCOAT) != 0).all()


def test_etas_outside_the_renderer_range_match_restatement():
    """Where a skip flag's premise fails, the skipped term matters: Fr NaN or infinite from such etas makes the
    reference's pdf NaN, and a kernel that kept TB_MAT_NO_FRESNEL would return brdfPdf there."""
    rng = np.random.default_rng(8)
    mats = flagged_materials(rng, 256)
    scene, keep = material_scene(mats)
    r = tb.Renderer(scene)
    c = odd_cases(rng, mats, 1 << 15)
    ev, _ = check(r, mats, c, "odd etas")
    # the NaN pdfs that the skip would have hidden are there, on front-facing views
    front = bsdf._dot(c["n"], c["v"]) > 0
    above = bsdf._dot(c["n"], c["l"]) > 0
    assert (np.isnan(ev[:, 3]) & front & above).sum() > 100
    r.close()


# ---- primitives outside the scene ----


def test_prims_outside_the_scene_give_zeros():
    snap = tb.Snapshot(tb.scene_path("cornell"))
    mats = materials_of(snap.scene.contents)
    r = tb.Renderer(snap.scene)
    rng = np.random.default_rng(2)
    c = hit_cases(r, snap.scene.contents, snap.camera, mats, rng, 4096)
    c["mat"] = np.array([-1, len(mats), INT_MIN, INT_MAX, 0, len(mats) - 1], np.int32)[np.arange(c.size) % 6]
    ev, s = check(r, mats, c, "prims outside")
    out = c["mat"] < 0
    out |= c["mat"] >= len(mats)
    assert (ev[out].view(np.uint32) == 0).all()
    assert (s[out][:, :7].view(np.uint32) == 0).all() and (s[out][:, 7].view(np.int32) == -1).all()
    r.close()
    snap.close()


# ---- the reference's own code ----


@pytest.mark.skipif(not refdrv.have_ref("detmath"), reason="oracle/_ref is not built")
def test_reference_code_agrees():
    mats, c, _ = _edge_cases(20261018)
    scene, keep = material_scene(mats)
    r = tb.Renderer(scene)
    ev, s = device(r, c)
    idx, ref = bsdf._reference(mats, c, 8)
    assert not mismatches(ev[idx], np.concatenate([ref["f"], ref["pdf"][:, None]], 1)).any()
    got = np.concatenate([s[idx, 0:4], s[idx, 7:8].view(np.int32).astype(np.int32).view(F32)], 1)
    want = np.concatenate([ref["light"], ref["spdf"][:, None], ref["type"].astype(np.int32).view(F32)[:, None]], 1)
    assert not mismatches(got, want).any()
    r.close()


# ---- variants, counts, streams, side effects, refusals ----


@pytest.mark.parametrize("variant", ["cached", "group"])
def test_variants_give_the_restatement_bits(variant, tmp_path):
    snap = tb.Snapshot(tb.scene_path("veach"))
    mats = materials_of(snap.scene.contents)
    plain = tb.Renderer(snap.scene)
    c = hit_cases(plain, snap.scene.contents, snap.camera, mats, np.random.default_rng(4), 8192)
    plain.close()
    r = queryscenes.variant_renderer(variant, snap, tmp_path)
    check(r, mats, c, variant)
    r.close()
    snap.close()


@pytest.mark.parametrize("count", [0, 1, 31, 33, 10 ** 6 + 7])
def test_query_counts(count):
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("cornell"))
    mats = materials_of(snap.scene.contents)
    r = tb.Renderer(snap.scene)
    base = hit_cases(r, snap.scene.contents, snap.camera, mats, np.random.default_rng(6), 4096)
    c = np.resize(base, count)
    if count <= 4096:
        ev, s = check(r, mats, c, "count %d" % count)
    else:
        # the restatement checks the 4096 distinct queries; the big batch must repeat their answers
        wev, ws = check(r, mats, base, "count %d, distinct queries" % count)
        ev, s = device(r, c)
        k = np.arange(count) % base.size
        assert not mismatches(ev, wev[k]).any() and not mismatches(s, ws[k]).any()
    assert ev.shape == (count, 4) and s.shape == (count, 8)
    launches = r.stats().kernelLaunches
    q = torch.zeros((count, 12), dtype=torch.float32, device="cuda")
    l, pdf, f, t = r.bsdf_sample(q, torch.zeros((count,), dtype=torch.int32, device="cuda"))
    assert l.shape == (count, 3) and pdf.shape == (count,) and f.shape == (count, 3) and t.dtype == torch.int32
    assert r.stats().kernelLaunches == launches + (count > 0)
    r.close()
    snap.close()


def test_queries_written_on_the_callers_stream():
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("meshlight"))
    mats = materials_of(snap.scene.contents)
    r = tb.Renderer(snap.scene)
    c = hit_cases(r, snap.scene.contents, snap.camera, mats, np.random.default_rng(9), 1 << 14)
    wev, ws = expected(mats, c)
    src = torch.from_numpy(_queries(c)).cuda()
    sd = torch.from_numpy(np.ascontiguousarray(c["seed"])).cuda()
    dst, dseeds = torch.zeros_like(src), torch.zeros_like(sd)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    r.set_stream(s.cuda_stream)
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)   # the copies below land well after the calls have been queued
        dst.copy_(src)
        dseeds.copy_(sd)
        ev = r.bsdf_eval(dst)
        l, pdf, f, t = r.bsdf_sample(dst, dseeds)
        smp = torch.cat([l, pdf[:, None], f, t.view(torch.float32)[:, None]], 1)
    s.synchronize()
    assert not mismatches(ev.cpu().numpy(), wev).any()
    assert not mismatches(smp.cpu().numpy(), ws).any()
    r.set_stream(None)
    r.close()
    snap.close()


def test_queries_have_no_side_effects():
    snap = tb.Snapshot(tb.scene_path("cornell"))
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = 64, 48
    mats = materials_of(snap.scene.contents)
    fresh = tb.Renderer(snap.scene)   # before tb200_init
    c = hit_cases(fresh, snap.scene.contents, cam, mats, np.random.default_rng(11), 4096)
    check(fresh, mats, c, "before Init")
    fresh.close()

    r = tb.Renderer(snap.scene)
    r.Init(64, 48)
    out = np.zeros((48, 64, 4), np.float32)
    r.Render(cam, opt, out)
    rad0, _ = r.trace_frame(cam, opt, 0)
    acc0, st0, kernel0 = r.read_accumulator(), r.stats(), r.last_kernel()
    torch = _torch()
    q = torch.from_numpy(_queries(c)).cuda()
    r.bsdf_eval(q)
    st1 = r.stats()
    assert st1.kernelLaunches == st0.kernelLaunches + 1 and st1.gpuMs > 0.0
    r.bsdf_sample(q, torch.from_numpy(np.ascontiguousarray(c["seed"])).cuda())
    st2 = r.stats()
    assert st2.kernelLaunches == st0.kernelLaunches + 2 and st2.gpuMs > 0.0
    assert (st2.frames, st2.samples) == (st0.frames, st0.samples)
    assert r.last_kernel() == kernel0
    assert (r.read_accumulator().view(np.uint32) == acc0.view(np.uint32)).all()
    rad1, _ = r.trace_frame(cam, opt, 0)
    assert (rad0.view(np.uint32) == rad1.view(np.uint32)).all()
    # the frame counter did not move: the next Render adds the same frame a fresh renderer adds second
    r.Render(cam, opt, out)
    other = tb.Renderer(snap.scene)
    other.Init(64, 48)
    out2 = np.zeros((48, 64, 4), np.float32)
    other.Render(cam, opt, out2)
    other.Render(cam, opt, out2)
    rel = np.linalg.norm((out - out2).astype(np.float64)) / np.linalg.norm(out2.astype(np.float64))
    assert rel < 1e-5, rel
    other.close()
    r.close()
    snap.close()


def test_bad_arguments_are_refused_before_any_launch():
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path("cornell"))
    r = tb.Renderer(snap.scene)
    lib = r.lib
    n = 64
    q = torch.zeros((n, 12), dtype=torch.float32, device="cuda")
    sd = torch.zeros((n,), dtype=torch.int32, device="cuda")
    ev = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    sm = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    host = np.zeros((n, 12), np.float32)
    launches = r.stats().kernelLaunches

    def refused(entry, args, count, words):
        assert getattr(lib, entry)(r.h, *args, count) != 0
        msg = tb.last_error()
        assert msg.startswith(entry + ":") and any(w in msg for w in words), msg

    for entry, args in (("tb200_bsdf_eval", [q.data_ptr(), ev.data_ptr()]),
                        ("tb200_bsdf_sample", [q.data_ptr(), sd.data_ptr(), sm.data_ptr()])):
        for k in range(len(args)):
            bad = list(args)
            bad[k] = None
            refused(entry, bad, n, ["null"])
            bad[k] = host.ctypes.data
            refused(entry, bad, n, ["not device memory"])
            bad[k] = args[k] + (2 if k == 1 and entry == "tb200_bsdf_sample" else 4)
            refused(entry, bad, n - 1, ["aligned"])
        refused(entry, args, -1, ["out of range"])
        assert getattr(lib, entry)(r.h, *[None] * len(args), 0) == 0   # nothing to do: nothing launched
    assert lib.tb200_bsdf_eval(None, q.data_ptr(), ev.data_ptr(), n) != 0 and "null renderer" in tb.last_error()
    # a tensor that owns its whole segment: the caching allocator gives a fresh 24 MiB tensor a segment of its own
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    big_n = (24 << 20) // 48
    big = torch.zeros((big_n, 12), dtype=torch.float32, device="cuda")
    big_ev = torch.empty((big_n + 1, 4), dtype=torch.float32, device="cuda")
    big_sd = torch.zeros((big_n + 1,), dtype=torch.int32, device="cuda")
    big_sm = torch.empty((big_n + 1, 8), dtype=torch.float32, device="cuda")
    refused("tb200_bsdf_eval", [big.data_ptr(), big_ev.data_ptr()], big_n + 1, ["past the end"])
    refused("tb200_bsdf_sample", [big.data_ptr(), big_sd.data_ptr(), big_sm.data_ptr()], big_n + 1, ["past the end"])
    assert r.stats().kernelLaunches == launches
    assert lib.tb200_bsdf_eval(r.h, big.data_ptr(), big_ev.data_ptr(), big_n) == 0
    assert r.stats().kernelLaunches == launches + 1
    # the Python interface checks shapes, dtypes, contiguity and the device itself
    with pytest.raises(TypeError):
        r.bsdf_eval(q.double())
    with pytest.raises(ValueError):
        r.bsdf_eval(q[:, :8].contiguous())
    with pytest.raises(ValueError):
        r.bsdf_eval(torch.zeros((12, n), dtype=torch.float32, device="cuda").t())
    with pytest.raises(ValueError):
        r.bsdf_eval(q.cpu())
    with pytest.raises(TypeError):
        r.bsdf_sample(q, sd.long())
    with pytest.raises(ValueError):
        r.bsdf_sample(q, sd[:n - 1])
    with pytest.raises(TypeError):
        r.bsdf_sample(q, None)
    with pytest.raises(ValueError):
        r.bsdf_sample(q, sd, out=torch.empty((n, 4), dtype=torch.float32, device="cuda"))
    r.close()
    snap.close()
