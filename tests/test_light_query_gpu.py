"""The light queries on the device (tb200_sample_lights / tb200_sky_eval, Renderer.sample_lights / sky) against the CPU
restatement: SampleLights per record (tests/light_oracle.cpp: oracle_sample_lights) and Sky::Eval / ProbePdf per
direction (oracle_sky_eval), bit for bit, a NaN matching any NaN.  Then a PathTrace built in torch from the queries,
against the restatement's PathTrace with the same per-call seeds (oracle_path_trace_reseeded); and the contract the
queries share with the others: batch order and size, streams, calls before Init, scene-cache and group renderers, side
effects and refusals."""
import ctypes as C

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import lightoracle
import queryscenes

pytestmark = pytest.mark.gpu

F32 = np.float32
RAY_EPS = F32(0.0001)   # kRayEpsilon, render.cpp:11


def _torch():
    import torch
    return torch


def _same(got, want):
    """Per row, whether every value matches: bits, except that a NaN matches any NaN."""
    return ((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all(1)


def _iors(scene):
    """material_ior of every primitive's material: the etaO of a path entering it."""
    n = scene.numPrimitives
    eta = np.array([scene.primitives[i].material.eta for i in range(n)], F32)
    spec = np.array([scene.primitives[i].material.specular for i in range(n)], F32)
    return tb.material_ior(eta, spec).reshape(n)


def _seeds(rng, n):
    return rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(np.int32)


def check_nee(r, scene_ptr, q, seeds, what):
    """Runs the NEE query on (N, 16) records q and int32 seeds (torch tensors on the head) and compares it with the
    restatement; returns the device's radiance as numpy."""
    got = r.sample_lights(q, seeds).cpu().numpy()
    want = lightoracle.sample_lights(scene_ptr, q.cpu().numpy(), seeds.cpu().numpy())
    bad = ~_same(got, want)
    if bad.any():
        k = int(np.argmax(bad))
        raise AssertionError("%s: %d of %d queries differ; first: record %s seed %d device %s restatement %s" % (
            what, int(bad.sum()), len(got), q[k].cpu().numpy(), int(seeds[k]), got[k], want[k]))
    return got


def _ff(n, l):
    """FaceForward(n, l) as the restatement's face_fwd: dot(l, n) < 0 ? -n : n, the dot summed left to right."""
    d = l[:, 0] * n[:, 0] + l[:, 1] * n[:, 1] + l[:, 2] * n[:, 2]
    return n.where((d >= 0)[:, None] | d.isnan()[:, None], -n)


def first_and_second_hits(r, snap, W, H, frames, rng):
    """The light queries PathTrace makes at the first and second hits of the image's own camera samples (frames
    0 .. frames-1 of a W x H image): (q1, q2) records, the second after bsdf_sample at the first, with inside-medium
    etas where the sampled direction transmits.  Misses keep prim -1."""
    torch = _torch()
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = W, H
    iors = torch.from_numpy(_iors(snap.scene.contents)).cuda()
    rays, _ = r.camera_rays(cam, opt, tb.frame_samples(W, H, 0, frames, device="cuda"))
    hits, prims = r.trace_rays(rays)
    o, d, t = rays[:, 0:3], rays[:, 4:7], rays[:, 3]
    p = o + d * hits[:, 0:1]
    n = hits[:, 1:4]
    eta_o = iors[prims.clamp(min=0).long()]
    q1 = tb.light_queries(prims, p, n, -d, 1.0, eta_o, t)
    seeds = torch.from_numpy(_seeds(rng, len(prims))).cuda()
    l, pdf, _, _ = r.bsdf_sample(tb.bsdf_queries(prims, n, -d, 1.0, eta_o), seeds)
    rays2 = torch.zeros_like(rays)
    rays2[:, 0:3] = p + _ff(n, l) * float(RAY_EPS)
    rays2[:, 3] = t
    rays2[:, 4:7] = l
    h2, p2 = r.trace_rays(rays2)
    p2 = torch.where((prims >= 0) & (pdf > 0), p2, torch.full_like(p2, -1))
    transmitted = (l[:, 0] * n[:, 0] + l[:, 1] * n[:, 1] + l[:, 2] * n[:, 2]) <= 0
    eta_o2 = iors[p2.clamp(min=0).long()]
    eta_i = torch.where(transmitted, eta_o, torch.ones_like(eta_o))
    eta_o2 = torch.where(transmitted, torch.ones_like(eta_o2), eta_o2)
    q2 = tb.light_queries(p2, rays2[:, 0:3] + l * h2[:, 0:1], h2[:, 1:4], -l, eta_i, eta_o2, t)
    return q1, q2


# ---- 1. real hits on every snapshot ----


@pytest.mark.parametrize("name", queryscenes.SNAPSHOTS)
def test_sample_lights_at_real_hits(name):
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path(name))
    r = tb.Renderer(snap.scene)
    rng = np.random.default_rng(11)
    q1, q2 = first_and_second_hits(r, snap, 64, 48, 2, rng)
    lit = False
    for k, q in enumerate((q1, q2)):
        seeds = torch.from_numpy(_seeds(rng, q.shape[0])).cuda()
        got = check_nee(r, snap.scene, q, seeds, "%s, bounce %d" % (name, k + 1))
        hit = q[:, 7].view(torch.int32).cpu().numpy() >= 0
        assert (got[~hit] == 0).all()
        lit = lit or bool((got != 0).any())
    scene = snap.scene.contents
    if _light_prims(scene) or scene.sky.probeValid:
        assert lit, "%s: no light reached any hit" % name
    r.close()
    snap.close()


# ---- 2. odd inputs ----


def _hit_records(name, n, rng):
    """(snap, renderer, q) for n first hits of `name`'s camera samples (misses dropped)."""
    snap = tb.Snapshot(tb.scene_path(name))
    r = tb.Renderer(snap.scene)
    q1, _ = first_and_second_hits(r, snap, 96, 64, 1, rng)
    q = q1[q1[:, 7].view(_torch().int32) >= 0][:n].contiguous()
    return snap, r, q


@pytest.mark.parametrize("name", ["veach", "cornell", "glass", "gloss", "envmini", "meshlight"])
def test_odd_etas_and_vectors(name):
    # etas outside any path's range and non-unit, zero, reversed or non-finite n and wo: the reference's full BSDF
    # arithmetic must run, so the renderer's Fresnel and clearcoat skips must not (they are exact only for a path's
    # own inputs)
    torch = _torch()
    rng = np.random.default_rng(12)
    snap, r, q = _hit_records(name, 6000, rng)
    m = q.shape[0]
    etas = torch.tensor([0.0, -1.0, 1e-30, 0.5, 1.0, 1.5, 3.0, 1e30, float("inf"), float("nan")])
    q[:, 11] = etas[torch.from_numpy(rng.integers(0, len(etas), m))].cuda()
    q[:, 12] = etas[torch.from_numpy(rng.integers(0, len(etas), m))].cuda()
    scale = torch.tensor([1.0, 0.0, -1.0, 0.25, 3.0, 1e-20, 1e20, float("inf")])
    q[:, 4:7] *= scale[torch.from_numpy(rng.integers(0, len(scale), m))].cuda()[:, None]
    q[:, 8:11] *= scale[torch.from_numpy(rng.integers(0, len(scale), m))].cuda()[:, None]
    check_nee(r, snap.scene, q, torch.from_numpy(_seeds(rng, m)).cuda(), "%s, odd etas and vectors" % name)
    r.close()
    snap.close()


def test_primitives_outside_the_scene_give_zeros():
    torch = _torch()
    rng = np.random.default_rng(13)
    snap, r, q = _hit_records("veach", 512, rng)
    np_ = snap.scene.contents.numPrimitives
    bad = torch.tensor([-1, -2, np_, np_ + 1, 2 ** 31 - 1, -2 ** 31], dtype=torch.int32)
    q[:, 7] = bad[torch.arange(q.shape[0]) % len(bad)].view(torch.float32).cuda()
    got = r.sample_lights(q, torch.zeros(q.shape[0], dtype=torch.int32, device="cuda"))
    assert (got.view(torch.int32) == 0).all()
    r.close()
    snap.close()


def _light_prims(scene):
    return [i for i in range(scene.numPrimitives) if scene.primitives[i].lightSamples > 0]


@pytest.mark.parametrize("name", ["veach", "emitter", "meshlight"])
def test_a_surface_that_is_a_light_and_points_inside_a_light(name):
    torch = _torch()
    rng = np.random.default_rng(14)
    snap, r, q = _hit_records(name, 4096, rng)
    scene = snap.scene.contents
    lights = _light_prims(scene)
    assert lights, name
    m = q.shape[0]
    # the surface primitive is a light: its material shades the connections, as PathTrace's call at a light hit does
    ql = q.clone()
    ql[:, 7] = torch.tensor(lights, dtype=torch.int32)[torch.arange(m) % len(lights)].view(torch.float32).cuda()
    check_nee(r, snap.scene, ql, torch.from_numpy(_seeds(rng, m)).cuda(), "%s, light surfaces" % name)
    # points at the centre of and just inside each sphere light, and on mesh lights' own instances
    centres = [list(scene.primitives[i].start.p) for i in lights]
    qc = q.clone()
    c = torch.tensor(centres, dtype=torch.float32)[torch.arange(m) % len(centres)].cuda()
    jitter = torch.from_numpy(rng.normal(size=(m, 3)).astype(F32) * 0.01).cuda()
    qc[:, 0:3] = c + jitter * (torch.arange(m, device="cuda") % 2)[:, None]
    check_nee(r, snap.scene, qc, torch.from_numpy(_seeds(rng, m)).cuda(), "%s, points inside lights" % name)
    r.close()
    snap.close()


def test_times_outside_the_shutter():
    torch = _torch()
    rng = np.random.default_rng(15)
    snap, r, q = _hit_records("motionblur", 4096, rng)
    m = q.shape[0]
    # finite times only: the renderer takes a static primitive's transform without interpolating, where the
    # reference's interpolation with a NaN or infinite time would give NaN (include/tinsel_b200.h)
    times = torch.tensor([-1.0, -0.0, 1.0, 1.5, 2.0, 10.0, -1e6, 1e6])
    q[:, 3] = times[torch.arange(m) % len(times)].cuda()
    check_nee(r, snap.scene, q, torch.from_numpy(_seeds(rng, m)).cuda(), "motionblur, times outside the shutter")
    r.close()
    snap.close()


# ---- 3. the sky ----


def _sky_directions(rng):
    u = rng.normal(size=(20000, 3))
    u = (u / np.linalg.norm(u, axis=1, keepdims=True)).astype(F32)
    eps = [0.0, 1e-5, -1e-5, 5e-5, 1e-4, 2e-4, 1e-7]
    poles = []
    for y in (1.0, -1.0):
        for e in eps:
            for x, z in ((e, 0.0), (0.0, e), (e, e), (-e, e)):
                poles.append((x, y, z))
                v = np.array([x, y, z], np.float64)
                poles.append(tuple(v / np.linalg.norm(v)))
    axis = [(0.0, y, 0.0) for y in (0.5, -0.5, 2.0, 0.0, -0.0, 1e-30)]
    odd = [(np.nan, 0.0, 1.0), (0.0, np.nan, 0.0), (1.0, 0.0, np.nan), (np.inf, 1.0, 0.0), (0.0, -np.inf, 0.0),
           (0.0, 0.0, 0.0), (-0.0, -0.0, -0.0)]
    # two infinite components: atan2f(+-inf, +-inf) is +-pi/4 or +-3pi/4 (C99 Annex F), not NaN
    odd += [(x, y, z) for x in (np.inf, -np.inf) for z in (np.inf, -np.inf) for y in (0.0, -0.0, 0.5, -1.0, np.inf)]
    return np.concatenate([u, u * F32(3.0), u * F32(1e-3), np.array(poles + axis + odd, F32)]).astype(F32)


@pytest.mark.parametrize("name", queryscenes.SNAPSHOTS)
def test_sky_matches_restatement(name):
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path(name))
    r = tb.Renderer(snap.scene)
    d = _sky_directions(np.random.default_rng(16))
    rays = np.zeros((len(d), 8), F32)
    rays[:, 4:7] = d
    rays[:, 0:4] = np.random.default_rng(17).normal(size=(len(d), 4))   # only dir is read
    got = r.sky(torch.from_numpy(rays).cuda()).cpu().numpy()
    want = lightoracle.sky_eval(snap.scene, d)
    bad = ~_same(got, want)
    assert not bad.any(), (name, int(bad.sum()), d[bad][:4], got[bad][:4], want[bad][:4])
    rgb, pdf = r.sky(torch.from_numpy(rays).cuda(), split=True)
    assert tuple(rgb.shape) == (len(d), 3) and tuple(pdf.shape) == (len(d),)
    sky = snap.scene.contents.sky
    if not sky.probeValid:
        assert (got[:, 3] == 0).all()
    else:
        assert (got[:, 3] > 0).any()
        # (inf, 0, inf) looks up u = (pi + pi/4) / (2 pi) = 0.625 and v = acos(0) / pi = 0.5
        k = int(np.flatnonzero((d[:, 0] == np.inf) & (d[:, 1] == 0) & (d[:, 2] == np.inf))[0])
        w, h = sky.probeWidth, sky.probeHeight
        texel = np.ctypeslib.as_array(sky.probeData, shape=(h * w * 4,)).reshape(h, w, 4)[int(0.5 * h), int(0.625 * w), :3]
        assert (got[k, :3].view(np.uint32) == texel.view(np.uint32)).all(), (name, got[k], texel)
    r.close()
    snap.close()


def test_both_kinds_of_sky_are_covered():
    kinds = set()
    for name in queryscenes.SNAPSHOTS:
        snap = tb.Snapshot(tb.scene_path(name))
        kinds.add(bool(snap.scene.contents.sky.probeValid))
        snap.close()
    assert kinds == {False, True}


# ---- 4. a PathTrace built from the queries ----


def torch_path_trace(r, snap, rays, seeds):
    """PathTrace (render.cpp:230-388) of every camera ray, in torch over the library's queries: trace_rays,
    sample_lights, bsdf_sample and sky, with primitive_areas and the materials for the emission MIS.  seeds: (N,
    maxDepth, 2) int32, bounce b's SampleLights and BSDFSample seeds.  Returns (radiance (N, 3), length (N,), prims
    (N, maxDepth)) as numpy, in oracle_path_trace_reseeded's conventions."""
    torch = _torch()
    scene = snap.scene.contents
    dev = rays.device
    n, depth = rays.shape[0], snap.options.maxDepth
    iors = torch.from_numpy(_iors(scene)).to(dev)
    mats = [scene.primitives[i].material for i in range(scene.numPrimitives)]
    emission = torch.tensor([list(m.emission) for m in mats], dtype=torch.float32, device=dev)
    absorption = torch.tensor([list(m.absorption) for m in mats], dtype=torch.float32, device=dev)
    light_samples = torch.tensor([scene.primitives[i].lightSamples for i in range(scene.numPrimitives)], device=dev)
    areas = torch.from_numpy(tb.primitive_areas(scene)).to(dev)
    probe = bool(scene.sky.probeValid)

    o, d, t = rays[:, 0:3].clone(), rays[:, 4:7].clone(), rays[:, 3].clone()
    T = torch.ones((n, 3), device=dev)
    L = torch.zeros((n, 3), device=dev)
    eta = torch.ones(n, device=dev)
    absorb = torch.zeros((n, 3), device=dev)
    ray_type = torch.full((n,), abi.BSDF_REFLECTED, dtype=torch.int32, device=dev)
    bsdf_pdf = torch.ones(n, device=dev)
    length = torch.zeros(n, dtype=torch.int32, device=dev)
    prims_out = torch.full((n, depth), -2, dtype=torch.int32, device=dev)
    alive = torch.arange(n, device=dev)
    for b in range(depth):
        if alive.numel() == 0:
            break
        ray = torch.zeros((alive.numel(), 8), device=dev)
        ray[:, 0:3], ray[:, 3], ray[:, 4:7] = o[alive], t[alive], d[alive]
        hits, prims = r.trace_rays(ray)
        length[alive] += 1
        prims_out[alive, b] = prims
        miss = prims < 0
        # the miss branch
        mi = alive[miss]
        if mi.numel():
            sky, sky_pdf = r.sky(ray[miss].contiguous(), split=True)
            w = torch.ones(mi.numel(), device=dev)
            if probe and b > 0:
                mis = 0.5 * bsdf_pdf[mi] / (0.5 * bsdf_pdf[mi] + 0.5 * sky_pdf)
                w = torch.where(ray_type[mi] != abi.BSDF_SPECULAR, mis, w)
            L[mi] = L[mi] + (sky * w[:, None]) * T[mi]
        # the hit branch
        hi, hp = alive[~miss], prims[~miss]
        if hi.numel() == 0:
            alive = hi
            break
        h = hits[~miss]
        ht = h[:, 0]
        air = eta[hi] == 1.0
        out_eta = torch.where(air, iors[hp.long()], torch.ones_like(ht))
        out_abs = torch.where(air[:, None], absorption[hp.long()], torch.zeros_like(T[hi]))
        T[hi] = T[hi] * torch.exp((-absorb[hi]) * ht[:, None])
        dd = d[hi]
        p = o[hi] + dd * ht[:, None]
        nn = h[:, 1:4]
        em = emission[hp.long()]
        if b == 0:
            L[hi] = L[hi] + em
        else:
            area = areas[hp.long()]
            lit = area > 0
            cosv = ((-dd)[:, 0] * nn[:, 0] + (-dd)[:, 1] * nn[:, 1] + (-dd)[:, 2] * nn[:, 2]).clamp(1e-3, 1.0)
            light_pdf = ((1.0 / area) * ht * ht) / cosv
            ls = light_samples[hp.long()]
            N = (ls.float() + 1.0).int().float()
            cb, cl = 1.0 / N, ls.float() / N
            w = cb * bsdf_pdf[hi] / (cb * bsdf_pdf[hi] + cl * light_pdf)
            w = torch.where(ray_type[hi] == abi.BSDF_SPECULAR, torch.ones_like(w), w)
            L[hi] = torch.where(lit[:, None], L[hi] + (T[hi] * w[:, None]) * em, L[hi])
        nee = r.sample_lights(tb.light_queries(hp, p, nn, -dd, eta[hi], out_eta, t[hi]), seeds[hi, b, 0].contiguous())
        L[hi] = L[hi] + T[hi] * nee
        ls_zero = light_samples[hp.long()] == 0   # PathTrace stops at a light after its NEE
        l, pdf, f, typ = r.bsdf_sample(tb.bsdf_queries(hp, nn, -dd, eta[hi], out_eta), seeds[hi, b, 1].contiguous())
        go = ls_zero & ~(pdf <= 0)
        cos_ln = l[:, 0] * nn[:, 0] + l[:, 1] * nn[:, 1] + l[:, 2] * nn[:, 2]
        trans = go & (cos_ln <= 0)
        hi_t = hi[trans]
        eta[hi_t] = out_eta[trans]
        absorb[hi_t] = out_abs[trans]
        gi = hi[go]
        cos_nl = (nn[:, 0] * l[:, 0] + nn[:, 1] * l[:, 1] + nn[:, 2] * l[:, 2]).abs()
        T[gi] = T[gi] * ((f[go] * cos_nl[go][:, None]) / pdf[go][:, None])
        bsdf_pdf[gi] = pdf[go]
        ray_type[gi] = typ[go]
        d[gi] = l[go]
        o[gi] = p[go] + _ff(nn[go], l[go]) * float(RAY_EPS)
        alive = gi
    return L.cpu().numpy(), length.cpu().numpy(), prims_out.cpu().numpy()


@pytest.mark.parametrize("name", ["cornell", "veach", "envmini", "meshlight"])
def test_a_path_built_from_the_queries_is_pathtrace(name):
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path(name))
    cam, opt = snap.camera, snap.options
    W, H, spp = 48, 32, 3
    opt.width, opt.height = W, H
    r = tb.Renderer(snap.scene)
    rays, _ = r.camera_rays(cam, opt, tb.frame_samples(W, H, 0, spp, device="cuda"))
    n, depth = rays.shape[0], opt.maxDepth
    seeds = _seeds(np.random.default_rng(18), n * depth * 2).reshape(n, depth, 2)
    got, glen, gprims = torch_path_trace(r, snap, rays, torch.from_numpy(seeds).cuda())
    rn = rays.cpu().numpy()
    want, wlen, wprims = lightoracle.path_trace_reseeded(snap.scene, rn[:, 0:3], rn[:, 4:7], rn[:, 3], depth, seeds)
    # every ray, hit point, eta and seed the queries see is the restatement's bit for bit (the torch ops that form
    # them, o + d*t, -d and p + n*eps, are single IEEE float32 operations, as in the restatement), so the paths are
    # the same paths
    assert (glen == wlen).all(), (int((glen != wlen).sum()), name)
    assert (gprims == wprims).all(), (int((gprims != wprims).any(1).sum()), name)
    assert (wlen > 1).any() and (wprims >= 0).any()
    # the radiance is summed by torch in the restatement's order, but its throughput goes through torch.exp instead
    # of the restatement's expf (a few ulp apart) and each bounce multiplies rounding errors of a few ulp into the
    # sum; over at most maxDepth bounces that stays below 1e-5 relative, plus 1e-6 absolute near zero
    nan = np.isnan(want)
    assert (np.isnan(got) == nan).all(), name
    err = np.abs(got[~nan] - want[~nan])
    tol = 1e-5 * np.abs(want[~nan]) + 1e-6
    assert (err <= tol).all(), (name, float((err / np.maximum(tol, 1e-30)).max()))
    assert (want[~nan] > 0).any()
    r.close()
    snap.close()


# ---- 5. the contract shared with the other queries ----


def _both(r, q, seeds, rays):
    return r.sample_lights(q, seeds).cpu().numpy(), r.sky(rays).cpu().numpy()


def _contract_inputs(name, n, rng):
    torch = _torch()
    snap, r, q = _hit_records(name, n, rng)
    seeds = torch.from_numpy(_seeds(rng, q.shape[0])).cuda()
    rays = torch.zeros((q.shape[0], 8), device="cuda")
    rays[:, 4:7] = torch.nn.functional.normalize(torch.from_numpy(rng.normal(size=(q.shape[0], 3)).astype(F32)), dim=1).cuda()
    return snap, r, q, seeds, rays


def test_batch_order_does_not_change_results():
    torch = _torch()
    rng = np.random.default_rng(19)
    snap, r, q, seeds, rays = _contract_inputs("envmini", 5000, rng)
    a, s = _both(r, q, seeds, rays)
    perm = torch.from_numpy(rng.permutation(q.shape[0])).cuda()
    b, t = _both(r, q[perm].contiguous(), seeds[perm].contiguous(), rays[perm].contiguous())
    pn = perm.cpu().numpy()
    assert (b.view(np.uint32) == a[pn].view(np.uint32)).all()
    assert (t.view(np.uint32) == s[pn].view(np.uint32)).all()
    for k in (1, 7, 100):   # sub-batches give the same bits
        c, u = _both(r, q[k:k + 37].contiguous(), seeds[k:k + 37].contiguous(), rays[k:k + 37].contiguous())
        assert (c.view(np.uint32) == a[k:k + 37].view(np.uint32)).all() and (u.view(np.uint32) == s[k:k + 37].view(np.uint32)).all()
    r.close()
    snap.close()


def _grid_capacity():
    # k_sample_lights holds two 256-thread CTAs per SM (128 registers a thread); one record per thread per claim
    torch = _torch()
    return torch.cuda.get_device_properties(0).multi_processor_count * 2 * 256


@pytest.mark.parametrize("count", [0, 1, 31, 33, "capacity+1"])
def test_counts(count):
    torch = _torch()
    if count == "capacity+1":
        count = _grid_capacity() + 1
    rng = np.random.default_rng(20)
    snap, r, q, seeds, rays = _contract_inputs("veach", 4096, rng)
    idx = torch.from_numpy(rng.integers(0, q.shape[0], count)).cuda()
    qq, ss, rr = q[idx].contiguous(), seeds[idx].contiguous(), rays[idx].contiguous()
    launches = r.stats().kernelLaunches
    got, sky = _both(r, qq, ss, rr)
    assert got.shape == (count, 3) and sky.shape == (count, 4)
    assert r.stats().kernelLaunches == launches + 2 * (count > 0)
    k = np.unique(np.linspace(0, max(count - 1, 0), min(count, 2048)).astype(np.int64)) if count else np.zeros(0, np.int64)
    want = lightoracle.sample_lights(snap.scene, qq.cpu().numpy()[k], ss.cpu().numpy()[k])
    assert _same(got[k], want).all()
    assert _same(sky[k], lightoracle.sky_eval(snap.scene, rr.cpu().numpy()[k, 4:7])).all()
    r.close()
    snap.close()


def test_queries_on_the_callers_stream_and_before_init():
    torch = _torch()
    rng = np.random.default_rng(21)
    snap, r, q, seeds, rays = _contract_inputs("meshlight", 4096, rng)   # r never Init
    want, wsky = _both(r, q, seeds, rays)
    assert _same(want, lightoracle.sample_lights(snap.scene, q.cpu().numpy(), seeds.cpu().numpy())).all()
    torch.cuda.synchronize()
    dq, ds, dr = torch.zeros_like(q), torch.zeros_like(seeds), torch.zeros_like(rays)
    st = torch.cuda.Stream()
    r.set_stream(st.cuda_stream)
    with torch.cuda.stream(st):
        torch.cuda._sleep(20_000_000)   # the copies land well after the calls have been queued
        dq.copy_(q)
        ds.copy_(seeds)
        dr.copy_(rays)
        got = r.sample_lights(dq, ds)
        sky = r.sky(dr)
    st.synchronize()
    r.set_stream(None)
    assert (got.cpu().numpy().view(np.uint32) == want.view(np.uint32)).all()
    assert (sky.cpu().numpy().view(np.uint32) == wsky.view(np.uint32)).all()
    r.close()
    snap.close()


@pytest.mark.parametrize("variant", ["cached", "group"])
def test_variants_give_the_same_bits(variant, tmp_path):
    rng = np.random.default_rng(22)
    snap, plain, q, seeds, rays = _contract_inputs("motionblur", 4096, rng)
    r = queryscenes.variant_renderer(variant, snap, tmp_path)
    a, s = _both(plain, q, seeds, rays)
    b, t = _both(r, q, seeds, rays)
    assert (a.view(np.uint32) == b.view(np.uint32)).all() and (s.view(np.uint32) == t.view(np.uint32)).all()
    r.close()
    plain.close()
    snap.close()


def test_no_side_effects():
    rng = np.random.default_rng(23)
    snap, r, q, seeds, rays = _contract_inputs("cornell", 2048, rng)
    cam, opt = snap.camera, snap.options
    W, H = 64, 48
    opt.width, opt.height = W, H
    r.Init(W, H)
    out = np.zeros((H, W, 4), np.float32)
    r.Render(cam, opt, out)
    acc0, st0, kernel0 = r.read_accumulator(), r.stats(), r.last_kernel()
    r.sample_lights(q, seeds)
    st1 = r.stats()
    assert st1.kernelLaunches == st0.kernelLaunches + 1 and st1.gpuMs > 0.0
    r.sky(rays)
    st2 = r.stats()
    assert st2.kernelLaunches == st0.kernelLaunches + 2 and st2.gpuMs > 0.0
    assert (st2.frames, st2.samples) == (st0.frames, st0.samples) and r.last_kernel() == kernel0
    assert (r.read_accumulator().view(np.uint32) == acc0.view(np.uint32)).all()
    # the frame counter did not move: the next Render adds frame 1, as a second Render of a fresh renderer does
    r.Render(cam, opt, out)
    other = tb.Renderer(snap.scene)
    other.Init(W, H)
    out2 = np.zeros((H, W, 4), np.float32)
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
    q = torch.zeros((n, 16), dtype=torch.float32, device="cuda")
    seeds = torch.zeros(n, dtype=torch.int32, device="cuda")
    rad = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
    rays = torch.zeros((n, 8), dtype=torch.float32, device="cuda")
    sky = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
    host = np.zeros((n, 16), np.float32)
    launches = r.stats().kernelLaunches

    def refused(entry, args, count, words):
        assert getattr(lib, entry)(r.h, *args, count) != 0
        msg = tb.last_error()
        assert msg.startswith(entry + ":") and any(w in msg for w in words), msg

    calls = (("tb200_sample_lights", [q.data_ptr(), seeds.data_ptr(), rad.data_ptr()], [8, 2, 2]),
             ("tb200_sky_eval", [rays.data_ptr(), sky.data_ptr()], [4, 8]))
    for entry, args, skew in calls:
        for k in range(len(args)):
            bad = list(args)
            bad[k] = None
            refused(entry, bad, n, ["null"])
            bad[k] = host.ctypes.data
            refused(entry, bad, n, ["not device memory"])
            bad[k] = args[k] + skew[k]
            refused(entry, bad, n - 1, ["aligned"])
        refused(entry, args, -1, ["out of range"])
        assert getattr(lib, entry)(r.h, *[None] * len(args), 0) == 0   # nothing to do: nothing launched
        assert getattr(lib, entry)(None, *args, n) != 0 and "null renderer" in tb.last_error()
    # spans past the end: tensors that own their segments (a fresh 24 MiB tensor gets a segment of its own)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    big = (24 << 20) // 64
    big_q = torch.zeros((big, 16), dtype=torch.float32, device="cuda")
    big_s = torch.zeros(big + 1, dtype=torch.int32, device="cuda")
    big_r = torch.zeros((big + 1, 3), dtype=torch.float32, device="cuda")
    refused("tb200_sample_lights", [big_q.data_ptr(), big_s.data_ptr(), big_r.data_ptr()], big + 1, ["past the end"])
    assert "q:" in tb.last_error()
    big_rays = torch.zeros((big * 2, 8), dtype=torch.float32, device="cuda")
    big_sky = torch.zeros((big * 2 + 1, 4), dtype=torch.float32, device="cuda")
    refused("tb200_sky_eval", [big_rays.data_ptr(), big_sky.data_ptr()], big * 2 + 1, ["past the end"])
    assert "rays:" in tb.last_error()
    assert r.stats().kernelLaunches == launches
    if torch.cuda.device_count() > 1:
        other = torch.zeros((n, 4), dtype=torch.float32, device="cuda:1")
        refused("tb200_sky_eval", [rays.data_ptr(), other.data_ptr()], n, ["lies on device"])
    # the Python interface checks shapes, dtypes, contiguity and the device itself
    with pytest.raises(TypeError):
        r.sample_lights(q, seeds.float())
    with pytest.raises(ValueError):
        r.sample_lights(q[:, :12].contiguous(), seeds)
    with pytest.raises(ValueError):
        r.sample_lights(q, seeds[:n - 1])
    with pytest.raises(ValueError):
        r.sky(rays.cpu())
    with pytest.raises(ValueError):
        r.sky(rays, torch.zeros((n, 3), device="cuda"))
    with pytest.raises(ValueError):
        r.sky(torch.zeros((8, n), device="cuda").t())
    r.close()
    snap.close()
