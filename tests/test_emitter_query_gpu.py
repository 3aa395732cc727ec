"""The emitter and probe sample queries on the device (tb200_sample_emitters / tb200_sample_probe,
Renderer.sample_emitters / sample_probe) against the CPU restatement's PrimitiveSample and ProbeSample
(tests/emitter_oracle.cpp: oracle_sample_emitters, oracle_sample_probe), bit for bit, a NaN matching any NaN.  Then
SampleLights rebuilt in torch from those queries, trace_rays and bsdf_eval, against the restatement's SampleLights with
a seed per slot (oracle_sample_lights_per_slot); and the contract the queries share with the others: batch order and
size, streams, calls before Init, scene-cache, group and no-flat renderers, side effects and refusals."""
import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import emitteroracle
import fuzzscene
import queryscenes

pytestmark = pytest.mark.gpu

F32 = np.float32
RAY_EPS = F32(0.0001)   # kRayEpsilon, render.cpp:11
TIMES = [0.0, -0.0, 0.25, 0.5, 1.0, -1.0, 1.5, 10.0, -1e6]   # finite times, inside the shutter and outside


def _torch():
    import torch
    return torch


def _same(got, want):
    """Per row, whether every value matches: bits, except that a NaN matches any NaN."""
    return ((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all(1)


def _seeds(rng, n):
    """n seeds as int32 (their bits are the uint32 seeds), the edge seeds first."""
    edge = np.array(list(emitteroracle.EDGE_SEEDS.values()) + emitteroracle.COL_END_SEEDS, np.uint32)
    rest = rng.integers(0, 2 ** 32, max(n - len(edge), 0), dtype=np.uint64).astype(np.uint32)
    return np.concatenate([edge, rest])[:n].view(np.int32)


def _lights(scene):
    return [i for i in range(scene.numPrimitives) if scene.primitives[i].lightSamples > 0]


def _cuda(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def check_emitters(r, scene_ptr, prims, times, seeds, what):
    """Runs sample_emitters on the int32 prims, float32 times and int32 seeds (numpy) and compares every record with
    the restatement; returns the device's (N, 8) records as numpy."""
    torch = _torch()
    q = tb.emitter_queries(_cuda(prims.astype(np.int32)), _cuda(times.astype(F32)))
    out = torch.full((len(prims), 8), float("nan"), device="cuda")   # the pads must be written
    pos, nrm = r.sample_emitters(q, _cuda(seeds), out)
    assert pos.data_ptr() == out.data_ptr() and nrm.data_ptr() == out.data_ptr() + 16
    got = out.cpu().numpy()
    want = emitteroracle.sample_emitters(scene_ptr, q.cpu().numpy(), seeds)
    bad = ~_same(got, want)
    if bad.any():
        k = int(np.argmax(bad))
        raise AssertionError("%s: %d of %d queries differ; first: prim %d time %r seed %d device %s restatement %s" % (
            what, int(bad.sum()), len(got), prims[k], times[k], seeds[k], got[k], want[k]))
    assert (got[:, 3].view(np.uint32) == 0).all() and (got[:, 7].view(np.uint32) == 0).all()
    return got


def check_probe(r, scene_ptr, seeds, what):
    torch = _torch()
    out = torch.full((len(seeds), 8), float("nan"), device="cuda")
    d, pdf, c = r.sample_probe(_cuda(seeds), out)
    assert tuple(d.shape) == (len(seeds), 3) and tuple(pdf.shape) == (len(seeds),) and tuple(c.shape) == (len(seeds), 3)
    got = out.cpu().numpy()
    want = emitteroracle.sample_probe(scene_ptr, seeds)
    bad = ~_same(got, want)
    if bad.any():
        k = int(np.argmax(bad))
        raise AssertionError("%s: %d of %d seeds differ; first: seed %d device %s restatement %s" % (
            what, int(bad.sum()), len(got), seeds[k], got[k], want[k]))
    assert (got[:, 7].view(np.uint32) == 0).all()
    return got


def check_scene(path, what, n=4096, times=TIMES):
    """Every light of the scene at `path` at every time of `times`, n seeds each; every other primitive and prims
    outside the scene give zeros; the probe (or its zeros)."""
    snap = tb.Snapshot(path)
    r = tb.Renderer(snap.scene)
    scene = snap.scene.contents
    rng = np.random.default_rng(41)
    lights = _lights(scene)
    for light in lights:
        seeds = _seeds(rng, n)
        t = np.array(times, F32)[np.arange(n) % len(times)]
        got = check_emitters(r, snap.scene, np.full(n, light, np.int32), t, seeds, "%s, light %d" % (what, light))
        assert (got[:, 0:3] != 0).any(1).all(), (what, light)
    others = [i for i in range(scene.numPrimitives) if i not in lights]
    bad = np.array(others + [-1, -2, scene.numPrimitives, scene.numPrimitives + 1, 2 ** 31 - 1, -2 ** 31], np.int32)
    got = check_emitters(r, snap.scene, bad, np.zeros(len(bad), F32), _seeds(rng, len(bad)), "%s, not lights" % what)
    assert (got.view(np.uint32) == 0).all()
    got = check_probe(r, snap.scene, _seeds(rng, 1 << 14), "%s, probe" % what)
    if not scene.sky.probeValid:
        assert (got.view(np.uint32) == 0).all()
    r.close()
    snap.close()
    return lights


# ---- 1. every light and probe ----


@pytest.mark.parametrize("name", queryscenes.SNAPSHOTS)
def test_snapshots(name):
    check_scene(tb.scene_path(name), name)


@pytest.mark.parametrize("family,seed,swap", queryscenes.FUZZ)
def test_fuzz_families(family, seed, swap, tmp_path):
    path = str(tmp_path / "s.tsnap")
    queryscenes.fuzz_scene(family, seed, swap, path)
    assert check_scene(path, "fuzz %s/%d" % (family, seed), n=2048)


@pytest.mark.parametrize("case", ["nee300_odd", "meshlight300", "probe255"])
def test_limit_scenes(case, tmp_path):
    path = str(tmp_path / "s.tsnap")
    info = fuzzscene.make_limit_scene(case, path)
    assert check_scene(path, case, n=2048) == info["lights"]


def test_every_kind_of_light_is_covered(tmp_path):
    # sphere and mesh lights, instanced and moving mesh lights, and mesh lights with zero-area triangles
    seen = {"sphere": False, "mesh": False, "moving mesh": False, "zero area": False}
    for k, (family, seed, swap) in enumerate(queryscenes.FUZZ):
        path = str(tmp_path / ("s%d.tsnap" % k))
        queryscenes.fuzz_scene(family, seed, swap, path)
        snap = tb.Snapshot(path)
        sc = snap.scene.contents
        for i in _lights(sc):
            p = sc.primitives[i]
            if p.type == abi.SPHERE:
                seen["sphere"] = True
            elif p.type == abi.MESH:
                seen["mesh"] = True
                seen["moving mesh"] |= list(p.start.p) != list(p.end.p) or p.start.s != p.end.s
                m = sc.meshes[p.mesh]
                pdf = np.diff(np.concatenate([[0.0], np.ctypeslib.as_array(m.cdf, (m.numIndices // 3,))]))
                seen["zero area"] |= bool((pdf == 0).any())
        snap.close()
    assert all(seen.values()), seen


def test_motion_blur_times():
    # motionblur's light is static: every finite time takes its transform as stored, as the reference's interpolation
    # between two equal transforms gives (the fuzz families' instanced mesh lights move and scale)
    times = list(np.linspace(0.0, 1.0, 17)) + [-0.5, 1.5, 3.0, -1e3, 1e3]
    check_scene(tb.scene_path("motionblur"), "motionblur", times=times)


def test_probe_edge_draws(tmp_path):
    # draws of exactly 0.0 and 1.0, and seeds whose column search ends one past the row (col == width), on envmini,
    # probe255 and the fuzz probe (black rows: plateaus in the row CDF and NaN column CDFs)
    paths = {"envmini": tb.scene_path("envmini"), "probe255": str(tmp_path / "a.tsnap"), "fuzz": str(tmp_path / "b.tsnap")}
    fuzzscene.make_limit_scene("probe255", paths["probe255"])
    fuzzscene.make_mesh_scene(0, paths["fuzz"], "probe")
    seeds = np.array(list(emitteroracle.EDGE_SEEDS.values()) + emitteroracle.COL_END_SEEDS, np.uint32).view(np.int32)
    col_end = 0
    for name, path in paths.items():
        snap = tb.Snapshot(path)
        sky = snap.scene.contents.sky
        assert sky.probeValid
        W, H = sky.probeWidth, sky.probeHeight
        cy = np.ctypeslib.as_array(sky.cdfValuesY, (H,))
        cx = np.ctypeslib.as_array(sky.cdfValuesX, (H * W,)).reshape(H, W)
        r = tb.Renderer(snap.scene)
        check_probe(r, snap.scene, seeds, name)
        for s in emitteroracle.COL_END_SEEDS:   # the second draw is 1.0: col == width where the row's CDF ends below 1
            row = int(np.searchsorted(cy, emitteroracle.randf(s, 1)[0], "left"))
            col_end += int(row < H and cx[row, -1] < 1.0)
        r.close()
        snap.close()
    assert col_end > 0


# ---- 2. the pieces suffice: SampleLights rebuilt from them ----


def _absf(x):
    """Abs as the reference's: x < 0 ? -x : x (so -0 stays -0)."""
    return x.where(~(x < 0), -x)


def _dot(a, b):
    return a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1] + a[:, 2] * b[:, 2]


def _ff(n, l):
    """FaceForward(n, l) as the restatement's face_fwd: dot(l, n) < 0 ? -n : n, the dot summed left to right."""
    return n.where(~(_dot(l, n) < 0)[:, None], -n)


def torch_sample_lights(r, snap, q, seeds):
    """SampleLights (render.cpp:103-227) of every (N, 16) light query record, in torch over the library's queries:
    sample_probe and sample_emitters for the draws, trace_rays for the shadow rays, bsdf_eval for the BSDF, with
    primitive_areas and the materials' emission.  Slot s of record k draws from Random(seeds[k, s]).  Every operation
    is the restatement's single float32 operation, in its order.  Returns (radiance (N, 3), hit (N, slots), accepted
    (N, slots)) as numpy, in oracle_sample_lights_per_slot's conventions."""
    torch = _torch()
    scene = snap.scene.contents
    n = q.shape[0]
    p, t, nn, prim, wo, eta_i, eta_o = q[:, 0:3], q[:, 3], q[:, 4:7], q[:, 7].view(torch.int32), q[:, 8:11], q[:, 11], q[:, 12]
    emission = _cuda(np.array([list(scene.primitives[i].material.emission) for i in range(scene.numPrimitives)], F32))
    areas = tb.primitive_areas(scene)
    total = torch.zeros((n, 3), device="cuda")
    hits, accepted = [], []

    def shadow(wi):
        ray = torch.zeros((n, 8), device="cuda")
        ray[:, 0:3] = p + _ff(nn, wi) * float(RAY_EPS)
        ray[:, 3] = t
        ray[:, 4:7] = wi
        h, hp = r.trace_rays(ray)
        return h[:, 0], hp

    def bsdf(wi):
        v = r.bsdf_eval(tb.bsdf_queries(prim, nn, wo, eta_i, eta_o, wi))
        return v[:, 0:3], v[:, 3]

    slot = 0
    if scene.sky.probeValid:
        wi, sky_pdf, color = r.sample_probe(seeds[:, slot].contiguous())
        _, hp = shadow(wi)
        f, bp = bsdf(wi)
        w = (0.5 * sky_pdf) / ((0.5 * bp) + (0.5 * sky_pdf))
        term = (((color * w[:, None]) * f) * _absf(_dot(wi, nn))[:, None]) * (torch.ones_like(sky_pdf) / sky_pdf)[:, None]
        total = torch.where(((hp < 0) & (bp > 0) & (w > 0))[:, None], total + term, total)
        total = total * 1.0
        hits.append(hp.clamp(min=-1))
        accepted.append(hp < 0)
        slot += 1
    for light in _lights(scene):
        ls = int(scene.primitives[light].lightSamples)
        N = int(F32(ls) + F32(1.0))
        cb, cl = float(F32(1.0) / F32(N)), float(F32(ls) / F32(N))
        inv_area = float(F32(1.0) / areas[light])
        L = torch.zeros((n, 3), device="cuda")
        for _ in range(ls):
            pos, lnrm = r.sample_emitters(tb.emitter_queries(torch.full((n,), light, dtype=torch.int32, device="cuda"), t),
                                          seeds[:, slot].contiguous())
            wi = pos - p
            d_sq = _dot(wi, wi)
            dist = torch.sqrt(d_sq)
            wi = wi * (torch.ones_like(dist) / dist)[:, None]
            st, hp = shadow(wi)
            t_sq = st * st
            near = (st - torch.sqrt(d_sq)).abs() <= float(F32(1e-2))
            nl = _absf(_dot(lnrm, wi))
            ok = (hp >= 0) & near & ~(_absf(nl) < float(F32(1e-6)))
            light_pdf = (inv_area * t_sq) / nl
            f, bp = bsdf(wi)
            w = (cl * light_pdf) / ((cb * bp) + (cl * light_pdf))
            e = emission[hp.clamp(min=0).long()]
            floor = light_pdf.where(float(F32(1e-3)) < light_pdf, torch.full_like(light_pdf, float(F32(1e-3))))
            term = ((f * w[:, None]) * e) * (_absf(_dot(wi, nn)) / floor)[:, None]
            L = torch.where((ok & (bp > 0))[:, None], L + term, L)
            hits.append(hp.clamp(min=-1))
            accepted.append(ok)
            slot += 1
        total = total + L * float(F32(1.0) / F32(ls))
    return (total.cpu().numpy(), torch.stack(hits, 1).cpu().numpy().astype(np.int32),
            torch.stack(accepted, 1).cpu().numpy())


def first_hits(r, snap, W, H, frames):
    """The light query records of the first hits of the image's own camera samples (misses dropped), with
    PathTrace's first-bounce etas."""
    torch = _torch()
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = W, H
    scene = snap.scene.contents
    eta = np.array([scene.primitives[i].material.eta for i in range(scene.numPrimitives)], F32)
    spec = np.array([scene.primitives[i].material.specular for i in range(scene.numPrimitives)], F32)
    iors = _cuda(tb.material_ior(eta, spec).reshape(-1))
    rays, _ = r.camera_rays(cam, opt, tb.frame_samples(W, H, 0, frames, device="cuda"))
    hits, prims = r.trace_rays(rays)
    keep = prims >= 0
    rays, hits, prims = rays[keep], hits[keep], prims[keep].contiguous()
    o, d, t = rays[:, 0:3], rays[:, 4:7], rays[:, 3].contiguous()
    return tb.light_queries(prims, o + d * hits[:, 0:1], hits[:, 1:4].contiguous(), (-d).contiguous(), 1.0,
                            iors[prims.long()], t)


@pytest.mark.parametrize("name", ["cornell", "veach", "envmini", "meshlight"])
def test_sample_lights_rebuilt_from_the_queries(name):
    torch = _torch()
    snap = tb.Snapshot(tb.scene_path(name))
    r = tb.Renderer(snap.scene)
    q = first_hits(r, snap, 64, 48, 2)
    m = emitteroracle.num_slots(snap.scene.contents)
    seeds = _seeds(np.random.default_rng(42), q.shape[0] * m).reshape(q.shape[0], m)
    got, ghit, gacc = torch_sample_lights(r, snap, q, _cuda(seeds))
    want, whit, wacc = emitteroracle.sample_lights_per_slot(snap.scene, q.cpu().numpy(), seeds)
    # every shadow ray and its acceptance are the restatement's
    assert (ghit == whit).all(), (name, int((ghit != whit).sum()))
    assert (gacc == wacc).all(), (name, int((gacc != wacc).sum()))
    assert wacc.any() and (whit >= -1).all()
    # and so is the radiance, bit for bit: each torch op is the restatement's single IEEE float32 operation
    bad = ~_same(got, want)
    assert not bad.any(), (name, int(bad.sum()), got[bad][:4], want[bad][:4])
    assert (want > 0).any()
    r.close()
    snap.close()


# ---- 3. the contract shared with the other queries ----


def _contract_inputs(name, n, rng, tmp_path=None):
    """(snap, renderer, emitter queries, seeds): queries over the scene's lights and other prims.  name: a snapshot,
    or one of fuzzscene.LIMIT_CASES written under tmp_path."""
    path = tb.scene_path(name)
    if name in fuzzscene.LIMIT_CASES:
        path = str(tmp_path / (name + ".tsnap"))
        fuzzscene.make_limit_scene(name, path)
    snap = tb.Snapshot(path)
    r = tb.Renderer(snap.scene)
    sc = snap.scene.contents
    prims = rng.integers(-1, sc.numPrimitives + 1, n).astype(np.int32)
    lights = np.array(_lights(sc), np.int32)
    if len(lights):
        prims[::2] = lights[rng.integers(0, len(lights), (n + 1) // 2)]
    times = rng.uniform(-0.5, 1.5, n).astype(F32)
    q = tb.emitter_queries(_cuda(prims), _cuda(times))
    return snap, r, q, _cuda(_seeds(rng, n))


def _both(r, q, seeds):
    torch = _torch()
    e = torch.empty((q.shape[0], 8), device="cuda")
    p = torch.empty((seeds.shape[0], 8), device="cuda")
    r.sample_emitters(q, seeds, e)
    r.sample_probe(seeds, p)
    return e.cpu().numpy(), p.cpu().numpy()


def test_batch_order_does_not_change_results(tmp_path):
    rng = np.random.default_rng(43)
    snap, r, q, seeds = _contract_inputs("probe255", 5000, rng, tmp_path)   # a light and a probe
    a, s = _both(r, q, seeds)
    perm = _cuda(rng.permutation(q.shape[0]))
    b, u = _both(r, q[perm].contiguous(), seeds[perm].contiguous())
    pn = perm.cpu().numpy()
    assert (b.view(np.uint32) == a[pn].view(np.uint32)).all() and (u.view(np.uint32) == s[pn].view(np.uint32)).all()
    for k in (1, 7, 100):   # sub-batches give the same bits
        c, v = _both(r, q[k:k + 37].contiguous(), seeds[k:k + 37].contiguous())
        assert (c.view(np.uint32) == a[k:k + 37].view(np.uint32)).all() and (v.view(np.uint32) == s[k:k + 37].view(np.uint32)).all()
    r.close()
    snap.close()


def _grid_capacity():
    # both kernels are grid-stride with one record per 256-thread CTA slot: k_sample_emitters holds 6 CTAs per SM
    # (40 registers a thread), k_sample_probe 8 (30); the larger is the one a batch past both must loop over
    torch = _torch()
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256


@pytest.mark.parametrize("count", [0, 1, 31, 33, "capacity-1", "capacity+1"])
def test_counts(count, tmp_path):
    if isinstance(count, str):
        count = _grid_capacity() + (1 if count.endswith("+1") else -1)
    rng = np.random.default_rng(44)
    snap, r, q, seeds = _contract_inputs("probe255", 4096, rng, tmp_path)
    idx = _cuda(rng.integers(0, q.shape[0], count))
    qq, ss = q[idx].contiguous(), seeds[idx].contiguous()
    launches = r.stats().kernelLaunches
    e, p = _both(r, qq, ss)
    assert e.shape == (count, 8) and p.shape == (count, 8)
    assert r.stats().kernelLaunches == launches + 2 * (count > 0)
    assert _same(e, emitteroracle.sample_emitters(snap.scene, qq.cpu().numpy(), ss.cpu().numpy())).all()
    assert _same(p, emitteroracle.sample_probe(snap.scene, ss.cpu().numpy())).all()
    r.close()
    snap.close()


def test_queries_on_the_callers_stream_and_before_init(tmp_path):
    torch = _torch()
    rng = np.random.default_rng(45)
    snap, r, q, seeds = _contract_inputs("probe255", 4096, rng, tmp_path)   # r never Init
    want, wp = _both(r, q, seeds)
    assert _same(want, emitteroracle.sample_emitters(snap.scene, q.cpu().numpy(), seeds.cpu().numpy())).all()
    assert _same(wp, emitteroracle.sample_probe(snap.scene, seeds.cpu().numpy())).all()
    torch.cuda.synchronize()
    dq, ds = torch.zeros_like(q), torch.zeros_like(seeds)
    st = torch.cuda.Stream()
    r.set_stream(st.cuda_stream)
    with torch.cuda.stream(st):
        torch.cuda._sleep(20_000_000)   # the copies land well after the calls have been queued
        dq.copy_(q)
        ds.copy_(seeds)
        pos, nrm = r.sample_emitters(dq, ds)
        d, pdf, c = r.sample_probe(ds)
    st.synchronize()
    r.set_stream(None)
    got = torch.cat([pos, nrm], 1).cpu().numpy()
    assert (got.view(np.uint32) == want[:, [0, 1, 2, 4, 5, 6]].view(np.uint32)).all()
    gp = torch.cat([d, pdf[:, None], c], 1).cpu().numpy()
    assert (gp.view(np.uint32) == wp[:, :7].view(np.uint32)).all()
    r.close()
    snap.close()


@pytest.mark.parametrize("variant", ["cached", "group", "no_flat"])
def test_variants_give_the_same_bits(variant, tmp_path):
    rng = np.random.default_rng(46)
    for name in ("motionblur", "meshlight", "envmini"):
        snap, plain, q, seeds = _contract_inputs(name, 4096, rng)
        r = queryscenes.variant_renderer(variant, snap, tmp_path)
        a, s = _both(plain, q, seeds)
        b, t = _both(r, q, seeds)
        assert (a.view(np.uint32) == b.view(np.uint32)).all() and (s.view(np.uint32) == t.view(np.uint32)).all(), name
        r.close()
        plain.close()
        snap.close()


def test_no_side_effects():
    rng = np.random.default_rng(47)
    snap, r, q, seeds = _contract_inputs("cornell", 2048, rng)
    cam, opt = snap.camera, snap.options
    W, H = 64, 48
    opt.width, opt.height = W, H
    r.Init(W, H)
    out = np.zeros((H, W, 4), np.float32)
    r.Render(cam, opt, out)
    acc0, st0, kernel0 = r.read_accumulator(), r.stats(), r.last_kernel()
    r.sample_emitters(q, seeds)
    st1 = r.stats()
    assert st1.kernelLaunches == st0.kernelLaunches + 1 and st1.gpuMs > 0.0
    r.sample_probe(seeds)
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
    snap = tb.Snapshot(tb.scene_path("envmini"))
    r = tb.Renderer(snap.scene)
    lib = r.lib
    n = 64
    q = torch.zeros((n, 2), dtype=torch.float32, device="cuda")
    seeds = torch.zeros(n, dtype=torch.int32, device="cuda")
    eo = torch.zeros((n, 8), dtype=torch.float32, device="cuda")
    po = torch.zeros((n, 8), dtype=torch.float32, device="cuda")
    host = np.zeros((n, 8), np.float32)
    launches = r.stats().kernelLaunches

    def refused(entry, args, count, words):
        assert getattr(lib, entry)(r.h, *args, count) != 0
        msg = tb.last_error()
        assert msg.startswith(entry + ":") and any(w in msg for w in words), msg

    calls = (("tb200_sample_emitters", [q.data_ptr(), seeds.data_ptr(), eo.data_ptr()], [4, 2, 8]),
             ("tb200_sample_probe", [seeds.data_ptr(), po.data_ptr()], [2, 8]))
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
    big = (24 << 20) // 8
    big_q = torch.zeros((big, 2), dtype=torch.float32, device="cuda")
    big_s = torch.zeros(big + 1, dtype=torch.int32, device="cuda")
    big_o = torch.zeros((big + 1, 8), dtype=torch.float32, device="cuda")
    refused("tb200_sample_emitters", [big_q.data_ptr(), big_s.data_ptr(), big_o.data_ptr()], big + 1, ["past the end"])
    assert "q:" in tb.last_error()
    big_s2 = torch.zeros(big * 2, dtype=torch.int32, device="cuda")
    big_p = torch.zeros((big * 2 + 1, 8), dtype=torch.float32, device="cuda")
    refused("tb200_sample_probe", [big_s2.data_ptr(), big_p.data_ptr()], big * 2 + 1, ["past the end"])
    assert "seeds:" in tb.last_error()
    assert r.stats().kernelLaunches == launches
    if torch.cuda.device_count() > 1:
        other = torch.zeros((n, 8), dtype=torch.float32, device="cuda:1")
        refused("tb200_sample_probe", [seeds.data_ptr(), other.data_ptr()], n, ["lies on device"])
    # the Python interface checks shapes, dtypes, contiguity and the device itself
    with pytest.raises(TypeError):
        r.sample_emitters(q, seeds.float())
    with pytest.raises(ValueError):
        r.sample_emitters(torch.zeros((n, 3), device="cuda"), seeds)
    with pytest.raises(ValueError):
        r.sample_emitters(q, seeds[:n - 1])
    with pytest.raises(ValueError):
        r.sample_emitters(q, seeds, torch.zeros((n, 6), device="cuda"))
    with pytest.raises(ValueError):
        r.sample_probe(seeds.cpu())
    with pytest.raises(ValueError):
        r.sample_probe(seeds[:, None].contiguous())
    with pytest.raises(TypeError):
        r.sample_probe(seeds.float())
    with pytest.raises(ValueError):
        r.sample_probe(seeds, torch.zeros((n, 4), device="cuda"))
    with pytest.raises(ValueError):
        r.sample_probe(torch.zeros(2 * n, dtype=torch.int32, device="cuda")[::2])
    r.close()
    snap.close()
