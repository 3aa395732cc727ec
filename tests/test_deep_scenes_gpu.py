"""The wide wavefront kernels (wf2_l2: 2048 slots per CTA, each path's cold half in a 128-byte record in global memory)
and the probe at the scale they were built for, on the stand-ins of tests/bigscene.py: ajax_like (a 512 000-triangle
mesh, instanced twice, one instance a mesh light) and env_like (glass lit only by a 4000 x 2000 probe).

  * one frame at the full size of BASELINE.json's ajax (1024^2) and env (2048^2) configurations, per sample and bit for
    bit against the CPU restatement (NaN matching NaN): launches of many samples per slot, so every slot is refilled
    and its cold record handed from path to path; ajax_like under every knob that selects another kernel or walk.
    The kernel that ran is pinned by name (test_route_gpu's rule), so a scene sent elsewhere fails loudly;
  * the split-queue tuner through its phases in one accumulation, against the float64 film of the restatement's
    samples (and in counting mode), then per sample on the route it decided;
  * the probe queries on 4 M seeds and the mesh-light query on 1 M seeds against the restatement, with draws that
    land on runs of equal cdfX values and on cdfX values exactly (where lower_bound's < and <= part);
  * a renderer from the scene cache (the probe's 8 M-entry tables) against the direct one."""
import os
import time

import numpy as np
import pytest

import tinsel_b200 as tb
import bigscene
import emitteroracle
import filmref
import lightoracle
import refdrv
import schedenv
from test_route_gpu import facts, kernel, route

pytestmark = pytest.mark.gpu

THREADS = min(os.cpu_count() or 8, 32)   # more threads than a cgroup CPU quota allows only thrash
SIZES = {"ajax_like": (1024, 1024), "env_like": (2048, 2048)}
FRAME = 3
AJAX_KNOBS = [{}, dict(SPLIT="1"), dict(SPLIT="0"), dict(CTA="512"), dict(QUEUES="lanes"), dict(TREELET="1"),
              dict(NO_FLAT="1")]
CASES = [("ajax_like", k) for k in AJAX_KNOBS] + [("env_like", {})]


@pytest.fixture(autouse=True)
def default_knobs():
    with schedenv.knobs():
        yield


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    d = tmp_path_factory.mktemp("deep")
    paths = {n: str(d / (n + ".tsnap")) for n in SIZES}
    bigscene.ajax_like(paths["ajax_like"])
    bigscene.env_like(paths["env_like"])
    return paths


@pytest.fixture(scope="module")
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


_port = {}


def port_frame(path, size, frame):
    """The restatement's (radiance, raster) of one frame, traced once per scene, size and frame."""
    key = (path, size, frame)
    if key not in _port:
        t0 = time.perf_counter()
        port = refdrv.PortScene.from_snapshot(path)
        port.set_size(*size)
        _port[key] = port.trace_frame(frame, THREADS)
        port.close()
        print("restatement %s %dx%d frame %d on %d threads: %.1f s" % (
            os.path.basename(path), size[0], size[1], frame, THREADS, time.perf_counter() - t0))
    return _port[key]


def compare(rad, ras, want, what):
    """Per sample, bit for bit (a NaN matches any NaN); returns the number of samples compared."""
    wrad, wras = want
    assert np.array_equal(ras, wras), "%s: raster positions differ" % what
    same = (rad.view(np.uint32) == wrad.view(np.uint32)).all(-1) | (np.isnan(rad).any(-1) & np.isnan(wrad).any(-1))
    bad = int((~same).sum())
    assert bad == 0, "%s: %d of %d samples differ (first at (y, x) %s)" % (
        what, bad, same.size, tuple(int(v) for v in np.argwhere(~same)[0]))
    return same.size


def _same(got, want):
    """Per row, whether every value matches: bits, except that a NaN matches any NaN."""
    return ((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all(1)


def _setup(path, size):
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = size
    return snap, cam, opt


@pytest.mark.parametrize("name,knobs", CASES, ids=["%s-%s" % (n, ",".join("%s=%s" % kv for kv in k.items()) or "default")
                                                   for n, k in CASES])
def test_full_size_frame_per_sample(name, knobs, scenes, num_sms):
    size = SIZES[name]
    assert size[0] * size[1] >= 6 * num_sms * 1024      # a large launch: several paths per slot
    want = port_frame(scenes[name], size, FRAME)
    snap, cam, opt = _setup(scenes[name], size)
    with schedenv.knobs(**knobs) as applied:
        expect = kernel(route(facts(scenes[name]), applied), size[0] * size[1], num_sms)
        r = tb.Renderer(snap.scene)
    r.Init(*size)
    t0 = time.perf_counter()
    rad, ras = r.trace_frame(cam, opt, FRAME)
    ran = r.last_kernel()
    n = compare(rad, ras, want, "%s %s" % (name, knobs))
    print("%-9s %-12s ran %-16s %8d samples bit-exact in %.1f s" % (
        name, ",".join("%s=%s" % kv for kv in knobs.items()) or "default", ran, n, time.perf_counter() - t0))
    assert ran == expect, "%s %s ran %s, the rule says %s" % (name, knobs, ran, expect)
    if not knobs:
        assert ran.startswith("wf2_l2."), ran
    r.close()
    snap.close()


def test_tuner_phases_in_one_accumulation(scenes):
    """Launches of 2^18 samples on a fresh renderer: split, split (timed), generic (timed), then the faster twice; the
    film of all five against the float64 film of the restatement's samples, in counting mode too; then one frame per
    sample on the route the tuner kept."""
    path, size, launches = scenes["ajax_like"], (512, 512), 5
    assert route(facts(path), {})["tune"]
    t0 = time.perf_counter()
    snap, cam, opt = _setup(path, size)
    copt = filmref.counting_options(opt)
    r, rc = tb.Renderer(snap.scene), tb.Renderer(snap.scene)
    r.Init(*size)
    rc.Init(*size)
    ran = {"gauss": [], "counting": []}
    for _ in range(launches):
        r.render_device(cam, opt, 1)
        ran["gauss"].append(r.last_kernel())
        rc.render_device(cam, copt, 1)
        ran["counting"].append(rc.last_kernel())
    for what, names in ran.items():
        assert names[:3] == ["wf2_l2.split", "wf2_l2.split", "wf2_l2.generic"], (what, names)
        assert names[3] in ("wf2_l2.split", "wf2_l2.generic") and names[4] == names[3], (what, names)
    gauss, counts = filmref.Film64(*size, opt), filmref.Film64(*size, copt)
    for f in range(launches):
        rad, ras = port_frame(path, size, f)
        gauss.add(ras, rad)
        counts.add(ras, rad)
    assert r.stats().samples == gauss.samples == launches * size[0] * size[1]
    filmref.assert_film_close(r.read_accumulator(), gauss, "ajax_like 512^2 x %d launches %s" % (launches, ran["gauss"]))
    img = rc.read_accumulator()
    filmref.assert_counts(img, counts, "ajax_like counting")
    filmref.assert_film_close(img, counts, "ajax_like counting")
    rad, ras = r.trace_frame(cam, opt, 2)
    assert r.last_kernel() == ran["gauss"][-1]
    n = compare(rad, ras, port_frame(path, size, 2), "ajax_like after the tuner decided %s" % r.last_kernel())
    print("tuner: %s; film of %d samples within bounds; %d samples bit-exact on %s; %.1f s" % (
        ran["gauss"], gauss.samples, n, r.last_kernel(), time.perf_counter() - t0))
    r.close()
    rc.close()
    snap.close()


def first_draws(seeds, k):
    """The first k Randf draws of Random(seed) for every uint32 seed, as float32 arrays (emitteroracle.randf,
    vectorised)."""
    m = np.uint64(0xffffffff)
    s1 = (seeds.astype(np.uint64) + np.uint64(315645664)) & m
    s2 = s1 ^ np.uint64(0x13ab45fe)
    out = []
    for _ in range(k):
        a, b = s1, s2
        s1 = (b ^ (((a << np.uint64(5)) | (a >> np.uint64(27))) & m)) ^ ((a * b) & m)
        s2 = s1 ^ (((b << np.uint64(12)) | (b >> np.uint64(20))) & m)
        out.append(s1.astype(np.float32) * np.float32(2.3283064365386963e-10))
    return out


def _seeds(rng, n):
    """n uint32 seeds, the edge seeds (draws of exactly 0 and 1, column searches that end past the row) first."""
    edge = np.array(list(emitteroracle.EDGE_SEEDS.values()) + emitteroracle.COL_END_SEEDS, np.uint32)
    return np.concatenate([edge, rng.integers(0, 2 ** 32, n - len(edge), dtype=np.uint64).astype(np.uint32)])


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_probe_queries_on_4m_seeds(scenes):
    """sample_probe on 4 M seeds and sky on the directions it returns, bit for bit; the draws that exercise
    LowerBound's tie-breaking are counted from the restatement's tables."""
    import torch
    t0 = time.perf_counter()
    n = 1 << 22
    snap = tb.Snapshot(scenes["env_like"])
    sky = snap.scene.contents.sky
    W, H = sky.probeWidth, sky.probeHeight
    seeds = _seeds(np.random.default_rng(61), n)
    r = tb.Renderer(snap.scene)
    out = torch.full((n, 8), float("nan"), device="cuda")
    r.sample_probe(_cuda(seeds.view(np.int32)), out)
    got = out.cpu().numpy()
    want = emitteroracle.sample_probe(snap.scene, seeds)
    bad = ~_same(got, want)
    assert not bad.any(), "%d of %d probe samples differ; first: seed %d device %s restatement %s" % (
        int(bad.sum()), n, seeds[np.argmax(bad)], got[np.argmax(bad)], want[np.argmax(bad)])
    rays = torch.zeros((n, 8), device="cuda")
    rays[:, 4:7] = out[:, 0:3]
    sky_got = r.sky(rays).cpu().numpy()
    sky_want = lightoracle.sky_eval(snap.scene, got[:, 0:3])
    bad = ~_same(sky_got, sky_want)
    assert not bad.any(), "%d of %d sky values differ" % (int(bad.sum()), n)
    # where each draw lands in the tables: LowerBound over cdfY, then over the row's cdfX
    r1, r2 = first_draws(seeds, 2)
    assert all([r1[k], r2[k]] == emitteroracle.randf(int(seeds[k]), 2) for k in range(64))
    _, cdf_x, _, cdf_y, _ = bigscene.probe_tables(sky)
    row = np.searchsorted(cdf_y, r1, "left")
    run = exact = 0
    for j in np.unique(row[row < H]):
        sel = row == j
        col = np.searchsorted(cdf_x[j], r2[sel], "left")
        inside = col < W
        value = cdf_x[j, col[inside]]
        nxt = cdf_x[j, np.minimum(col[inside] + 1, W - 1)]
        run += int(((value == nxt) & (col[inside] + 1 < W)).sum())
        exact += int((value == r2[sel][inside]).sum())
    print("probe: %d seeds, dir/pdf/color and sky bit-exact; %d draws land on a run of equal cdfX values, %d equal a "
          "cdfX value exactly; %.1f s" % (n, run, exact, time.perf_counter() - t0))
    assert run > 0 and exact > 0
    r.close()
    snap.close()


def test_mesh_light_samples_on_1m_seeds(scenes):
    """sample_emitters on the ajax_like mesh light (an area CDF of 512 000 entries), bit for bit."""
    import torch
    t0 = time.perf_counter()
    n = 1 << 20
    snap = tb.Snapshot(scenes["ajax_like"])
    sc = snap.scene.contents
    lights = [i for i in range(sc.numPrimitives) if sc.primitives[i].lightSamples > 0 and sc.primitives[i].type == tb.abi.MESH]
    assert len(lights) == 1
    rng = np.random.default_rng(62)
    seeds = _seeds(rng, n)
    times = rng.uniform(0.0, 1.0, n).astype(np.float32)
    r = tb.Renderer(snap.scene)
    q = tb.emitter_queries(torch.full((n,), lights[0], dtype=torch.int32, device="cuda"), _cuda(times))
    out = torch.full((n, 8), float("nan"), device="cuda")
    r.sample_emitters(q, _cuda(seeds.view(np.int32)), out)
    got = out.cpu().numpy()
    want = emitteroracle.sample_emitters(snap.scene, q.cpu().numpy(), seeds)
    bad = ~_same(got, want)
    assert not bad.any(), "%d of %d mesh light samples differ; first: seed %d device %s restatement %s" % (
        int(bad.sum()), n, seeds[np.argmax(bad)], got[np.argmax(bad)], want[np.argmax(bad)])
    m = sc.meshes[sc.primitives[lights[0]].mesh]
    cdf = np.ctypeslib.as_array(m.cdf, (m.numIndices // 3,))
    tris = np.unique(np.minimum(np.searchsorted(cdf, first_draws(seeds, 1)[0], "left"), len(cdf) - 1)).size
    print("mesh light: %d seeds over %d triangles (%d of them drawn) bit-exact; %.1f s" % (
        n, len(cdf), tris, time.perf_counter() - t0))
    r.close()
    snap.close()


def test_renderer_from_cache(scenes, tmp_path):
    """env_like through tb200_create_cached (the probe and its four tables, 8 M entries each for data, pdfX and
    cdfX) equals the direct renderer per sample."""
    size = (256, 256)
    snap, cam, opt = _setup(scenes["env_like"], size)
    path = str(tmp_path / "env_like.tcache")
    tb.scene_cache_save(snap.scene, path)
    a = tb.Renderer(snap.scene)
    b = tb.Renderer(None, cache=path)
    for x in (a, b):
        x.Init(*size)
    for frame in (0, 2):
        ra, sa = a.trace_frame(cam, opt, frame)
        rb, sb = b.trace_frame(cam, opt, frame)
        assert np.array_equal(sa, sb)
        assert np.array_equal(ra.view(np.uint32), rb.view(np.uint32)), "frame %d" % frame
    assert b.stats().h2dBytes == a.stats().h2dBytes
    print("cache: env_like %dx%d, 2 frames bit-identical to the direct renderer (%d bytes uploaded)" % (
        size[0], size[1], a.stats().h2dBytes))
    a.close()
    b.close()
    snap.close()
