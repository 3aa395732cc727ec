"""The accumulated image, the number people see and bench.py times, against the float64 film reference
(tests/filmref.py) per pixel and channel, in the shapes the benchmark and the API launch it.

Per-sample inputs come from the CPU restatement (PortScene.trace_frame), so the reference is independent of the
GPU.  assert_film_close allows only what a correct GPU film can differ by: the order of its fp32 additions and
the L2 adder's flush to zero.  Counting mode (box filter of width 0) checks that every pixel received exactly
the samples it should have, bit for bit."""
import os

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import sharding
import filmref
import fuzzscene
import refdrv
import schedenv
from test_filmref import NAN_FILTER, NAN_SEED, VARIANTS, apply

pytestmark = pytest.mark.gpu

THREADS = min(os.cpu_count() or 8, 32)   # more threads than a cgroup CPU quota allows only thrash
MATRIX_SCENES = ["meshlight", "motionblur", "many", "veach", "big-mesh"]
MATRIX_VARIANTS = [(s, c) for s in schedenv.SCHEDS for c in schedenv.CTAS] + [("mega", None), ("no-flat", None)]


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    """name -> snapshot path; "big-mesh" is a fuzz scene with a mesh of more than 4096 triangles, so that the
    split trace queue and the treelet engage."""
    paths = {n: tb.scene_path(n) for n in ("cornell", "veach", "meshlight", "motionblur", "many")}
    d = tmp_path_factory.mktemp("film")
    paths["big-mesh"] = str(d / "big.tsnap")
    info = fuzzscene.make_mesh_scene(0, paths["big-mesh"], "big", width=256, height=256)
    assert max(info["tris"]) > 4096, info
    paths["nan-probe"] = str(d / "probe.tsnap")
    fuzzscene.make_mesh_scene(NAN_SEED, paths["nan-probe"], "probe")
    for n, p in paths.items():
        if not os.path.exists(p):
            pytest.skip("snapshot %s not present" % p)
    return paths


@pytest.fixture(autouse=True)
def default_knobs():
    with schedenv.knobs():
        yield


_refs = {}


def reference(path, size, frames, options_list, sample_mask=None, key=None):
    """Film64s of the restatement's samples of `frames`, one per options (cached per key)."""
    if key is not None and key in _refs:
        return _refs[key]
    port = refdrv.PortScene.from_snapshot(path)
    port.set_size(*size)
    films = filmref.films_of_frames(size[0], size[1], options_list, lambda f: port.trace_frame(f, 1), frames, THREADS,
                                    sample_mask)
    port.close()
    if key is not None:
        _refs[key] = films
    return films


def setup(path, size, changes=None):
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = size
    if changes:
        apply(opt, changes)
    return snap, cam, opt


def renderer(snap, opt):
    r = tb.Renderer(snap.scene)
    r.Init(opt.width, opt.height)
    return r


# ---- the benchmark's shape and the other full-size shapes ----

def test_benchmark_shape_cornell_1024(scenes):
    """bench.py measure_one_gpu: warm-up, Init, then two render_device(32) steps on a torch stream handed to
    set_stream (frames 0-63, the lane-owned queue layout); then Render() e2e, 3 + 8 calls into a pinned host
    buffer with the streamed read-back (frames 0-10); then render_n(7), a head launch of 6 frames and a
    streamed tail (frames 0-6)."""
    import torch
    size = (1024, 1024)
    snap, cam, opt = setup(scenes["cornell"], size)
    f07 = reference(scenes["cornell"], size, range(0, 7), [opt])[0]
    f011 = f07.copy()
    f011 += reference(scenes["cornell"], size, range(7, 11), [opt])[0]
    f064 = f011.copy()
    f064 += reference(scenes["cornell"], size, range(11, 64), [opt])[0]
    r = renderer(snap, opt)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        r.set_stream(stream.cuda_stream)
        r.render_device(cam, opt, 32)
        r.Init(*size)
        torch.cuda.synchronize()
        s0 = r.stats().samples
        for _ in range(2):
            r.render_device(cam, opt, 32)
        torch.cuda.synchronize()
        img = r.read_accumulator()
    assert r.stats().samples - s0 == f064.samples
    filmref.assert_film_close(img, f064, "cornell 1024^2 2 x render_device(32)")
    r.set_stream(None)
    r.Init(*size)
    host = np.zeros((size[1], size[0], 4), np.float32)
    r.pin_output(host)
    for _ in range(3 + 8):
        r.Render(cam, opt, host)
    filmref.assert_film_close(host, f011, "cornell 1024^2 11 x Render")
    r.unpin_output()
    r.Init(*size)
    out = np.zeros_like(host)
    r.render_n(cam, opt, 7, out)
    filmref.assert_film_close(out, f07, "cornell 1024^2 render_n(7)")
    r.close()
    snap.close()


def test_veach_1920x1080_render_device_16(scenes):
    size = (1920, 1080)
    snap, cam, opt = setup(scenes["veach"], size)
    ref = reference(scenes["veach"], size, range(16), [opt])[0]
    r = renderer(snap, opt)
    r.render_device(cam, opt, 16)
    filmref.assert_film_close(r.read_accumulator(), ref, "veach 1920x1080 render_device(16)")
    r.close()
    snap.close()


# ---- every scheduler variant in the steady state: about 1 M samples in one launch ----

def matrix_reference(scenes, name):
    snap, cam, opt = setup(scenes[name], (256, 256))
    films = reference(scenes[name], (256, 256), range(16), [opt, filmref.counting_options(opt)], key=("matrix", name))
    return snap, cam, opt, films


def variant_knobs(sched, cta):
    return schedenv.sched_env(sched, cta) if cta else schedenv.knobs(**schedenv.ROUTES[sched])


@pytest.mark.parametrize("sched,cta", MATRIX_VARIANTS, ids=["%s-%s" % v if v[1] else v[0] for v in MATRIX_VARIANTS])
def test_scheduler_variants_steady_state(sched, cta, scenes):
    for name in MATRIX_SCENES:
        snap, cam, opt, (gauss, counts) = matrix_reference(scenes, name)
        copt = filmref.counting_options(opt)
        with variant_knobs(sched, cta):
            r = renderer(snap, opt)
            rc = renderer(snap, copt)
        what = "%s %s/%s 256^2 x 16" % (name, sched, cta)
        s0 = r.stats().samples
        r.render_device(cam, opt, 16)
        assert r.stats().samples - s0 == gauss.samples
        filmref.assert_film_close(r.read_accumulator(), gauss, what)
        rc.render_device(cam, copt, 16)
        img = rc.read_accumulator()
        filmref.assert_counts(img, counts, what + " counting")
        filmref.assert_film_close(img, counts, what + " counting")
        r.close()
        rc.close()
        snap.close()


# ---- work splitting ----

def test_interleaved_shards(scenes):
    """tb200_set_shard, 3 shards: each accumulator against the reference of its own samples only (tile rows
    t % 3 == shard); every pixel that none of them reaches must stay exactly zero."""
    size = (256, 192)
    snap, cam, opt = setup(scenes["cornell"], size)
    copt = filmref.counting_options(opt)
    rows = np.arange(size[1])
    for shard in range(3):
        mask = np.broadcast_to(((rows // sharding.TILE_ROWS) % 3 == shard)[:, None], (size[1], size[0]))
        gauss, counts = reference(scenes["cornell"], size, range(4), [opt, copt], mask)
        assert gauss.samples == sharding.shard_sample_count(size[0], size[1], shard, 3, 4)
        for o, ref, check in ((opt, gauss, filmref.assert_film_close), (copt, counts, filmref.assert_counts)):
            r = renderer(snap, o)
            r.set_shard(shard, 3)
            r.render_device(cam, o, 4)
            assert r.stats().samples == ref.samples
            check(r.read_accumulator(), ref, "cornell %dx%d shard %d of 3" % (size + (shard,)))
            r.close()
    snap.close()


SLAB_CASES = [("cornell", (200, 150), 3), ("veach", (160, 90), 2), ("cornell", (64, 9), 4),
              ("cornell", (64, 37), [(0, 13), (13, 1), (14, 0), (14, 23)])]   # cuts off the 4-row tile grid
SLAB_FILTERS = [("scene", {}), ("gauss-1.5", {"filterWidth": 1.5}), ("gauss-3.5", {"filterWidth": 3.5}),
                ("box-0.5", {"filterType": tb.abi.FILTER_BOX, "filterWidth": 0.5})]
SENTINEL = -7.0


@pytest.mark.parametrize("queues", ["rings", "lanes"])
@pytest.mark.parametrize("filt", SLAB_FILTERS, ids=[f[0] for f in SLAB_FILTERS])
@pytest.mark.parametrize("name,size,parts", SLAB_CASES)
def test_row_slabs(name, size, parts, filt, queues, scenes):
    """Owner-computes row slabs: set_slab renderers side by side, 4 Render() calls and one render_device(4) each, and
    a create_multi group whose members share the one device.  The rows each owner delivers, into a buffer filled with
    a sentinel, must equal the whole image's reference.  `parts`: a number of tile-row slabs (sharding.slab_rows),
    or a list of (first row, rows)."""
    fname, changes = filt
    snap, cam, opt = setup(scenes[name], size, changes)
    ref = reference(scenes[name], size, range(4), [opt], key=("slab", name, size, fname))[0]
    cuts = [sharding.slab_rows(size[1], k, parts) for k in range(parts)] if isinstance(parts, int) else parts
    what = "%s %dx%d %s queues=%s" % (name, size[0], size[1], fname, queues)
    with schedenv.knobs(**schedenv.ROUTES[queues]):
        render_out = np.full((size[1], size[0], 4), SENTINEL, np.float32)
        device_out = render_out.copy()
        for row0, nrows in cuts:
            r = renderer(snap, opt)
            r.set_slab(row0, nrows)
            for _ in range(4):
                r.Render(cam, opt, render_out)
            r.Init(*size)
            r.render_device(cam, opt, 4)
            if queues == "lanes" and nrows:
                assert r.last_kernel().startswith("wf2_lq"), r.last_kernel()
            r.read_accumulator(device_out)
            r.close()
        filmref.assert_film_close(render_out, ref, "%s: %d set_slab renderers, Render() x 4" % (what, len(cuts)))
        filmref.assert_film_close(device_out, ref, "%s: %d set_slab renderers, render_device(4)" % (what, len(cuts)))
        with schedenv.knobs(TEST_DUP_DEVICES="1", **schedenv.ROUTES[queues]):
            m = tb.Renderer(snap.scene, devices=[0] * len(cuts))
        m.Init(*size)
        out = np.full_like(render_out, SENTINEL)
        for _ in range(4):
            m.Render(cam, opt, out)
        assert m.stats().samples == 4 * size[0] * size[1]
        filmref.assert_film_close(out, ref, "%s: create_multi of %d, Render() x 4" % (what, len(cuts)))
        m.Init(*size)
        m.render_device(cam, opt, 4)
        out = m.read_accumulator(np.full_like(render_out, SENTINEL))
        filmref.assert_film_close(out, ref, "%s: create_multi of %d, render_device(4)" % (what, len(cuts)))
        m.close()
    snap.close()


@pytest.mark.parametrize("queues", ["ring", "lanes"])
@pytest.mark.parametrize("size", [(1, 1), (37, 23), (129, 65), (1021, 515)])
def test_ragged_sizes(size, queues, scenes):
    """Image sizes that are not multiples of the 8x4 sample tiles: tile padding must neither splat nor count."""
    snap, cam, opt = setup(scenes["cornell"], size)
    copt = filmref.counting_options(opt)
    gauss, counts = reference(scenes["cornell"], size, range(4), [opt, copt])
    for o, ref, check in ((opt, gauss, filmref.assert_film_close), (copt, counts, filmref.assert_counts)):
        with schedenv.knobs(QUEUES=queues):
            r = renderer(snap, o)
        r.render_device(cam, o, 4)
        assert r.stats().samples == ref.samples
        check(r.read_accumulator(), ref, "cornell %dx%d queues=%s" % (size + (queues,)))
        r.close()
    snap.close()


# ---- the film's edges: every filter variant in every kernel ----

FILTER_CASES = [(v[0], v[1], v[2], "cornell") for v in VARIANTS] + [("nan-probe", (40, 30), NAN_FILTER, "nan-probe")]
FILTER_RUNS = [(c, p) for c in FILTER_CASES for p in ("mega", "rings", "lanes", "lanes-generic")
               if p != "lanes-generic" or c[3] == "cornell"]


def expected_kernel(pipeline, scene):
    """The kernel each forced pipeline must run (kernels.cu: launch_mega, launch_wavefront2)."""
    if pipeline == "mega":
        return "k_mega"
    if pipeline == "rings":
        # cornell has one shadow ray per hit and runs free; the probe scene has a light too, so it runs hard phases
        return "wf2_smem.generic" if scene == "cornell" else "wf2_smem.hard"
    return "wf2_lq.specialized" if pipeline == "lanes" and scene == "cornell" else "wf2_lq.generic"


def run_id(case, pipeline):
    """<case>-<pipeline>; a ring-queue run also names the ring kernel's scheduling mode it pins (rings-generic,
    rings-hard), which the scene decides."""
    if pipeline == "rings":
        return "%s-rings-%s" % (case[0], expected_kernel(pipeline, case[3]).split(".")[1])
    return "%s-%s" % (case[0], pipeline)


@pytest.mark.parametrize("case,pipeline", FILTER_RUNS, ids=[run_id(c, p) for c, p in FILTER_RUNS])
def test_filter_variants(case, pipeline, scenes):
    what, size, changes, scene = case
    snap, cam, opt = setup(scenes[scene], size, changes)
    ref = reference(scenes[scene], size, range(4), [opt], key=("filter", what))[0]
    if scene == "nan-probe":
        assert np.isnan(ref.sums).any() and np.isfinite(ref.sums).any()
    with schedenv.knobs(**schedenv.ROUTES[pipeline]):
        r = renderer(snap, opt)
    r.render_device(cam, opt, 4)
    assert r.last_kernel() == expected_kernel(pipeline, scene)
    filmref.assert_film_close(r.read_accumulator(), ref, "%s %dx%d %s %s" % (scene, size[0], size[1], what, pipeline))
    r.close()
    snap.close()


# ---- jobs split into several launches (api.cu: launch_frames) ----

@pytest.mark.parametrize("pipeline", ["mega", "wavefront"])
def test_launch_split_small(pipeline, scenes):
    """A per-launch cap of 2 frames plus a bit (TINSEL_B200_TEST_LAUNCH_SAMPLES): render_device(8) then (5) take
    4 and 3 launches, render_n(7) a head of 3 launches and a tail.  Each launch must start at its own frame."""
    size = (96, 64)
    spf = 12 * 16 * 32    # samples per frame, tile padding included
    snap, cam, opt = setup(scenes["cornell"], size)
    f8 = reference(scenes["cornell"], size, range(8), [opt])[0]
    f13 = f8.copy()
    f13 += reference(scenes["cornell"], size, range(8, 13), [opt])[0]
    f7 = reference(scenes["cornell"], size, range(7), [opt])[0]
    with schedenv.knobs(TEST_LAUNCH_SAMPLES=2 * spf + 100, **schedenv.ROUTES[pipeline]):
        r = renderer(snap, opt)
    with schedenv.knobs(**schedenv.ROUTES[pipeline]):
        whole = renderer(snap, opt)
    l0 = r.stats().kernelLaunches
    r.render_device(cam, opt, 8)
    whole.render_device(cam, opt, 8)
    assert r.stats().kernelLaunches - l0 > whole.stats().kernelLaunches   # the cap did split the job
    filmref.assert_film_close(r.read_accumulator(), f8, "cornell %s 8 frames in 4 launches" % pipeline)
    r.render_device(cam, opt, 5)
    filmref.assert_film_close(r.read_accumulator(), f13, "cornell %s + 5 frames in 3 launches" % pipeline)
    r.Init(*size)
    out = np.zeros((size[1], size[0], 4), np.float32)
    r.render_n(cam, opt, 7, out)
    filmref.assert_film_close(out, f7, "cornell %s render_n(7) split" % pipeline)
    r.close()
    whole.close()
    snap.close()


def test_launch_split_at_the_31_bit_boundary(scenes):
    """cornell 64x64 has 4096 samples per frame: render_device(524289) is two launches, of 524287 frames (sample
    indices up to 2^31 - 4097) and of 2.  Counting mode: every pixel's weight equals the host's count of the
    samples that land on it (raster positions that round up onto the next pixel included), and the rgb/w image
    agrees with a 2048-frame mean of the restatement within 8 sigma.  The radiance is clamped to length 1 so
    that the spread of 2048 samples is a fair estimate (no rare firefly dominates the mean).  The spread comes
    from the same skewed samples as the mean, so the worst of 12288 such ratios runs past a normal 6 sigma: 6.3
    here, and 6.2 between two independent 2048-frame means of the restatement."""
    from concurrent.futures import ThreadPoolExecutor
    size, frames = (64, 64), 524289
    snap, cam, opt = setup(scenes["cornell"], size, {"clamp": 1.0})
    copt = filmref.counting_options(opt)
    port = refdrv.PortScene.from_snapshot(scenes["cornell"])
    port.set_size(*size)
    port.options = copt
    expect = port.box_counts(0, frames, THREADS)
    r = renderer(snap, copt)
    r.render_device(cam, copt, frames)
    assert r.stats().samples == frames * 4096
    img = r.read_accumulator()
    r.close()
    filmref.assert_counts(img, expect, "cornell 64x64 x %d frames" % frames)
    assert frames * 4096 - 4096 < int(expect.sum()) <= frames * 4096    # a few samples round off the image

    def moments(k0):   # ClampLength in fp32, as add_sample does it
        rad = np.stack([port.trace_frame(f, 1)[0] for f in range(k0, k0 + 64)])
        l = np.sqrt((rad[..., 0] * rad[..., 0] + rad[..., 1] * rad[..., 1]) + rad[..., 2] * rad[..., 2])
        c = np.where((l > np.float32(1.0))[..., None], rad * (np.float32(1.0) / l)[..., None], rad).astype(np.float64)
        return c.sum(0), (c * c).sum(0)

    with ThreadPoolExecutor(THREADS) as ex:
        parts = list(ex.map(moments, range(0, 2048, 64)))
    port.close()
    mean = sum(p[0] for p in parts) / 2048
    var = np.maximum(sum(p[1] for p in parts) / 2048 - mean ** 2, 0.0)
    gpu = img[..., :3].astype(np.float64) / img[..., 3:].astype(np.float64)
    assert np.isfinite(gpu).all()
    # a pixel whose 2048 samples all agree can still receive rarer values in 524289: the spread is floored at
    # that of one unit-length outlier in 2048 samples
    var = np.maximum(var, 1.0 / 2048)
    sigma = np.sqrt(var / 2048 + var / frames)
    z = np.abs(gpu - mean) / sigma
    print("cornell 64x64 x %d frames: worst |gpu - cpu| / sigma %.2f" % (frames, float(z.max())))
    assert float(z.max()) <= 8.0, np.unravel_index(int(np.argmax(z)), z.shape)
    snap.close()
