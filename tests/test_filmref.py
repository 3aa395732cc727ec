"""The float64 film reference (tests/filmref.py) against the reference renderer's own framebuffer, without a GPU.

splat64 of the CPU restatement's per-sample output must reproduce the golden 4-spp accumulators that the
reference's own AddSample summed (tools/make_golden.py), and the restatement's render_seeded under every filter
variant, within the summation-order bound.  Negative controls show that the bound is tight enough to notice one
lost, duplicated, moved or mis-seeded sample."""
import os
import subprocess

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import filmref
import fuzzscene
import refdrv

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# the golden scenes whose snapshot is in the repository (ajax, env and table have golden vectors only)
GOLDEN_SCENES = ["cornell", "veach", "glass", "meshlight", "motionblur", "gloss", "emitter", "furnace", "conservation",
                 "many", "mini", "envmini", "simple"]
INF = float("inf")

# filter variants: (id, size, option changes)
VARIANTS = [
    ("scene", (37, 23), {}),
    ("gauss-0.5", (37, 23), {"filterWidth": 0.5}),
    ("gauss-1.5", (37, 23), {"filterWidth": 1.5}),
    ("gauss-3.5", (37, 23), {"filterWidth": 3.5}),
    ("steep", (37, 23), {"filterWidth": 2.5, "filterFalloff": 9.0}),
    ("offset-0", (37, 23), {"filterWidth": 1.5, "filterOffset": 0.0}),
    ("offset-1", (37, 23), {"filterOffset": 1.0}),
    ("offset-1.5", (37, 23), {"filterOffset": 1.5}),
    ("box-0", (37, 23), {"filterType": abi.FILTER_BOX, "filterWidth": 0.0}),
    ("box-0.5", (37, 23), {"filterType": abi.FILTER_BOX, "filterWidth": 0.5}),
    ("box-3.5", (37, 23), {"filterType": abi.FILTER_BOX, "filterWidth": 3.5}),
    ("clamp-0", (37, 23), {"clamp": 0.0}),
    ("clamp-0.75", (37, 23), {"clamp": 0.75}),
    ("clamp-inf", (37, 23), {"clamp": INF}),
    ("1x1", (1, 1), {}),
    ("5x3", (5, 3), {}),
    ("5x3-gauss-3.5", (5, 3), {"filterWidth": 3.5}),
]
# NaN samples (a probe with black rows, see fuzzscene._probe); falloff and offset leave zero weights inside the
# footprint, which the NaN samples must still poison
NAN_SEED = 4
NAN_FILTER = {"filterWidth": 1.0, "filterFalloff": 3.0, "filterOffset": 0.1}


@pytest.fixture(scope="module", autouse=True)
def port_built():
    subprocess.check_call(["make", "-s", "-C", os.path.join(refdrv.ROOT, "oracle"), "port"])


def apply(options, changes):
    for k, v in changes.items():
        setattr(options, k, v)
    return options


def film(port, frames, options=None):
    o = port.options if options is None else options
    f = filmref.Film64(o.width, o.height, o)
    for k in frames:
        rad, ras = port.trace_frame(k, 4)
        f.add(ras, rad)
    return f


@pytest.mark.parametrize("name", GOLDEN_SCENES)
def test_splat64_matches_reference_addsample(name):
    """The restatement's samples of frames 0-3, splatted in float64, against the reference's own fp32 sums."""
    g = np.load(os.path.join(GOLD, "scene_%s.npz" % name))
    port = refdrv.PortScene.from_snapshot(tb.scene_path(name))
    port.set_size(int(g["width"]), int(g["height"]))
    worst = filmref.assert_film_close(g["accum_4spp"], film(port, range(4)), name)
    assert worst > 0.0     # the sums really are compared in another order
    port.close()


@pytest.mark.parametrize("case", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_splat64_matches_restatement_filter_variants(case):
    _, (w, h), changes = case
    port = refdrv.PortScene.from_snapshot(tb.scene_path("cornell"))
    port.set_size(w, h)
    apply(port.options, changes)
    ref = film(port, range(4))
    filmref.assert_film_close(port.render_seeded(0, 4, 2), ref, "cornell %dx%d %s" % (w, h, case[0]))
    o = port.options
    if o.filterType == abi.FILTER_GAUSSIAN and o.filterOffset >= 1.0:
        assert not ref.sums.any() and ref.n.all()    # every weight is zero, and every term is still counted
    if o.filterType == abi.FILTER_BOX and o.filterWidth == 0.0:
        assert (ref.n == ref.sums[..., 3]).all() and ref.samples == 4 * w * h
    port.close()


def test_splat64_matches_restatement_with_nan_samples(tmp_path):
    path = str(tmp_path / "probe.tsnap")
    fuzzscene.make_mesh_scene(NAN_SEED, path, "probe")
    port = refdrv.PortScene.from_snapshot(path)
    apply(port.options, NAN_FILTER)
    ref = film(port, range(4))
    nan = np.isnan(ref.sums).any(-1)
    assert 0.05 < nan.mean() < 0.95     # NaN pixels and finite pixels to compare
    filmref.assert_film_close(port.render_seeded(0, 4, 2), ref, "probe seed %d" % NAN_SEED)
    # without the zero-weight terms of the NaN samples, fewer pixels would be NaN
    o = port.options
    finite_only = filmref.Film64(o.width, o.height, o)
    for k in range(4):
        rad, ras = port.trace_frame(k, 4)
        finite_only.add(ras, rad, np.isfinite(rad).all(-1))
    assert not np.isnan(finite_only.sums).any()
    port.close()


def test_box_counts_match_splat64():
    """oracle_box_counts (raster positions only) gives the counts splat64 gives from traced samples, also where a
    raster position rounds up onto the next pixel or off the image."""
    port = refdrv.PortScene.from_snapshot(tb.scene_path("cornell"))
    port.set_size(37, 23)
    gauss = port.options
    for width in (0.0, 0.5, 1.5):
        port.options = apply(filmref.counting_options(gauss), {"filterWidth": width})
        ref = film(port, range(8))
        assert np.array_equal(port.box_counts(0, 8, 3), ref.n), width
        assert np.array_equal(port.render_seeded(0, 8, 2)[..., 3], ref.n.astype(np.float32)), width
    port.close()


# ---- negative controls: each mutation of the sample set must break the bound or the count ----

def _cornell_golden():
    g = np.load(os.path.join(GOLD, "scene_cornell.npz"))
    port = refdrv.PortScene.from_snapshot(tb.scene_path("cornell"))
    port.set_size(int(g["width"]), int(g["height"]))
    samples = [port.trace_frame(k, 4) for k in range(5)]
    return g["accum_4spp"], port, samples


def _mutated(samples, how):
    rad = [s[0].copy() for s in samples[:4]]
    ras = [s[1].copy() for s in samples[:4]]
    keep = [np.ones(r.shape[:2], bool) for r in rad]
    j, i = 20, 30
    if how == "drop":
        keep[2][j, i] = False
    elif how == "duplicate":
        rad.append(rad[2][j:j + 1, i:i + 1])
        ras.append(ras[2][j:j + 1, i:i + 1])
        keep.append(np.ones((1, 1), bool))
    elif how == "move":
        ras[2][j, i, 0] += 1.0
    elif how == "frame4":
        rad[3], ras[3] = samples[4][0].copy(), samples[4][1].copy()
    return rad, ras, keep


@pytest.mark.parametrize("how", ["drop", "duplicate", "move", "frame4"])
def test_negative_controls_break_the_bound(how):
    acc, port, samples = _cornell_golden()
    o = port.options
    rad, ras, keep = _mutated(samples, how)
    ref = filmref.Film64(o.width, o.height, o)
    for a, b, k in zip(rad, ras, keep):
        ref.add(b, a, k)
    worst, bad = filmref.film_error(acc, ref)
    assert bad is not None, "%s: the bound did not notice (worst error/bound %.3f)" % (how, worst)
    print("%-9s worst error/bound %.3g" % (how, worst))
    if how != "frame4":
        # counting mode notices the same sample-set change exactly
        co = filmref.counting_options(o)
        port.options = co
        counts = port.render_seeded(0, 4, 2)
        cref = filmref.Film64(o.width, o.height, co)
        for a, b, k in zip(rad, ras, keep):
            cref.add(b, a, k)
        with pytest.raises(AssertionError):
            filmref.assert_counts(counts, cref, how)
    port.close()
