"""The lane-owned wavefront kernel has two instantiations (wf2_lanes.cuh; kernels.cu: launch_wavefront2): one with every
scene feature (probe, motion, transmission, subsurface, clearcoat, absorption) and one compiled without them, which
scenes that have none of them run (api.cu: scene_features).  Routing to the right one, and the same bits from both."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import refdrv
import schedenv

pytestmark = pytest.mark.gpu

SPECIALIZED, GENERIC = "wf2_lq.specialized", "wf2_lq.generic"
SIZE = (96, 64)


@pytest.fixture(autouse=True)
def lane_layout():
    with schedenv.knobs(**schedenv.ROUTES["lanes"]):
        yield


def _port(path):
    subprocess.check_call(["make", "-s", "-C", os.path.join(refdrv.ROOT, "oracle"), "port"])
    p = refdrv.PortScene.from_snapshot(path)
    p.set_size(*SIZE)
    return p


def _trace(path, frame=2):
    """Per-sample radiance and raster position of one frame on the GPU, and the name of the kernel that traced it.
    The lane-owned kernel carries each sample's raster position in its slot from the sample's generation to its
    splat (wf2_common.cuh: wf2_stage_r, wf2_lanes.cuh: wf2_splat), past every stage that must leave it alone."""
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = SIZE
    r = tb.Renderer(snap.scene)
    r.Init(*SIZE)
    rad, ras = r.trace_frame(cam, opt, frame)
    kernel = r.last_kernel()
    r.close()
    snap.close()
    return (rad, ras), kernel


def _assert_matches_port(path, traced, frame=2):
    rad, ras = traced
    port = _port(path)
    prad, pras = port.trace_frame(frame, nthreads=8)
    port.close()
    same = (rad.view(np.uint32) == prad.view(np.uint32)).all(-1) | (np.isnan(rad).any(-1) & np.isnan(prad).any(-1))
    assert same.all(), "%s: %d of %d samples differ from the CPU restatement" % (path, int((~same).sum()), same.size)
    same = (ras.view(np.uint32) == pras.view(np.uint32)).all(-1)
    assert same.all(), "%s: %d of %d raster positions differ from the CPU restatement" % (path, int((~same).sum()), same.size)


@pytest.mark.parametrize("name,kernel", [("cornell", SPECIALIZED), ("simple", SPECIALIZED), ("gloss", SPECIALIZED),
                                         ("meshlight", SPECIALIZED), ("glass", GENERIC), ("mini", GENERIC),
                                         ("furnace", GENERIC), ("many", GENERIC), ("motionblur", GENERIC)])
def test_routing(name, kernel):
    _, ran = _trace(tb.scene_path(name))
    assert ran == kernel


def test_override_runs_generic():
    with schedenv.knobs(**schedenv.ROUTES["lanes-generic"]):
        _, ran = _trace(tb.scene_path("cornell"))
    assert ran == GENERIC


@pytest.mark.parametrize("name", ["cornell", "meshlight"])
def test_specialized_equals_generic_and_restatement(name):
    path = tb.scene_path(name)
    rad, ran = _trace(path)
    assert ran == SPECIALIZED
    with schedenv.knobs(**schedenv.ROUTES["lanes-generic"]):
        grad, gran = _trace(path)
    assert gran == GENERIC
    assert all((a.view(np.uint32) == b.view(np.uint32)).all() for a, b in zip(rad, grad))
    _assert_matches_port(path, rad)


def _spheres(scene):
    return [i for i in range(scene.numPrimitives) if scene.primitives[i].type == abi.SPHERE and scene.primitives[i].lightSamples == 0]


def _cornell_variant(tmp_path, *features):
    """cornell with the given features switched on, saved as a snapshot."""
    snap = tb.Snapshot(tb.scene_path("cornell"))
    scene = snap.scene.contents
    cam, opt = snap.camera, snap.options
    keep = []
    sphere = _spheres(scene)[0]
    prim = scene.primitives[sphere]
    for feature in features:
        _switch_on(scene, prim, feature, keep)
    path = str(tmp_path / ("cornell_%s.tsnap" % "_".join(features)))
    assert tb.load_library().tb200_snapshot_save(path.encode(), C.byref(scene), C.byref(cam), C.byref(opt)) == 0
    for k in keep:
        k.close()
    snap.close()
    return path


def _switch_on(scene, prim, feature, keep):
    if feature == "probe":
        env = tb.Snapshot(tb.scene_path("envmini"))
        keep.append(env)
        scene.sky = abi.copy_struct(env.scene.contents.sky)
    elif feature == "motion":
        prim.end.p[1] = prim.start.p[1] + 0.25
    elif feature in ("transmission", "subsurface", "clearcoat"):
        setattr(prim.material, feature, 0.5)
    elif feature == "absorption":
        # on the sphere when it transmits, else on the roughest opaque material
        if prim.material.transmission == 0.0:
            mats = [i for i in range(scene.numPrimitives) if scene.primitives[i].lightSamples == 0]
            prim = scene.primitives[max(mats, key=lambda i: scene.primitives[i].material.roughness)]
        prim.material.absorption[:] = [1.5, 0.5, 3.0]


@pytest.mark.parametrize("feature", ["probe", "motion", "transmission", "subsurface", "clearcoat", "absorption"])
def test_one_feature_variants_run_generic(feature, tmp_path):
    path = _cornell_variant(tmp_path, feature)
    rad, ran = _trace(path)
    assert ran == GENERIC
    _assert_matches_port(path, rad)


def test_absorption_reaches_the_image(tmp_path):
    """On an opaque material a BSDF sample below the surface has pdf 0 and ends the path before it can enter the
    medium, so absorption alone leaves cornell's image as it is.  Under a transmissive sphere the Beer-Lambert
    branch runs: the image differs from the one without absorption, and matches the restatement."""
    clear, ran = _trace(_cornell_variant(tmp_path, "transmission"))
    path = _cornell_variant(tmp_path, "transmission", "absorption")
    rad, ran = _trace(path)
    assert ran == GENERIC
    assert not (rad[0].view(np.uint32) == clear[0].view(np.uint32)).all()
    _assert_matches_port(path, rad)
