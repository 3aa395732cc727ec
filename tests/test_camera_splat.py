"""The camera-sample and splat queries without a GPU: the record layout of include/tinsel_b200.h, the order of
tinsel_b200.frame_samples, and the restatement's camera samples (oracle_camera_samples, tests/camera_oracle.cpp)
against its trace_frame raster positions and oracle_generate_ray."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import cameraoracle
import refdrv

F32 = np.float32
HEADER = tb.ROOT + "/include/tinsel_b200.h"


def _header_layout():
    src = r'''
#include <stddef.h>
#include <stdio.h>
#include "tinsel_b200.h"
int main(void)
{
    printf("size %zu pixel %zu frame %zu\n", sizeof(tb200_camera_sample), offsetof(tb200_camera_sample, pixel),
           offsetof(tb200_camera_sample, frame));
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call(["cc", "-I", os.path.dirname(HEADER), c, "-o", exe])
        return subprocess.check_output([exe], text=True)


def test_record_layout_matches_the_header():
    got = dict(re.findall(r"(\w+) (\d+)", _header_layout()))
    assert int(got["size"]) == C.sizeof(abi.CameraSample) == abi.CAMERA_SAMPLE_DTYPE.itemsize == 8
    assert int(got["pixel"]) == abi.CameraSample.pixel.offset == abi.CAMERA_SAMPLE_DTYPE.fields["pixel"][1] == 0
    assert int(got["frame"]) == abi.CameraSample.frame.offset == abi.CAMERA_SAMPLE_DTYPE.fields["frame"][1] == 4
    assert "tb200_camera_rays" in abi.EXPORTS and "tb200_splat" in abi.EXPORTS


@pytest.mark.parametrize("size", [(1, 1), (7, 5), (1, 9), (640, 480)])
def test_frame_samples_order(size):
    torch = pytest.importorskip("torch")
    W, H = size
    s = tb.frame_samples(W, H, 5, 3, device="cpu")
    assert s.dtype == torch.int32 and tuple(s.shape) == (3 * W * H, 2) and s.is_contiguous()
    a = s.numpy()
    assert (a[:, 0] == np.tile(np.arange(W * H), 3)).all()
    assert (a[:, 1] == np.repeat([5, 6, 7], W * H)).all()
    rec = a.view(abi.CAMERA_SAMPLE_DTYPE).reshape(-1)
    assert rec["pixel"][W * H - 1] == W * H - 1 and rec["frame"][W * H] == 6


def test_frame_samples_edges():
    pytest.importorskip("torch")
    # frames wrap as the renderer's int32 counter does
    a = tb.frame_samples(2, 1, 2 ** 31 - 1, 2, device="cpu").numpy()
    assert a[:, 1].tolist() == [2 ** 31 - 1, 2 ** 31 - 1, -2 ** 31, -2 ** 31]
    assert tb.frame_samples(2, 1, -1, 1, device="cpu").numpy()[:, 1].tolist() == [-1, -1]
    assert tuple(tb.frame_samples(3, 3, 0, 0, device="cpu").shape) == (0, 2)
    for bad in ((0, 1, 0, 1), (1, 0, 0, 1), (-2, 3, 0, 1), (2, 2, 0, -1)):
        with pytest.raises(ValueError):
            tb.frame_samples(*bad, device="cpu")


def _cameras():
    """The snapshot cameras of cornell and motionblur (its shutter is open), and a rotated camera with a wide and a
    narrow field of view."""
    out = []
    for name in ("cornell", "motionblur"):
        snap = tb.Snapshot(tb.scene_path(name))
        out.append((name, snap.camera))
        snap.close()
    base = out[0][1]
    for name, fov, rot in (("rotated wide", 2.6, (0.1, 0.3, -0.2, 0.927)), ("narrow", 0.05, (0.0, 0.0, 0.0, 1.0))):
        cam = abi.copy_struct(base)
        cam.fov = fov
        r = np.asarray(rot, np.float64)
        cam.rotation[:] = (r / np.linalg.norm(r)).astype(F32).tolist()
        cam.shutterStart, cam.shutterEnd = 0.25, 0.75
        out.append((name, cam))
    return out


@pytest.mark.parametrize("size", [(1, 1), (7, 5), (33, 20)])
def test_oracle_camera_samples_match_trace_frame_and_generate_ray(size):
    """oracle_camera_samples (tests/camera_oracle.cpp) draws what the restatement's trace_sample draws: the raster
    positions of trace_frame bit for bit, in the same build and in oracle/libtinsel_oracle.so, and the ray
    oracle_generate_ray makes through them."""
    W, H = size
    port = refdrv.PortScene.from_snapshot(tb.scene_path("cornell"))
    port.set_size(W, H)
    port.set_max_depth(1)
    for frame in (0, 3, 2 ** 31 - 1, -1):
        _, ras = port.trace_frame(frame)
        _, ras_same_build = cameraoracle.trace_frame(port.lib.tb200_snapshot_scene(port._keep), port.camera, port.options,
                                                      frame)
        s = np.stack([np.arange(W * H), np.full(W * H, frame)], 1).astype(np.int32)
        for name, cam in _cameras():
            o, d, t, r = cameraoracle.camera_samples(cam, W, H, s)
            # the raster position depends on the seed alone, not on the camera
            assert (r.view(np.uint32) == ras.reshape(-1, 2).view(np.uint32)).all(), (name, size, frame)
            assert (r.view(np.uint32) == ras_same_build.reshape(-1, 2).view(np.uint32)).all(), (name, size, frame)
            assert ((t >= min(cam.shutterStart, cam.shutterEnd)) & (t <= max(cam.shutterStart, cam.shutterEnd))).all()
            for k in list(range(min(W * H, 8))) + [W * H - 1]:
                go, gd = cameraoracle.generate_ray(cam, W, H, r[k, 0], r[k, 1])
                assert (o[k].view(np.uint32) == go.view(np.uint32)).all() and (d[k].view(np.uint32) == gd.view(np.uint32)).all(), (name, k)
    port.close()


def test_oracle_camera_samples_out_of_range_pixels():
    W, H = 7, 5
    _, cam = _cameras()[0]
    s = np.array([[-1, 0], [W * H, 0], [-2 ** 31, 7], [2 ** 31 - 1, -1], [W * H - 1, 2]], np.int32)
    o, d, t, r = cameraoracle.camera_samples(cam, W, H, s)
    assert (o[:4] == 0).all() and (d[:4] == 0).all() and (t[:4] == 0).all() and np.isnan(r[:4]).all()
    assert np.isfinite(r[4]).all() and (np.floor(r[4]) == [W - 1, H - 1]).all()
