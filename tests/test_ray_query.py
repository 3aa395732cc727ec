"""The batched closest-hit query's CPU side: the restatement's batch form (tests/rayoracle.py, the arm the device query
is checked against) equals the restatement's own per-ray Trace, and the ctypes mirrors of tb200_ray / tb200_hit have the
header's layout."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import rayoracle
import raysets
import refdrv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SNAPSHOTS = sorted(f[:-6] for f in os.listdir(os.path.join(ROOT, "scenes")) if f.endswith(".tsnap"))


@pytest.fixture(scope="module", autouse=True)
def port_built():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "port"])


@pytest.mark.parametrize("name", SNAPSHOTS)
def test_batch_equals_per_ray_trace(name):
    snap = tb.Snapshot(tb.scene_path(name))
    port = refdrv.PortScene.from_snapshot(tb.scene_path(name))
    batch = rayoracle.RayOracle.from_snapshot(tb.scene_path(name))
    rng = np.random.RandomState(7)
    cam = raysets.camera_rays(port.camera, 1500, rng)
    hits, prims = batch.trace_rays(cam, nthreads=1)
    rays = np.concatenate([cam, raysets.random_rays(snap.scene.contents, 1500, rng, (-0.5, 1.5)),
                           raysets.secondary_rays(cam, hits, prims, rng)[:500], raysets.fallback_rays(snap.scene.contents, rng, 100)])
    hits, prims = batch.trace_rays(rays, nthreads=3)
    want_h = np.zeros_like(hits)
    want_p = np.zeros_like(prims)
    for i, r in enumerate(rays):
        prim, t, n = port.trace(r[0:3], r[4:7], float(r[3]))
        want_p[i] = prim
        want_h[i] = [t, n[0], n[1], n[2]]
    bad = raysets.mismatches(hits, prims, want_h, want_p)
    assert len(bad) == 0, "%d of %d rays differ, first %s" % (len(bad), len(rays), rays[bad[0]])
    assert (prims >= 0).any() and (prims < 0).any()
    batch.close()
    port.close()
    snap.close()


def test_ray_and_hit_layout_matches_header():
    assert C.sizeof(abi.Ray) == 32 and C.sizeof(abi.Hit) == 16
    assert [(f, abi.Ray.__dict__[f].offset) for f, _ in abi.Ray._fields_] == [("origin", 0), ("time", 12), ("dir", 16), ("pad", 28)]
    assert [(f, abi.Hit.__dict__[f].offset) for f, _ in abi.Hit._fields_] == [("t", 0), ("normal", 4)]
    header = open(os.path.join(ROOT, "include", "tinsel_b200.h")).read()
    ray = re.search(r"typedef struct tb200_ray \{([^}]*)\}", header).group(1)
    hit = re.search(r"typedef struct tb200_hit \{([^}]*)\}", header).group(1)
    assert re.findall(r"float (\w+)", ray) == [f for f, _ in abi.Ray._fields_]
    assert re.findall(r"float (\w+)", hit) == [f for f, _ in abi.Hit._fields_]
    # the Python interface hands torch's (N, 8) float32 rows to the library as tb200_ray records
    assert np.dtype(np.float32).itemsize * 8 == C.sizeof(abi.Ray)
