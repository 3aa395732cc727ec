"""The closest-hit query with the hit triangle, CPU side: the restatement's batch form (tests/trioracle.py, the arm
tb200_trace_rays_tri is checked against) returns tb200_trace_rays' arm's hits and primitives bit for bit, and a triangle
record that passes the checks that need no restatement (trioracle.check_semantics); and the ctypes mirror of
tb200_tri_hit has the header's layout."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import fuzzscene
import rayoracle
import raysets
import trioracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SNAPSHOTS = sorted(f[:-6] for f in os.listdir(os.path.join(ROOT, "scenes")) if f.endswith(".tsnap"))
N = 8192


def _check(path, rng, time=(0.0, 1.0)):
    snap = tb.Snapshot(path)
    scene = snap.scene.contents
    plain = rayoracle.RayOracle.from_snapshot(path)
    tri_oracle = trioracle.TriOracle.from_snapshot(path)
    cam = raysets.camera_rays(snap.camera, N, rng)
    h, p = plain.trace_rays(cam)
    rays = np.concatenate([cam, raysets.random_rays(scene, N, rng, time), raysets.secondary_rays(cam, h, p, rng),
                           raysets.fallback_rays(scene, rng)])
    want_h, want_p = plain.trace_rays(rays)
    hits, prims, tri, uvw = tri_oracle.trace_rays_tri(rays, nthreads=3)
    bad = raysets.mismatches(hits, prims, want_h, want_p)
    assert len(bad) == 0, "%d of %d rays differ from oracle_trace_rays, first %s" % (len(bad), len(rays), rays[bad[0]])
    counts = trioracle.check_semantics(scene, rays, hits, prims, tri, uvw, os.path.basename(path))
    types = {p.type for p in C.cast(scene.primitives, C.POINTER(abi.Primitive * scene.numPrimitives)).contents}
    assert counts[0] > 0 or abi.MESH not in types, "no mesh hit in a scene with meshes"
    assert counts[1] > 0 or not types & {abi.SPHERE, abi.PLANE}, "no sphere or plane hit in a scene with them"
    tri_oracle.close()
    plain.close()
    snap.close()
    return counts


@pytest.mark.parametrize("name", SNAPSHOTS)
def test_snapshot_records_match_trace(name):
    _check(tb.scene_path(name), np.random.RandomState(3), (-0.5, 1.5) if name == "motionblur" else (0.0, 1.0))


@pytest.mark.parametrize("family,seed,swap", [("ties", 0, False), ("ties", 0, True), ("instanced", 1, False), ("big", 0, False)])
def test_fuzz_records_match_trace(family, seed, swap, tmp_path):
    path = str(tmp_path / "s.tsnap")
    fuzzscene.make_mesh_scene(seed, path, family, swap_ties=swap)
    mesh_hits, _ = _check(path, np.random.RandomState(seed + 5), (-0.5, 1.5))
    assert mesh_hits > 0


def test_tri_hit_layout_matches_header():
    assert C.sizeof(abi.TriHit) == 16
    assert [(f, abi.TriHit.__dict__[f].offset) for f, _ in abi.TriHit._fields_] == [("tri", 0), ("u", 4), ("v", 8), ("w", 12)]
    header = open(os.path.join(ROOT, "include", "tinsel_b200.h")).read()
    rec = re.search(r"typedef struct tb200_tri_hit \{([^}]*)\}", header).group(1)
    assert re.findall(r"(\w+)[,;]", rec) == [f for f, _ in abi.TriHit._fields_]
    # Renderer.trace_rays_tri hands an (N, 4) int32 tensor to the library as tb200_tri_hit records
    assert np.dtype(np.int32).itemsize * 4 == C.sizeof(abi.TriHit)
