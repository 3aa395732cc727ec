"""The generator of the large stand-in scenes (tests/bigscene.py) delivers what tests/test_deep_scenes_gpu.py relies
on: a mesh of more than 500 000 triangles whose BVH is a valid tree in the reference's format within the traversal
stack's 31 interior levels, the area CDF by MeshData's rule, and a 4000 x 2000 probe whose importance tables the
snapshot builds (snapshot.cpp: build_probe_tables) exactly as Probe::BuildCDF does, with runs of equal cdfX values and
NaN rows.  No GPU: the snapshot is written and read by the host library."""
import ctypes as C
import time

import numpy as np
import pytest

import tinsel_b200 as tb
import bigscene
from test_bvh_build import MAX_LEVELS, _check_structure


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    d = tmp_path_factory.mktemp("bigscene")
    paths = {"ajax_like": str(d / "ajax_like.tsnap"), "env_like": str(d / "env_like.tsnap")}
    return paths, bigscene.ajax_like(paths["ajax_like"]), bigscene.env_like(paths["env_like"])


def _running_sum(values):
    """MeshData's loop: the running float32 sum, one addition at a time."""
    out = np.zeros(len(values), np.float32)
    total = np.float32(0.0)
    for i, a in enumerate(values):
        total = np.float32(total + a)
        out[i] = total
    return out


def test_ajax_like_mesh(scenes):
    paths, info, _ = scenes
    m = info["mesh"]
    t0 = time.perf_counter()
    levels = _check_structure(m.nodes, m.pos, m.idx) - 1
    assert info["tris"] >= 500000 and info["tris"] == len(m.idx)
    assert levels == info["levels"] <= MAX_LEVELS
    run = _running_sum(m.areas)
    assert np.array_equal(m.cdf, (run / run[-1]).astype(np.float32)) and m.area == float(run[-1])
    # the snapshot holds the mesh as generated, with one static instance and one rotated, scaled mesh light
    snap = tb.Snapshot(paths["ajax_like"])
    sc = snap.scene.contents
    mesh = sc.meshes[0]
    assert (mesh.numIndices // 3, mesh.numNodes) == (info["tris"], len(m.nodes))
    assert np.array_equal(np.ctypeslib.as_array(mesh.cdf, (info["tris"],)), m.cdf)
    assert C.string_at(mesh.nodes, mesh.numNodes * 32) == m.nodes.tobytes()
    inst = [sc.primitives[i] for i in range(sc.numPrimitives) if sc.primitives[i].type == tb.abi.MESH]
    assert len(inst) == 2 and all(bytes(p.start) == bytes(p.end) for p in inst)
    assert inst[1].lightSamples > 0 and inst[1].end.s != 1.0 and list(inst[1].end.r) != [0.0, 0.0, 0.0, 1.0]
    snap.close()
    print("ajax_like: %d triangles, %d BVH nodes in %d interior levels, generated in %.1f s (checked in %.1f s)" % (
        info["tris"], len(m.nodes), levels, info["seconds"], time.perf_counter() - t0))


def test_env_like_probe_tables(scenes):
    """The snapshot's tables equal BuildCDF restated in numpy bit for bit (NaN rows included); in float64 every
    row's CDF rises, ends within one ulp of 1, and the pdf sums to 1."""
    paths, _, info = scenes
    W, H = bigscene.PROBE_SIZE
    assert info["probe"].shape == (H, W, 4) and info["tris"] > 4096
    snap = tb.Snapshot(paths["env_like"])
    sky = snap.scene.contents.sky
    assert sky.probeValid and (sky.probeWidth, sky.probeHeight) == (W, H)
    pdf_x, cdf_x, pdf_y, cdf_y, slack = bigscene.probe_tables(sky)
    want = bigscene.build_cdf(info["probe"])
    for name, got, exp in zip(("pdfX", "cdfX", "pdfY", "cdfY"), (pdf_x, cdf_x, pdf_y, cdf_y), want):
        same = (got.view(np.uint32) == exp.view(np.uint32)) | (np.isnan(got) & np.isnan(exp))
        assert same.all(), "%s: %d values differ from BuildCDF" % (name, int((~same).sum()))
    assert not slack.any()
    snap.close()
    black = np.isnan(cdf_x).any(1)
    assert black.any() and np.isnan(cdf_x[black]).all() and (info["probe"][black, :, :3] == 0).all()
    lit = ~black
    cx = cdf_x[lit].astype(np.float64)
    assert (np.diff(cx, axis=1) >= 0).all() and (np.diff(cdf_y.astype(np.float64)) >= 0).all()
    ulp = np.spacing(np.float32(1.0))
    assert (np.abs(cx[:, -1] - 1.0) <= ulp).all() and abs(float(cdf_y[-1]) - 1.0) <= ulp
    # each pdf is a weight over its row's float32 running sum, whose n additions may each round by 2^-24: a row of
    # 4000 texels sums to 1 within about 2.4e-4 only, not 1e-5 (the rows here deviate by up to 9e-5)
    u = 2.0 ** -24
    row_err = np.abs(pdf_x[lit].astype(np.float64).sum(1) - 1.0).max()
    y_err = abs(pdf_y.astype(np.float64).sum() - 1.0)
    joint_err = abs((pdf_x[lit].astype(np.float64) * pdf_y[lit, None].astype(np.float64)).sum() - 1.0)
    assert row_err <= (W + 2) * u and y_err <= (H + 2) * u and joint_err <= (W + H + 4) * u, (row_err, y_err, joint_err)
    runs = bigscene.equal_runs(cdf_x)
    assert runs > 0
    print("env_like: %dx%d probe, %d black rows, %d equal neighbours in cdfX, pdf sums off 1 by %.1e (row), %.1e (rows), "
          "%.1e (joint); glass mesh of %d triangles; generated in %.1f s" % (
              W, H, int(black.sum()), runs, row_err, y_err, joint_err, info["tris"], info["seconds"]))
