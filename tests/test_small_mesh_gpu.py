"""Meshes whose BVH is one leaf or one interior pair over two leaves (a quad: cornell's light) are walked inline
without the traversal stack, and transforms whose rotation is exactly (+0, +0, +0, +1) skip the quaternion
arithmetic (tb_math.cuh: rotate_xf).  Both are exact: per sample in both pipelines against the CPU restatement,
and per ray through the batched closest-hit and occlusion queries, for quads that are unrotated, rotated, scaled, or carry a -0 quaternion
component, beside a one-triangle mesh, a bent quad whose triangles' boxes differ (the near-first swap) and a mesh
too deep for the inline walk.  Rays aimed at the quads' shared diagonal, where the two triangles tie in t, and
rays along it in the quad's plane, are traced on their own."""
import os
import subprocess

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import fuzzscene
import occlusionsets
import rayoracle
import raysets
import refdrv

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q_ROT = np.array([0.3, -0.5, 0.2, 0.78], np.float64) / np.linalg.norm([0.3, -0.5, 0.2, 0.78])
VARIANTS = {
    "unrotated": ((0.0, 0.0, 0.0, 1.0), 1.0),
    "rotated": (tuple(Q_ROT), 1.0),
    "scaled": ((0.0, 0.0, 0.0, 1.0), 0.625),
    "negzero": ((-0.0, 0.0, 0.0, 1.0), 1.0),
    "negzero_y": ((0.0, -0.0, 0.0, 1.0), 1.0),
}


def _quad(half, bend=0.0):
    """Two triangles over [-half, half]^2 in z = 0 sharing the diagonal from vertex 0 to vertex 3; `bend` lifts
    vertex 1 and lowers vertex 2, so that the triangles' boxes differ.  Vertex normals differ per vertex."""
    p = np.array([[-half, -half, 0.0], [half, -half, bend], [-half, half, -bend], [half, half, 0.0]])
    n = np.array([[0.1, 0.0, 1.0], [0.0, 0.2, 1.0], [-0.2, 0.1, 1.0], [0.0, -0.1, 1.0]])
    return fuzzscene.MeshData(p, n / np.linalg.norm(n, axis=1, keepdims=True), np.array([[0, 1, 3], [0, 3, 2]]))


def _triangle():
    p = np.array([[-0.4, -0.3, 0.0], [0.5, -0.2, 0.1], [0.0, 0.45, -0.1]])
    return fuzzscene.MeshData(p, np.tile([0.0, 0.0, 1.0], (3, 1)), np.array([[0, 1, 2]]))


def _make_scene(path, variant, seed=0):
    """Floor, a quad light above, a flat quad, a bent quad, a one-triangle mesh, an 8-triangle grid (walked with
    the stack) and a diffuse sphere.  Every mesh carries the variant's rotation and scale."""
    q, s = VARIANTS[variant]
    rng = np.random.RandomState(seed)
    g = fuzzscene._grid(2)
    meshes = [_quad(0.5), _quad(0.6), _quad(0.5, bend=0.25), _triangle(), fuzzscene.MeshData(g[0] * 0.5, g[1], g[2])]
    prims = (abi.Primitive * 7)()
    bounds = [fuzzscene._floor(prims[0], rng)]
    placement = [(0.0, 2.4, -0.5), (-1.1, 1.0, -0.8), (0.9, 1.1, -0.6), (0.0, 0.6, 0.4), (-0.2, 1.6, -1.4)]
    for k, (m, pos) in enumerate(zip(meshes, placement)):
        pr = prims[1 + k]
        pr.material = fuzzscene._material(rng, k == 0)
        pr.material.transmission = 0.0
        pr.lightSamples = 1 if k == 0 else 0
        bounds.append(fuzzscene._instance(pr, k, m, pos, q, s))
    bounds.append(fuzzscene._sphere(prims[6], (1.2, 0.4, 0.5), 0.35, fuzzscene._material(rng, False)))
    tree = fuzzscene._build_bvh(bounds)
    fuzzscene._save(rng, path, prims, tree, meshes, 96, 64)
    return meshes, placement, q, s


def _rotate(q, v):
    x, y, z, w = q
    u = np.array([x, y, z])
    t = 2.0 * np.cross(u, v)
    return v + w * t + np.cross(u, t)


def _diagonal_rays(mesh, pos, q, s, origin, rng, n=2048):
    """Rays from `origin` to points of the quad's shared diagonal, and rays along the diagonal in the quad's plane."""
    a, c = mesh.pos[0].astype(np.float64), mesh.pos[3].astype(np.float64)
    k = rng.uniform(0.0, 1.0, n)
    k[:4] = [0.0, 0.25, 0.5, 1.0]
    world = np.array([_rotate(q, s * (a + (c - a) * kk)) + pos for kk in k])
    d = world - np.asarray(origin, np.float64)
    aim = raysets.pack(np.tile(np.asarray(origin, np.float32), (n, 1)), (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32),
                       np.full(n, 0.5, np.float32))
    along = _rotate(q, c - a)
    along = along / np.linalg.norm(along)
    starts = np.array([_rotate(q, s * (a + (a - c) * kk)) + pos for kk in rng.uniform(0.05, 1.0, 64)])
    flat = raysets.pack(starts.astype(np.float32), np.tile(along.astype(np.float32), (64, 1)), np.full(64, 0.5, np.float32))
    return np.concatenate([aim, flat])


@pytest.fixture(scope="module", autouse=True)
def port_built():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "port"])


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_small_meshes_per_sample(variant, tmp_path):
    path = str(tmp_path / "s.tsnap")
    _make_scene(path, variant)
    port = refdrv.PortScene.from_snapshot(path)
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    lit = 0.0
    try:
        for pipeline in ("mega", "wavefront"):
            os.environ["TINSEL_B200_PIPELINE"] = pipeline
            r = tb.Renderer(snap.scene)
            r.Init(opt.width, opt.height)
            for frame in (0, 3):
                rad, ras = r.trace_frame(cam, opt, frame)
                prad, pras = port.trace_frame(frame, 8)
                assert np.array_equal(ras, pras)
                same = (rad.view(np.uint32) == prad.view(np.uint32)) | (np.isnan(rad) & np.isnan(prad))
                bad = int((~same.all(-1)).sum())
                assert bad == 0, "%s/%s frame %d: %d of %d samples differ" % (variant, pipeline, frame, bad, rad.shape[0] * rad.shape[1])
                lit += float(np.nan_to_num(rad).sum())
            r.close()
    finally:
        os.environ.pop("TINSEL_B200_PIPELINE", None)
    assert lit > 0.0
    port.close()
    snap.close()


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_small_meshes_per_ray(variant, tmp_path):
    import torch
    path = str(tmp_path / "s.tsnap")
    meshes, placement, q, s = _make_scene(path, variant)
    snap = tb.Snapshot(path)
    port = rayoracle.RayOracle.from_snapshot(path)
    r = tb.Renderer(snap.scene)
    rng = np.random.RandomState(7)
    cam = raysets.camera_rays(snap.camera, 1 << 15, rng)
    h, p = port.trace_rays(cam)
    sets = {"camera": cam, "random": raysets.random_rays(snap.scene.contents, 1 << 15, rng), "secondary": raysets.secondary_rays(cam, h, p, rng)}
    for k in range(3):   # the light, the flat quad, the bent quad
        pos = np.array(placement[k])
        sets["diagonal%d" % k] = _diagonal_rays(meshes[k], pos, q, s, (0.0, 1.2, 6.0), rng)
        sets["diagonal%d_below" % k] = _diagonal_rays(meshes[k], pos, q, s, pos + (0.3, -0.6, 0.9), rng)
    hit_meshes = set()
    for what, rays in sets.items():
        hits, prims = r.trace_rays(torch.from_numpy(np.ascontiguousarray(rays)).cuda())
        hits, prims = hits.cpu().numpy(), prims.cpu().numpy()
        want_h, want_p = port.trace_rays(rays)
        bad = raysets.mismatches(hits, prims, want_h, want_p)
        assert len(bad) == 0, "%s/%s: %d of %d rays differ; first ray %s: device %s %s, port %s %s" % (
            variant, what, len(bad), len(rays), rays[bad[0]], prims[bad[0]], hits[bad[0]], want_p[bad[0]], want_h[bad[0]])
        hit_meshes.update(int(x) for x in np.unique(prims))
        tmax_sets = occlusionsets.tmax_sets(want_h, want_p, rng)
        for name in ("inf", "t", "t_up", "t_down"):
            sub = occlusionsets.with_tmax(rays, tmax_sets[name])
            got = r.occluded(torch.from_numpy(np.ascontiguousarray(sub)).cuda()).cpu().numpy()
            want = occlusionsets.occluded(want_h, want_p, tmax_sets[name])
            bad = np.nonzero(got != want)[0]
            assert len(bad) == 0, "%s/%s/tmax=%s: %d of %d occlusion verdicts differ; first ray %s: device %s, port %s (prim %d, t %r)" % (
                variant, what, name, len(bad), len(rays), sub[bad[0]], got[bad[0]], want[bad[0]], want_p[bad[0]], float(want_h[bad[0], 0]))
    assert {1, 2, 3, 4, 5} <= hit_meshes, hit_meshes   # every mesh was hit
    r.close()
    port.close()
    snap.close()
