"""TEST INFRASTRUCTURE: checks of tb200_trace_rays_tri's triangle records that need no restatement (the restatement's
own records come from rayoracle.RayOracle.trace_rays_tri)."""
import ctypes as C

import numpy as np

from tinsel_b200 import abi


def _rotate(q, v):
    """q v q* for the quaternions q (N, 4) = (x, y, z, w), normalised here, and vectors v (N, 3), in float64."""
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    u, w = q[:, :3], q[:, 3:4]
    t = 2.0 * np.cross(u, v)
    return v + w * t + np.cross(u, t)


def check_semantics(scene, rays, hits, prims, tri, uvw, what=""):
    """Checks what tb200_trace_rays_tri promises about tri / uvw without the restatement, and returns the number of
    mesh hits and of sphere or plane hits.  Everywhere: tri = -1 and u = v = w = +0 unless a mesh was hit.  On mesh
    hits: tri indexes the mesh, u == (1 - v) - w in float32, and u, v, w lie in [0, 1].  On mesh hits of primitives
    whose transform does not move: u*A + v*B + w*C, transformed, is the hit point o + t*d to a relative 2e-5, and
    u*N0 + v*N1 + w*N2, transformed, normalised and face-forwarded, is the returned normal to 1e-6 (8 ulps of 1)."""
    n = len(rays)
    prim_arr = C.cast(scene.primitives, C.POINTER(abi.Primitive * scene.numPrimitives)).contents
    types = np.array([p.type for p in prim_arr] + [-1], np.int32)[prims]   # prims == -1 picks the -1 appended
    mesh = types == abi.MESH
    bits = uvw.view(np.uint32)
    assert (tri[~mesh] == -1).all() and (bits[~mesh] == 0).all(), what + ": a triangle record off a mesh hit"
    u, v, w = uvw[:, 0], uvw[:, 1], uvw[:, 2]
    assert (u[mesh].view(np.uint32) == ((np.float32(1.0) - v[mesh]) - w[mesh]).view(np.uint32)).all(), what + ": u != 1 - v - w"
    assert ((uvw[mesh] >= 0.0) & (uvw[mesh] <= 1.0)).all(), what + ": a weight outside [0, 1]"

    for k, p in enumerate(prim_arr):
        sel = np.nonzero(prims == k)[0]
        if p.type != abi.MESH or len(sel) == 0:
            continue
        m = scene.meshes[p.mesh]
        ntris = m.numIndices // 3
        assert ((tri[sel] >= 0) & (tri[sel] < ntris)).all(), what + ": a triangle index outside the mesh"
        if bytes(p.start) != bytes(p.end):
            continue
        idx = np.ctypeslib.as_array(m.indices, (ntris, 3))[tri[sel]]
        pos = np.ctypeslib.as_array(m.positions, (m.numVertices, 3)).astype(np.float64)
        nrm = np.ctypeslib.as_array(m.normals, (m.numVertices, 3)).astype(np.float64)
        wts = uvw[sel].astype(np.float64)
        q = np.tile(np.array(p.start.r[:], np.float64), (len(sel), 1))
        local = sum(wts[:, j:j + 1] * pos[idx[:, j]] for j in range(3))
        world = np.array(p.start.p[:], np.float64) + _rotate(q, local * p.start.s)
        r = rays[sel].astype(np.float64)
        want = r[:, 0:3] + r[:, 4:7] * hits[sel, 0:1].astype(np.float64)
        scale = np.linalg.norm(r[:, 0:3], axis=1) + np.linalg.norm(want, axis=1) + 1e-3
        err = np.linalg.norm(world - want, axis=1) / scale
        assert err.max() < 2e-5, "%s: hit point off by %g (prim %d)" % (what, err.max(), k)
        s = _rotate(q, sum(wts[:, j:j + 1] * nrm[idx[:, j]] for j in range(3)))
        length = np.linalg.norm(s, axis=1, keepdims=True)
        s = s / np.maximum(length, 1e-300)
        face = np.sum(s * -r[:, 4:7], axis=1)
        s = np.where(face[:, None] < 0.0, -s, s)
        # where the smooth normal is close to 0 (normalize's fallback) or to the ray's plane (face-forward's sign),
        # float32 rounding may decide differently than float64: only well-conditioned hits are compared
        ok = (length[:, 0] > 1e-3) & (np.abs(face) > 1e-3 * np.linalg.norm(r[:, 4:7], axis=1))
        nerr = np.abs(s[ok] - hits[sel][ok, 1:4]).max() if ok.any() else 0.0
        assert nerr < 1e-6, "%s: normal off by %g (prim %d)" % (what, nerr, k)
    return int(mesh.sum()), int(((types == abi.SPHERE) | (types == abi.PLANE)).sum())
