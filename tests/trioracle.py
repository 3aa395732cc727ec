"""TEST INFRASTRUCTURE: the CPU restatement's closest hit with the hit triangle over a whole batch of rays
(tests/trace_rays_tri_oracle.cpp), the arm the device's tb200_trace_rays_tri is checked against.  Built like
tests/rayoracle.py, with the same flags, into a temporary directory keyed by the sources' hash; the library also
holds rayoracle's entry points, so TriOracle is a RayOracle over it."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tinsel_b200 import abi
import rayoracle

ROOT = rayoracle.ROOT
SOURCES = [os.path.join(ROOT, "tests", "trace_rays_tri_oracle.cpp"), os.path.join(ROOT, "tinsel_b200", "csrc", "snapshot.cpp")]
DEPS = SOURCES + rayoracle.DEPS

_lib = None


def library_path():
    h = hashlib.sha1(" ".join([rayoracle.CXX] + rayoracle.FLAGS).encode())
    for p in DEPS:
        with open(p, "rb") as f:
            h.update(f.read())
    return os.path.join(tempfile.gettempdir(), "tinsel_b200_trioracle_%s.so" % h.hexdigest()[:16])


def load():
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        tmp = "%s.%d.tmp" % (path, os.getpid())
        subprocess.check_call([rayoracle.CXX, *rayoracle.FLAGS, "-I", ROOT, "-I", os.path.join(ROOT, "include"), "-o", tmp,
                               *SOURCES])
        os.replace(tmp, path)
    lib = C.CDLL(path)
    lib.oracle_create.restype = C.c_void_p
    lib.oracle_create.argtypes = [C.POINTER(abi.Scene)]
    lib.oracle_destroy.argtypes = [C.c_void_p]
    lib.oracle_trace_rays.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_longlong, C.POINTER(C.c_float),
                                      C.POINTER(C.c_int32), C.c_int]
    lib.oracle_trace_rays_tri.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_longlong, C.POINTER(C.c_float),
                                          C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int]
    abi.declare_snapshot_api(lib)
    _lib = lib
    return lib


class TriOracle(rayoracle.RayOracle):
    """RayOracle over this library, plus trace_rays_tri(rays (N, 8) float32) -> (hits (N, 4), prims (N,), tri (N,),
    uvw (N, 3) float32), the shapes and meaning of Renderer.trace_rays_tri."""

    def __init__(self, scene_ptr, keepalive=None):
        self.lib = load()
        h = self.lib.oracle_create(scene_ptr)
        if not h:
            raise RuntimeError("the CPU restatement refused the scene: a BVH is not a tree or is too deep for its stack")
        self.h = C.c_void_p(h)
        self._keep = keepalive
        self._snap = None

    @classmethod
    def from_snapshot(cls, path):
        lib = load()
        snap = lib.tb200_snapshot_load(path.encode())
        if not snap:
            raise RuntimeError("cannot load " + path)
        o = cls(lib.tb200_snapshot_scene(snap))
        o._snap = snap
        return o

    def trace_rays_tri(self, rays, nthreads=None):
        rays = np.ascontiguousarray(rays, np.float32).reshape(-1, 8)
        hits = np.zeros((len(rays), 4), np.float32)
        prims = np.zeros(len(rays), np.int32)
        tris = np.zeros((len(rays), 4), np.int32)
        self.lib.oracle_trace_rays_tri(self.h, rays.ctypes.data_as(C.POINTER(C.c_float)), len(rays),
                                       hits.ctypes.data_as(C.POINTER(C.c_float)), prims.ctypes.data_as(C.POINTER(C.c_int32)),
                                       tris.ctypes.data_as(C.POINTER(C.c_int32)), nthreads or os.cpu_count() or 1)
        return hits, prims, tris[:, 0], tris[:, 1:].view(np.float32)


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
