"""TEST INFRASTRUCTURE: the CPU restatement's Trace over a whole batch of rays (tests/trace_rays_oracle.cpp), the arm
the device's closest-hit queries are checked against.  The library is compiled on first use, with oracle/Makefile's
flags, from the restatement's unchanged source, into a temporary directory keyed by the sources' hash (the
repository tree may be read-only)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tinsel_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = [os.path.join(ROOT, "tests", "trace_rays_oracle.cpp"), os.path.join(ROOT, "tinsel_b200", "csrc", "snapshot.cpp")]
DEPS = SOURCES + [os.path.join(ROOT, "oracle", "tinsel_oracle.cpp"), os.path.join(ROOT, "include", "tinsel_b200.h"),
                  os.path.join(ROOT, "include", "tb200_detmath.h")]
# oracle/Makefile's CXXFLAGS (the restatement's numerics depend on them), plus -Bsymbolic as for its other libraries
FLAGS = ["-O2", "-DNDEBUG", "-w", "-fPIC", "-std=c++17", "-ffp-contract=off", "-pthread", "-shared", "-Wl,-Bsymbolic"]
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"

_lib = None


def library_path():
    h = hashlib.sha1(" ".join([CXX] + FLAGS).encode())
    for p in DEPS:
        with open(p, "rb") as f:
            h.update(f.read())
    return os.path.join(tempfile.gettempdir(), "tinsel_b200_rayoracle_%s.so" % h.hexdigest()[:16])


def load():
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        tmp = "%s.%d.tmp" % (path, os.getpid())
        subprocess.check_call([CXX, *FLAGS, "-I", ROOT, "-I", os.path.join(ROOT, "include"), "-o", tmp, *SOURCES])
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


class RayOracle:
    """The restatement over a tb200_scene; trace_rays(rays (N, 8) float32) -> (hits (N, 4), prims (N,)), and
    trace_rays_tri(rays) -> (hits, prims, tri (N,), uvw (N, 3) float32), the shapes and meaning of
    Renderer.trace_rays_tri."""

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

    def trace_rays(self, rays, nthreads=None):
        rays = np.ascontiguousarray(rays, np.float32).reshape(-1, 8)
        hits = np.zeros((len(rays), 4), np.float32)
        prims = np.zeros(len(rays), np.int32)
        self.lib.oracle_trace_rays(self.h, rays.ctypes.data_as(C.POINTER(C.c_float)), len(rays),
                                   hits.ctypes.data_as(C.POINTER(C.c_float)), prims.ctypes.data_as(C.POINTER(C.c_int32)),
                                   nthreads or os.cpu_count() or 1)
        return hits, prims

    def trace_rays_tri(self, rays, nthreads=None):
        rays = np.ascontiguousarray(rays, np.float32).reshape(-1, 8)
        hits = np.zeros((len(rays), 4), np.float32)
        prims = np.zeros(len(rays), np.int32)
        tris = np.zeros((len(rays), 4), np.int32)
        self.lib.oracle_trace_rays_tri(self.h, rays.ctypes.data_as(C.POINTER(C.c_float)), len(rays),
                                       hits.ctypes.data_as(C.POINTER(C.c_float)), prims.ctypes.data_as(C.POINTER(C.c_int32)),
                                       tris.ctypes.data_as(C.POINTER(C.c_int32)), nthreads or os.cpu_count() or 1)
        return hits, prims, tris[:, 0], tris[:, 1:].view(np.float32)

    def close(self):
        if self.h:
            self.lib.oracle_destroy(self.h)
            self.h = None
        if self._snap:
            self.lib.tb200_snapshot_free(self._snap)
            self._snap = None
