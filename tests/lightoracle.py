"""TEST INFRASTRUCTURE: the CPU restatement's SampleLights over a batch of surface records and its PathTrace with a
seed per call (tests/light_oracle.cpp), the arms the device's next-event-estimation query and a path built from the
queries are checked against.  The library is compiled on first use, with oracle/Makefile's flags, from the
restatement's unchanged source, into a temporary directory keyed by the sources' hash (the repository tree may be
read-only).  Besides its own two functions it exports every entry point of the restatement (oracle_sky_eval,
oracle_primitive_sample, ...)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tinsel_b200 import abi
import rayoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = [os.path.join(ROOT, "tests", "light_oracle.cpp"), os.path.join(ROOT, "tinsel_b200", "csrc", "snapshot.cpp")]
DEPS = SOURCES + [os.path.join(ROOT, "oracle", "tinsel_oracle.cpp"), os.path.join(ROOT, "include", "tinsel_b200.h"),
                  os.path.join(ROOT, "include", "tb200_detmath.h")]

_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int32)
_u32p = C.POINTER(C.c_uint32)
_lib = None


def library_path():
    h = hashlib.sha1(" ".join([rayoracle.CXX] + rayoracle.FLAGS).encode())
    for p in DEPS:
        with open(p, "rb") as f:
            h.update(f.read())
    return os.path.join(tempfile.gettempdir(), "tinsel_b200_lightoracle_%s.so" % h.hexdigest()[:16])


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
    lib.oracle_sample_lights.argtypes = [C.POINTER(abi.Scene), C.c_longlong, C.c_void_p, _u32p, _f32p]
    lib.oracle_path_trace_reseeded.argtypes = [C.POINTER(abi.Scene), C.c_longlong, _f32p, _f32p, _f32p, C.c_int, _u32p,
                                               _f32p, _i32p, _i32p]
    lib.oracle_create.restype = C.c_void_p
    lib.oracle_create.argtypes = [C.POINTER(abi.Scene)]
    lib.oracle_destroy.argtypes = [C.c_void_p]
    lib.oracle_sky_eval.argtypes = [C.c_void_p, _f32p, _f32p, _f32p]
    lib.oracle_primitive_sample.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_int, _f32p, _f32p, _f32p]
    abi.declare_snapshot_api(lib)
    _lib = lib
    return lib


def _fp(a):
    return a.ctypes.data_as(_f32p)


def sample_lights(scene_ptr, records, seeds):
    """The restatement's SampleLights of every tb200_light_query record ((n, 16) float32 rows, as
    tinsel_b200.light_queries packs them) from Random(seeds[k]): (n, 3) float32."""
    records = np.ascontiguousarray(records, np.float32).reshape(-1, 16)
    seeds = np.ascontiguousarray(seeds).view(np.uint32).reshape(-1)
    assert seeds.shape[0] == records.shape[0]
    out = np.zeros((records.shape[0], 3), np.float32)
    load().oracle_sample_lights(scene_ptr, records.shape[0], records.ctypes.data_as(C.c_void_p),
                                seeds.ctypes.data_as(_u32p), _fp(out))
    return out


def path_trace_reseeded(scene_ptr, origin, direction, time, max_depth, seeds):
    """The restatement's PathTrace of n rays with bounce b's SampleLights drawing from Random(seeds[k, b, 0]) and its
    BSDFSample from Random(seeds[k, b, 1]); seeds: (n, max_depth, 2) 32-bit integers.  Returns (radiance (n, 3)
    float32, length (n,) int32: the Trace calls made, prims (n, max_depth) int32: each bounce's hit primitive, -1 on
    a miss, -2 after the path ended)."""
    origin = np.ascontiguousarray(origin, np.float32).reshape(-1, 3)
    direction = np.ascontiguousarray(direction, np.float32).reshape(-1, 3)
    time = np.ascontiguousarray(time, np.float32).reshape(-1)
    n = origin.shape[0]
    seeds = np.ascontiguousarray(seeds).view(np.uint32).reshape(n, max_depth, 2)
    rad = np.zeros((n, 3), np.float32)
    length = np.zeros(n, np.int32)
    prims = np.zeros((n, max_depth), np.int32)
    load().oracle_path_trace_reseeded(scene_ptr, n, _fp(origin), _fp(direction), _fp(time), max_depth,
                                      seeds.ctypes.data_as(_u32p), _fp(rad), length.ctypes.data_as(_i32p),
                                      prims.ctypes.data_as(_i32p))
    return rad, length, prims


def sky_eval(scene_ptr, dirs):
    """The restatement's Sky::Eval and ProbePdf (0 without a probe) of every direction: (n, 4) float32."""
    lib = load()
    h = lib.oracle_create(scene_ptr)
    assert h, "the restatement refused the scene"
    dirs = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
    out = np.zeros((dirs.shape[0], 4), np.float32)
    c, p = np.zeros(3, np.float32), np.zeros(1, np.float32)
    for k in range(dirs.shape[0]):
        lib.oracle_sky_eval(h, _fp(dirs[k]), _fp(c), _fp(p))
        out[k, :3], out[k, 3] = c, p[0]
    lib.oracle_destroy(h)
    return out


def primitive_areas(scene_ptr):
    """The restatement's prim_area of every primitive, as oracle_primitive_sample returns it: (numPrimitives,)
    float32."""
    lib = load()
    h = lib.oracle_create(scene_ptr)
    assert h, "the restatement refused the scene"
    n = scene_ptr.contents.numPrimitives
    out = np.zeros(n, np.float32)
    pos, nrm, a = np.zeros(3, np.float32), np.zeros(3, np.float32), np.zeros(1, np.float32)
    for i in range(n):
        lib.oracle_primitive_sample(h, i, 0.0, 1, _fp(pos), _fp(nrm), _fp(a))
        out[i] = a[0]
    lib.oracle_destroy(h)
    return out
