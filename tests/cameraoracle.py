"""TEST INFRASTRUCTURE: the CPU restatement's camera samples over a batch of (pixel, frame) records
(tests/camera_oracle.cpp), the arm the device's camera-ray query is checked against.  The library is compiled on first
use, with oracle/Makefile's flags, from the restatement's unchanged source, into a temporary directory keyed by the
sources' hash (the repository tree may be read-only).  Besides oracle_camera_samples it exports every entry point of
the restatement, so a test can check the samples against that same build's trace_frame and generate_ray."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tinsel_b200 import abi
import rayoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = [os.path.join(ROOT, "tests", "camera_oracle.cpp"), os.path.join(ROOT, "tinsel_b200", "csrc", "snapshot.cpp")]
DEPS = SOURCES + [os.path.join(ROOT, "oracle", "tinsel_oracle.cpp"), os.path.join(ROOT, "include", "tinsel_b200.h"),
                  os.path.join(ROOT, "include", "tb200_detmath.h")]

_f32p = C.POINTER(C.c_float)
_lib = None


def library_path():
    h = hashlib.sha1(" ".join([rayoracle.CXX] + rayoracle.FLAGS).encode())
    for p in DEPS:
        with open(p, "rb") as f:
            h.update(f.read())
    return os.path.join(tempfile.gettempdir(), "tinsel_b200_cameraoracle_%s.so" % h.hexdigest()[:16])


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
    lib.oracle_camera_samples.argtypes = [C.POINTER(abi.Camera), C.c_int, C.c_int, C.c_longlong, C.POINTER(C.c_int32),
                                          _f32p, _f32p, _f32p, _f32p]
    lib.oracle_create.restype = C.c_void_p
    lib.oracle_create.argtypes = [C.POINTER(abi.Scene)]
    lib.oracle_destroy.argtypes = [C.c_void_p]
    lib.oracle_trace_frame.argtypes = [C.c_void_p, C.POINTER(abi.Camera), C.POINTER(abi.Options), C.c_int, _f32p, _f32p,
                                       C.c_int]
    lib.oracle_generate_ray.argtypes = [C.POINTER(abi.Camera), C.c_int, C.c_int, C.c_float, C.c_float, _f32p, _f32p]
    abi.declare_snapshot_api(lib)
    _lib = lib
    return lib


def _fp(a):
    return a.ctypes.data_as(_f32p)


def camera_samples(camera, width, height, samples):
    """The restatement's camera samples (trace_sample's draws and ray) of `samples`, (n, 2) int32 (pixel, frame)
    records of a width x height image: (origin (n, 3), dir (n, 3), time (n,), raster (n, 2)), float32.  A pixel
    outside [0, width*height) gives zeros and a NaN raster."""
    samples = np.ascontiguousarray(samples, np.int32).reshape(-1, 2)
    n = samples.shape[0]
    origin, d = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float32)
    time, raster = np.zeros(n, np.float32), np.zeros((n, 2), np.float32)
    load().oracle_camera_samples(C.byref(camera), width, height, n, samples.ctypes.data_as(C.POINTER(C.c_int32)),
                                 _fp(origin), _fp(d), _fp(time), _fp(raster))
    return origin, d, time, raster


def trace_frame(scene_ptr, camera, options, frame, nthreads=4):
    """This build's oracle_trace_frame: (radiance (H, W, 3), raster (H, W, 2)) of every pixel's sample in `frame`."""
    lib = load()
    h = lib.oracle_create(scene_ptr)
    assert h, "the restatement refused the scene"
    rad = np.zeros((options.height, options.width, 3), np.float32)
    ras = np.zeros((options.height, options.width, 2), np.float32)
    lib.oracle_trace_frame(h, C.byref(camera), C.byref(options), frame, _fp(rad), _fp(ras), nthreads)
    lib.oracle_destroy(h)
    return rad, ras


def generate_ray(camera, width, height, x, y):
    """This build's oracle_generate_ray through raster position (x, y): (origin (3,), dir (3,)) float32."""
    o, d = np.zeros(3, np.float32), np.zeros(3, np.float32)
    load().oracle_generate_ray(C.byref(camera), width, height, float(x), float(y), _fp(o), _fp(d))
    return o, d
