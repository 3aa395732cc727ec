"""TEST INFRASTRUCTURE: the CPU restatement's PrimitiveSample and ProbeSample over a batch and its SampleLights with a
seed per slot (tests/emitter_oracle.cpp), the arms the device's emitter and probe sample queries and a SampleLights
built from them are checked against; the restatement's single-call oracle_primitive_sample and oracle_probe_sample;
and seeds whose Random draws are exactly 0.0 or 1.0.  The library is compiled on first use, with oracle/Makefile's
flags, from the restatement's unchanged source, into a temporary directory keyed by the sources' hash (the repository
tree may be read-only)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tinsel_b200 import abi
import rayoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = [os.path.join(ROOT, "tests", "emitter_oracle.cpp"), os.path.join(ROOT, "tinsel_b200", "csrc", "snapshot.cpp")]
DEPS = SOURCES + [os.path.join(ROOT, "oracle", "tinsel_oracle.cpp"), os.path.join(ROOT, "include", "tinsel_b200.h"),
                  os.path.join(ROOT, "include", "tb200_detmath.h")]

# Seeds whose Random draws are exactly 0.0 or 1.0 (Randf can return 1.0: the largest uint32 values round up to 2^32),
# found by an exhaustive search: {(draw index, value): seed}
EDGE_SEEDS = {(0, 0.0): 3569454725, (0, 1.0): 31056728, (1, 0.0): 2426648011, (1, 1.0): 32418902,
              (2, 0.0): 1389320875, (2, 1.0): 6778759, (3, 0.0): 1848853012, (3, 1.0): 39639462}
# more seeds whose second draw is 1.0: ProbeSample's column search returns col == width in every row whose CDF ends
# below 1 (build_probe_tables' slack element is there for the last row)
COL_END_SEEDS = [32418902, 65966622, 95789306, 110558804, 220241688, 379624053, 410227903, 452831547]

_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int32)
_u32p = C.POINTER(C.c_uint32)
_lib = None


def library_path():
    h = hashlib.sha1(" ".join([rayoracle.CXX] + rayoracle.FLAGS).encode())
    for p in DEPS:
        with open(p, "rb") as f:
            h.update(f.read())
    return os.path.join(tempfile.gettempdir(), "tinsel_b200_emitteroracle_%s.so" % h.hexdigest()[:16])


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
    lib.oracle_sample_emitters.argtypes = [C.POINTER(abi.Scene), C.c_longlong, C.c_void_p, _u32p, _f32p]
    lib.oracle_sample_probe.argtypes = [C.POINTER(abi.Scene), C.c_longlong, _u32p, _f32p]
    lib.oracle_sample_lights_per_slot.argtypes = [C.POINTER(abi.Scene), C.c_longlong, C.c_void_p, _u32p, C.c_int, _f32p,
                                                  _i32p]
    lib.oracle_create.restype = C.c_void_p
    lib.oracle_create.argtypes = [C.POINTER(abi.Scene)]
    lib.oracle_destroy.argtypes = [C.c_void_p]
    lib.oracle_primitive_sample.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_int, _f32p, _f32p, _f32p]
    lib.oracle_probe_sample.argtypes = [C.c_void_p, C.c_int, _f32p, _f32p, _f32p]
    _lib = lib
    return lib


def randf(seed, k):
    """The first k Randf draws of Random(seed) (src/maths.h:1036-1076), as float32."""
    s1 = (315645664 + int(seed)) & 0xffffffff
    s2 = s1 ^ 0x13ab45fe
    out = []
    for _ in range(k):
        a, b = s1, s2
        s1 = (b ^ (((a << 5) | (a >> 27)) & 0xffffffff)) ^ ((a * b) & 0xffffffff)
        s2 = s1 ^ (((b << 12) | (b >> 20)) & 0xffffffff)
        out.append(np.float32(s1) * np.float32(2.3283064365386963e-10))
    return out


def _fp(a):
    return a.ctypes.data_as(_f32p)


def _seeds(seeds, n):
    seeds = np.ascontiguousarray(seeds).view(np.uint32).reshape(-1)
    assert seeds.shape[0] == n
    return seeds


def sample_emitters(scene_ptr, records, seeds):
    """The restatement's PrimitiveSample of every tb200_emitter_query record ((n, 2) float32 rows, as
    tinsel_b200.emitter_queries packs them) from Random(seeds[k]): (n, 8) float32 rows pos, 0, normal, 0; zeros for a
    primitive that is not a light or lies outside the scene."""
    records = np.ascontiguousarray(records, np.float32).reshape(-1, 2)
    seeds = _seeds(seeds, records.shape[0])
    out = np.zeros((records.shape[0], 8), np.float32)
    load().oracle_sample_emitters(scene_ptr, records.shape[0], records.ctypes.data_as(C.c_void_p),
                                  seeds.ctypes.data_as(_u32p), _fp(out))
    return out


def sample_probe(scene_ptr, seeds):
    """The restatement's ProbeSample from Random(seed) of every seed: (n, 8) float32 rows dir, pdf, color, 0; zeros
    without a probe."""
    seeds = np.ascontiguousarray(seeds).view(np.uint32).reshape(-1)
    out = np.zeros((seeds.shape[0], 8), np.float32)
    load().oracle_sample_probe(scene_ptr, seeds.shape[0], seeds.ctypes.data_as(_u32p), _fp(out))
    return out


def num_slots(scene):
    """SampleLights' slots: the probe sample when the sky has a probe, then every light sample."""
    return int(bool(scene.sky.probeValid)) + sum(max(scene.primitives[i].lightSamples, 0) for i in range(scene.numPrimitives))


def sample_lights_per_slot(scene_ptr, records, seeds):
    """The restatement's SampleLights of every tb200_light_query record with slot s of record k drawing from
    Random(seeds[k, s]); seeds: (n, num_slots) 32-bit integers.  Returns (radiance (n, 3) float32, hit (n, num_slots)
    int32: each slot's shadow-ray hit primitive, -1 on a miss, -2 when nothing was traced, accepted (n, num_slots)
    bool: whether the slot's sample reached the BSDF evaluation)."""
    records = np.ascontiguousarray(records, np.float32).reshape(-1, 16)
    n, m = records.shape[0], num_slots(scene_ptr.contents)
    seeds = _seeds(seeds, n * m)
    rad = np.zeros((n, 3), np.float32)
    slots = np.zeros((n, m, 2), np.int32)
    load().oracle_sample_lights_per_slot(scene_ptr, n, records.ctypes.data_as(C.c_void_p), seeds.ctypes.data_as(_u32p), m,
                                         _fp(rad), slots.ctypes.data_as(_i32p))
    return rad, slots[..., 0], slots[..., 1] != 0


def primitive_sample(scene_ptr, prim, time, seed):
    """The restatement's single-call oracle_primitive_sample: (pos (3,), normal (3,)) float32."""
    lib = load()
    h = lib.oracle_create(scene_ptr)
    assert h, "the restatement refused the scene"
    pos, nrm, a = np.zeros(3, np.float32), np.zeros(3, np.float32), np.zeros(1, np.float32)
    lib.oracle_primitive_sample(h, prim, time, int(np.int64(seed).astype(np.uint32).view(np.int32)), _fp(pos), _fp(nrm),
                                _fp(a))
    lib.oracle_destroy(h)
    return pos, nrm


def probe_sample(scene_ptr, seed):
    """The restatement's single-call oracle_probe_sample: (dir (3,), pdf, color (3,)) float32."""
    lib = load()
    h = lib.oracle_create(scene_ptr)
    assert h, "the restatement refused the scene"
    d, c, p = np.zeros(3, np.float32), np.zeros(3, np.float32), np.zeros(1, np.float32)
    lib.oracle_probe_sample(h, int(np.int64(seed).astype(np.uint32).view(np.int32)), _fp(d), _fp(c), _fp(p))
    lib.oracle_destroy(h)
    return d, p[0], c
