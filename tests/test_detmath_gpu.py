"""The math layer on the device against its host build and float64.

include/tb200_detmath.h is compiled twice: for the device, with the __dmul_rn/__dadd_rn/... intrinsics, and for the
host, with plain operators and -ffp-contract=off (the CPU restatement, the detmath flavour of the reference, api.cu's
host code).  Per-sample parity rests on both giving the same bits, for every argument a caller can pass.  This module
checks it directly: tests/math_harness.cu evaluates the functions on the device, one input per thread, and
tests/math_host.cpp recomputes each result with the host build and with glibc's double function rounded once.

- sinf, cosf, the out-of-line tb_sincosf, expf inline and the out-of-line tb_expf, and acosf on all 2^32 floats: the
  device equals the host bit for bit (a NaN matches any NaN), the host equals float64 except where the header documents
  otherwise (|x| >= 1e6 gives exactly (+0, 1), sin(-0) gives +0, both asserted as exact values), and expf never
  decreases as its argument increases.
- atan2f and powf on a cross product of special values, on every (sign, exponent) pair with random mantissas, and
  powf on the finish step's domain: device = host = float64, which follows C99 Annex F at the special values.
- the double-precision cores those functions round (tbm_sincos_d, tbm_exp_d, tbm_log_d, tbm_atan2_d) on millions
  of arguments: the device equals the host to the last bit of the double, which a contraction on either side breaks.
- tb_math.cuh's transforms on the device: bit for bit with their nvcc host build and with the full quaternion
  arithmetic their shortcuts stand for; interpolate_transform bit for bit with its host build.

tests/test_detmath.py and tests/test_transform_exact.py check the host builds alone."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import cuda_harness
import rayoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_SOURCES = [os.path.join(ROOT, "tests", "math_host.cpp")]
HOST_DEPS = HOST_SOURCES + [os.path.join(ROOT, "include", "tb200_detmath.h")]

F32 = np.float32
# math_unary's and math_binary's functions (math_harness.cu)
SINF, COSF, SINCOSF, EXPF, TB_EXPF, ACOSF = range(6)
ATAN2F, POWF = range(2)
# math_double's and math_double_host's double-precision cores
SINCOS_D, EXP_D, LOG_D, ATAN2_D = range(4)
# math_check_unary's host functions (math_host.cpp); math_check_binary takes ATAN2F and POWF
HOST_SINCOS, HOST_EXP, HOST_ACOS = range(3)
# each host function with the device functions it checks, and which host output each device output must equal
UNARY = {
    "sincos": (HOST_SINCOS, [(SINF, (0,)), (COSF, (1,)), (SINCOSF, (0, 1))]),
    "exp": (HOST_EXP, [(EXPF, (0,)), (TB_EXPF, (0,))]),
    "acos": (HOST_ACOS, [(ACOSF, (0,))]),
}
# math_host.cpp's failure classes, in order
DEVICE, REF, BIG, NEG_ZERO, ORDER, NEAR_TIE = range(6)
CLASSES = ("device != host", "host != float64", "|x| >= 1e6", "sin(-0)", "decreasing exp", "powf 1 ulp at a near-tie")
MAX_FAILS = 8

CHUNK = 1 << 26
ALL = 1 << 32
# finite floats with |x| >= 1e6 (1e6 is the float 0x49742400)
N_BIG = 2 * (0x7f800000 - 0x49742400)


def _threads():
    return len(os.sched_getaffinity(0))


# ---- the two helpers ----

_dev = None
_host = None


def device_lib():
    global _dev
    if _dev is None:
        lib = C.CDLL(cuda_harness.harness_path("math_harness"))
        lib.math_sizeof_xf.restype = C.c_int
        lib.math_unary.restype = C.c_int
        lib.math_unary.argtypes = [C.c_int, C.c_uint32, C.c_longlong, C.c_void_p, C.c_void_p]
        lib.math_binary.restype = C.c_int
        lib.math_binary.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]
        lib.math_double.restype = C.c_int
        lib.math_double.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]
        lib.math_transforms.restype = C.c_int
        lib.math_transforms.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        lib.math_transforms_host.restype = None
        lib.math_transforms_host.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        lib.math_interpolate.restype = C.c_int
        lib.math_interpolate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        lib.math_interpolate_host.restype = None
        lib.math_interpolate_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        _dev = lib
    return _dev


def host_path():
    """tests/math_host.cpp built with the CPU restatement's flags (rayoracle.FLAGS) into a temporary directory keyed by
    its sources' hash (the repository tree may be read-only), on first use."""
    h = hashlib.sha1(" ".join([rayoracle.CXX] + rayoracle.FLAGS).encode())
    for p in HOST_DEPS:
        with open(p, "rb") as f:
            h.update(f.read())
    path = os.path.join(tempfile.gettempdir(), "tinsel_b200_mathhost_%s.so" % h.hexdigest()[:16])
    if not os.path.exists(path):
        tmp = "%s.%d.tmp" % (path, os.getpid())
        subprocess.check_call([rayoracle.CXX, *rayoracle.FLAGS, "-I", os.path.join(ROOT, "include"), "-o", tmp,
                               *HOST_SOURCES])
        os.replace(tmp, path)
    return path


def host_lib():
    global _host
    if _host is None:
        lib = C.CDLL(host_path())
        lib.math_check_unary.restype = None
        lib.math_check_unary.argtypes = [C.c_int, C.c_uint32, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p]
        lib.math_double_host.restype = None
        lib.math_double_host.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]
        lib.math_check_binary.restype = None
        lib.math_check_binary.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_int,
                                          C.c_void_p, C.c_void_p]
        _host = lib
    return _host


def test_math_helpers_compile():
    """Both helpers against the headers as they are (no GPU needed): a header change that breaks either fails here."""
    cuda_harness.harness_path("math_harness")
    host_lib()


# ---- one-argument functions: all 2^32 floats ----


def _torch():
    import torch
    return torch


def _ok(rc):
    assert rc == 0, "CUDA error %d" % rc


def _report(counts, fails, where):
    """Per failure class, the count and the first failing inputs (where(position) names one)."""
    out = []
    for k, name in enumerate(CLASSES):
        if counts[k]:
            out.append("%s: %d, first at %s" % (name, counts[k], ", ".join(where(int(i)) for i in fails[k] if i >= 0)))
    return "; ".join(out)


@pytest.mark.gpu
@pytest.mark.parametrize("family", list(UNARY))
def test_unary_on_every_float(family):
    torch = _torch()
    dev, host = device_lib(), host_lib()
    fn, variants = UNARY[family]
    outs = [(v, o) for v, os_ in variants for o in os_]
    da = torch.empty(CHUNK, dtype=torch.float32, device="cuda")
    db = torch.empty(CHUNK, dtype=torch.float32, device="cuda")
    ha = [torch.empty(CHUNK, dtype=torch.float32, pin_memory=True) for _ in outs]
    ptrs = (C.c_void_p * len(outs))(*[h.data_ptr() for h in ha])
    which = (C.c_int * len(outs))(*[o for _, o in outs])
    counts = np.zeros(len(CLASSES), np.int64)
    c = np.zeros(len(CLASSES), np.int64)
    f = np.zeros(len(CLASSES) * MAX_FAILS, np.int64)
    fails = [[] for _ in CLASSES]
    prev = None
    t0 = time.time()
    for first in range(0, ALL, CHUNK):
        k = 0
        for v, os_ in variants:
            _ok(dev.math_unary(v, first, CHUNK, da.data_ptr(), db.data_ptr()))
            for o in range(len(os_)):
                ha[k].copy_(da if o == 0 else db)
                k += 1
        host.math_check_unary(fn, first, CHUNK, ptrs, which, len(outs), _threads(), c.ctypes.data, f.ctypes.data)
        counts += c
        for j in range(len(CLASSES)):
            fails[j] += [first + int(i) for i in f[j * MAX_FAILS:(j + 1) * MAX_FAILS] if i >= 0]
        if fn == HOST_EXP:
            # the order across the chunk boundary: bits first - 1 and first, unless first - 1 is +-inf or a NaN
            u = first - 1
            if prev is not None and (u & 0x7fffffff) < 0x7f800000:
                a, b = prev, float(ha[0][0])
                if not (b <= a if u >> 31 else a <= b):
                    counts[ORDER] += 1
                    fails[ORDER].append(u)
            prev = float(ha[0][CHUNK - 1])
    secs = time.time() - t0
    fails = np.array([(x + [-1] * MAX_FAILS)[:MAX_FAILS] for x in fails])

    def where(u):
        x = np.array([u], np.uint32).view(F32)[0]
        return "%08x (%r)" % (u, float(x))

    msg = _report(counts, fails, where)
    print("%s: device != host: %d of %d; host != float64: %d; %.1f s on %d host threads" % (
        family, counts[DEVICE], ALL, counts[REF], secs, _threads()))
    assert counts[DEVICE] == 0 and counts[REF] == 0 and counts[ORDER] == 0, "%s: %s" % (family, msg)
    if fn == HOST_SINCOS:
        # the documented exceptions, each with its exact value (math_host.cpp counts only those)
        assert counts[BIG] == N_BIG, msg
        assert counts[NEG_ZERO] == 1 and fails[NEG_ZERO][0] == 0x80000000, msg


# ---- two-argument functions ----


def _bits(u):
    return np.asarray(u, np.uint32).view(F32)


def _specials():
    """+-0, the smallest and largest subnormals, +-FLT_MIN, +-0.5, 1, 2, 3, 2.2, 1/2.2, odd and even integers around
    2^24, +-FLT_MAX, +-inf and NaN."""
    pos = np.concatenate([
        _bits([0x00000000, 0x00000001, 0x007fffff, 0x00800000, 0x7f7fffff, 0x7f800000]),
        np.array([0.5, 1.0, 2.0, 3.0, 2.2, 1.0 / 2.2, 16777213.0, 16777215.0, 16777216.0, 16777218.0, 33554430.0,
                  33554432.0], F32),
        np.array([F32(1.0) / F32(2.2)], F32),
    ])
    return np.concatenate([pos, -pos, _bits([0x7fc00000])]).astype(F32)


def _check_binary(fn, x, y):
    """fn over the pairs (x[i], y[i]) (float32 arrays) on the device, checked by the host arm; returns
    (counts, fails) with fails as positions."""
    torch = _torch()
    dev, host = device_lib(), host_lib()
    n = len(x)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    out = torch.empty(n, dtype=torch.float32, device="cuda")
    _ok(dev.math_binary(fn, xd.data_ptr(), yd.data_ptr(), n, out.data_ptr()))
    got = out.cpu().numpy()
    c = np.zeros(len(CLASSES), np.int64)
    f = np.zeros(len(CLASSES) * MAX_FAILS, np.int64)
    host.math_check_binary(fn, x.ctypes.data, y.ctypes.data, n, got.ctypes.data, _threads(), c.ctypes.data,
                           f.ctypes.data)
    return c, f.reshape(len(CLASSES), MAX_FAILS)


def _assert_binary(fn, x, y, what):
    """device = host on every pair, host = float64 but for powf's near-ties; returns the number of those."""
    x, y = np.ascontiguousarray(x, F32), np.ascontiguousarray(y, F32)
    counts, fails = _check_binary(fn, x, y)
    msg = _report(counts, fails, lambda i: "(%r, %r)" % (float(x[i]), float(y[i])))
    assert counts[DEVICE] == 0 and counts[REF] == 0, "%s, %s of %d pairs: %s" % (
        ("atan2f", "powf")[fn], what, len(x), msg)
    return int(counts[NEAR_TIE])


@pytest.mark.gpu
@pytest.mark.parametrize("fn", [ATAN2F, POWF], ids=["atan2f", "powf"])
def test_binary_on_special_values(fn):
    s = _specials()
    x, y = np.repeat(s, len(s)), np.tile(s, len(s))
    _assert_binary(fn, x, y, "specials")


@pytest.mark.gpu
@pytest.mark.parametrize("fn", [ATAN2F, POWF], ids=["atan2f", "powf"])
def test_binary_on_every_sign_and_exponent(fn):
    # every (sign, exponent) of x with every one of y, 16 random mantissas each: 4.2 M pairs, NaNs and infinities too
    rng = np.random.default_rng(31 + fn)
    se = np.arange(512, dtype=np.uint32) << 23
    sx, sy = np.repeat(se, 512 * 16), np.tile(np.repeat(se, 16), 512)
    x = _bits(sx | rng.integers(0, 1 << 23, sx.size, dtype=np.uint32))
    y = _bits(sy | rng.integers(0, 1 << 23, sy.size, dtype=np.uint32))
    _assert_binary(fn, x, y, "(sign, exponent) pairs")


@pytest.mark.gpu
@pytest.mark.parametrize("gamma", [F32(2.2), F32(1.0) / F32(2.2)], ids=["2.2", "1/2.2"])
def test_powf_on_the_finish_domain(gamma):
    # the finish step (k_finish: SrgbToLinear, LinearToSrgb) raises values in [0, 1] to 2.2 and 1/2.2: every float there
    end = 0x3f800000 + 1
    ties = 0
    t0 = time.time()
    for first in range(0, end, CHUNK):
        x = _bits(np.arange(first, min(first + CHUNK, end), dtype=np.uint32))
        ties += _assert_binary(POWF, x, np.full(x.size, gamma, F32), "x in [0, 1], y = %r" % float(gamma))
    print("powf(x in [0, 1], %r): device != host: 0 of %d; 1 ulp from float64 at a near-tie: %d; %.1f s" % (
        float(gamma), end, ties, time.time() - t0))
    # the header's bound: a misrounded result in about 1e-7 of the calls
    assert ties <= end * 1e-6


# ---- the double-precision cores ----


def _double_args(rng, fn, n):
    """n arguments (x, y) in the domain of a core: |x| < 1e6 for sincos (phases of a few pi mostly), the exponents
    powf passes to tbm_exp_d, positive normal doubles for tbm_log_d, any signs and magnitudes for tbm_atan2_d."""
    mag = lambda lo, hi: np.exp(rng.uniform(np.log(lo), np.log(hi), n)) * rng.choice([-1.0, 1.0], n)
    y = np.zeros(n)
    if fn == SINCOS_D:
        x = np.where(rng.random(n) < 0.5, rng.uniform(-8.0, 8.0, n), mag(1e-300, 9.99e5))
    elif fn == EXP_D:
        x = rng.uniform(-110.0, 100.0, n)
    elif fn == LOG_D:
        x = np.abs(mag(1e-300, 1e300))
    else:
        x, y = mag(1e-300, 1e300), mag(1e-300, 1e300)
        x[: n // 4], y[n // 4: n // 2] = 0.0, -0.0
    return np.ascontiguousarray(x), np.ascontiguousarray(y)


@pytest.mark.gpu
@pytest.mark.parametrize("fn", [SINCOS_D, EXP_D, LOG_D, ATAN2_D], ids=["sincos_d", "exp_d", "log_d", "atan2_d"])
def test_double_cores_match_their_host_build(fn):
    # The float functions round these once, so a contraction or a reordered step on the device changes a float result
    # only where the double lies within its own error of a float midpoint: rarely enough to pass every float above.
    # Their double results must be the host's to the last bit.
    torch = _torch()
    n = 1 << 22
    x, y = _double_args(np.random.default_rng(51 + fn), fn, n)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    ad = torch.empty(n, dtype=torch.float64, device="cuda")
    bd = torch.zeros(n, dtype=torch.float64, device="cuda")
    _ok(device_lib().math_double(fn, xd.data_ptr(), yd.data_ptr(), n, ad.data_ptr(), bd.data_ptr()))
    a, b = np.zeros(n), np.zeros(n)
    host_lib().math_double_host(fn, x.ctypes.data, y.ctypes.data, n, a.ctypes.data, b.ctypes.data)
    got = np.stack([ad.cpu().numpy(), bd.cpu().numpy()], 1)
    want = np.stack([a, b], 1)
    bad = ~((got.view(np.uint64) == want.view(np.uint64)) | (np.isnan(got) & np.isnan(want))).all(1)
    assert not bad.any(), "%d of %d differ from the host build; first at (%s, %s): device %s host %s" % (
        int(bad.sum()), n, float(x[bad][0]).hex(), float(y[bad][0]).hex(), [float(v).hex() for v in got[bad][0]],
        [float(v).hex() for v in want[bad][0]])


# ---- transforms ----

# struct Xf in tb_math.cuh: p, r (x, y, z, w), s
XF_DTYPE = np.dtype([("p", F32, 3), ("r", F32, 4), ("s", F32)])


def _vectors(rng):
    """tests/test_transform_exact.py's vectors: every triple of 19 special components, then 400 k random bit patterns,
    every other one with a magnitude around 1."""
    sp = np.array([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -5.9e-39, 1.17549435e-38, -1.17549435e-38, 1.0, -1.0, 0.5,
                   3.75, -1234.5, 3.4028235e38, -3.4028235e38, np.inf, -np.inf, np.nan, -np.nan], F32)
    special = np.stack(np.meshgrid(sp, sp, sp, indexing="ij"), -1).reshape(-1, 3)
    u = rng.integers(0, 1 << 32, (400000, 3), dtype=np.uint32)
    u[1::2] = (u[1::2] & 0x807fffff) | ((100 + (u[1::2] >> 24) % 56) << 23)
    return np.ascontiguousarray(np.concatenate([special, _bits(u)]), F32)


def _transforms():
    """The 8 quaternions (identity, -0 components, a negated w, rotations) x 4 scales x 3 translations."""
    h = 0.5
    qs = [(0.0, 0.0, 0.0, 1.0), (-0.0, 0.0, 0.0, 1.0), (0.0, -0.0, 0.0, 1.0), (0.0, 0.0, -0.0, 1.0),
          (-0.0, -0.0, -0.0, 1.0), (0.0, 0.0, 0.0, -1.0), (h, -h, h, h), (0.36, 0.0, -0.48, 0.8)]
    ss = [1.0, 0.625, 2.5, 0.3]
    ps = [(0.0, 0.0, 0.0), (-0.0, 1.5, -2.25), (0.1, 1e30, -3.0)]
    t = np.zeros(len(qs) * len(ss) * len(ps), XF_DTYPE)
    k = 0
    for q in qs:
        for s in ss:
            for p in ps:
                t[k] = (p, q, s)
                k += 1
    return t


def _same(a, b):
    """Element-wise: the same bits, or both NaN (which NaN an operation returns is not specified: the device gives the
    canonical one, and x86 the payload of one operand, whose order the compiler may swap)."""
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


@pytest.mark.gpu
def test_transforms_match_their_host_build_and_the_full_arithmetic():
    torch = _torch()
    lib = device_lib()
    assert lib.math_sizeof_xf() == XF_DTYPE.itemsize
    v = _vectors(np.random.default_rng(41))
    ts = _transforms()
    vd = torch.from_numpy(v).cuda()
    out = torch.empty((len(v), 8, 3), dtype=torch.float32, device="cuda")
    want = np.zeros((len(v), 8, 3), F32)
    names = ("transform_vector", "transform_point", "inverse_transform_vector", "inverse_transform_point")
    # the host build on a slice of the vectors per thread (ctypes releases the GIL)
    cuts = np.linspace(0, len(v), _threads() + 1).astype(int)
    spans = list(zip(cuts[:-1], cuts[1:]))
    pool = ThreadPoolExecutor(len(spans))
    fast = 0
    for t in ts:
        t = np.ascontiguousarray(t.reshape(1))
        td = torch.from_numpy(t.view(np.uint8)).cuda()
        _ok(lib.math_transforms(td.data_ptr(), 1, vd.data_ptr(), len(v), out.data_ptr()))
        got = out.cpu().numpy()
        list(pool.map(lambda s: lib.math_transforms_host(t.ctypes.data, 1, v[s[0]:].ctypes.data, int(s[1] - s[0]),
                                                         want[s[0]:].ctypes.data), spans))
        if tuple(t[0]["r"].view(np.uint32)) == (0, 0, 0, 0x3f800000):
            fast += int(np.isfinite(v).all(-1).sum())
        # the host build, then the shortcuts of rotate_xf and inverse_scale against the full quaternion arithmetic
        host = _same(got, want).all(-1)
        full = _same(got[:, :4], got[:, 4:]).all(-1)
        if host.all() and full.all():
            continue
        for k in range(4):
            bad = ~host[:, k] | ~host[:, 4 + k]
            assert not bad.any(), "%s by %s differs from its host build at %d vectors, first %r: device %r host %r" % (
                names[k], t[0], int(bad.sum()), v[bad][0], got[bad][0, [k, 4 + k]], want[bad][0, [k, 4 + k]])
            bad = ~full[:, k]
            assert not bad.any(), "%s by %s differs from the full arithmetic at %d vectors, first %r: %r vs %r" % (
                names[k], t[0], int(bad.sum()), v[bad][0], got[bad][0, k], got[bad][0, 4 + k])
    pool.shutdown()
    assert fast > 0   # the shortcut of an unrotated transform was taken


@pytest.mark.gpu
def test_interpolate_transform_matches_its_host_build():
    torch = _torch()
    lib = device_lib()
    rng = np.random.default_rng(43)
    ts = _transforms()
    rnd = np.zeros(64, XF_DTYPE)
    rnd["p"] = rng.normal(size=(64, 3)) * 10.0
    q = rng.normal(size=(64, 4))
    rnd["r"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    rnd["s"] = rng.uniform(0.1, 4.0, 64)
    xs = np.concatenate([ts, rnd])
    times = np.array([0.0, -0.0, 1.0, 0.5, 0.25, 0.3, 1e-8, 0.99999994, 1.5, -1.0], F32)
    n = len(xs)
    a, b = np.repeat(xs, n * len(times)), np.tile(np.repeat(xs, len(times)), n)
    t = np.tile(times, n * n)
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    ad, bd = (torch.from_numpy(z.view(np.uint8)).cuda() for z in (a, b))
    tdev = torch.from_numpy(t).cuda()
    out = torch.empty(len(t) * 8, dtype=torch.float32, device="cuda")
    _ok(lib.math_interpolate(ad.data_ptr(), bd.data_ptr(), tdev.data_ptr(), len(t), out.data_ptr()))
    got = out.cpu().numpy().reshape(-1, 8)
    want = np.zeros(len(t), XF_DTYPE)
    lib.math_interpolate_host(a.ctypes.data, b.ctypes.data, t.ctypes.data, len(t), want.ctypes.data)
    want = want.view(F32).reshape(-1, 8)
    bad = ~_same(got, want).all(-1)
    assert not bad.any(), "%d of %d interpolations differ, first %s, %s at %r: device %r host %r" % (
        int(bad.sum()), len(t), a[bad][0], b[bad][0], float(t[bad][0]), got[bad][0], want[bad][0])
