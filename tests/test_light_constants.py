"""The light constants of a primitive record (tb_scene.cuh: set_light_constants), which path_hit and nee_connect read
instead of dividing on every bounce: 1/area, 1/N, lightSamples/N and 1/lightSamples with N = int(lightSamples + 1.0f).
The host's values must have the bits the device's own evaluation of those expressions gave, so they are compared
with the expressions restated in numpy float32 (IEEE division, round-to-nearest conversions: the device's
-prec-div=true arithmetic).  Covered: lightSamples of 0, 1, 2, 7, 2^24 - 1, 2^24 and negative counts; areas of +-0,
denormals, 1, FLT_MAX, infinity and what the sphere and mesh rules give.  The helper is built with nvcc and the
library's host flags (host code only), and the scene cache, which stores the records as the library built them, is
checked over the snapshots' primitives.  A cache written before the records held the constants is refused.  No GPU."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import tinsel_b200 as tb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
FIELDS = ("invArea", "cbsdf", "clight", "invLightSamples")

SRC = r"""
#include "tb_scene.cuh"
#include <cstddef>
#include <cstdio>

int main()
{
    printf("%zu %zu %zu", sizeof(DPrim), offsetof(DPrim, area), offsetof(DPrim, lightSamples));
    printf(" %zu %zu %zu %zu\n", offsetof(DPrim, invArea), offsetof(DPrim, cbsdf), offsetof(DPrim, clight), offsetof(DPrim, invLightSamples));
    unsigned areaBits;
    int lightSamples;
    while (scanf("%x %d", &areaBits, &lightSamples) == 2) {
        DPrim d;
        memset(&d, 0, sizeof(d));
        memcpy(&d.area, &areaBits, 4);
        d.lightSamples = lightSamples;
        set_light_constants(d);
        printf("%08x %08x %08x %08x\n", tb_float_bits(d.invArea), tb_float_bits(d.cbsdf), tb_float_bits(d.clight),
               tb_float_bits(d.invLightSamples));
    }
    return 0;
}
"""


def device_expressions(area, light_samples):
    """what path_hit and nee_connect computed per bounce, in float32: 1.0f / area, N = int(lightSamples + 1.0f),
    1.0f / N, float(lightSamples) / N and 1.0f / lightSamples (an int operand converts to float first)"""
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        n = int(F(light_samples) + F(1))   # float -> int truncates toward zero, as the C conversion does
        return [F(1) / F(area), F(1) / F(n), F(light_samples) / F(n), F(1) / F(light_samples)]


def bits(x):
    return int(np.asarray(x, F).view(np.uint32))


@pytest.fixture(scope="module")
def helper(tmp_path_factory):
    """(layout, run): the DPrim offsets the helper program reports, and run(cases) -> its four values' bits per case"""
    tmp = tmp_path_factory.mktemp("light_constants")
    src = tmp / "t.cu"
    src.write_text(SRC)
    exe = str(tmp / "t")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    subprocess.check_call([nvcc, "-ccbin", "/usr/bin/g++", "-std=c++17", "-Xcompiler", "-ffp-contract=off,-O2",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tinsel_b200", "csrc"), str(src), "-o", exe])
    layout = [int(v) for v in subprocess.check_output([exe], input=b"").split()]

    def run(cases):
        stdin = "".join("%08x %d\n" % (bits(a), n) for a, n in cases).encode()
        lines = subprocess.check_output([exe], input=stdin).decode().split("\n")[1:]
        return [[int(w, 16) for w in line.split()] for line in lines if line]
    return layout, run


LIGHT_SAMPLES = [0, 1, 2, 7, 2 ** 24 - 1, 2 ** 24, -1, -2, -7]


def sphere_area(radius):
    # PrimitiveArea of a sphere, as api.cu computes it: 4.0f * kPi * r * r
    with np.errstate(over="ignore", under="ignore"):
        return F(4) * F(3.141592653589793) * F(radius) * F(radius)


def mesh_area(area, scale):
    # PrimitiveArea of a mesh: the mesh's area times the end transform's scale
    with np.errstate(over="ignore", under="ignore"):
        return F(area) * F(scale)


AREAS = ([F(0), F(-0.0), F(1.4e-45), F(1.1754942e-38), F(5.9e-39), np.finfo(F).tiny, F(1), F(0.3), np.finfo(F).max, F(np.inf)] +
         [sphere_area(r) for r in (0.0, 1e-23, 0.05, 0.5, 1.0, 7.25, 1e18, 1e19)] +
         [mesh_area(a, s) for a, s in ((0.0, 1.0), (4.0e-6, 1.0), (0.1156, 1.0), (0.1156, 2.5), (3.0e38, 2.0), (1.0e-30, 1.0e-15))])


def test_host_constants_match_the_device_expressions(helper):
    layout, run = helper
    assert layout[0] % 4 == 0 and len(set(layout[1:])) == len(layout) - 1
    cases = [(a, n) for a in AREAS for n in LIGHT_SAMPLES]
    got = run(cases)
    assert len(got) == len(cases)
    bad = []
    for (a, n), g in zip(cases, got):
        want = [bits(v) for v in device_expressions(a, n)]
        if g != want:
            bad.append("area %r lightSamples %d: host %s, device expressions %s" % (float(a), n, ["%08x" % v for v in g], ["%08x" % v for v in want]))
    assert not bad, "%d of %d cases differ:\n%s" % (len(bad), len(cases), "\n".join(bad[:20]))
    # the cases reach what they are meant to: 2^24 + 1 rounds to 2^24 in float, so 2^24 - 1 and 2^24 share N
    assert device_expressions(1.0, 2 ** 24)[1] == device_expressions(1.0, 2 ** 24 - 1)[1] == F(1) / F(2 ** 24)
    assert np.isinf(device_expressions(1.0, 0)[3]) and np.isinf(device_expressions(1.0, -1)[1])
    assert device_expressions(np.finfo(F).max, 1)[0] < np.finfo(F).tiny   # a denormal reciprocal, not flushed


def _cache_records(tmp_path, name, layout):
    """the primitive records of scenes/<name>.tsnap as tb200_scene_cache_save stores them: (area, lightSamples, the four
    constants' bits) per primitive, and the snapshot's areas by the loader's rules (tb.primitive_areas)"""
    path = tb.scene_path(name)
    if not os.path.exists(path):
        pytest.skip("snapshot scenes/%s.tsnap not present" % name)
    snap = tb.Snapshot(path)
    out = str(tmp_path / (name + ".tcache"))
    tb.scene_cache_save(snap.scene, out)
    rules = tb.primitive_areas(snap.scene)
    snap.close()
    data = open(out, "rb").read()
    size, off_area, off_ls = layout[:3]
    offs = layout[3:]
    assert data[:8] == b"TB2CACHE" and int.from_bytes(data[12:16], "little") == size
    count = int.from_bytes(data[24:32], "little")
    assert count == len(rules)
    recs = []
    for i in range(count):
        rec = data[32 + i * size: 32 + (i + 1) * size]
        area = np.frombuffer(rec[off_area:off_area + 4], F)[0]
        ls = int(np.frombuffer(rec[off_ls:off_ls + 4], np.int32)[0])
        recs.append((area, ls, [int.from_bytes(rec[o:o + 4], "little") for o in offs]))
    return recs, rules, data


@pytest.mark.parametrize("name", ["cornell", "veach", "meshlight", "emitter", "many", "simple"])
def test_cached_records_carry_the_device_expressions(tmp_path, helper, name):
    recs, rules, _ = _cache_records(tmp_path, name, helper[0])
    lights = 0
    for i, (area, ls, got) in enumerate(recs):
        assert bits(area) == bits(rules[i]), "primitive %d: area %r, the sphere / mesh rule gives %r" % (i, area, rules[i])
        want = [bits(v) for v in device_expressions(area, ls)]
        assert got == want, "%s primitive %d (area %r, lightSamples %d): %s" % (name, i, float(area), ls, dict(zip(FIELDS, got)))
        lights += ls > 0 and area > 0
    assert lights > 0


def test_version_3_cache_without_the_light_constants_is_refused(tmp_path, helper):
    """a version-3 cache holds records without the light constants: it is refused, not read with the wrong layout (the
    current version is 5: version 4 records marked primitives with a -0 component static, test_motion_time.py)"""
    _, _, data = _cache_records(tmp_path, "cornell", helper[0])
    assert int.from_bytes(data[8:12], "little") == 5
    lib = tb.load_library()
    old = bytearray(data)
    old[8:12] = (3).to_bytes(4, "little")
    p = str(tmp_path / "v3.tcache")
    open(p, "wb").write(bytes(old))
    h = lib.tb200_create_cached(p.encode(), 0)
    if h:
        lib.tb200_destroy(h)
    assert not h and "another build" in tb.last_error()
