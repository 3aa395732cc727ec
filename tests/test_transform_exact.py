"""The shortcuts of tb_math.cuh's transforms, on the host: rotate_xf returns v + 0.0f for a rotation of exactly
(+0, +0, +0, +1) and a finite v, and inverse_scale skips the division for a unit scale.  All four transform
functions are compared bit for bit with the full quaternion arithmetic of maths.h:558-619 over zeros of both
signs, denormals, +-FLT_MAX, +-inf and NaN in every component, random vectors, quaternions with a -0 component and
rotated ones, and unit and other scales.  Built with nvcc (host code only, the device build's host flags)."""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include "tb_math.cuh"
#include <cstdio>
#include <cmath>
#include <vector>

static V3 full_tv(const Xf& t, V3 v) { return rotate(t.r, t.s * v); }
static V3 full_tp(const Xf& t, V3 v) { return t.p + rotate(t.r, t.s * v); }
static V3 full_itv(const Xf& t, V3 v) { return (1.0f / t.s) * rotate(qconj(t.r), v); }
static V3 full_itp(const Xf& t, V3 v) { return (1.0f / t.s) * rotate(qconj(t.r), v - t.p); }

static bool same(V3 a, V3 b)
{
    return tb_float_bits(a.x) == tb_float_bits(b.x) && tb_float_bits(a.y) == tb_float_bits(b.y) && tb_float_bits(a.z) == tb_float_bits(b.z);
}

int main()
{
    const float sp[] = {0.0f, -0.0f, 1e-45f, -1e-45f, 1.1754942e-38f, -5.9e-39f, FLT_MIN, -FLT_MIN, 1.0f, -1.0f, 0.5f, 3.75f, -1234.5f,
                        FLT_MAX, -FLT_MAX, INFINITY, -INFINITY, NAN, -NAN};
    const int ns = sizeof(sp) / sizeof(sp[0]);
    std::vector<V3> vs;
    for (int i = 0; i < ns; ++i)
        for (int j = 0; j < ns; ++j)
            for (int k = 0; k < ns; ++k) vs.push_back(v3(sp[i], sp[j], sp[k]));
    uint32_t s = 2463534242u;
    auto bits = [&]() { s ^= s << 13; s ^= s >> 17; s ^= s << 5; return s; };
    for (int i = 0; i < 400000; ++i) {
        float c[3];
        for (int k = 0; k < 3; ++k) {
            uint32_t u = bits();
            if (i & 1) u = (u & 0x807fffffu) | ((100u + (u >> 24) % 56u) << 23);   // magnitudes around 1 as well
            memcpy(&c[k], &u, 4);
        }
        vs.push_back(v3(c[0], c[1], c[2]));
    }
    const float h = 0.5f;
    const Q4 qs[] = {q4(0.0f, 0.0f, 0.0f, 1.0f), q4(-0.0f, 0.0f, 0.0f, 1.0f), q4(0.0f, -0.0f, 0.0f, 1.0f), q4(0.0f, 0.0f, -0.0f, 1.0f),
                     q4(-0.0f, -0.0f, -0.0f, 1.0f), q4(0.0f, 0.0f, 0.0f, -1.0f), q4(h, -h, h, h), q4(0.36f, 0.0f, -0.48f, 0.8f)};
    const float ss[] = {1.0f, 0.625f, 2.5f, 0.3f};
    const V3 ps[] = {v3(0.0f, 0.0f, 0.0f), v3(-0.0f, 1.5f, -2.25f), v3(0.1f, 1e30f, -3.0f)};
    long bad = 0, fast = 0, cases = 0;
    for (const Q4& q : qs)
        for (float sc : ss)
            for (const V3& p : ps) {
                Xf t;
                t.p = p;
                t.r = q;
                t.s = sc;
                for (const V3& v : vs) {
                    bad += !same(transform_vector(t, v), full_tv(t, v));
                    bad += !same(transform_point(t, v), full_tp(t, v));
                    bad += !same(inverse_transform_vector(t, v), full_itv(t, v));
                    bad += !same(inverse_transform_point(t, v), full_itp(t, v));
                    fast += (&q == &qs[0]) && std::isfinite(v.x) && std::isfinite(v.y) && std::isfinite(v.z);
                    cases += 4;
                }
            }
    printf("%ld %ld %ld\n", bad, fast, cases);
    return 0;
}
"""


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def test_transform_shortcuts_are_bit_exact(tmp_path):
    src = tmp_path / "t.cu"
    src.write_text(SRC)
    exe = str(tmp_path / "t")
    subprocess.check_call([_nvcc(), "-ccbin", "/usr/bin/g++", "-std=c++17", "-Xcompiler", "-ffp-contract=off,-O2",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tinsel_b200", "csrc"), str(src), "-o", exe])
    bad, fast, cases = map(int, subprocess.check_output([exe]).split())
    assert fast > 0
    assert bad == 0, "%d of %d transforms differ from the full quaternion arithmetic" % (bad, cases)
