// tb_math.cuh -- fp32 vector / quaternion / RNG primitives for the sm_90a kernels.
//
// Every function evaluates in exactly the operation order of the reference expression it
// stands for (cited per function, paths under /root/reference/src), because per-sample parity
// with src/render.cpp is a bit-exactness problem: this TU is compiled with -fmad=false
// -prec-div=true -prec-sqrt=true -ftz=false so +,-,*,/,sqrt are IEEE and un-contracted, just
// like the x86-64 (no-FMA) build of the reference.  Where the reference silently promotes to
// double (`Vec3/float` is `a*(1.0/s)`, maths.h:242) the double rounding is innocuous for a
// single division (53 >= 2*24+2 bits), so `1.0f/s` in fp32 gives the same bits.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <float.h>
#include <string.h>

#include "tb200_detmath.h"

#define TB_DEV __device__ __forceinline__
// usable from host code too (api.cu hoists per-primitive constants with the same arithmetic)
#define TB_HD __host__ __device__ __forceinline__

struct V3 {
    float x, y, z;
};

TB_HD V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
TB_HD V3 v3s(float s) { return v3(s, s, s); }

// maths.h:237-251
TB_HD V3 operator-(V3 a) { return v3(-a.x, -a.y, -a.z); }
TB_HD V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
TB_HD V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
TB_HD V3 operator*(V3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }
TB_HD V3 operator*(float s, V3 a) { return v3(a.x * s, a.y * s, a.z * s); }
TB_HD V3 operator*(V3 a, V3 b) { return v3(a.x * b.x, a.y * b.y, a.z * b.z); }
// Vec3/float == a*(1.0/s), maths.h:242
TB_HD V3 operator/(V3 a, float s) { const float r = 1.0f / s; return v3(a.x * r, a.y * r, a.z * r); }

// maths.h:256-258
TB_HD V3 cross(V3 a, V3 b) { return v3(a.y * b.z - b.y * a.z, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
TB_HD float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
TB_HD float length_sq(V3 a) { return dot(a, a); }
TB_HD float length(V3 a) { return sqrtf(length_sq(a)); }
// maths.h:260
TB_HD V3 normalize(V3 a) { return a / length(a); }
// maths.h:261-273
TB_HD V3 safe_normalize(V3 a, V3 fallback)
{
    const float m = length_sq(a);
    if (m > 0.0f) return a * (1.0f / sqrtf(m));
    return fallback;
}

// maths.h:56-77: Min/Max/Clamp/Abs templates (their NaN and -0 behaviour differs from fminf/fabsf)
TB_HD float tb_min(float a, float b) { return (a < b) ? a : b; }
TB_HD float tb_max(float a, float b) { return (a < b) ? b : a; }
TB_HD int tb_min(int a, int b) { return (a < b) ? a : b; }
TB_HD int tb_max(int a, int b) { return (a < b) ? b : a; }
TB_HD float tb_clamp(float x, float lo, float hi) { return tb_min(tb_max(x, lo), hi); }
TB_HD int tb_clamp(int x, int lo, int hi) { return tb_min(tb_max(x, lo), hi); }
TB_HD float tb_abs(float x) { return (x < 0.0f) ? -x : x; }
// maths.h:79-83
TB_HD float tb_lerp(float a, float b, float t) { return a + (b - a) * t; }
TB_HD V3 tb_lerp(V3 a, V3 b, float t) { return a + (b - a) * t; }
TB_HD float tb_sqr(float x) { return x * x; }

// maths.h:1591-1598
TB_HD V3 face_forward(V3 n, V3 v) { return (dot(v, n) < 0.0f) ? -n : n; }

// ---- quaternion / transform (maths.h:502-620) ------------------------------------------------

struct Q4 {
    float x, y, z, w;
};
TB_HD Q4 q4(float x, float y, float z, float w) { Q4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }

// maths.h:531-537
TB_HD Q4 qmul(Q4 a, Q4 b)
{
    return q4(a.w * b.x + b.w * a.x + a.y * b.z - b.y * a.z,
              a.w * b.y + b.w * a.y + a.z * b.x - b.z * a.x,
              a.w * b.z + b.w * a.z + a.x * b.y - b.x * a.y,
              a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z);
}
TB_HD Q4 qconj(Q4 q) { return q4(-q.x, -q.y, -q.z, q.w); }
// maths.h:558-563: q * (v,0) * q'
TB_HD V3 rotate(Q4 q, V3 v)
{
    const Q4 t = qmul(qmul(q, q4(v.x, v.y, v.z, 0.0f)), qconj(q));
    return v3(t.x, t.y, t.z);
}

struct Xf {
    V3 p;
    Q4 r;
    float s;
};

TB_HD uint32_t tb_float_bits(float f)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, sizeof(u));
    return u;
#endif
}

#if defined(__CUDA_ARCH__)
#define TB_COLD __noinline__   // rarely executed on the device: keep a single out-of-line copy
#else
#define TB_COLD
#endif

// rotate_xf's full arithmetic, out of line on the device: inline, its two qmuls were copied into every transform of
// every kernel, while scenes without rotations (cornell, veach) only ever take the shortcut
static __host__ __device__ TB_COLD V3 rotate_xf_full(Q4 q, V3 v, bool inverse) { return rotate(inverse ? qconj(q) : q, v); }

// rotate(q, v), or rotate(qconj(q), v) when `inverse`, for the rotation of a transform.  When q is (+0, +0, +0, +1)
// bit for bit and v is finite, every sum in both qmuls adds only exact zeros to the one product v.c * 1, and the +0
// among them turns a -0 into +0: the result is v + 0.0f, in either direction.  Any other quaternion (a -0 component
// included) and a non-finite v (0 * inf is NaN) take the full rotation.
TB_HD V3 rotate_xf(Q4 q, V3 v, bool inverse)
{
    const bool unrotated = (tb_float_bits(q.x) | tb_float_bits(q.y) | tb_float_bits(q.z)) == 0u && tb_float_bits(q.w) == 0x3f800000u;
    if (unrotated && fabsf(v.x) <= FLT_MAX && fabsf(v.y) <= FLT_MAX && fabsf(v.z) <= FLT_MAX) return v + v3s(0.0f);
    return rotate_xf_full(q, v, inverse);
}
// 1.0f / s, without the IEEE division for the common unit scale (1.0f / 1.0f is 1.0f)
TB_HD float inverse_scale(float s) { return s == 1.0f ? 1.0f : 1.0f / s; }

// maths.h:601-619
TB_HD V3 transform_vector(const Xf& t, V3 v) { return rotate_xf(t.r, t.s * v, false); }
TB_HD V3 transform_point(const Xf& t, V3 v) { return t.p + rotate_xf(t.r, t.s * v, false); }
TB_HD V3 inverse_transform_vector(const Xf& t, V3 v) { return inverse_scale(t.s) * rotate_xf(t.r, v, true); }
TB_HD V3 inverse_transform_point(const Xf& t, V3 v) { return inverse_scale(t.s) * rotate_xf(t.r, v - t.p, true); }

// maths.h:1566-1569 with Quat Lerp (maths.h:79-83 over Quat ops) and Normalize(Quat) (maths.h:547-553)
static __host__ __device__ TB_COLD Xf interpolate_transform(const Xf& a, const Xf& b, float t)
{
    Xf r;
    r.p = a.p + (b.p - a.p) * t;
    const Q4 q = q4(a.r.x + (b.r.x - a.r.x) * t, a.r.y + (b.r.y - a.r.y) * t, a.r.z + (b.r.z - a.r.z) * t,
                    a.r.w + (b.r.w - a.r.w) * t);
    const float len = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    const float rcp = 1.0f / len;
    r.r = q4(q.x * rcp, q.y * rcp, q.z * rcp, q.w * rcp);
    r.s = a.s + (b.s - a.s) * t;
    return r;
}

// ---- Random (maths.h:1036-1091) ---------------------------------------------------------------

struct Rng {
    uint32_t s1, s2;
};

TB_DEV Rng rng_seed(uint32_t seed)
{
    Rng r;
    r.s1 = 315645664u + seed;
    r.s2 = r.s1 ^ 0x13ab45feu;
    return r;
}

TB_DEV uint32_t rng_next(Rng& r)
{
    const uint32_t a = r.s1, b = r.s2;
    r.s1 = (b ^ ((a << 5) | (a >> 27))) ^ (a * b);
    r.s2 = r.s1 ^ ((b << 12) | (b >> 20));
    return r.s1;
}

// Randf (maths.h:1066-1076): float(value) * (1.0f/float(0xffffffff)); the constant is exactly 2^-32.
// Sample1D/Sample2D (sampler.h:238-258) go through Randf(0,1) = (1-t)*0 + t*1 == t.
TB_DEV float rng_float(Rng& r) { return (float)rng_next(r) * 2.3283064365386963e-10f; }

// device copy of tb200_sample_seed() (tinsel_b200/csrc/snapshot.cpp)
TB_DEV uint32_t tb_mix32(uint32_t h)
{
    h ^= h >> 16;
    h *= 0x7FEB352Du;
    h ^= h >> 15;
    h *= 0x846CA68Bu;
    h ^= h >> 16;
    return h;
}
TB_DEV uint32_t tb_sample_seed(uint32_t pixel, uint32_t frame)
{
    const uint32_t h = tb_mix32(pixel + 0x9E3779B9u);
    return tb_mix32(h ^ (frame * 0x85EBCA6Bu + 0xC2B2AE35u));
}

// Out-of-line device copies of the double-precision transcendentals: they are called from a dozen
// sites and inlining every copy bloats the kernel far past the instruction cache.  Results come back
// as return values, which stay in registers; out-pointers would go through the caller's stack.
#define TB_NOINLINE static __device__ __noinline__
// (sinf(x), cosf(x))
TB_NOINLINE float2 tb_sincosf(float x)
{
    float s, c;
    tbm_sincosf(x, &s, &c);
    return make_float2(s, c);
}
TB_NOINLINE float tb_expf(float x) { return tbm_expf(x); }

#define TB_PI 3.141592653589793f
#define TB_2PI (3.141592653589793f * 2.0f)
#define TB_INV_PI (1.0f / TB_PI)
#define TB_INV_2PI (1.0f / TB_2PI)

// ---- sampling warps (maths.h:1261-1325) -------------------------------------------------------

// BasisFromVector, maths.h:1261-1275 (1.0/sqrt(float) in double == 1.0f/sqrtf in fp32)
TB_DEV void basis_from_vector(V3 w, V3* u, V3* v)
{
    if (fabsf(w.x) > fabsf(w.y)) {
        const float invLen = 1.0f / sqrtf(w.x * w.x + w.z * w.z);
        *u = v3(-w.z * invLen, 0.0f, w.x * invLen);
    } else {
        const float invLen = 1.0f / sqrtf(w.y * w.y + w.z * w.z);
        *u = v3(0.0f, w.z * invLen, -w.y * invLen);
    }
    *v = cross(w, *u);
}

// UniformSampleSphere, maths.h:1278-1287
TB_DEV V3 uniform_sample_sphere(float u1, float u2)
{
    const float z = 1.f - 2.f * u1;
    const float r = sqrtf(tb_max(0.f, 1.f - z * z));
    const float phi = 2.f * TB_PI * u2;
    const float2 sc = tb_sincosf(phi);
    const float s = sc.x, c = sc.y;
    return v3(r * c, r * s, z);
}

// UniformSampleHemisphere(Random&), maths.h:1291-1302
TB_DEV V3 uniform_sample_hemisphere(Rng& rng)
{
    const float z = rng_float(rng);
    const float w = sqrtf(1.0f - z * z);
    const float phi = TB_2PI * rng_float(rng);
    const float2 sc = tb_sincosf(phi);
    const float s = sc.x, c = sc.y;
    return v3(c * w, s * w, z);
}

// CosineSampleHemisphere, maths.h:1319-1325 via UniformSampleDisc, maths.h:1304-1310
TB_DEV V3 cosine_sample_hemisphere(float u1, float u2)
{
    const float r = sqrtf(u1);
    const float theta = TB_2PI * u2;
    const float2 sc = tb_sincosf(theta);
    const float s = sc.x, c = sc.y;
    const float sx = r * c, sy = r * s;
    const float z = sqrtf(tb_max(0.0f, 1.0f - sx * sx - sy * sy));
    return v3(sx, sy, z);
}
