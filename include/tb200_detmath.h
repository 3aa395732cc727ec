/*
 * tb200_detmath.h -- deterministic single-precision transcendentals, identical on host and device.
 *
 * tinsel's hot path calls libm's sinf/cosf/expf/acosf/atan2f (src/disney.h:189-190,
 * src/maths.h:253,1282-1284,1298-1299,1309, src/probe.h:107-108,120-122,150,228,
 * src/render.h:31).  glibc and CUDA libdevice round these differently in ~0.1-1 % of calls,
 * which is enough to flip `rand < F`-style branches, so neither is usable for per-sample
 * parity.  These versions evaluate in IEEE double with only +,-,*,/,sqrt,rint (bit-identical
 * on x86-64 and sm_90a as long as no FMA contraction happens: build with -fmad=false /
 * -ffp-contract=off) and round once to float.  The double result is accurate to < 1e-15
 * relative, so the float result is the correctly rounded one except with probability ~1e-7;
 * glibc 2.39's own float functions are "nearly always" correctly rounded too, hence the two
 * agree to the last bit in > 99.8 % of calls (tests/test_detmath.py measures it).
 *
 * Used by: the CUDA kernels, the oracle port, and the "detmath" flavour of oracle/_ref (the
 * reference's own source compiled with these substituted for libm).
 */
#ifndef TB200_DETMATH_H
#define TB200_DETMATH_H

#include <stdint.h>
#include <string.h>
#include <math.h>

#if defined(__CUDACC__)
#define TBM_HD __host__ __device__ __forceinline__
#else
#define TBM_HD static inline
#endif

#if defined(__CUDA_ARCH__)
#define TBM_MUL(a, b) __dmul_rn((a), (b))
#define TBM_ADD(a, b) __dadd_rn((a), (b))
#define TBM_SUB(a, b) __dsub_rn((a), (b))
#define TBM_DIV(a, b) __ddiv_rn((a), (b))
#define TBM_SQRT(a) __dsqrt_rn((a))
#else
#define TBM_MUL(a, b) ((a) * (b))
#define TBM_ADD(a, b) ((a) + (b))
#define TBM_SUB(a, b) ((a) - (b))
#define TBM_DIV(a, b) ((a) / (b))
#define TBM_SQRT(a) sqrt((a))
#endif

/* p*z + c without contraction */
#define TBM_HORNER(p, z, c) TBM_ADD(TBM_MUL((p), (z)), (c))

TBM_HD double tbm_bits_to_double(uint64_t u)
{
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double d;
    memcpy(&d, &u, 8);
    return d;
#endif
}

/* sin and cos of a double argument of moderate size (|x| < 1e6), both to < 1e-16 absolute. */
TBM_HD void tbm_sincos_d(double x, double* s, double* c)
{
    if (!(fabs(x) < 1.0e6)) {
        /* inf/nan -> nan.  Huge finite arguments never occur on the hot path (phases are at
         * most a few pi); they get an arbitrary but deterministic answer. */
        *s = x - x;
        *c = (x - x) + 1.0;
        return;
    }
    const double kd = rint(TBM_MUL(x, 0.6366197723675814 /* 2/pi */));
    /* Cody-Waite: pi/2 = P1 + P2, P1 has 33 significant bits so kd*P1 is exact */
    double r = TBM_SUB(x, TBM_MUL(kd, 1.5707963267341256));
    r = TBM_SUB(r, TBM_MUL(kd, 6.077100506506192e-11));
    const double z = TBM_MUL(r, r);

    /* sin r = r + r*z*(S1 + z*(S2 + ...)), Taylor to r^17 */
    double ps = -2.8114572543455206e-15; /* -1/17! */
    ps = TBM_HORNER(ps, z, 7.6471637318198164e-13);  /*  1/15! */
    ps = TBM_HORNER(ps, z, -1.6059043836821613e-10); /* -1/13! */
    ps = TBM_HORNER(ps, z, 2.5052108385441720e-08);  /*  1/11! */
    ps = TBM_HORNER(ps, z, -2.7557319223985893e-06); /* -1/9!  */
    ps = TBM_HORNER(ps, z, 1.9841269841269841e-04);  /*  1/7!  */
    ps = TBM_HORNER(ps, z, -8.3333333333333332e-03); /* -1/5!  */
    ps = TBM_HORNER(ps, z, 1.6666666666666666e-01);  /*  1/3! (sign applied below) */
    /* note: signs alternate; the chain above already carries them except the last */
    const double sr = TBM_SUB(r, TBM_MUL(TBM_MUL(r, z), ps));

    /* cos r = 1 - z/2 + z^2*(C1 + z*(C2 + ...)), Taylor to r^18 */
    double pc = -1.5619206968586226e-16; /* -1/18! */
    pc = TBM_HORNER(pc, z, 4.7794773323873853e-14);  /*  1/16! */
    pc = TBM_HORNER(pc, z, -1.1470745597729725e-11); /* -1/14! */
    pc = TBM_HORNER(pc, z, 2.0876756987868100e-09);  /*  1/12! */
    pc = TBM_HORNER(pc, z, -2.7557319223985888e-07); /* -1/10! */
    pc = TBM_HORNER(pc, z, 2.4801587301587302e-05);  /*  1/8!  */
    pc = TBM_HORNER(pc, z, -1.3888888888888889e-03); /* -1/6!  */
    pc = TBM_HORNER(pc, z, 4.1666666666666664e-02);  /*  1/4!  */
    const double cr = TBM_ADD(TBM_SUB(1.0, TBM_MUL(0.5, z)), TBM_MUL(TBM_MUL(z, z), pc));

    const int n = ((int)kd) & 3;
    if (n == 0) { *s = sr; *c = cr; }
    else if (n == 1) { *s = cr; *c = -sr; }
    else if (n == 2) { *s = -sr; *c = -cr; }
    else { *s = -cr; *c = sr; }
}

/* sin(-0) gives +0, not C99's -0 (r = -0 - kd*P1 with kd = -0 is +0).  No caller passes -0: every phase is a product of
 * non-negative draws or uv coordinates (tb_shade.cuh, tb_math.cuh's sampling warps), so a select on the hot path would
 * only serve a case that cannot occur.  Every other |x| < 1e6 gives the correctly rounded value. */
TBM_HD float tbm_sinf(float x)
{
    double s, c;
    tbm_sincos_d((double)x, &s, &c);
    return (float)s;
}

TBM_HD float tbm_cosf(float x)
{
    double s, c;
    tbm_sincos_d((double)x, &s, &c);
    return (float)c;
}

TBM_HD void tbm_sincosf(float x, float* s, float* c)
{
    double sd, cd;
    tbm_sincos_d((double)x, &sd, &cd);
    *s = (float)sd;
    *c = (float)cd;
}

TBM_HD float tbm_expf(float xf)
{
    const double x = (double)xf;
    if (!(x == x)) return xf;
    if (x > 100.0) return (float)(1.0e300 * 1.0e300); /* +inf */
    if (x < -110.0) return 0.0f;
    const double kd = rint(TBM_MUL(x, 1.4426950408889634 /* log2(e) */));
    double r = TBM_SUB(x, TBM_MUL(kd, 0.6931471803691238));
    r = TBM_SUB(r, TBM_MUL(kd, 1.9082149292705877e-10));
    /* e^r, |r| <= 0.347, Taylor to r^13 */
    double p = 1.6059043836821613e-10;           /* 1/13! */
    p = TBM_HORNER(p, r, 2.0876756987868100e-09); /* 1/12! */
    p = TBM_HORNER(p, r, 2.5052108385441720e-08); /* 1/11! */
    p = TBM_HORNER(p, r, 2.7557319223985888e-07); /* 1/10! */
    p = TBM_HORNER(p, r, 2.7557319223985893e-06); /* 1/9!  */
    p = TBM_HORNER(p, r, 2.4801587301587302e-05); /* 1/8!  */
    p = TBM_HORNER(p, r, 1.9841269841269841e-04); /* 1/7!  */
    p = TBM_HORNER(p, r, 1.3888888888888889e-03); /* 1/6!  */
    p = TBM_HORNER(p, r, 8.3333333333333332e-03); /* 1/5!  */
    p = TBM_HORNER(p, r, 4.1666666666666664e-02); /* 1/4!  */
    p = TBM_HORNER(p, r, 1.6666666666666666e-01); /* 1/3!  */
    p = TBM_HORNER(p, r, 0.5);
    p = TBM_HORNER(p, r, 1.0);
    p = TBM_HORNER(p, r, 1.0);
    const int k = (int)kd;
    const double scale = tbm_bits_to_double((uint64_t)(k + 1023) << 52);
    return (float)TBM_MUL(p, scale);
}

/* atan(q) for q in [0,1]: q = c + delta with c = i/16, atan(q) = atan(c) + atan((q-c)/(1+q*c)) */
TBM_HD double tbm_atan_unit_d(double q)
{
    const int i = (int)rint(TBM_MUL(q, 16.0));
    double base;
    switch (i) {
        case 0: base = 0.0; break;
        case 1: base = 0.06241880999595735; break;
        case 2: base = 0.12435499454676144; break;
        case 3: base = 0.18534794999569476; break;
        case 4: base = 0.24497866312686414; break;
        case 5: base = 0.3028848683749714; break;
        case 6: base = 0.35877067027057225; break;
        case 7: base = 0.4124104415973873; break;
        case 8: base = 0.4636476090008061; break;
        case 9: base = 0.5123894603107377; break;
        case 10: base = 0.5585993153435624; break;
        case 11: base = 0.6022873461349642; break;
        case 12: base = 0.6435011087932844; break;
        case 13: base = 0.6823165548747481; break;
        case 14: base = 0.7188299996216245; break;
        case 15: base = 0.7531512809621944; break;
        default: base = 0.7853981633974483; break;
    }
    const double c = TBM_MUL((double)i, 0.0625);
    const double u = TBM_DIV(TBM_SUB(q, c), TBM_ADD(1.0, TBM_MUL(q, c)));
    const double z = TBM_MUL(u, u);
    /* atan u = u - u^3/3 + u^5/5 - ... - u^15/15, |u| <= 1/32 */
    double p = -6.6666666666666666e-02;            /* -1/15 */
    p = TBM_HORNER(p, z, 7.6923076923076927e-02);  /*  1/13 */
    p = TBM_HORNER(p, z, -9.0909090909090912e-02); /* -1/11 */
    p = TBM_HORNER(p, z, 1.1111111111111110e-01);  /*  1/9  */
    p = TBM_HORNER(p, z, -1.4285714285714285e-01); /* -1/7  */
    p = TBM_HORNER(p, z, 2.0000000000000001e-01);  /*  1/5  */
    p = TBM_HORNER(p, z, -3.3333333333333331e-01); /* -1/3  */
    const double au = TBM_ADD(u, TBM_MUL(TBM_MUL(u, z), p));
    return TBM_ADD(base, au);
}

/* atan2(y, x) in double for finite arguments, with the C99 signed-zero conventions */
TBM_HD double tbm_atan2_d(double y, double x)
{
    const double kPiD = 3.141592653589793;
    const double kHalfPiD = 1.5707963267948966;
    const double ay = fabs(y), ax = fabs(x);
    double a;
    if (ax == 0.0 && ay == 0.0) a = 0.0;
    else if (ay <= ax) a = tbm_atan_unit_d(TBM_DIV(ay, ax));
    else a = TBM_SUB(kHalfPiD, tbm_atan_unit_d(TBM_DIV(ax, ay)));
    if (signbit(x)) a = TBM_SUB(kPiD, a);
    return signbit(y) ? -a : a;
}

TBM_HD float tbm_atan2f(float y, float x)
{
    if (!(y == y) || !(x == x)) return y + x;
    double yd = (double)y, xd = (double)x;
    /* C99 F.9.1.4: atan2(+-inf, +inf) = +-pi/4 and atan2(+-inf, -inf) = +-3pi/4, which are atan2(+-1, +-1); inf/inf
     * would give NaN.  One call site, so that the inlined atan2 is not duplicated. */
    const double kInfD = tbm_bits_to_double(0x7ff0000000000000ull);
    if (fabs(yd) == kInfD && fabs(xd) == kInfD) {
        yd = copysign(1.0, yd);
        xd = copysign(1.0, xd);
    }
    return (float)tbm_atan2_d(yd, xd);
}

TBM_HD float tbm_acosf(float xf)
{
    const double x = (double)xf;
    if (!(fabs(x) <= 1.0)) return (float)tbm_bits_to_double(0x7ff8000000000000ull); /* nan, like libm for |x|>1 */
    /* acos x = atan2(sqrt((1-x)(1+x)), x); 1-x and 1+x are exact in double for float x */
    const double s = TBM_SQRT(TBM_MUL(TBM_SUB(1.0, x), TBM_ADD(1.0, x)));
    return (float)tbm_atan2_d(s, x);
}

/* ---- powf ----------------------------------------------------------------------------------
 * Used by the display/finish step (ToneMap -> SrgbToLinear -> LinearToSrgb, util.h:25-42,
 * maths.h:1545-1555): pow(x, y) = exp(y * log x) evaluated in double, rounded once to float. */

/* e^x in double for |x| <= 745 (same reduction and polynomial as tbm_expf) */
TBM_HD double tbm_exp_d(double x)
{
    const double kd = rint(TBM_MUL(x, 1.4426950408889634 /* log2(e) */));
    double r = TBM_SUB(x, TBM_MUL(kd, 0.6931471803691238));
    r = TBM_SUB(r, TBM_MUL(kd, 1.9082149292705877e-10));
    double p = 1.6059043836821613e-10;           /* 1/13! */
    p = TBM_HORNER(p, r, 2.0876756987868100e-09); /* 1/12! */
    p = TBM_HORNER(p, r, 2.5052108385441720e-08); /* 1/11! */
    p = TBM_HORNER(p, r, 2.7557319223985888e-07); /* 1/10! */
    p = TBM_HORNER(p, r, 2.7557319223985893e-06); /* 1/9!  */
    p = TBM_HORNER(p, r, 2.4801587301587302e-05); /* 1/8!  */
    p = TBM_HORNER(p, r, 1.9841269841269841e-04); /* 1/7!  */
    p = TBM_HORNER(p, r, 1.3888888888888889e-03); /* 1/6!  */
    p = TBM_HORNER(p, r, 8.3333333333333332e-03); /* 1/5!  */
    p = TBM_HORNER(p, r, 4.1666666666666664e-02); /* 1/4!  */
    p = TBM_HORNER(p, r, 1.6666666666666666e-01); /* 1/3!  */
    p = TBM_HORNER(p, r, 0.5);
    p = TBM_HORNER(p, r, 1.0);
    p = TBM_HORNER(p, r, 1.0);
    /* 2^k in two factors so that results in the float-denormal range stay exact powers of two */
    const int k = (int)kd;
    const int k1 = k / 2, k2 = k - k1;
    const double s1 = tbm_bits_to_double((uint64_t)(k1 + 1023) << 52);
    const double s2 = tbm_bits_to_double((uint64_t)(k2 + 1023) << 52);
    return TBM_MUL(TBM_MUL(p, s1), s2);
}

/* log x in double for finite x > 0 (x a normal double): x = m 2^e, m in [sqrt(.5), sqrt 2),
 * log m = 2 atanh(s), s = (m-1)/(m+1), |s| <= 0.1716, odd series to s^25 */
TBM_HD double tbm_log_d(double x)
{
    uint64_t u;
#if defined(__CUDA_ARCH__)
    u = (uint64_t)__double_as_longlong(x);
#else
    memcpy(&u, &x, sizeof(u));
#endif
    int e = (int)((u >> 52) & 0x7ffu) - 1023;
    uint64_t mant = u & 0x000fffffffffffffull;
    /* mantissa bits above sqrt(2)-1 go to the next binade: m in [sqrt(.5), sqrt 2) */
    if (mant > 0x6a09e667f3bcdull) e += 1;
    const double m = tbm_bits_to_double(mant | ((mant > 0x6a09e667f3bcdull ? 1022ull : 1023ull) << 52));
    const double f = TBM_SUB(m, 1.0);
    const double sq = TBM_DIV(f, TBM_ADD(m, 1.0));
    const double z = TBM_MUL(sq, sq);
    double p = 8.0000000000000002e-02;            /* 2/25 */
    p = TBM_HORNER(p, z, 8.6956521739130432e-02); /* 2/23 */
    p = TBM_HORNER(p, z, 9.5238095238095233e-02); /* 2/21 */
    p = TBM_HORNER(p, z, 1.0526315789473684e-01); /* 2/19 */
    p = TBM_HORNER(p, z, 1.1764705882352941e-01); /* 2/17 */
    p = TBM_HORNER(p, z, 1.3333333333333333e-01); /* 2/15 */
    p = TBM_HORNER(p, z, 1.5384615384615385e-01); /* 2/13 */
    p = TBM_HORNER(p, z, 1.8181818181818182e-01); /* 2/11 */
    p = TBM_HORNER(p, z, 2.2222222222222221e-01); /* 2/9  */
    p = TBM_HORNER(p, z, 2.8571428571428570e-01); /* 2/7  */
    p = TBM_HORNER(p, z, 4.0000000000000002e-01); /* 2/5  */
    p = TBM_HORNER(p, z, 6.6666666666666663e-01); /* 2/3  */
    /* log m = 2 s + s^3 p */
    const double lm = TBM_ADD(TBM_MUL(2.0, sq), TBM_MUL(TBM_MUL(sq, z), p));
    const double ed = (double)e;
    return TBM_ADD(TBM_MUL(ed, 0.6931471803691238), TBM_ADD(TBM_MUL(ed, 1.9082149292705877e-10), lm));
}

TBM_HD float tbm_powf(float xf, float yf)
{
    const double x = (double)xf, y = (double)yf;
    const double kInfD = tbm_bits_to_double(0x7ff0000000000000ull);
    if (y == 0.0 || x == 1.0) return 1.0f;                     /* C99: also for NaN in the other argument */
    if (!(x == x) || !(y == y)) return xf + yf;
    const int yIsInt = (fabs(y) >= 9007199254740992.0) || (rint(y) == y);
    const int yIsOdd = yIsInt && fabs(y) < 9007199254740992.0 && (rint(TBM_MUL(y, 0.5)) != TBM_MUL(y, 0.5));
    if (fabs(y) == kInfD) {
        const double ax = fabs(x);
        if (ax == 1.0) return 1.0f;
        return ((ax > 1.0) == (y > 0.0)) ? (float)kInfD : 0.0f;
    }
    if (x == 0.0 || fabs(x) == kInfD) {
        const int big = (fabs(x) == kInfD) == (y > 0.0);       /* result magnitude inf (else 0) */
        const double mag = big ? kInfD : 0.0;
        return (float)((signbit(x) && yIsOdd) ? -mag : mag);
    }
    if (x < 0.0 && !yIsInt) return (float)tbm_bits_to_double(0x7ff8000000000000ull);
    const double t = TBM_MUL(y, tbm_log_d(fabs(x)));
    double r;
    if (t > 100.0) r = kInfD;
    else if (t < -110.0) r = 0.0;
    else r = tbm_exp_d(t);
    return (float)((x < 0.0 && yIsOdd) ? -r : r);
}

#endif /* TB200_DETMATH_H */
