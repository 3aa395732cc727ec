// math_host.cpp -- TEST INFRASTRUCTURE: the host arm of tests/test_detmath_gpu.py.  Given a chunk of the device's
// results (tests/math_harness.cu), it recomputes every value with the host build of include/tb200_detmath.h (built
// with the CPU restatement's flags, -ffp-contract=off) and with glibc's double function rounded once to float, on a
// few threads, and returns per class of failure a count and the first failing positions, so that the 2^32 results of
// a function never have to pass through numpy.
#include "tb200_detmath.h"

#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

// failure classes: counts[k] and fails[k * MATH_MAX_FAILS ...]
enum {
    MATH_DEVICE = 0,    // a device result differs from the host build (a NaN matches any NaN, all else bit for bit)
    MATH_REF = 1,       // the host build differs from float64 rounded once, outside the documented exceptions
    MATH_BIG = 2,       // sincos: finite |x| >= 1e6, where the host build gives exactly (+0, 1) (counted, not failures)
    MATH_NEG_ZERO = 3,  // sincos: x = -0, where the host build gives exactly (+0, 1) (counted, not a failure)
    MATH_ORDER = 4,     // exp: a result below the one of the next smaller input
    MATH_NEAR_TIE = 5,  // pow: 1 ulp from float64 rounded once, which lies within the header's error of a midpoint
    MATH_CLASSES = 6,
    MATH_MAX_FAILS = 8,
};
// the host functions of math_check_unary
enum { HOST_SINCOS, HOST_EXP, HOST_ACOS };
// math_check_binary's functions (math_binary's numbers in math_harness.cu)
enum { HOST_ATAN2, HOST_POW };
// math_double_host's functions (math_double's numbers in math_harness.cu)
enum { HOST_SINCOS_D, HOST_EXP_D, HOST_LOG_D, HOST_ATAN2_D };

static inline uint32_t bits_of(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
}

static inline float float_of(uint32_t u)
{
    float f;
    memcpy(&f, &u, 4);
    return f;
}

static inline bool same(float a, float b) { return (std::isnan(a) && std::isnan(b)) || bits_of(a) == bits_of(b); }

struct Tally {
    long long counts[MATH_CLASSES] = {};
    std::vector<long long> fails[MATH_CLASSES];
    void add(int k, long long i)
    {
        if ((int)fails[k].size() < MATH_MAX_FAILS) fails[k].push_back(i);
        counts[k]++;
    }
};

// runs body(lo, hi, tally) over [0, n) on nthreads threads and merges the tallies in order of position
template <class F>
static void run(long long n, int nthreads, long long* counts, long long* fails, F body)
{
    if (nthreads < 1) nthreads = 1;
    std::vector<Tally> t(nthreads);
    std::vector<std::thread> th;
    for (int k = 0; k < nthreads; ++k)
        th.emplace_back([&, k]() { body(n * k / nthreads, n * (k + 1) / nthreads, t[k]); });
    for (auto& x : th) x.join();
    for (int c = 0; c < MATH_CLASSES; ++c) {
        int m = 0;
        counts[c] = 0;
        for (int k = 0; k < nthreads; ++k) {
            counts[c] += t[k].counts[c];
            for (long long i : t[k].fails[c])
                if (m < MATH_MAX_FAILS) fails[c * MATH_MAX_FAILS + m++] = i;
        }
        for (; m < MATH_MAX_FAILS; ++m) fails[c * MATH_MAX_FAILS + m] = -1;
    }
}

extern "C" {

// The floats whose bits are first + i, i < n.  dev[j] (j < ndev) holds the device's results of one variant of host
// function fn, output which[j] of it (HOST_SINCOS: 0 the sine, 1 the cosine; otherwise 0); ndev >= 1.  counts:
// MATH_CLASSES counts; fails: MATH_MAX_FAILS positions i per class, -1 where there are fewer failures.  The order of
// HOST_EXP's results is checked within the chunk; the caller checks it across chunks.
void math_check_unary(int fn, uint32_t first, long long n, const float* const* dev, const int* which, int ndev,
                      int nthreads, long long* counts, long long* fails)
{
    run(n, nthreads, counts, fails, [&](long long lo, long long hi, Tally& t) {
        for (long long i = lo; i < hi; ++i) {
            const uint32_t u = first + (uint32_t)i;
            const float x = float_of(u);
            float h[2];
            bool ok = true;
            if (fn == HOST_SINCOS) {
                tbm_sincosf(x, &h[0], &h[1]);
                if (!std::isfinite(x)) {
                    ok = std::isnan(h[0]) && std::isnan(h[1]);   // sin, cos(+-inf or NaN) are NaN
                } else if (std::fabs(x) >= 1.0e6f) {
                    ok = bits_of(h[0]) == 0u && bits_of(h[1]) == 0x3f800000u;
                    if (ok) t.add(MATH_BIG, i);
                } else if (u == 0x80000000u) {
                    ok = bits_of(h[0]) == 0u && bits_of(h[1]) == 0x3f800000u;
                    if (ok) t.add(MATH_NEG_ZERO, i);
                } else {
                    ok = same(h[0], (float)std::sin((double)x)) && same(h[1], (float)std::cos((double)x));
                }
            } else if (fn == HOST_EXP) {
                h[0] = tbm_expf(x);
                ok = same(h[0], (float)std::exp((double)x));
                // the device's first variant at x and at the next float away from zero (bits u + 1): the value
                // increases with the bits for +x and decreases for -x.  +-inf and NaN have no such neighbour.
                if (i + 1 < n && (u & 0x7fffffffu) < 0x7f800000u) {
                    const float a = dev[0][i], b = dev[0][i + 1];
                    if (!((u & 0x80000000u) ? b <= a : a <= b)) t.add(MATH_ORDER, i);
                }
            } else {
                h[0] = tbm_acosf(x);
                ok = std::fabs(x) <= 1.0f ? same(h[0], (float)std::acos((double)x)) : std::isnan(h[0]);
            }
            if (!ok) t.add(MATH_REF, i);
            for (int j = 0; j < ndev; ++j)
                if (!same(dev[j][i], h[which[j]])) {
                    t.add(MATH_DEVICE, i);
                    break;
                }
        }
    });
}

// math_double on the host: a[i] (and b[i]) = the double-precision core fn at x[i] (and y[i])
void math_double_host(int fn, const double* x, const double* y, long long n, double* a, double* b)
{
    for (long long i = 0; i < n; ++i) {
        if (fn == HOST_SINCOS_D) tbm_sincos_d(x[i], &a[i], &b[i]);
        else if (fn == HOST_EXP_D) a[i] = tbm_exp_d(x[i]);
        else if (fn == HOST_LOG_D) a[i] = tbm_log_d(x[i]);
        else a[i] = tbm_atan2_d(x[i], y[i]);
    }
}

// dev[i]: the device's tbm_atan2f(x[i], y[i]) (HOST_ATAN2) or tbm_powf(x[i], y[i]) (HOST_POW).  counts and fails as
// for math_check_unary, MATH_DEVICE, MATH_REF and MATH_NEAR_TIE only, with positions that index the arrays.
void math_check_binary(int fn, const float* x, const float* y, long long n, const float* dev, int nthreads,
                       long long* counts, long long* fails)
{
    run(n, nthreads, counts, fails, [&](long long lo, long long hi, Tally& t) {
        for (long long i = lo; i < hi; ++i) {
            const float a = x[i], b = y[i];
            float h, r;
            double w = 0.0;
            if (fn == HOST_ATAN2) {
                h = tbm_atan2f(a, b);
                r = (float)std::atan2((double)a, (double)b);
            } else {
                h = tbm_powf(a, b);
                w = std::pow((double)a, (double)b);
                r = (float)w;
            }
            if (!same(h, r)) {
                // tbm_powf's exp(y log x) in double is within ~3e-14 relative of x^y (|y log x| < 110), so it
                // rounds to the neighbour of the correctly rounded float only when x^y is that close to a midpoint
                const long long d = (long long)bits_of(h) - (long long)bits_of(r);
                const double mid = 0.5 * ((double)h + (double)r);
                const bool nearTie = fn == HOST_POW && std::isfinite(h) && std::isfinite(r) && (d == 1 || d == -1) &&
                                     std::fabs(w - mid) <= 1e-13 * std::fabs(mid);
                t.add(nearTie ? MATH_NEAR_TIE : MATH_REF, i);
            }
            if (!same(dev[i], h)) t.add(MATH_DEVICE, i);
        }
    });
}

}
