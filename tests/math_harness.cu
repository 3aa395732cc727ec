// math_harness.cu -- TEST INFRASTRUCTURE: the math layer the kernels build on, one case per thread on the device:
// the single-precision transcendentals of include/tb200_detmath.h (inline, and through tb_math.cuh's out-of-line
// tb_sincosf / tb_expf the kernels call), the double-precision cores they round, tb_math.cuh's four transform
// functions and interpolate_transform.  The transforms also run on the host from this translation unit (nvcc's host
// build of the same header), and beside them the full quaternion arithmetic (maths.h:558-619) that their shortcuts
// stand for.  tests/test_detmath_gpu.py compiles it with the library's own nvcc flags (tinsel_b200.build) into a
// temporary directory and loads it with ctypes.
#include "tb_math.cuh"

// math_unary's functions; tests/test_detmath_gpu.py has the same numbers
enum { MATH_SINF, MATH_COSF, MATH_SINCOSF, MATH_EXPF, MATH_TB_EXPF, MATH_ACOSF };
// math_binary's functions; tests/test_detmath_gpu.py has the same numbers
enum { MATH_ATAN2F, MATH_POWF };
// math_double's functions: the double-precision cores, whose every bit must match the host build (a contraction or
// a changed reduction shows in their low bits long before it flips a rounded float); math_host.cpp and
// tests/test_detmath_gpu.py have the same numbers
enum { MATH_SINCOS_D, MATH_EXP_D, MATH_LOG_D, MATH_ATAN2_D };

__global__ void unary_cases(int fn, uint32_t firstBits, long long n, float* a, float* b)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float x = __uint_as_float(firstBits + (uint32_t)i);
        switch (fn) {
            case MATH_SINF: a[i] = tbm_sinf(x); break;
            case MATH_COSF: a[i] = tbm_cosf(x); break;
            case MATH_SINCOSF: {
                const float2 sc = tb_sincosf(x);
                a[i] = sc.x;
                b[i] = sc.y;
                break;
            }
            case MATH_EXPF: a[i] = tbm_expf(x); break;
            case MATH_TB_EXPF: a[i] = tb_expf(x); break;
            default: a[i] = tbm_acosf(x); break;
        }
    }
}

__global__ void binary_cases(int fn, const float* x, const float* y, long long n, float* out)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = fn == MATH_ATAN2F ? tbm_atan2f(x[i], y[i]) : tbm_powf(x[i], y[i]);
}

__global__ void double_cases(int fn, const double* x, const double* y, long long n, double* a, double* b)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        switch (fn) {
            case MATH_SINCOS_D: tbm_sincos_d(x[i], &a[i], &b[i]); break;
            case MATH_EXP_D: a[i] = tbm_exp_d(x[i]); break;
            case MATH_LOG_D: a[i] = tbm_log_d(x[i]); break;
            default: a[i] = tbm_atan2_d(x[i], y[i]); break;
        }
    }
}

// maths.h:601-619 without the shortcuts of rotate_xf and inverse_scale
TB_HD V3 full_tv(const Xf& t, V3 v) { return rotate(t.r, t.s * v); }
TB_HD V3 full_tp(const Xf& t, V3 v) { return t.p + rotate(t.r, t.s * v); }
TB_HD V3 full_itv(const Xf& t, V3 v) { return (1.0f / t.s) * rotate(qconj(t.r), v); }
TB_HD V3 full_itp(const Xf& t, V3 v) { return (1.0f / t.s) * rotate(qconj(t.r), v - t.p); }

// the 8 results of transform t on vector v: transform_vector, transform_point, inverse_transform_vector,
// inverse_transform_point, then the same four by the full arithmetic
TB_HD void transform_case(const Xf& t, V3 v, V3* out)
{
    out[0] = transform_vector(t, v);
    out[1] = transform_point(t, v);
    out[2] = inverse_transform_vector(t, v);
    out[3] = inverse_transform_point(t, v);
    out[4] = full_tv(t, v);
    out[5] = full_tp(t, v);
    out[6] = full_itv(t, v);
    out[7] = full_itp(t, v);
}

__global__ void transform_cases(const Xf* t, int nt, const V3* v, int nv, V3* out)
{
    const long long n = (long long)nt * nv;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        transform_case(t[i / nv], v[i % nv], out + 8 * i);
}

__global__ void interpolate_cases(const Xf* a, const Xf* b, const float* t, int n, Xf* out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = interpolate_transform(a[i], b[i], t[i]);
}

static int finish()
{
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

static const int kThreads = 256;
static int blocks(long long n)
{
    const long long b = (n + kThreads - 1) / kThreads;
    return (int)(b < 65536 ? (b > 0 ? b : 1) : 65536);
}

extern "C" {

int math_sizeof_xf() { return (int)sizeof(Xf); }

// Thread i evaluates function fn at the float whose bits are firstBits + i (wrapping), for i < n.  a, b: device
// arrays of n floats; b receives the cosine of MATH_SINCOSF and is not touched otherwise.  Returns a cudaError_t.
int math_unary(int fn, uint32_t firstBits, long long n, float* a, float* b)
{
    if (n > 0) unary_cases<<<blocks(n), kThreads>>>(fn, firstBits, n, a, b);
    return finish();
}

// out[i] = tbm_atan2f(x[i], y[i]) or tbm_powf(x[i], y[i]); device arrays.  Returns a cudaError_t.
int math_binary(int fn, const float* x, const float* y, long long n, float* out)
{
    if (n > 0) binary_cases<<<blocks(n), kThreads>>>(fn, x, y, n, out);
    return finish();
}

// a[i] (and b[i], the cosine of MATH_SINCOS_D) = the double-precision core fn at x[i] (and y[i] for MATH_ATAN2_D);
// device arrays.  Returns a cudaError_t.
int math_double(int fn, const double* x, const double* y, long long n, double* a, double* b)
{
    if (n > 0) double_cases<<<blocks(n), kThreads>>>(fn, x, y, n, a, b);
    return finish();
}

// Every transform t[0..nt) on every vector v[0..nv): out[(ti * nv + vi) * 8 + k] is transform_case's result k.
// Device arrays.  Returns a cudaError_t.
int math_transforms(const void* t, int nt, const void* v, int nv, void* out)
{
    if ((long long)nt * nv > 0) transform_cases<<<blocks((long long)nt * nv), kThreads>>>((const Xf*)t, nt, (const V3*)v, nv, (V3*)out);
    return finish();
}

// the same on the host, from this translation unit's host build of tb_math.cuh
void math_transforms_host(const void* t, int nt, const void* v, int nv, void* out)
{
    for (long long i = 0; i < (long long)nt * nv; ++i) transform_case(((const Xf*)t)[i / nv], ((const V3*)v)[i % nv], (V3*)out + 8 * i);
}

// out[i] = interpolate_transform(a[i], b[i], t[i]); device arrays.  Returns a cudaError_t.
int math_interpolate(const void* a, const void* b, const float* t, int n, void* out)
{
    if (n > 0) interpolate_cases<<<(n + kThreads - 1) / kThreads, kThreads>>>((const Xf*)a, (const Xf*)b, t, n, (Xf*)out);
    return finish();
}

// the same on the host
void math_interpolate_host(const void* a, const void* b, const float* t, int n, void* out)
{
    for (int i = 0; i < n; ++i) ((Xf*)out)[i] = interpolate_transform(((const Xf*)a)[i], ((const Xf*)b)[i], t[i]);
}

}
