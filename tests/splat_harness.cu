// splat_harness.cu -- TEST INFRASTRUCTURE: the film's splat (tinsel_b200/csrc/tb_film.cuh) one case per thread, each
// into its own film, so that every term add_sample or add_sample_small writes can be read back alone and compared
// with the CPU restatement bit for bit.  tests/test_splat_gpu.py compiles it with the library's own nvcc flags
// (tinsel_b200.build) into a temporary directory and loads it with ctypes.
#include "tb_film.cuh"

// one case; CASE_DTYPE in tests/test_splat_gpu.py has the same layout
struct SplatCase {
    int32_t width, height, filterType, rowLo, rowHi;
    float filterWidth, filterFalloff, filterOffset, clamp, filterArgZero;
    float rasterX, rasterY, r, g, b, pad;
};

enum { SPLAT_ADD_SAMPLE = 0, SPLAT_ADD_SAMPLE_SMALL = 1, SPLAT_ADD_SAMPLE_NO_SHORTCUT = 2 };

// case k splats into films + k * stride + guard: its film of width x height pixels lies between zeroed guard zones
__global__ void splat_cases(const SplatCase* cases, int n, float4* films, long long stride, long long guard, int mode)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const SplatCase c = cases[k];
    DFilm f;
    f.width = c.width;
    f.height = c.height;
    f.filterType = c.filterType;
    f.filterWidth = c.filterWidth;
    f.filterFalloff = c.filterFalloff;
    f.filterOffset = c.filterOffset;
    f.clamp = c.clamp;
    f.maxDepth = 0;
    f.filterArgZero = mode == SPLAT_ADD_SAMPLE_NO_SHORTCUT ? -INFINITY : c.filterArgZero;
    f.rowLo = c.rowLo;
    f.rowHi = c.rowHi;
    float4* film = films + k * stride + guard;
    if (mode == SPLAT_ADD_SAMPLE_SMALL)
        add_sample_small(f, film, c.rasterX, c.rasterY, v3(c.r, c.g, c.b));
    else
        add_sample(f, film, c.rasterX, c.rasterY, v3(c.r, c.g, c.b));
}

extern "C" {

// the renderer's DFilm::filterArgZero rule (film_filter_arg_zero, as fill_params applies it) for n offsets
void splat_filter_arg_zero(const float* offsets, float* out, int n)
{
    for (int k = 0; k < n; ++k) out[k] = film_filter_arg_zero(offsets[k]);
}

// cases, films: device pointers; films holds n * stride float4, zeroed by the caller.  Returns a cudaError_t.
int splat_run(const void* cases, int n, void* films, long long stride, long long guard, int mode)
{
    if (n > 0) splat_cases<<<(n + 127) / 128, 128>>>((const SplatCase*)cases, n, (float4*)films, stride, guard, mode);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

}
