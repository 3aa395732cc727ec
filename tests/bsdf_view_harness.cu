// bsdf_view_harness.cu -- TEST INFRASTRUCTURE: bsdf_eval_pdf (tinsel_b200/csrc/tb_shade.cuh) with and without the
// view terms a bounce computes once (bsdf_view), one case per thread, in both instantiations the kernels use
// (TB_FEAT_ALL and TB_FEAT_NONE), so that tests/test_bsdf_view_gpu.py can compare the two bit for bit.  The cases and
// materials are tests/bsdf_harness.cu's (struct BsdfCase, DMaterial records from bsdf_make_materials there).
// Compiled like that harness, with the library's own nvcc flags, into a temporary directory.
#include "tb_shade.cuh"

// struct BsdfCase in tests/bsdf_harness.cu
struct BsdfCase {
    int32_t mat, seed;
    float etaI, etaO;
    float n[3], v[3], l[3];
};

// one result; OUT_DTYPE in tests/test_bsdf_view_gpu.py has the same layout
struct ViewOut {
    float f[3], pdf;     // bsdf_eval_pdf(mat, etaI, etaO, N, V, L)
    float fv[3], pdfv;   // bsdf_eval_pdf(mat, etaI, etaO, N, V, L, bsdf_view(mat, N, V))
};

template <uint32_t FEAT>
__global__ void view_cases(const DMaterial* mats, const BsdfCase* cases, int n, ViewOut* out)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const BsdfCase c = cases[k];
    const DMaterial& m = mats[c.mat];
    const V3 N = v3(c.n[0], c.n[1], c.n[2]), V = v3(c.v[0], c.v[1], c.v[2]), L = v3(c.l[0], c.l[1], c.l[2]);
    const BsdfValue a = bsdf_eval_pdf<FEAT>(m, c.etaI, c.etaO, N, V, L);
    const BsdfValue b = bsdf_eval_pdf<FEAT>(m, c.etaI, c.etaO, N, V, L, bsdf_view<FEAT>(m, N, V));
    ViewOut o;
    o.f[0] = a.f.x; o.f[1] = a.f.y; o.f[2] = a.f.z;
    o.pdf = a.pdf;
    o.fv[0] = b.f.x; o.fv[1] = b.f.y; o.fv[2] = b.f.z;
    o.pdfv = b.pdf;
    out[k] = o;
}

extern "C" {

// mats, cases, out: device pointers; all: TB_FEAT_ALL, else TB_FEAT_NONE.  Returns a cudaError_t.
int view_run(const void* mats, const void* cases, int n, void* out, int all)
{
    if (n > 0) {
        if (all)
            view_cases<TB_FEAT_ALL><<<(n + 127) / 128, 128>>>((const DMaterial*)mats, (const BsdfCase*)cases, n, (ViewOut*)out);
        else
            view_cases<TB_FEAT_NONE><<<(n + 127) / 128, 128>>>((const DMaterial*)mats, (const BsdfCase*)cases, n, (ViewOut*)out);
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

}
