// bsdf_harness.cu -- TEST INFRASTRUCTURE: the Disney BSDF (tinsel_b200/csrc/tb_shade.cuh) one case per thread, in
// both instantiations the kernels use (TB_FEAT_ALL and TB_FEAT_NONE), so that every output of bsdf_pdf, bsdf_eval,
// bsdf_eval_pdf and bsdf_sample_dir can be compared with the CPU restatement bit for bit.  The materials go through
// the renderer's own host code (tb_scene.cuh: make_material, set_fresnel_flags, material_features).
// tests/test_bsdf_gpu.py compiles it with the library's own nvcc flags (tinsel_b200.build) into a temporary
// directory and loads it with ctypes.
#include "tb_shade.cuh"

// one case; CASE_DTYPE in tests/test_bsdf_gpu.py has the same layout
struct BsdfCase {
    int32_t mat, seed;
    float etaI, etaO;
    float n[3], v[3], l[3];
};

// one result; OUT_DTYPE in tests/test_bsdf_gpu.py has the same layout
struct BsdfOut {
    float f[3], pdf;           // bsdf_eval, bsdf_pdf
    float fp[3], pdfp;         // bsdf_eval_pdf
    float light[3], spdf;      // bsdf_sample_dir, then the pdf as path_scatter takes it
    int32_t type, fromBsdf;    // the sampled BSDFType; whether the pdf is BSDFPdf(light)
    uint32_t rng[2];           // the RNG state after sampling
};

template <uint32_t FEAT>
__global__ void bsdf_cases(const DMaterial* mats, const BsdfCase* cases, int n, BsdfOut* out)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const BsdfCase c = cases[k];
    const DMaterial& m = mats[c.mat];
    const V3 N = v3(c.n[0], c.n[1], c.n[2]), V = v3(c.v[0], c.v[1], c.v[2]), L = v3(c.l[0], c.l[1], c.l[2]);
    BsdfOut o;
    const V3 f = bsdf_eval<FEAT>(m, c.etaI, c.etaO, N, V, L);
    o.pdf = bsdf_pdf<FEAT>(m, c.etaI, c.etaO, N, V, L);
    const BsdfValue b = bsdf_eval_pdf<FEAT>(m, c.etaI, c.etaO, N, V, L);
    o.f[0] = f.x; o.f[1] = f.y; o.f[2] = f.z;
    o.fp[0] = b.f.x; o.fp[1] = b.f.y; o.fp[2] = b.f.z;
    o.pdfp = b.pdf;
    // path_scatter (tb_shade.cuh) with the case's surface
    V3 u, v;
    basis_from_vector(N, &u, &v);
    V3 dir = v3s(0.0f);
    int type = TB_REFLECTED;
    float pdf = 0.0f;
    Rng rng = rng_seed((uint32_t)c.seed);
    const bool fromBsdf = bsdf_sample_dir<FEAT>(m, c.etaI, c.etaO, u, v, N, V, dir, pdf, type, rng);
    if (fromBsdf) pdf = bsdf_eval_pdf<FEAT>(m, c.etaI, c.etaO, N, V, dir).pdf;
    o.light[0] = dir.x; o.light[1] = dir.y; o.light[2] = dir.z;
    o.spdf = pdf;
    o.type = type;
    o.fromBsdf = fromBsdf;
    o.rng[0] = rng.s1;
    o.rng[1] = rng.s2;
    out[k] = o;
}

extern "C" {

int bsdf_sizeof_material() { return (int)sizeof(DMaterial); }

// n materials in scenes of sceneSize consecutive ones (n a multiple of sceneSize): each through make_material, then
// set_fresnel_flags per scene, as api.cu builds a scene.  out receives the DMaterial records (bsdf_sizeof_material()
// bytes each); flags, features and ior (optional) each material's DMaterial::flags, material_features and ior.
void bsdf_make_materials(const tb200_material* mats, int n, int sceneSize, void* out, uint32_t* flags, uint32_t* features,
                         float* ior)
{
    DMaterial* d = (DMaterial*)out;
    for (int i = 0; i < n; ++i) d[i] = make_material(mats[i]);
    for (int s = 0; s + sceneSize <= n; s += sceneSize)
        set_fresnel_flags((size_t)sceneSize, [&](size_t i) -> DMaterial& { return d[s + i]; });
    for (int i = 0; i < n; ++i) {
        if (flags) flags[i] = d[i].flags;
        if (features) features[i] = material_features(d[i]);
        if (ior) ior[i] = d[i].ior;
    }
}

// mats, cases, out: device pointers; all: TB_FEAT_ALL, else TB_FEAT_NONE.  Returns a cudaError_t.
int bsdf_run(const void* mats, const void* cases, int n, void* out, int all)
{
    if (n > 0) {
        if (all)
            bsdf_cases<TB_FEAT_ALL><<<(n + 127) / 128, 128>>>((const DMaterial*)mats, (const BsdfCase*)cases, n, (BsdfOut*)out);
        else
            bsdf_cases<TB_FEAT_NONE><<<(n + 127) / 128, 128>>>((const DMaterial*)mats, (const BsdfCase*)cases, n, (BsdfOut*)out);
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

}
