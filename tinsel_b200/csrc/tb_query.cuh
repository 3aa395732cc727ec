// tb_query.cuh -- batched closest-hit ray query (tb200_trace_rays): Trace(scene, Ray(origin, dir, time)) of
// render.cpp:17-62 for every ray of a caller's batch, bit for bit, through the same trace_closest() the
// renderer runs; the same query reporting the hit triangle and its barycentric weights (tb200_trace_rays_tri); and
// the batched occlusion query (tb200_occluded_rays) over trace_occluded(); and the batched BSDF queries
// (tb200_bsdf_eval, tb200_bsdf_sample) over the renderer's Disney BSDF functions; and the two ends of a path: the
// renderer's camera samples (tb200_camera_rays, over camera_sample) and the film's splat (tb200_splat, over
// add_sample_small); and the light queries: next-event estimation (tb200_sample_lights, over nee_generate and
// nee_connect) and the sky of a miss (tb200_sky_eval, over sky_eval and probe_pdf); and the two draws NEE is made of:
// emitter samples (tb200_sample_emitters, over prim_sample) and probe samples (tb200_sample_probe, over
// probe_sample).  Included once, by kernels.cu.
//
// The ray queries and the NEE query run a persistent kernel: as many CTAs as the SMs hold at once, for the whole
// batch.  Their warps claim chunks of 32 records from a global counter: a static split would leave SMs idle, because
// a ray that hits a plane costs a few dozen instructions and one that walks a deep mesh BVH more than ten times that.

#define TB_QUERY_THREADS 256

// The body of the query kernels.  One copy of the scene descriptor per CTA: the walks take it by reference, and a
// per-thread copy would live in local memory.  The scene tables stay in global memory: staging the primitive
// records, scene-level BVH pairs and flat scene program in shared memory with TMA bulk copies, as k_wavefront2 does,
// measured no faster (DESIGN §5.6).  No mesh treelet either (the host leaves DScene::treelet null).
// Then one atomic per warp claims 32 consecutive records, and each lane hands its record's index to
// record(sc, i), which loads the record and writes its answer with streaming stores, so that the outputs do not
// evict mesh BVH lines from L2.
template <class Record>
static __device__ __forceinline__ void query_claim(const QueryParams& P, Record record)
{
    __shared__ struct { DScene scene; } S;
    if (threadIdx.x == 0) S.scene = P.scene;
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const unsigned long long n = (unsigned long long)P.numRays;
    for (;;) {
        unsigned long long base = 0ull;
        if (lane == 0) base = atomicAdd(P.counter, 32ull);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= n) break;
        const unsigned long long i = base + (unsigned long long)lane;
        if (i < n) record(S.scene, i);
    }
}

// query_claim over the ray records: each lane loads its ray (two 16-byte loads) and hands it to ray(sc, i, a, b).
template <class Ray>
static __device__ __forceinline__ void query_claim_rays(const QueryParams& P, Ray ray)
{
    query_claim(P, [&](const DScene& sc, unsigned long long i) { ray(sc, i, __ldg(&P.rays[2 * i]), __ldg(&P.rays[2 * i + 1])); });
}

// Closest hit (QueryKind::Closest) and, with TRI, closest hit with the hit triangle (QueryKind::ClosestTri):
// the same hits and primitives bit for bit, and with TRI the winner's triangle record from the same walk.
template <bool TRI>
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_trace_rays(const __grid_constant__ QueryParams P)
{
    // a: origin.xyz, time; b: dir.xyz, pad
    query_claim_rays(P, [&](const DScene& sc, unsigned long long i, float4 a, float4 b) {
        const TraceHit<TRI> h = trace_closest<TB_FEAT_ALL, TRI>(sc, v3(a.x, a.y, a.z), v3(b.x, b.y, b.z), a.w, true);
        // the walks leave a sphere's or plane's record unset, or holding an earlier mesh candidate's triangle
        int4 tri = make_int4(-1, 0, 0, 0);
        if constexpr (TRI) {
            if (h.prim >= 0 && sc.prims[h.prim].type == TB200_MESH)
                tri = make_int4(h.rec.tri, __float_as_int(h.rec.u), __float_as_int(h.rec.v), __float_as_int(h.rec.w));
        }
        __stcs(&P.hits[i], make_float4(h.t, h.n.x, h.n.y, h.n.z));
        __stcs(&P.prims[i], h.prim);
        if constexpr (TRI) __stcs(&P.tris[i], tri);
    });
}

// Occlusion (QueryKind::Occluded): per ray, whether Trace hits a primitive with t < tmax, the ray record's last
// float; trace_occluded() stops at the first blocker.
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_occluded_rays(const __grid_constant__ QueryParams P)
{
    // a: origin.xyz, time; b: dir.xyz, tmax
    query_claim_rays(P, [&](const DScene& sc, unsigned long long i, float4 a, float4 b) {
        const bool occ = trace_occluded<TB_FEAT_ALL>(sc, v3(a.x, a.y, a.z), v3(b.x, b.y, b.z), a.w, b.w);
        __stcs(&P.occluded[i], (unsigned char)occ);
    });
}

// bsdf_eval_pdf()'s body, inlined: that function is out of line and takes the material by reference, so the
// kernel's copy of it, whose flags it changes, would live in a 112-byte local-memory frame (DESIGN §5.1); inlined,
// the copy stays in registers.  bsdf_pdf() and bsdf_eval() are the functions bsdf_eval_pdf() calls.
static __device__ __forceinline__ BsdfValue query_eval_pdf(const DMaterial& mat, float etaI, float etaO, V3 N, V3 V, V3 L)
{
    BsdfValue r;
    r.pdf = bsdf_pdf<TB_FEAT_ALL>(mat, etaI, etaO, N, V, L);
    r.f = bsdf_eval<TB_FEAT_ALL>(mat, etaI, etaO, N, V, L);
    return r;
}

// The BSDF queries: BSDFEval + BSDFPdf (QueryKind::BsdfEval) or, with SAMPLE, one BSDFSample step of PathTrace
// followed by BSDFEval of the sampled direction (QueryKind::BsdfSample), per query record, bit for bit.
// Every query costs about the same (one BSDF call, no walk), so a grid-stride loop with one query per thread needs
// no work counter.  Each thread loads its record with three 16-byte loads and writes with streaming stores.
//
// The material is the primitive's DMaterial with TB_MAT_NO_FRESNEL and TB_MAT_NO_CLEARCOAT cleared: those skips are
// exact only for the etas and the front-facing unit vectors a path produces (tb_scene.cuh: make_material,
// set_fresnel_flags), and a caller may pass any.  TB_MAT_GTR1_WIDE picks GTR1's value, not a skip, and stays.  So
// the TB_FEAT_ALL instantiation runs the reference's full arithmetic.
template <bool SAMPLE>
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_bsdf_query(const __grid_constant__ QueryParams P)
{
    const unsigned long long n = (unsigned long long)P.numRays;
    const unsigned long long stride = (unsigned long long)gridDim.x * TB_QUERY_THREADS;
    for (unsigned long long i = (unsigned long long)blockIdx.x * TB_QUERY_THREADS + threadIdx.x; i < n; i += stride) {
        // a: n.xyz, prim bits; b: v.xyz, etaI; c: l.xyz, etaO
        const float4 a = __ldg(&P.bsdfQueries[3 * i]), b = __ldg(&P.bsdfQueries[3 * i + 1]);
        const float4 c = __ldg(&P.bsdfQueries[3 * i + 2]);
        const int prim = __float_as_int(a.w);
        const bool inScene = prim >= 0 && prim < P.scene.numPrims;
        DMaterial mat;
        if (inScene) {
            mat = P.scene.prims[prim].mat;
            mat.flags &= ~(uint32_t)(TB_MAT_NO_FRESNEL | TB_MAT_NO_CLEARCOAT);
        }
        const V3 N = v3(a.x, a.y, a.z), V = v3(b.x, b.y, b.z);
        if constexpr (!SAMPLE) {
            BsdfValue r = {v3s(0.0f), 0.0f};
            if (inScene) r = query_eval_pdf(mat, b.w, c.w, N, V, v3(c.x, c.y, c.z));
            __stcs(&P.bsdfValues[i], make_float4(r.f.x, r.f.y, r.f.z, r.pdf));
        } else {
            V3 L = v3s(0.0f), f = v3s(0.0f);
            float pdf = 0.0f;
            int type = -1;
            if (inScene) {
                // path_scatter (tb_shade.cuh), less its path state
                Rng rng = rng_seed(__ldg(&P.seeds[i]));
                V3 u, v;
                basis_from_vector(N, &u, &v);
                type = TB_REFLECTED;
                const bool pdfFromBsdf = bsdf_sample_dir<TB_FEAT_ALL>(mat, b.w, c.w, u, v, N, V, L, pdf, type, rng);
                if (pdfFromBsdf || pdf > 0.0f) {
                    const BsdfValue r = query_eval_pdf(mat, b.w, c.w, N, V, L);
                    f = r.f;
                    if (pdfFromBsdf) pdf = r.pdf;
                }
                if (!(pdf > 0.0f)) f = v3s(0.0f);   // PathTrace ends the path before it evaluates
            }
            __stcs(&P.bsdfSamples[2 * i], make_float4(L.x, L.y, L.z, pdf));
            __stcs(&P.bsdfSamples[2 * i + 1], make_float4(f.x, f.y, f.z, __int_as_float(type)));
        }
    }
}

// The camera rays (QueryKind::CameraRays): per sample record (pixel, frame), what sample_begin computes for that
// pixel in that frame (camera_sample), bit for bit.  A pixel outside [0, width*height) gets an all-zero ray, which
// trace_rays answers with a miss, and a NaN raster position, which k_splat skips.  Grid-stride, one sample per
// thread: one 8-byte load, three streaming stores.
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_camera_rays(const __grid_constant__ QueryParams P)
{
    const unsigned long long n = (unsigned long long)P.numRays;
    const unsigned long long stride = (unsigned long long)gridDim.x * TB_QUERY_THREADS;
    const int W = P.film.width;
    for (unsigned long long i = (unsigned long long)blockIdx.x * TB_QUERY_THREADS + threadIdx.x; i < n; i += stride) {
        const int2 s = __ldg(&P.cameraSamples[i]);   // pixel, frame
        float4 a = make_float4(0.0f, 0.0f, 0.0f, 0.0f), b = a;
        float2 raster = make_float2(__int_as_float(0x7fffffff), __int_as_float(0x7fffffff));
        if (s.x >= 0 && s.x < W * P.film.height) {   // the host refuses images of more than INT32_MAX pixels
            Rng rng;
            V3 o, d;
            float time;
            camera_sample(P.camera, W, s.x % W, s.x / W, (uint32_t)s.y, rng, o, d, time, raster.x, raster.y);
            a = make_float4(o.x, o.y, o.z, time);
            b = make_float4(d.x, d.y, d.z, __int_as_float(0x7f800000));   // +inf: occluded_rays reads it as tmax
        }
        __stcs(&P.cameraRays[2 * i], a);
        __stcs(&P.cameraRays[2 * i + 1], b);
        __stcs(&P.rasterOut[i], raster);
    }
}

// The splat (QueryKind::Splat): per sample, AddSample (render.cpp:401-445) of its radiance at its raster position
// into P.accum through add_sample_small, the lane-owned wavefront kernel's splat, over every row of the film.  A
// raster coordinate that is NaN or 2^30 or more in magnitude is skipped: AddSample's int conversion of
// raster +- filterWidth is undefined there (the host has refused filter widths of 2^30 or more).  Grid-stride, one
// sample per thread; the reductions go to L2 (tb_film.cuh: accum_add).
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_splat(const __grid_constant__ QueryParams P)
{
    const unsigned long long n = (unsigned long long)P.numRays;
    const unsigned long long stride = (unsigned long long)gridDim.x * TB_QUERY_THREADS;
    for (unsigned long long i = (unsigned long long)blockIdx.x * TB_QUERY_THREADS + threadIdx.x; i < n; i += stride) {
        const float2 r = __ldg(&P.rasterIn[i]);
        if (!(fabsf(r.x) < 1073741824.0f && fabsf(r.y) < 1073741824.0f)) continue;
        const V3 c = v3(__ldg(&P.radiance[3 * i]), __ldg(&P.radiance[3 * i + 1]), __ldg(&P.radiance[3 * i + 2]));
        add_sample_small(P.film, P.accum, r.x, r.y, c);
    }
}

// Next-event estimation (QueryKind::SampleLights): per surface record, SampleLights (render.cpp:103-227) from
// Random(seed), bit for bit, through k_mega's NEE loop: nee_begin, nee_generate over every primitive, a closest-hit
// shadow trace per sample and nee_connect.  The result is `sum`, which PathTrace multiplies by the throughput.  A
// prim outside [0, numPrims) gives zeros and traces nothing.  Every query of a scene takes the same number of shadow
// rays, but their walks differ in cost as the ray queries' do, so the records are claimed as rays are.
// The BSDF evaluations run on a copy of the surface's material with TB_MAT_NO_FRESNEL and TB_MAT_NO_CLEARCOAT
// cleared, as in k_bsdf_query and for the same reason: a caller may pass any etas and vectors.  bsdf_eval_pdf()
// takes that copy by reference and is out of line, so the copy lives in the kernel's local frame (DESIGN §5.11).
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_sample_lights(const __grid_constant__ QueryParams P)
{
    query_claim(P, [&](const DScene& sc, unsigned long long i) {
        // a: p.xyz, time; b: n.xyz, prim bits; c: wo.xyz, etaI; d: etaO, pad
        const float4 a = __ldg(&P.lightQueries[4 * i]), b = __ldg(&P.lightQueries[4 * i + 1]);
        const float4 c = __ldg(&P.lightQueries[4 * i + 2]), d = __ldg(&P.lightQueries[4 * i + 3]);
        const int prim = __float_as_int(b.w);
        NeeCursor cur;
        nee_begin(cur);
        if (prim >= 0 && prim < sc.numPrims) {
            Surface sf;
            sf.prim = prim;
            sf.p = v3(a.x, a.y, a.z);
            sf.n = v3(b.x, b.y, b.z);
            sf.wo = v3(c.x, c.y, c.z);
            sf.etaI = c.w;
            sf.etaO = d.x;
            sf.outAbsorb = v3s(0.0f);   // not read by NEE
            DMaterial mat = sc.prims[prim].mat;
            mat.flags &= ~(uint32_t)(TB_MAT_NO_FRESNEL | TB_MAT_NO_CLEARCOAT);
            Rng rng = rng_seed(__ldg(&P.seeds[i]));
            ShadowRay sr;
            while (nee_generate(sc, sf, a.w, cur, rng, sr)) {
                const Hit sh = trace_closest<TB_FEAT_ALL>(sc, sr.o, sr.d, a.w, false);
                nee_connect(sc, sf, sr, sh, cur, nullptr, &mat);
            }
        }
        __stcs(&P.lightRadiance[3 * i], cur.sum.x);
        __stcs(&P.lightRadiance[3 * i + 1], cur.sum.y);
        __stcs(&P.lightRadiance[3 * i + 2], cur.sum.z);
    });
}

// The sky of a miss (QueryKind::Sky): per ray, Sky::Eval(dir) and ProbePdf(dir) (scene.h:168-178, probe.h:136-160),
// bit for bit, with one ProbeDirToUV shared by both as in path_miss; pdf 0 for the gradient sky.  Only dir is read.
// Every query costs the same, so grid-stride, one ray per thread: one 16-byte load, one streaming store.
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_sky(const __grid_constant__ QueryParams P)
{
    const unsigned long long n = (unsigned long long)P.numRays;
    const unsigned long long stride = (unsigned long long)gridDim.x * TB_QUERY_THREADS;
    for (unsigned long long i = (unsigned long long)blockIdx.x * TB_QUERY_THREADS + threadIdx.x; i < n; i += stride) {
        const float4 b = __ldg(&P.rays[2 * i + 1]);   // dir.xyz, pad
        const V3 dir = v3(b.x, b.y, b.z);
        float u = 0.0f, v = 0.0f, pdf = 0.0f;
        if (P.scene.probe.valid) {
            const float2 uv = probe_dir_to_uv(dir);
            u = uv.x;
            v = uv.y;
            pdf = probe_pdf(P.scene.probe, u, v);
        }
        const V3 c = sky_eval<TB_FEAT_ALL>(P.scene, dir, u, v);
        __stcs(&P.skyOut[i], make_float4(c.x, c.y, c.z, pdf));
    }
}

// The emitter samples (QueryKind::SampleEmitters): per record (prim, time), PrimitiveSample (intersection.h:855-904)
// from Random(seed), bit for bit, through the prim_sample nee_generate calls, on the primitive record in global
// memory.  Only lights (lightSamples > 0) are sampled; any other prim, or one outside [0, numPrims), gives zeros and
// draws nothing.  A query costs at most one binary search of a mesh's CDF, so grid-stride, one record per thread:
// one 8-byte load, two streaming stores.
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_sample_emitters(const __grid_constant__ QueryParams P)
{
    const unsigned long long n = (unsigned long long)P.numRays;
    const unsigned long long stride = (unsigned long long)gridDim.x * TB_QUERY_THREADS;
    for (unsigned long long i = (unsigned long long)blockIdx.x * TB_QUERY_THREADS + threadIdx.x; i < n; i += stride) {
        const float2 q = __ldg(&P.emitterQueries[i]);   // prim bits, time
        const int prim = __float_as_int(q.x);
        V3 pos = v3s(0.0f), normal = v3s(0.0f);
        if (prim >= 0 && prim < P.scene.numPrims && P.scene.prims[prim].lightSamples > 0) {
            Rng rng = rng_seed(__ldg(&P.seeds[i]));
            prim_sample<TB_FEAT_ALL>(P.scene, P.scene.prims[prim], q.y, pos, normal, rng);
        }
        __stcs(&P.emitterOut[2 * i], make_float4(pos.x, pos.y, pos.z, 0.0f));
        __stcs(&P.emitterOut[2 * i + 1], make_float4(normal.x, normal.y, normal.z, 0.0f));
    }
}

// The probe samples (QueryKind::SampleProbe): per seed, ProbeSample (probe.h:205-236) from Random(seed), bit for
// bit, through the probe_sample nee_generate calls; zeros without a probe.  Two binary searches per seed, so
// grid-stride, one seed per thread: one 4-byte load, two streaming stores.
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_sample_probe(const __grid_constant__ QueryParams P)
{
    const unsigned long long n = (unsigned long long)P.numRays;
    const unsigned long long stride = (unsigned long long)gridDim.x * TB_QUERY_THREADS;
    for (unsigned long long i = (unsigned long long)blockIdx.x * TB_QUERY_THREADS + threadIdx.x; i < n; i += stride) {
        V3 dir = v3s(0.0f), color = v3s(0.0f);
        float pdf = 0.0f;
        if (P.scene.probe.valid) {
            Rng rng = rng_seed(__ldg(&P.seeds[i]));
            probe_sample(P.scene.probe, dir, color, pdf, rng);
        }
        __stcs(&P.probeOut[2 * i], make_float4(dir.x, dir.y, dir.z, pdf));
        __stcs(&P.probeOut[2 * i + 1], make_float4(color.x, color.y, color.z, 0.0f));
    }
}

void launch_query(QueryKind kind, const QueryParams& p, int numSMs, cudaStream_t stream, unsigned long long* launchCount)
{
    if (p.numRays <= 0) return;
    const bool perThread = kind != QueryKind::Closest && kind != QueryKind::ClosestTri && kind != QueryKind::Occluded &&
                           kind != QueryKind::SampleLights;
    void (*kernel)(QueryParams) = kind == QueryKind::Closest          ? k_trace_rays<false>
                                  : kind == QueryKind::ClosestTri     ? k_trace_rays<true>
                                  : kind == QueryKind::Occluded       ? k_occluded_rays
                                  : kind == QueryKind::BsdfEval       ? k_bsdf_query<false>
                                  : kind == QueryKind::BsdfSample     ? k_bsdf_query<true>
                                  : kind == QueryKind::CameraRays     ? k_camera_rays
                                  : kind == QueryKind::Splat          ? k_splat
                                  : kind == QueryKind::SampleLights   ? k_sample_lights
                                  : kind == QueryKind::Sky            ? k_sky
                                  : kind == QueryKind::SampleEmitters ? k_sample_emitters
                                                                      : k_sample_probe;
    // as many CTAs as the SMs hold at once, but no more than there are 32-ray chunks (the grid-stride queries: one
    // record per thread)
    int perSM = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, kernel, TB_QUERY_THREADS, 0) != cudaSuccess || perSM < 1) perSM = 1;
    const unsigned long long grid = (unsigned long long)(numSMs > 0 ? numSMs : 1) * (unsigned long long)perSM;
    unsigned long long needed;
    if (perThread) {
        needed = ((unsigned long long)p.numRays + TB_QUERY_THREADS - 1ull) / TB_QUERY_THREADS;
    } else {
        const unsigned long long chunks = ((unsigned long long)p.numRays + 31ull) / 32ull;
        const unsigned long long warps = (unsigned long long)TB_QUERY_THREADS / 32ull;
        needed = (chunks + warps - 1ull) / warps;
        cudaMemsetAsync(p.counter, 0, sizeof(unsigned long long), stream);
    }
    kernel<<<(unsigned)std::min(grid, needed), TB_QUERY_THREADS, 0, stream>>>(p);
    if (launchCount) ++*launchCount;
}
