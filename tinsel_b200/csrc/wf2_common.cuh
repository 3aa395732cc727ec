// wf2_common.cuh -- what the two wavefront kernels share: the slot state both keep, the scene staging prologue,
// stage R, the shading tail (wf2_surface, wf2_scatter) and the launcher.
//
// The product pipeline is a persistent, CTA-resident wavefront path tracer with a dedicated traversal stage.  One
// CTA per SM stays resident for the whole launch and owns TB_WF2_PATHS path slots whose inter-stage state stays on
// chip (or in L2).  A global-memory wavefront (tinsel's own unfinished wavefront.cu keeps ~150 B/path in DRAM and
// re-reads it in five kernels per bounce, wavefront.cu:765-796,1357-1375) would make queue traffic, not the scene,
// the HBM consumer; here HBM only sees scene misses and the framebuffer reductions.
//
// Every slot that is alive sits in exactly one CTA-shared stage queue.  Each WARP claims a chunk of up to 32 slots
// from a stage queue, processes it and appends the slots to the queues of their next stages:
//   R  finish + regenerate: splat the finished sample into the accumulator, claim a new sample
//      index from the global counter (one atomic per warp), generate its camera ray      -> T
//   T  trace the pending ray: closest hit -> hit record
//   A  extension result: miss -> sky -> R; hit -> shading, NEE -> next extension ray -> T, or termination -> R
// Regeneration keeps the slots populated until the sample counter runs dry; the CTA exits when its last slot dies.
// Two kernels build on this: wf2_lanes.cuh (namespace wf2_lq) and wf2_rings.cuh (wf2_smem, wf2_l2; see kernels.cu).
// Included in each namespace, so no include guard, and only macros whose text is the same every time.

#ifndef TB_WF2_THREADS
#define TB_WF2_THREADS 512
#endif
#ifndef TB_WF2_THREADS_WIDE
#define TB_WF2_THREADS_WIDE 768
#endif
#ifndef TB_WF2_CTAS_PER_SM
#define TB_WF2_CTAS_PER_SM 1
#endif
static_assert(TB_WF2_PATHS <= TB_WF2_SLOTS, "the host sizes the cold slot state with TB_WF2_SLOTS");
#define TB_WF2_MAX_PRIMS 40     // scene tables up to this size are staged in shared memory (the flat program: up to 16 primitives)
#define TB_WF2_MAX_PAIRS 40

enum { WF2_PH_EXT = 0, WF2_PH_NEE = 1 };
#define WF2_FLAG_EMPTY 1u   // the slot holds no sample (before its first camera ray)

// Cold half of a slot's state: 16-byte chunks, one record per slot, accessed by the one lane that owns the slot at
// the time (ownership moves through the stage queues, whose pushes are preceded by a block-scope fence).  Chunks 0-3:
//   0: T.xyz, eta        1: L.xyz, bsdfPdf     2: absorption.xyz, sample index     3: rng1, rng2, raster x, y (stage
// R's generation stores the sample's raster position in .zw; the ring layout overwrites it with NEE bookkeeping)
// TB_WF2_COLD_SMEM: the records live in shared memory (Wf2Shared::cold); otherwise in global memory (P.cold),
// read with ld.global.cg / written with st.global.cg.
enum { CC_T = 0, CC_L = 1, CC_A = 2, CC_RNG = 3 };
#ifdef TB_WF2_COLD_SMEM
TB_DEV float4 cold_ld(const float4* rec, int c) { return rec[c]; }
TB_DEV void cold_st(float4* rec, int c, float x, float y, float z, float w) { rec[c] = make_float4(x, y, z, w); }
TB_DEV void cold_st2(float4* rec, int c, float x, float y) { *reinterpret_cast<float2*>(rec + c) = make_float2(x, y); }
#else
TB_DEV float4 cold_ld(const float4* rec, int c) { return __ldcg(rec + c); }
TB_DEV void cold_st(float4* rec, int c, float x, float y, float z, float w) { __stcg(rec + c, make_float4(x, y, z, w)); }
TB_DEV void cold_st2(float4* rec, int c, float x, float y) { __stcg(reinterpret_cast<float2*>(rec + c), make_float2(x, y)); }
#endif
TB_DEV float u2f(uint32_t v) { return __uint_as_float(v); }
TB_DEV uint32_t f2u(float v) { return __float_as_uint(v); }

// HOT half of the slot state, which every layout's Wf2Shared starts with: what stage T (trace) reads and writes for
// every ray.  The cold half is kept apart (see cold_ld): the wavefront is bound by the number of paths an SM has in
// flight (halving the slots halves the throughput on every scene, measured in round 2), so the hot half stays small.
struct Wf2SharedBase {
    float ox[TB_WF2_PATHS], oy[TB_WF2_PATHS], oz[TB_WF2_PATHS];
    float dx[TB_WF2_PATHS], dy[TB_WF2_PATHS], dz[TB_WF2_PATHS];
    float time[TB_WF2_PATHS];
    uint32_t flags[TB_WF2_PATHS];     // bit 0 empty (no sample yet), bits 1-2 rayType, bit 3 phase, bits 8.. bounce
    // extension-ray hit
    float ht[TB_WF2_PATHS], hnx[TB_WF2_PATHS], hny[TB_WF2_PATHS], hnz[TB_WF2_PATHS];
    int hprim[TB_WF2_PATHS];
};

// The members every layout's Wf2Shared ends with, after its own (a common prefix would move the layout's members and
// change the kernels' shared-memory vector accesses: veach ran 1 % slower on an H100 at 700 W).
#define WF2_SHARED_TABLES                                                                                             \
    int pref;      /* stage the warps currently prefer (see the kernel's scheduler) */                                \
    int live;      /* slots that still hold (or may still receive) a path */                                          \
    int exhausted;                                                                                                    \
    /* the scene descriptor every stage reads, pointing at the staged tables below: one copy per CTA, filled by    */ \
    /* thread 0 (a per-thread copy would live in local memory, a dependent round trip at the head of each stage)   */ \
    DScene scene;                                                                                                     \
    /* tables staged on chip by bulk copies (TMA) that complete on `stageBar`; +1: copies round up to 16 bytes     */ \
    alignas(16) DPrim prims[TB_WF2_MAX_PRIMS + 1];                                                                    \
    alignas(16) BvhPair pairs[TB_WF2_MAX_PAIRS];                                                                      \
    alignas(16) ProgOp flat[32];                                                                                      \
    alignas(8) unsigned long long stageBar

// the layout's shared-memory state, defined by the kernel's own header
struct Wf2Shared;

// dynamic shared memory of a CTA: the slot state, then from the next 128-byte boundary the treelet (if any)
#define TB_WF2_TREELET_OFFSET(Shared) ((sizeof(Shared) + 127) & ~size_t(127))

TB_DEV Surface wf2_surface(const Wf2SharedBase& S, const DScene& sc, int s, float eta)
{
    // the quantities path_hit() derives from the path and the hit record (render.cpp:255-278)
    Surface sf;
    const V3 o = v3(S.ox[s], S.oy[s], S.oz[s]);
    const V3 d = v3(S.dx[s], S.dy[s], S.dz[s]);
    sf.prim = S.hprim[s];
    sf.p = o + d * S.ht[s];
    sf.n = v3(S.hnx[s], S.hny[s], S.hnz[s]);
    sf.wo = -d;
    sf.etaI = eta;
    const DPrim& prim = sc.prims[sf.prim];
    if (sf.etaI == 1.0f) {
        sf.etaO = prim.mat.ior;
        sf.outAbsorb = prim.mat.absorption;
    } else {
        sf.etaO = 1.0f;
        sf.outAbsorb = v3s(0.0f);
    }
    return sf;
}

// Streamed read-back bookkeeping (LaunchParams::bandFlags): called by a whole warp after its lanes
// with `have` set have retired sample `idx` (splatted it, or skipped it as tile padding).  Every
// lane fences its own framebuffer reductions, equal bands are counted with one atomic, and whoever
// completes a band publishes it to the host.
static __device__ __noinline__ void wf2_band_report(unsigned int* bandCount, volatile unsigned int* bandFlags, uint32_t bandSamples,
                                                    uint32_t samplesPerFrame, uint32_t bandTag, uint32_t idx, bool have)
{
    __threadfence();
    const unsigned act = __ballot_sync(0xffffffffu, have);
    if (!have) return;
    const uint32_t band = idx / bandSamples;
    const unsigned peers = __match_any_sync(act, band);
    if ((int)(threadIdx.x & 31u) != __ffs(peers) - 1) return;
    const uint32_t n = (uint32_t)__popc(peers);
    const uint32_t size = min(bandSamples, samplesPerFrame - band * bandSamples);
    if (atomicAdd(&bandCount[band], n) + n == size) {
        __threadfence_system();
        bandFlags[band] = bandTag;
    }
}

static __device__ __noinline__ void wf2_band_pad(unsigned int* bandCount, volatile unsigned int* bandFlags, uint32_t bandSamples,
                                                 uint32_t samplesPerFrame, uint32_t bandTag, uint32_t idx)
{
    const uint32_t band = idx / bandSamples;
    const uint32_t size = min(bandSamples, samplesPerFrame - band * bandSamples);
    if (atomicAdd(&bandCount[band], 1u) + 1u == size) {
        __threadfence_system();
        bandFlags[band] = bandTag;
    }
}

// Stage A's opening for slot s (cold chunks CC_T, CC_L: ct, cl).  A miss adds the sky (hprim -1; -2: maxDepth 0) and
// returns false, the path is finished.  A hit runs the hit prologue (path_hit, render.cpp:255-310) on the slot's path
// state and returns true with that state in ps, the surface in sf and chunk CC_A in ca.
template <uint32_t FEAT>
TB_DEV bool wf2_hit(const Wf2SharedBase& S, float4* rec, const DScene& sc, int s, float4 ct, float4 cl, float4& ca, PathState& ps, Surface& sf)
{
    const uint32_t fl = S.flags[s];
    const int bounce = (int)(fl >> 8);
    const int hprim = S.hprim[s];
    if (hprim < 0) {
        if (hprim == -1) {
            ps.d = v3(S.dx[s], S.dy[s], S.dz[s]);
            ps.T = v3(ct.x, ct.y, ct.z);
            ps.L = v3(cl.x, cl.y, cl.z);
            ps.rayType = (int)((fl >> 1) & 3u);
            ps.bsdfPdf = cl.w;
            path_miss<FEAT>(sc, ps, bounce);
            cold_st(rec, CC_L, ps.L.x, ps.L.y, ps.L.z, cl.w);
        }
        return false;
    }
    ca = cold_ld(rec, CC_A);
    const float4 cr = cold_ld(rec, CC_RNG);
    ps.o = v3(S.ox[s], S.oy[s], S.oz[s]);
    ps.d = v3(S.dx[s], S.dy[s], S.dz[s]);
    ps.time = S.time[s];
    ps.T = v3(ct.x, ct.y, ct.z);
    ps.L = v3(cl.x, cl.y, cl.z);
    ps.eta = ct.w;
    ps.absorb = v3(ca.x, ca.y, ca.z);
    ps.rayType = (int)((fl >> 1) & 3u);
    ps.bsdfPdf = cl.w;
    ps.rng.s1 = f2u(cr.x);
    ps.rng.s2 = f2u(cr.y);
    Hit h;
    h.t = S.ht[s];
    h.n = v3(S.hnx[s], S.hny[s], S.hnz[s]);
    h.prim = hprim;
    path_hit<FEAT>(sc, ps, h, bounce, sf);
    return true;
}

// finish the shading of a surface hit once all NEE samples are folded: BSDF sample, next ray
// (path_scatter) or termination.  Returns true when the slot continues with a new extension ray.  view: the surface's
// bsdf_view(), or nullptr (see nee_connect).
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV bool wf2_scatter(Wf2SharedBase& S, float4* rec, const DScene& sc, int s, const Surface& sf, V3 T, V3 L, Rng rng, float time, V3 neeSum,
                        int bounce, int maxDepth, V3 absorb, float bsdfPdf, uint32_t sample, const BsdfView* view = nullptr)
{
    PathState ps;
    ps.o = v3s(0.0f);
    ps.d = v3s(0.0f);
    ps.time = time;
    ps.T = T;
    ps.L = L;
    ps.eta = sf.etaI;
    ps.absorb = absorb;
    ps.rayType = (int)((S.flags[s] >> 1) & 3u);
    ps.bsdfPdf = bsdfPdf;
    ps.rng = rng;
    bool go;
    if (bounce + 1 >= maxDepth) {
        // the scattered ray of the final bounce is never traced (render.cpp:250): fold NEE only
        ps.L = ps.L + ps.T * neeSum;
        go = false;
    } else {
        go = path_scatter<FEAT>(sc, ps, sf, neeSum, view);
    }
    cold_st(rec, CC_L, ps.L.x, ps.L.y, ps.L.z, ps.bsdfPdf);
    if (!go) return false;
    S.ox[s] = ps.o.x; S.oy[s] = ps.o.y; S.oz[s] = ps.o.z;
    S.dx[s] = ps.d.x; S.dy[s] = ps.d.y; S.dz[s] = ps.d.z;
    cold_st(rec, CC_T, ps.T.x, ps.T.y, ps.T.z, ps.eta);
    cold_st(rec, CC_A, ps.absorb.x, ps.absorb.y, ps.absorb.z, u2f(sample));
    cold_st2(rec, CC_RNG, u2f(ps.rng.s1), u2f(ps.rng.s2));   // .zw left alone: the lane-owned splat reads the raster position there
    S.flags[s] = ((uint32_t)ps.rayType << 1) | ((uint32_t)WF2_PH_EXT << 3) | ((uint32_t)(bounce + 1) << 8);
    return true;
}

// THREADS: 512 (16 warps, up to 128 registers) for scenes held in shared memory, where more warps
// only add instruction-cache pressure; 768 (24 warps, 80 registers) for scenes with deep mesh BVHs,
// whose traversal is latency bound on L2 and pays for the extra warps (Wf2Route::wideCta).
// MODE: the ring-queue kernel's scheduler, compiled in per instantiation because the kernel's speed is sensitive to
// register allocation and code layout (measured in round 2); the lane-owned kernel takes GENERIC.
//   WF2_MODE_GENERIC  both schedulers, run-time flag, no split trace queue (the free-running default;
//                     its own specialisation measured slower on cornell)
//   WF2_MODE_HARD     hard phases only (faster on veach)
//   WF2_MODE_SPLIT    free-running with the split trace queue TM (scenes with a big mesh)
// FEAT: the scene features (TB_FEAT_*) compiled in; only the lane-owned kernel has an instantiation without them.
enum { WF2_MODE_GENERIC = 0, WF2_MODE_HARD = 1, WF2_MODE_SPLIT = 2 };
template <int THREADS, int MODE, uint32_t FEAT = TB_FEAT_ALL>
__global__ void __launch_bounds__(THREADS, TB_WF2_CTAS_PER_SM) k_wavefront2(const __grid_constant__ LaunchParams P, unsigned long long total);

TB_DEV uint32_t wf2_smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// a generic address the compiler cannot trace back to shared memory: loads through it are generic loads
// (LD), so one instruction serves lanes that read the staged treelet and lanes that read global memory
TB_DEV const unsigned char* wf2_opaque(const void* p)
{
    unsigned long long a = (unsigned long long)p;
    asm volatile("" : "+l"(a));
    return reinterpret_cast<const unsigned char*>(a);
}

// Prologue, thread 0: primitive records, the scene-level BVH (child-pair records) and the flat scene program go to
// shared memory as TMA bulk copies (cp.async.bulk -> UBLKCP) on an mbarrier armed with the byte count, which everybody
// waits on (wf2_await_scene); the treelet goes to `tl`, past the slot state (TB_WF2_TREELET_OFFSET).  Also sets the
// CTA's counters: every slot is alive and starts in queue `first` (stage R's).
template <class Shared>
TB_DEV void wf2_stage_scene(Shared& S, const LaunchParams& P, unsigned char* tl, int first)
{
    const bool stagePrims = P.scene.numPrims <= TB_WF2_MAX_PRIMS;
    const bool stagePairs = P.scene.numPairs > 0 && P.scene.numPairs <= TB_WF2_MAX_PAIRS;
    const bool stageFlat = P.scene.numFlat > 0 && P.scene.numFlat <= 32;
    const uint32_t bar = wf2_smem_addr(&S.stageBar);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // device arrays are padded by one element (api.cu: upload_image), so rounding up stays inside them
    const uint32_t primBytes = stagePrims ? (((uint32_t)P.scene.numPrims * (uint32_t)sizeof(DPrim) + 15u) & ~15u) : 0u;
    const uint32_t pairBytes = stagePairs ? (uint32_t)P.scene.numPairs * (uint32_t)sizeof(BvhPair) : 0u;
    const uint32_t flatBytes = stageFlat ? (uint32_t)P.scene.numFlat * (uint32_t)sizeof(ProgOp) : 0u;
    const bool stageTreelet = P.treeletBytes >= (int)sizeof(BvhPair) && P.scene.treeletMesh >= 0;
    const uint32_t treeBytes = stageTreelet ? (uint32_t)min(P.scene.treeletPairs, P.treeletBytes / (int)sizeof(BvhPair)) * (uint32_t)sizeof(BvhPair) : 0u;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(primBytes + pairBytes + flatBytes + treeBytes) : "memory");
    if (treeBytes) {
        const unsigned char* src = reinterpret_cast<const unsigned char*>(P.scene.meshes[P.scene.treeletMesh].pairs);
        for (uint32_t off = 0; off < treeBytes; off += 32768u) {
            const uint32_t n = min(32768u, treeBytes - off);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(wf2_smem_addr(tl + off)),
                         "l"(src + off), "r"(n), "r"(bar)
                         : "memory");
        }
    }
    if (primBytes)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(wf2_smem_addr(S.prims)),
                     "l"(P.scene.prims), "r"(primBytes), "r"(bar)
                     : "memory");
    if (pairBytes)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(wf2_smem_addr(S.pairs)),
                     "l"(P.scene.pairs), "r"(pairBytes), "r"(bar)
                     : "memory");
    if (flatBytes)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(wf2_smem_addr(S.flat)),
                     "l"(P.scene.flat), "r"(flatBytes), "r"(bar)
                     : "memory");
    // the CTA's scene descriptor (Wf2SharedBase::scene), published by the barrier in wf2_await_scene
    DScene d = P.scene;
    if (stagePrims) d.prims = S.prims;
    if (stagePairs) d.pairs = S.pairs;
    if (stageFlat) d.flat = S.flat;
    // the top of the biggest mesh's BVH goes into whatever shared memory the slot arrays leave (P.treeletBytes,
    // set by the launch from the device's limit): the first levels of every inline mesh walk are then shared-
    // memory reads instead of dependent L2 round trips
    d.treelet = nullptr;
    if (P.treeletBytes >= (int)sizeof(BvhPair) && d.treeletMesh >= 0) {
        d.treeletPairs = min(d.treeletPairs, P.treeletBytes / (int)sizeof(BvhPair));
        d.treelet = wf2_opaque(tl);
    } else {
        d.treeletPairs = 0;
    }
    S.scene = d;
    S.pref = first;
    S.live = TB_WF2_PATHS;
    S.exhausted = 0;
}

// Prologue, every thread: wait for thread 0's set-up (barrier word, S.scene, queues), then for the staged tables
template <class Shared>
TB_DEV void wf2_await_scene(Shared& S)
{
    __syncthreads();
    uint32_t landed = 0;
    while (!landed)
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(landed)
                     : "r"(wf2_smem_addr(&S.stageBar)), "r"(0u)
                     : "memory");
}

// stage R's parts, timed separately in the clock build (tools/stage_clocks.py)
enum { WF2_R_SPLAT = 0, WF2_R_CLAIM = 1, WF2_R_REGEN = 2, WF2_R_PARTS = 3 };
#ifdef TB_WF2_STAGE_CLOCKS
// (at a point where the warp has converged, so that lane 0's clock, the one counted, includes every lane's work)
TB_DEV unsigned int wf2_now()
{
    __syncwarp();
    return (unsigned int)clock64();
}
#else
TB_DEV unsigned int wf2_now() { return 0u; }
#endif

// Splat finished sample `doneSample` (cold record `rec`, its chunk CC_L in cl) into the accumulator, defined by the
// layout's own header: the splat is the one part of stage R the layouts do differently.
TB_DEV void wf2_splat(const LaunchParams& P, const float4* rec, float4 cl, uint32_t doneSample);

// Stage R, by a whole warp (`active` lanes hold slot s, cold record `rec`): splat the finished sample, claim a new one
// and generate its camera ray.  Returns true where one was; the caller pushes those, then wf2_retire()s the others.
// rparts: the cycles of each part (WF2_R_*) add up there in the clock build.
template <class Shared>
TB_DEV bool wf2_stage_r(Shared& S, const LaunchParams& P, unsigned long long total, float4* rec, int s, bool active,
                        unsigned int (&rparts)[WF2_R_PARTS])
{
    const unsigned int t0 = wf2_now();
    const int lane = threadIdx.x & 31;
    const bool finished = active && !(S.flags[s] & WF2_FLAG_EMPTY);
    uint32_t doneSample = 0xffffffffu;
    if (finished) {
        const float4 cl = cold_ld(rec, CC_L), ca = cold_ld(rec, CC_A);
        doneSample = f2u(ca.w);
        wf2_splat(P, rec, cl, doneSample);
    }
    if (P.bandFlags)
        wf2_band_report(P.bandCount, P.bandFlags, P.bandSamples, (uint32_t)P.samplesPerFrame, P.bandTag, doneSample, finished);
    if (active) S.flags[s] = WF2_FLAG_EMPTY;
    rparts[WF2_R_SPLAT] += wf2_now() - t0;
    // claim a new sample; indices on tile padding outside the image are skipped
    bool want = active && !*(volatile int*)&S.exhausted;
    bool fresh = false;
    for (int attempt = 0; attempt < 64; ++attempt) {
        if (!__any_sync(0xffffffffu, want)) break;
        const unsigned int t1 = wf2_now();
        const unsigned m = __ballot_sync(0xffffffffu, want);
        const int leader = __ffs(m) - 1;
        unsigned long long base = 0ull;
        if (lane == leader) {
            base = atomicAdd(P.sampleCounter, (unsigned long long)__popc(m));
            if (base + __popc(m) >= total) *(volatile int*)&S.exhausted = 1;
        }
        base = __shfl_sync(0xffffffffu, base, leader);
        const unsigned long long idx = base + (unsigned long long)__popc(m & ((1u << lane) - 1u));
        const unsigned int t2 = wf2_now();
        rparts[WF2_R_CLAIM] += t2 - t1;
        if (want) {
            if (idx >= total) {
                want = false;
            } else {
                int px, py, frame;
                if (decode_sample(P, idx, px, py, frame)) {
                    PathState ps;
                    float rx, ry;
                    sample_begin(P, px, py, frame, ps, rx, ry);
                    S.ox[s] = ps.o.x; S.oy[s] = ps.o.y; S.oz[s] = ps.o.z;
                    S.dx[s] = ps.d.x; S.dy[s] = ps.d.y; S.dz[s] = ps.d.z;
                    S.time[s] = ps.time;
                    cold_st(rec, CC_T, 1.0f, 1.0f, 1.0f, 1.0f);                     // throughput 1, eta 1
                    cold_st(rec, CC_L, 0.0f, 0.0f, 0.0f, 1.0f);                     // radiance 0, bsdfPdf 1
                    cold_st(rec, CC_A, 0.0f, 0.0f, 0.0f, u2f((uint32_t)idx));      // no absorption, the sample index
                    cold_st(rec, CC_RNG, u2f(ps.rng.s1), u2f(ps.rng.s2), rx, ry);      // the RNG, the raster position
                    S.flags[s] = ((uint32_t)TB_REFLECTED << 1) | ((uint32_t)WF2_PH_EXT << 3);
                    fresh = true;
                    want = false;
                } else if (P.bandFlags) {
                    // tile padding outside the image retires at once
                    wf2_band_pad(P.bandCount, P.bandFlags, P.bandSamples, (uint32_t)P.samplesPerFrame, P.bandTag, (uint32_t)idx);
                }
            }
        }
        rparts[WF2_R_REGEN] += wf2_now() - t2;
    }
    return fresh;
}

// after stage R: slots that could not be refilled die, and the CTA exits when none is left
template <class Shared>
TB_DEV void wf2_retire(Shared& S, bool dead)
{
    const unsigned m = __ballot_sync(0xffffffffu, dead);
    if (m && (threadIdx.x & 31) == 0) atomicSub(&S.live, __popc(m));
}

// The opt-in to > 48 KB of dynamic shared memory and the occupancy answer are PER DEVICE (and the
// attribute applies to the current device only), so they are kept per device ordinal and set up once
// per device under a lock: a host may own renderers on several GPUs, driven from several threads.
#define TB_WF2_MAX_DEVICES 64
template <int THREADS, int MODE, uint32_t FEAT, class Shared>
static int wavefront2_ctas_per_sm()
{
    static std::mutex lock;
    static int ctasPerSM[TB_WF2_MAX_DEVICES] = {};   // 0 = not configured yet
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= TB_WF2_MAX_DEVICES) dev = 0;
    std::lock_guard<std::mutex> guard(lock);
    if (ctasPerSM[dev] == 0) {
        int n = 0;
        cudaFuncSetAttribute(k_wavefront2<THREADS, MODE, FEAT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)std::max(wavefront2_smem_limit(), sizeof(Shared)));
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_wavefront2<THREADS, MODE, FEAT>, THREADS, sizeof(Shared)) != cudaSuccess || n < 1)
            n = 1;
        if (n > TB_WF2_MAX_CTAS_PER_SM) n = TB_WF2_MAX_CTAS_PER_SM;
        ctasPerSM[dev] = n;
    }
    return ctasPerSM[dev];
}

// Launch k_wavefront2<THREADS, MODE, FEAT> over `total` samples (> 0; the caller has reset P.sampleCounter).
// Shared is the layout's Wf2Shared, complete where the launcher is instantiated.
template <int THREADS, int MODE, uint32_t FEAT = TB_FEAT_ALL, class Shared = Wf2Shared>
static void launch_wavefront2_t(const LaunchParams& p0, int numSMs, cudaStream_t stream, unsigned long long total)
{
    const int ctasPerSM = wavefront2_ctas_per_sm<THREADS, MODE, FEAT, Shared>();
    // shared memory beyond the slot arrays holds the treelet
    LaunchParams p = p0;
    const size_t slotBytes = TB_WF2_TREELET_OFFSET(Shared);
    p.treeletBytes = 0;
    if (p.scene.treeletMesh >= 0 && p.scene.treeletPairs > 0 && wavefront2_smem_limit() > slotBytes) {
        const size_t room = (wavefront2_smem_limit() - slotBytes) / sizeof(BvhPair) * sizeof(BvhPair);
        p.treeletBytes = (int)std::min(room, (size_t)p.scene.treeletPairs * sizeof(BvhPair));
    }
    const size_t smemBytes = p.treeletBytes > 0 ? slotBytes + (size_t)p.treeletBytes : sizeof(Shared);
    // TB_WF2_CTAS_PER_SM resident CTAs per SM; small jobs use fewer so that every CTA has a full slot array
    const unsigned long long want = (total + TB_WF2_PATHS - 1) / TB_WF2_PATHS;
    int grid = (numSMs > 0 ? numSMs : 132) * ctasPerSM;
    if (want < (unsigned long long)grid) grid = (int)want;
    if (grid < 1) grid = 1;
    k_wavefront2<THREADS, MODE, FEAT><<<grid, THREADS, smemBytes, stream>>>(p, total);
}
