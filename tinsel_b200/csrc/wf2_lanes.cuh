// wf2_lanes.cuh -- the lane-owned wavefront kernel, included after wf2_common.cuh in namespace wf2_lq (kernels.cu):
// scenes held on chip under the free-running scheduler, in launches long enough to reach a steady state.
//
// Slot s is only ever handled by lane (s & 31) of whichever warp claims it, so every access to the slot arrays is
// free of bank conflicts (lane i touches bank i; with ring queues the slot ids of a chunk are a random permutation,
// so most accesses to the slot arrays conflict), and a stage queue needs no ring: it is one bit per slot, the 32
// slots of a lane in one word.  A push is one atomicOr by the owning lane on its own word: no ballot, no prefix sum,
// no reserved-but-unwritten cell.  The price is the FIFO order, which costs scenes with deep BVHs their traversal
// coherence: those keep the ring queues (wf2_rings.cuh).
//
// There is no stage B: stage A shades the whole bounce in place, in k_mega's order (see there), so no shadow ray
// ever waits in a slot and stage T only traces extension rays.  Stage R is the common one (wf2_stage_r); only its
// splat (wf2_splat, below) is this layout's own.

#ifndef TB_WF2_COLD_SMEM
#error "the lane-owned layout keeps the cold state in shared memory"
#endif
static_assert(TB_WF2_PATHS == 1024, "one word per lane and queue");

enum { CC_CHUNKS = 4 };   // cold chunks 0-3 (wf2_common.cuh); chunk 3 holds the RNG alone
enum { WF2_Q_T = 0, WF2_Q_A = 1, WF2_Q_R = 2, WF2_NUM_Q = 3 };

struct Wf2Shared : Wf2SharedBase {
    float4 cold[TB_WF2_PATHS * CC_CHUNKS];
    // stage queues as bit sets: one word per queue and lane
    unsigned int lq[WF2_NUM_Q][32];
    // every primitive with lightSamples > 0 lies in [lightBegin, lightEnd): stage A's NEE scan starts and stops
    // there instead of loading every primitive's lightSamples in turn (a dependent chain on every hit)
    int lightBegin, lightEnd;
    WF2_SHARED_TABLES;
};

#ifndef WF2_R_MIN_LANES
#define WF2_R_MIN_LANES 24   // stage R waits for that many lanes with a finished slot while T or A has work
#endif
#ifndef WF2_STICK_LANES
#define WF2_STICK_LANES 16     // a warp stays with the preferred stage while that many lanes have a slot waiting there
#endif

// The caller has fenced its slot-state writes (__threadfence_block).
TB_DEV void wf2_push(Wf2Shared& S, int q, bool flag, int slot)
{
    if (flag) atomicOr(&S.lq[q][slot & 31], 1u << (slot >> 5));
}

// Claim one waiting slot per lane.  All three queues (T, A, R) are looked at in one go -- three independent
// loads of the lane's own words and three ballots -- and the warp takes the CTA's preferred stage while at least
// `stick` lanes have something there, else the stage with the most lanes ready (which becomes the preference:
// the warps of a CTA herd through the stages, and share the instruction cache -- a per-warp preference instead
// of the CTA-wide one is much slower).  Every lane then picks a set bit of its word -- starting at a position that
// differs from warp to warp, so that two warps claiming at once rarely want the same one -- and clears it with
// an atomicAnd; whoever sees the bit set in the value returned owns the slot.  Returns the mask of lanes that
// got a slot (0: nothing waits anywhere) and the stage.
TB_DEV unsigned wf2_claim_fullest(Wf2Shared& S, int stick, int& slot, int& stage)
{
    const int lane = threadIdx.x & 31;
    const int rot = (int)(threadIdx.x >> 5) * 2 + 1;
    for (;;) {
        // the preference and the three queue words load side by side (no load depends on another)
        int pref = *(volatile int*)&S.pref;   // every lane loads (a broadcast, no branch); lane 0's copy is the one used
        const unsigned m0 = *(volatile unsigned int*)&S.lq[0][lane], m1 = *(volatile unsigned int*)&S.lq[1][lane];
        const unsigned m2 = *(volatile unsigned int*)&S.lq[2][lane];
        pref = __shfl_sync(0xffffffffu, pref, 0);
        // lanes ready per queue, one byte each (selections by shifts, not branches)
        unsigned cc = (unsigned)__popc(__ballot_sync(0xffffffffu, m0 != 0u)) | ((unsigned)__popc(__ballot_sync(0xffffffffu, m1 != 0u)) << 8) |
                      ((unsigned)__popc(__ballot_sync(0xffffffffu, m2 != 0u)) << 16);
        // R's work is per lane (the splat's atomics, a new camera ray), so a thin R chunk costs nearly what a full
        // one does: R only counts as ready with WF2_R_MIN_LANES lanes, or when nothing else is (cornell: about +1.5 %)
        if (((cc >> (8 * WF2_Q_R)) & 0xffu) < WF2_R_MIN_LANES && (cc & ~(0xffu << (8 * WF2_Q_R))) != 0u) cc &= ~(0xffu << (8 * WF2_Q_R));
        int q = pref;
        unsigned bc = (cc >> (8 * pref)) & 0xffu;
        if (bc < (unsigned)stick) {
#pragma unroll
            for (int k = 1; k < WF2_NUM_Q; ++k) {
                const int qq = pref + k < WF2_NUM_Q ? pref + k : pref + k - WF2_NUM_Q;
                const unsigned cq = (cc >> (8 * qq)) & 0xffu;
                q = cq > bc ? qq : q;
                bc = cq > bc ? cq : bc;
            }
        }
        if (bc == 0u) return 0u;
        const unsigned mine = q == 0 ? m0 : q == 1 ? m1 : m2;
        bool got = false;
        if (mine != 0u) {
            const int k = (__ffs(__funnelshift_r(mine, mine, rot)) - 1 + rot) & 31;
            const unsigned bit = 1u << k;
            got = (atomicAnd(&S.lq[q][lane], ~bit) & bit) != 0u;
            slot = lane + 32 * k;
        }
        const unsigned act = __ballot_sync(0xffffffffu, got);
        if (act != 0u) {
            __threadfence_block();   // the producer's state writes precede its atomicOr
            if (q != pref && lane == 0) *(volatile int*)&S.pref = q;
            stage = q;
            return act;
        }
        // every lane lost its bit to another warp, which made progress: look again
    }
}

// stage A's parts, timed separately in the clock build (tools/stage_clocks.py): the hit prologue (wf2_hit), the light
// samples (nee_generate), the shadow traces, the connections (wf2_surface, nee_connect) and the BSDF sample
// (wf2_scatter).  The lanes of a chunk leave the NEE loop at different times, so no lane can wait for the others
// inside it: each lane reads the clock on its own (wf2_lane_now), and the chunk counts the longest any lane spent.
enum { WF2_A_HIT = 0, WF2_A_LIGHT = 1, WF2_A_SHADOW = 2, WF2_A_CONNECT = 3, WF2_A_SCATTER = 4, WF2_A_PARTS = 5 };
#ifdef TB_WF2_STAGE_CLOCKS
TB_DEV unsigned int wf2_lane_now() { return (unsigned int)clock64(); }
#else
TB_DEV unsigned int wf2_lane_now() { return 0u; }
#endif

#ifdef TB_WF2_STAGE_CLOCKS
// Per-stage cycle accounting (development builds with -DTB_WF2_STAGE_CLOCKS, read by tb200_stage_clocks, see
// tools/stage_clocks.py).  Every warp sums clock64() deltas in registers and adds its totals here when it exits.
// Stage kinds k: 0 R, 1 T, 2 A, 3 B (no B in this kernel: its counters stay 0).
//   [0] claims that got slots   [1] idle: empty claims and the back-off   [2 + k] cycles in stage k
//   [6 + k] chunks of stage k   [10 + k] lanes active in those chunks      [14] warps
//   [15 + p] stage R's cycles in part p: WF2_R_SPLAT, WF2_R_CLAIM, WF2_R_REGEN (see wf2_stage_r)
//   [18 + p] stage A's cycles in part p: WF2_A_HIT ... WF2_A_SCATTER (see the kernel)
enum { WF2_CLK_CLAIM = 0, WF2_CLK_IDLE = 1, WF2_CLK_CYCLES = 2, WF2_CLK_CHUNKS = 6, WF2_CLK_LANES = 10, WF2_CLK_WARPS = 14, WF2_CLK_R_PARTS = 15,
       WF2_CLK_A_PARTS = 18, WF2_CLK_N = 23 };
static_assert(WF2_CLK_N == TB_WF2_STAGE_CLOCK_WORDS, "tb_kernels.cuh states the counter count");
__device__ unsigned long long g_wf2StageClocks[WF2_CLK_N];

// A warp's sums are 32 bits wide (fewer registers, so the accounting itself spills less): a warp lives for one
// launch, and the tool's launches last far fewer than 2^32 cycles.
struct Wf2Clocks {
    static constexpr int kinds = 3;   // R, T, A: this kernel has no stage B
    unsigned int claim = 0, idle = 0, cyc[kinds] = {}, chunks[kinds] = {}, lanes[kinds] = {}, rparts[WF2_R_PARTS] = {}, aparts[WF2_A_PARTS] = {};

    // a chunk of stage A: each part counts the longest any lane spent in it (lane_parts: per lane, see the kernel)
    TB_DEV void add_a(const unsigned int (&lane_parts)[WF2_A_PARTS])
    {
#pragma unroll
        for (int p = 0; p < WF2_A_PARTS; ++p) aparts[p] += __reduce_max_sync(0xffffffffu, lane_parts[p]);
    }

    // the stage kind as a constant index, so the arrays stay in registers
    TB_DEV void add(int stage, unsigned int dt, unsigned act)
    {
#pragma unroll
        for (int k = 0; k < kinds; ++k) {
            const int q = k == 0 ? (int)WF2_Q_R : k == 1 ? (int)WF2_Q_T : (int)WF2_Q_A;
            if (stage == q) {
                cyc[k] += dt;
                chunks[k] += 1u;
                lanes[k] += (unsigned)__popc(act);
            }
        }
    }
    TB_DEV void flush() const
    {
        if ((threadIdx.x & 31) != 0) return;
        atomicAdd(&g_wf2StageClocks[WF2_CLK_CLAIM], (unsigned long long)claim);
        atomicAdd(&g_wf2StageClocks[WF2_CLK_IDLE], (unsigned long long)idle);
#pragma unroll
        for (int k = 0; k < kinds; ++k) {
            atomicAdd(&g_wf2StageClocks[WF2_CLK_CYCLES + k], (unsigned long long)cyc[k]);
            atomicAdd(&g_wf2StageClocks[WF2_CLK_CHUNKS + k], (unsigned long long)chunks[k]);
            atomicAdd(&g_wf2StageClocks[WF2_CLK_LANES + k], (unsigned long long)lanes[k]);
        }
#pragma unroll
        for (int p = 0; p < WF2_R_PARTS; ++p) atomicAdd(&g_wf2StageClocks[WF2_CLK_R_PARTS + p], (unsigned long long)rparts[p]);
#pragma unroll
        for (int p = 0; p < WF2_A_PARTS; ++p) atomicAdd(&g_wf2StageClocks[WF2_CLK_A_PARTS + p], (unsigned long long)aparts[p]);
        atomicAdd(&g_wf2StageClocks[WF2_CLK_WARPS], 1ull);
    }
};

void wf2_stage_clocks(unsigned long long* out, bool reset)
{
    cudaMemcpyFromSymbol(out, g_wf2StageClocks, sizeof(g_wf2StageClocks));
    if (reset) {
        static const unsigned long long zero[WF2_CLK_N] = {};
        cudaMemcpyToSymbol(g_wf2StageClocks, zero, sizeof(zero));
    }
}
#endif

// The lane-owned splat (stage R: wf2_stage_r).  It neither decodes the sample index nor draws the raster position
// again: the slot's RNG chunk carries it in .zw from the sample's generation (wf2_scatter leaves .zw alone), and
// add_sample_small weighs a 3x3 footprint with one filter evaluation per column and per row.  The per-sample capture
// (P.outRadiance, for trace_frame) is out of line: renders never take it.
static __device__ __noinline__ void wf2_capture(const LaunchParams& P, uint32_t doneSample, float rasterX, float rasterY, V3 radiance)
{
    int px, py, frame;
    decode_sample(P, (unsigned long long)doneSample, px, py, frame);
    sample_end(P, px, py, rasterX, rasterY, radiance);
}

TB_DEV void wf2_splat(const LaunchParams& P, const float4* rec, float4 cl, uint32_t doneSample)
{
    const float4 cr = cold_ld(rec, CC_RNG);
    if (P.outRadiance) {
        wf2_capture(P, doneSample, cr.z, cr.w, v3(cl.x, cl.y, cl.z));
    } else {
        add_sample_small(P.film, P.accum, cr.z, cr.w, v3(cl.x, cl.y, cl.z));
    }
}

template <int THREADS, int MODE, uint32_t FEAT>
__global__ void __launch_bounds__(THREADS, TB_WF2_CTAS_PER_SM) k_wavefront2(const __grid_constant__ LaunchParams P, unsigned long long total)
{
    static_assert(MODE == WF2_MODE_GENERIC, "the lane-owned layout serves the free-running scheduler only");
    extern __shared__ __align__(16) unsigned char wf_smem_raw[];
    Wf2Shared& S = *reinterpret_cast<Wf2Shared*>(wf_smem_raw);
    const int tid = threadIdx.x;
    if (tid == 0) {
        wf2_stage_scene(S, P, wf_smem_raw + TB_WF2_TREELET_OFFSET(Wf2Shared), WF2_Q_R);
        int lb = 0, le = 0;
        for (int i = P.scene.numPrims - 1; i >= 0; --i)
            if (P.scene.prims[i].lightSamples > 0) {
                if (le == 0) le = i + 1;
                lb = i;
            }
        S.lightBegin = lb;
        S.lightEnd = le;
    }
    const DScene& sc = S.scene;
    // every slot starts in the R queue "finished with nothing to splat": stage R fills it with a camera sample
    for (int s = tid; s < TB_WF2_PATHS; s += THREADS) S.flags[s] = WF2_FLAG_EMPTY;
    if (tid < WF2_NUM_Q * 32) S.lq[tid >> 5][tid & 31] = (tid >> 5) == WF2_Q_R ? 0xffffffffu : 0u;
    wf2_await_scene(S);

    const int maxDepth = P.film.maxDepth;
    const int lane = tid & 31;
    float4* const coldBase = S.cold;
#ifdef TB_WF2_STAGE_CLOCKS
    Wf2Clocks clk;
    unsigned int (&rparts)[WF2_R_PARTS] = clk.rparts;
#else
    unsigned int rparts[WF2_R_PARTS];   // written only in the clock build
#endif
    for (;;) {
        int s = 0, stage = -1;
#ifdef TB_WF2_STAGE_CLOCKS
        const unsigned int t0 = (unsigned int)clock64();
#endif
        const unsigned act = wf2_claim_fullest(S, WF2_STICK_LANES, s, stage);
        if (act == 0u) {
            if (*(volatile int*)&S.live <= 0) break;
            __nanosleep(200);
#ifdef TB_WF2_STAGE_CLOCKS
            clk.idle += (unsigned int)clock64() - t0;
#endif
            continue;
        }
        const bool active = ((act >> lane) & 1u) != 0u;
#ifdef TB_WF2_STAGE_CLOCKS
        const unsigned int t1 = (unsigned int)clock64();
        clk.claim += t1 - t0;
#endif

        if (stage == WF2_Q_R) {
            // ===================== R: splat the finished sample, regenerate =======================
            const bool fresh = wf2_stage_r(S, P, total, coldBase + (size_t)s * CC_CHUNKS, s, active, rparts);
            __threadfence_block();
            wf2_push(S, WF2_Q_T, fresh, s);
            wf2_retire(S, active && !fresh);
        } else if (stage == WF2_Q_T) {
            // ===================== T: trace the extension ray =====================================
            if (active) {
                if (maxDepth > 0) {
                    // S.flat, not sc.flat: shared-memory loads (wf2_stage_scene stages every flat program -- api.cu's
                    // build_program keeps them to the 32 ops S.flat holds -- and with numFlat == 0 no op is read)
                    const Hit h = trace_closest<FEAT, false, true>(sc, S.flat, v3(S.ox[s], S.oy[s], S.oz[s]), v3(S.dx[s], S.dy[s], S.dz[s]), S.time[s], true);
                    S.ht[s] = h.t;
                    S.hnx[s] = h.n.x; S.hny[s] = h.n.y; S.hnz[s] = h.n.z;
                    S.hprim[s] = h.prim;
                } else {
                    S.hprim[s] = -2;   // maxDepth == 0: no trace at all, radiance stays 0
                }
            }
            __threadfence_block();
            wf2_push(S, WF2_Q_A, active, s);
        } else if (stage == WF2_Q_A) {
            // ===================== A: the whole bounce ============================================
            bool cont = false, fin = false;
            unsigned int ap[WF2_A_PARTS] = {};   // this lane's cycles per part, in the clock build
            if (active) {
                float4* rec = coldBase + (size_t)s * CC_CHUNKS;
                const float4 ct = cold_ld(rec, CC_T), cl = cold_ld(rec, CC_L);
                float4 ca;
                PathState ps;
                Surface sf;
                unsigned int ta = wf2_lane_now();
                if (!wf2_hit<FEAT>(S, rec, sc, s, ct, cl, ca, ps, sf)) {
                    ap[WF2_A_HIT] += wf2_lane_now() - ta;
                    fin = true;
                } else {
                    ap[WF2_A_HIT] += wf2_lane_now() - ta;
                    NeeCursor c;
                    ShadowRay sr;
                    nee_begin(c, S.lightBegin);
                    const int lightEnd = S.lightEnd;
                    // The whole bounce in place, in k_mega's order: every NEE sample traced and connected, then
                    // the BSDF sample.  What the traces do not need stays in the slot and is read back after
                    // them instead of being held in registers across them: the throughput and radiance path_hit
                    // left, and the surface (wf2_surface rebuilds it bit for bit, as stage B of the ring kernel
                    // does).  s2 is s behind an empty asm, so the compiler cannot forward the stores to the reads.
                    // (Measured on cornell: keeping it all in registers spills, 160 bytes.)  The BSDF's view terms
                    // (bsdf_view) are the exception: three floats (four with clearcoat), computed once here for every
                    // BSDF evaluation of the bounce, fit in registers across the traces.
                    cold_st(rec, CC_T, ps.T.x, ps.T.y, ps.T.z, ct.w);
                    cold_st(rec, CC_L, ps.L.x, ps.L.y, ps.L.z, cl.w);
                    const float time = ps.time;
                    Rng rng = ps.rng;
                    const BsdfView view = bsdf_view<FEAT>(sc.prims[sf.prim].mat, sf.n, sf.wo);
                    int s2 = s;
                    ta = wf2_lane_now();
                    while (nee_generate<FEAT>(sc, sf, time, c, rng, sr, lightEnd)) {
                        unsigned int tb = wf2_lane_now();
                        ap[WF2_A_LIGHT] += tb - ta;
                        const Hit sh = trace_closest<FEAT, false, true>(sc, S.flat, sr.o, sr.d, time, false);
                        asm volatile("" : "+r"(s2) : "f"(sh.t));
                        ta = wf2_lane_now();
                        ap[WF2_A_SHADOW] += ta - tb;
                        sf = wf2_surface(S, sc, s2, ct.w);
                        nee_connect<FEAT>(sc, sf, sr, sh, c, &view);
                        tb = wf2_lane_now();
                        ap[WF2_A_CONNECT] += tb - ta;
                        ta = tb;
                    }
                    ap[WF2_A_LIGHT] += wf2_lane_now() - ta;   // the call that found no further sample
                    asm volatile("" : "+r"(s2));
                    const float4* rec2 = coldBase + (size_t)s2 * CC_CHUNKS;
                    const float4 t2 = cold_ld(rec2, CC_T), l2 = cold_ld(rec2, CC_L), a2 = cold_ld(rec2, CC_A);
                    ta = wf2_lane_now();
                    cont = wf2_scatter<FEAT>(S, rec, sc, s, sf, v3(t2.x, t2.y, t2.z), v3(l2.x, l2.y, l2.z), rng, time, c.sum, (int)(S.flags[s] >> 8), maxDepth,
                                       v3(a2.x, a2.y, a2.z), l2.w, f2u(a2.w), &view);
                    ap[WF2_A_SCATTER] += wf2_lane_now() - ta;
                    fin = !cont;
                }
            }
#ifdef TB_WF2_STAGE_CLOCKS
            clk.add_a(ap);
#endif
            __threadfence_block();
            wf2_push(S, WF2_Q_T, cont, s);
            wf2_push(S, WF2_Q_R, fin, s);
        }
#ifdef TB_WF2_STAGE_CLOCKS
        clk.add(stage, (unsigned int)clock64() - t1, act);
#endif
    }
#ifdef TB_WF2_STAGE_CLOCKS
    clk.flush();
#endif
}
