// wf2_rings.cuh -- the ring-queue wavefront kernel, included after wf2_common.cuh in namespaces wf2_smem and wf2_l2
// (kernels.cu).  Its FIFO order traces rays that were pushed together together, which deep mesh BVHs gain from.
//
// Every slot that is alive has exactly one pending ray, its extension ray or one shadow ray.  Stage T traces either
// kind; stage A takes the extension-ray results, stage B the shadow-ray ones:
//   A  extension result: miss -> sky -> R; hit -> absorption, emission MIS, first NEE sample -> T
//   B  shadow result: connect the NEE sample; next NEE sample -> T, or BSDF sample, throughput
//      update and next extension ray -> T, or termination -> R
// Stage R is the common one (wf2_common.cuh: wf2_stage_r); only its splat (wf2_splat, below) is this layout's own.
//
// The queues are lock-free rings in shared memory: producers reserve cells with one warp-aggregated atomicAdd on
// `tail` and store lap-tagged slot ids, so a chunk is always full while the queue holds >= 32 entries.
//
// Who runs what when is the scheduler's business: hard phases, free running, or free running with a second trace
// queue for rays that enter a big mesh (template MODE, see wf2_common.cuh, and the kernel below).

// The cold chunks past 0-3 (wf2_common.cuh) hold the pending shadow ray's NEE bookkeeping:
//   3: rng1, rng2, NEE cursor, sampled light      4: shadow dist, light normal.xyz
//   5: sky pdf, NEE sum.xyz                        6: NEE radiance accumulator.xyz
// The NEE cursor word (wf2_store_shadow): bit 0 "a shadow ray has been drawn at this hit" (NeeCursor::slot is only
// ever compared with 0, and a hit draws up to 1 + 4095 * 4095 of them), the primitive scan position in bits
// 8..19, the sample index within that light in bits 20..31.
// A record in global memory is 128 bytes (8 chunks, seven used); in shared memory (TB_WF2_COLD_SMEM) the stride is 7
// chunks: the cold half then costs 7 128-bit accesses per stage instead of 27 32-bit ones.
#ifdef TB_WF2_COLD_SMEM
enum { CC_SH = 4, CC_SUM = 5, CC_LA = 6, CC_CHUNKS = 7 };
#else
enum { CC_SH = 4, CC_SUM = 5, CC_LA = 6, CC_CHUNKS = 8 };
#endif

// stage queues.  T, A, B, R in the cyclic order of the free-running sweep; F0/F1 hold the freshly regenerated camera
// rays in hard-phase mode (double-buffered: R fills one while T drains the other).  TM (WF2_MODE_SPLIT): rays
// that enter the big mesh's box; same stage code as T, but a chunk taken from TM walks the mesh with all of its
// lanes and a chunk taken from T with none.
enum { WF2_Q_T = 0, WF2_Q_A = 1, WF2_Q_B = 2, WF2_Q_R = 3, WF2_Q_F0 = 4, WF2_Q_F1 = 5, WF2_Q_TM = 6 };

struct Wf2Shared : Wf2SharedBase {
    // pending shadow ray (origin is recomputed from the surface point) and its result
    float sdx[TB_WF2_PATHS], sdy[TB_WF2_PATHS], sdz[TB_WF2_PATHS];
    float st[TB_WF2_PATHS];
    int sprim[TB_WF2_PATHS];
#ifdef TB_WF2_COLD_SMEM
    float4 cold[TB_WF2_PATHS * CC_CHUNKS];
#endif
    // stage queues: rings of lap-tagged slot ids
    uint16_t ring[7][TB_WF2_PATHS];
    unsigned int head[7], tail[7];
    unsigned int snap[5];             // hard-phase mode: the tail each stage of the current phase runs with
    WF2_SHARED_TABLES;
};

#define WF2_MASK (TB_WF2_PATHS - 1)
#define WF2_LOG2_PATHS (TB_WF2_PATHS == 2048 ? 11 : TB_WF2_PATHS == 1024 ? 10 : TB_WF2_PATHS == 512 ? 9 : TB_WF2_PATHS == 256 ? 8 : 7)
#define WF2_SLOT_BITS 11                      // queue cells: slot id in the low 11 bits, lap tag (1..31) above
#define WF2_SLOT_MASK ((1u << WF2_SLOT_BITS) - 1u)
static_assert(TB_WF2_PATHS <= (1 << WF2_SLOT_BITS) && (TB_WF2_PATHS & (TB_WF2_PATHS - 1)) == 0, "slot ids must fit the queue cells");

// cell value of ring index i holding slot s: the lap tag (1..31, never 0) makes "reserved but not
// yet written" and "left over from the previous lap" distinguishable from the expected entry
TB_DEV uint16_t wf2_cell(unsigned int index, int slot)
{
    const unsigned int lap = ((index >> WF2_LOG2_PATHS) % 31u) + 1u;
    return (uint16_t)((unsigned)slot | (lap << WF2_SLOT_BITS));
}

// append `slot` to stage queue q for every lane with flag == true: ballot + prefix sum, one shared
// atomic per warp.  The caller has fenced its slot-state writes (__threadfence_block).
TB_DEV void wf2_push(Wf2Shared& S, int q, bool flag, int slot)
{
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (m == 0u) return;
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(m) - 1;
    unsigned int base = 0;
    if (lane == leader) base = atomicAdd(&S.tail[q], (unsigned)__popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (flag) {
        const unsigned int idx = base + (unsigned)__popc(m & ((1u << lane) - 1u));
        *(volatile uint16_t*)&S.ring[q][idx & WF2_MASK] = wf2_cell(idx, slot);
    }
}

// Push a slot whose pending ray is ready to be traced.  With `split` set the ray (extension ray, or
// the shadow ray from the hit point) is classified against the big mesh's bounds first; the test
// is a scheduling heuristic, so the unoffset hit point is good enough as the shadow-ray origin.
TB_DEV void wf2_push_trace(Wf2Shared& S, const DScene& sc, bool split, int q, bool flag, int s)
{
    if (!split) {
        wf2_push(S, q, flag, s);
        return;
    }
    bool big = false;
    if (flag) {
        V3 o = v3(S.ox[s], S.oy[s], S.oz[s]);
        V3 d = v3(S.dx[s], S.dy[s], S.dz[s]);
        if (((S.flags[s] >> 3) & 1u) != WF2_PH_EXT) {
            o = o + d * S.ht[s];
            d = v3(S.sdx[s], S.sdy[s], S.sdz[s]);
        }
        V3 rcp;
        rcp.x = 1.0f / d.x;
        rcp.y = 1.0f / d.y;
        rcp.z = 1.0f / d.z;
        float t;
        big = ray_aabb(o, rcp, sc.splitLo.x, sc.splitLo.y, sc.splitLo.z, sc.splitHi.x, sc.splitHi.y, sc.splitHi.z, t);
    }
    wf2_push(S, q, flag && !big, s);
    wf2_push(S, WF2_Q_TM, flag && big, s);
}

// Claim up to 32 entries of queue q for this warp.  Returns the number claimed (warp-uniform);
// lane i < n receives its slot.  Lock-free: cells are read first, ownership is taken with a CAS
// on head, so a stalled warp can never read a cell that a producer has already recycled.
TB_DEV int wf2_claim(Wf2Shared& S, int q, int minCount, int& slot)
{
    const int lane = threadIdx.x & 31;
    int notReady = 0;
    for (;;) {
        unsigned int h = 0, t = 0;
        if (lane == 0) {
            h = *(volatile unsigned int*)&S.head[q];
            t = *(volatile unsigned int*)&S.tail[q];
        }
        h = __shfl_sync(0xffffffffu, h, 0);
        t = __shfl_sync(0xffffffffu, t, 0);
        int n = (int)(t - h);
        if (n < minCount) return 0;
        if (n > 32) n = 32;
        // optimistic read; entries reserved by a producer but not yet stored end the chunk early
        const unsigned int idx = h + (unsigned)lane;
        const uint16_t cell = *(volatile uint16_t*)&S.ring[q][idx & WF2_MASK];
        const bool ok = lane < n && (unsigned)(cell >> WF2_SLOT_BITS) == (((idx >> WF2_LOG2_PATHS) % 31u) + 1u);
        const unsigned good = __ballot_sync(0xffffffffu, ok);
        n = (good == 0xffffffffu) ? 32 : __ffs(~good) - 1;   // length of the valid prefix
        if (n <= 0) {
            if (++notReady > 8) return 0;   // a producer is between its reservation and its store
            continue;
        }
        unsigned int got = 0;
        if (lane == 0) got = atomicCAS(&S.head[q], h, h + (unsigned)n);
        got = __shfl_sync(0xffffffffu, got, 0);
        if (got == h) {
            __threadfence_block();   // the producer's state writes precede its cell store
            slot = (int)(cell & WF2_SLOT_MASK);
            return n;
        }
        // lost the race to another warp, which made progress: try again
    }
}

// Hard-phase variant: while a stage runs nobody pushes into its queue, so `tail` is fixed and a
// ticket (atomicAdd on head) can never overshoot into entries that do not exist yet.  `head` is
// put back to `tail` by thread 0 after the barrier that ends the stage.
TB_DEV int wf2_claim_ticket(Wf2Shared& S, int q, unsigned int tail, int& slot)
{
    const int lane = threadIdx.x & 31;
    unsigned int base = 0;
    if (lane == 0) base = atomicAdd(&S.head[q], 32u);
    base = __shfl_sync(0xffffffffu, base, 0);
    const int avail = (int)(tail - base);
    if (avail <= 0) return 0;
    const int n = avail < 32 ? avail : 32;
    if (lane < n) slot = (int)(*(volatile uint16_t*)&S.ring[q][(base + (unsigned)lane) & WF2_MASK] & WF2_SLOT_MASK);
    return n;
}

// The stored primitive position runs up to numPrims (past the last light, after the probe sample of a scene
// without lights), the stored sample index up to lightSamples - 1: both fit the cursor's 12-bit fields.
static_assert(TB200_MAX_PRIMITIVES <= 0xfff && TB200_MAX_LIGHT_SAMPLES <= 0xfff, "the NEE cursor holds 12-bit primitive and sample indices");

// the pending shadow ray and the NEE bookkeeping that waits for its result
TB_DEV void wf2_store_shadow(Wf2Shared& S, float4* rec, int s, const ShadowRay& sr, const NeeCursor& c, Rng rng)
{
    S.sdx[s] = sr.d.x; S.sdy[s] = sr.d.y; S.sdz[s] = sr.d.z;
    const uint32_t cursor = (c.slot != 0 ? 1u : 0u) | ((uint32_t)c.prim << 8) | ((uint32_t)c.sample << 20);
    cold_st(rec, CC_RNG, u2f(rng.s1), u2f(rng.s2), u2f(cursor), __int_as_float(sr.light));
    cold_st(rec, CC_SH, sr.dist, sr.lightN.x, sr.lightN.y, sr.lightN.z);
    cold_st(rec, CC_SUM, sr.skyPdf, c.sum.x, c.sum.y, c.sum.z);
    cold_st(rec, CC_LA, c.Lacc.x, c.Lacc.y, c.Lacc.z, 0.0f);
}

// The ring layout's splat (stage R: wf2_stage_r).  The RNG chunk's .zw holds NEE bookkeeping by now, so the raster
// position is drawn again from the sample's seed.  (The lane-owned splat, add_sample_small, would make veach's
// hard-phase kernel bigger and slower.)
TB_DEV void wf2_splat(const LaunchParams& P, const float4* rec, float4 cl, uint32_t doneSample)
{
    int px, py, frame;
    decode_sample(P, (unsigned long long)doneSample, px, py, frame);
    // raster position of the sample: its first two RNG draws (render.cpp:476,481-482)
    Rng rr = rng_seed(tb_sample_seed((uint32_t)(py * P.film.width + px), (uint32_t)frame));
    float rx = rng_float(rr);
    float ry = rng_float(rr);
    rx += px;
    ry += py;
    sample_end(P, px, py, rx, ry, v3(cl.x, cl.y, cl.z));
}

template <int THREADS, int MODE, uint32_t FEAT>
__global__ void __launch_bounds__(THREADS, TB_WF2_CTAS_PER_SM) k_wavefront2(const __grid_constant__ LaunchParams P, unsigned long long total)
{
    static_assert(FEAT == TB_FEAT_ALL, "only the lane-owned layout has a specialised instantiation");
    extern __shared__ __align__(16) unsigned char wf_smem_raw[];
    Wf2Shared& S = *reinterpret_cast<Wf2Shared*>(wf_smem_raw);
    const int tid = threadIdx.x;
    if (tid == 0) wf2_stage_scene(S, P, wf_smem_raw + TB_WF2_TREELET_OFFSET(Wf2Shared), WF2_Q_R);
    const DScene& sc = S.scene;
    // every slot starts in the R queue "finished with nothing to splat": stage R fills it with a camera sample
    for (int s = tid; s < TB_WF2_PATHS; s += THREADS) {
        S.ring[WF2_Q_R][s] = wf2_cell((unsigned)s, s);
        S.ring[WF2_Q_T][s] = 0;
        S.ring[WF2_Q_A][s] = 0;
        S.ring[WF2_Q_B][s] = 0;
        S.ring[WF2_Q_F0][s] = 0;
        S.ring[WF2_Q_F1][s] = 0;
        S.ring[WF2_Q_TM][s] = 0;
        S.flags[s] = WF2_FLAG_EMPTY;
    }
    if (tid == 0) {
        for (int q = 0; q < 7; ++q) S.head[q] = S.tail[q] = 0u;
        S.tail[WF2_Q_R] = TB_WF2_PATHS;
        S.snap[0] = TB_WF2_PATHS;
        S.snap[1] = S.snap[2] = S.snap[3] = S.snap[4] = 0u;
    }
    wf2_await_scene(S);

    const int maxDepth = P.film.maxDepth;
    const int lane = tid & 31;
#ifdef TB_WF2_COLD_SMEM
    float4* const coldBase = S.cold;
#else
    float4* const coldBase = P.cold + (size_t)blockIdx.x * TB_WF2_PATHS * CC_CHUNKS;
#endif

    // Two scheduling modes share the stage code below (P.hardPhases, uniform for the launch):
    //  * hard phases: all warps of the CTA work through the same short list of stages, claiming chunks dynamically
    //    until each queue is empty, and meet at a block barrier twice per cycle.  The kernel is far larger than the
    //    instruction cache (32 KB of L1.5 against ~150 KB), so warps that execute the same code at the same time
    //    share every instruction line; this is the faster mode when rays cost about the same (small scenes held in
    //    shared memory).
    //  * free running: no barriers at all; every warp picks the next stage itself, starting at a CTA-wide preferred
    //    stage and moving on cyclically when that queue has no full chunk left (dragging the preference along).
    //    Nobody ever waits for a slow ray, which wins when ray cost varies wildly (deep mesh BVHs) and the hot loop
    //    is small enough to stay cached.
    const bool hard = MODE == WF2_MODE_HARD ? true : MODE == WF2_MODE_SPLIT ? false : (P.hardPhases != 0);
    constexpr bool split = MODE == WF2_MODE_SPLIT;
    // hard-phase schedule: each cycle is two block-synchronous phases,
    //   phase 0:  R (finished slots -> fresh camera rays into F[cycle&1]),  T,  F[~cycle&1]
    //   phase 1:  A,  B
    // Inside a phase the stages run back to back without a barrier: they consume queues that were completed before the
    // phase began (so their tails are fixed and tickets cannot overshoot into missing entries) and touch disjoint
    // slots.  step 0..4 = R, T, F, A, B.
    int step = 0, cycle = 0;
    unsigned int stepTail = TB_WF2_PATHS;   // every slot starts in the R queue
    int stepQueue = WF2_Q_R;
    unsigned int rparts[WF2_R_PARTS];   // stage R's part timing: only the lane-owned kernel reports it

    for (;;) {
        int s = 0, n = 0, stage = -1;
        if (hard) {
            n = wf2_claim_ticket(S, stepQueue, stepTail, s);
            if (n > 0) {
                stage = stepQueue;
            } else {
                // this stage's queue is drained; at the end of a phase meet the other warps, undo the overshoot of the
                // failed ticket requests (head back to the tail the stage ran with)
                const bool endOfPhase = (step == 2 || step == 4);
                if (endOfPhase) {
                    __syncthreads();
                    if (tid == 0) {
                        if (step == 2) {
                            S.head[WF2_Q_R] = S.snap[0];
                            S.head[WF2_Q_T] = S.snap[1];
                            S.head[WF2_Q_F0 + ((cycle + 1) & 1)] = S.snap[2];
                        } else {
                            S.head[WF2_Q_A] = S.snap[3];
                            S.head[WF2_Q_B] = S.snap[4];
                        }
                    }
                    if (step == 2 && *(volatile int*)&S.live <= 0) {
                        // `live` only changes during R; nothing is left anywhere once it reaches zero
                        break;
                    }
                }
                if (step == 4) {
                    step = 0;
                    ++cycle;
                } else {
                    ++step;
                }
                stepQueue = step == 0 ? WF2_Q_R : step == 1 ? WF2_Q_T : step == 2 ? WF2_Q_F0 + ((cycle + 1) & 1)
                          : step == 3 ? WF2_Q_A : WF2_Q_B;
                // the queue was completed before this phase began; thread 0 publishes the tail every
                // warp of the CTA uses (and that the head is reset to afterwards)
                stepTail = *(volatile unsigned int*)&S.tail[stepQueue];
                if (tid == 0) S.snap[step] = stepTail;
                continue;
            }
        } else {
            int p = 0;
            if (lane == 0) p = *(volatile int*)&S.pref | (*(volatile int*)&S.exhausted << 8);
            p = __shfl_sync(0xffffffffu, p, 0);
            // Once the sample counter has run dry the CTA is draining: nothing refills the queues any more, so
            // waiting for full 32-entry chunks only adds latency -- take whatever is there.  (A 1-spp Render() on
            // one of N GPUs is ALL drain: a single partial fill of the slot arrays.)
            const int full = (p >> 8) ? 1 : 32;
            p &= 0xff;
            if (!split) {
                for (int k = 0; k < 8 && stage < 0; ++k) {
                    // k = 0..3: full chunks only; k = 4..7: whatever is left
                    const int q = (p + k) & 3;
                    n = wf2_claim(S, q, k < 4 ? full : 1, s);
                    if (n > 0) stage = q;
                }
            } else {
                // same sweep over five queues: T, TM, A, B, R (pref holds the position in this order)
                for (int k = 0; k < 10 && stage < 0; ++k) {
                    const int pos = (p + k) % 5;
                    const int q = pos == 0 ? WF2_Q_T : pos == 1 ? WF2_Q_TM : pos == 2 ? WF2_Q_A : pos == 3 ? WF2_Q_B : WF2_Q_R;
                    n = wf2_claim(S, q, k < 5 ? full : 1, s);
                    if (n > 0) {
                        stage = q;
                        if (pos != p && lane == 0) *(volatile int*)&S.pref = pos;
                    }
                }
            }
            if (!split && stage >= 0 && stage != p && lane == 0) *(volatile int*)&S.pref = stage;
            if (stage < 0) {
                if (*(volatile int*)&S.live <= 0) break;
                __nanosleep(200);
                continue;
            }
        }
        const bool active = lane < n;

        if (stage == WF2_Q_R) {
            // ===================== R: splat the finished sample, regenerate =======================
            const bool fresh = wf2_stage_r(S, P, total, coldBase + (size_t)s * CC_CHUNKS, s, active, rparts);
            __threadfence_block();
            wf2_push_trace(S, sc, split, hard ? WF2_Q_F0 + (cycle & 1) : WF2_Q_T, fresh, s);
            wf2_retire(S, active && !fresh);
        } else if (stage == WF2_Q_T || stage >= WF2_Q_F0) {
            // ===================== T: trace the pending ray =======================================
            bool isExt = false, isNee = false;
            if (active) {
                const uint32_t fl = S.flags[s];
                V3 o = v3(S.ox[s], S.oy[s], S.oz[s]);
                V3 d = v3(S.dx[s], S.dy[s], S.dz[s]);
                const float time = S.time[s];
                isExt = ((fl >> 3) & 1u) == WF2_PH_EXT;
                isNee = !isExt;
                if (isNee) {
                    // shadow ray from the surface point: origin = p + FaceForward(n, wi)*eps (render.cpp:121,170)
                    const V3 p = o + d * S.ht[s];
                    const V3 nn = v3(S.hnx[s], S.hny[s], S.hnz[s]);
                    d = v3(S.sdx[s], S.sdy[s], S.sdz[s]);
                    o = p + face_forward(nn, d) * TB_RAY_EPS;
                }
                if (isNee || maxDepth > 0) {
                    // one traversal instance serves both ray kinds (normals only for extension rays)
                    const Hit h = trace_closest(sc, o, d, time, isExt);
                    if (isExt) {
                        S.ht[s] = h.t;
                        S.hnx[s] = h.n.x; S.hny[s] = h.n.y; S.hnz[s] = h.n.z;
                        S.hprim[s] = h.prim;
                    } else {
                        S.st[s] = h.t;
                        S.sprim[s] = h.prim;
                    }
                } else {
                    S.hprim[s] = -2;   // maxDepth == 0: no trace at all, radiance stays 0
                }
            }
            __threadfence_block();
            wf2_push(S, WF2_Q_A, isExt, s);
            wf2_push(S, WF2_Q_B, isNee, s);
        } else if (stage == WF2_Q_A) {
            // ===================== A: extension-ray results =======================================
            bool cont = false, fin = false;
            if (active) {
                float4* rec = coldBase + (size_t)s * CC_CHUNKS;
                const float4 ct = cold_ld(rec, CC_T), cl = cold_ld(rec, CC_L);
                float4 ca;
                PathState ps;
                Surface sf;
                if (!wf2_hit<FEAT>(S, rec, sc, s, ct, cl, ca, ps, sf)) {
                    fin = true;
                } else {
                    const uint32_t fl = S.flags[s];
                    NeeCursor c;
                    ShadowRay sr;
                    nee_begin(c);
                    if (nee_generate(sc, sf, ps.time, c, ps.rng, sr)) {
                        cold_st(rec, CC_T, ps.T.x, ps.T.y, ps.T.z, ct.w);
                        cold_st(rec, CC_L, ps.L.x, ps.L.y, ps.L.z, cl.w);
                        wf2_store_shadow(S, rec, s, sr, c, ps.rng);
                        S.flags[s] = (fl & ~(1u << 3)) | ((uint32_t)WF2_PH_NEE << 3);
                        cont = true;
                    } else {
                        // scene without lights or probe: straight to the BSDF
                        cont = wf2_scatter(S, rec, sc, s, sf, ps.T, ps.L, ps.rng, ps.time, c.sum, (int)(fl >> 8), maxDepth, ps.absorb, ps.bsdfPdf, f2u(ca.w));
                        fin = !cont;
                    }
                }
            }
            __threadfence_block();
            wf2_push_trace(S, sc, split, WF2_Q_T, cont, s);
            wf2_push(S, WF2_Q_R, fin, s);
        } else {
            // ===================== B: shadow-ray results ==========================================
            bool cont = false, fin = false;
            if (active) {
                float4* rec = coldBase + (size_t)s * CC_CHUNKS;
                const float4 ct = cold_ld(rec, CC_T), cl = cold_ld(rec, CC_L), ca = cold_ld(rec, CC_A), cr = cold_ld(rec, CC_RNG);
                const float4 csh = cold_ld(rec, CC_SH), csum = cold_ld(rec, CC_SUM), cla = cold_ld(rec, CC_LA);
                const uint32_t fl = S.flags[s];
                const int bounce = (int)(fl >> 8);
                const Surface sf = wf2_surface(S, sc, s, ct.w);
                ShadowRay sr;
                sr.o = v3s(0.0f);
                sr.d = v3(S.sdx[s], S.sdy[s], S.sdz[s]);
                sr.dist = csh.x;
                sr.lightN = v3(csh.y, csh.z, csh.w);
                sr.skyPdf = csum.x;
                sr.light = __float_as_int(cr.w);
                NeeCursor c;
                const uint32_t cw = f2u(cr.z);
                c.slot = (int)(cw & 1u);
                c.prim = (int)((cw >> 8) & 0xfffu);
                c.sample = (int)(cw >> 20);
                c.sum = v3(csum.y, csum.z, csum.w);
                c.Lacc = v3(cla.x, cla.y, cla.z);
                Hit sh;
                sh.t = S.st[s];
                sh.prim = S.sprim[s];
                sh.n = v3s(0.0f);
                nee_connect(sc, sf, sr, sh, c);

                Rng rng;
                rng.s1 = f2u(cr.x);
                rng.s2 = f2u(cr.y);
                const float time = S.time[s];
                if (nee_generate(sc, sf, time, c, rng, sr)) {
                    wf2_store_shadow(S, rec, s, sr, c, rng);
                    cont = true;
                } else {
                    cont = wf2_scatter(S, rec, sc, s, sf, v3(ct.x, ct.y, ct.z), v3(cl.x, cl.y, cl.z), rng, time, c.sum, bounce, maxDepth,
                                       v3(ca.x, ca.y, ca.z), cl.w, f2u(ca.w));
                    fin = !cont;
                }
            }
            __threadfence_block();
            wf2_push_trace(S, sc, split, WF2_Q_T, cont, s);
            wf2_push(S, WF2_Q_R, fin, s);
        }
    }
}
