// wavefront2.cuh -- the product pipeline: a persistent, CTA-resident wavefront path tracer with a
// dedicated traversal stage.
//
// One CTA per SM stays resident for the whole launch and owns TB_WF2_PATHS path slots whose ENTIRE
// inter-stage state lives in SHARED MEMORY (SoA, 45 words per path: path state, pending shadow ray,
// hit records, next-event-estimation cursor).  A global-memory wavefront (tinsel's own unfinished
// wavefront.cu keeps ~150 B/path in DRAM and re-reads it in five kernels per bounce,
// wavefront.cu:765-796,1357-1375) would make queue traffic, not the scene, the HBM consumer; here
// HBM only sees scene misses and the framebuffer reductions.
//
// Every slot that is alive has exactly one pending ray: its extension ray or one shadow ray, and
// sits in exactly one CTA-shared stage queue.  Each WARP claims a chunk of up to 32 entries from a
// stage queue, processes it and appends the slots to the queues of their next stages:
//
//   R  finish + regenerate: splat the finished sample into the accumulator, claim a new sample
//      index from the global counter (one atomic per warp), generate its camera ray      -> T
//   T  trace the pending ray: closest hit -> hit record                        -> A (extension) / B (shadow)
//   A  extension result: miss -> sky -> R; hit -> absorption, emission MIS, first NEE sample -> T
//   B  shadow result: connect the NEE sample; next NEE sample -> T, or BSDF sample, throughput
//      update and next extension ray -> T, or termination -> R
//
// The lane-owned layout (wf2_lq, below) has no stage B: its stage A shades the whole bounce in place, in
// k_mega's order -- every NEE sample is generated, traced and connected right there, then the BSDF sample
// -> T, or termination -> R.  That saves the claim, push and slot-state round trip a shadow ray took through
// stage T (the claims halve), though on cornell the fused stage A costs nearly all of it back (DESIGN §5.1).
//
// The queues are lock-free rings in shared memory: producers reserve cells with one warp-
// aggregated atomicAdd on `tail` (ballot + prefix sum) and store lap-tagged slot ids, so a chunk
// is always full while the queue holds >= 32 entries (compaction is implicit in the queue).
// Regeneration keeps the slots populated until the sample counter runs dry; the CTA exits when
// its last slot dies.
//
// Who runs what when is the scheduler's business, and there are three of them (template MODE,
// chosen per scene on the host, see the comment at the kernel): free-running warps with no block
// barrier at all and a shared stage preference that keeps them loosely in step (they share the
// instruction cache: 32 KB of L1.5 against ~150 KB of kernel); block-synchronous hard phases with
// ticket claims for scenes where every hit spawns several shadow rays; and free-running with a
// second trace queue for rays that enter a big mesh.
//
// This header is compiled THREE TIMES by kernels.cu, in three namespaces, for the three layouts of the slot
// state and its queues (chosen with TB_WF2_PATHS / TB_WF2_COLD_SMEM / TB_WF2_LANEQ before each inclusion):
//   wf2_smem  1024 slots per CTA, the whole state in shared memory, ring queues -- scenes held on chip under
//             the hard-phase scheduler (several shadow rays per hit), 512-thread CTAs
//   wf2_lq    the same state with LANE-OWNED slots and bit-set queues (see wf2_push) -- scenes held on chip
//             under the free-running scheduler: no bank conflicts, cheap queue operations, no FIFO order
//   wf2_l2    2048 slots per CTA, the cold half of the state in global memory (L2), ring queues -- scenes with
//             deep mesh BVHs (768-thread CTAs), which gain from more paths in flight and from the rings' FIFO
//             order (rays pushed together are traced together)
// so it has no include guard, and only defines macros whose text is the same every time.

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

// Cold half of a slot's state: eight 16-byte chunks (seven used) per slot in global memory, read with
// ld.global.cg / written with st.global.cg by the one lane that owns the slot at the time (ownership
// moves through the stage queues, whose pushes are preceded by a block-scope fence).
//   0: T.xyz, eta        1: L.xyz, bsdfPdf     2: absorption.xyz, sample index
//   3: rng1, rng2, NEE cursor, sampled light   4: shadow dist, light normal.xyz
//   5: sky pdf, NEE sum.xyz                     6: NEE radiance accumulator.xyz
// The NEE cursor word (wf2_store_shadow): bit 0 "a shadow ray has been drawn at this hit" (NeeCursor::slot is only
// ever compared with 0, and a hit draws up to 1 + 4095 * 4095 of them), the primitive scan position in bits
// 8..19, the sample index within that light in bits 20..31.
// TB_WF2_COLD_SMEM: the same records in SHARED memory instead (stride 7 chunks), for builds with few enough
// slots per CTA: the cold half then costs 7 128-bit accesses per stage instead of 27 32-bit ones.
// TB_WF2_LANEQ: no shadow ray ever waits in a slot (stage A traces them in place), so only chunks 0-3 exist
// and chunk 3 holds the RNG alone.
#if defined(TB_WF2_LANEQ)
#ifndef TB_WF2_COLD_SMEM
#error "the lane-owned layout keeps the cold state in shared memory"
#endif
enum { CC_T = 0, CC_L = 1, CC_A = 2, CC_RNG = 3, CC_CHUNKS = 4 };
TB_DEV float4 cold_ld(const float4* rec, int c) { return rec[c]; }
TB_DEV void cold_st(float4* rec, int c, float x, float y, float z, float w) { rec[c] = make_float4(x, y, z, w); }
#elif defined(TB_WF2_COLD_SMEM)
enum { CC_T = 0, CC_L = 1, CC_A = 2, CC_RNG = 3, CC_SH = 4, CC_SUM = 5, CC_LA = 6, CC_CHUNKS = 7 };
TB_DEV float4 cold_ld(const float4* rec, int c) { return rec[c]; }
TB_DEV void cold_st(float4* rec, int c, float x, float y, float z, float w) { rec[c] = make_float4(x, y, z, w); }
#else
enum { CC_T = 0, CC_L = 1, CC_A = 2, CC_RNG = 3, CC_SH = 4, CC_SUM = 5, CC_LA = 6, CC_CHUNKS = 8 };
TB_DEV float4 cold_ld(const float4* rec, int c) { return __ldcg(rec + c); }
TB_DEV void cold_st(float4* rec, int c, float x, float y, float z, float w) { __stcg(rec + c, make_float4(x, y, z, w)); }
#endif
TB_DEV float u2f(uint32_t v) { return __uint_as_float(v); }
TB_DEV uint32_t f2u(float v) { return __float_as_uint(v); }

struct Wf2Shared {
    // HOT half of the slot state: what stage T (trace) reads and writes for every ray.  The cold half --
    // throughput, radiance, medium, RNG, the NEE bookkeeping: 27 words that only stages R, A and B touch,
    // once per ray -- lives in a 128-byte record per slot in global memory (Wf2Cold, L2-resident).  The
    // wavefront is bound by the number of paths an SM has in flight (halving the slots halves the
    // throughput on every scene, measured in round 2), and 18 words instead of 45 per slot double it.
    float ox[TB_WF2_PATHS], oy[TB_WF2_PATHS], oz[TB_WF2_PATHS];
    float dx[TB_WF2_PATHS], dy[TB_WF2_PATHS], dz[TB_WF2_PATHS];
    float time[TB_WF2_PATHS];
    uint32_t flags[TB_WF2_PATHS];     // bit 0 empty (no sample yet), bits 1-2 rayType, bit 3 phase, bits 8.. bounce
    // extension-ray hit
    float ht[TB_WF2_PATHS], hnx[TB_WF2_PATHS], hny[TB_WF2_PATHS], hnz[TB_WF2_PATHS];
    int hprim[TB_WF2_PATHS];
#ifndef TB_WF2_LANEQ
    // pending shadow ray (origin is recomputed from the surface point) and its result
    float sdx[TB_WF2_PATHS], sdy[TB_WF2_PATHS], sdz[TB_WF2_PATHS];
    float st[TB_WF2_PATHS];
    int sprim[TB_WF2_PATHS];
#endif
#ifdef TB_WF2_COLD_SMEM
    float4 cold[TB_WF2_PATHS * CC_CHUNKS];
#endif
#ifdef TB_WF2_LANEQ
    // stage queues as bit sets (lane-owned slots, see wf2_push below): one word per queue and lane
    unsigned int lq[3][32];
    // every primitive with lightSamples > 0 lies in [lightBegin, lightEnd): stage A's NEE scan starts and stops
    // there instead of loading every primitive's lightSamples in turn (a dependent chain on every hit)
    int lightBegin, lightEnd;
#else
    // stage queues: rings of lap-tagged slot ids
    uint16_t ring[7][TB_WF2_PATHS];
    unsigned int head[7], tail[7];
    unsigned int snap[5];             // hard-phase mode: the tail each stage of the current phase runs with
#endif
    int pref;                         // stage the warps currently prefer (soft phases, see the main loop)
    int live;                         // slots that still hold (or may still receive) a path
    int exhausted;
    // the scene descriptor every stage reads, pointing at the staged tables below: one copy per CTA, filled by
    // thread 0 in the prologue.  A per-thread copy would live in local memory (the stages take it by reference),
    // where every field read is a dependent L1 / L2 round trip at the head of a stage.
    DScene scene;
    // scene tables staged on chip by bulk copies (TMA) that complete on `stageBar`
    alignas(16) DPrim prims[TB_WF2_MAX_PRIMS + 1];   // +1: the copy length is rounded up to 16 bytes
    alignas(16) BvhPair pairs[TB_WF2_MAX_PAIRS];
    alignas(16) ProgOp flat[32];
    alignas(8) unsigned long long stageBar;
};

// dynamic shared memory of a CTA: the slot arrays
#define TB_WF2_SMEM_BYTES sizeof(Wf2Shared)

// stage queues.  T, A, B, R in the cyclic order of the free-running sweep; F0/F1 hold the freshly
// regenerated camera rays in hard-phase mode (double-buffered: R fills one while T drains the other)
// TM (free-running mode, scenes with DScene::splitValid): rays that enter the big mesh's box; same
// stage code as T, but a chunk taken from TM walks the mesh with all of its lanes and a chunk taken
// from T with none.
#ifdef TB_WF2_LANEQ
enum { WF2_Q_T = 0, WF2_Q_A = 1, WF2_Q_R = 2, WF2_NUM_Q = 3 };   // no B, no hard phases, no split trace queue
#else
enum { WF2_Q_T = 0, WF2_Q_A = 1, WF2_Q_B = 2, WF2_Q_R = 3, WF2_Q_F0 = 4, WF2_Q_F1 = 5, WF2_Q_TM = 6 };
#endif
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

#ifdef TB_WF2_LANEQ
// Lane-owned slots (the third layout, wf2_lq: scenes held on chip, free-running warps).  Slot s is only ever
// handled by lane (s & 31) of whichever warp claims it, so every access to the slot arrays is free of bank
// conflicts (lane i touches bank i; with ring queues the slot ids of a chunk are a random permutation, so most
// accesses to the slot arrays conflict), and a stage queue needs no ring: it is one bit per
// slot, the 32 slots of a lane in one word.  A push is one atomicOr by the owning lane on its own word -- no
// ballot, no prefix sum, no reserved-but-unwritten cell for a consumer to trip over.  The price is the FIFO
// order (a chunk is no longer a run of rays that were pushed together), which costs scenes with deep BVHs
// their traversal coherence: those keep the ring queues.
// The caller has fenced its slot-state writes (__threadfence_block).
static_assert(TB_WF2_PATHS == 1024, "one word per lane and queue");
#ifndef WF2_R_MIN_LANES
#define WF2_R_MIN_LANES 24   // stage R waits for that many lanes with a finished slot while T or A has work
#endif
#ifndef WF2_STICK_LANES
#define WF2_STICK_LANES 16     // a warp stays with the preferred stage while that many lanes have a slot waiting there
#endif
TB_DEV void wf2_push(Wf2Shared& S, int q, bool flag, int slot)
{
    if (flag) atomicOr(&S.lq[q][slot & 31], 1u << (slot >> 5));
}
#else
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
#endif

// Push a slot whose pending ray is ready to be traced.  With `split` set the ray (extension ray, or
// the shadow ray from the hit point) is classified against the big mesh's bounds first; the test
// is a scheduling heuristic, so the unoffset hit point is good enough as the shadow-ray origin.
TB_DEV void wf2_push_trace(Wf2Shared& S, const DScene& sc, bool split, int q, bool flag, int s)
{
#ifdef TB_WF2_LANEQ
    wf2_push(S, q, flag, s);   // no split trace queue in this layout
#else
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
#endif
}

#ifdef TB_WF2_LANEQ
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
#else
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

// the same claims as lane masks (lanes 0..n-1), the form the kernel body works with
TB_DEV unsigned wf2_lanes(int n) { return n >= 32 ? 0xffffffffu : ((1u << n) - 1u); }
#endif

TB_DEV Surface wf2_surface(const Wf2Shared& S, const DScene& sc, int s, float eta)
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

#ifndef TB_WF2_LANEQ
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
#endif

// finish the shading of a surface hit once all NEE samples are folded: BSDF sample, next ray
// (path_scatter) or termination.  Returns true when the slot continues with a new extension ray.
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV bool wf2_scatter(Wf2Shared& S, float4* rec, const DScene& sc, int s, const Surface& sf, V3 T, V3 L, Rng rng, float time, V3 neeSum,
                        int bounce, int maxDepth, V3 absorb, float bsdfPdf, uint32_t sample)
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
        go = path_scatter<FEAT>(sc, ps, sf, neeSum);
    }
    cold_st(rec, CC_L, ps.L.x, ps.L.y, ps.L.z, ps.bsdfPdf);
    if (!go) return false;
    S.ox[s] = ps.o.x; S.oy[s] = ps.o.y; S.oz[s] = ps.o.z;
    S.dx[s] = ps.d.x; S.dy[s] = ps.d.y; S.dz[s] = ps.d.z;
    cold_st(rec, CC_T, ps.T.x, ps.T.y, ps.T.z, ps.eta);
    cold_st(rec, CC_A, ps.absorb.x, ps.absorb.y, ps.absorb.z, u2f(sample));
    cold_st(rec, CC_RNG, u2f(ps.rng.s1), u2f(ps.rng.s2), 0.0f, 0.0f);
    S.flags[s] = ((uint32_t)ps.rayType << 1) | ((uint32_t)WF2_PH_EXT << 3) | ((uint32_t)(bounce + 1) << 8);
    return true;
}

// THREADS: 512 (16 warps, up to 128 registers) for scenes held in shared memory, where more warps
// only add instruction-cache pressure; 768 (24 warps, 80 registers) for scenes with deep mesh BVHs,
// whose traversal is latency bound on L2 and pays for the extra warps (LaunchParams::wideCta).
// MODE selects the scheduler that is compiled in -- measured, not principled: the kernel's speed is
// sensitive to register allocation and code layout, so every variant that is not needed is kept out
// of the others' bodies (measured in round 2):
//   WF2_MODE_GENERIC  both schedulers, run-time flag, no split trace queue (the free-running default;
//                     its own specialisation measured slower on cornell)
//   WF2_MODE_HARD     hard phases only (faster on veach)
//   WF2_MODE_SPLIT    free-running with the split trace queue TM (scenes with a big mesh)
enum { WF2_MODE_GENERIC = 0, WF2_MODE_HARD = 1, WF2_MODE_SPLIT = 2 };

#if defined(TB_WF2_STAGE_CLOCKS) && defined(TB_WF2_LANEQ)
// Per-stage cycle accounting of the lane-owned layout (development builds with -DTB_WF2_STAGE_CLOCKS, read by
// tb200_stage_clocks, see tools/stage_clocks.py).  Every warp sums clock64() deltas in registers and adds its
// totals here when it exits.  Stage kinds k: 0 R, 1 T, 2 A, 3 B (no B in this layout: its counters stay 0).
//   [0] claims that got slots   [1] idle: empty claims and the back-off   [2 + k] cycles in stage k
//   [6 + k] chunks of stage k   [10 + k] lanes active in those chunks      [14] warps
enum { WF2_CLK_CLAIM = 0, WF2_CLK_IDLE = 1, WF2_CLK_CYCLES = 2, WF2_CLK_CHUNKS = 6, WF2_CLK_LANES = 10, WF2_CLK_WARPS = 14, WF2_CLK_N = 15 };
static_assert(WF2_CLK_N == TB_WF2_STAGE_CLOCK_WORDS, "tb_kernels.cuh states the counter count");
__device__ unsigned long long g_wf2StageClocks[WF2_CLK_N];

// A warp's sums are 32 bits wide (fewer registers, so the accounting itself spills less): a warp lives for one
// launch, and the tool's launches last far fewer than 2^32 cycles.
struct Wf2Clocks {
    static constexpr int kinds = 3;   // R, T, A: this layout has no stage B
    unsigned int claim = 0, idle = 0, cyc[kinds] = {}, chunks[kinds] = {}, lanes[kinds] = {};

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

TB_DEV uint32_t wf2_smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// a generic address the compiler cannot trace back to shared memory: loads through it are generic loads
// (LD), so one instruction serves lanes that read the staged treelet and lanes that read global memory
TB_DEV const unsigned char* wf2_opaque(const void* p)
{
    unsigned long long a = (unsigned long long)p;
    asm volatile("" : "+l"(a));
    return reinterpret_cast<const unsigned char*>(a);
}

// FEAT: the scene features (TB_FEAT_*) compiled in.  The lane-owned layout has a second instantiation without any
// of them, for scenes that have none (wf2_lq::launch_layout); every other instantiation has them all.
template <int THREADS, int MODE, uint32_t FEAT = TB_FEAT_ALL>
__global__ void __launch_bounds__(THREADS, TB_WF2_CTAS_PER_SM) k_wavefront2(const __grid_constant__ LaunchParams P, unsigned long long total)
{
    extern __shared__ __align__(16) unsigned char wf_smem_raw[];
    Wf2Shared& S = *reinterpret_cast<Wf2Shared*>(wf_smem_raw);
    const int tid = threadIdx.x;

    // ---- prologue: stage the scene tables on chip ---------------------------------------------
    // Primitive records, the scene-level BVH (child-pair records) and the flat scene program go from
    // global to shared memory as TMA bulk copies (cp.async.bulk -> UBLKCP): thread 0 arms an mbarrier
    // with the byte count and issues up to three copies, everybody waits on the barrier's phase.
    const bool stagePrims = P.scene.numPrims <= TB_WF2_MAX_PRIMS;
    const bool stagePairs = P.scene.numPairs > 0 && P.scene.numPairs <= TB_WF2_MAX_PAIRS;
    const bool stageFlat = P.scene.numFlat > 0 && P.scene.numFlat <= 32;
    if (tid == 0) {
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
            unsigned char* tl = wf_smem_raw + ((sizeof(Wf2Shared) + 127) & ~size_t(127));
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
        // the CTA's scene descriptor (Wf2Shared::scene), published by the barrier below
        DScene d = P.scene;
        if (stagePrims) d.prims = S.prims;
        if (stagePairs) d.pairs = S.pairs;
        if (stageFlat) d.flat = S.flat;
        // the top of the biggest mesh's BVH goes into whatever shared memory the slot arrays leave (P.treeletBytes,
        // set by the launch from the device's limit): the first levels of every inline mesh walk are then shared-
        // memory reads instead of dependent L2 round trips
        d.treelet = nullptr;
        if (P.treeletBytes >= (int)sizeof(BvhPair) && d.treeletMesh >= 0) {
            unsigned char* tl = wf_smem_raw + ((sizeof(Wf2Shared) + 127) & ~size_t(127));
            d.treeletPairs = min(d.treeletPairs, P.treeletBytes / (int)sizeof(BvhPair));
            d.treelet = wf2_opaque(tl);
        } else {
            d.treeletPairs = 0;
        }
        S.scene = d;
#ifdef TB_WF2_LANEQ
        int lb = 0, le = 0;
        for (int i = P.scene.numPrims - 1; i >= 0; --i)
            if (P.scene.prims[i].lightSamples > 0) {
                if (le == 0) le = i + 1;
                lb = i;
            }
        S.lightBegin = lb;
        S.lightEnd = le;
#endif
    }
    const DScene& sc = S.scene;
    // every slot starts in the R queue "finished with nothing to splat": stage R fills it with a
    // camera sample
#ifdef TB_WF2_LANEQ
    for (int s = tid; s < TB_WF2_PATHS; s += THREADS) S.flags[s] = WF2_FLAG_EMPTY;
    if (tid < WF2_NUM_Q * 32) S.lq[tid >> 5][tid & 31] = (tid >> 5) == WF2_Q_R ? 0xffffffffu : 0u;
    if (tid == 0) {
#else
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
#endif
        S.pref = WF2_Q_R;
        S.live = TB_WF2_PATHS;
        S.exhausted = 0;
    }
    __syncthreads();   // the barrier word and S.scene are initialised (thread 0, above) before anybody reads them
    {
        uint32_t landed = 0;
        while (!landed)
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(landed)
                         : "r"(wf2_smem_addr(&S.stageBar)), "r"(0u)
                         : "memory");
    }

    const int maxDepth = P.film.maxDepth;
    const int lane = tid & 31;
#ifdef TB_WF2_COLD_SMEM
    float4* const coldBase = S.cold;
#else
    float4* const coldBase = P.cold + (size_t)blockIdx.x * TB_WF2_PATHS * CC_CHUNKS;
#endif

    // Two scheduling modes share the stage code below (P.hardPhases, uniform for the launch):
    //
    //  * hard phases: all warps of the CTA work through the same short list of stages, claiming
    //    chunks dynamically until each queue is empty, and meet at a block barrier twice per cycle.
    //    The kernel is far larger than the instruction cache, so warps that execute the same
    //    code at the same time share every instruction line; this is the faster mode when rays
    //    cost about the same (small scenes held in shared memory).
    //  * free running: no barriers at all; every warp picks the next stage itself, starting at a
    //    CTA-wide preferred stage and moving on cyclically when that queue has no full chunk left
    //    (dragging the preference along).  Nobody ever waits for a slow ray, which wins when ray
    //    cost varies wildly (deep mesh BVHs) and the hot loop is small enough to stay cached.
#ifdef TB_WF2_LANEQ
    static_assert(MODE == WF2_MODE_GENERIC, "the lane-owned layout serves the free-running scheduler only");
#else
    static_assert(FEAT == TB_FEAT_ALL, "only the lane-owned layout has a specialised instantiation");
#endif
#ifdef TB_WF2_LANEQ
    constexpr bool split = false;
#ifdef TB_WF2_STAGE_CLOCKS
    Wf2Clocks clk;
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
#else
    const bool hard = MODE == WF2_MODE_HARD ? true : MODE == WF2_MODE_SPLIT ? false : (P.hardPhases != 0);
    constexpr bool split = MODE == WF2_MODE_SPLIT;
    // hard-phase schedule: each cycle is two block-synchronous phases,
    //   phase 0:  R (finished slots -> fresh camera rays into F[cycle&1]),  T,  F[~cycle&1]
    //   phase 1:  A,  B
    // Inside a phase the stages run back to back without a barrier: they consume queues that were
    // completed before the phase began (so their tails are fixed and tickets cannot overshoot into
    // missing entries) and touch disjoint slots.  step 0..4 = R, T, F, A, B.
    int step = 0, cycle = 0;
    unsigned int stepTail = TB_WF2_PATHS;   // every slot starts in the R queue
    int stepQueue = WF2_Q_R;

    for (;;) {
        int s = 0, n = 0, stage = -1;
        if (hard) {
            n = wf2_claim_ticket(S, stepQueue, stepTail, s);
            if (n > 0) {
                stage = stepQueue;
            } else {
                // this stage's queue is drained; at the end of a phase meet the other warps, undo the
                // overshoot of the failed ticket requests (head back to the tail the stage ran with)
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
#endif

        if (stage == WF2_Q_R) {
            // ===================== R: splat the finished sample, regenerate =======================
            float4* rec = coldBase + (size_t)s * CC_CHUNKS;
            const bool finished = active && !(S.flags[s] & WF2_FLAG_EMPTY);
            uint32_t doneSample = 0xffffffffu;
            if (finished) {
                const float4 cl = cold_ld(rec, CC_L), ca = cold_ld(rec, CC_A);
                doneSample = f2u(ca.w);
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
            if (P.bandFlags)
                wf2_band_report(P.bandCount, P.bandFlags, P.bandSamples, (uint32_t)P.samplesPerFrame, P.bandTag, doneSample, finished);
            if (active) S.flags[s] = WF2_FLAG_EMPTY;
            // claim a new sample; indices on tile padding outside the image are skipped
            bool want = active && !*(volatile int*)&S.exhausted;
            bool fresh = false;
            for (int attempt = 0; attempt < 64; ++attempt) {
                if (!__any_sync(0xffffffffu, want)) break;
                const unsigned m = __ballot_sync(0xffffffffu, want);
                const int leader = __ffs(m) - 1;
                unsigned long long base = 0ull;
                if (lane == leader) {
                    base = atomicAdd(P.sampleCounter, (unsigned long long)__popc(m));
                    if (base + __popc(m) >= total) *(volatile int*)&S.exhausted = 1;
                }
                base = __shfl_sync(0xffffffffu, base, leader);
                const unsigned long long idx = base + (unsigned long long)__popc(m & ((1u << lane) - 1u));
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
                            cold_st(rec, CC_RNG, u2f(ps.rng.s1), u2f(ps.rng.s2), 0.0f, 0.0f);
                            S.flags[s] = ((uint32_t)TB_REFLECTED << 1) | ((uint32_t)WF2_PH_EXT << 3);
                            fresh = true;
                            want = false;
                        } else if (P.bandFlags) {
                            // tile padding outside the image retires at once
                            wf2_band_pad(P.bandCount, P.bandFlags, P.bandSamples, (uint32_t)P.samplesPerFrame, P.bandTag, (uint32_t)idx);
                        }
                    }
                }
            }
            __threadfence_block();
#ifdef TB_WF2_LANEQ
            wf2_push(S, WF2_Q_T, fresh, s);
#else
            wf2_push_trace(S, sc, split, hard ? WF2_Q_F0 + (cycle & 1) : WF2_Q_T, fresh, s);
#endif
            // slots that could not be refilled die: the CTA exits when none is left
            const unsigned dead = __ballot_sync(0xffffffffu, active && !fresh);
            if (dead && lane == 0) atomicSub(&S.live, __popc(dead));
#ifdef TB_WF2_LANEQ
        } else if (stage == WF2_Q_T) {
            // ===================== T: trace the extension ray (the only kind this layout queues) ==
            if (active) {
                if (maxDepth > 0) {
                    const Hit h = trace_closest<FEAT>(sc, v3(S.ox[s], S.oy[s], S.oz[s]), v3(S.dx[s], S.dy[s], S.dz[s]), S.time[s], true);
                    S.ht[s] = h.t;
                    S.hnx[s] = h.n.x; S.hny[s] = h.n.y; S.hnz[s] = h.n.z;
                    S.hprim[s] = h.prim;
                } else {
                    S.hprim[s] = -2;   // maxDepth == 0: no trace at all, radiance stays 0
                }
            }
            __threadfence_block();
            wf2_push(S, WF2_Q_A, active, s);
#else
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
#endif
        } else if (stage == WF2_Q_A) {
            // ===================== A: extension-ray results =======================================
            bool cont = false, fin = false;
            if (active) {
                float4* rec = coldBase + (size_t)s * CC_CHUNKS;
                const float4 ct = cold_ld(rec, CC_T), cl = cold_ld(rec, CC_L);
                const uint32_t fl = S.flags[s];
                const int bounce = (int)(fl >> 8);
                const int hprim = S.hprim[s];
                if (hprim < 0) {
                    if (hprim == -1) {
                        PathState ps;
                        ps.d = v3(S.dx[s], S.dy[s], S.dz[s]);
                        ps.T = v3(ct.x, ct.y, ct.z);
                        ps.L = v3(cl.x, cl.y, cl.z);
                        ps.rayType = (int)((fl >> 1) & 3u);
                        ps.bsdfPdf = cl.w;
                        path_miss<FEAT>(sc, ps, bounce);
                        cold_st(rec, CC_L, ps.L.x, ps.L.y, ps.L.z, cl.w);
                    }
                    fin = true;
                } else {
                    // hit prologue (render.cpp:255-310)
                    const float4 ca = cold_ld(rec, CC_A), cr = cold_ld(rec, CC_RNG);
                    PathState ps;
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
                    Surface sf;
                    path_hit<FEAT>(sc, ps, h, bounce, sf);
                    NeeCursor c;
                    ShadowRay sr;
#ifdef TB_WF2_LANEQ
                    nee_begin(c, S.lightBegin);
                    const int lightEnd = S.lightEnd;
                    // The whole bounce in place, in k_mega's order: every NEE sample traced and connected, then
                    // the BSDF sample.  What the traces do not need stays in the slot and is read back after
                    // them instead of being held in registers across them: the throughput and radiance path_hit
                    // left, and the surface (wf2_surface rebuilds it bit for bit, as stage B of the other layouts
                    // does).  s2 is s behind an empty asm, so the compiler cannot forward the stores to the reads.
                    // (Measured on cornell: keeping it all in registers spills, 160 bytes.)
                    cold_st(rec, CC_T, ps.T.x, ps.T.y, ps.T.z, ct.w);
                    cold_st(rec, CC_L, ps.L.x, ps.L.y, ps.L.z, cl.w);
                    const float time = ps.time;
                    Rng rng = ps.rng;
                    int s2 = s;
                    while (nee_generate<FEAT>(sc, sf, time, c, rng, sr, lightEnd)) {
                        const Hit sh = trace_closest<FEAT>(sc, sr.o, sr.d, time, false);
                        asm volatile("" : "+r"(s2) : "f"(sh.t));
                        sf = wf2_surface(S, sc, s2, ct.w);
                        nee_connect<FEAT>(sc, sf, sr, sh, c);
                    }
                    asm volatile("" : "+r"(s2));
                    const float4* rec2 = coldBase + (size_t)s2 * CC_CHUNKS;
                    const float4 t2 = cold_ld(rec2, CC_T), l2 = cold_ld(rec2, CC_L), a2 = cold_ld(rec2, CC_A);
                    cont = wf2_scatter<FEAT>(S, rec, sc, s, sf, v3(t2.x, t2.y, t2.z), v3(l2.x, l2.y, l2.z), rng, time, c.sum, (int)(S.flags[s] >> 8), maxDepth,
                                       v3(a2.x, a2.y, a2.z), l2.w, f2u(a2.w));
                    fin = !cont;
#else
                    nee_begin(c);
                    if (nee_generate(sc, sf, ps.time, c, ps.rng, sr)) {
                        cold_st(rec, CC_T, ps.T.x, ps.T.y, ps.T.z, ct.w);
                        cold_st(rec, CC_L, ps.L.x, ps.L.y, ps.L.z, cl.w);
                        wf2_store_shadow(S, rec, s, sr, c, ps.rng);
                        S.flags[s] = (fl & ~(1u << 3)) | ((uint32_t)WF2_PH_NEE << 3);
                        cont = true;
                    } else {
                        // scene without lights or probe: straight to the BSDF
                        cont = wf2_scatter(S, rec, sc, s, sf, ps.T, ps.L, ps.rng, ps.time, c.sum, bounce, maxDepth, ps.absorb, ps.bsdfPdf, f2u(ca.w));
                        fin = !cont;
                    }
#endif
                }
            }
            __threadfence_block();
            wf2_push_trace(S, sc, split, WF2_Q_T, cont, s);
            wf2_push(S, WF2_Q_R, fin, s);
        }
#ifndef TB_WF2_LANEQ
        else {
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
#endif
#if defined(TB_WF2_STAGE_CLOCKS) && defined(TB_WF2_LANEQ)
        clk.add(stage, (unsigned int)clock64() - t1, act);
#endif
    }
#if defined(TB_WF2_STAGE_CLOCKS) && defined(TB_WF2_LANEQ)
    clk.flush();
#endif
}

// The opt-in to > 48 KB of dynamic shared memory and the occupancy answer are PER DEVICE (and the
// attribute applies to the current device only), so they are kept per device ordinal and set up once
// per device under a lock: a host may own renderers on several GPUs, driven from several threads.
#define TB_WF2_MAX_DEVICES 64
template <int THREADS, int MODE, uint32_t FEAT>
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
                             (int)std::max(wavefront2_smem_limit(), (size_t)TB_WF2_SMEM_BYTES));
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_wavefront2<THREADS, MODE, FEAT>, THREADS, TB_WF2_SMEM_BYTES) != cudaSuccess || n < 1)
            n = 1;
        if (n > TB_WF2_MAX_CTAS_PER_SM) n = TB_WF2_MAX_CTAS_PER_SM;
        ctasPerSM[dev] = n;
    }
    return ctasPerSM[dev];
}

template <int THREADS, int MODE, uint32_t FEAT = TB_FEAT_ALL>
static void launch_wavefront2_t(const LaunchParams& p0, int numSMs, cudaStream_t stream, unsigned long long total)
{
    const int ctasPerSM = wavefront2_ctas_per_sm<THREADS, MODE, FEAT>();
    // shared memory beyond the slot arrays holds the treelet
    LaunchParams p = p0;
    const size_t slotBytes = (TB_WF2_SMEM_BYTES + 127) & ~size_t(127);
    p.treeletBytes = 0;
    if (p.scene.treeletMesh >= 0 && p.scene.treeletPairs > 0 && wavefront2_smem_limit() > slotBytes) {
        const size_t room = (wavefront2_smem_limit() - slotBytes) / sizeof(BvhPair) * sizeof(BvhPair);
        p.treeletBytes = (int)std::min(room, (size_t)p.scene.treeletPairs * sizeof(BvhPair));
    }
    const size_t smemBytes = p.treeletBytes > 0 ? slotBytes + (size_t)p.treeletBytes : TB_WF2_SMEM_BYTES;
    // TB_WF2_CTAS_PER_SM resident CTAs per SM; small jobs use fewer so that every CTA has a full slot array
    const unsigned long long want = (total + TB_WF2_PATHS - 1) / TB_WF2_PATHS;
    int grid = (numSMs > 0 ? numSMs : 132) * ctasPerSM;
    if (want < (unsigned long long)grid) grid = (int)want;
    if (grid < 1) grid = 1;
    k_wavefront2<THREADS, MODE, FEAT><<<grid, THREADS, smemBytes, stream>>>(p, total);
}

// the launches of this layout (see the top of the file for which scheduler variants each layout serves); returns
// the name of the kernel launched (nullptr: nothing to do)
const char* launch_layout(const LaunchParams& p, int numSMs, cudaStream_t stream, unsigned long long* launchCount)
{
    const unsigned long long total = p.samplesPerFrame * (unsigned long long)p.numFrames;
    if (total == 0ull) return nullptr;
    cudaMemsetAsync(p.sampleCounter, 0, sizeof(unsigned long long), stream);
#if !defined(TB_WF2_LANEQ)
    const bool split = !p.hardPhases && p.scene.splitValid;
#endif
    const char* name;
#if defined(TB_WF2_LANEQ)
    // scenes with none of the TB_FEAT_* features run the instantiation without them (LaunchParams::specialized).
    // Also 512 threads: at 640 (20 warps, 96 registers) it spills 128 bytes and measured no faster on cornell.
    if (p.specialized) {
        launch_wavefront2_t<TB_WF2_THREADS, WF2_MODE_GENERIC, TB_FEAT_NONE>(p, numSMs, stream, total);
        name = "wf2_lq.specialized";
    } else {
        launch_wavefront2_t<TB_WF2_THREADS, WF2_MODE_GENERIC>(p, numSMs, stream, total);
        name = "wf2_lq.generic";
    }
#elif defined(TB_WF2_COLD_SMEM)
    if (p.hardPhases) launch_wavefront2_t<TB_WF2_THREADS, WF2_MODE_HARD>(p, numSMs, stream, total);
    else if (split) launch_wavefront2_t<TB_WF2_THREADS, WF2_MODE_SPLIT>(p, numSMs, stream, total);
    else launch_wavefront2_t<TB_WF2_THREADS, WF2_MODE_GENERIC>(p, numSMs, stream, total);
    name = "wf2_smem";
#else
    if (split) {
        launch_wavefront2_t<TB_WF2_THREADS_WIDE, WF2_MODE_SPLIT>(p, numSMs, stream, total);
    } else {
        launch_wavefront2_t<TB_WF2_THREADS_WIDE, WF2_MODE_GENERIC>(p, numSMs, stream, total);   // hard phases too (run-time flag)
    }
    name = "wf2_l2";
#endif
    if (launchCount) ++*launchCount;
    return name;
}
