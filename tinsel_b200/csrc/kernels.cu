// kernels.cu -- sm_90a kernels of the tinsel_b200 path tracer.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false -prec-div=true -prec-sqrt=true
//        -ftz=false -lineinfo  (see tb_math.cuh for why contraction is off)
#include "tb_kernels.cuh"

// ------------------------------------------------------------------------------------------------
// Work decomposition.  A launch covers numFrames x (the 8x4 pixel tiles of this shard inside the
// row range).  Consecutive sample indices walk one tile (32 samples = one warp's worth of coherent
// camera rays), then the next tile of the row, then the shard's next tile row.
// ------------------------------------------------------------------------------------------------
void finalize_params(LaunchParams* p)
{
    if (p->numShards < 1) p->numShards = 1;
    p->tilesX = (p->film.width + 7) >> 3;
    const int tileRowsAll = (p->numRows + 3) >> 2;
    // tile rows t in [0, tileRowsAll) with t % numShards == shard
    p->tileRows = tileRowsAll > p->shard ? (tileRowsAll - p->shard + p->numShards - 1) / p->numShards : 0;
    p->samplesPerFrame = (unsigned long long)p->tilesX * (unsigned long long)p->tileRows * 32ull;
    divisor_magic((uint32_t)p->samplesPerFrame, &p->spfMul, &p->spfShift);
    divisor_magic((uint32_t)p->tilesX, &p->tilesXMul, &p->tilesXShift);
}

// Division by an invariant integer (Granlund and Montgomery, "Division by invariant integers using
// multiplication", 1994, section 4): with l = ceil(log2 d) and m = floor(2^32 (2^l - d) / d) + 1, which fits 32 bits,
// n / d = (mulhi(n, m) + n) >> l for every 32-bit n, the sum formed in 64 bits.  d = 0 (no samples) gives 0, 0.
void divisor_magic(uint32_t d, uint32_t* mul, uint32_t* shift)
{
    uint32_t l = 0;
    while (l < 32 && (1ull << l) < d) ++l;
    *mul = d ? (uint32_t)((((1ull << 32) * ((1ull << l) - d)) / d) + 1ull) : 0u;
    *shift = l;
}

TB_DEV uint32_t div_magic(uint32_t n, uint32_t mul, uint32_t shift) { return (uint32_t)(((unsigned long long)__umulhi(n, mul) + n) >> shift); }

// (launches are split on the host so that idx and samplesPerFrame fit 31 bits: 32-bit division, by the
// multipliers finalize_params computed)
TB_DEV bool decode_sample(const LaunchParams& P, unsigned long long idx64, int& px, int& py, int& frame)
{
    const uint32_t idx = (uint32_t)idx64, spf = (uint32_t)P.samplesPerFrame;
    const uint32_t f = div_magic(idx, P.spfMul, P.spfShift);
    frame = P.frame0 + (int)f;
    const uint32_t local = idx - f * spf;
    const uint32_t tile = local >> 5, in = local & 31u;
    const uint32_t tileY = div_magic(tile, P.tilesXMul, P.tilesXShift);
    px = (int)((tile - tileY * (uint32_t)P.tilesX) * 8u + (in & 7u));
    const int tileRow = (int)tileY * P.numShards + P.shard;
    const int ry = tileRow * 4 + (int)(in >> 3);
    py = P.firstRow + ry;
    return px < P.film.width && ry < P.numRows;
}

// ------------------------------------------------------------------------------------------------
// Shared per-sample prologue: the camera sample of (pixel, frame) (tb_film.cuh: camera_sample), then the path's
// start from its ray and the Random state after its draws.
// ------------------------------------------------------------------------------------------------
TB_DEV void sample_begin(const LaunchParams& P, int px, int py, int frame, PathState& ps, float& rasterX, float& rasterY)
{
    Rng rng;
    V3 origin, dir;
    float time;
    camera_sample(P.camera, P.film.width, px, py, (uint32_t)frame, rng, origin, dir, time, rasterX, rasterY);
    path_init(ps, origin, dir, time, rng);
}

TB_DEV void sample_end(const LaunchParams& P, int px, int py, float rasterX, float rasterY, V3 radiance)
{
    if (P.outRadiance) {
        const size_t p = (size_t)py * P.film.width + px;
        P.outRadiance[p * 3 + 0] = radiance.x;
        P.outRadiance[p * 3 + 1] = radiance.y;
        P.outRadiance[p * 3 + 2] = radiance.z;
        P.outRaster[p * 2 + 0] = rasterX;
        P.outRaster[p * 2 + 1] = rasterY;
    } else {
        add_sample(P.film, P.accum, rasterX, rasterY, radiance);
    }
}

// ------------------------------------------------------------------------------------------------
// Validation pipeline: one thread = one path, PathTrace's loop (render.cpp:250-385) verbatim in
// terms of the stage functions.  Kept as the simplest possible arrangement of the same device
// functions the wavefront kernel uses, so that a parity failure can be bisected between "math"
// and "scheduling".
// ------------------------------------------------------------------------------------------------
// (P is __grid_constant__: the stage functions take P.scene by reference, which would otherwise make a per-thread
// copy of the parameters in local memory)
__global__ void __launch_bounds__(128) k_mega(const __grid_constant__ LaunchParams P)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P.samplesPerFrame * (unsigned long long)P.numFrames) return;
    int px, py, frame;
    if (!decode_sample(P, idx, px, py, frame)) return;

    PathState ps;
    float rasterX, rasterY;
    sample_begin(P, px, py, frame, ps, rasterX, rasterY);

    for (int bounce = 0; bounce < P.film.maxDepth; ++bounce) {
        const Hit h = trace_closest(P.scene, ps.o, ps.d, ps.time, true);
        if (h.prim < 0) {
            path_miss(P.scene, ps, bounce);
            break;
        }
        Surface sf;
        path_hit(P.scene, ps, h, bounce, sf);

        NeeCursor cur;
        nee_begin(cur);
        ShadowRay sr;
        while (nee_generate(P.scene, sf, ps.time, cur, ps.rng, sr)) {
            const Hit sh = trace_closest(P.scene, sr.o, sr.d, ps.time, false);
            nee_connect(P.scene, sf, sr, sh, cur);
        }
        if (!path_scatter(P.scene, ps, sf, cur.sum)) break;
    }
    sample_end(P, px, py, rasterX, rasterY, ps.L);
}

const char* launch_mega(const LaunchParams& p, cudaStream_t stream, unsigned long long* launchCount)
{
    const unsigned long long total = p.samplesPerFrame * (unsigned long long)p.numFrames;
    if (total == 0ull) return nullptr;
    const int block = 128;
    const unsigned long long grid = (total + block - 1) / block;
    k_mega<<<(unsigned)grid, block, 0, stream>>>(p);
    if (launchCount) ++*launchCount;
    return "k_mega";
}

// ------------------------------------------------------------------------------------------------
// eNormals (render.cpp:494-515): ray through the integer raster position, time 1.0, overwrite.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_normals(const __grid_constant__ LaunchParams P)
{
    const int W = P.film.width;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P.numRows * W) return;
    const int ry = idx / W;
    // image-plane shards own the 4-row tile rows t with t % numShards == shard (decode_sample)
    if ((ry >> 2) % P.numShards != P.shard) return;
    const int py = P.firstRow + ry;
    const int px = idx % W;
    V3 origin, dir;
    generate_ray(P.camera, (float)px, (float)py, origin, dir);
    const Hit h = trace_closest(P.scene, origin, dir, 1.0f, true);
    float4 out = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (h.prim >= 0) {
        const V3 n = h.n * 0.5f + v3s(0.5f);
        out = make_float4(n.x, n.y, n.z, 1.0f);
    }
    P.accum[py * W + px] = out;
}

void launch_normals(const LaunchParams& p, cudaStream_t stream, unsigned long long* launchCount)
{
    const int total = p.numRows * p.film.width;
    if (total <= 0) return;
    k_normals<<<(total + 127) / 128, 128, 0, stream>>>(p);
    if (launchCount) ++*launchCount;
}

// ------------------------------------------------------------------------------------------------
// Wavefront pipeline: see wf2_common.cuh and launch_wavefront2 below
// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// Display/finish step: exposure / weight normalisation, filmic tone map, sRGB, 8-bit with the PNG
// writer's dither.  One thread = four consecutive pixels, so that the 8-bit output leaves as three
// 32-bit words per thread; 64 B read + 64 B (+12 B) written per thread, nothing re-read.
// ------------------------------------------------------------------------------------------------
static __device__ __noinline__ float tb_powf(float x, float y) { return tbm_powf(x, y); }

// ToneMap (util.h:25-42, filmic branch) followed by LinearToSrgb (maths.h:1545-1549), one channel
TB_DEV float finish_channel(float t)
{
    const float b = t - 0.004f;
    const float x = (0.0f < b) ? b : 0.0f;                       // Max(Vec3(0), texColor - Vec3(0.004))
    const float num = x * (6.2f * x + 0.5f);
    const float den = x * (6.2f * x + 1.7f) + 0.06f;             // Vec3(0.06): the double literal narrows to float
    const float ret = num / den;
    const float lin = tb_powf(ret, 2.2f);                        // SrgbToLinear
    return tb_powf(lin, 1.0f / 2.2f);                            // LinearToSrgb, kInvGamma = 1.0f/2.2f
}

// Quantize(c*255.0 + Randf() + Randf() - 0.5f), png.cpp:324-343: the sum is formed in double
// (255.0 is a double literal), narrowed to float at the call, clamped with Min(Max(x,0),255)
// (maths.h:55-65: a NaN ends up as 255) and truncated.
TB_DEV unsigned int finish_quantize(float c, Rng& rng)
{
    const float r1 = rng_float(rng);
    const float r2 = rng_float(rng);
    const double v = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)c, 255.0), (double)r1), (double)r2), (double)0.5f);
    float x = (float)v;
    x = (x < 0.0f) ? 0.0f : x;
    x = (x < 255.0f) ? x : 255.0f;
    return (unsigned int)(unsigned char)x;
}

__global__ void __launch_bounds__(128) k_finish(FinishParams P)
{
    const int quad = blockIdx.x * blockDim.x + threadIdx.x;
    const int first = quad * 4;
    if (first >= P.numPixels) return;
    unsigned int bytes[12];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int i = first + k;
        float4 f = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (i < P.numPixels) {
            const float4 p = __ldcs(&P.accum[i]);
            const float s = P.exposure / p.w;                    // main.cpp:267
            f.x = finish_channel(p.x * s);
            f.y = finish_channel(p.y * s);
            f.z = finish_channel(p.z * s);
            f.w = 0.0f;                                          // ToneMap builds Color(retColor, 0.0f)
            if (P.filtered) __stcs(&P.filtered[i], f);
            if (P.rgb8) {
                const uint2 st = __ldg(&P.ditherState[i]);
                Rng rng;
                rng.s1 = st.x;
                rng.s2 = st.y;
                bytes[k * 3 + 0] = finish_quantize(f.x, rng);
                bytes[k * 3 + 1] = finish_quantize(f.y, rng);
                bytes[k * 3 + 2] = finish_quantize(f.z, rng);
            }
        } else {
            bytes[k * 3 + 0] = bytes[k * 3 + 1] = bytes[k * 3 + 2] = 0u;
        }
    }
    if (P.rgb8) {
        // the buffer is allocated in multiples of 12 bytes, so the last thread may write its padding
        unsigned int* out = (unsigned int*)P.rgb8 + quad * 3;
#pragma unroll
        for (int w = 0; w < 3; ++w)
            out[w] = bytes[w * 4] | (bytes[w * 4 + 1] << 8) | (bytes[w * 4 + 2] << 16) | (bytes[w * 4 + 3] << 24);
    }
}

void launch_finish(const FinishParams& p, cudaStream_t stream, unsigned long long* launchCount)
{
    if (p.numPixels <= 0) return;
    const int quads = (p.numPixels + 3) / 4;
    k_finish<<<(quads + 127) / 128, 128, 0, stream>>>(p);
    if (launchCount) ++*launchCount;
}

// ------------------------------------------------------------------------------------------------
// Non-local means on the finished image (src/nlm.cpp).  One thread per pixel, 32x8 pixel blocks so
// that the window taps of a block overlap in L1; sums run in the reference's order (columns outer,
// rows inner) because fp32 addition order is part of the result.
// ------------------------------------------------------------------------------------------------
TB_DEV float4 f4_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
TB_DEV float4 f4_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }

// AverageFilter, nlm.cpp:4-34
__global__ void __launch_bounds__(256) k_nlm_mean(NlmParams P)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= P.width || y >= P.height) return;
    const int xlower = max(0, x - P.radius), xupper = min(P.width - 1, x + P.radius);
    const int ylower = max(0, y - P.radius), yupper = min(P.height - 1, y + P.radius);
    int count = 0;
    float4 sum = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    for (int fx = xlower; fx <= xupper; ++fx)
        for (int fy = ylower; fy <= yupper; ++fy) {
            sum = f4_add(sum, __ldg(&P.in[fy * P.width + fx]));
            count += 1;
        }
    P.means[y * P.width + x] = f4_scale(sum, 1.0f / (float)count);
}

// NonLocalMeansFilter, nlm.cpp:36-73
__global__ void __launch_bounds__(256) k_nlm(NlmParams P)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= P.width || y >= P.height) return;
    const int xlower = max(0, x - P.radius), xupper = min(P.width - 1, x + P.radius);
    const int ylower = max(0, y - P.radius), yupper = min(P.height - 1, y + P.radius);
    float totalWeight = 0.0f;
    float4 sum = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    const float4 mean = P.means[y * P.width + x];
    for (int fx = xlower; fx <= xupper; ++fx)
        for (int fy = ylower; fy <= yupper; ++fy) {
            const float4 m = P.means[fy * P.width + fx];
            const float dx = mean.x - m.x, dy = mean.y - m.y, dz = mean.z - m.z, dw = mean.w - m.w;
            const float lsq = dx * dx + dy * dy + dz * dz + dw * dw;       // LengthSq(Vec4), maths.h:331-332
            const float weight = tb_expf(-P.falloff * lsq);
            sum = f4_add(sum, f4_scale(__ldg(&P.in[fy * P.width + fx]), weight));
            totalWeight += weight;
        }
    __stcs(&P.out[y * P.width + x], f4_scale(sum, 1.0f / totalWeight));
}

void launch_nlm(const NlmParams& p, cudaStream_t stream, unsigned long long* launchCount)
{
    if (p.width <= 0 || p.height <= 0) return;
    const dim3 grid((p.width + 31) / 32, (p.height + 7) / 8);
    k_nlm_mean<<<grid, 256, 0, stream>>>(p);
    k_nlm<<<grid, 256, 0, stream>>>(p);
    if (launchCount) *launchCount += 2;
}

#include <algorithm>
#include <cstdlib>
#include <mutex>

// dynamic shared memory a CTA may opt in to on the current device (227 KB on sm_90a)
static size_t wavefront2_smem_limit()
{
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess || v <= 0) return 0;
    return (size_t)v;
}

// Three layouts of the wavefront's slot state and queues, each in its own namespace (see wf2_common.cuh):
//  * wf2_smem: the ring-queue kernel with 1024 slots per CTA, hot + cold state in shared memory.  Scenes held on
//    chip (cornell, veach): they are issue-bound, and fetching the cold half from L2 slows them down.
//  * wf2_l2: the ring-queue kernel with 2048 slots per CTA, the cold half in a 128-byte record per slot in global
//    memory, L2-resident.  Scenes with deep mesh BVHs (ajax, env): their rays take long, and twice the
//    paths in flight hide it.
//  * wf2_lq: the lane-owned kernel, 1024 slots per CTA in shared memory with LANE-OWNED slots and bit-set stage
//    queues instead of rings, free-running scheduler only: no shared-memory bank conflicts and far cheaper queue
//    operations, at the price of the rings' FIFO order (scenes held on chip do not care; deep BVHs such as ajax do).
namespace wf2_smem {
#undef TB_WF2_PATHS
#define TB_WF2_PATHS 1024
#define TB_WF2_COLD_SMEM 1
#include "wf2_common.cuh"
#include "wf2_rings.cuh"
#undef TB_WF2_COLD_SMEM
}  // namespace wf2_smem
namespace wf2_l2 {
#undef TB_WF2_PATHS
#define TB_WF2_PATHS 2048
#include "wf2_common.cuh"
#include "wf2_rings.cuh"
}  // namespace wf2_l2
namespace wf2_lq {
#undef TB_WF2_PATHS
#define TB_WF2_PATHS 1024
#define TB_WF2_COLD_SMEM 1
#include "wf2_common.cuh"
#include "wf2_lanes.cuh"
#undef TB_WF2_COLD_SMEM
}  // namespace wf2_lq

#ifdef TB_WF2_STAGE_CLOCKS
void read_stage_clocks(unsigned long long* out, bool reset) { wf2_lq::wf2_stage_clocks(out, reset); }
#endif

// The seven wavefront kernels, in the order launch_wavefront2 chooses between them.
using Wf2Launcher = void (*)(const LaunchParams&, int, cudaStream_t, unsigned long long);
static const struct {
    Wf2Launcher launch;
    const char* name;   // reported by tb200_last_kernel
} kWavefront2[] = {
    {wf2_l2::launch_wavefront2_t<TB_WF2_THREADS_WIDE, wf2_l2::WF2_MODE_SPLIT>, "wf2_l2.split"},
    {wf2_l2::launch_wavefront2_t<TB_WF2_THREADS_WIDE, wf2_l2::WF2_MODE_GENERIC>, "wf2_l2.generic"},
    {wf2_lq::launch_wavefront2_t<TB_WF2_THREADS, wf2_lq::WF2_MODE_GENERIC, TB_FEAT_NONE>, "wf2_lq.specialized"},
    {wf2_lq::launch_wavefront2_t<TB_WF2_THREADS, wf2_lq::WF2_MODE_GENERIC>, "wf2_lq.generic"},
    {wf2_smem::launch_wavefront2_t<TB_WF2_THREADS, wf2_smem::WF2_MODE_HARD>, "wf2_smem.hard"},
    {wf2_smem::launch_wavefront2_t<TB_WF2_THREADS, wf2_smem::WF2_MODE_SPLIT>, "wf2_smem.split"},
    {wf2_smem::launch_wavefront2_t<TB_WF2_THREADS, wf2_smem::WF2_MODE_GENERIC>, "wf2_smem.generic"},
};
enum { WF2_L2_SPLIT, WF2_L2_GENERIC, WF2_LQ_NONE, WF2_LQ_ALL, WF2_SMEM_HARD, WF2_SMEM_SPLIT, WF2_SMEM_GENERIC };

// Which of the seven kernels runs: every one produces the same bits, so the choice is speed alone.
// Per scene (wavefront2_route, at upload in tb200_create / tb200_create_cached, from the knobs read at its start):
//  * hardPhases = numNee > 1 && maxTris <= 4096 (TINSEL_B200_SCHED=hard|free overrides).  Block-synchronous stages
//    win when every hit spawns several shadow rays (the barrier keeps all warps on one stage's code); free-running
//    warps win otherwise, by a wide margin when ray cost varies (deep mesh BVHs).
//  * wideCta = !hardPhases && maxTris > 4096 (TINSEL_B200_CTA=768|512 overrides): more warps hide the L2 latency of
//    deep mesh BVHs; on scenes held in shared memory they only thrash the instruction cache.
//  * The split trace queue (rays entering the largest mesh's box queued apart) is in use when that box exists and
//    maxTris > 4096 or TINSEL_B200_SPLIT=1, never with TINSEL_B200_SPLIT=0; split = !hardPhases && in use.
//    tune = split && TINSEL_B200_SPLIT unset: api.cu: tune_update keeps the faster of split on and off.
//  * laneQueues = 1 (TINSEL_B200_QUEUES=ring: 0, =lanes: 2); specialized = no TB_FEAT_* feature and
//    TINSEL_B200_SPECIALIZE is not 0.
// Per launch (launch_wavefront2), with small = fewer than 6 x numSMs x 1024 samples, the first rule that applies:
//  1. wideCta: wf2_l2.split when split, else wf2_l2.generic (which runs hard phases too: P.hardPhases is read there).
//  2. !hardPhases, !split, and laneQueues 2, or 1 and not small: wf2_lq.specialized when specialized, else
//     wf2_lq.generic.  The lane-owned layout wins in the steady state (cornell 32 spp on an H100: 1131 vs 893
//     Msamples/s) and loses while the slots fill and drain (1-spp frames, slabs of a multi-GPU render; measured in
//     round 2).  The specialised kernel has 512-thread CTAs too: at 640 (20 warps, 96 registers) it spills 128
//     bytes and measured no faster on cornell.
//  3. Otherwise wf2_smem.hard when hardPhases, else wf2_smem.split when split, else wf2_smem.generic.
Wf2Route wavefront2_route(int numNee, int maxTris, bool splitBox, uint32_t features, const Knobs& knobs)
{
    Wf2Route r;
    r.hardPhases = numNee > 1 && maxTris <= 4096;
    if (knobs.sched == 1) r.hardPhases = true;
    if (knobs.sched == 0) r.hardPhases = false;
    r.wideCta = !r.hardPhases && maxTris > 4096;
    if (knobs.cta == 768) r.wideCta = true;
    if (knobs.cta == 512) r.wideCta = false;
    const bool splitQueue = splitBox && (maxTris > 4096 || (knobs.splitSet && knobs.split == 1)) && !(knobs.splitSet && knobs.split == 0);
    r.split = !r.hardPhases && splitQueue;
    r.tune = r.split && !knobs.splitSet;
    r.laneQueues = knobs.laneQueues;
    r.specialized = features == TB_FEAT_NONE && knobs.specialize;
    return r;
}

// Launches the kernel the route calls for (see above); returns its name (nullptr: nothing to do).
const char* launch_wavefront2(const LaunchParams& p, const Wf2Route& route, int numSMs, cudaStream_t stream, unsigned long long* launchCount)
{
    const unsigned long long total = p.samplesPerFrame * (unsigned long long)p.numFrames;
    if (total == 0ull) return nullptr;
    const bool small = total < 6ull * (unsigned long long)(numSMs > 0 ? numSMs : 132) * 1024ull;
    int k;
    if (route.wideCta)
        k = route.split ? WF2_L2_SPLIT : WF2_L2_GENERIC;
    else if (!route.hardPhases && !route.split && (route.laneQueues == 2 || (route.laneQueues == 1 && !small)))
        k = route.specialized ? WF2_LQ_NONE : WF2_LQ_ALL;
    else
        k = route.hardPhases ? WF2_SMEM_HARD : route.split ? WF2_SMEM_SPLIT : WF2_SMEM_GENERIC;
    LaunchParams q = p;
    q.hardPhases = route.hardPhases;
    cudaMemsetAsync(q.sampleCounter, 0, sizeof(unsigned long long), stream);
    kWavefront2[k].launch(q, numSMs, stream, total);
    if (launchCount) ++*launchCount;
    return kWavefront2[k].name;
}

// ------------------------------------------------------------------------------------------------
// Batched closest-hit ray query: see tb_query.cuh
// ------------------------------------------------------------------------------------------------
#include "tb_query.cuh"

// ------------------------------------------------------------------------------------------------
// The probe's sampling tables (Probe::BuildCDF): see tb_probe.cuh
// ------------------------------------------------------------------------------------------------
#include "tb_probe.cuh"
