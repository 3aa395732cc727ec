// tb_kernels.cuh -- kernel launch interface shared by api.cu (host side) and kernels.cu.
#pragma once

#include "tb_film.cuh"

// path slots per CTA of the wavefront kernel, at most (the layouts of kernels.cu use 1024 and 2048): the host
// sizes the cold slot state with it
#define TB_WF2_SLOTS 2048
#define TB_WF2_MAX_CTAS_PER_SM 2   // the launch never places more CTAs per SM (the host sizes the cold state with it)

struct LaunchParams {
    DScene scene;
    DCamera camera;
    DFilm film;
    float4* accum;        // width*height running sums
    unsigned long long* sampleCounter;   // per-renderer work counter of the wavefront kernel
    int hardPhases;       // wavefront scheduling mode: 1 = block-synchronous stages, 0 = free-running warps (set by launch_wavefront2)
    int frame0;           // first frame (sample index per pixel)
    int numFrames;        // frames to trace in this launch
    int firstRow;         // pixel rows [firstRow, firstRow+numRows) are traced ...
    int numRows;
    int shard, numShards; // ... restricted to 4-row tile rows t with t % numShards == shard
    int tilesX;           // 8-pixel tile columns
    int tileRows;         // tile rows owned by this shard inside the row range
    unsigned long long samplesPerFrame;   // tilesX * tileRows * 32 (includes padding outside the image)
    uint32_t spfMul, spfShift;            // division by samplesPerFrame and by tilesX: divisor_magic, set by finalize_params
    uint32_t tilesXMul, tilesXShift;
    // tb200_trace_frame outputs (nullptr in normal rendering)
    float* outRadiance;   // 3 floats per pixel
    float* outRaster;     // 2 floats per pixel
    // streamed read-back (tb200_render, single-frame launches; nullptr/0 otherwise): the sample range
    // is cut into bands of `bandSamples` consecutive indices (whole tile rows); the thread that
    // retires the last sample of a band stores `bandTag` into bandFlags[band] (mapped host memory),
    // so the host can copy finished rows while the kernel is still tracing the rest.
    unsigned int* bandCount;          // device counters, zeroed before the launch
    volatile unsigned int* bandFlags; // device pointer to pinned, mapped host memory
    unsigned int bandSamples;
    unsigned int bandTag;
    // cold half of the wavefront's slot state: 8 x float4 per slot, TB_WF2_PATHS slots per CTA of the launch
    float4* cold;
    int treeletBytes;     // shared memory behind the slot arrays that the prologue fills with the top of DScene::treeletMesh's BVH
};

// The per-scene part of the choice of wavefront kernel (kernels.cu: wavefront2_route, launch_wavefront2).
struct Wf2Route {
    bool hardPhases;    // block-synchronous stages rather than free-running warps
    bool wideCta;       // 768-thread CTAs (wf2_l2) rather than 512
    bool split;         // free-running with the split trace queue; the tuner may change it between launches
    bool tune;          // the split-queue tuner decides `split` by measurement (api.cu: tune_update)
    bool specialized;   // no TB_FEAT_* feature: the lane-owned kernel compiled without them
    int laneQueues;     // lane-owned slots with bit-set queues: 0 never, 1 for launches that are not small, 2 always
};

// The run-time knobs (README, "Run-time knobs"): environment variables that choose between variants which all give
// the same bits.  api.cu: read_knobs is the library's only reader of them; each tb200_create* call reads them once,
// at its start.  Each variable, how its value is read, and what it does:
//   TINSEL_B200_PIPELINE=mega          mega: the validation kernel k_mega (one thread per path) instead of the wavefront kernel
//   TINSEL_B200_READBACK=plain         plainReadback: tb200_render copies after the launch instead of streaming rows under it
//   TINSEL_B200_TEST_LAUNCH_SAMPLES=n  launchSamples (strtoull): test hook, n > 0 lowers the 2^31-1 samples per launch
//   TINSEL_B200_TEST_DUP_DEVICES       dupDevices (set at all): test hook, tb200_create_multi accepts a device twice
//   TINSEL_B200_SCHED=hard|free        sched (1, 0; -1 for any other value): forces Wf2Route::hardPhases
//   TINSEL_B200_SPLIT=1|0              splitSet, split (atoi): 1 forces the split trace queue on, 0 off; set to any
//                                      value at all, it turns off the tuner (Wf2Route::tune)
//   TINSEL_B200_CTA=768|512            cta (atoi): forces Wf2Route::wideCta on or off; other values leave the rule's
//   TINSEL_B200_QUEUES=ring|lanes      laneQueues: Wf2Route::laneQueues 0 or 2; unset or any other value gives 1
//   TINSEL_B200_SPECIALIZE=0           specialize (false when atoi is 0, non-numeric text included): featureless
//                                      scenes run the generic lane-owned kernel
//   TINSEL_B200_NO_FLAT                noFlat (set at all, even to 0): the scene level runs the reference-order BVH
//                                      walk instead of the flat scene program
//   TINSEL_B200_TREELET=1              treelet (atoi is 1): stage the top of the biggest mesh's BVH in shared memory
struct Knobs {
    bool mega;
    bool plainReadback;
    unsigned long long launchSamples;   // 0 when unset
    bool dupDevices;
    int sched;
    bool splitSet;
    int split;
    int cta;
    int laneQueues;
    bool specialize;
    bool noFlat;
    bool treelet;
};

#define TB_MAX_BANDS 64

// fills tilesX / tileRows / samplesPerFrame and their division multipliers from the row range and shard
void finalize_params(LaunchParams* p);
// multiplier and shift that divide every 32-bit integer by d exactly (kernels.cu; tb200_divisor_magic)
void divisor_magic(uint32_t d, uint32_t* mul, uint32_t* shift);

// The launches below return the name of the kernel they ran (nullptr when there was no work), for tb200_last_kernel.
// one thread per (pixel, frame): the whole path in registers.  Validation / fallback pipeline.
const char* launch_mega(const LaunchParams& p, cudaStream_t stream, unsigned long long* launchCount);
// persistent CTA-resident wavefront pipeline with a dedicated traversal stage (the product path), and its route for
// a scene of numNee shadow rays per hit, largest mesh maxTris triangles (splitBox: its box in DScene), features,
// under the renderer's knobs
Wf2Route wavefront2_route(int numNee, int maxTris, bool splitBox, uint32_t features, const Knobs& knobs);
const char* launch_wavefront2(const LaunchParams& p, const Wf2Route& route, int numSMs, cudaStream_t stream, unsigned long long* launchCount);
#ifdef TB_WF2_STAGE_CLOCKS
// development builds: the per-stage cycle counters of the lane-owned wavefront layout (wf2_lanes.cuh), summed
// over every launch since the last reset
#define TB_WF2_STAGE_CLOCK_WORDS 23
void read_stage_clocks(unsigned long long* out, bool reset);
#endif
// eNormals mode (render.cpp:494-515)
void launch_normals(const LaunchParams& p, cudaStream_t stream, unsigned long long* launchCount);

// Display/finish step (src/main.cpp:258-271, src/png.cpp:329-343), see tb200_finish.
struct FinishParams {
    const float4* accum;      // width*height running sums
    int numPixels;
    float exposure;
    float4* filtered;         // device, or nullptr
    unsigned char* rgb8;      // device (numPixels*3 bytes, allocated in multiples of 12), or nullptr
    const uint2* ditherState; // WritePng's Random state in front of each pixel's six draws (when rgb8)
};
void launch_finish(const FinishParams& p, cudaStream_t stream, unsigned long long* launchCount);

// NonLocalMeansFilter (src/nlm.cpp:4-73) on the finished image; see tb200_nlm.
struct NlmParams {
    const float4* in;     // finished image (k_finish output)
    float4* means;        // scratch: AverageFilter output
    float4* out;
    int width, height, radius;
    float falloff;
};
void launch_nlm(const NlmParams& p, cudaStream_t stream, unsigned long long* launchCount);

// The batched queries (tb_query.cuh): the ray queries, each Trace (render.cpp:17-62) of every ray of a caller's
// batch; the BSDF queries, one Disney BSDF call (disney.h) per query record; the two ends of a path, the
// renderer's camera sample and the film's AddSample, per sample record; the light queries, SampleLights per
// surface record and the sky of a miss per ray; and the two draws SampleLights is made of, PrimitiveSample per
// emitter record and ProbeSample per seed:
enum class QueryKind {
    Closest,      // tb200_trace_rays: the closest hit
    ClosestTri,   // tb200_trace_rays_tri: the closest hit and the winner's triangle and barycentric weights
    Occluded,     // tb200_occluded_rays: whether Trace hits something before the ray's tmax
    BsdfEval,     // tb200_bsdf_eval: BSDFEval and BSDFPdf
    BsdfSample,   // tb200_bsdf_sample: BSDFSample, then BSDFEval of the sampled direction
    CameraRays,   // tb200_camera_rays: the camera ray and raster position of a (pixel, frame) sample
    Splat,        // tb200_splat: AddSample of a caller's radiance at a raster position
    SampleLights, // tb200_sample_lights: SampleLights (next-event estimation) at a surface point
    Sky,          // tb200_sky_eval: Sky::Eval and ProbePdf of a direction
    SampleEmitters,   // tb200_sample_emitters: PrimitiveSample of a light primitive
    SampleProbe,      // tb200_sample_probe: ProbeSample of the sky's probe
};
// Every query's parameters.  The input and output pointers a query does not use stay null.
struct QueryParams {
    DScene scene;
    const float4* rays;   // Closest, ClosestTri, Occluded: 2 per ray: origin.xyz, time; dir.xyz, pad (Occluded: tmax)
    float4* hits;         // Closest, ClosestTri: 1 per ray: t, normal.xyz
    int* prims;           // Closest, ClosestTri: 1 per ray: closest primitive, -1 on a miss
    int4* tris;           // ClosestTri: 1 per ray: triangle, then the bits of u, v, w; -1, 0, 0, 0 unless a mesh was hit
    unsigned char* occluded;   // Occluded: 1 per ray: 1 when occluded, else 0
    const float4* bsdfQueries;  // BsdfEval, BsdfSample: 3 per query: n.xyz, prim bits; v.xyz, etaI; l.xyz, etaO
    const uint32_t* seeds;      // BsdfSample: 1 per query: the Random seed
    float4* bsdfValues;         // BsdfEval: 1 per query: f.rgb, pdf
    float4* bsdfSamples;        // BsdfSample: 2 per query: l.xyz, pdf; f.rgb, type bits
    long long numRays;    // records in the batch (rays, BSDF queries or samples)
    unsigned long long* counter;   // work counter of the ray queries, cleared by the launch
    // (the members below come after the others, so that the five kernels above keep their parameter offsets)
    DCamera camera;       // CameraRays: the camera, set up for film.width x film.height
    DFilm film;           // CameraRays: the image size; Splat: the film and its filter, rows [0, height)
    const int2* cameraSamples;   // CameraRays: 1 per sample: pixel, frame
    float4* cameraRays;          // CameraRays: 2 per sample: origin.xyz, time; dir.xyz, +inf
    float2* rasterOut;           // CameraRays: 1 per sample: raster position
    const float2* rasterIn;      // Splat: 1 per sample: raster position
    const float* radiance;       // Splat: 3 per sample: rgb
    float4* accum;               // Splat: film.width * film.height running sums
    // (and these after those, so that the seven kernels above keep theirs)
    const float4* lightQueries;  // SampleLights: 4 per query: p.xyz, time; n.xyz, prim bits; wo.xyz, etaI; etaO, pad
    float* lightRadiance;        // SampleLights: 3 per query: rgb (seeds: 1 per query, the Random seed)
    float4* skyOut;              // Sky: 1 per ray (of rays, whose dir alone is read): Sky::Eval rgb, ProbePdf
    // (and these after all those, so that the nine kernels above keep theirs)
    const float2* emitterQueries;   // SampleEmitters: 1 per query: prim bits, time (seeds: 1 per query)
    float4* emitterOut;             // SampleEmitters: 2 per query: pos.xyz, 0; normal.xyz, 0
    float4* probeOut;               // SampleProbe: 2 per seed: dir.xyz, pdf; color.rgb, 0
};
// Unlike the launches above, it leaves tb200_last_kernel alone and so returns no kernel name.
void launch_query(QueryKind kind, const QueryParams& p, int numSMs, cudaStream_t stream, unsigned long long* launchCount);

// Probe::BuildCDF (src/probe.h:31-79) on the device (tb_probe.cuh): from width*height RGBA texels, pdfX and cdfX
// (width*height floats each), pdfY and cdfY (height floats each).  width*height < INT32_MAX.  Three launches.
struct ProbeTablesParams {
    const float4* probe;
    int width, height;
    float *pdfX, *cdfX, *pdfY, *cdfY;
};
void launch_probe_tables(const ProbeTablesParams& p, cudaStream_t stream, unsigned long long* launchCount);
