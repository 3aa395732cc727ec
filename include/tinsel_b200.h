/*
 * tinsel_b200.h -- C ABI of the H100-native wavefront path tracer.
 *
 * This is the drop-in boundary for tinsel's one data-parallel hot path
 * (ray-gen -> two-level BVH traversal -> Disney BSDF -> MIS next-event
 * estimation -> filtered framebuffer accumulation).  Plain pointers and sizes
 * only: no C++ types, no torch types.  The reference-side C++ adapter that
 * turns these entry points back into tinsel's
 *     Renderer* CreateGpuWavefrontRenderer(const Scene* s);     (src/render.h:78)
 *     virtual void Renderer::Init(int width, int height);       (src/render.h:70)
 *     virtual void Renderer::Render(const Camera&, const Options&, Color*);  (src/render.h:71)
 * lives in tinsel_b200/plugin/tinsel_plugin.cpp and is shown in INTEGRATION.md.
 *
 * Every POD struct below mirrors a reference struct field-for-field in meaning
 * (not in byte layout: pointers-to-host-Mesh become mesh indices, the unused
 * bump-map fields are dropped).  File:line citations are under /root/reference.
 */
#ifndef TINSEL_B200_H
#define TINSEL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- POD mirrors of the reference's input types ------------------------------------------ */

/* Transform (src/maths.h:575-589): rigid transform with uniform scale. */
typedef struct tb200_transform {
    float p[3];      /* translation                     */
    float r[4];      /* rotation quaternion x,y,z,w     */
    float s;         /* uniform scale                   */
} tb200_transform;

/* Material (src/scene.h:45-102) without the unused bump-map fields. */
typedef struct tb200_material {
    float emission[3];
    float color[3];
    float absorption[3];
    float eta;
    float metallic;
    float subsurface;
    float specular;
    float roughness;
    float specularTint;
    float anisotropic;     /* parsed, unused by the reference BSDF (src/disney.h) */
    float sheen;           /* parsed, unused */
    float sheenTint;       /* parsed, unused */
    float clearcoat;
    float clearcoatGloss;
    float transmission;
} tb200_material;

/* GeometryType (src/scene.h:104-109) */
enum { TB200_SPHERE = 0, TB200_PLANE = 1, TB200_MESH = 2 };

/* Primitive (src/scene.h:142-159).  `mesh` indexes tb200_scene::meshes (the reference
 * identifies shared meshes by MeshGeometry::id, src/util.h:20). */
typedef struct tb200_primitive {
    tb200_transform start;       /* startTransform */
    tb200_transform end;         /* endTransform   */
    int32_t type;                /* TB200_SPHERE / TB200_PLANE / TB200_MESH */
    float radius;                /* SphereGeometry::radius  */
    float plane[4];              /* PlaneGeometry::plane    */
    int32_t mesh;                /* index into meshes, -1 if not a mesh */
    tb200_material material;
    int32_t lightSamples;        /* >0: explicitly sampled area light */
} tb200_primitive;

/* BVHNode (src/bvh.h:9-19), identical 32-byte layout: the reference's bitfield
 * `rightIndex:31, leaf:1` is the low 31 bits / top bit of right_leaf. */
typedef struct tb200_bvh_node {
    float lower[3];
    float upper[3];
    uint32_t left;               /* leaf: item index; interior: left child node index */
    uint32_t right_leaf;         /* bits 0..30 right child node index, bit 31 leaf flag */
} tb200_bvh_node;

/* The most levels of interior nodes a BVH (scene level or mesh) may have: the traversal keeps its
 * pending nodes in a fixed 32-entry stack, as the reference does.  Every BVH is also a tree: walked
 * from node 0, no node is reached twice.  tb200_create, tb200_scene_cache_save and
 * tb200_create_cached refuse a scene that breaks either rule; tb200_bvh_build never returns one. */
#define TB200_MAX_BVH_LEVELS 31

/* The most primitives a scene may have, and the most lightSamples one primitive may take: the wavefront
 * kernel keeps a hit's next-event-estimation position (a primitive index, and a sample index within that
 * light) in two 12-bit fields.  tb200_create, tb200_scene_cache_save and tb200_create_cached refuse more. */
#define TB200_MAX_PRIMITIVES 4095
#define TB200_MAX_LIGHT_SAMPLES 4095

/* MeshGeometry (src/scene.h:121-139).  All pointers are borrowed host memory. */
typedef struct tb200_mesh {
    const float* positions;      /* numVertices * 3 */
    const float* normals;        /* numVertices * 3 */
    const int32_t* indices;      /* numIndices      */
    const tb200_bvh_node* nodes; /* numNodes        */
    const float* cdf;            /* numIndices / 3, area CDF (src/mesh.cpp RebuildCDF) */
    int32_t numVertices;
    int32_t numIndices;
    int32_t numNodes;
    float area;
} tb200_mesh;

/* Sky + Probe (src/scene.h:161-181, src/probe.h:9-86). */
typedef struct tb200_sky {
    float horizon[3];
    float zenith[3];
    int32_t probeValid;
    int32_t probeWidth;
    int32_t probeHeight;
    const float* probeData;      /* width*height*4 (Color rgba) */
    const float* pdfValuesX;     /* width*height */
    const float* cdfValuesX;     /* width*height */
    const float* pdfValuesY;     /* height */
    const float* cdfValuesY;     /* height */
} tb200_sky;

/* Scene (src/scene.h:183-217): primitives + scene-level BVH over them + sky. */
typedef struct tb200_scene {
    const tb200_primitive* primitives;
    int32_t numPrimitives;
    const tb200_mesh* meshes;
    int32_t numMeshes;
    const tb200_bvh_node* bvhNodes;  /* Scene::bvh.nodes */
    int32_t numBvhNodes;
    tb200_sky sky;
} tb200_scene;

/* Camera (src/scene.h:11-31) */
typedef struct tb200_camera {
    float position[3];
    float rotation[4];
    float fov;
    float shutterStart;
    float shutterEnd;
} tb200_camera;

/* Options + Filter (src/render.h:13-63); same field order as the reference.
 * Every call that takes options refuses them (returns -1, tb200_last_error says why, nothing is launched and
 * the accumulator is untouched) when filterType is neither TB200_FILTER_BOX nor TB200_FILTER_GAUSSIAN, or when
 * filterWidth is not finite or is 2^30 or more in magnitude: the splat converts raster +- filterWidth to int,
 * and only below that bound does the conversion mean the same on every side.  filterFalloff, filterOffset and
 * clamp only enter arithmetic and are taken as they are, NaN and infinities included. */
enum { TB200_FILTER_BOX = 0, TB200_FILTER_GAUSSIAN = 1 };
enum { TB200_MODE_NORMALS = 0, TB200_MODE_COMPLEXITY = 1, TB200_MODE_PATHTRACE = 2 };
typedef struct tb200_options {
    int32_t mode;
    int32_t width;
    int32_t height;
    int32_t filterType;
    float filterWidth;
    float filterFalloff;
    float filterOffset;   /* used as handed in, never recomputed (loader quirk, src/loader.cpp:75) */
    float exposure;
    float limit;
    float clamp;
    int32_t maxDepth;
    int32_t maxSamples;
} tb200_options;

/* Per-renderer counters since tb200_init (all monotonically increasing). */
typedef struct tb200_stats {
    uint64_t frames;          /* Render() calls (1 spp each) since Init      */
    uint64_t samples;         /* camera paths traced                          */
    uint64_t kernelLaunches;  /* CUDA kernels launched by this renderer       */
    uint64_t d2hBytes;        /* bytes copied device->host                    */
    uint64_t h2dBytes;        /* bytes copied host->device (scene upload etc) */
    double   gpuMs;           /* CUDA-event time of the last render call      */
} tb200_stats;

typedef struct tb200_renderer tb200_renderer;

/* ---- entry points ------------------------------------------------------------------------- */

/* Replaces CreateGpuWavefrontRenderer(const Scene*) (src/render.h:78; the reference's own
 * definition, src/wavefront.cu:1384, is in no build).  Uploads and re-lays-out the scene for
 * the GPU.  `device` is the CUDA ordinal.  Returns NULL on failure (see tb200_last_error). */
tb200_renderer* tb200_create(const tb200_scene* scene, int device);

/* The same renderer spread over several GPUs of one box (one process, one host thread per further
 * device inside the library): the scene is replicated, tb200_init cuts the image into one contiguous
 * slab of pixel rows per device (cut at 4-row tile rows), every device traces the samples of its slab
 * plus those of the rows within the filter's reach outside it -- so it holds COMPLETE sums for the
 * rows it owns, from bit-identical duplicated samples (SURVEY 8e) -- and tb200_render has each device
 * stream its own rows into `output` over its own PCIe link: no per-call reduction, no collective.
 * Every call below that takes the returned handle acts on the whole group unless it says otherwise.
 * This is what CreateGpuWavefrontRenderer returns when TINSEL_GPUS=N is set (tinsel_plugin.cpp).
 * `devices`: numDevices distinct CUDA ordinals; devices[0] is the head (finish / denoise run there). */
#define TB200_MAX_DEVICES 16
tb200_renderer* tb200_create_multi(const tb200_scene* scene, const int* devices, int numDevices);
int tb200_num_devices(const tb200_renderer* r);

/* The slab rule tb200_init applies to a multi-device renderer, for hosts that run one process per GPU
 * and call tb200_set_slab themselves: member k of n owns pixel rows [*firstRow, *firstRow + *numRows)
 * (contiguous, cut at 4-row tile rows).  tb200_slab_traced_rows: the rows whose samples the owner of
 * [firstRow, firstRow+numRows) traces -- the slab plus the filter's reach (ceil(width)+1 rows,
 * render.cpp:404-407) on either side, clipped to the image. */
void tb200_slab_rows(int height, int member, int numMembers, int* firstRow, int* numRows);
void tb200_slab_traced_rows(int height, int firstRow, int numRows, float filterWidth, int* firstTraced, int* numTraced);

/* The multiplier and shift with which the kernels divide sample indices by a launch's samples per frame and
 * tile index by its 8-pixel tile columns: for every 32-bit n, n / d == (((n * mul) >> 32) + n) >> shift, the
 * product and the sum formed in 64 bits.  d = 0 gives 0, 0. */
void tb200_divisor_magic(unsigned int d, unsigned int* mul, unsigned int* shift);

/* Replaces Renderer::Init (src/render.h:70; semantics of src/render.cu:1070-1075):
 * (re)allocates and zeroes the device accumulator, resets the frame counter. Returns 0 on success. */
int tb200_init(tb200_renderer* r, int width, int height);

/* Replaces Renderer::Render (src/render.h:71; semantics of src/render.cpp:447-524):
 * ePathTrace adds exactly one sample per pixel and leaves output[0..w*h) = running sums
 * (sum w*r, sum w*g, sum w*b, sum w) since Init; eNormals overwrites with normals; eComplexity
 * is a no-op.  `output` is HOST memory, width*height*4 floats.  Synchronous. Returns 0 on success. */
int tb200_render(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options, float* output);

/* Batch form of the same path: adds `spp` samples per pixel (frames k..k+spp-1 of the same
 * per-sample seed sequence as `spp` tb200_render calls) and leaves the sums on the device.
 * If firstRow/numRows restrict the pixel rows whose samples are traced (image-plane sharding
 * across GPUs); splats still land wherever the filter footprint reaches.  Returns 0 on success. */
int tb200_render_device(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options,
                        int spp, int firstRow, int numRows);

/* Image-plane sharding across GPUs: this renderer traces only the 4-pixel-high tile rows t with
 * t % numShards == shard (interleaved for load balance).  Every sample is traced by exactly one
 * shard with the same per-(pixel,frame) seed, so the sum over shards of the accumulators equals
 * the unsharded image up to fp32 summation order.  Default: shard 0 of 1. */
int tb200_set_shard(tb200_renderer* r, int shard, int numShards);

/* external != 0: launch all work of this renderer on the caller's CUDA stream `cudaStream` (a
 * cudaStream_t passed as void*; handle 0 is CUDA's legacy default stream), so that the caller's own
 * events bracket it.  external == 0: back to the renderer's private stream (`cudaStream` ignored).
 * Single-device renderers only. */
int tb200_set_stream(tb200_renderer* r, void* cudaStream, int external);

/* Owner-computes row slab (the multi-GPU building block, also usable one process per GPU): this
 * renderer owns pixel rows [firstRow, firstRow+numRows).  It traces their samples plus those of the
 * rows within the filter's reach outside the slab, splats into the owned rows only, and
 * tb200_render / tb200_read_accumulator / tb200_render_n write only the owned rows of `output`.
 * numRows < 0 removes the slab (whole image).  Not combinable with tb200_set_shard. */
int tb200_set_slab(tb200_renderer* r, int firstRow, int numRows);

/* Page-locks a CALLER-OWNED host buffer (cudaHostRegister, portable across devices) so that the
 * read-backs of tb200_render & co. into it run at PCIe speed, asynchronously, and -- for a
 * multi-device renderer -- from all devices at once.  The library never pins caller memory on its
 * own: the caller owns the buffer's lifetime and must call tb200_unpin_output (or tb200_destroy)
 * BEFORE freeing or reallocating it.  Unpinned buffers work too, through the driver's staged copy.
 * Returns 0 on success. */
int tb200_pin_output(tb200_renderer* r, float* output, size_t bytes);
int tb200_unpin_output(tb200_renderer* r);

/* Multi-device renderers: copies every device's slab into the head device's accumulator (device to
 * device, NVLink), so that tb200_device_accumulator(head) holds the whole image.  tb200_finish does
 * this itself.  No-op for a single device. */
int tb200_gather_device(tb200_renderer* r);

/* Accumulate into caller-owned DEVICE memory (width*height*4 floats, e.g. a torch tensor that is
 * then reduced with NCCL) instead of the renderer's own buffer.  Call after tb200_init; NULL
 * switches back.  The caller zeroes its buffer. */
int tb200_bind_accumulator(tb200_renderer* r, float* deviceAccum);

/* Device pointer of the accumulator (width*height*4 floats) so that callers can reduce it
 * across GPUs (NCCL) without a host round trip.  Valid until the next tb200_init/destroy. */
float* tb200_device_accumulator(tb200_renderer* r);

/* Copies the accumulator to host memory (width*height*4 floats).  Returns 0 on success. */
int tb200_read_accumulator(tb200_renderer* r, float* output);

/* `n` x tb200_render in one call with ONE read-back: adds frames k..k+n-1 (the per-sample seeds of
 * n consecutive Render calls) and leaves the running sums in `output` (HOST, width*height*4
 * floats).  Replaces the `for (i < numSamples) g_renderer->Render(...)` loop of src/main.cpp:242-251
 * (16 calls, 16 read-backs per displayed frame).  ePathTrace only.  Returns 0 on success. */
int tb200_render_n(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options, int n, float* output);

/* The display/finish step that follows the path in src/main.cpp:258-271 and src/png.cpp:329-343,
 * on the device, reading the accumulator where it lies:
 *   filtered[i] = LinearToSrgb(ToneMap(pixels[i] * (exposure / pixels[i].w), limit))
 *                 (util.h:25-42 filmic curve, maths.h:1545-1555; alpha comes out 0 as in the reference)
 *   rgb8[i*3+c] = Quantize(filtered[i][c]*255.0 + Randf + Randf - 0.5f)  with WritePng's own
 *                 sequential Random() dither stream (6 draws per pixel, pixel-major)
 * `filtered` (HOST, width*height*4 floats) and `rgb8` (HOST, width*height*3 bytes) are each
 * optional (NULL = not wanted): a caller that only displays or writes the PNG reads back 3 bytes
 * per pixel instead of 16.  Arithmetic is the reference's expression order with powf from
 * include/tb200_detmath.h.  Returns 0 on success. */
int tb200_finish(tb200_renderer* r, float exposure, float limit, float* filtered, unsigned char* rgb8);

/* NonLocalMeansFilter(g_filtered, g_exposed, width, height, falloff, radius) of src/nlm.cpp:36-73
 * (called from src/main.cpp:273-277 on the finished image when the viewer's denoise toggle is on),
 * on the device, applied to the image the last tb200_finish produced (which stays resident):
 * box means over the clamped (2*radius+1)^2 window (AverageFilter, nlm.cpp:4-34), then per pixel
 * sum in[q]*w / sum w with w = expf(-falloff * |mean[p]-mean[q]|^2) over the same window, summed in
 * the reference's order (columns outer, rows inner).  `out` is HOST memory, width*height*4 floats.
 * Returns 0 on success, -1 if tb200_finish has not run since the last tb200_init. */
int tb200_nlm(tb200_renderer* r, float falloff, int radius, float* out);

/* Per-sample radiance probe used by the parity tests: traces frame `frame` only and writes,
 * for pixel p (row-major), radiance[3p..3p+2] = PathTrace() result and raster[2p..2p+1] =
 * jittered raster position, WITHOUT touching the accumulator.  Host pointers.  0 on success. */
int tb200_trace_frame(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options,
                      int frame, float* radiance, float* raster);

/* ---- batched closest-hit ray query ---------------------------------------------------------
 * Per ray i, exactly Trace(scene, Ray(origin, dir, time)) of src/render.cpp:17-62, bit for bit:
 *   prims[i]       index of the closest primitive with t > 0, or -1 on a miss
 *   hits[i].t      its distance in units of |dir| (dir is used as given, never normalised)
 *   hits[i].normal the shading normal after FaceForward(n, -dir)
 * A miss leaves t = FLT_MAX and the face-forwarded zero normal.  `time` drives the motion-blur
 * interpolation of primitive transforms; `pad` is ignored here (tb200_occluded_rays reads it as
 * tmax, so one array of rays can feed both queries).  Any finite `time`, inside the shutter or not, is exact.  A NaN
 * or infinite time is the one exception: the device keeps a static primitive's transform (a sphere or mesh whose
 * start and end transforms match bit for bit and have no -0 component), where the reference's interpolation gives
 * NaN.  A primitive that moves is exact at any time, and so is a plane, which ignores transforms.
 * `rays`, `hits` and `prims` are DEVICE memory of the renderer's device (a multi-device renderer: its
 * head, devices[0]); `rays` and `hits` 16-byte aligned.  Host or foreign-device pointers, null pointers,
 * numRays < 0 and spans past the end of their allocation are refused before anything is launched.
 * The work runs on the renderer's stream (tb200_set_stream) and the call returns when the results are
 * in place.  Needs no tb200_init; leaves the accumulator, the frame counter, stats.frames,
 * stats.samples and tb200_last_kernel as they are; adds 1 to stats.kernelLaunches and sets stats.gpuMs
 * to the query kernel's time.  numRays == 0 launches nothing.  Returns 0 on success. */
/* `pad`: tmax of the occlusion query (tb200_occluded_rays); the closest-hit query ignores it. */
typedef struct tb200_ray { float origin[3]; float time; float dir[3]; float pad; } tb200_ray;   /* 32 B */
typedef struct tb200_hit { float t; float normal[3]; } tb200_hit;                               /* 16 B */
int tb200_trace_rays(tb200_renderer* r, const tb200_ray* rays, tb200_hit* hits, int32_t* prims, int64_t numRays);

/* ---- batched occlusion (any-hit) ray query --------------------------------------------------
 * Per ray i, exactly: occluded[i] = 1 iff Trace(scene, Ray(origin, dir, time)) of src/render.cpp:17-62
 * returns a primitive (prims[i] >= 0 from tb200_trace_rays) and its t < tmax, where tmax is the
 * ray's `pad` field; else 0.  t is in units of |dir|, so dir = target - origin with tmax = 1 asks
 * whether anything lies between two points.  tmax <= 0 or NaN gives 0, tmax = +inf "hits anything";
 * a miss (t = FLT_MAX) is never occluded.  The walk stops at the first blocker and computes no normal.
 * Any finite `time`, inside the shutter or not, is exact.  A NaN or infinite time is the one exception:
 * the device keeps a static primitive's transform (a sphere or mesh whose start and end transforms match bit for bit
 * and have no -0 component), where the reference's interpolation gives NaN.  A primitive that moves is exact at any
 * time, and so is a plane, which ignores transforms.
 * `rays` (16-byte aligned) and `occluded` (numRays bytes) are DEVICE memory of the renderer's
 * device, with the refusals, stream, synchronisation and side effects of tb200_trace_rays: it adds
 * 1 to stats.kernelLaunches, sets stats.gpuMs to its kernel's time, and touches nothing else.
 * numRays == 0 launches nothing.  Returns 0 on success. */
int tb200_occluded_rays(tb200_renderer* r, const tb200_ray* rays, uint8_t* occluded, int64_t numRays);

/* ---- batched closest-hit ray query with the hit triangle -----------------------------------
 * hits[i] and prims[i] are bit for bit what tb200_trace_rays writes for the same ray.  When prims[i] is
 * a mesh primitive, tris[i] describes the triangle whose hit Trace kept:
 *   tri      its index in that primitive's mesh: its vertices are indices[3*tri .. 3*tri+2] of the
 *            tb200_mesh the scene was created from
 *   u, v, w  IntersectRayTriTwoSided's barycentric weights (intersection.h:117-145): v weights
 *            indices[3*tri+1], w weights indices[3*tri+2], and u = 1 - v - w as the reference rounds it
 * so u*N[i0] + v*N[i1] + w*N[i2] is the smooth normal before its flip, transform and normalisation
 * (intersection.h:994-1013).  The weights are in the mesh's own space: an instance transform, motion
 * included, does not change them.  Ties are Trace's: the first primitive in the reference's order wins,
 * and inside a mesh the first triangle in walk order.  A sphere hit, a plane hit or a miss gives
 * tri = -1 and u = v = w = 0.  tris (numRays records, 16-byte aligned) is DEVICE memory like the other
 * arrays; the refusals, stream, synchronisation and side effects are tb200_trace_rays': it adds 1 to
 * stats.kernelLaunches, sets stats.gpuMs to its kernel's time, and touches nothing else.  numRays == 0
 * launches nothing.  `pad` is ignored.  Any finite `time`, inside the shutter or not, is exact.  A NaN or infinite
 * time is the one exception: the device keeps a static primitive's transform (a sphere or mesh whose start and end
 * transforms match bit for bit and have no -0 component), where the reference's interpolation gives NaN.  A primitive
 * that moves is exact at any time, and so is a plane, which ignores transforms.  Returns 0 on success. */
typedef struct tb200_tri_hit { int32_t tri; float u, v, w; } tb200_tri_hit;   /* 16 B */
int tb200_trace_rays_tri(tb200_renderer* r, const tb200_ray* rays, tb200_hit* hits, int32_t* prims,
                         tb200_tri_hit* tris, int64_t numRays);

/* ---- batched BSDF queries --------------------------------------------------------------------
 * The material half of a bounce, for a caller's batch: per query i, the Disney BSDF of src/disney.h
 * bit for bit (a NaN may have another payload), with the material the path tracer shades primitive
 * `prim` with (a mesh primitive has one material).  `n`, `v` (towards the viewer) and `l` (towards the
 * light) are used as given, never normalised, as are the etas, which may take any value.  PathTrace's
 * convention (src/render.cpp:259-269): a ray in air hitting a surface has etaI = 1, etaO = the
 * material's ior (tb200_material eta, or Material::GetIndexOfRefraction's value from `specular` when
 * eta == 0); a ray inside a medium of ior eta has etaI = eta, etaO = 1.
 *   tb200_bsdf_eval:   out[i].f = BSDFEval(mat, etaI, etaO, n, v, l), out[i].pdf = BSDFPdf(same).
 *   tb200_bsdf_sample: one step of PathTrace (src/render.cpp:327-341): BSDFSample with the basis
 *                      BasisFromVector(n) and Random(seeds[i]) (src/maths.h:1040-1044) gives l, pdf
 *                      and type; then f = BSDFEval(l) when pdf > 0, else f = 0.  q[i].l is ignored.
 * A prim outside [0, numPrimitives) gives f = 0, pdf = 0 and, when sampling, l = 0, type = -1, so the
 * prims of tb200_trace_rays can be passed straight through on misses (-1).
 * `q`, `seeds` and `out` are DEVICE memory of the renderer's device (a multi-device renderer: its head);
 * `q` and `out` 16-byte aligned, `seeds` 4-byte aligned.  The refusals, stream, synchronisation and side
 * effects are tb200_trace_rays': null pointers, n < 0, host or foreign-device memory and spans past the
 * end of their allocation are refused before any launch; needs no tb200_init; adds 1 to
 * stats.kernelLaunches, sets stats.gpuMs to its kernel's time, and touches nothing else.  n == 0
 * launches nothing.  Returns 0 on success. */
typedef struct tb200_bsdf_query {   /* 48 B */
    float n[3];
    int32_t prim;
    float v[3];
    float etaI;
    float l[3];
    float etaO;
} tb200_bsdf_query;
typedef struct tb200_bsdf_value { float f[3]; float pdf; } tb200_bsdf_value;                              /* 16 B */
typedef struct tb200_bsdf_sampled { float l[3]; float pdf; float f[3]; int32_t type; } tb200_bsdf_sampled;   /* 32 B */
/* tb200_bsdf_sampled.type: BSDFType, src/disney.h:27-32 (-1 for a prim outside the scene) */
enum { TB200_BSDF_REFLECTED = 0, TB200_BSDF_TRANSMITTED = 1, TB200_BSDF_SPECULAR = 2 };
int tb200_bsdf_eval(tb200_renderer* r, const tb200_bsdf_query* q, tb200_bsdf_value* out, int64_t n);
int tb200_bsdf_sample(tb200_renderer* r, const tb200_bsdf_query* q, const uint32_t* seeds, tb200_bsdf_sampled* out,
                      int64_t n);

/* ---- batched camera samples and film splats --------------------------------------------------
 * The two ends of a path, for a caller's batch, exactly as the renderer runs them, so that a caller can trace the
 * image's own samples (depth, normal or primitive maps aligned with the image; an integrator of its own) and put
 * its own radiance into a film with the image's filter (custom AOVs; tb200_finish and tb200_nlm of its results).
 *   tb200_camera_rays: per record i, the camera sample the renderer traces for pixel p = samples[i].pixel of a
 *     W x H image (px = p % W, py = p / W) in frame samples[i].frame (any int32, read as its uint32 bits):
 *     Random(tb200_sample_seed(p, frame)), then the draws x, y, t (src/render.cpp:476-482), time =
 *     Lerp(shutterStart, shutterEnd, t) and GenerateRay(px + x, py + y) of the camera (src/util.h:45-83), bit for
 *     bit.  rays[i] = {origin, time, dir, pad = +inf} (+inf: tb200_occluded_rays reads the same record as "anything
 *     in front of the camera"); raster[2i..2i+1] = px + x, py + y, where the renderer splats that sample.  A pixel
 *     outside [0, W*H) gives an all-zero ray (a miss for tb200_trace_rays) and a NaN raster (skipped by
 *     tb200_splat).  Only options->width and options->height are read.
 *   tb200_splat: per sample i, AddSample(raster[2i..2i+1], radiance[3i..3i+2]) (src/render.cpp:401-445) into
 *     `accum`, W*H float4 running sums (sum w*rgb, sum w), added to what is there (the caller zeroes), with the
 *     options' filter type, width, falloff, offset and clamp, over every row [0, H) (slab and shard settings do
 *     not apply).  Filter options are refused as by the render calls.  A raster coordinate that is NaN or 2^30 or
 *     more in magnitude is skipped (AddSample's int conversion is undefined there); every other sample is splatted
 *     as the renderer splats it, including one outside the image whose footprint reaches in, and a non-finite
 *     radiance, which poisons its footprint as in the reference.  The sums are formed in the order the reductions
 *     reach memory, as the renderer's are.  accum = tb200_device_accumulator(r) puts the samples into the
 *     renderer's own film, for tb200_finish, tb200_nlm and tb200_read_accumulator.
 * All arrays are DEVICE memory of the renderer's device (a multi-device renderer: its head); alignment: samples 8
 * bytes, rays 16, raster 8, radiance 4, accum 16; accum spans W*H*16 bytes whatever n is.  Refused before any
 * launch, besides what tb200_trace_rays refuses (null pointers, n < 0, host or foreign-device memory, spans past
 * the end of their allocation): null options or camera, width or height <= 0 and W*H > INT32_MAX.  The stream,
 * synchronisation and side effects are tb200_trace_rays': needs no tb200_init; adds 1 to stats.kernelLaunches,
 * sets stats.gpuMs to its kernel's time, and changes nothing else but `accum`.  n == 0 launches nothing.  Returns 0
 * on success. */
typedef struct tb200_camera_sample { int32_t pixel; int32_t frame; } tb200_camera_sample;   /* 8 B */
int tb200_camera_rays(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options,
                      const tb200_camera_sample* samples, tb200_ray* rays, float* raster, int64_t n);
int tb200_splat(tb200_renderer* r, const tb200_options* options, const float* raster, const float* radiance,
                float* accum, int64_t n);

/* ---- batched next-event estimation and sky queries -------------------------------------------
 * The two stages of PathTrace (src/render.cpp:230-388) the queries above leave out, for a caller's batch:
 *   tb200_sample_lights: per query i, radiance[3i..3i+2] = SampleLights(scene, prims[prim], etaI, etaO, p, n, wo,
 *     time, Random(seeds[i])) (src/render.cpp:103-227), bit for bit (a NaN may have another payload): the probe
 *     sample and its shadow ray when the sky has a probe, then for every primitive with lightSamples > 0, in scene
 *     order, its samples, each with a full closest-hit Trace shadow ray at `time`, the |t - dist| <= 1e-2
 *     acceptance, the light-normal test and the balance-heuristic MIS, weighted by the emission of whatever the
 *     shadow ray hit.  That is the `sum` PathTrace multiplies by the path throughput; PathTrace calls it at every
 *     hit, a hit on a light included.  The record follows PathTrace's convention: p the hit point, n the shading
 *     normal as tb200_trace_rays returns it (face-forwarded), wo = -dir of the incoming ray, and the etas of
 *     tb200_bsdf_eval; all are used as given, never normalised, and the etas may take any value.  The BSDF is the
 *     material the path tracer shades `prim` with.  A prim outside [0, numPrimitives) gives zeros and traces
 *     nothing, so the prims of tb200_trace_rays can be passed straight through on misses (-1).  The three floats
 *     per query are the layout tb200_splat reads its radiance in.  Any finite `time`, inside the shutter or not, is
 *     exact.  A NaN or infinite time is the one exception: the device keeps a static primitive's transform (a sphere
 *     or mesh whose start and end transforms match bit for bit and have no -0 component), where the reference's
 *     interpolation gives NaN.  A primitive that moves is exact at any time, and so is a plane, which ignores
 *     transforms.
 *   tb200_sky_eval: per ray i (only rays[i].dir is read, so the records of tb200_trace_rays and tb200_camera_rays can
 *     be passed as they are), out[4i..4i+2] = Sky::Eval(dir) (src/scene.h:168-178) and out[4i+3] = ProbePdf(dir)
 *     (src/probe.h:136-160) when the sky has a probe, else 0; bit for bit.  The miss branch's MIS weight
 *     (src/render.cpp:365-384) depends on path state and stays with the caller.
 * All arrays are DEVICE memory of the renderer's device (a multi-device renderer: its head); alignment: q and rays
 * 16 bytes, seeds 4, radiance 4, out 16.  The refusals, stream, synchronisation and side effects are
 * tb200_trace_rays': null pointers, n < 0, host or foreign-device memory and spans past the end of their
 * allocation are refused before any launch; needs no tb200_init; adds 1 to stats.kernelLaunches, sets stats.gpuMs
 * to its kernel's time, and touches nothing else.  n == 0 launches nothing.  Returns 0 on success. */
typedef struct tb200_light_query {   /* 64 B */
    float p[3];  float time;     /* surface point; ray time (motion blur of the lights and the shadow rays) */
    float n[3];  int32_t prim;   /* shading normal as trace_rays returns it (face-forwarded); surface primitive */
    float wo[3]; float etaI;     /* towards the viewer (-dir of the incoming ray) */
    float etaO;  float pad[3];
} tb200_light_query;
int tb200_sample_lights(tb200_renderer* r, const tb200_light_query* q, const uint32_t* seeds, float* radiance,
                        int64_t n);
int tb200_sky_eval(tb200_renderer* r, const tb200_ray* rays, float* out, int64_t n);

/* ---- batched emitter and probe samples -------------------------------------------------------
 * The two draws SampleLights makes its light samples from, for a caller's batch, so that a caller can build a
 * light estimator of its own (one light picked by power, resampled candidates, the power heuristic, the start
 * points of light paths):
 *   tb200_sample_emitters: per query i, PrimitiveSample(primitives[prim], time, pos, normal, Random(seeds[i]))
 *     (src/intersection.h:855-904), bit for bit (a NaN may have another payload).  A sphere draws 2 numbers; a
 *     mesh draws 4: the triangle from the mesh's area CDF, UniformSampleTriangle's two, at the instance transform
 *     of `time`.  Only the primitives SampleLights samples are sampled: those with lightSamples > 0 (tb200_create
 *     refuses a mesh light without a CDF).  Any other primitive -- not a light, a plane, or a prim outside
 *     [0, numPrimitives), so that the prims of tb200_trace_rays can be passed straight through on misses (-1) --
 *     gives pos = normal = 0.  A degenerate triangle can give a zero normal too, so a zero normal does not mean
 *     "not a light".  Any finite `time`, inside the shutter or not, is exact.  A NaN or infinite time is the one
 *     exception: the device keeps a static primitive's transform (a sphere or mesh whose start and end transforms
 *     match bit for bit and have no -0 component), where the reference's interpolation gives NaN.  A primitive that
 *     moves is exact at any time, and so is a plane, which ignores transforms.
 *     The area pdf of a sample is 1 / PrimitiveArea (tinsel_b200.primitive_areas gives it as the renderer computes
 *     it: 4 pi r^2 of the unscaled radius for a sphere, the mesh's area times the end transform's scale for a mesh).
 *   tb200_sample_probe: per seed i, ProbeSample(probe, dir, color, pdf, Random(seeds[i])) (src/probe.h:205-236),
 *     bit for bit, including pdf = 0 where sinTheta == 0; all zeros when the sky has no probe.  The solid-angle pdf
 *     of any direction, for MIS against other strategies, is ProbePdf, which tb200_sky_eval returns.
 * The pads are written as 0.  All arrays are DEVICE memory of the renderer's device (a multi-device renderer: its
 * head); alignment: q 8 bytes, seeds 4, out 16.  The refusals, stream, synchronisation and side effects are
 * tb200_trace_rays': null pointers, n < 0, host or foreign-device memory and spans past the end of their
 * allocation are refused before any launch; needs no tb200_init; adds 1 to stats.kernelLaunches, sets stats.gpuMs
 * to its kernel's time, and touches nothing else.  n == 0 launches nothing.  Returns 0 on success. */
typedef struct tb200_emitter_query { int32_t prim; float time; } tb200_emitter_query;                      /* 8 B */
typedef struct tb200_emitter_sampled { float pos[3]; float pad0; float normal[3]; float pad1; } tb200_emitter_sampled;
                                                                                                            /* 32 B */
typedef struct tb200_probe_sampled { float dir[3]; float pdf; float color[3]; float pad; } tb200_probe_sampled;
                                                                                                            /* 32 B */
int tb200_sample_emitters(tb200_renderer* r, const tb200_emitter_query* q, const uint32_t* seeds,
                          tb200_emitter_sampled* out, int64_t n);
int tb200_sample_probe(tb200_renderer* r, const uint32_t* seeds, tb200_probe_sampled* out, int64_t n);

/* ---- the probe's sampling tables, and a new sky for a live renderer ---------------------------
 *   tb200_probe_tables: Probe::BuildCDF (src/probe.h:31-79) on the device, bit for bit (a NaN may have another
 *     payload), for the width x height RGBA texels at `probe` (the layout of tb200_sky::probeData; alpha is
 *     ignored): per texel the weight (r*0.3f + g*0.6f) + b*0.1f; per row its sequential fp32 running sum, pdfX and
 *     cdfX = weight and running sum times the IEEE 1.0f / row total (a black row gives NaN: 0 * inf); pdfY and cdfY
 *     = the row total and the rows' sequential running sum, each divided by the sum of all rows.  Writes
 *     width*height floats to pdfX and cdfX and height floats to pdfY and cdfY, the tb200_sky tables of that probe.
 *     Non-finite, negative and subnormal texels go through the arithmetic as they are.  All five arrays are DEVICE
 *     memory of the renderer's device (a multi-device renderer: its head); `probe` 16-byte aligned, the tables 4.
 *     Refused before any launch: width or height <= 0, width*height + 1 > INT32_MAX (the sampler indexes rows
 *     with int), and, as by tb200_trace_rays, null pointers, host or foreign-device memory and spans past the end of
 *     their allocation.  The stream, synchronisation and side effects are tb200_trace_rays': needs no tb200_init;
 *     adds 3 to stats.kernelLaunches, sets stats.gpuMs to the kernels' time, and touches nothing else.  It does not
 *     read or change the renderer's sky.  Returns 0 on success.
 *   tb200_set_sky: replaces the renderer's sky -- its gradient colours and its probe -- and leaves it as
 *     tb200_create would have built it from the same scene with this sky: every render call and every query after
 *     it (tb200_sky_eval, tb200_sample_probe, tb200_sample_lights, ...) sees the new sky, the probe's shadow ray per
 *     hit is counted in or out, and the wavefront kernel is chosen again for the scene with this sky under the knobs
 *     read at create time (tb200_last_kernel reports the new choice at the next render).  probe == NULL gives the
 *     gradient sky, and then width and height must be 0.  Otherwise `probe` is width x height RGBA texels as for
 *     tb200_probe_tables, in HOST memory or in DEVICE memory of the renderer's device (its head; 16-byte aligned,
 *     spanning width*height*16 bytes); a pointer to another device's memory is refused.  The renderer copies the
 *     texels (the caller's buffer is free once the call returns) and builds the four tables with tb200_probe_tables'
 *     kernels.  Colours and texels are taken as given, non-finite ones included.  A multi-device renderer sets the
 *     same sky on every device (a device probe is copied from the head to each).  Atomic: the new probe is built in
 *     full before anything changes, and after a refusal or a CUDA failure (-1, tb200_last_error says why) the
 *     renderer renders exactly as before; on success the previous probe's memory is freed.  The accumulator, the
 *     frame counter, stats.frames, stats.samples and tb200_last_kernel are left as they are: an image accumulated so
 *     far keeps its samples of the old sky, and restarting it (tb200_init) is the caller's choice, as it is after a
 *     camera change.  Adds the bytes copied from the host to stats.h2dBytes and the table build's launches to
 *     stats.kernelLaunches, and sets stats.gpuMs to the build's time (0 for the gradient sky).  Runs on the
 *     renderer's stream; returns when the new sky is in place.  Needs no tb200_init.  Returns 0 on success. */
int tb200_probe_tables(tb200_renderer* r, const float* probe, int width, int height, float* pdfX, float* cdfX,
                       float* pdfY, float* cdfY);
int tb200_set_sky(tb200_renderer* r, const float horizon[3], const float zenith[3], const float* probe, int width,
                  int height);

/* Sets the frame counter (frame k seeds sample k of every pixel). */
void tb200_set_frame(tb200_renderer* r, int frame);

void tb200_get_stats(tb200_renderer* r, tb200_stats* out);

/* Name of the path-tracing kernel the renderer's last launch ran, one per kernel: "wf2_lq.specialized" or
 * "wf2_lq.generic" (lane-owned wavefront with or without the scene-feature code), "wf2_smem.hard",
 * "wf2_smem.split", "wf2_smem.generic", "wf2_l2.split", "wf2_l2.generic" (ring-queue wavefront: layout before the
 * dot, scheduling mode after it), "k_mega"; "" before the first launch.  A static string.  Multi-device renderers:
 * the head's. */
const char* tb200_last_kernel(tb200_renderer* r);

/* The counters of ONE member of a multi-device renderer (0 = the head) and the pixel rows it owns: how the
 * work of the last call was spread (gpuMs per device).  Returns 0 on success. */
int tb200_get_member_stats(tb200_renderer* r, int member, tb200_stats* out, int* firstRow, int* numRows);

/* Deletes the renderer and all its device memory (reference: `delete g_renderer`, src/main.cpp:323). */
void tb200_destroy(tb200_renderer* r);

/* Sticky, thread-local description of the last failure ("" if none). */
const char* tb200_last_error(void);

/* The per-(pixel,frame) seed handed to Random(seed) (src/maths.h:1040-1044).  The reference
 * CPU renderer has one sequential stream (src/render.cpp:399); a parallel renderer needs a
 * per-sample rule, and this is it -- shared with the oracle so streams match draw for draw. */
uint32_t tb200_sample_seed(uint32_t pixelIndex, uint32_t frame);

/* ---- scene snapshots (".tsnap") ----------------------------------------------------------- */
/* A flat little-endian dump of everything the renderer consumes (tb200_scene + camera +
 * options as the reference loader produced them).  Written in this container by
 * oracle/ref_driver (which links the reference's own loader/BVH builder); read anywhere. */
typedef struct tb200_snapshot tb200_snapshot;

tb200_snapshot* tb200_snapshot_load(const char* path);
const tb200_scene* tb200_snapshot_scene(const tb200_snapshot* s);
const tb200_camera* tb200_snapshot_camera(const tb200_snapshot* s);
const tb200_options* tb200_snapshot_options(const tb200_snapshot* s);
int tb200_snapshot_save(const char* path, const tb200_scene* scene, const tb200_camera* camera,
                        const tb200_options* options);
void tb200_snapshot_free(tb200_snapshot* s);

/* ---- tinsel binary meshes (".bin") --------------------------------------------------------------
 * The reference's own mesh cache (src/mesh.cpp:809-880, ImportMeshFromBin / ExportMeshToBin, written
 * by `tinsel -convert`, src/main.cpp:151-169): int numVertices, numIndices, numNodes; Vec3
 * positions[numVertices]; Vec3 normals[numVertices]; int indices[numIndices]; BVHNode
 * nodes[numNodes]; float area; float cdf[numIndices/3].  It holds exactly what a tb200_mesh needs --
 * geometry, the built SAH BVH and the light-sampling CDF -- so a host can assemble a tb200_scene from
 * cached meshes without the OBJ/PLY importers and the BVH builder (3.5 s for ajax, SURVEY 8f).
 * The loaded object owns the arrays the returned tb200_mesh points into; files written by
 * tb200_mesh_bin_save are byte-identical to the reference writer's. */
typedef struct tb200_mesh_file tb200_mesh_file;
tb200_mesh_file* tb200_mesh_bin_load(const char* path);            /* NULL on failure (tb200_last_error) */
const tb200_mesh* tb200_mesh_bin_mesh(const tb200_mesh_file* f);
int tb200_mesh_bin_save(const char* path, const tb200_mesh* mesh);  /* 0 on success */
void tb200_mesh_bin_free(tb200_mesh_file* f);

/* ---- scene cache (".tcache") -------------------------------------------------------------------------
 * Everything tb200_create derives from a tb200_scene -- primitive records with their hoisted constants,
 * child-pair BVH records in breadth-first order, pre-gathered triangles and vertex normals, the flat scene
 * program, and the probe WITH its four sampling tables (Probe::BuildCDF, src/probe.h:31-79) -- stored in
 * exactly the layouts the device holds, so that tb200_create_cached goes from the file to device memory
 * array by array: no .tin/OBJ loader, no BVH builder, no re-packing, no per-triangle gather, no BuildCDF.
 * It plays the role the reference gives its `.bin` mesh cache (src/mesh.cpp:809-880, `tinsel -convert`,
 * src/main.cpp:151-169), for the whole scene.  The file is this build's device layout, not an interchange
 * format: a file written by another build is refused (layout stamp) and the caller uses tb200_create.
 * tb200_scene_cache_save needs no GPU.  A renderer from a cache is bit-identical to one from the scene. */
int tb200_scene_cache_save(const tb200_scene* scene, const char* path);   /* 0 on success */
tb200_renderer* tb200_create_cached(const char* path, int device);         /* NULL on failure (tb200_last_error) */

/* ---- mesh BVH construction on the GPU ---------------------------------------------------------------
 * Replaces Mesh::RebuildBVH + BVHBuilder::Build (src/mesh.cpp:314-338, src/bvh.h:30-263: one Bounds per
 * triangle, recursive full-sweep SAH on one host core, 1.33 s for ajax) for triangle meshes: a PLOC
 * (parallel locally-ordered clustering) build on the device, milliseconds for half a million triangles.
 * Writes 2*numTriangles-1 nodes in the reference's own BVHNode format (root at 0, one triangle per leaf,
 * leaf.left = triangle index, node boxes = exact unions of triangle boxes), usable as tb200_mesh::nodes,
 * by the reference's IntersectRayMesh, and in the .bin mesh cache.  `positions`, `indices`, `outNodes`
 * are HOST arrays.  The tree differs from the reference builder's (an equally valid input to the same
 * traversal).  Returns 0 on success; tb200_bvh_build_error() describes a failure.  A tree with more
 * than TB200_MAX_BVH_LEVELS levels of interior nodes is a failure: outNodes is then zeroed. */
typedef struct tb200_bvh_build_info {
    int32_t numNodes;          /* 2*numTriangles - 1 */
    int32_t rounds;            /* clustering rounds */
    uint64_t kernelLaunches;   /* this library's kernels (the radix sort and prefix sums are CUB calls on top) */
    double buildMs;            /* device time from the triangle boxes to the finished node array (CUDA events) */
} tb200_bvh_build_info;
int tb200_bvh_build(const float* positions, int numVertices, const int32_t* indices, int numIndices,
                    tb200_bvh_node* outNodes, int device, tb200_bvh_build_info* info);
const char* tb200_bvh_build_error(void);

#ifdef __cplusplus
}
#endif
#endif /* TINSEL_B200_H */
