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

/* Options + Filter (src/render.h:13-63); same field order as the reference. */
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

/* Sets the frame counter (frame k seeds sample k of every pixel). */
void tb200_set_frame(tb200_renderer* r, int frame);

void tb200_get_stats(tb200_renderer* r, tb200_stats* out);

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
