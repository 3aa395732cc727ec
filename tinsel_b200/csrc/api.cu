// api.cu -- host side of the C ABI (include/tinsel_b200.h): scene translation into the GPU
// layout, accumulator management, frame sequencing, host read-back.
//
// Host arithmetic here restates reference *host-side* or *per-primitive-constant* expressions
// (cited inline) and is compiled without contraction (-Xcompiler -ffp-contract=off, no fast-math)
// so that it matches the reference's x86-64 build.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "tb_kernels.cuh"

const char* tb200_snapshot_error();   // snapshot.cpp
unsigned long long tb200_snapshot_error_stamp();
unsigned long long tb200_error_tick();

namespace {

thread_local std::string g_error;
thread_local unsigned long long g_errorStamp = 0;

bool set_error(const std::string& what)
{
    g_error = what;
    g_errorStamp = tb200_error_tick();
    fprintf(stderr, "[tinsel_b200] %s\n", what.c_str());
    return false;
}

#define TB_CUDA(call)                                                                                   \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess) {                                                                        \
            set_error(std::string(#call) + ": " + cudaGetErrorString(e_));                              \
            return false;                                                                               \
        }                                                                                               \
    } while (0)

// Owners of one cudaMalloc'd (DevPtr) or cudaHostAlloc'd (HostPtr) allocation.  Moving an owner keeps the address.
struct CudaFree {
    void operator()(void* p) const { cudaFree(p); }
};
struct CudaFreeHost {
    void operator()(void* p) const { cudaFreeHost(p); }
};
template <typename T>
using DevPtr = std::unique_ptr<T, CudaFree>;
template <typename T>
using HostPtr = std::unique_ptr<T, CudaFreeHost>;

// *out = a new allocation of n elements.  What *out held is freed first, so that a resize never holds both.
template <typename T>
cudaError_t dev_alloc(DevPtr<T>* out, size_t n)
{
    out->reset();
    T* p = nullptr;
    const cudaError_t e = cudaMalloc((void**)&p, n * sizeof(T));
    if (e == cudaSuccess) out->reset(p);
    return e;
}

V3 hv3(const float* f) { return v3(f[0], f[1], f[2]); }

Xf to_xf(const tb200_transform& t)
{
    Xf x;
    x.p = hv3(t.p);
    x.r = q4(t.r[0], t.r[1], t.r[2], t.r[3]);
    x.s = t.s;
    return x;
}

// BVHNode[] (bvh.h:9-19) -> BvhPair[]; see tb_scene.cuh.  Returns the root reference.  Pairs are laid out
// in breadth-first order from the root, so that the first K records are the top of the tree: the treelet
// (DScene::treelet) stages exactly that prefix in shared memory with bulk copies, and the upper levels
// share cache lines for everybody else.  Record indices are
// private to this layout; topology, child order and therefore visit order are the reference's.
// *depth (optional) receives the number of levels of interior nodes.
uint32_t build_pairs(const tb200_bvh_node* nodes, int numNodes, std::vector<BvhPair>* out, int* depth = nullptr)
{
    out->clear();
    if (depth) *depth = 0;
    if (numNodes <= 0) return TB_LEAF;   // never traversed: callers skip empty trees
    if (nodes[0].right_leaf >> 31) return TB_LEAF | nodes[0].left;
    std::vector<uint32_t> pairIndex(numNodes, 0xffffffffu);
    std::vector<uint32_t> order;   // interior nodes in breadth-first order
    order.reserve(numNodes / 2 + 1);
    pairIndex[0] = 0;
    order.push_back(0);
    size_t levelEnd = 1;
    int levels = 1;
    for (size_t k = 0; k < order.size(); ++k) {
        if (k == levelEnd) {
            levelEnd = order.size();
            levels += 1;
        }
        const tb200_bvh_node& n = nodes[order[k]];
        const uint32_t kids[2] = {n.left, n.right_leaf & 0x7fffffffu};
        for (uint32_t c : kids) {
            if ((nodes[c].right_leaf >> 31) || pairIndex[c] != 0xffffffffu) continue;   // leaf, or already placed (malformed input)
            pairIndex[c] = (uint32_t)order.size();
            order.push_back(c);
        }
    }
    if (depth) *depth = levels;
    out->resize(order.size());
    auto ref_of = [&](uint32_t idx) -> uint32_t {
        const tb200_bvh_node& n = nodes[idx];
        return (n.right_leaf >> 31) ? (TB_LEAF | n.left) : pairIndex[idx];
    };
    for (size_t k = 0; k < order.size(); ++k) {
        const tb200_bvh_node& n = nodes[order[k]];
        const uint32_t li = n.left, ri = n.right_leaf & 0x7fffffffu;
        const tb200_bvh_node& L = nodes[li];
        const tb200_bvh_node& R = nodes[ri];
        BvhPair p;
        p.a = make_float4(L.lower[0], L.lower[1], L.lower[2], L.upper[0]);
        p.b = make_float4(L.upper[1], L.upper[2], R.lower[0], R.lower[1]);
        p.c = make_float4(R.lower[2], R.upper[0], R.upper[1], R.upper[2]);
        p.left = ref_of(li);
        p.right = ref_of(ri);
        p.pad0 = p.pad1 = 0;
        (*out)[k] = p;
    }
    return ref_of(0);
}

// Flat scene program for trace_closest() (tb_scene.cuh).  Walks the scene BVH once; infinite
// boxes (planes' +-1e8 bounds and every ancestor of one) are transparent, finite interior boxes get
// a bit in the per-ray mask, leaves become LEAF / LEAFBOX / PLANE ops guarded by the bit of their
// nearest finite ancestor.  Built only for scenes of at most 16 primitives.
void build_program(const tb200_scene* sc, std::vector<ProgOp>* out)
{
    out->clear();
    const tb200_bvh_node* nodes = sc->bvhNodes;
    if (sc->numBvhNodes <= 0 || sc->numPrimitives > 16) return;
    struct Item { uint32_t node; int guard; bool isRoot; };
    std::vector<Item> todo;
    todo.push_back({0u, TB_BIT_ALWAYS, true});
    int nextBit = 0;
    while (!todo.empty()) {
        const Item it = todo.back();
        todo.pop_back();
        const tb200_bvh_node& n = nodes[it.node];
        const bool leaf = (n.right_leaf >> 31) != 0;
        bool infinite = true;
        for (int k = 0; k < 3; ++k) infinite = infinite && n.lower[k] <= -5.0e7f && n.upper[k] >= 5.0e7f;
        if (it.isRoot) infinite = true;   // the root's own box is never tested (intersection.h:759-763)
        ProgOp op;
        memset(&op, 0, sizeof(op));
        op.a[0] = n.lower[0]; op.a[1] = n.lower[1]; op.a[2] = n.lower[2]; op.a[3] = n.upper[0];
        op.b[0] = n.upper[1]; op.b[1] = n.upper[2];
        if (leaf) {
            const tb200_primitive& p = sc->primitives[n.left];
            int kind = infinite ? TB_OP_LEAF : TB_OP_LEAFBOX;
            if (infinite && p.type == TB200_PLANE) {
                kind = TB_OP_PLANE;
                memcpy(op.a, p.plane, 16);
            }
            op.kindPrim = kind | (int(n.left) << 8);
            op.bits = it.guard;
            out->push_back(op);
        } else {
            int guard = it.guard;
            if (!infinite) {
                if (nextBit >= 31) { out->clear(); return; }
                op.kindPrim = TB_OP_BOX;
                op.bits = it.guard | (nextBit << 8);
                out->push_back(op);
                guard = nextBit++;
            }
            todo.push_back({n.right_leaf & 0x7fffffffu, guard, false});
            todo.push_back({n.left, guard, false});
        }
    }
    if (out->size() > 32) out->clear();
}

// CameraSampler constructor, util.h:49-71, with Mat44(Transform) (maths.h:841-849), Mat33(Quat)
// (maths.h:658-667) and MatrixMultiply<4,4,4> (maths.h:86-101: t = 0; t += a*b for k = 0..3).
struct M44 {
    float c[4][4];   // column major: c[col][row]
};

M44 mat_mul(const M44& a, const M44& b)
{
    M44 r;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float t = 0.0f;
            for (int k = 0; k < 4; ++k) t += a.c[k][i] * b.c[j][k];
            r.c[j][i] = t;
        }
    return r;
}

M44 mat_rows(float m11, float m12, float m13, float m14, float m21, float m22, float m23, float m24, float m31, float m32,
             float m33, float m34, float m41, float m42, float m43, float m44)
{
    M44 m;
    m.c[0][0] = m11; m.c[0][1] = m21; m.c[0][2] = m31; m.c[0][3] = m41;
    m.c[1][0] = m12; m.c[1][1] = m22; m.c[1][2] = m32; m.c[1][3] = m42;
    m.c[2][0] = m13; m.c[2][1] = m23; m.c[2][2] = m33; m.c[2][3] = m43;
    m.c[3][0] = m14; m.c[3][1] = m24; m.c[3][2] = m34; m.c[3][3] = m44;
    return m;
}

void camera_setup(const tb200_camera& cam, int width, int height, DCamera* out)
{
    Xf t;
    t.p = hv3(cam.position);
    t.r = q4(cam.rotation[0], cam.rotation[1], cam.rotation[2], cam.rotation[3]);
    t.s = 1.0f;   // Transform(camera.position, camera.rotation), render.cpp:450-452

    M44 c2w;
    const V3 c0 = rotate(t.r, v3(1.0f, 0.0f, 0.0f)) * t.s;
    const V3 c1 = rotate(t.r, v3(0.0f, 1.0f, 0.0f)) * t.s;
    const V3 c2 = rotate(t.r, v3(0.0f, 0.0f, 1.0f)) * t.s;
    const V3 c3 = t.p * t.s;
    c2w.c[0][0] = c0.x; c2w.c[0][1] = c0.y; c2w.c[0][2] = c0.z; c2w.c[0][3] = 0.0f;
    c2w.c[1][0] = c1.x; c2w.c[1][1] = c1.y; c2w.c[1][2] = c1.z; c2w.c[1][3] = 0.0f;
    c2w.c[2][0] = c2.x; c2w.c[2][1] = c2.y; c2w.c[2][2] = c2.z; c2w.c[2][3] = 0.0f;
    c2w.c[3][0] = c3.x; c2w.c[3][1] = c3.y; c2w.c[3][2] = c3.z; c2w.c[3][3] = 1.0f;

    const M44 rasterToScreen = mat_rows(2.0f / width, 0.0f, 0.0f, -1.0f,
                                        0.0f, -2.0f / height, 0.0f, 1.0f,
                                        0.0f, 0.0f, 1.0f, 1.0f,
                                        0.0f, 0.0f, 0.0f, 1.0f);
    const float f = tanf(cam.fov * 0.5f);
    const float aspect = float(width) / height;
    const M44 screenToCamera = mat_rows(f * aspect, 0.0f, 0.0f, 0.0f,
                                        0.0f, f, 0.0f, 0.0f,
                                        0.0f, 0.0f, -1.0f, 0.0f,
                                        0.0f, 0.0f, 0.0f, 1.0f);
    const M44 r2w = mat_mul(mat_mul(c2w, screenToCamera), rasterToScreen);
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r) out->r2w[c * 4 + r] = r2w.c[c][r];
    out->origin = v3(c2w.c[3][0], c2w.c[3][1], c2w.c[3][2]);
    out->shutterStart = cam.shutterStart;
    out->shutterEnd = cam.shutterEnd;
}

}  // namespace

struct tb200_renderer {
    int device = 0;
    int numSMs = 0;
    cudaStream_t stream = nullptr;        // the stream work is launched on
    cudaStream_t ownStream = nullptr;     // the renderer's private stream (default for `stream`)
    int shard = 0, numShards = 1;
    float4* boundAccum = nullptr;         // caller-owned accumulator (tb200_bind_accumulator)
    cudaEvent_t evStart = nullptr, evStop = nullptr;

    // Device memory.  Every owner frees its allocation when it is reset, reassigned or destroyed; tb200_destroy
    // releases them all at once, with the renderer's device current and before its streams go.
    struct Memory {
        std::vector<DevPtr<void>> scene;   // the scene's arrays (`scene` below points into them)
        DevPtr<float4> accum;
        DevPtr<float> radiance, raster;   // tb200_trace_frame scratch, allocated on first use per image size
        DevPtr<unsigned long long> counter;
        DevPtr<float4> cold;              // cold half of the wavefront's slot state (wf2_common.cuh): 128 B per slot
        DevPtr<float4> filtered;          // tb200_finish, per image size
        DevPtr<unsigned char> rgb8;
        DevPtr<uint2> dither;
        DevPtr<float4> means, denoised;   // tb200_nlm scratch + output, allocated on first use per finish size
        DevPtr<unsigned int> bandCount;   // streamed read-back: band counters on the device,
        HostPtr<unsigned int> bandFlags;  // completion flags in mapped host memory
    } mem;

    DScene scene;

    // film
    int width = 0, height = 0;
    int frame = 0;

    // display/finish step (tb200_finish)
    int finishWidth = 0, finishHeight = 0;   // size mem.filtered, rgb8 and dither were made for
    bool ditherReady = false;
    bool filteredValid = false;              // mem.filtered holds the image of a tb200_finish since the last tb200_init

    // streamed read-back (tb200_render): the band flags' device alias and a private copy stream
    unsigned int* dBandFlags = nullptr;
    cudaStream_t copyStream = nullptr;
    unsigned int bandTag = 0;

    // host read-back: a caller-owned buffer pinned on request (tb200_pin_output), never implicitly
    void* registered = nullptr;
    size_t registeredBytes = 0;

    // owner-computes row slab (tb200_set_slab; slabRows < 0: the whole image)
    int slabRow0 = 0, slabRows = -1;

    // multi-device group (tb200_create_multi): the head owns one renderer per further device, each
    // driven by its own host thread
    std::vector<tb200_renderer*> peers;
    struct Worker* worker = nullptr;      // peers only
    std::string workerError;              // a peer's failure message, handed to the calling thread
    bool peerAccess = false;

    Knobs knobs = {};             // read once, at the start of tb200_create* (read_knobs)
    Wf2Route route = {};          // the wavefront kernel's scheduling, decided at upload (kernels.cu: wavefront2_route)
    const char* lastKernel = "";  // the kernel the last path-tracing launch ran (tb200_last_kernel)
    // Split trace queue on/off is decided by measurement when route.tune (every variant produces the same bits):
    // the second and third sizeable launches after tb200_create time one setting each, the faster stays.
    int tunePhase = 3;            // 0 warm-up (split), 1 measuring split, 2 measuring no split, 3 decided
    double tuneRate[2] = {0.0, 0.0};   // samples per ms with / without the split queue
    unsigned long long launchSamples = 0;   // samples of the launch whose time is in stats.gpuMs
    // most samples (tile padding included) per launch: slot records keep a 32-bit sample index.
    // knobs.launchSamples lowers it, so that tests reach the split at small sizes.
    unsigned long long maxLaunchSamples = 0x7fffffffull;
    tb200_stats stats;
};

namespace {

// ---------------------------------------------------------------------------------------------------
// Scene image: everything build_scene() derives from a tb200_scene, in exactly the layouts the device
// holds -- DPrim records with their hoisted constants, child-pair BVH records in breadth-first order,
// pre-gathered triangles, the flat scene program, the probe with its four sampling tables.  It is
// built on the host (no GPU needed), uploaded array by array, and it is what the scene cache stores
// (tb200_scene_cache_save / tb200_create_cached): a cached scene goes from the file to the device
// without the loader, the BVH re-packing, the per-triangle gather or Probe::BuildCDF.
// ---------------------------------------------------------------------------------------------------
struct MeshImage {
    std::vector<BvhPair> pairs;
    std::vector<float4> verts, norms;
    std::vector<float> cdf;
    int numTris = 0;
    uint32_t rootRef = TB_LEAF;
    int depth = 0;
};

struct SceneImage {
    std::vector<DPrim> prims;
    std::vector<BvhPair> scenePairs;
    uint32_t sceneRoot = TB_LEAF;
    std::vector<ProgOp> flat;
    std::vector<MeshImage> meshes;
    V3 horizon = v3s(0.0f), zenith = v3s(0.0f);
    int numNee = 0;
    // scheduling hints: the largest mesh, and its primitive's world bounds (its leaf of the scene BVH)
    int maxTris = 0;
    int splitBoxValid = 0;
    V3 splitLo = v3s(0.0f), splitHi = v3s(0.0f);
    // probe (src/probe.h:9-86), each table with one element of slack (see below)
    int probeValid = 0, probeW = 0, probeH = 0;
    std::vector<float4> probeData;
    std::vector<float> pdfX, cdfX, pdfY, cdfY;
};

bool image_from_scene(const tb200_scene* s, SceneImage* img)
{
    // meshes: pairs + pre-gathered triangles
    img->meshes.resize(s->numMeshes);
    for (int m = 0; m < s->numMeshes; ++m) {
        const tb200_mesh& g = s->meshes[m];
        MeshImage& mi = img->meshes[m];
        mi.rootRef = build_pairs(g.nodes, g.numNodes, &mi.pairs, &mi.depth);
        const int numTris = g.numIndices / 3;
        mi.numTris = numTris;
        img->maxTris = std::max(img->maxTris, numTris);
        mi.verts.resize(size_t(numTris) * 3);
        mi.norms.resize(size_t(numTris) * 3);
        for (int t = 0; t < numTris; ++t) {
            const int i0 = g.indices[t * 3 + 0], i1 = g.indices[t * 3 + 1], i2 = g.indices[t * 3 + 2];
            const float* a = g.positions + size_t(i0) * 3;
            const float* b = g.positions + size_t(i1) * 3;
            const float* c = g.positions + size_t(i2) * 3;
            mi.verts[size_t(t) * 3 + 0] = make_float4(a[0], a[1], a[2], b[0]);
            mi.verts[size_t(t) * 3 + 1] = make_float4(b[1], b[2], c[0], c[1]);
            mi.verts[size_t(t) * 3 + 2] = make_float4(c[2], 0.0f, 0.0f, 0.0f);
            const float* n1 = g.normals + size_t(i0) * 3;
            const float* n2 = g.normals + size_t(i1) * 3;
            const float* n3 = g.normals + size_t(i2) * 3;
            mi.norms[size_t(t) * 3 + 0] = make_float4(n1[0], n1[1], n1[2], n2[0]);
            mi.norms[size_t(t) * 3 + 1] = make_float4(n2[1], n2[2], n3[0], n3[1]);
            mi.norms[size_t(t) * 3 + 2] = make_float4(n3[2], 0.0f, 0.0f, 0.0f);
        }
        mi.cdf.assign(size_t(numTris), 0.0f);   // only read when the mesh is sampled as a light
        if (g.cdf) memcpy(mi.cdf.data(), g.cdf, size_t(numTris) * sizeof(float));
    }
    // the largest mesh's primitive and its world bounds = that primitive's leaf in the scene BVH
    {
        int bigPrim = -1, bigTris = 0;
        for (int i = 0; i < s->numPrimitives; ++i) {
            const tb200_primitive& p = s->primitives[i];
            if (p.type == TB200_MESH && p.mesh >= 0 && p.mesh < s->numMeshes && s->meshes[p.mesh].numIndices / 3 > bigTris) {
                bigTris = s->meshes[p.mesh].numIndices / 3;
                bigPrim = i;
            }
        }
        for (int n = 0; n < s->numBvhNodes && bigPrim >= 0; ++n) {
            const tb200_bvh_node& node = s->bvhNodes[n];
            if ((node.right_leaf >> 31) != 0 && (int)node.left == bigPrim) {
                img->splitLo = v3(node.lower[0], node.lower[1], node.lower[2]);
                img->splitHi = v3(node.upper[0], node.upper[1], node.upper[2]);
                img->splitBoxValid = 1;
                break;
            }
        }
    }

    // primitives
    img->prims.resize(s->numPrimitives);
    img->numNee = s->sky.probeValid ? 1 : 0;
    for (int i = 0; i < s->numPrimitives; ++i) {
        const tb200_primitive& p = s->primitives[i];
        DPrim& d = img->prims[i];
        memset(&d, 0, sizeof(d));
        d.start = to_xf(p.start);
        d.end = to_xf(p.end);
        d.isStatic = memcmp(&p.start, &p.end, sizeof(tb200_transform)) == 0;
        // with start == end, Lerp(a,b,t) = a + (b-a)*t = a + 0*t is time independent
        d.fixed = interpolate_transform(d.start, d.end, 0.0f);
        d.type = p.type;
        d.radius = p.radius;
        memcpy(d.plane, p.plane, 16);
        d.mesh = p.mesh;
        d.lightSamples = p.lightSamples;
        if (p.type == TB200_MESH && (p.mesh < 0 || p.mesh >= s->numMeshes)) return set_error("primitive references a missing mesh");
        // PrimitiveArea, intersection.h:833-853
        if (p.type == TB200_SPHERE)
            d.area = 4.0f * TB_PI * p.radius * p.radius;
        else if (p.type == TB200_MESH)
            d.area = s->meshes[p.mesh].area * p.end.s;
        else
            d.area = 0.0f;
        d.mat = make_material(p.material);
        if (p.lightSamples > 0) img->numNee += p.lightSamples;
    }
    set_fresnel_flags(img->prims.size(), [&](size_t i) -> DMaterial& { return img->prims[i].mat; });
    img->sceneRoot = build_pairs(s->bvhNodes, s->numBvhNodes, &img->scenePairs);
    build_program(s, &img->flat);
    img->horizon = hv3(s->sky.horizon);
    img->zenith = hv3(s->sky.zenith);
    if (s->sky.probeValid) {
        const size_t n = size_t(s->sky.probeWidth) * s->sky.probeHeight;
        img->probeValid = 1;
        img->probeW = s->sky.probeWidth;
        img->probeH = s->sky.probeHeight;
        // one element of slack after each table: ProbeSample's column search may land on
        // col == width (probe.h:217-220) and read one past the last row
        img->probeData.assign(n + 1, make_float4(0.0f, 0.0f, 0.0f, 0.0f));
        memcpy(img->probeData.data(), s->sky.probeData, n * 16);
        img->pdfX.assign(n + 1, 0.0f);
        img->cdfX.assign(n + 1, 0.0f);
        img->pdfY.assign(size_t(s->sky.probeHeight) + 1, 0.0f);
        img->cdfY.assign(size_t(s->sky.probeHeight) + 1, 0.0f);
        memcpy(img->pdfX.data(), s->sky.pdfValuesX, n * 4);
        memcpy(img->cdfX.data(), s->sky.cdfValuesX, n * 4);
        memcpy(img->pdfY.data(), s->sky.pdfValuesY, size_t(s->sky.probeHeight) * 4);
        memcpy(img->cdfY.data(), s->sky.cdfValuesY, size_t(s->sky.probeHeight) * 4);
    }
    return true;
}

// The scene's features (tb_scene.cuh: TB_FEAT_*).  A scene without any of them runs the lane-owned kernel compiled
// without them (kernels.cu: launch_wavefront2).
uint32_t scene_features(const SceneImage& img)
{
    uint32_t f = img.probeValid ? TB_FEAT_PROBE : TB_FEAT_NONE;
    for (const DPrim& p : img.prims) {
        if (!p.isStatic) f |= TB_FEAT_MOTION;
        f |= material_features(p.mat);
    }
    return f;
}

// Copies `host` and padElems zeroed elements after it into a new allocation of r's scene memory; *dev = its
// address, null for no elements
template <typename T>
bool upload(tb200_renderer* r, const std::vector<T>& host, const T** dev, size_t padElems = 0)
{
    *dev = nullptr;
    const size_t n = host.size() + padElems;
    if (n == 0) return true;
    DevPtr<T> mem;
    TB_CUDA(dev_alloc(&mem, n));
    if (padElems) TB_CUDA(cudaMemset(mem.get(), 0, n * sizeof(T)));
    if (!host.empty()) TB_CUDA(cudaMemcpy(mem.get(), host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice));
    r->stats.h2dBytes += host.size() * sizeof(T);
    *dev = mem.get();
    r->mem.scene.push_back(std::move(mem));
    return true;
}

// device upload of a scene image + the per-scene scheduling decisions (from r->knobs)
bool upload_image(tb200_renderer* r, const SceneImage& img)
{
    memset(&r->scene, 0, sizeof(r->scene));
    std::vector<DMesh> meshes(img.meshes.size());
    for (size_t m = 0; m < img.meshes.size(); ++m) {
        const MeshImage& mi = img.meshes[m];
        if (!upload(r, mi.pairs, &meshes[m].pairs) || !upload(r, mi.verts, &meshes[m].triVerts) ||
            !upload(r, mi.norms, &meshes[m].triNormals) || !upload(r, mi.cdf, &meshes[m].cdf))
            return false;
        meshes[m].numTris = mi.numTris;
        meshes[m].rootRef = mi.rootRef;
    }
    DScene& sc = r->scene;
    if (!upload(r, meshes, &sc.meshes)) return false;
    sc.splitValid = img.splitBoxValid;
    sc.splitLo = img.splitLo;
    sc.splitHi = img.splitHi;
    r->route = wavefront2_route(img.numNee, img.maxTris, img.splitBoxValid, scene_features(img), r->knobs);
    r->tunePhase = r->route.tune ? 0 : 3;
    // one element of padding each: the kernels' bulk copies round their length up to 16 bytes
    if (!upload(r, img.prims, &sc.prims, 1)) return false;
    if (!upload(r, img.scenePairs, &sc.pairs, 1)) return false;
    sc.numPrims = (int)img.prims.size();
    sc.numPairs = (int)img.scenePairs.size();
    static const std::vector<ProgOp> noFlat;
    const std::vector<ProgOp>& flat = r->knobs.noFlat ? noFlat : img.flat;
    if (!upload(r, flat, &sc.flat, 1)) return false;
    sc.numFlat = (int)flat.size();
    // treelet: the top of the largest mesh's BVH staged in the shared memory the slot arrays leave, for the
    // mesh walk.  Measured in round 2: slower on every scene (ajax, env, meshlight) because the top levels already
    // live in L1, and claiming the last 45 KB of shared memory shrinks L1 from 60 to 28 KB.  Off unless TINSEL_B200_TREELET=1.
    sc.treelet = nullptr;
    sc.treeletMesh = -1;
    sc.treeletPairs = 0;
    {
        int big = -1;
        for (size_t m = 0; m < img.meshes.size(); ++m)
            if (img.meshes[m].numTris > 1024 && (big < 0 || img.meshes[m].numTris > img.meshes[big].numTris)) big = (int)m;
        if (big >= 0 && r->knobs.treelet) {
            sc.treeletMesh = big;
            sc.treeletPairs = (int)img.meshes[big].pairs.size();
        }
    }
    sc.rootRef = img.sceneRoot;
    sc.numMeshes = (int)img.meshes.size();
    sc.horizon = img.horizon;
    sc.zenith = img.zenith;
    sc.numNee = img.numNee;
    if (img.probeValid) {
        if (!upload(r, img.probeData, &sc.probe.data) || !upload(r, img.pdfX, &sc.probe.pdfX) || !upload(r, img.cdfX, &sc.probe.cdfX) ||
            !upload(r, img.pdfY, &sc.probe.pdfY) || !upload(r, img.cdfY, &sc.probe.cdfY))
            return false;
        sc.probe.valid = 1;
        sc.probe.width = img.probeW;
        sc.probe.height = img.probeH;
    }
    return true;
}

bool build_scene(tb200_renderer* r, const tb200_scene* s)
{
    SceneImage img;
    return image_from_scene(s, &img) && upload_image(r, img);
}

// ---- scene cache file ------------------------------------------------------------------------------
// "TB2CACHE", a layout stamp (the records are this build's device structs, not an interchange format:
// a stamp mismatch is refused and the caller falls back to tb200_create), then the SceneImage fields in
// declaration order; every array as a 64-bit count followed by its bytes.
const char kCacheMagic[8] = {'T', 'B', '2', 'C', 'A', 'C', 'H', 'E'};
const uint32_t kCacheVersion = 3;   // 3: DMaterial::flags

struct CacheStamp {
    uint32_t version, sizeofPrim, sizeofPair, sizeofOp;
};

struct CacheWriter {
    FILE* f;
    template <typename T>
    bool pod(const T& v) { return fwrite(&v, sizeof(T), 1, f) == 1; }
    template <typename T>
    bool vec(const std::vector<T>& v)
    {
        const uint64_t n = v.size();
        return pod(n) && (n == 0 || fwrite(v.data(), sizeof(T), n, f) == n);
    }
    bool count(const std::vector<MeshImage>& v) { return pod(uint64_t(v.size())); }
};

// Every count is checked against the file's size before anything is allocated for it.
struct CacheReader {
    FILE* f;
    uint64_t fileBytes;
    template <typename T>
    bool pod(T& v) { return fread(&v, sizeof(T), 1, f) == 1; }
    template <typename T>
    bool vec(std::vector<T>& v)
    {
        uint64_t n = 0;
        if (!pod(n) || n > fileBytes / sizeof(T)) return false;   // a count can never exceed the file
        v.resize(size_t(n));
        return n == 0 || fread(v.data(), sizeof(T), size_t(n), f) == n;
    }
    bool count(std::vector<MeshImage>& v)
    {
        uint64_t n = 0;
        if (!pod(n) || n > fileBytes) return false;
        v.resize(size_t(n));
        return true;
    }
};

// The SceneImage fields in file order, for a CacheWriter (Image = const SceneImage) or a CacheReader: the one
// statement of the format after the stamp.  vec(v) is a 64-bit count followed by the elements; count(meshes) is
// the number of meshes, whose fields follow mesh by mesh.
template <typename IO, typename Image>
bool cache_fields(IO& io, Image& img)
{
    bool ok = io.vec(img.prims) && io.vec(img.scenePairs) && io.pod(img.sceneRoot) && io.vec(img.flat) && io.count(img.meshes);
    for (auto& m : img.meshes)
        ok = ok && io.vec(m.pairs) && io.vec(m.verts) && io.vec(m.norms) && io.vec(m.cdf) && io.pod(m.numTris) && io.pod(m.rootRef) &&
             io.pod(m.depth);
    return ok && io.pod(img.horizon) && io.pod(img.zenith) && io.pod(img.numNee) && io.pod(img.maxTris) && io.pod(img.splitBoxValid) &&
           io.pod(img.splitLo) && io.pod(img.splitHi) && io.pod(img.probeValid) && io.pod(img.probeW) && io.pod(img.probeH) &&
           io.vec(img.probeData) && io.vec(img.pdfX) && io.vec(img.cdfX) && io.vec(img.pdfY) && io.vec(img.cdfY);
}

bool image_save(const SceneImage& img, const char* path)
{
    FILE* f = fopen(path, "wb");
    if (!f) return set_error(std::string("tb200_scene_cache_save: cannot open ") + path);
    const CacheStamp stamp = {kCacheVersion, (uint32_t)sizeof(DPrim), (uint32_t)sizeof(BvhPair), (uint32_t)sizeof(ProgOp)};
    CacheWriter w{f};
    bool ok = fwrite(kCacheMagic, 1, 8, f) == 8 && w.pod(stamp) && cache_fields(w, img);
    ok = (fclose(f) == 0) && ok;
    return ok ? true : set_error(std::string("tb200_scene_cache_save: write failed: ") + path);
}

bool image_load(const char* path, SceneImage* img)
{
    FILE* f = fopen(path, "rb");
    if (!f) return set_error(std::string("tb200_create_cached: cannot open ") + path);
    fseek(f, 0, SEEK_END);
    const uint64_t fileBytes = (uint64_t)std::max(0L, ftell(f));
    fseek(f, 0, SEEK_SET);
    char magic[8];
    CacheStamp stamp;
    CacheReader rd{f, fileBytes};
    bool ok = fread(magic, 1, 8, f) == 8 && memcmp(magic, kCacheMagic, 8) == 0 && rd.pod(stamp);
    if (ok && (stamp.version != kCacheVersion || stamp.sizeofPrim != sizeof(DPrim) || stamp.sizeofPair != sizeof(BvhPair) ||
               stamp.sizeofOp != sizeof(ProgOp))) {
        fclose(f);
        return set_error(std::string("tb200_create_cached: ") + path + " was written by another build of this library (layout stamp differs): recreate it");
    }
    ok = ok && cache_fields(rd, *img);
    fclose(f);
    if (!ok) return set_error(std::string("tb200_create_cached: truncated or malformed cache file ") + path);
    return true;
}

// levels: tb_tree_levels' result for the BVH called `what`
bool bvh_levels_ok(int levels, const std::string& what, std::string* why)
{
    if (levels < 0) return *why = what + ": a BVH node is reached twice from the root (shared subtree or cycle)", false;
    if (levels > TB200_MAX_BVH_LEVELS)
        return *why = what + ": BVH has " + std::to_string(levels) + " levels of interior nodes, more than the " +
                      std::to_string(TB200_MAX_BVH_LEVELS) + " the traversal stack holds", false;
    return true;
}

// levels of the BvhPair tree below `root`, or -1 (see tb_tree_levels)
int pair_levels(const std::vector<BvhPair>& pairs, uint32_t root)
{
    return tb_tree_levels(root, pairs.size(), [&pairs](uint32_t ref, uint32_t* c) {
        if (ref & TB_LEAF) return false;
        c[0] = pairs[ref].left;
        c[1] = pairs[ref].right;
        return true;
    });
}

// every index a kernel will follow stays inside its array, and every BVH is a tree the traversal stack can
// hold (a cache file is as untrusted as a tb200_scene)
bool validate_image(const SceneImage& img, std::string* why)
{
    const size_t np = img.prims.size();
    if (np == 0 || np > TB200_MAX_PRIMITIVES) return *why = "bad primitive count", false;
    auto ref_ok = [](uint32_t ref, size_t pairs, size_t items) { return (ref & TB_LEAF) ? (ref & ~TB_LEAF) < items : ref < pairs; };
    if (!ref_ok(img.sceneRoot, img.scenePairs.size(), np)) return *why = "scene root reference out of range", false;
    for (const BvhPair& p : img.scenePairs)
        if (!ref_ok(p.left, img.scenePairs.size(), np) || !ref_ok(p.right, img.scenePairs.size(), np)) return *why = "scene BVH reference out of range", false;
    if (!bvh_levels_ok(pair_levels(img.scenePairs, img.sceneRoot), "scene", why)) return false;
    for (size_t k = 0; k < img.meshes.size(); ++k) {
        const MeshImage& m = img.meshes[k];
        const size_t nt = (size_t)std::max(0, m.numTris);
        if (nt == 0 || m.verts.size() != nt * 3 || m.norms.size() != nt * 3 || m.cdf.size() != nt) return *why = "mesh arrays do not match the triangle count", false;
        if (!ref_ok(m.rootRef, m.pairs.size(), nt)) return *why = "mesh root reference out of range", false;
        for (const BvhPair& p : m.pairs)
            if (!ref_ok(p.left, m.pairs.size(), nt) || !ref_ok(p.right, m.pairs.size(), nt)) return *why = "mesh BVH reference out of range", false;
        const std::string name = "mesh " + std::to_string(k);
        if (m.depth < 0 || m.depth > TB200_MAX_BVH_LEVELS)
            return *why = name + ": stored BVH depth " + std::to_string(m.depth) + " is outside 0.." + std::to_string(TB200_MAX_BVH_LEVELS), false;
        const int levels = pair_levels(m.pairs, m.rootRef);
        if (!bvh_levels_ok(levels, name, why)) return false;
        if (levels != m.depth) return *why = name + ": stored BVH depth does not match the tree", false;
    }
    for (const DPrim& p : img.prims) {
        if (p.type != TB200_SPHERE && p.type != TB200_PLANE && p.type != TB200_MESH) return *why = "unknown primitive type", false;
        if (p.type == TB200_MESH && (p.mesh < 0 || (size_t)p.mesh >= img.meshes.size())) return *why = "primitive references a missing mesh", false;
        if (p.lightSamples < 0 || p.lightSamples > TB200_MAX_LIGHT_SAMPLES) return *why = "lightSamples out of range", false;
    }
    for (const ProgOp& op : img.flat)
        if ((size_t)(op.kindPrim >> 8) >= np && (op.kindPrim & 0xff) != TB_OP_BOX) return *why = "scene program references a missing primitive", false;
    if (img.flat.size() > 32) return *why = "scene program too long", false;
    if (img.probeValid) {
        const size_t n = (size_t)std::max(0, img.probeW) * (size_t)std::max(0, img.probeH);
        if (n == 0 || img.probeData.size() != n + 1 || img.pdfX.size() != n + 1 || img.cdfX.size() != n + 1 ||
            img.pdfY.size() != (size_t)img.probeH + 1 || img.cdfY.size() != (size_t)img.probeH + 1)
            return *why = "probe tables do not match the probe size", false;
    }
    return true;
}

// pixel rows a sample of row y can splat into: y - reach .. y + reach (render.cpp:404-407).  The width is
// clamped to [0, 2^30] first (NaN counts as 0), the widths fill_params accepts, so that no width -- infinite, NaN
// or huge -- converts to int out of range; row + reach then stays in range for images of fewer than 2^30 rows.
int filter_reach(float filterWidth) { return (int)ceilf(std::min(std::max(0.0f, filterWidth), 1073741824.0f)) + 1; }

// add_sample converts raster +- filterWidth to int.  Below 2^30 in magnitude that conversion is defined on the
// device and the host alike for every image size; a NaN, infinite or larger width saturates on the device and is
// undefined on the host.  Any filter type but the two known ones is read as Gaussian by the device and as a box
// by the CPU restatement.
bool filter_options_ok(const tb200_options* o)
{
    if (o->filterType != TB200_FILTER_BOX && o->filterType != TB200_FILTER_GAUSSIAN)
        return set_error("options.filterType " + std::to_string(o->filterType) + " is neither TB200_FILTER_BOX nor TB200_FILTER_GAUSSIAN");
    if (!(std::fabs(o->filterWidth) < 1073741824.0f))
        return set_error("options.filterWidth " + std::to_string(o->filterWidth) + " is not finite or is 2^30 or more in magnitude");
    return true;
}

bool fill_params(tb200_renderer* r, const tb200_camera* camera, const tb200_options* o, LaunchParams* P)
{
    if (!r->mem.accum) return set_error("tb200_init has not been called");
    if (o->width != r->width || o->height != r->height)
        return set_error("options.width/height differ from the last tb200_init");
    if (!filter_options_ok(o)) return false;
    memset(P, 0, sizeof(*P));
    P->scene = r->scene;
    camera_setup(*camera, o->width, o->height, &P->camera);
    P->film.width = o->width;
    P->film.height = o->height;
    P->film.filterType = o->filterType;
    P->film.filterWidth = o->filterWidth;
    P->film.filterFalloff = o->filterFalloff;
    P->film.filterOffset = o->filterOffset;
    P->film.clamp = o->clamp;
    P->film.maxDepth = o->maxDepth;
    P->film.filterArgZero = film_filter_arg_zero(o->filterOffset);
    P->accum = r->boundAccum ? r->boundAccum : r->mem.accum.get();
    P->sampleCounter = r->mem.counter.get();
    P->cold = r->mem.cold.get();
    P->firstRow = 0;
    P->numRows = o->height;
    P->film.rowLo = 0;
    P->film.rowHi = o->height;
    if (r->slabRows >= 0) {
        // owner-computes slab: trace the owned rows plus every row whose samples can reach them
        // (render.cpp:404-407: a sample of row y splats into rows int(y' - w) .. int(y' + w), y' in [y, y+1]),
        // splat into the owned rows only
        const int reach = filter_reach(o->filterWidth);
        const int lo = std::max(0, std::min(r->slabRow0, o->height));
        const int hi = std::max(lo, std::min(r->slabRow0 + r->slabRows, o->height));
        P->film.rowLo = lo;
        P->film.rowHi = hi;
        P->firstRow = std::max(0, lo - reach);
        P->numRows = hi > lo ? std::min(o->height, hi + reach) - P->firstRow : 0;
    }
    P->shard = r->shard;
    P->numShards = r->numShards;
    finalize_params(P);
    return true;
}

bool launch_frames(tb200_renderer* r, LaunchParams& P, bool recordStart = true)
{
    unsigned long long launches = 0;
    if (recordStart) TB_CUDA(cudaEventRecord(r->evStart, r->stream));
    if (P.samplesPerFrame > 0) {
        // slot records keep a 32-bit sample index: split very long jobs into several launches
        const int framesPerLaunch = (int)std::max<unsigned long long>(1ull, r->maxLaunchSamples / P.samplesPerFrame);
        const int frame0 = P.frame0, frames = P.numFrames;
        for (int f = 0; f < frames; f += framesPerLaunch) {
            P.frame0 = frame0 + f;
            P.numFrames = std::min(framesPerLaunch, frames - f);
            const char* name = r->knobs.mega ? launch_mega(P, r->stream, &launches) : launch_wavefront2(P, r->route, r->numSMs, r->stream, &launches);
            if (name) r->lastKernel = name;
        }
        P.frame0 = frame0;
        P.numFrames = frames;
    }
    TB_CUDA(cudaEventRecord(r->evStop, r->stream));
    TB_CUDA(cudaGetLastError());
    r->stats.kernelLaunches += launches;
    {
        // samples inside the image (tile padding excluded; with a slab: the owned rows, not their halo)
        uint64_t rows = 0;
        if (r->slabRows >= 0)
            rows = (uint64_t)(P.film.rowHi - P.film.rowLo);
        else
            for (int t = P.shard; t * 4 < P.numRows; t += P.numShards) rows += (uint64_t)((P.numRows - t * 4) < 4 ? (P.numRows - t * 4) : 4);
        r->stats.samples += rows * (uint64_t)P.film.width * (uint64_t)P.numFrames;
        r->launchSamples = rows * (uint64_t)P.film.width * (uint64_t)P.numFrames;
    }
    return true;
}

// called once the time of a path-tracing launch is in stats.gpuMs
void tune_update(tb200_renderer* r)
{
    if (r->tunePhase >= 3 || r->launchSamples < (1ull << 18) || !(r->stats.gpuMs > 0.0)) return;
    const double rate = (double)r->launchSamples / r->stats.gpuMs;
    if (r->tunePhase == 1) r->tuneRate[0] = rate;
    if (r->tunePhase == 2) r->tuneRate[1] = rate;
    r->tunePhase += 1;
    // phase 2 runs without the split queue; once it is measured, the faster setting stays
    if (r->tunePhase >= 2) r->route.split = r->tunePhase == 3 && r->tuneRate[0] >= r->tuneRate[1];
}

// waits for the work between evStart and evStop and sets stats.gpuMs to its time
bool sync_gpu_ms(tb200_renderer* r)
{
    TB_CUDA(cudaEventSynchronize(r->evStop));
    float ms = 0.0f;
    TB_CUDA(cudaEventElapsedTime(&ms, r->evStart, r->evStop));
    r->stats.gpuMs = ms;
    return true;
}

// pixel rows [row0, row1) this renderer is responsible for delivering to the host
void owned_rows(const tb200_renderer* r, int* row0, int* row1)
{
    if (r->slabRows < 0) {
        *row0 = 0;
        *row1 = r->height;
    } else {
        *row0 = std::max(0, std::min(r->slabRow0, r->height));
        *row1 = std::max(*row0, std::min(r->slabRow0 + r->slabRows, r->height));
    }
}

// device -> host copy of the owned rows of the accumulator after the stream's work.  `output` is
// the caller's whole-image buffer; whether it is pinned (tb200_pin_output) is the caller's choice:
// a pageable buffer takes the driver's staged path.
bool read_back(tb200_renderer* r, float* output)
{
    int row0, row1;
    owned_rows(r, &row0, &row1);
    const size_t rowBytes = size_t(r->width) * sizeof(float4);
    const size_t bytes = size_t(row1 - row0) * rowBytes;
    const char* accum = (const char*)(r->boundAccum ? r->boundAccum : r->mem.accum.get());
    if (bytes)
        TB_CUDA(cudaMemcpyAsync((char*)output + size_t(row0) * rowBytes, accum + size_t(row0) * rowBytes, bytes, cudaMemcpyDeviceToHost, r->stream));
    TB_CUDA(cudaStreamSynchronize(r->stream));
    r->stats.d2hBytes += bytes;
    return true;
}

// One frame of the wavefront kernel with the read-back streamed underneath it: samples are handed
// out in tile-row order, the kernel flags each band of tile rows as its last sample retires
// (wf2_common.cuh, wf2_band_report), and this thread copies every owned pixel row that no
// unfinished sample can still touch while the kernel is tracing the rest.  What is left when the
// kernel ends is the last band or two instead of the whole slab.
bool render_streamed(tb200_renderer* r, LaunchParams& P, float* output, bool recordStart)
{
    const float4* accum = P.accum;
    const size_t rowBytes = size_t(r->width) * sizeof(float4);
    // bands of whole tile rows, at most TB_MAX_BANDS, about 256 KiB each: what is left to copy when the
    // kernel ends is one band plus the filter's reach, and consecutive finished bands go out in one copy
    int bandTileRows = std::max(1, (int)((size_t(1) << 18) / (rowBytes * 4)));
    bandTileRows = std::max(bandTileRows, (P.tileRows + TB_MAX_BANDS - 1) / TB_MAX_BANDS);
    const int numBands = (P.tileRows + bandTileRows - 1) / bandTileRows;
    const int reach = filter_reach(P.film.filterWidth);
    int own0, own1;
    owned_rows(r, &own0, &own1);

    r->bandTag += 1;
    if (r->bandTag == 0) r->bandTag = 1;
    P.bandCount = r->mem.bandCount.get();
    P.bandFlags = r->dBandFlags;
    P.bandSamples = (unsigned)bandTileRows * (unsigned)P.tilesX * 32u;
    P.bandTag = r->bandTag;
    if (recordStart) TB_CUDA(cudaEventRecord(r->evStart, r->stream));
    TB_CUDA(cudaMemsetAsync(P.bandCount, 0, TB_MAX_BANDS * sizeof(unsigned int), r->stream));
    if (!launch_frames(r, P, false)) return false;

    const volatile unsigned int* bandFlags = r->mem.bandFlags.get();
    int done = 0;          // bands 0..done-1 are complete
    int copied = own0;     // owned pixel rows [own0, copied) are already on their way to the host
    bool copyFailed = false;
    auto copy_rows_below = [&](int limit) {
        limit = std::min(limit, own1);
        if (limit <= copied) return;
        if (cudaMemcpyAsync((char*)output + size_t(copied) * rowBytes, (const char*)accum + size_t(copied) * rowBytes,
                            size_t(limit - copied) * rowBytes, cudaMemcpyDeviceToHost, r->copyStream) != cudaSuccess)
            copyFailed = true;
        copied = limit;
    };
    unsigned spins = 0;
    for (;;) {
        while (done < numBands && bandFlags[done] == r->bandTag) ++done;
        if (done >= numBands) break;
        // unfinished samples sit in local tile rows >= done*bandTileRows, i.e. global pixel rows
        // >= firstRow + done*bandTileRows*numShards*4 (decode_sample)
        copy_rows_below(P.firstRow + done * bandTileRows * P.numShards * 4 - reach);
        // The band flags (plain reads of mapped host memory) are the signal; the event is only the safety net for a
        // launch that failed -- and a driver call per spin from every device's thread of a multi-device renderer
        // contends on the driver's locks, so it is asked rarely.
        ++spins;
        if ((spins & 1023u) == 0u && cudaEventQuery(r->evStop) != cudaErrorNotReady) break;   // finished (or failed): stop polling
        // back off: the calling thread may be the host application's UI thread (tinsel's GLUT loop)
        if (spins < 4096u)
            __builtin_ia32_pause();
        else
            std::this_thread::yield();
    }
    TB_CUDA(cudaStreamSynchronize(r->stream));
    copy_rows_below(own1);
    TB_CUDA(cudaStreamSynchronize(r->copyStream));
    if (copyFailed) TB_CUDA(cudaErrorUnknown);
    r->stats.d2hBytes += size_t(own1 - own0) * rowBytes;
    return true;
}

// Runs frames r->frame .. r->frame + n - 1 (n >= 1) of P, filled by fill_params, and sets stats.gpuMs to the time
// from the first launch to the end of the last.  With `output`, the caller's whole image, it also delivers the owned
// rows there: streamed under the last frame when the wavefront kernel runs it and its sample indices fit in 31 bits,
// else copied after the frames.  The frame counters advance only when all of this succeeded.
bool run_frames(tb200_renderer* r, LaunchParams& P, int n, float* output)
{
    const bool streamed = output && !r->knobs.plainReadback && !r->knobs.mega &&P.samplesPerFrame > 0 && P.samplesPerFrame < 0x7fffffffull;
    const int head = streamed ? n - 1 : n;   // frames launched before the streamed one
    P.frame0 = r->frame;
    P.numFrames = head;
    if (head > 0 && !launch_frames(r, P)) return false;
    if (streamed) {
        P.frame0 = r->frame + head;
        P.numFrames = 1;
        if (!render_streamed(r, P, output, head == 0)) return false;
    } else if (output && !read_back(r, output)) {
        return false;
    }
    if (!sync_gpu_ms(r)) return false;
    r->frame += n;
    r->stats.frames += n;
    return true;
}

}  // namespace

// One host thread per further device of a multi-device renderer.  Render() is called back to back
// (16 times per displayed frame, src/main.cpp:242-251) and a frame's kernel takes a fraction of a
// millisecond, so a worker spins briefly for its next job before it goes to sleep on the condition
// variable: a wake-up through the kernel would cost as much as the job.
struct Worker {
    std::thread thread;
    std::mutex lock;
    std::condition_variable wake;
    std::function<int(tb200_renderer*)> job;
    std::atomic<uint32_t> posted{0}, done{0};
    bool sleeping = false;
    std::atomic<bool> quit{false};
    int rc = 0;
};

namespace {

void worker_main(tb200_renderer* r)
{
    Worker* w = r->worker;
    cudaSetDevice(r->device);
    uint32_t seen = 0;
    for (;;) {
        int spins = 0;
        while (w->posted.load(std::memory_order_acquire) == seen) {
            if (++spins < 200000) {
                __builtin_ia32_pause();
                continue;
            }
            std::unique_lock<std::mutex> guard(w->lock);
            w->sleeping = true;
            w->wake.wait(guard, [&] { return w->posted.load(std::memory_order_acquire) != seen || w->quit.load(); });
            w->sleeping = false;
            spins = 0;
        }
        // tb200_destroy bumps `posted` to get a spinning worker out of its loop: that is not a job (the last one is
        // still in `job` -- running it again would render one more frame into a buffer the caller may have freed)
        if (w->quit.load(std::memory_order_acquire)) return;
        seen += 1;
        g_error.clear();
        w->rc = w->job(r);
        r->workerError = w->rc != 0 ? g_error : std::string();
        w->done.store(seen, std::memory_order_release);
    }
}

void worker_post(tb200_renderer* r, const std::function<int(tb200_renderer*)>& job)
{
    Worker* w = r->worker;
    w->job = job;
    w->posted.fetch_add(1, std::memory_order_release);
    std::lock_guard<std::mutex> guard(w->lock);
    if (w->sleeping) w->wake.notify_one();
}

int worker_wait(tb200_renderer* r)
{
    Worker* w = r->worker;
    const uint32_t want = w->posted.load(std::memory_order_relaxed);
    unsigned spins = 0;
    while (w->done.load(std::memory_order_acquire) != want) {
        if (++spins < 4096u)
            __builtin_ia32_pause();
        else
            std::this_thread::yield();
    }
    return w->rc;
}

// runs `job` on the head (calling thread) and on every peer (its worker thread) at the same time;
// returns 0 when all succeeded, else -1 with the first failure as this thread's last error
int group_run(tb200_renderer* head, const std::function<int(tb200_renderer*)>& job)
{
    for (tb200_renderer* p : head->peers) worker_post(p, job);
    cudaSetDevice(head->device);
    int rc = job(head);
    for (tb200_renderer* p : head->peers) {
        if (worker_wait(p) != 0 && rc == 0) {
            rc = -1;
            set_error("device " + std::to_string(p->device) + ": " + p->workerError);
        }
    }
    return rc;
}

// contiguous row slabs, cut at tile rows (4 pixel rows): member k of n owns [cut(k), cut(k+1))
int slab_cut(int height, int k, int n)
{
    if (k >= n) return height;
    const int tileRows = (height + 3) / 4;
    return std::min(height, (int)((long long)tileRows * k / n) * 4);
}

}  // namespace

extern "C" {

const char* tb200_last_error(void)
{
    // two sticky messages (this file's and snapshot.cpp's): the more recent one
    if (!g_error.empty() && g_errorStamp > tb200_snapshot_error_stamp()) return g_error.c_str();
    const char* snap = tb200_snapshot_error();
    if (snap && snap[0]) return snap;
    return g_error.c_str();
}

// Structural checks on the caller's scene before anything is uploaded: every index the kernels will
// follow must stay inside its array, and every BVH must be a tree no deeper than the traversal stack holds
// (the reference trusts its own loader; a C ABI cannot).
static bool validate_bvh(const tb200_bvh_node* nodes, int numNodes, int numItems, const char* what, std::string* why)
{
    if (numNodes <= 0 || !nodes) {
        *why = std::string(what) + ": no BVH nodes";
        return false;
    }
    for (int i = 0; i < numNodes; ++i) {
        const bool leaf = (nodes[i].right_leaf >> 31) != 0;
        const uint32_t left = nodes[i].left, right = nodes[i].right_leaf & 0x7fffffffu;
        if (leaf ? left >= (uint32_t)numItems : (left >= (uint32_t)numNodes || right >= (uint32_t)numNodes)) {
            *why = std::string(what) + ": BVH node " + std::to_string(i) + " points outside its array";
            return false;
        }
    }
    const int levels = tb_tree_levels(0u, (size_t)numNodes, [nodes](uint32_t i, uint32_t* c) {
        if (nodes[i].right_leaf >> 31) return false;
        c[0] = nodes[i].left;
        c[1] = nodes[i].right_leaf & 0x7fffffffu;
        return true;
    });
    return bvh_levels_ok(levels, what, why);
}

static bool validate_scene(const tb200_scene* s, std::string* why)
{
    if (s->numPrimitives <= 0 || !s->primitives) return *why = "scene has no primitives", false;
    if (s->numPrimitives > TB200_MAX_PRIMITIVES)
        return *why = "more than " + std::to_string(TB200_MAX_PRIMITIVES) + " primitives (the wavefront's NEE cursor holds 12-bit primitive indices)", false;
    if (s->numMeshes < 0 || (s->numMeshes > 0 && !s->meshes)) return *why = "bad mesh array", false;
    if (!validate_bvh(s->bvhNodes, s->numBvhNodes, s->numPrimitives, "scene", why)) return false;
    for (int m = 0; m < s->numMeshes; ++m) {
        const tb200_mesh& g = s->meshes[m];
        const std::string name = "mesh " + std::to_string(m);
        if (g.numVertices <= 0 || g.numIndices <= 0 || g.numIndices % 3 != 0 || !g.positions || !g.normals || !g.indices)
            return *why = name + ": empty or incomplete geometry", false;
        for (int i = 0; i < g.numIndices; ++i)
            if (g.indices[i] < 0 || g.indices[i] >= g.numVertices) return *why = name + ": vertex index out of range", false;
        if (!validate_bvh(g.nodes, g.numNodes, g.numIndices / 3, name.c_str(), why)) return false;
    }
    for (int i = 0; i < s->numPrimitives; ++i) {
        const tb200_primitive& p = s->primitives[i];
        if (p.type != TB200_SPHERE && p.type != TB200_PLANE && p.type != TB200_MESH)
            return *why = "primitive " + std::to_string(i) + ": unknown type", false;
        if (p.type == TB200_MESH && (p.mesh < 0 || p.mesh >= s->numMeshes))
            return *why = "primitive " + std::to_string(i) + ": mesh index out of range", false;
        if (p.type == TB200_MESH && p.lightSamples > 0 && !s->meshes[p.mesh].cdf)
            return *why = "primitive " + std::to_string(i) + ": mesh light without a sampling CDF", false;
        if (p.lightSamples < 0 || p.lightSamples > TB200_MAX_LIGHT_SAMPLES)
            return *why = "primitive " + std::to_string(i) + ": lightSamples out of range", false;
    }
    if (s->sky.probeValid) {
        const tb200_sky& k = s->sky;
        if (k.probeWidth <= 0 || k.probeHeight <= 0 || !k.probeData || !k.pdfValuesX || !k.cdfValuesX || !k.pdfValuesY || !k.cdfValuesY)
            return *why = "sky probe: missing tables", false;
    }
    return true;
}

static tb200_renderer* create_with(int device, const std::function<bool(tb200_renderer*)>& build);

tb200_renderer* tb200_create(const tb200_scene* scene, int device)
{
    g_error.clear();
    if (!scene) {
        set_error("tb200_create: null scene");
        return nullptr;
    }
    {
        std::string why;
        if (!validate_scene(scene, &why)) {
            set_error("tb200_create: invalid scene: " + why);
            return nullptr;
        }
    }
    return create_with(device, [scene](tb200_renderer* r) { return build_scene(r, scene); });
}

int tb200_scene_cache_save(const tb200_scene* scene, const char* path)
{
    g_error.clear();
    if (!scene || !path) {
        set_error("tb200_scene_cache_save: null argument");
        return -1;
    }
    std::string why;
    if (!validate_scene(scene, &why)) {
        set_error("tb200_scene_cache_save: invalid scene: " + why);
        return -1;
    }
    SceneImage img;
    if (!image_from_scene(scene, &img)) return -1;
    return image_save(img, path) ? 0 : -1;
}

tb200_renderer* tb200_create_cached(const char* path, int device)
{
    g_error.clear();
    if (!path) {
        set_error("tb200_create_cached: null path");
        return nullptr;
    }
    // SceneImage is heavy (hundreds of MB for a big mesh + probe): shared with the build step, freed after it
    std::shared_ptr<SceneImage> img(new SceneImage());
    try {
        if (!image_load(path, img.get())) return nullptr;
    } catch (const std::exception& e) {   // bad_alloc from a corrupt count that passed the size check
        set_error(std::string("tb200_create_cached: ") + e.what());
        return nullptr;
    }
    std::string why;
    if (!validate_image(*img, &why)) {
        set_error("tb200_create_cached: invalid cache file: " + why);
        return nullptr;
    }
    return create_with(device, [img](tb200_renderer* r) { return upload_image(r, *img); });
}

// The library's one reader of the environment (tb_kernels.cuh: Knobs lists each variable and its parsing)
static Knobs read_knobs()
{
    const auto is = [](const char* value, const char* word) { return value && strcmp(value, word) == 0; };
    const char* cap = getenv("TINSEL_B200_TEST_LAUNCH_SAMPLES");
    const char* sched = getenv("TINSEL_B200_SCHED");
    const char* split = getenv("TINSEL_B200_SPLIT");
    const char* cta = getenv("TINSEL_B200_CTA");
    const char* queues = getenv("TINSEL_B200_QUEUES");
    const char* spec = getenv("TINSEL_B200_SPECIALIZE");
    const char* treelet = getenv("TINSEL_B200_TREELET");
    Knobs k;
    k.mega = is(getenv("TINSEL_B200_PIPELINE"), "mega");
    k.plainReadback = is(getenv("TINSEL_B200_READBACK"), "plain");
    k.launchSamples = cap ? strtoull(cap, nullptr, 10) : 0;
    k.dupDevices = getenv("TINSEL_B200_TEST_DUP_DEVICES") != nullptr;
    k.sched = is(sched, "hard") ? 1 : is(sched, "free") ? 0 : -1;
    k.splitSet = split != nullptr;
    k.split = split ? atoi(split) : 0;
    k.cta = cta ? atoi(cta) : 0;
    k.laneQueues = is(queues, "ring") ? 0 : is(queues, "lanes") ? 2 : 1;
    k.specialize = !(spec && atoi(spec) == 0);
    k.noFlat = getenv("TINSEL_B200_NO_FLAT") != nullptr;
    k.treelet = treelet && atoi(treelet) == 1;
    return k;
}

static tb200_renderer* create_with(int device, const std::function<bool(tb200_renderer*)>& build)
{
    const Knobs knobs = read_knobs();
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
        cudaGetLastError();
        set_error("tb200_create: no CUDA device available (this library has no CPU fallback)");
        return nullptr;
    }
    if (device < 0 || device >= count) {
        set_error("tb200_create: bad device ordinal");
        return nullptr;
    }
    tb200_renderer* r = new tb200_renderer();
    memset(&r->stats, 0, sizeof(r->stats));
    r->device = device;
    r->knobs = knobs;
    if (knobs.launchSamples > 0) r->maxLaunchSamples = std::min(knobs.launchSamples, r->maxLaunchSamples);   // test hook: lowers the cap, never raises it
    bool ok = cudaSetDevice(device) == cudaSuccess;
    cudaDeviceProp prop;
    ok = ok && cudaGetDeviceProperties(&prop, device) == cudaSuccess;
    if (ok) r->numSMs = prop.multiProcessorCount;
    ok = ok && cudaStreamCreateWithFlags(&r->ownStream, cudaStreamNonBlocking) == cudaSuccess;
    r->stream = r->ownStream;
    ok = ok && cudaEventCreate(&r->evStart) == cudaSuccess && cudaEventCreate(&r->evStop) == cudaSuccess;
    if (!ok) {
        set_error(std::string("tb200_create: device setup failed: ") + cudaGetErrorString(cudaGetLastError()));
        delete r;
        return nullptr;
    }
    unsigned int* hostFlags = nullptr;
    // cold slot state for every CTA a launch can have (one or two per SM, see launch_wavefront2): 8 float4 per slot
    ok = dev_alloc(&r->mem.cold, size_t(r->numSMs) * TB_WF2_MAX_CTAS_PER_SM * TB_WF2_SLOTS * 8) == cudaSuccess &&
         dev_alloc(&r->mem.counter, 1) == cudaSuccess && dev_alloc(&r->mem.bandCount, TB_MAX_BANDS) == cudaSuccess &&
         cudaHostAlloc((void**)&hostFlags, TB_MAX_BANDS * sizeof(unsigned int), cudaHostAllocMapped) == cudaSuccess;
    if (ok) r->mem.bandFlags.reset(hostFlags);
    if (!ok || cudaHostGetDevicePointer((void**)&r->dBandFlags, hostFlags, 0) != cudaSuccess ||
        cudaStreamCreateWithFlags(&r->copyStream, cudaStreamNonBlocking) != cudaSuccess) {
        set_error("tb200_create: counter allocation failed");
        tb200_destroy(r);
        return nullptr;
    }
    memset(hostFlags, 0, TB_MAX_BANDS * sizeof(unsigned int));
    if (!build(r)) {
        tb200_destroy(r);
        return nullptr;
    }
    return r;
}

tb200_renderer* tb200_create_multi(const tb200_scene* scene, const int* devices, int numDevices)
{
    if (!devices || numDevices < 1 || numDevices > TB200_MAX_DEVICES) {
        set_error("tb200_create_multi: bad device list");
        return nullptr;
    }
    const bool dupDevices = read_knobs().dupDevices;   // test hook: a one-GPU box
    for (int a = 0; a < numDevices; ++a)
        for (int b = 0; b < a; ++b)
            if (devices[a] == devices[b] && !dupDevices) {
                set_error("tb200_create_multi: a device is listed twice");
                return nullptr;
            }
    // one complete renderer per device (the scene is replicated: SURVEY 8e, at most ~250 MB), built
    // side by side because most of the time is the host-side re-layout of the meshes
    std::vector<tb200_renderer*> members(numDevices, nullptr);
    std::vector<std::string> errors(numDevices);
    {
        std::vector<std::thread> builders;
        for (int k = 0; k < numDevices; ++k)
            builders.emplace_back([&, k] {
                members[k] = tb200_create(scene, devices[k]);
                if (!members[k]) errors[k] = g_error;
            });
        for (std::thread& t : builders) t.join();
    }
    for (int k = 0; k < numDevices; ++k)
        if (!members[k]) {
            set_error("tb200_create_multi: device " + std::to_string(devices[k]) + ": " + errors[k]);
            for (tb200_renderer* m : members) tb200_destroy(m);
            return nullptr;
        }
    tb200_renderer* head = members[0];
    for (int k = 1; k < numDevices; ++k) {
        tb200_renderer* p = members[k];
        head->peers.push_back(p);
        // device-to-device gathers go over NVLink when the pair allows peer access
        int can = 0;
        if (p->device != head->device && cudaDeviceCanAccessPeer(&can, p->device, head->device) == cudaSuccess && can) {
            cudaSetDevice(p->device);
            if (cudaDeviceEnablePeerAccess(head->device, 0) != cudaSuccess) cudaGetLastError();
        }
        p->worker = new Worker();
        p->worker->thread = std::thread(worker_main, p);
    }
    cudaSetDevice(head->device);
    return head;
}

static int init_one(tb200_renderer* r, int width, int height)
{
    cudaSetDevice(r->device);
    const size_t n = size_t(width) * height;
    if (width != r->width || height != r->height || !r->mem.accum) {
        r->mem.radiance.reset();
        r->mem.raster.reset();
        if (dev_alloc(&r->mem.accum, n) != cudaSuccess) {
            set_error("tb200_init: accumulator allocation failed");
            return -1;
        }
        r->width = width;
        r->height = height;
    }
    if (cudaMemsetAsync(r->mem.accum.get(), 0, n * sizeof(float4), r->stream) != cudaSuccess ||
        cudaStreamSynchronize(r->stream) != cudaSuccess) {
        set_error("tb200_init: accumulator clear failed");
        return -1;
    }
    r->frame = 0;
    r->stats.frames = 0;
    r->boundAccum = nullptr;
    r->filteredValid = false;
    return 0;
}

int tb200_init(tb200_renderer* r, int width, int height)
{
    if (!r || width <= 0 || height <= 0) {
        set_error("tb200_init: bad arguments");
        return -1;
    }
    if (!r->peers.empty()) {
        // multi-device: contiguous row slabs cut at tile rows, one per device
        const int n = (int)r->peers.size() + 1;
        r->slabRow0 = 0;
        r->slabRows = slab_cut(height, 1, n);
        for (int k = 1; k < n; ++k) {
            r->peers[k - 1]->slabRow0 = slab_cut(height, k, n);
            r->peers[k - 1]->slabRows = slab_cut(height, k + 1, n) - slab_cut(height, k, n);
        }
    }
    return group_run(r, [=](tb200_renderer* m) { return init_one(m, width, height); });
}

static bool render_one(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options, float* output)
{
    cudaSetDevice(r->device);
    LaunchParams P;
    if (!fill_params(r, camera, options, &P)) return false;
    if (options->mode == TB200_MODE_NORMALS) {
        unsigned long long launches = 0;
        if (r->slabRows >= 0) {
            // eNormals writes each pixel from its own primary ray: the owned rows, no halo
            P.firstRow = P.film.rowLo;
            P.numRows = P.film.rowHi - P.film.rowLo;
            finalize_params(&P);
        }
        TB_CUDA(cudaEventRecord(r->evStart, r->stream));
        launch_normals(P, r->stream, &launches);
        TB_CUDA(cudaEventRecord(r->evStop, r->stream));
        TB_CUDA(cudaGetLastError());
        r->stats.kernelLaunches += launches;
        return read_back(r, output) && sync_gpu_ms(r);
    }
    if (!run_frames(r, P, 1, output)) return false;
    // The tuner compares launchSamples with stats.gpuMs.  tb200_render_n does not call it: with a streamed read-back
    // its gpuMs spans the launch of the first n - 1 frames and the last frame's launch, while launchSamples counts
    // only the last frame's launch.
    tune_update(r);
    return true;
}

int tb200_render(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options, float* output)
{
    if (!r || !camera || !options || !output) {
        set_error("tb200_render: null argument");
        return -1;
    }
    if (options->mode == TB200_MODE_COMPLEXITY) return 0;   // render.cpp:516-519
    // every device traces its slab and streams its own rows into `output` over its own PCIe link
    return group_run(r, [=](tb200_renderer* m) { return render_one(m, camera, options, output) ? 0 : -1; });
}

static int render_device_one(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options, int spp,
                             int firstRow, int numRows)
{
    cudaSetDevice(r->device);
    if (options->mode != TB200_MODE_PATHTRACE) {
        set_error("tb200_render_device: only ePathTrace is batched");
        return -1;
    }
    LaunchParams P;
    if (!fill_params(r, camera, options, &P)) return -1;
    if (numRows >= 0) {
        if (r->slabRows >= 0) {
            set_error("tb200_render_device: a row range cannot be combined with a row slab (tb200_set_slab / multi-device)");
            return -1;
        }
        if (firstRow < 0 || firstRow + numRows > options->height) {
            set_error("tb200_render_device: row range outside the image");
            return -1;
        }
        P.firstRow = firstRow;
        P.numRows = numRows;
        finalize_params(&P);
    }
    if (spp == 0 || P.numRows <= 0) {   // nothing to trace: the frames count, stats.gpuMs keeps the last launch's time
        r->frame += spp;
        r->stats.frames += spp;
        return 0;
    }
    if (!run_frames(r, P, spp, nullptr)) return -1;
    tune_update(r);
    return 0;
}

int tb200_render_device(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options, int spp,
                        int firstRow, int numRows)
{
    if (!r || !camera || !options || spp < 0) {
        set_error("tb200_render_device: bad argument");
        return -1;
    }
    return group_run(r, [=](tb200_renderer* m) { return render_device_one(m, camera, options, spp, firstRow, numRows); });
}

#define TB_SINGLE_DEVICE_ONLY(r, what)                                                              \
    if (!(r)->peers.empty()) {                                                                      \
        set_error(what ": not available on a multi-device renderer");                               \
        return -1;                                                                                  \
    }

int tb200_set_shard(tb200_renderer* r, int shard, int numShards)
{
    if (!r || numShards < 1 || shard < 0 || shard >= numShards) {
        set_error("tb200_set_shard: bad arguments");
        return -1;
    }
    TB_SINGLE_DEVICE_ONLY(r, "tb200_set_shard")
    r->shard = shard;
    r->numShards = numShards;
    return 0;
}

int tb200_set_stream(tb200_renderer* r, void* cudaStream, int external)
{
    if (!r) {
        set_error("tb200_set_stream: null renderer");
        return -1;
    }
    TB_SINGLE_DEVICE_ONLY(r, "tb200_set_stream")
    cudaSetDevice(r->device);
    cudaStreamSynchronize(r->stream);
    // handle 0 with external != 0 is CUDA's legacy default stream, a perfectly good caller stream
    r->stream = external ? (cudaStream_t)cudaStream : r->ownStream;
    return 0;
}

int tb200_set_slab(tb200_renderer* r, int firstRow, int numRows)
{
    if (!r || (numRows >= 0 && firstRow < 0)) {
        set_error("tb200_set_slab: bad arguments");
        return -1;
    }
    TB_SINGLE_DEVICE_ONLY(r, "tb200_set_slab")
    if (numRows >= 0 && r->numShards > 1) {
        set_error("tb200_set_slab: cannot be combined with tb200_set_shard");
        return -1;
    }
    r->slabRow0 = numRows >= 0 ? firstRow : 0;
    r->slabRows = numRows >= 0 ? numRows : -1;
    return 0;
}

int tb200_pin_output(tb200_renderer* r, float* output, size_t bytes)
{
    if (!r || !output || bytes == 0) {
        set_error("tb200_pin_output: bad arguments");
        return -1;
    }
    cudaSetDevice(r->device);
    if (r->registered == output && r->registeredBytes == bytes) return 0;
    if (r->registered) tb200_unpin_output(r);
    // portable: every device of a multi-device renderer copies its rows straight into this buffer
    if (cudaHostRegister(output, bytes, cudaHostRegisterPortable) != cudaSuccess) {
        set_error(std::string("tb200_pin_output: cudaHostRegister: ") + cudaGetErrorString(cudaGetLastError()));
        return -1;
    }
    r->registered = output;
    r->registeredBytes = bytes;
    return 0;
}

int tb200_unpin_output(tb200_renderer* r)
{
    if (!r) return -1;
    if (r->registered) {
        cudaSetDevice(r->device);
        cudaHostUnregister(r->registered);
        cudaGetLastError();
        r->registered = nullptr;
        r->registeredBytes = 0;
    }
    return 0;
}

int tb200_bind_accumulator(tb200_renderer* r, float* deviceAccum)
{
    if (!r || !r->mem.accum) {
        set_error("tb200_bind_accumulator: call tb200_init first");
        return -1;
    }
    TB_SINGLE_DEVICE_ONLY(r, "tb200_bind_accumulator")
    r->boundAccum = (float4*)deviceAccum;
    return 0;
}

float* tb200_device_accumulator(tb200_renderer* r)
{
    if (!r) return nullptr;
    return (float*)(r->boundAccum ? r->boundAccum : r->mem.accum.get());
}

int tb200_read_accumulator(tb200_renderer* r, float* output)
{
    if (!r || !output || !r->mem.accum) {
        set_error("tb200_read_accumulator: bad argument");
        return -1;
    }
    return group_run(r, [=](tb200_renderer* m) {
        cudaSetDevice(m->device);
        return read_back(m, output) ? 0 : -1;
    });
}

int tb200_gather_device(tb200_renderer* r)
{
    if (!r || !r->mem.accum) {
        set_error("tb200_gather_device: call tb200_init first");
        return -1;
    }
    // every peer's slab -> the head's accumulator, device to device (NVLink when peer access is on)
    const size_t rowBytes = size_t(r->width) * sizeof(float4);
    for (tb200_renderer* p : r->peers) {
        int row0, row1;
        owned_rows(p, &row0, &row1);
        if (row1 <= row0) continue;
        cudaSetDevice(p->device);
        if (cudaMemcpyPeerAsync((char*)r->mem.accum.get() + size_t(row0) * rowBytes, r->device, (const char*)p->mem.accum.get() + size_t(row0) * rowBytes,
                                p->device, size_t(row1 - row0) * rowBytes, p->stream) != cudaSuccess) {
            set_error(std::string("tb200_gather_device: ") + cudaGetErrorString(cudaGetLastError()));
            return -1;
        }
    }
    for (tb200_renderer* p : r->peers) {
        cudaSetDevice(p->device);
        if (cudaStreamSynchronize(p->stream) != cudaSuccess) {
            set_error(std::string("tb200_gather_device: ") + cudaGetErrorString(cudaGetLastError()));
            return -1;
        }
    }
    cudaSetDevice(r->device);
    return 0;
}

int tb200_num_devices(const tb200_renderer* r) { return r ? (int)r->peers.size() + 1 : 0; }

void tb200_slab_rows(int height, int member, int numMembers, int* firstRow, int* numRows)
{
    if (numMembers < 1) numMembers = 1;
    member = std::max(0, std::min(member, numMembers - 1));
    const int a = slab_cut(std::max(0, height), member, numMembers), b = slab_cut(std::max(0, height), member + 1, numMembers);
    if (firstRow) *firstRow = a;
    if (numRows) *numRows = b - a;
}

void tb200_slab_traced_rows(int height, int firstRow, int numRows, float filterWidth, int* firstTraced, int* numTraced)
{
    const int reach = filter_reach(filterWidth);
    const int lo = std::max(0, std::min(firstRow, height)), hi = std::max(lo, std::min(firstRow + std::max(0, numRows), height));
    const int t0 = std::max(0, lo - reach);
    if (firstTraced) *firstTraced = t0;
    if (numTraced) *numTraced = hi > lo ? std::min(height, hi + reach) - t0 : 0;
}

void tb200_divisor_magic(unsigned int d, unsigned int* mul, unsigned int* shift)
{
    uint32_t m = 0, l = 0;
    divisor_magic(d, &m, &l);
    if (mul) *mul = m;
    if (shift) *shift = l;
}

static int render_n_one(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options, int n, float* output)
{
    cudaSetDevice(r->device);
    LaunchParams P;
    return fill_params(r, camera, options, &P) && run_frames(r, P, n, output) ? 0 : -1;
}

int tb200_render_n(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options, int n, float* output)
{
    if (!r || !camera || !options || !output || n < 1) {
        set_error("tb200_render_n: bad argument");
        return -1;
    }
    if (options->mode != TB200_MODE_PATHTRACE) {
        set_error("tb200_render_n: only ePathTrace is batched");
        return -1;
    }
    return group_run(r, [=](tb200_renderer* m) { return render_n_one(m, camera, options, n, output); });
}

int tb200_finish(tb200_renderer* r, float exposure, float limit, float* filtered, unsigned char* rgb8)
{
    (void)limit;   // ToneMap's filmic branch ignores it (util.h:25-42), kept for the call shape of main.cpp:269
    if (!r || !r->mem.accum) {
        set_error("tb200_finish: tb200_init has not been called");
        return -1;
    }
    if (!r->peers.empty() && tb200_gather_device(r) != 0) return -1;   // the finish step runs on the head device
    cudaSetDevice(r->device);
    const int W = r->width, H = r->height;
    const size_t n = size_t(W) * H;
    const size_t rgbBytes = ((n + 3) / 4) * 12;
    if (r->finishWidth != W || r->finishHeight != H) {
        r->mem.means.reset();
        r->mem.denoised.reset();
        r->ditherReady = false;
        r->filteredValid = false;
        r->finishWidth = r->finishHeight = 0;
        if (dev_alloc(&r->mem.filtered, n) != cudaSuccess || dev_alloc(&r->mem.rgb8, rgbBytes) != cudaSuccess ||
            dev_alloc(&r->mem.dither, n) != cudaSuccess) {
            set_error("tb200_finish: buffer allocation failed");
            return -1;
        }
        r->finishWidth = W;
        r->finishHeight = H;
    }
    if (rgb8 && !r->ditherReady) {
        // WritePng (png.cpp:329-343) draws its dither from one sequential Random(): six draws per pixel
        // in pixel order.  The stream does not depend on the image, so the state in front of every
        // pixel is tabulated once per image size and the kernel continues from there.
        std::vector<uint2> states(n);
        uint32_t s1 = 315645664u, s2 = s1 ^ 0x13ab45feu;   // Random(0), maths.h:1041-1045
        for (size_t i = 0; i < n; ++i) {
            states[i] = make_uint2(s1, s2);
            for (int k = 0; k < 6; ++k) {
                const uint32_t a = s1, b = s2;
                s1 = (b ^ ((a << 5) | (a >> 27))) ^ (a * b);
                s2 = s1 ^ ((b << 12) | (b >> 20));
            }
        }
        if (cudaMemcpyAsync(r->mem.dither.get(), states.data(), n * sizeof(uint2), cudaMemcpyHostToDevice, r->stream) != cudaSuccess ||
            cudaStreamSynchronize(r->stream) != cudaSuccess) {
            set_error("tb200_finish: dither table upload failed");
            return -1;
        }
        r->stats.h2dBytes += n * sizeof(uint2);
        r->ditherReady = true;
    }
    FinishParams F;
    F.accum = r->boundAccum ? r->boundAccum : r->mem.accum.get();
    F.numPixels = (int)n;
    F.exposure = exposure;
    F.filtered = r->mem.filtered.get();   // always kept on the device: tb200_nlm reads it
    F.rgb8 = rgb8 ? r->mem.rgb8.get() : nullptr;
    F.ditherState = r->mem.dither.get();
    unsigned long long launches = 0;
    cudaEventRecord(r->evStart, r->stream);
    launch_finish(F, r->stream, &launches);
    cudaEventRecord(r->evStop, r->stream);
    r->stats.kernelLaunches += launches;
    bool ok = cudaGetLastError() == cudaSuccess;
    if (ok && filtered) {
        ok = cudaMemcpyAsync(filtered, r->mem.filtered.get(), n * sizeof(float4), cudaMemcpyDeviceToHost, r->stream) == cudaSuccess;
        r->stats.d2hBytes += n * sizeof(float4);
    }
    if (ok && rgb8) {
        ok = cudaMemcpyAsync(rgb8, r->mem.rgb8.get(), n * 3, cudaMemcpyDeviceToHost, r->stream) == cudaSuccess;
        r->stats.d2hBytes += n * 3;
    }
    ok = ok && cudaStreamSynchronize(r->stream) == cudaSuccess;
    if (!ok) {
        set_error(std::string("tb200_finish: ") + cudaGetErrorString(cudaGetLastError()));
        return -1;
    }
    r->filteredValid = true;
    return sync_gpu_ms(r) ? 0 : -1;
}

int tb200_nlm(tb200_renderer* r, float falloff, int radius, float* out)
{
    if (!r || !out || radius < 0) {
        set_error("tb200_nlm: bad argument");
        return -1;
    }
    if (!r->filteredValid || r->finishWidth != r->width || r->finishHeight != r->height) {
        set_error("tb200_nlm: tb200_finish has not produced an image since the last tb200_init");
        return -1;
    }
    cudaSetDevice(r->device);
    const size_t n = size_t(r->width) * r->height;
    if (!r->mem.means || !r->mem.denoised) {
        if (dev_alloc(&r->mem.means, n) != cudaSuccess || dev_alloc(&r->mem.denoised, n) != cudaSuccess) {
            set_error("tb200_nlm: buffer allocation failed");
            return -1;
        }
    }
    NlmParams N;
    N.in = r->mem.filtered.get();
    N.means = r->mem.means.get();
    N.out = r->mem.denoised.get();
    N.width = r->width;
    N.height = r->height;
    N.radius = radius;
    N.falloff = falloff;
    unsigned long long launches = 0;
    cudaEventRecord(r->evStart, r->stream);
    launch_nlm(N, r->stream, &launches);
    cudaEventRecord(r->evStop, r->stream);
    r->stats.kernelLaunches += launches;
    if (cudaGetLastError() != cudaSuccess ||
        cudaMemcpyAsync(out, r->mem.denoised.get(), n * sizeof(float4), cudaMemcpyDeviceToHost, r->stream) != cudaSuccess ||
        cudaStreamSynchronize(r->stream) != cudaSuccess) {
        set_error(std::string("tb200_nlm: ") + cudaGetErrorString(cudaGetLastError()));
        return -1;
    }
    r->stats.d2hBytes += n * sizeof(float4);
    return sync_gpu_ms(r) ? 0 : -1;
}

int tb200_trace_frame(tb200_renderer* r, const tb200_camera* camera, const tb200_options* options, int frame,
                      float* radiance, float* raster)
{
    if (!r || !camera || !options || !radiance || !raster) {
        set_error("tb200_trace_frame: null argument");
        return -1;
    }
    cudaSetDevice(r->device);
    LaunchParams P;
    {
        // a probe of the whole frame on this device, whatever slab it owns when rendering
        const int slabRows = r->slabRows;
        r->slabRows = -1;
        const bool ok = fill_params(r, camera, options, &P);
        r->slabRows = slabRows;
        if (!ok) return -1;
    }
    const size_t n = size_t(r->width) * r->height;
    if (!r->mem.radiance || !r->mem.raster) {
        if (dev_alloc(&r->mem.radiance, n * 3) != cudaSuccess || dev_alloc(&r->mem.raster, n * 2) != cudaSuccess) {
            set_error("tb200_trace_frame: scratch allocation failed");
            return -1;
        }
    }
    P.frame0 = frame;
    P.numFrames = 1;
    P.outRadiance = r->mem.radiance.get();
    P.outRaster = r->mem.raster.get();
    // pixels of other shards (tb200_set_shard) are not traced by this renderer: they read back as zero
    if (cudaMemsetAsync(P.outRadiance, 0, n * 3 * sizeof(float), r->stream) != cudaSuccess ||
        cudaMemsetAsync(P.outRaster, 0, n * 2 * sizeof(float), r->stream) != cudaSuccess) {
        set_error("tb200_trace_frame: scratch clear failed");
        return -1;
    }
    const uint64_t samplesBefore = r->stats.samples;
    if (!launch_frames(r, P)) return -1;
    r->stats.samples = samplesBefore;
    if (cudaMemcpyAsync(radiance, P.outRadiance, n * 3 * sizeof(float), cudaMemcpyDeviceToHost, r->stream) != cudaSuccess ||
        cudaMemcpyAsync(raster, P.outRaster, n * 2 * sizeof(float), cudaMemcpyDeviceToHost, r->stream) != cudaSuccess ||
        cudaStreamSynchronize(r->stream) != cudaSuccess) {
        set_error(std::string("tb200_trace_frame: ") + cudaGetErrorString(cudaGetLastError()));
        return -1;
    }
    r->stats.d2hBytes += n * 5 * sizeof(float);
    return 0;
}

// cuMemGetAddressRange (driver API), reached through the runtime so that the library needs no -lcuda
typedef int (*MemRangeFn)(unsigned long long* base, size_t* size, unsigned long long ptr);

static MemRangeFn mem_range_fn()
{
    static MemRangeFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult status = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &p, cudaEnableDefault, &status) != cudaSuccess ||
            status != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            p = nullptr;
        }
        return (MemRangeFn)p;
    }();
    return fn;
}

// `bytes` from `ptr` lie inside one allocation of device memory on r's device
static bool check_device_span(const char* entry, const tb200_renderer* r, const void* ptr, size_t bytes, size_t align, const char* what)
{
    const std::string name = std::string(entry) + ": " + what;
    if (!ptr) return set_error(name + " is null");
    if ((uintptr_t)ptr % align != 0) return set_error(name + " is not aligned to " + std::to_string(align) + " bytes");
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, ptr) != cudaSuccess) {
        cudaGetLastError();
        return set_error(name + " is not a CUDA pointer");
    }
    if (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged)
        return set_error(name + " is not device memory (host memory is not accepted)");
    if (attr.device != r->device)
        return set_error(name + " lies on device " + std::to_string(attr.device) + ", not on the renderer's device " + std::to_string(r->device));
    const MemRangeFn range = mem_range_fn();
    if (!range) return set_error(std::string(entry) + ": cuMemGetAddressRange is not available from the driver");
    unsigned long long base = 0;
    size_t size = 0;
    if (range(&base, &size, (unsigned long long)(uintptr_t)ptr) != 0) return set_error(name + ": the driver knows no allocation at this address");
    const unsigned long long p = (unsigned long long)(uintptr_t)ptr;
    if (bytes > size || p - base > size - bytes)
        return set_error(name + ": " + std::to_string(bytes) + " bytes from this address run past the end of its allocation");
    return true;
}

// One output of a ray query, as the caller passed it: checked by check_device_span for numRays records
struct QuerySpan {
    const void* ptr;
    size_t bytesPerRay;
    size_t align;
    const char* what;   // its name in refusals
};

// Every ray query: checks the renderer, the ray count, the rays and then the outputs in the order given (the first
// refusal sets the error), makes the renderer's device current, runs the query's kernel on r's stream with Q's
// outputs, waits for it and sets stats.gpuMs to its time.  No rays: returns 0 before the pointers are checked.
static int run_query(const char* entry, tb200_renderer* r, QueryKind kind, const tb200_ray* rays, int64_t numRays,
                     std::initializer_list<QuerySpan> outputs, QueryParams Q)
{
    auto fail = [&](const std::string& why) {
        set_error(std::string(entry) + ": " + why);
        return -1;
    };
    if (!r) return fail("null renderer");
    if (numRays < 0 || numRays > (int64_t)(SIZE_MAX / sizeof(tb200_ray)))
        return fail("numRays " + std::to_string((long long)numRays) + " is out of range");
    if (numRays == 0) return 0;
    cudaSetDevice(r->device);   // a multi-device renderer answers on its head, which holds a full copy of the scene
    const size_t n = (size_t)numRays;
    if (!check_device_span(entry, r, rays, n * sizeof(tb200_ray), 16, "rays")) return -1;
    for (const QuerySpan& s : outputs)
        if (!check_device_span(entry, r, s.ptr, n * s.bytesPerRay, s.align, s.what)) return -1;
    Q.scene = r->scene;
    Q.rays = reinterpret_cast<const float4*>(rays);
    Q.numRays = numRays;
    Q.counter = r->mem.counter.get();   // the wavefront's work counter: free between launches on this stream

    unsigned long long launches = 0;
    if (cudaEventRecord(r->evStart, r->stream) != cudaSuccess) return fail(cudaGetErrorString(cudaGetLastError()));
    launch_query(kind, Q, r->numSMs, r->stream, &launches);
    r->stats.kernelLaunches += launches;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaEventRecord(r->evStop, r->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(r->stream);
    if (e != cudaSuccess) return fail(cudaGetErrorString(e));
    return sync_gpu_ms(r) ? 0 : -1;
}

static_assert(sizeof(tb200_ray) == 32 && sizeof(tb200_hit) == 16, "the query kernels read two float4 per ray and write one hit");
static_assert(sizeof(tb200_tri_hit) == 16, "the query kernel writes one int4 per triangle record");

int tb200_trace_rays(tb200_renderer* r, const tb200_ray* rays, tb200_hit* hits, int32_t* prims, int64_t numRays)
{
    QueryParams Q = {};
    Q.hits = reinterpret_cast<float4*>(hits);
    Q.prims = prims;
    return run_query("tb200_trace_rays", r, QueryKind::Closest, rays, numRays,
                     {{hits, sizeof(tb200_hit), 16, "hits"}, {prims, sizeof(int32_t), 4, "prims"}}, Q);
}

int tb200_occluded_rays(tb200_renderer* r, const tb200_ray* rays, uint8_t* occluded, int64_t numRays)
{
    QueryParams Q = {};
    Q.occluded = occluded;
    return run_query("tb200_occluded_rays", r, QueryKind::Occluded, rays, numRays, {{occluded, 1, 1, "occluded"}}, Q);
}

int tb200_trace_rays_tri(tb200_renderer* r, const tb200_ray* rays, tb200_hit* hits, int32_t* prims, tb200_tri_hit* tris, int64_t numRays)
{
    QueryParams Q = {};
    Q.hits = reinterpret_cast<float4*>(hits);
    Q.prims = prims;
    Q.tris = reinterpret_cast<int4*>(tris);
    return run_query("tb200_trace_rays_tri", r, QueryKind::ClosestTri, rays, numRays,
                     {{hits, sizeof(tb200_hit), 16, "hits"}, {prims, sizeof(int32_t), 4, "prims"},
                      {tris, sizeof(tb200_tri_hit), 16, "tris"}}, Q);
}

#ifdef TB_WF2_STAGE_CLOCKS
// development builds only (-DTB_WF2_STAGE_CLOCKS, tools/stage_clocks.py): copies the lane-owned wavefront
// layout's per-stage cycle counters of the current device into out[0..n) (n >= 15 words, see wf2_lanes.cuh:
// Wf2Clocks) after the work queued so far has finished, and zeroes them when `reset` is set
int tb200_stage_clocks(unsigned long long* out, int n, int reset)
{
    if (!out || n < TB_WF2_STAGE_CLOCK_WORDS) {
        set_error("tb200_stage_clocks: need room for 18 counters");
        return -1;
    }
    if (cudaDeviceSynchronize() != cudaSuccess) {
        set_error(std::string("tb200_stage_clocks: ") + cudaGetErrorString(cudaGetLastError()));
        return -1;
    }
    read_stage_clocks(out, reset != 0);
    return TB_WF2_STAGE_CLOCK_WORDS;
}
#endif

void tb200_set_frame(tb200_renderer* r, int frame)
{
    if (!r) return;
    r->frame = frame;
    for (tb200_renderer* p : r->peers) p->frame = frame;
}

void tb200_get_stats(tb200_renderer* r, tb200_stats* out)
{
    if (!r || !out) return;
    *out = r->stats;
    for (const tb200_renderer* p : r->peers) {
        out->samples += p->stats.samples;
        out->kernelLaunches += p->stats.kernelLaunches;
        out->d2hBytes += p->stats.d2hBytes;
        out->h2dBytes += p->stats.h2dBytes;
        out->gpuMs = std::max(out->gpuMs, p->stats.gpuMs);
    }
}

const char* tb200_last_kernel(tb200_renderer* r)
{
    return r ? r->lastKernel : "";
}

int tb200_get_member_stats(tb200_renderer* r, int member, tb200_stats* out, int* firstRow, int* numRows)
{
    if (!r || !out || member < 0 || member > (int)r->peers.size()) {
        set_error("tb200_get_member_stats: bad argument");
        return -1;
    }
    const tb200_renderer* m = member == 0 ? r : r->peers[member - 1];
    *out = m->stats;
    int row0, row1;
    owned_rows(m, &row0, &row1);
    if (firstRow) *firstRow = row0;
    if (numRows) *numRows = row1 - row0;
    return 0;
}

void tb200_destroy(tb200_renderer* r)
{
    if (!r) return;
    for (tb200_renderer* p : r->peers) tb200_destroy(p);
    r->peers.clear();
    if (r->worker) {
        {
            std::lock_guard<std::mutex> guard(r->worker->lock);
            r->worker->quit.store(true, std::memory_order_release);
        }
        r->worker->posted.fetch_add(1, std::memory_order_release);   // leave the spin, see `quit`
        r->worker->wake.notify_one();
        if (r->worker->thread.joinable()) r->worker->thread.join();
        delete r->worker;
        r->worker = nullptr;
    }
    tb200_unpin_output(r);
    cudaSetDevice(r->device);
    if (r->stream) cudaStreamSynchronize(r->stream);
    r->mem = tb200_renderer::Memory();
    r->stream = r->ownStream;
    if (r->evStart) cudaEventDestroy(r->evStart);
    if (r->evStop) cudaEventDestroy(r->evStop);
    if (r->stream) cudaStreamDestroy(r->stream);
    if (r->copyStream) cudaStreamDestroy(r->copyStream);
    delete r;
}

}  // extern "C"
