// bvh_build.cu -- mesh BVH construction on the GPU (SURVEY.md 8f rank 3).
//
// Replaces, for triangle meshes, the reference's host-side builder: Mesh::RebuildBVH
// (src/mesh.cpp:314-338: one Bounds per triangle, AddPoint x 3) + BVHBuilder::Build
// (src/bvh.h:30-263: recursive full-sweep SAH, std::sort per node, one item per leaf; 1.33 s for
// ajax's 544 566 triangles on one host core).  Output is the reference's own node format
// (BVHNode, bvh.h:9-19: 32 bytes, bounds + leftIndex + rightIndex:31/leaf:1, leaf.leftIndex = triangle)
// with the root at index 0, one triangle per leaf, 2n-1 nodes -- so it drops into tb200_mesh::nodes,
// into the reference's own IntersectRayMesh, and into the .bin mesh cache (tb200_mesh_bin_save).
//
// Algorithm: PLOC -- parallel locally-ordered clustering (Meister & Bittner 2018) -- an agglomerative
// builder whose trees are on a par with top-down SAH builds:
//   1. triangle bounds + centroid bounds (one reduction), 30-bit Morton codes, radix sort;
//   2. clusters = the leaves in Morton order; repeat until one cluster is left:
//        a. every cluster looks at its PLOC_RADIUS neighbours on either side and picks the one whose
//           merged box has the smallest surface area;
//        b. mutual nearest neighbours merge into a new interior node (kept at the lower position);
//        c. the cluster array is compacted (prefix sum).
//      About 40 % of the clusters merge per round: ~30 rounds for half a million triangles.
//   3. interior nodes are renumbered so that the root is node 0 (creation order reversed), leaves
//      follow: node n-1+i is the leaf of triangle i.
// Node boxes are exact unions of triangle boxes (fp32 min/max: order-independent), as the reference's.
//
// Parity: a different tree is a different -- equally valid -- input to the same traversal.  Visit
// order changes, so only exact ties in t between two triangles can be resolved differently from the
// reference's tree; the criterion (tests/test_bvh_build.py) is therefore: hand the GPU-built tree to
// the oracle as the mesh's BVH and compare per sample, bit for bit, on that same tree.
#include <algorithm>
#include <cfloat>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "tinsel_b200.h"

namespace {

#define PLOC_RADIUS 16
#define PLOC_BLOCK 256

struct Box {
    float lo[3], hi[3];
};

__device__ __forceinline__ Box box_union(const Box& a, const Box& b)
{
    Box r;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        r.lo[k] = fminf(a.lo[k], b.lo[k]);
        r.hi[k] = fmaxf(a.hi[k], b.hi[k]);
    }
    return r;
}

__device__ __forceinline__ float box_area(const Box& b)
{
    const float ex = b.hi[0] - b.lo[0], ey = b.hi[1] - b.lo[1], ez = b.hi[2] - b.lo[2];
    return ex * ey + ey * ez + ez * ex;   // half the surface area: a monotone proxy
}

// Build-time node: box + children as BUILD ids (leaf i = i, interior c = numTris + c)
struct BuildNode {
    Box box;
    int left, right;
};

__device__ __forceinline__ void atomic_min_float(float* addr, float v)
{
    // bounds are finite: order-preserving integer views
    if (v >= 0.0f) atomicMin((int*)addr, __float_as_int(v));
    else atomicMax((unsigned int*)addr, __float_as_uint(v));
}
__device__ __forceinline__ void atomic_max_float(float* addr, float v)
{
    if (v >= 0.0f) atomicMax((int*)addr, __float_as_int(v));
    else atomicMin((unsigned int*)addr, __float_as_uint(v));
}

// Mesh::RebuildBVH's triangleBounds (mesh.cpp:320-331) + the box of the centroids
__global__ void k_tri_bounds(const float* __restrict__ positions, const int* __restrict__ indices, int numTris, BuildNode* nodes,
                             float* centroidBox /* lo[3], hi[3] */)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float c[3] = {0.0f, 0.0f, 0.0f};
    const bool live = i < numTris;
    if (live) {
        Box b;
        const int i0 = indices[i * 3 + 0], i1 = indices[i * 3 + 1], i2 = indices[i * 3 + 2];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float a = positions[(size_t)i0 * 3 + k], bb = positions[(size_t)i1 * 3 + k], cc = positions[(size_t)i2 * 3 + k];
            b.lo[k] = fminf(a, fminf(bb, cc));
            b.hi[k] = fmaxf(a, fmaxf(bb, cc));
            c[k] = 0.5f * (b.lo[k] + b.hi[k]);
        }
        nodes[i].box = b;
        nodes[i].left = i;
        nodes[i].right = -1;
    }
    // block reduction of the centroid box, one atomic per block and component
    typedef cub::BlockReduce<float, PLOC_BLOCK> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float lo = Reduce(tmp).Reduce(live ? c[k] : FLT_MAX, cub::Min());
        __syncthreads();
        const float hi = Reduce(tmp).Reduce(live ? c[k] : -FLT_MAX, cub::Max());
        __syncthreads();
        if (threadIdx.x == 0) {
            atomic_min_float(&centroidBox[k], lo);
            atomic_max_float(&centroidBox[3 + k], hi);
        }
    }
}

__device__ __forceinline__ unsigned int expand_bits10(unsigned int v)
{
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}

__global__ void k_morton(const BuildNode* nodes, int numTris, const float* centroidBox, unsigned int* keys, int* values)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= numTris) return;
    unsigned int code = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float lo = centroidBox[k], hi = centroidBox[3 + k];
        const float c = 0.5f * (nodes[i].box.lo[k] + nodes[i].box.hi[k]);
        const float ext = hi - lo;
        float u = ext > 0.0f ? (c - lo) / ext : 0.0f;
        u = fminf(fmaxf(u * 1024.0f, 0.0f), 1023.0f);
        code |= expand_bits10((unsigned int)u) << (2 - k);
    }
    keys[i] = code;
    values[i] = i;
}

// 2a: nearest neighbour within PLOC_RADIUS positions (ties: the lower position), one thread per cluster;
// the block stages its window of boxes in shared memory
__global__ void k_nearest(const int* __restrict__ clusters, int count, const BuildNode* __restrict__ nodes, int* __restrict__ nearest)
{
    __shared__ Box sbox[PLOC_BLOCK + 2 * PLOC_RADIUS];
    const int base = blockIdx.x * PLOC_BLOCK - PLOC_RADIUS;
    for (int k = threadIdx.x; k < PLOC_BLOCK + 2 * PLOC_RADIUS; k += PLOC_BLOCK) {
        const int j = base + k;
        if (j >= 0 && j < count) sbox[k] = nodes[clusters[j]].box;
    }
    __syncthreads();
    const int i = blockIdx.x * PLOC_BLOCK + threadIdx.x;
    if (i >= count) return;
    const Box me = sbox[threadIdx.x + PLOC_RADIUS];
    float best = FLT_MAX;
    int bestJ = -1;
    for (int dj = -PLOC_RADIUS; dj <= PLOC_RADIUS; ++dj) {
        const int j = i + dj;
        if (dj == 0 || j < 0 || j >= count) continue;
        const float a = box_area(box_union(me, sbox[threadIdx.x + PLOC_RADIUS + dj]));
        if (a < best) {
            best = a;
            bestJ = j;
        }
    }
    nearest[i] = bestJ;
}

// 2b: mutual nearest neighbours merge; the lower position keeps the new node, the upper one is vacated
__global__ void k_merge(int* clusters, int count, BuildNode* nodes, const int* nearest, int numTris, int* interiorCount, int* valid)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const int j = nearest[i];
    int keep = 1;
    if (j >= 0 && nearest[j] == i) {
        if (i < j) {
            const int c = atomicAdd(interiorCount, 1);
            const int a = clusters[i], b = clusters[j];
            BuildNode n;
            n.box = box_union(nodes[a].box, nodes[b].box);
            n.left = a;
            n.right = b;
            nodes[numTris + c] = n;
            clusters[i] = numTris + c;
        } else {
            keep = 0;
        }
    }
    valid[i] = keep;
}

// 2c: compaction with the exclusive prefix sum of `valid`
__global__ void k_compact(const int* clustersIn, const int* valid, const int* offset, int count, int* clustersOut)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    if (valid[i]) clustersOut[offset[i]] = clustersIn[i];
}

// 3: build ids -> reference node indices.  Interior c (creation order) -> numInterior-1-c, so the root,
// created last, is node 0; leaf of triangle i -> numInterior + i.
__global__ void k_emit(const BuildNode* nodes, int numTris, int numInterior, tb200_bvh_node* out)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= numTris + numInterior) return;
    const BuildNode n = nodes[k];
    tb200_bvh_node o;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        o.lower[a] = n.box.lo[a];
        o.upper[a] = n.box.hi[a];
    }
    if (k < numTris) {
        o.left = (uint32_t)k;                 // leaf: the triangle
        o.right_leaf = 0x80000000u;
        out[numInterior + k] = o;
    } else {
        auto map = [&](int id) -> uint32_t { return id < numTris ? (uint32_t)(numInterior + id) : (uint32_t)(numInterior - 1 - (id - numTris)); };
        o.left = map(n.left);
        o.right_leaf = map(n.right) & 0x7fffffffu;
        out[numInterior - 1 - (k - numTris)] = o;
    }
}

thread_local std::string g_buildError;

bool fail(const std::string& what)
{
    g_buildError = what;
    fprintf(stderr, "[tinsel_b200] tb200_bvh_build: %s\n", what.c_str());
    return false;
}

#define BB_CUDA(call)                                                              \
    do {                                                                           \
        cudaError_t e_ = (call);                                                   \
        if (e_ != cudaSuccess) {                                                   \
            fail(std::string(#call) + ": " + cudaGetErrorString(e_));              \
            return false;                                                          \
        }                                                                          \
    } while (0)

struct DeviceBuffers {
    std::vector<void*> ptrs;
    ~DeviceBuffers()
    {
        for (void* p : ptrs) cudaFree(p);
    }
    template <typename T>
    bool alloc(T** p, size_t n)
    {
        *p = nullptr;
        if (cudaMalloc((void**)p, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return false;
        ptrs.push_back(*p);
        return true;
    }
};

bool build_on_device(const float* positions, int numVertices, const int32_t* indices, int numIndices, tb200_bvh_node* outNodes,
                     int device, tb200_bvh_build_info* info)
{
    const int numTris = numIndices / 3;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
        cudaGetLastError();
        return fail("no CUDA device available (this library has no CPU fallback)");
    }
    if (device < 0 || device >= count) return fail("bad device ordinal");
    BB_CUDA(cudaSetDevice(device));
    cudaStream_t stream;
    BB_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    struct StreamGuard {
        cudaStream_t s;
        ~StreamGuard() { cudaStreamDestroy(s); }
    } guard{stream};
    cudaEvent_t ev0, ev1;
    BB_CUDA(cudaEventCreate(&ev0));
    BB_CUDA(cudaEventCreate(&ev1));

    DeviceBuffers mem;
    float *dPos, *dCentroidBox;
    int *dIdx, *dClustersA, *dClustersB, *dValues, *dNearest, *dValid, *dOffset, *dInterior;
    unsigned int *dKeys, *dKeysSorted;
    BuildNode* dNodes;
    tb200_bvh_node* dOut;
    const size_t n = (size_t)numTris;
    if (!mem.alloc(&dPos, (size_t)numVertices * 3) || !mem.alloc(&dIdx, (size_t)numIndices) || !mem.alloc(&dNodes, 2 * n) ||
        !mem.alloc(&dCentroidBox, 6) || !mem.alloc(&dKeys, n) || !mem.alloc(&dKeysSorted, n) || !mem.alloc(&dValues, n) ||
        !mem.alloc(&dClustersA, n) || !mem.alloc(&dClustersB, n) || !mem.alloc(&dNearest, n) || !mem.alloc(&dValid, n) ||
        !mem.alloc(&dOffset, n) || !mem.alloc(&dInterior, 1) || !mem.alloc(&dOut, 2 * n))
        return fail("device allocation failed");
    BB_CUDA(cudaMemcpyAsync(dPos, positions, (size_t)numVertices * 3 * sizeof(float), cudaMemcpyHostToDevice, stream));
    BB_CUDA(cudaMemcpyAsync(dIdx, indices, (size_t)numIndices * sizeof(int), cudaMemcpyHostToDevice, stream));
    const float boxInit[6] = {FLT_MAX, FLT_MAX, FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX};
    BB_CUDA(cudaMemcpyAsync(dCentroidBox, boxInit, sizeof(boxInit), cudaMemcpyHostToDevice, stream));
    BB_CUDA(cudaMemsetAsync(dInterior, 0, sizeof(int), stream));

    // cub scratch for the sort and the scans
    size_t sortBytes = 0, scanBytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, dKeys, dKeysSorted, dValues, dClustersA, numTris, 0, 30, stream);
    cub::DeviceScan::ExclusiveSum(nullptr, scanBytes, dValid, dOffset, numTris, stream);
    unsigned char* dScratch;
    if (!mem.alloc(&dScratch, std::max(sortBytes, scanBytes))) return fail("device allocation failed");
    size_t scratchBytes = std::max(sortBytes, scanBytes);

    BB_CUDA(cudaEventRecord(ev0, stream));
    const int grid = (numTris + PLOC_BLOCK - 1) / PLOC_BLOCK;
    unsigned long long launches = 0;
    k_tri_bounds<<<grid, PLOC_BLOCK, 0, stream>>>(dPos, dIdx, numTris, dNodes, dCentroidBox);
    k_morton<<<grid, PLOC_BLOCK, 0, stream>>>(dNodes, numTris, dCentroidBox, dKeys, dValues);
    launches += 2;
    BB_CUDA(cub::DeviceRadixSort::SortPairs(dScratch, scratchBytes, dKeys, dKeysSorted, dValues, dClustersA, numTris, 0, 30, stream));

    int* cur = dClustersA;
    int* nxt = dClustersB;
    int clusters = numTris, rounds = 0;
    while (clusters > 1) {
        const int g = (clusters + PLOC_BLOCK - 1) / PLOC_BLOCK;
        k_nearest<<<g, PLOC_BLOCK, 0, stream>>>(cur, clusters, dNodes, dNearest);
        k_merge<<<g, PLOC_BLOCK, 0, stream>>>(cur, clusters, dNodes, dNearest, numTris, dInterior, dValid);
        BB_CUDA(cub::DeviceScan::ExclusiveSum(dScratch, scratchBytes, dValid, dOffset, clusters, stream));
        k_compact<<<g, PLOC_BLOCK, 0, stream>>>(cur, dValid, dOffset, clusters, nxt);
        launches += 3;
        // the new count = interior nodes created so far: n - created
        int created = 0;
        BB_CUDA(cudaMemcpyAsync(&created, dInterior, sizeof(int), cudaMemcpyDeviceToHost, stream));
        BB_CUDA(cudaStreamSynchronize(stream));
        const int next = numTris - created;
        if (next >= clusters) return fail("clustering made no progress");   // cannot happen: the globally closest pair is always mutual
        clusters = next;
        std::swap(cur, nxt);
        ++rounds;
    }
    const int numInterior = numTris - 1;
    k_emit<<<(2 * numTris - 1 + PLOC_BLOCK - 1) / PLOC_BLOCK, PLOC_BLOCK, 0, stream>>>(dNodes, numTris, numInterior, dOut);
    launches += 1;
    BB_CUDA(cudaEventRecord(ev1, stream));
    BB_CUDA(cudaMemcpyAsync(outNodes, dOut, (size_t)(2 * numTris - 1) * sizeof(tb200_bvh_node), cudaMemcpyDeviceToHost, stream));
    BB_CUDA(cudaStreamSynchronize(stream));
    BB_CUDA(cudaGetLastError());
    float ms = 0.0f;
    cudaEventElapsedTime(&ms, ev0, ev1);
    cudaEventDestroy(ev0);
    cudaEventDestroy(ev1);
    // PLOC puts no bound on depth (a nested series of ever smaller triangles clusters into a chain), and
    // tb200_create refuses a tree deeper than the traversal stack holds.  Levels in one pass: k_emit numbers
    // interior nodes in reverse creation order and children are created before their parent, so every
    // child's index is larger than its parent's.
    {
        std::vector<int> level((size_t)numInterior, 0);
        int levels = 1;
        level[0] = 1;
        for (int i = 0; i < numInterior; ++i) {
            const uint32_t kids[2] = {outNodes[i].left, outNodes[i].right_leaf & 0x7fffffffu};
            for (uint32_t c : kids)
                if (c < (uint32_t)numInterior) {
                    level[c] = level[i] + 1;
                    levels = std::max(levels, level[c]);
                }
        }
        if (levels > TB200_MAX_BVH_LEVELS) {
            memset(outNodes, 0, (size_t)(2 * numTris - 1) * sizeof(tb200_bvh_node));
            return fail("the tree has " + std::to_string(levels) + " levels of interior nodes, more than the " +
                        std::to_string(TB200_MAX_BVH_LEVELS) + " the traversal stack holds");
        }
    }
    if (info) {
        info->numNodes = 2 * numTris - 1;
        info->rounds = rounds;
        info->kernelLaunches = launches;
        info->buildMs = ms;
    }
    return true;
}

}  // namespace

extern "C" int tb200_bvh_build(const float* positions, int numVertices, const int32_t* indices, int numIndices, tb200_bvh_node* outNodes,
                               int device, tb200_bvh_build_info* info)
{
    g_buildError.clear();
    if (info) memset(info, 0, sizeof(*info));
    if (!positions || !indices || !outNodes || numVertices <= 0 || numIndices < 3 || numIndices % 3 != 0) {
        fail("bad arguments");
        return -1;
    }
    for (int i = 0; i < numIndices; ++i)
        if (indices[i] < 0 || indices[i] >= numVertices) {
            fail("vertex index out of range");
            return -1;
        }
    if (numIndices == 3) {
        // one triangle: a single leaf (BVHBuilder::BuildRecursive with n == 1, bvh.h:224-233)
        tb200_bvh_node o;
        for (int k = 0; k < 3; ++k) {
            const float a = positions[indices[0] * 3 + k], b = positions[indices[1] * 3 + k], c = positions[indices[2] * 3 + k];
            o.lower[k] = std::min(a, std::min(b, c));
            o.upper[k] = std::max(a, std::max(b, c));
        }
        o.left = 0;
        o.right_leaf = 0x80000000u;
        outNodes[0] = o;
        if (info) info->numNodes = 1;
        return 0;
    }
    return build_on_device(positions, numVertices, indices, numIndices, outNodes, device, info) ? 0 : -1;
}

extern "C" const char* tb200_bvh_build_error(void) { return g_buildError.c_str(); }
