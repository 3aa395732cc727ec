// tb_query.cuh -- batched closest-hit ray query (tb200_trace_rays): Trace(scene, Ray(origin, dir, time)) of
// render.cpp:17-62 for every ray of a caller's batch, bit for bit, through the same trace_closest() the
// renderer runs; the same query reporting the hit triangle and its barycentric weights (tb200_trace_rays_tri); and
// the batched occlusion query (tb200_occluded_rays) over trace_occluded().  Included once, by kernels.cu.
//
// A persistent kernel: as many CTAs as the SMs hold at once, for the whole batch.  Their warps claim chunks of 32
// rays from a global counter: a static split would leave SMs idle, because a ray that hits a plane costs a few
// dozen instructions and one that walks a deep mesh BVH more than ten times that.

#define TB_QUERY_THREADS 256

// The body of the query kernels.  One copy of the scene descriptor per CTA: the walks take it by reference, and a
// per-thread copy would live in local memory.  The scene tables stay in global memory: staging the primitive
// records, scene-level BVH pairs and flat scene program in shared memory with TMA bulk copies, as k_wavefront2 does,
// measured no faster (DESIGN §5.6).  No mesh treelet either (the host leaves DScene::treelet null).
// Then one atomic per warp claims 32 consecutive rays; each lane loads its ray (two 16-byte loads) and hands it to
// ray(sc, i, a, b), which writes its answer with streaming stores, so that the outputs do not evict mesh BVH lines
// from L2.
template <class Ray>
static __device__ __forceinline__ void query_claim_rays(const QueryParams& P, Ray ray)
{
    __shared__ struct { DScene scene; } S;
    if (threadIdx.x == 0) S.scene = P.scene;
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const unsigned long long n = (unsigned long long)P.numRays;
    for (;;) {
        unsigned long long base = 0ull;
        if (lane == 0) base = atomicAdd(P.counter, 32ull);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= n) break;
        const unsigned long long i = base + (unsigned long long)lane;
        if (i < n) ray(S.scene, i, __ldg(&P.rays[2 * i]), __ldg(&P.rays[2 * i + 1]));
    }
}

// Closest hit (QueryKind::Closest) and, with TRI, closest hit with the hit triangle (QueryKind::ClosestTri):
// the same hits and primitives bit for bit, and with TRI the winner's triangle record from the same walk.
template <bool TRI>
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_trace_rays(const __grid_constant__ QueryParams P)
{
    // a: origin.xyz, time; b: dir.xyz, pad
    query_claim_rays(P, [&](const DScene& sc, unsigned long long i, float4 a, float4 b) {
        const TraceHit<TRI> h = trace_closest<TB_FEAT_ALL, TRI>(sc, v3(a.x, a.y, a.z), v3(b.x, b.y, b.z), a.w, true);
        // the walks leave a sphere's or plane's record unset, or holding an earlier mesh candidate's triangle
        int4 tri = make_int4(-1, 0, 0, 0);
        if constexpr (TRI) {
            if (h.prim >= 0 && sc.prims[h.prim].type == TB200_MESH)
                tri = make_int4(h.rec.tri, __float_as_int(h.rec.u), __float_as_int(h.rec.v), __float_as_int(h.rec.w));
        }
        __stcs(&P.hits[i], make_float4(h.t, h.n.x, h.n.y, h.n.z));
        __stcs(&P.prims[i], h.prim);
        if constexpr (TRI) __stcs(&P.tris[i], tri);
    });
}

// Occlusion (QueryKind::Occluded): per ray, whether Trace hits a primitive with t < tmax, the ray record's last
// float; trace_occluded() stops at the first blocker.
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_occluded_rays(const __grid_constant__ QueryParams P)
{
    // a: origin.xyz, time; b: dir.xyz, tmax
    query_claim_rays(P, [&](const DScene& sc, unsigned long long i, float4 a, float4 b) {
        const bool occ = trace_occluded<TB_FEAT_ALL>(sc, v3(a.x, a.y, a.z), v3(b.x, b.y, b.z), a.w, b.w);
        __stcs(&P.occluded[i], (unsigned char)occ);
    });
}

void launch_query(QueryKind kind, const QueryParams& p, int numSMs, cudaStream_t stream, unsigned long long* launchCount)
{
    if (p.numRays <= 0) return;
    void (*kernel)(QueryParams) = kind == QueryKind::Closest    ? k_trace_rays<false>
                                  : kind == QueryKind::ClosestTri ? k_trace_rays<true>
                                                                  : k_occluded_rays;
    // as many CTAs as the SMs hold at once, but no more than there are 32-ray chunks
    int perSM = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, kernel, TB_QUERY_THREADS, 0) != cudaSuccess || perSM < 1) perSM = 1;
    const unsigned long long chunks = ((unsigned long long)p.numRays + 31ull) / 32ull;
    const unsigned long long warps = (unsigned long long)TB_QUERY_THREADS / 32ull;
    const unsigned long long grid = (unsigned long long)(numSMs > 0 ? numSMs : 1) * (unsigned long long)perSM;
    cudaMemsetAsync(p.counter, 0, sizeof(unsigned long long), stream);
    kernel<<<(unsigned)std::min(grid, (chunks + warps - 1ull) / warps), TB_QUERY_THREADS, 0, stream>>>(p);
    if (launchCount) ++*launchCount;
}
