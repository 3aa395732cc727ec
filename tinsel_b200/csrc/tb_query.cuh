// tb_query.cuh -- batched closest-hit ray query (tb200_trace_rays): Trace(scene, Ray(origin, dir, time)) of
// render.cpp:17-62 for every ray of a caller's batch, bit for bit, through the same trace_closest() the
// renderer runs; the same query reporting the hit triangle and its barycentric weights (tb200_trace_rays_tri); and
// the batched occlusion query (tb200_occluded_rays) over trace_occluded().  Included once, by kernels.cu.
//
// A persistent kernel: as many CTAs as the SMs hold at once, for the whole batch.  Their warps claim chunks of 32
// rays from a global counter: a static split would leave SMs idle, because a ray that hits a plane costs a few
// dozen instructions and one that walks a deep mesh BVH more than ten times that.

#define TB_QUERY_THREADS 256

// The claim loop of the query kernels: one atomic per warp claims 32 consecutive rays; each lane loads its ray (two
// 16-byte loads) and hands it to ray(i, a, b), which writes its answer with streaming stores, so that the outputs
// do not evict mesh BVH lines from L2.
template <class Ray>
static __device__ __forceinline__ void query_claim_rays(unsigned long long* counter, long long numRays, const float4* rays, Ray ray)
{
    const int lane = threadIdx.x & 31;
    const unsigned long long n = (unsigned long long)numRays;
    for (;;) {
        unsigned long long base = 0ull;
        if (lane == 0) base = atomicAdd(counter, 32ull);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= n) break;
        const unsigned long long i = base + (unsigned long long)lane;
        if (i < n) ray(i, __ldg(&rays[2 * i]), __ldg(&rays[2 * i + 1]));
    }
}

__global__ void __launch_bounds__(TB_QUERY_THREADS) k_trace_rays(const __grid_constant__ QueryParams P)
{
    // one copy of the scene descriptor per CTA: trace_closest takes it by reference, and a per-thread copy would
    // live in local memory
    __shared__ struct { DScene scene; } S;

    // The scene tables stay in global memory: staging the primitive records, scene-level BVH pairs and flat scene
    // program in shared memory with TMA bulk copies, as k_wavefront2 does, measured no faster (DESIGN §5.6).  No
    // mesh treelet either (the host leaves DScene::treelet null).
    if (threadIdx.x == 0) S.scene = P.scene;
    __syncthreads();
    const DScene& sc = S.scene;

    // a: origin.xyz, time; b: dir.xyz, pad
    query_claim_rays(P.counter, P.numRays, P.rays, [&](unsigned long long i, float4 a, float4 b) {
        const Hit h = trace_closest<TB_FEAT_ALL>(sc, v3(a.x, a.y, a.z), v3(b.x, b.y, b.z), a.w, true);
        __stcs(&P.hits[i], make_float4(h.t, h.n.x, h.n.y, h.n.z));
        __stcs(&P.prims[i], h.prim);
    });
}

// CTAs of a persistent query kernel: as many as the SMs hold at once, but no more than there are 32-ray chunks
template <class Kernel>
static unsigned query_grid(Kernel kernel, long long numRays, int numSMs)
{
    int perSM = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, kernel, TB_QUERY_THREADS, 0) != cudaSuccess || perSM < 1) perSM = 1;
    const unsigned long long chunks = ((unsigned long long)numRays + 31ull) / 32ull;
    const unsigned long long warps = (unsigned long long)TB_QUERY_THREADS / 32ull;
    const unsigned long long grid = (unsigned long long)(numSMs > 0 ? numSMs : 1) * (unsigned long long)perSM;
    return (unsigned)std::min(grid, (chunks + warps - 1ull) / warps);
}

const char* launch_trace_rays(const QueryParams& p, int numSMs, cudaStream_t stream, unsigned long long* launchCount)
{
    if (p.numRays <= 0) return nullptr;
    const unsigned grid = query_grid(k_trace_rays, p.numRays, numSMs);
    cudaMemsetAsync(p.counter, 0, sizeof(unsigned long long), stream);
    k_trace_rays<<<grid, TB_QUERY_THREADS, 0, stream>>>(p);
    if (launchCount) ++*launchCount;
    return "k_trace_rays";
}

// Batched occlusion query (tb200_occluded_rays): per ray, whether Trace hits a primitive with t < tmax, the ray
// record's last float; trace_occluded() stops at the first blocker.  The shape of k_trace_rays, writing one byte per ray.
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_occluded_rays(const __grid_constant__ OcclusionParams P)
{
    __shared__ struct { DScene scene; } S;
    if (threadIdx.x == 0) S.scene = P.scene;
    __syncthreads();
    const DScene& sc = S.scene;

    // a: origin.xyz, time; b: dir.xyz, tmax
    query_claim_rays(P.counter, P.numRays, P.rays, [&](unsigned long long i, float4 a, float4 b) {
        const bool occ = trace_occluded<TB_FEAT_ALL>(sc, v3(a.x, a.y, a.z), v3(b.x, b.y, b.z), a.w, b.w);
        __stcs(&P.occluded[i], (unsigned char)occ);
    });
}

const char* launch_occluded_rays(const OcclusionParams& p, int numSMs, cudaStream_t stream, unsigned long long* launchCount)
{
    if (p.numRays <= 0) return nullptr;
    const unsigned grid = query_grid(k_occluded_rays, p.numRays, numSMs);
    cudaMemsetAsync(p.counter, 0, sizeof(unsigned long long), stream);
    k_occluded_rays<<<grid, TB_QUERY_THREADS, 0, stream>>>(p);
    if (launchCount) ++*launchCount;
    return "k_occluded_rays";
}

// Batched closest-hit query with the hit triangle (tb200_trace_rays_tri): k_trace_rays' hit and primitive, bit for bit,
// plus the winner's triangle record from the same walk.  The shape of k_trace_rays, writing a third, 16-byte record.
__global__ void __launch_bounds__(TB_QUERY_THREADS) k_trace_rays_tri(const __grid_constant__ TriQueryParams P)
{
    __shared__ struct { DScene scene; } S;
    if (threadIdx.x == 0) S.scene = P.scene;
    __syncthreads();
    const DScene& sc = S.scene;

    // a: origin.xyz, time; b: dir.xyz, pad
    query_claim_rays(P.counter, P.numRays, P.rays, [&](unsigned long long i, float4 a, float4 b) {
        const HitRec h = trace_closest<TB_FEAT_ALL, true>(sc, v3(a.x, a.y, a.z), v3(b.x, b.y, b.z), a.w, true);
        // the walks leave a sphere's or plane's record unset, or holding an earlier mesh candidate's triangle
        int4 tri = make_int4(-1, 0, 0, 0);
        if (h.prim >= 0 && sc.prims[h.prim].type == TB200_MESH)
            tri = make_int4(h.rec.tri, __float_as_int(h.rec.u), __float_as_int(h.rec.v), __float_as_int(h.rec.w));
        __stcs(&P.hits[i], make_float4(h.t, h.n.x, h.n.y, h.n.z));
        __stcs(&P.prims[i], h.prim);
        __stcs(&P.tris[i], tri);
    });
}

const char* launch_trace_rays_tri(const TriQueryParams& p, int numSMs, cudaStream_t stream, unsigned long long* launchCount)
{
    if (p.numRays <= 0) return nullptr;
    const unsigned grid = query_grid(k_trace_rays_tri, p.numRays, numSMs);
    cudaMemsetAsync(p.counter, 0, sizeof(unsigned long long), stream);
    k_trace_rays_tri<<<grid, TB_QUERY_THREADS, 0, stream>>>(p);
    if (launchCount) ++*launchCount;
    return "k_trace_rays_tri";
}
