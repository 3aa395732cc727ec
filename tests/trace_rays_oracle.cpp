// trace_rays_oracle.cpp -- TEST INFRASTRUCTURE: the batch form of the CPU restatement's Trace, the arm the device's
// closest-hit query (tb200_trace_rays) is checked against.  It compiles the restatement (oracle/tinsel_oracle.cpp)
// unchanged into the same translation unit and adds one entry point that applies its closest_hit() to a whole batch
// on host threads: per-ray calls through ctypes are far too slow for the test sizes.  tests/rayoracle.py builds it
// with oracle/Makefile's flags into a temporary directory and loads it.
#include <atomic>

#include "oracle/tinsel_oracle.cpp"

extern "C" {

// tb200_trace_rays' contract over host arrays: rays n x (origin.xyz, time, dir.xyz, pad), hits n x (t, normal.xyz),
// prims n.  `h` is an oracle_create handle of this library.  Threads take chunks of 4096 rays in turn.
void oracle_trace_rays(void* h, const float* rays, long long n, float* hits, int* prims, int nthreads)
{
    const tb200_scene& sc = *((Oracle*)h)->scene;
    const long long chunk = 4096;
    std::atomic<long long> cursor(0);
    auto work = [&] {
        for (;;) {
            const long long i0 = cursor.fetch_add(chunk);
            if (i0 >= n) return;
            const long long i1 = i0 + chunk < n ? i0 + chunk : n;
            for (long long i = i0; i < i1; ++i) {
                const float* r = rays + 8 * i;
                hit_t hit = closest_hit(sc, from(r), from(r + 4), r[3]);
                hits[4 * i + 0] = hit.t;
                hits[4 * i + 1] = hit.n.x;
                hits[4 * i + 2] = hit.n.y;
                hits[4 * i + 3] = hit.n.z;
                prims[i] = hit.prim;
            }
        }
    };
    if (nthreads < 1) nthreads = 1;
    std::vector<std::thread> th;
    for (int t = 1; t < nthreads; ++t) th.emplace_back(work);
    work();
    for (auto& x : th) x.join();
}

}  // extern "C"
