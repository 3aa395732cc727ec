// trace_rays_oracle.cpp -- TEST INFRASTRUCTURE: the batch form of the CPU restatement's Trace, the arm the device's
// closest-hit queries (tb200_trace_rays, tb200_trace_rays_tri) are checked against.  It compiles the restatement
// (oracle/tinsel_oracle.cpp) unchanged into the same translation unit and adds entry points that apply its
// closest_hit() to a whole batch on host threads: per-ray calls through ctypes are far too slow for the test sizes.
// tests/rayoracle.py builds it with oracle/Makefile's flags into a temporary directory and loads it.
#include <atomic>

#include "oracle/tinsel_oracle.cpp"

namespace {

// closest_hit(), plus the triangle record of its winner: prim_hit() reads it from mesh_closest() and keeps only the
// normal, so the winner's mesh_closest() runs once more here, on the same primitive, transform and ray.  It is a pure
// function of those, so it returns the record Trace's own call computed.  tri = -1 and u = v = w = 0 unless a mesh
// was hit.
hit_t closest_hit_tri(const tb200_scene& sc, vec3 o, vec3 d, float time, int& tri, float& u, float& v, float& w)
{
    const hit_t hit = closest_hit(sc, o, d, time);
    tri = -1;
    u = v = w = 0.0f;
    if (hit.prim >= 0 && sc.primitives[hit.prim].type == TB200_MESH) {
        const tb200_primitive& p = sc.primitives[hit.prim];
        const xform xf = xf_lerp(xf_from(p.start), xf_from(p.end), time);
        mesh_hit mh;
        if (mesh_closest(sc.meshes[p.mesh], xf_inv_point(xf, o), xf_inv_vector(xf, d), mh) && mh.t == hit.t) {
            tri = mh.tri;
            u = mh.u;
            v = mh.v;
            w = mh.w;
        }
    }
    return hit;
}

// ray(i) for every i < n, on nthreads host threads that take chunks of 4096 rays in turn
template <class Ray>
void for_each_ray(long long n, int nthreads, Ray ray)
{
    const long long chunk = 4096;
    std::atomic<long long> cursor(0);
    auto work = [&] {
        for (;;) {
            const long long i0 = cursor.fetch_add(chunk);
            if (i0 >= n) return;
            const long long i1 = i0 + chunk < n ? i0 + chunk : n;
            for (long long i = i0; i < i1; ++i) ray(i);
        }
    };
    if (nthreads < 1) nthreads = 1;
    std::vector<std::thread> th;
    for (int t = 1; t < nthreads; ++t) th.emplace_back(work);
    work();
    for (auto& x : th) x.join();
}

void put_hit(const hit_t& hit, float* hits, int* prims, long long i)
{
    hits[4 * i + 0] = hit.t;
    hits[4 * i + 1] = hit.n.x;
    hits[4 * i + 2] = hit.n.y;
    hits[4 * i + 3] = hit.n.z;
    prims[i] = hit.prim;
}

}  // namespace

extern "C" {

// tb200_trace_rays' contract over host arrays: rays n x (origin.xyz, time, dir.xyz, pad), hits n x (t, normal.xyz),
// prims n.  `h` is an oracle_create handle of this library.
void oracle_trace_rays(void* h, const float* rays, long long n, float* hits, int* prims, int nthreads)
{
    const tb200_scene& sc = *((Oracle*)h)->scene;
    for_each_ray(n, nthreads, [&](long long i) {
        const float* r = rays + 8 * i;
        put_hit(closest_hit(sc, from(r), from(r + 4), r[3]), hits, prims, i);
    });
}

// tb200_trace_rays_tri's contract over host arrays: oracle_trace_rays' rays, hits and prims, and tris n x (tri, then
// the bits of u, v, w).
void oracle_trace_rays_tri(void* h, const float* rays, long long n, float* hits, int* prims, int* tris, int nthreads)
{
    const tb200_scene& sc = *((Oracle*)h)->scene;
    for_each_ray(n, nthreads, [&](long long i) {
        const float* r = rays + 8 * i;
        float u, v, w;
        put_hit(closest_hit_tri(sc, from(r), from(r + 4), r[3], tris[4 * i], u, v, w), hits, prims, i);
        memcpy(&tris[4 * i + 1], &u, 4);
        memcpy(&tris[4 * i + 2], &v, 4);
        memcpy(&tris[4 * i + 3], &w, 4);
    });
}

}  // extern "C"
