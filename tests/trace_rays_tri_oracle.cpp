// trace_rays_tri_oracle.cpp -- TEST INFRASTRUCTURE: the CPU restatement's closest hit together with the hit triangle,
// the arm the device's tb200_trace_rays_tri is checked against.  It compiles tests/trace_rays_oracle.cpp (and with it
// the unchanged restatement, oracle/tinsel_oracle.cpp) into the same translation unit and adds one batch entry point.
// tests/trioracle.py builds it with oracle/Makefile's flags into a temporary directory and loads it.
#include "tests/trace_rays_oracle.cpp"

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

}  // namespace

extern "C" {

// tb200_trace_rays_tri's contract over host arrays: oracle_trace_rays' rays, hits and prims, and tris n x (tri, then
// the bits of u, v, w).  Threads take chunks of 4096 rays in turn.
void oracle_trace_rays_tri(void* h, const float* rays, long long n, float* hits, int* prims, int* tris, int nthreads)
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
                float u, v, w;
                hit_t hit = closest_hit_tri(sc, from(r), from(r + 4), r[3], tris[4 * i], u, v, w);
                hits[4 * i + 0] = hit.t;
                hits[4 * i + 1] = hit.n.x;
                hits[4 * i + 2] = hit.n.y;
                hits[4 * i + 3] = hit.n.z;
                prims[i] = hit.prim;
                memcpy(&tris[4 * i + 1], &u, 4);
                memcpy(&tris[4 * i + 2], &v, 4);
                memcpy(&tris[4 * i + 3], &w, 4);
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
