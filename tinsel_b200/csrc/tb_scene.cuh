// tb_scene.cuh -- GPU-side scene layout and the two-level closest-hit traversal.
//
// Layout (built on the host by api.cu from a tb200_scene):
//   * DPrim[]     one record per Primitive (scene.h:142-159) with the per-primitive constants the
//                 reference recomputes per ray hoisted out: the interpolated transform when
//                 start==end (InterpolateTransform is then time-independent), PrimitiveArea,
//                 GetIndexOfRefraction and the material-only subexpressions of BSDFEval.
//   * BvhPair[]   the reference's BVHNode arrays (bvh.h:9-19) re-packed so that ONE interior
//                 visit is ONE 64-byte record holding both children's boxes and references,
//                 instead of three dependent 32-byte node fetches (self + 2 children,
//                 intersection.h:694-708).  Tree topology, child order and visit order are
//                 unchanged, so tie-breaks and the `tLeft < tmax` culling decisions are the
//                 reference's, bit for bit.  A reference is (leaf << 31) | index.
//   * tri verts   per-triangle pre-gathered positions (3 x float4, 48 B) replacing the
//                 index -> vertex double indirection (intersection.h:638-644).
#pragma once

#include <algorithm>
#include <utility>
#include <vector>

#include "tinsel_b200.h"
#include "tb_math.cuh"

#define TB_LEAF 0x80000000u
// the ordered scene walk is the rarely taken fallback of trace_closest(); out of line by default
#ifdef TB_ORDERED_INLINE
#define TB_ORDERED_ATTR static __device__ __forceinline__
#else
#define TB_ORDERED_ATTR static __device__ __noinline__
#endif
#define TB_STACK 32  // the reference uses int stack[32] (intersection.h:688,759)
// Interior levels a BVH may have (TB200_MAX_BVH_LEVELS, checked by validate_bvh / validate_image in api.cu).
// The walks below pop one entry and push up to both children.  Visiting an interior node at level k
// (root = 1) leaves at most k + 1 entries on the stack: one pending sibling per level above plus its own
// two children.  So a tree with L interior levels needs L + 1 entries, and L <= TB_STACK - 1.
static_assert(TB200_MAX_BVH_LEVELS == TB_STACK - 1, "the BVH depth bound must match the traversal stack");

// Host side: interior levels of the binary tree below `root` (0 when the root is a leaf), or -1 when a node
// is reached twice (a shared subtree or a cycle).  children(id, c) returns false for a leaf, else stores the
// two child ids in c.  Ids >= numIds are leaves that need no tracking (the TB_LEAF references of BvhPair
// records); every id below it is checked to be reached once.  Child ids must already be range-checked.
template <class Children>
inline int tb_tree_levels(uint32_t root, size_t numIds, Children children)
{
    std::vector<unsigned char> seen(numIds, 0);
    std::vector<std::pair<uint32_t, int>> todo(1, std::make_pair(root, 1));
    int levels = 0;
    uint32_t c[2];
    while (!todo.empty()) {
        const std::pair<uint32_t, int> it = todo.back();
        todo.pop_back();
        if (it.first < numIds) {
            if (seen[it.first]) return -1;
            seen[it.first] = 1;
        }
        if (!children(it.first, c)) continue;
        levels = std::max(levels, it.second);
        todo.push_back(std::make_pair(c[0], it.second + 1));
        todo.push_back(std::make_pair(c[1], it.second + 1));
    }
    return levels;
}

struct __align__(16) BvhPair {
    float4 a;   // L.lower.xyz, L.upper.x
    float4 b;   // L.upper.yz, R.lower.xy
    float4 c;   // R.lower.z, R.upper.xyz
    uint32_t left, right;   // child references
    uint32_t pad0, pad1;
};

struct DMaterial {
    V3 emission;
    V3 color;
    V3 absorption;
    float metallic, subsurface, specular, roughness, specularTint;
    float clearcoat, clearcoatGloss, transmission;
    // hoisted material-only subexpressions
    float ior;            // Material::GetIndexOfRefraction, scene.h:72-78
    V3 cspec0;            // disney.h:305-310
    V3 sqrtColor;         // disney.h:358
    float alpha;          // Max(0.001f, roughness), disney.h:139
    float gtr1A2m1;       // a2-1 for the clearcoat GTR1, disney.h:61-63,387
    float gtr1PiLogA2;    // kPi*logf(a2)
    int gtr1Wide;         // a >= 1 -> GTR1 returns kInvPi
};

struct DMesh {
    const BvhPair* pairs;
    const float4* triVerts;     // 3 float4 per triangle: (ax ay az bx)(by bz cx cy)(cz - - -)
    const float4* triNormals;   // same packing for the three vertex normals
    const float* cdf;
    int numTris;
    uint32_t rootRef;
};

struct DPrim {
    Xf start, end;
    Xf fixed;             // InterpolateTransform(start,end,t) when isStatic
    int isStatic;
    int type;
    float radius;
    float plane[4];
    int mesh;
    int lightSamples;
    float area;           // PrimitiveArea, intersection.h:833-853
    DMaterial mat;
};

struct DProbe {
    int valid, width, height;
    const float4* data;
    const float* pdfX;
    const float* cdfX;
    const float* pdfY;
    const float* cdfY;
};

struct DScene {
    const DPrim* prims;
    int numPrims;
    const BvhPair* pairs;     // scene-level BVH
    int numPairs;
    uint32_t rootRef;
    const DMesh* meshes;
    int numMeshes;
    V3 horizon, zenith;
    DProbe probe;
    int numNee;               // shadow rays per surface hit: probe + sum(lightSamples)
    const struct ProgOp* flat;     // flat scene program (numFlat == 0: use the ordered walk)
    int numFlat;
    // Scheduling hint only (never changes a result): world-space bounds of the scene's largest mesh
    // when it is big enough for its BVH walk to dominate a ray's cost.  The wavefront kernel queues
    // rays that enter this box separately from the rest, so that a warp's 32 rays either all walk
    // the mesh or none does.
    int splitValid;
    V3 splitLo, splitHi;
    // Offload mode of the wavefront kernel (wavefront_walk.cuh): bit i set = primitive i is a big mesh
    // whose BVH walk runs on the walker CTAs; trace_partial() skips it and reports the rays that reach it.
    uint32_t deferMask;
    // Treelet: the first `treeletPairs` pair records (breadth-first = the top levels) of mesh `treeletMesh`'s BVH,
    // staged in shared memory by the wavefront kernel's prologue (a TMA bulk copy); ray_mesh() reads records
    // below that index from there.  The host sets treeletMesh and the mesh's total pair count; the kernel clips
    // the count to the shared memory it has left and sets the pointer.  Null / 0 everywhere else.
    const unsigned char* treelet;
    int treeletPairs;
    int treeletMesh;
};

struct Hit {
    float t;
    V3 n;        // FaceForward'ed (render.cpp:58)
    int prim;    // -1: miss
};

TB_DEV Xf prim_transform(const DPrim& p, float time)
{
    if (p.isStatic) return p.fixed;
    return interpolate_transform(p.start, p.end, time);
}

// IntersectRayAABBFast, intersection.h:373-397 (minf/maxf are the ternaries of :368-369)
TB_DEV bool ray_aabb(V3 pos, V3 rcp, float lx, float ly, float lz, float ux, float uy, float uz, float& t)
{
    float l1 = (lx - pos.x) * rcp.x;
    float l2 = (ux - pos.x) * rcp.x;
    float lmin = tb_min(l1, l2);
    float lmax = (l1 > l2) ? l1 : l2;

    l1 = (ly - pos.y) * rcp.y;
    l2 = (uy - pos.y) * rcp.y;
    float mn = tb_min(l1, l2), mx = (l1 > l2) ? l1 : l2;
    lmin = (mn > lmin) ? mn : lmin;
    lmax = tb_min(mx, lmax);

    l1 = (lz - pos.z) * rcp.z;
    l2 = (uz - pos.z) * rcp.z;
    mn = tb_min(l1, l2);
    mx = (l1 > l2) ? l1 : l2;
    lmin = (mn > lmin) ? mn : lmin;
    lmax = tb_min(mx, lmax);

    const bool hit = (lmax >= 0.f) & (lmax >= lmin);
    if (hit) t = lmin;
    return hit;
}

// IntersectRayTriTwoSided, intersection.h:117-145
TB_DEV bool ray_tri(V3 p, V3 dir, V3 a, V3 b, V3 c, float& t, float& u, float& v, float& w, float& sign, V3& normal)
{
    const V3 ab = b - a;
    const V3 ac = c - a;
    const V3 n = cross(ab, ac);

    const float d = dot(-dir, n);
    const float ood = 1.0f / d;
    const V3 ap = p - a;

    t = dot(ap, n) * ood;
    if (t < 0.0f) return false;

    const V3 e = cross(-dir, ap);
    v = dot(ac, e) * ood;
    if (v < 0.0f || v > 1.0f) return false;
    w = -dot(ab, e) * ood;
    if (w < 0.0f || v + w > 1.0f) return false;

    u = 1.0f - v - w;
    normal = n;
    sign = d;
    return true;
}

struct MeshHit {
    float t, u, v, w;
    int tri;
    V3 n;   // closestNormal = n*sign, unnormalised (intersection.h:658)
};

// IntersectRayMesh + MeshQuery, intersection.h:629-749
//
// The lanes of a warp that walk a mesh together do it in PHASES, chosen by vote among them (TB_MESH_PHASES):
//   BOX  interior-node steps, repeated while most of the lanes have one.  A lane that reaches a triangle parks
//        it in `pend` and keeps descending -- speculatively: its later box tests use a stale, larger tmax, so it
//        visits a superset of the reference's nodes; everything in the extra nodes lies at t >= the closest hit
//        and fails the strict `t < closestT`, and triangles are still tested in the reference's order, so the
//        result is the reference's bit for bit (the walker CTAs of wavefront_walk.cuh run the same scheme);
//   TRI  the parked triangles are tested.
// A data-dependent `if (leaf) ... else ...` per lane makes the warp execute both bodies in almost every
// iteration; this way each pass runs one body with the lanes that are ready for it.  Measured in round 2:
// bit-exact, but the votes cost more than the divergence they remove (ajax, table and cornell all ran slower),
// so the plain loop below is the default (-DTB_MESH_PHASES=1 builds
// the voted one; the walker CTAs of the offload mode, which have nothing else to do, keep theirs).
#ifndef TB_MESH_PHASES
#define TB_MESH_PHASES 0
#endif
static __device__ __noinline__ bool ray_mesh(const DMesh& m, const unsigned char* top, uint32_t topCount, V3 origin, V3 dir, MeshHit& out)
{
    V3 rcp;
    rcp.x = 1.0f / dir.x;
    rcp.y = 1.0f / dir.y;
    rcp.z = 1.0f / dir.z;

    uint32_t stack[TB_STACK];
    float closestT = FLT_MAX;
    float tmax = FLT_MAX;
    out.tri = -1;
#if TB_MESH_PHASES
    const uint32_t EMPTY = 0xffffffffu;
    const unsigned mask = __activemask();   // the lanes that entered together; every vote below is among them
    const int group = __popc(mask);
    const int boxMin = (group * 5 + 7) / 8, triMin = (group + 3) / 4;
    int sp = 0;
    uint32_t cur = m.rootRef, pend = EMPTY;
    if (cur & TB_LEAF) {   // a one-triangle mesh
        pend = cur;
        cur = EMPTY;
    }
    for (;;) {
        // ---- BOX ---------------------------------------------------------------------------------------------
        int nBox;
        for (;;) {
            const bool wBox = cur != EMPTY && (cur & TB_LEAF) == 0u;
            nBox = __popc(__ballot_sync(mask, wBox));
            if (nBox == 0) break;
            if (wBox) {
                // IntersectRayMesh interior step, intersection.h:702-727; top of the tree from the staged treelet
                // (shared memory) when there is one, the rest from global memory: one generic load path for both
                const unsigned char* base = cur < topCount ? top : reinterpret_cast<const unsigned char*>(m.pairs);
                const BvhPair* pr = reinterpret_cast<const BvhPair*>(base + (size_t)cur * sizeof(BvhPair));
                const float4 a = pr->a, b = pr->b, c = pr->c;
                const uint2 kids = *reinterpret_cast<const uint2*>(&pr->left);
                float tLeft, tRight;
                const bool hitLeft = ray_aabb(origin, rcp, a.x, a.y, a.z, a.w, b.x, b.y, tLeft) && tLeft < tmax;
                const bool hitRight = ray_aabb(origin, rcp, b.z, b.w, c.x, c.y, c.z, c.w, tRight) && tRight < tmax;
                // "traverse closest first": the reference pushes the far child, then the near one, and pops the near
                // one at once (intersection.h:716-727) -- the near child is next, the far one goes on the stack
                const bool both = hitLeft && hitRight;
                const bool swap = both && (tLeft < tRight);
                const uint32_t far = swap ? kids.y : kids.x;
                uint32_t nxt = both ? (swap ? kids.x : kids.y) : (hitLeft ? kids.x : kids.y);
                if (both) stack[sp++] = far;
                if (!(hitLeft || hitRight)) nxt = sp > 0 ? stack[--sp] : EMPTY;
                if (nxt != EMPTY && (nxt & TB_LEAF) != 0u && pend == EMPTY) {
                    // park the triangle, go on with what the reference would pop after testing it
                    pend = nxt;
                    nxt = sp > 0 ? stack[--sp] : EMPTY;
                }
                cur = nxt;
            }
            if (nBox < boxMin) break;   // give the triangle phase a turn (one step per turn keeps every lane progressing)
        }
        // ---- TRI ---------------------------------------------------------------------------------------------
        const bool wTri = pend != EMPTY;
        const int nPend = __popc(__ballot_sync(mask, wTri));
        if (nPend > 0 && (nPend >= triMin || nBox < boxMin)) {
            if (wTri) {
                // MeshQuery, intersection.h:629-674
                const uint32_t i = pend & ~TB_LEAF;
                const float4 q0 = __ldg(&m.triVerts[i * 3 + 0]);
                const float4 q1 = __ldg(&m.triVerts[i * 3 + 1]);
                const float4 q2 = __ldg(&m.triVerts[i * 3 + 2]);
                float t, u, v, w, sign;
                V3 n;
                if (ray_tri(origin, dir, v3(q0.x, q0.y, q0.z), v3(q0.w, q1.x, q1.y), v3(q1.z, q1.w, q2.x), t, u, v, w, sign, n)) {
                    if (t > 0.0f && t < closestT) {
                        closestT = t;
                        out.u = u;
                        out.v = v;
                        out.w = w;
                        out.tri = (int)i;
                        out.n = n * sign;
                    }
                }
                tmax = closestT;   // "truncate ray", intersection.h:700
                pend = EMPTY;
                if (cur != EMPTY && (cur & TB_LEAF) != 0u) {
                    // a second triangle was waiting behind the first
                    pend = cur;
                    cur = sp > 0 ? stack[--sp] : EMPTY;
                }
            }
        }
        if (__ballot_sync(mask, cur != EMPTY || pend != EMPTY) == 0u) break;   // every lane of the group is done
    }
#else
    stack[0] = m.rootRef;
    int count = 1;
    while (count) {
        const uint32_t ref = stack[--count];
        if (ref & TB_LEAF) {
            const uint32_t i = ref & ~TB_LEAF;
            const float4 q0 = __ldg(&m.triVerts[i * 3 + 0]);
            const float4 q1 = __ldg(&m.triVerts[i * 3 + 1]);
            const float4 q2 = __ldg(&m.triVerts[i * 3 + 2]);
            float t, u, v, w, sign;
            V3 n;
            if (ray_tri(origin, dir, v3(q0.x, q0.y, q0.z), v3(q0.w, q1.x, q1.y), v3(q1.z, q1.w, q2.x), t, u, v, w, sign, n)) {
                if (t > 0.0f && t < closestT) {
                    closestT = t;
                    out.u = u;
                    out.v = v;
                    out.w = w;
                    out.tri = (int)i;
                    out.n = n * sign;
                }
            }
            tmax = closestT;  // "truncate ray", intersection.h:700
        } else {
            const unsigned char* base = ref < topCount ? top : reinterpret_cast<const unsigned char*>(m.pairs);
            const BvhPair* pr = reinterpret_cast<const BvhPair*>(base + (size_t)ref * sizeof(BvhPair));
            const float4 a = pr->a, b = pr->b, c = pr->c;
            const uint2 kids = *reinterpret_cast<const uint2*>(&pr->left);
            float tLeft, tRight;
            const bool hitLeft = ray_aabb(origin, rcp, a.x, a.y, a.z, a.w, b.x, b.y, tLeft) && tLeft < tmax;
            const bool hitRight = ray_aabb(origin, rcp, b.z, b.w, c.x, c.y, c.z, c.w, tRight) && tRight < tmax;
            uint32_t left = kids.x, right = kids.y;
            // "traverse closest first": only the indices swap, not the hit flags (intersection.h:716-727)
            if (hitLeft && hitRight && (tLeft < tRight)) {
                const uint32_t tmp = left;
                left = right;
                right = tmp;
            }
            if (hitLeft) stack[count++] = left;
            if (hitRight) stack[count++] = right;
        }
    }
#endif
    if (closestT < FLT_MAX) {
        out.t = closestT;
        return true;
    }
    return false;
}

// PrimitiveIntersect, intersection.h:951-1020, split in two: prim_test() decides hit / t exactly
// as the reference does, prim_normal() produces *outNormal for a recorded hit.  The reference
// computes the normal of every candidate (no side effects); only the winner's is ever used, so
// the traversals below call prim_normal() once, for the closest hit (and never for shadow rays:
// SampleLights only reads t and the hit primitive).
struct PrimHit {
    float t;
    int tri;
    float u, v, w;
    V3 gn;     // MeshQuery::closestNormal (n*sign, unnormalised)
};

TB_DEV bool prim_test(const DScene& sc, const DPrim& p, V3 o, V3 d, float time, PrimHit& ph)
{
    if (p.type == TB200_PLANE) {
        // IntersectRayPlane, intersection.h:85-99; Dot(Vec4,Vec4) adds plane.w*0 resp. plane.w*1
        const float dd = p.plane[0] * d.x + p.plane[1] * d.y + p.plane[2] * d.z + p.plane[3] * 0.0f;
        if (dd == 0.0f) return false;
        const float t = -(p.plane[0] * o.x + p.plane[1] * o.y + p.plane[2] * o.z + p.plane[3] * 1.0f) / dd;
        ph.t = t;
        return t > 0.0f;
    }
    const Xf xf = prim_transform(p, time);
    if (p.type == TB200_SPHERE) {
        // SolveQuadratic with a == 1 + IntersectRaySphere, intersection.h:30-83
        const V3 q = o - xf.p;
        const float radius = p.radius * xf.s;
        const float a = 1.0f;
        const float b = 2.0f * dot(q, d);
        const float c = dot(q, q) - (radius * radius);
        const float disc = b * b - 4.0f * a * c;
        if (disc < 0.0f) return false;   // the reference falls through with r == false and returns it
        const float tt = -0.5f * (b + ((b < 0.0f) ? -1.0f : 1.0f) * sqrtf(disc));
        float minT = tt / a;
        float maxT = c / tt;
        if (maxT < minT) { const float s = minT; minT = maxT; maxT = s; }   // Sort2
        if (minT < 0.0f && maxT < 0.0f) return false;
        if (minT < 0.0f && maxT > 0.0f) minT = maxT;
        ph.t = minT;
        return true;
    }
    // mesh
    const V3 lo = inverse_transform_point(xf, o);
    const V3 ld = inverse_transform_vector(xf, d);
    MeshHit mh;
    const bool staged = p.mesh == sc.treeletMesh && sc.treelet != nullptr;
    if (!ray_mesh(sc.meshes[p.mesh], sc.treelet, staged ? (uint32_t)sc.treeletPairs : 0u, lo, ld, mh)) return false;
    ph.t = mh.t;
    ph.tri = mh.tri;
    ph.u = mh.u;
    ph.v = mh.v;
    ph.w = mh.w;
    ph.gn = mh.n;
    return true;
}

TB_DEV V3 prim_normal(const DScene& sc, const DPrim& p, V3 o, V3 d, float time, const PrimHit& ph)
{
    if (p.type == TB200_PLANE) return v3(p.plane[0], p.plane[1], p.plane[2]);
    const Xf xf = prim_transform(p, time);
    if (p.type == TB200_SPHERE) return normalize((o + d * ph.t) - xf.p);   // intersection.h:76-79
    const DMesh& m = sc.meshes[p.mesh];
    const float4 q0 = __ldg(&m.triNormals[ph.tri * 3 + 0]);
    const float4 q1 = __ldg(&m.triNormals[ph.tri * 3 + 1]);
    const float4 q2 = __ldg(&m.triNormals[ph.tri * 3 + 2]);
    const V3 n1 = v3(q0.x, q0.y, q0.z), n2 = v3(q0.w, q1.x, q1.y), n3 = v3(q1.z, q1.w, q2.x);
    V3 smooth = ph.u * n1 + ph.v * n2 + ph.w * n3;
    if (dot(smooth, ph.gn) < 0.0f) smooth = smooth * -1.0f;
    return safe_normalize(transform_vector(xf, smooth), ph.gn);   // intersection.h:994-1013
}

// Trace + QueryBVH, render.cpp:17-62 + intersection.h:751-799: near-first DFS over the scene
// BVH with NO closest-t culling; the callback keeps `t < minT && t > 0` (first found wins ties).
// This is the reference's visit order, bit for bit.
TB_ORDERED_ATTR Hit trace_ordered(const DScene& sc, V3 o, V3 d, float time, bool wantNormal)
{
    V3 rcp;
    rcp.x = 1.0f / d.x;
    rcp.y = 1.0f / d.y;
    rcp.z = 1.0f / d.z;

    uint32_t stack[TB_STACK];
    stack[0] = sc.rootRef;
    int count = 1;

    float minT = FLT_MAX;
    int closest = -1;
    PrimHit best;
    best.t = 0.0f; best.tri = 0; best.u = best.v = best.w = 0.0f; best.gn = v3s(0.0f);

    while (count) {
        const uint32_t ref = stack[--count];
        if (ref & TB_LEAF) {
            const int index = (int)(ref & ~TB_LEAF);
            PrimHit ph;
            if (prim_test(sc, sc.prims[index], o, d, time, ph)) {
                if (ph.t < minT && ph.t > 0.0f) {
                    minT = ph.t;
                    closest = index;
                    best = ph;
                }
            }
        } else {
            const BvhPair* pr = &sc.pairs[ref];
            const float4 a = pr->a, b = pr->b, c = pr->c;
            float tLeft, tRight;
            const bool hitLeft = ray_aabb(o, rcp, a.x, a.y, a.z, a.w, b.x, b.y, tLeft);
            const bool hitRight = ray_aabb(o, rcp, b.z, b.w, c.x, c.y, c.z, c.w, tRight);
            uint32_t left = pr->left, right = pr->right;
            if (hitLeft && hitRight && (tLeft < tRight)) {
                const uint32_t tmp = left;
                left = right;
                right = tmp;
            }
            if (hitLeft) stack[count++] = left;
            if (hitRight) stack[count++] = right;
        }
    }
    Hit h;
    h.t = minT;
    h.prim = closest;
    V3 n = v3s(0.0f);
    if (wantNormal && closest >= 0) n = prim_normal(sc, sc.prims[closest], o, d, time, best);
    h.n = face_forward(n, -d);
    return h;
}

// Flat scene program.  For small scenes (<= 16 primitives) the ordered walk above spends most of
// its instructions on boxes that cannot miss: planes have +-1e8 bounds (intersection.h:919-924),
// so every subtree holding one is "hit" for any ray that starts inside |o| < 1e7.  Because the
// scene level has no closest-t culling, the SET of primitives tested depends only on which nodes'
// slab tests pass, never on the visit order; the order matters only when two primitives return
// exactly the same t.  The host (api.cu: build_program) therefore compiles the scene BVH into a
// short list of ops executed in a fixed, warp-uniform order:
//   BOX      finite interior box: same slab test as the reference, result kept in a bit mask
//   LEAFBOX  finite leaf box + primitive test          LEAF  primitive test behind infinite boxes
//   PLANE    static plane with its coefficients inline (IntersectRayPlane ignores transforms)
// each guarded by the bit of its nearest finite ancestor (infinite boxes are transparent).
// trace_closest() keeps min t and -- if it ever sees an exact tie, a NaN direction, or an origin
// outside the guard -- redoes the ray with trace_ordered().  Same result bit for bit, a fraction
// of the instructions, no stack, no type-switch divergence.
enum { TB_OP_BOX = 0, TB_OP_LEAFBOX = 1, TB_OP_LEAF = 2, TB_OP_PLANE = 3 };
#define TB_BIT_ALWAYS 32

struct __align__(16) ProgOp {
    float a[4];      // BOX/LEAFBOX: lo.xyz, hi.x      PLANE: plane coefficients
    float b[2];      // BOX/LEAFBOX: hi.y, hi.z
    int kindPrim;    // kind | primitive index << 8
    int bits;        // guard bit (TB_BIT_ALWAYS: unconditional) | own bit << 8 (BOX only)
};

TB_DEV Hit trace_closest(const DScene& sc, V3 o, V3 d, float time, bool wantNormal)
{
    const int n = sc.numFlat;
    const bool guard = (fabsf(o.x) < 1.0e7f) & (fabsf(o.y) < 1.0e7f) & (fabsf(o.z) < 1.0e7f) & (d.x == d.x) & (d.y == d.y) &
                       (d.z == d.z);
    if (n == 0 || !guard) return trace_ordered(sc, o, d, time, wantNormal);

    V3 rcp;
    rcp.x = 1.0f / d.x;
    rcp.y = 1.0f / d.y;
    rcp.z = 1.0f / d.z;

    float minT = FLT_MAX;
    int closest = -1;
    bool tie = false;
    // triangle record of the closest mesh hit.  Kept in (local) memory behind a run-time index on
    // purpose: as a register struct it is copied around on every iteration of the op loop, planes
    // included, which costs more than the whole plane test.
    PrimHit rec[2];
    int ri = 0;
    rec[0].t = 0.0f; rec[0].tri = 0; rec[0].u = rec[0].v = rec[0].w = 0.0f; rec[0].gn = v3s(0.0f);
    uint32_t visited = 0u;

    for (int i = 0; i < n; ++i) {
        const float4 a = *reinterpret_cast<const float4*>(sc.flat[i].a);
        const float4 bk = *reinterpret_cast<const float4*>(sc.flat[i].b);   // b[0], b[1], kindPrim, bits
        const int kindPrim = __float_as_int(bk.z), bits = __float_as_int(bk.w);
        const int gbit = bits & 0xff;
        if (gbit != TB_BIT_ALWAYS && !((visited >> gbit) & 1u)) continue;
        const int kind = kindPrim & 0xff;
        float t;
        if (kind == TB_OP_PLANE) {
            // IntersectRayPlane, intersection.h:85-99
            const float dd = a.x * d.x + a.y * d.y + a.z * d.z + a.w * 0.0f;
            if (dd == 0.0f) continue;
            t = -(a.x * o.x + a.y * o.y + a.z * o.z + a.w * 1.0f) / dd;
        } else {
            if (kind != TB_OP_LEAF) {
                float tbox;
                if (!ray_aabb(o, rcp, a.x, a.y, a.z, a.w, bk.x, bk.y, tbox)) continue;
                if (kind == TB_OP_BOX) {
                    visited |= 1u << ((bits >> 8) & 0xff);
                    continue;
                }
            }
            PrimHit* ph = &rec[ri ^ 1];
            if (!prim_test(sc, sc.prims[kindPrim >> 8], o, d, time, *ph)) continue;
            t = ph->t;
            if (t > 0.0f && t < minT) ri ^= 1;   // the record just written becomes the best one
        }
        if (t > 0.0f) {
            if (t < minT) {
                minT = t;
                closest = kindPrim >> 8;
            } else if (t == minT) {
                tie = true;
            }
        }
    }
    if (tie) return trace_ordered(sc, o, d, time, wantNormal);
    Hit h;
    h.t = minT;
    h.prim = closest;
    V3 nrm = v3s(0.0f);
    if (wantNormal && closest >= 0) {
        rec[ri].t = minT;
        nrm = prim_normal(sc, sc.prims[closest], o, d, time, rec[ri]);
    }
    h.n = face_forward(nrm, -d);
    return h;
}


// trace_closest() for the offload mode of the wavefront kernel: the primitives of sc.deferMask (big
// meshes) are not intersected here -- a ray that reaches one (its box test passed, or it sits behind
// infinite boxes) gets that primitive's bit in `pending` and the caller posts it to the walker CTAs.
// The hit returned covers all other primitives; merging it with the walkers' answer gives exactly
// trace_closest()'s result, because the closest hit over a set of primitives does not depend on the
// order they are tested in, EXCEPT for exact ties in t -- which the scene program detects among its
// own primitives (below), the walkers among theirs, and the merge between the two; every tie is redone
// with the reference-order walk.  Falls back to the complete trace_ordered() (pending == 0) for the
// same rays trace_closest() does.
TB_DEV Hit trace_partial(const DScene& sc, V3 o, V3 d, float time, bool wantNormal, uint32_t& pending)
{
    pending = 0u;
    const int n = sc.numFlat;
    const bool guard = (fabsf(o.x) < 1.0e7f) & (fabsf(o.y) < 1.0e7f) & (fabsf(o.z) < 1.0e7f) & (d.x == d.x) & (d.y == d.y) &
                       (d.z == d.z);
    if (n == 0 || !guard) return trace_ordered(sc, o, d, time, wantNormal);

    V3 rcp;
    rcp.x = 1.0f / d.x;
    rcp.y = 1.0f / d.y;
    rcp.z = 1.0f / d.z;

    float minT = FLT_MAX;
    int closest = -1;
    bool tie = false;
    PrimHit rec[2];
    int ri = 0;
    rec[0].t = 0.0f; rec[0].tri = 0; rec[0].u = rec[0].v = rec[0].w = 0.0f; rec[0].gn = v3s(0.0f);
    uint32_t visited = 0u;
    uint32_t wait = 0u;

    for (int i = 0; i < n; ++i) {
        const float4 a = *reinterpret_cast<const float4*>(sc.flat[i].a);
        const float4 bk = *reinterpret_cast<const float4*>(sc.flat[i].b);   // b[0], b[1], kindPrim, bits
        const int kindPrim = __float_as_int(bk.z), bits = __float_as_int(bk.w);
        const int gbit = bits & 0xff;
        if (gbit != TB_BIT_ALWAYS && !((visited >> gbit) & 1u)) continue;
        const int kind = kindPrim & 0xff;
        float t;
        if (kind == TB_OP_PLANE) {
            const float dd = a.x * d.x + a.y * d.y + a.z * d.z + a.w * 0.0f;
            if (dd == 0.0f) continue;
            t = -(a.x * o.x + a.y * o.y + a.z * o.z + a.w * 1.0f) / dd;
        } else {
            if (kind != TB_OP_LEAF) {
                float tbox;
                if (!ray_aabb(o, rcp, a.x, a.y, a.z, a.w, bk.x, bk.y, tbox)) continue;
                if (kind == TB_OP_BOX) {
                    visited |= 1u << ((bits >> 8) & 0xff);
                    continue;
                }
            }
            const int prim = kindPrim >> 8;
            if ((sc.deferMask >> prim) & 1u) {
                wait |= 1u << prim;
                continue;
            }
            PrimHit* ph = &rec[ri ^ 1];
            if (!prim_test(sc, sc.prims[prim], o, d, time, *ph)) continue;
            t = ph->t;
            if (t > 0.0f && t < minT) ri ^= 1;
        }
        if (t > 0.0f) {
            if (t < minT) {
                minT = t;
                closest = kindPrim >> 8;
            } else if (t == minT) {
                tie = true;
            }
        }
    }
    if (tie) return trace_ordered(sc, o, d, time, wantNormal);
    pending = wait;
    Hit h;
    h.t = minT;
    h.prim = closest;
    V3 nrm = v3s(0.0f);
    if (wantNormal && closest >= 0) {
        rec[ri].t = minT;
        nrm = prim_normal(sc, sc.prims[closest], o, d, time, rec[ri]);
    }
    h.n = face_forward(nrm, -d);
    return h;
}
