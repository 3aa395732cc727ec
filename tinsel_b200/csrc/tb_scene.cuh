// tb_scene.cuh -- GPU-side scene layout and the two-level traversal of the closest-hit and occlusion queries.
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

// DMaterial::flags.  The two skips are decided on the host (make_material, set_fresnel_flags), because whether
// they are exact depends on parameter values the loader accepts without checking.
enum : uint32_t {
    TB_MAT_GTR1_WIDE = 1u << 0,     // clearcoat alpha >= 1: GTR1 returns kInvPi (disney.h:58)
    TB_MAT_NO_CLEARCOAT = 1u << 1,  // BSDFEval may skip the clearcoat lobe (tb_shade.cuh: bsdf_eval)
    TB_MAT_NO_FRESNEL = 1u << 2,    // BSDFPdf may skip Fr for a front-facing view (tb_shade.cuh: bsdf_pdf)
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
    uint32_t flags;       // TB_MAT_*
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
    // (splitValid: splitLo/splitHi hold them).  With the split trace queue (kernels.cu: wavefront2_route) the
    // wavefront kernel queues rays that enter this box separately from the rest, so that a warp's 32 rays
    // either all walk the mesh or none does.
    int splitValid;
    V3 splitLo, splitHi;
    // Treelet: the first `treeletPairs` pair records (breadth-first = the top levels) of mesh `treeletMesh`'s BVH,
    // staged in shared memory by the wavefront kernel's prologue (a TMA bulk copy); ray_mesh() reads records
    // below that index from there.  The host sets treeletMesh and the mesh's total pair count; the kernel clips
    // the count to the shared memory it has left and sets the pointer.  Null / 0 everywhere else.
    const unsigned char* treelet;
    int treeletPairs;
    int treeletMesh;
};
// each CTA of the wavefront kernel copies DScene into its shared memory (Wf2Shared::scene): a change of its size
// moves the shared-memory layout behind it (one such shift cost veach 1 %)
static_assert(sizeof(DScene) == 192, "DScene's size moves the wavefront kernel's shared-memory layout");

struct Hit {
    float t;
    V3 n;        // FaceForward'ed (render.cpp:58)
    int prim;    // -1: miss
};

// Scene features that the trace and shading code tests for at run time (the host computes a scene's set in
// api.cu: scene_features).  The device functions that test them take the set as a template parameter FEAT and
// guard each such branch with a constant test of their bit: with a bit clear, the branches only that feature
// can take -- and the code and registers behind them -- drop out of the instantiation.  Every test is still
// made at run time in the default instantiation (TB_FEAT_ALL), which serves every scene.
enum : uint32_t {
    TB_FEAT_NONE = 0u,
    TB_FEAT_PROBE = 1u << 0,          // the sky has an environment probe
    TB_FEAT_MOTION = 1u << 1,         // a primitive moves (start != end transform)
    TB_FEAT_TRANSMISSION = 1u << 2,   // a material has transmission != 0, or BSDFPdf must evaluate Fr for it
    TB_FEAT_SUBSURFACE = 1u << 3,     // a material has subsurface != 0
    TB_FEAT_CLEARCOAT = 1u << 4,      // a material has clearcoat != 0, or a clearcoat lobe that is not finite
    TB_FEAT_ABSORPTION = 1u << 5,     // a material has a non-zero absorption component
    TB_FEAT_ALL = (1u << 6) - 1u,
};

// ---- per-material constants (host side; api.cu and tests/bsdf_harness.cu) ---------------------------------

// The double intermediates are the reference's own (SURVEY.md 7.2c):
//   GetIndexOfRefraction  scene.h:72-78    2.0f/(1.0f-sqrtf(0.08*specular)) - 1.0f
//   Cdlum                 disney.h:307     .3*r + .6*g + .1*b   (double, rounded to float)
//   Ctint, Cspec0         disney.h:309-310 specular*.08 is a double product converted to Real
//   clearcoat alpha       disney.h:387     Lerp(.1,.001,gloss) in double, converted to float
// Sets every flag but TB_MAT_NO_FRESNEL, which depends on the whole scene (set_fresnel_flags).
inline DMaterial make_material(const tb200_material& m)
{
    DMaterial d;
    d.emission = v3(m.emission[0], m.emission[1], m.emission[2]);
    d.color = v3(m.color[0], m.color[1], m.color[2]);
    d.absorption = v3(m.absorption[0], m.absorption[1], m.absorption[2]);
    d.metallic = m.metallic;
    d.subsurface = m.subsurface;
    d.specular = m.specular;
    d.roughness = m.roughness;
    d.specularTint = m.specularTint;
    d.clearcoat = m.clearcoat;
    d.clearcoatGloss = m.clearcoatGloss;
    d.transmission = m.transmission;

    if (m.eta == 0.0f)
        d.ior = 2.0f / (1.0f - sqrtf(float(0.08 * double(m.specular)))) - 1.0f;
    else
        d.ior = m.eta;

    const float Cdlum = float(.3 * double(m.color[0]) + .6 * double(m.color[1]) + .1 * double(m.color[2]));
    const V3 Cdlin = d.color;
    const V3 Ctint = Cdlum > 0.0f ? Cdlin / Cdlum : v3s(1.0f);
    const float spec08 = float(double(m.specular) * .08);
    d.cspec0 = tb_lerp(spec08 * tb_lerp(v3s(1.0f), Ctint, m.specularTint), Cdlin, m.metallic);

    d.sqrtColor = v3(sqrtf(m.color[0]), sqrtf(m.color[1]), sqrtf(m.color[2]));
    d.alpha = tb_max(0.001f, m.roughness);

    const float a = float(.1 + (.001 - .1) * double(m.clearcoatGloss));
    const float a2 = a * a;
    d.gtr1A2m1 = a2 - 1;
    d.gtr1PiLogA2 = TB_PI * logf(a2);
    d.flags = (a >= 1) ? TB_MAT_GTR1_WIDE : 0u;
    // The clearcoat lobe is clearcoat*Gr*Fc*Dr.  With NDotL > 0 and NDotV >= 0, Gr and Fc are finite, so with
    // clearcoat == 0 the lobe is +-0 -- and adding it changes at most the sign of a zero -- iff Dr = GTR1(NDotH) is
    // finite.  The wide branch is kInvPi.  Otherwise Dr = (a2-1) / (kPi*logf(a2) * t), t = 1 + (a2-1)*NDotH^2,
    // needs a finite a2 != 1 (logf(a2) == 0 at 1) and t > 0 for every NDotH^2 up to 1 plus the rounding of unit
    // vectors (2^-20 bounds it): a2 > 1 gives t >= 1; for a2 < 1, t is smallest at the largest NDotH^2, and a tiny
    // a2 -- a gloss near 1/.99, where the alpha crosses 0 -- makes it 0 there and Dr infinite.
    const float t = 1 + d.gtr1A2m1 * 1.00000095367431640625f;   // 1 + 2^-20
    const bool gtr1Finite = (d.flags & TB_MAT_GTR1_WIDE) || (a2 <= FLT_MAX && a2 != 1.0f && (a2 > 1.0f || t > 0.0f));
    if (m.clearcoat == 0.0f && gtr1Finite) d.flags |= TB_MAT_NO_CLEARCOAT;
    return d;
}

// Fr(VDotN, etaI, etaT) is finite for every VDotN > 0 when both etas lie in [1/256, 256]: the squared ratio and
// eta*LDotN stay below 2^32, and no denominator of r1 or r2 can be 0.  A path's etaI and etaO are 1 or the ior of
// some material of the scene (path_hit), so the bound is a property of the scene, not of one material.  Outside
// it Fr can be NaN or infinite (a NaN, infinite, zero or negative ior: eta == 0 with specular < 0 or >= 12.5).
inline bool ior_fresnel_safe(float ior) { return ior >= 1.0f / 256.0f && ior <= 256.0f; }

// Sets TB_MAT_NO_FRESNEL on the materials of one scene: BSDFPdf's `Lerp(brdfPdf, pdfSpec*F, transmission)` is
// brdfPdf plus (finite)*0 -- so Fr may be skipped -- when transmission == 0 and F is finite.  mat(i) returns a
// reference to the scene's i-th DMaterial.
template <class Mat>
inline void set_fresnel_flags(size_t n, Mat mat)
{
    bool safe = true;
    for (size_t i = 0; i < n; ++i) safe = safe && ior_fresnel_safe(mat(i).ior);
    for (size_t i = 0; i < n; ++i)
        if (safe && mat(i).transmission == 0.0f) mat(i).flags |= TB_MAT_NO_FRESNEL;
}

// The material's part of a scene's features (api.cu: scene_features); a NaN parameter counts as present.  The
// kernel compiled without transmission and clearcoat skips Fr and the clearcoat lobe unconditionally, so a
// material counts as having them unless both skips are exact (each flag implies transmission resp. clearcoat 0).
inline uint32_t material_features(const DMaterial& m)
{
    uint32_t f = TB_FEAT_NONE;
    if (!(m.flags & TB_MAT_NO_FRESNEL)) f |= TB_FEAT_TRANSMISSION;
    if (m.subsurface != 0.0f) f |= TB_FEAT_SUBSURFACE;
    if (!(m.flags & TB_MAT_NO_CLEARCOAT)) f |= TB_FEAT_CLEARCOAT;
    if (m.absorption.x != 0.0f || m.absorption.y != 0.0f || m.absorption.z != 0.0f) f |= TB_FEAT_ABSORPTION;
    return f;
}

template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV Xf prim_transform(const DPrim& p, float time)
{
    if (!(FEAT & TB_FEAT_MOTION) || p.isStatic) return p.fixed;
    return interpolate_transform(p.start, p.end, time);
}

// the reciprocal direction of the slab tests: three IEEE divisions, as the reference computes it
TB_DEV V3 ray_rcp(const V3& d)
{
    V3 rcp;
    rcp.x = 1.0f / d.x;
    rcp.y = 1.0f / d.y;
    rcp.z = 1.0f / d.z;
    return rcp;
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

// ray_tri() against triangle i of mesh m, read from its pre-gathered vertices
TB_DEV bool tri_hit(const DMesh& m, uint32_t i, const V3& origin, const V3& dir, float& t, float& u, float& v, float& w, float& sign, V3& n)
{
    const float4 q0 = __ldg(&m.triVerts[i * 3 + 0]);
    const float4 q1 = __ldg(&m.triVerts[i * 3 + 1]);
    const float4 q2 = __ldg(&m.triVerts[i * 3 + 2]);
    return ray_tri(origin, dir, v3(q0.x, q0.y, q0.z), v3(q0.w, q1.x, q1.y), v3(q1.z, q1.w, q2.x), t, u, v, w, sign, n);
}

struct MeshHit {
    float t, u, v, w;
    int tri;
    V3 n;   // closestNormal = n*sign, unnormalised (intersection.h:658)
};

// IntersectRayMesh + MeshQuery, intersection.h:629-749: the reference's stack walk, one triangle or interior pair
// per iteration in the reference's order, with children culled at the mesh's own closest hit.  Pair records below
// `topCount` are read from `top` (the staged treelet), the rest from the mesh's own array.  Each triangle with
// 0 < t < closestT lowers closestT to t and is handed to record(t, i, u, v, w, sign, n); the walk stops when that
// returns true.  Returns closestT: FLT_MAX when nothing was recorded.
template <class Record>
TB_DEV float mesh_walk(const DMesh& m, const unsigned char* top, uint32_t topCount, const V3& origin, const V3& dir, Record record)
{
    const V3 rcp = ray_rcp(dir);
    uint32_t stack[TB_STACK];
    float closestT = FLT_MAX;
    float tmax = FLT_MAX;
    stack[0] = m.rootRef;
    int count = 1;
    while (count) {
        const uint32_t ref = stack[--count];
        if (ref & TB_LEAF) {
            const uint32_t i = ref & ~TB_LEAF;
            float t, u, v, w, sign;
            V3 n;
            if (tri_hit(m, i, origin, dir, t, u, v, w, sign, n)) {
                if (t > 0.0f && t < closestT) {
                    closestT = t;
                    if (record(t, i, u, v, w, sign, n)) break;
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
    return closestT;
}

// The closest hit of mesh_walk(); tri == -1 (and t == FLT_MAX) when the ray misses the mesh.
static __device__ __noinline__ MeshHit ray_mesh(const DMesh& m, const unsigned char* top, uint32_t topCount, V3 origin, V3 dir)
{
    MeshHit out;
    out.tri = -1;
    out.u = out.v = out.w = 0.0f;
    out.n = v3s(0.0f);
    out.t = mesh_walk(m, top, topCount, origin, dir, [&](float, uint32_t i, float u, float v, float w, float sign, V3 n) {
        out.u = u;
        out.v = v;
        out.w = w;
        out.tri = (int)i;
        out.n = n * sign;
        return false;
    });
    return out;
}

// The leaves of a BVH that is one leaf, or one interior pair over two leaves (a quad: cornell's light), in the order
// the reference pops them; a reference without TB_LEAF ends the list.  The reference pops the root, pushes each
// child whose box passes `tChild < tmax` (tmax is still FLT_MAX), the nearer one last when both do, then pops and
// tests the triangles in turn; no box test follows, so the truncation of the ray changes nothing and the walk needs
// no stack.  Returns false for any other tree.
TB_DEV bool small_mesh_leaves(const DMesh& m, const V3& origin, const V3& dir, uint32_t& first, uint32_t& second)
{
    first = m.rootRef;
    second = 0u;
    if (first & TB_LEAF) return true;
    const BvhPair* pr = &m.pairs[first];
    const uint2 kids = *reinterpret_cast<const uint2*>(&pr->left);
    if (!(kids.x & kids.y & TB_LEAF)) return false;
    const float4 a = pr->a, b = pr->b, c = pr->c;
    const V3 rcp = ray_rcp(dir);
    float tLeft, tRight;
    const bool hitLeft = ray_aabb(origin, rcp, a.x, a.y, a.z, a.w, b.x, b.y, tLeft) && tLeft < FLT_MAX;
    const bool hitRight = ray_aabb(origin, rcp, b.z, b.w, c.x, c.y, c.z, c.w, tRight) && tRight < FLT_MAX;
    const bool both = hitLeft && hitRight;
    const bool swap = both && (tLeft < tRight);   // left pushed last: it pops first
    first = hitRight ? (swap ? kids.x : kids.y) : (hitLeft ? kids.x : 0u);
    second = both ? (swap ? kids.y : kids.x) : 0u;
    return true;
}

// ray_mesh() for small_mesh_leaves()' trees, inline and without the stack.  Returns false, having done nothing, for
// any other tree.
TB_DEV bool ray_mesh_small(const DMesh& m, V3 origin, V3 dir, MeshHit& out)
{
    uint32_t first, second;
    if (!small_mesh_leaves(m, origin, dir, first, second)) return false;
    float closestT = FLT_MAX;
    out.tri = -1;
    out.u = out.v = out.w = 0.0f;
    out.n = v3s(0.0f);
#pragma unroll 1
    for (uint32_t ref = first; ref & TB_LEAF; ref = second, second = 0u) {
        const uint32_t i = ref & ~TB_LEAF;
        float t, u, v, w, sign;
        V3 n;
        if (tri_hit(m, i, origin, dir, t, u, v, w, sign, n)) {
            if (t > 0.0f && t < closestT) {
                closestT = t;
                out.u = u;
                out.v = v;
                out.w = w;
                out.tri = (int)i;
                out.n = n * sign;
            }
        }
    }
    out.t = closestT;
    return true;
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

template <uint32_t FEAT = TB_FEAT_ALL>
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
    const Xf xf = prim_transform<FEAT>(p, time);
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
    const DMesh& m = sc.meshes[p.mesh];
    MeshHit mh;
    if (!ray_mesh_small(m, lo, ld, mh)) {
        const bool staged = p.mesh == sc.treeletMesh && sc.treelet != nullptr;
        mh = ray_mesh(m, sc.treelet, staged ? (uint32_t)sc.treeletPairs : 0u, lo, ld);
    }
    if (mh.tri < 0) return false;
    ph.t = mh.t;
    ph.tri = mh.tri;
    ph.u = mh.u;
    ph.v = mh.v;
    ph.w = mh.w;
    ph.gn = mh.n;
    return true;
}

template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV V3 prim_normal(const DScene& sc, const DPrim& p, V3 o, V3 d, float time, const PrimHit& ph)
{
    if (p.type == TB200_PLANE) return v3(p.plane[0], p.plane[1], p.plane[2]);
    const Xf xf = prim_transform<FEAT>(p, time);
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
template <uint32_t FEAT = TB_FEAT_ALL>
TB_ORDERED_ATTR Hit trace_ordered(const DScene& sc, V3 o, V3 d, float time, bool wantNormal)
{
    const V3 rcp = ray_rcp(d);
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
            if (prim_test<FEAT>(sc, sc.prims[index], o, d, time, ph)) {
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
    if (wantNormal && closest >= 0) n = prim_normal<FEAT>(sc, sc.prims[closest], o, d, time, best);
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

// The rays the flat program serves: the origin inside |o| < 1e7, where the planes' +-1e8 boxes cannot miss, and a
// direction without NaN.  Every other ray takes the stack walk.
TB_DEV bool flat_guard(const V3& o, const V3& d)
{
    return (fabsf(o.x) < 1.0e7f) & (fabsf(o.y) < 1.0e7f) & (fabsf(o.z) < 1.0e7f) & (d.x == d.x) & (d.y == d.y) & (d.z == d.z);
}

// `flat` is sc.flat, or the same program where the caller can name it in shared memory (the lane-owned wavefront
// kernel: Wf2Shared::flat), so that the op loads compile to shared-memory loads instead of generic ones.
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV Hit trace_closest(const DScene& sc, const ProgOp* flat, V3 o, V3 d, float time, bool wantNormal)
{
    const int n = sc.numFlat;
    if (n == 0 || !flat_guard(o, d)) return trace_ordered<FEAT>(sc, o, d, time, wantNormal);

    const V3 rcp = ray_rcp(d);

    float minT = FLT_MAX;
    int closest = -1;
    bool tie = false;
    // triangle record of the closest mesh hit.  Kept in (local) memory behind a run-time index on
    // purpose: as a register struct it is copied around on every iteration of the op loop, planes
    // included, which costs more than the whole plane test.  (A register copy of the winner written only
    // on the sphere / mesh branch also measured slower: cornell 1153 against 1171 Msamples/s, H100 at 700 W.)
    PrimHit rec[2];
    int ri = 0;
    rec[0].t = 0.0f; rec[0].tri = 0; rec[0].u = rec[0].v = rec[0].w = 0.0f; rec[0].gn = v3s(0.0f);
    uint32_t visited = 0u;

    for (int i = 0; i < n; ++i) {
        const float4 a = *reinterpret_cast<const float4*>(flat[i].a);
        const float4 bk = *reinterpret_cast<const float4*>(flat[i].b);   // b[0], b[1], kindPrim, bits
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
            if (!prim_test<FEAT>(sc, sc.prims[kindPrim >> 8], o, d, time, *ph)) continue;
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
    if (tie) return trace_ordered<FEAT>(sc, o, d, time, wantNormal);
    Hit h;
    h.t = minT;
    h.prim = closest;
    V3 nrm = v3s(0.0f);
    if (wantNormal && closest >= 0) {
        rec[ri].t = minT;
        nrm = prim_normal<FEAT>(sc, sc.prims[closest], o, d, time, rec[ri]);
    }
    h.n = face_forward(nrm, -d);
    return h;
}

template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV Hit trace_closest(const DScene& sc, V3 o, V3 d, float time, bool wantNormal)
{
    return trace_closest<FEAT>(sc, sc.flat, o, d, time, wantNormal);
}

// ---- occlusion (any-hit) query: trace_occluded() answers `Trace(o, d, time) hits a primitive with t < tmax`
// (tb200_occluded_rays) exactly, without finding the closest hit.
//
// Why stopping at the first blocker is exact:
//   * Scene level.  Trace has no closest-t culling, so the set of primitives it tests depends only on the slab
//     tests, never on what it has found or in which order (the premise of the flat scene program).  It records a
//     primitive when 0 < t < minT, minT starting at FLT_MAX, so its closest t is below tmax iff some tested
//     primitive has 0 < t < min(tmax, FLT_MAX).  Any visit order may stop at the first such primitive, and exact-t
//     ties do not matter: no tie fallback, no winner records.
//   * Mesh level.  The mesh walk does cull boxes with its own closest hit, so it keeps the reference's order and
//     truncation, starting from FLT_MAX.  A triangle is recorded only when 0 < t < closestT, so the records
//     strictly decrease: the first record below tmax proves that the mesh's final t is below tmax, and no record
//     below tmax proves that it is not.
//   * Boxes are never culled with the query's tmax.  A box's slab entry can round above the t of a triangle inside
//     it; the reference, whose bound is its own closest hit, still descends into that box, and a walk culled at
//     tmax would not (DESIGN §8b).
// No u/v/w, no normals, no treelet (the query kernel stages none).

// mesh_walk() that stops at the first recorded triangle with t < tmax; true when there is one (the walk then
// returns that t, and otherwise a closestT that no record brought below tmax).
static __device__ __noinline__ bool ray_mesh_occluded(const DMesh& m, V3 origin, V3 dir, float tmax)
{
    return mesh_walk(m, nullptr, 0u, origin, dir, [&](float t, uint32_t, float, float, float, float, V3) { return t < tmax; }) <
           tmax;
}

// small_mesh_leaves()' trees: the reference tests every leaf whose box passes `tChild < FLT_MAX` and no box test
// follows, so the triangles tested, and with them the verdict, do not depend on their order.
// Returns false, having done nothing, for any other tree; else sets `occluded`.
TB_DEV bool ray_mesh_small_occluded(const DMesh& m, V3 origin, V3 dir, float tmax, bool& occluded)
{
    uint32_t first, second;
    if (!small_mesh_leaves(m, origin, dir, first, second)) return false;
    occluded = false;
#pragma unroll 1
    for (uint32_t ref = first; (ref & TB_LEAF) && !occluded; ref = second, second = 0u) {
        float t, u, v, w, sign;
        V3 n;
        // a triangle with 0 < t < tmax is recorded unless an earlier record is already below it, so either way the
        // mesh's closest t is below tmax
        occluded = tri_hit(m, ref & ~TB_LEAF, origin, dir, t, u, v, w, sign, n) && t > 0.0f && t < tmax;
    }
    return true;
}

// prim_test() and the scene-level acceptance `0 < t`, then `t < tmax`: whether primitive p has a hit that makes the
// ray occluded.  Meshes take the early-exit walks above; prim_test serves only spheres and planes here (a sphere
// hit can have t <= 0).
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV bool prim_occludes(const DScene& sc, const DPrim& p, V3 o, V3 d, float time, float tmax)
{
    if (p.type != TB200_PLANE && p.type != TB200_SPHERE) {
        const Xf xf = prim_transform<FEAT>(p, time);
        const V3 lo = inverse_transform_point(xf, o);
        const V3 ld = inverse_transform_vector(xf, d);
        const DMesh& m = sc.meshes[p.mesh];
        bool occluded;
        if (ray_mesh_small_occluded(m, lo, ld, tmax, occluded)) return occluded;
        return ray_mesh_occluded(m, lo, ld, tmax);
    }
    PrimHit ph;
    return prim_test<FEAT>(sc, p, o, d, time, ph) && ph.t > 0.0f && ph.t < tmax;
}

// trace_ordered()'s stack walk, stopping at the first primitive that occludes.  The near-first order is kept only
// because it tends to find a blocker sooner.  This walk and trace_occluded()'s op loop stay separate from
// trace_ordered()'s and trace_closest()'s: sharing them through a template that takes the query's action changed
// the closest-hit kernels' register allocation and cost the cornell benchmark 3 % (DESIGN §5.7).
template <uint32_t FEAT = TB_FEAT_ALL>
TB_ORDERED_ATTR bool occluded_ordered(const DScene& sc, V3 o, V3 d, float time, float tmax)
{
    const V3 rcp = ray_rcp(d);
    uint32_t stack[TB_STACK];
    stack[0] = sc.rootRef;
    int count = 1;
    while (count) {
        const uint32_t ref = stack[--count];
        if (ref & TB_LEAF) {
            if (prim_occludes<FEAT>(sc, sc.prims[ref & ~TB_LEAF], o, d, time, tmax)) return true;
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
    return false;
}

// Whether Trace(o, d, time) returns a primitive with t < tmax.  tmax <= 0 or NaN: never; a miss (t = FLT_MAX):
// never, whatever tmax.  The flat scene program where trace_closest() runs it (the same guard), else the early-exit
// stack walk.
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV bool trace_occluded(const DScene& sc, V3 o, V3 d, float time, float tmax)
{
    if (!(tmax > 0.0f)) return false;
    if (tmax > FLT_MAX) tmax = FLT_MAX;   // Trace records only t < FLT_MAX
    const int n = sc.numFlat;
    if (n == 0 || !flat_guard(o, d)) return occluded_ordered<FEAT>(sc, o, d, time, tmax);

    const V3 rcp = ray_rcp(d);
    uint32_t visited = 0u;
    for (int i = 0; i < n; ++i) {
        const float4 a = *reinterpret_cast<const float4*>(sc.flat[i].a);
        const float4 bk = *reinterpret_cast<const float4*>(sc.flat[i].b);   // b[0], b[1], kindPrim, bits
        const int kindPrim = __float_as_int(bk.z), bits = __float_as_int(bk.w);
        const int gbit = bits & 0xff;
        if (gbit != TB_BIT_ALWAYS && !((visited >> gbit) & 1u)) continue;
        const int kind = kindPrim & 0xff;
        if (kind == TB_OP_PLANE) {
            // IntersectRayPlane, intersection.h:85-99
            const float dd = a.x * d.x + a.y * d.y + a.z * d.z + a.w * 0.0f;
            if (dd == 0.0f) continue;
            const float t = -(a.x * o.x + a.y * o.y + a.z * o.z + a.w * 1.0f) / dd;
            if (t > 0.0f && t < tmax) return true;
            continue;
        }
        if (kind != TB_OP_LEAF) {
            float tbox;
            if (!ray_aabb(o, rcp, a.x, a.y, a.z, a.w, bk.x, bk.y, tbox)) continue;
            if (kind == TB_OP_BOX) {
                visited |= 1u << ((bits >> 8) & 0xff);
                continue;
            }
        }
        if (prim_occludes<FEAT>(sc, sc.prims[kindPrim >> 8], o, d, time, tmax)) return true;
    }
    return false;
}
