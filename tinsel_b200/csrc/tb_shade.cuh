// tb_shade.cuh -- Disney BSDF, HDR probe / sky, next-event estimation and the per-bounce path
// logic of PathTrace (render.cpp:230-388), split into stage functions so that the same code
// serves the one-thread-per-path validation kernel and the wavefront pipeline.
//
// Operation order follows the cited reference expressions exactly (see tb_math.cuh header).
#pragma once

#include "tb_scene.cuh"

enum { TB_REFLECTED = 0, TB_TRANSMITTED = 1, TB_SPECULAR = 2 };   // BSDFType, disney.h:27-32

#define TB_RAY_EPS 0.0001f   // kRayEpsilon, render.cpp:11

// ---- Disney BSDF (disney.h) -------------------------------------------------------------------

// SchlickFresnel, disney.h:49-54
TB_DEV float schlick_fresnel(float u)
{
    const float m = tb_clamp(1 - u, 0.0f, 1.0f);
    const float m2 = m * m;
    return m2 * m2 * m;
}

// GTR2, disney.h:64-69
TB_DEV float gtr2(float NDotH, float a)
{
    const float a2 = a * a;
    const float t = 1.0f + (a2 - 1.0f) * NDotH * NDotH;
    return a2 / (TB_PI * t * t);
}

// GTR1 with the material-constant parts hoisted, disney.h:56-62
TB_DEV float gtr1_clearcoat(const DMaterial& m, float NDotH)
{
    if (m.flags & TB_MAT_GTR1_WIDE) return TB_INV_PI;
    const float t = 1 + m.gtr1A2m1 * NDotH * NDotH;
    return m.gtr1A2m1 / (m.gtr1PiLogA2 * t);
}

// SmithGGX, disney.h:71-76
TB_DEV float smith_ggx(float NDotv, float alphaG)
{
    const float a = alphaG * alphaG;
    const float b = NDotv * NDotv;
    return 1 / (NDotv + sqrtf(a + b - a * b));
}

// Fr, disney.h:79-96
TB_NOINLINE float fresnel_dielectric(float VDotN, float etaI, float etaT)
{
    const float SinThetaT2 = tb_sqr(etaI / etaT) * (1.0f - VDotN * VDotN);
    if (SinThetaT2 > 1.0f) return 1.0f;
    const float LDotN = sqrtf(1.0f - SinThetaT2);
    const float eta = etaT / etaI;
    const float r1 = (VDotN - eta * LDotN) / (VDotN + eta * LDotN);
    const float r2 = (LDotN - eta * VDotN) / (LDotN + eta * VDotN);
    return 0.5f * (tb_sqr(r1) + tb_sqr(r2));
}

// Refract, disney.h:34-47
TB_DEV bool refract_dir(V3 wi, V3 n, float eta, V3& wt)
{
    const float cosThetaI = dot(n, wi);
    const float sin2ThetaI = tb_max(0.0f, 1.0f - cosThetaI * cosThetaI);
    const float sin2ThetaT = eta * eta * sin2ThetaI;
    if (sin2ThetaT >= 1) return false;
    const float cosThetaT = sqrtf(1.0f - sin2ThetaT);
    wt = eta * -wi + (eta * cosThetaI - cosThetaT) * n;
    return true;
}

// BSDFPdf, disney.h:125-166
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV float bsdf_pdf(const DMaterial& mat, float etaI, float etaO, V3 n, V3 V, V3 L)
{
    if (dot(L, n) <= 0.0f) {
        const float bsdfPdf = 0.0f;
        const float brdfPdf = TB_INV_2PI * mat.subsurface * 0.5f;
        return tb_lerp(brdfPdf, bsdfPdf, mat.transmission);
    }
    const float NV = dot(n, V);
    const float a = mat.alpha;
    const V3 half = safe_normalize(L + V, v3s(0.0f));
    const float cosThetaHalf = tb_abs(dot(half, n));
    const float pdfHalf = gtr2(cosThetaHalf, a) * cosThetaHalf;
    const float pdfSpec = 0.25f * pdfHalf / tb_max(1.e-6f, dot(L, half));
    const float pdfDiff = tb_abs(dot(L, n)) * TB_INV_PI * (1.0f - mat.subsurface);
    const float brdfPdf = tb_lerp(pdfDiff, pdfSpec, 0.5f);
    // Lerp(brdfPdf, pdfSpec*F, transmission): with transmission == 0, a front-facing view and every ior of the
    // scene in the range where Fr is finite (TB_MAT_NO_FRESNEL, tb_scene.cuh: set_fresnel_flags), the lerp adds
    // (finite)*0 = +-0 and returns brdfPdf up to the sign of a zero; Fr is skipped then.
    if ((!(FEAT & TB_FEAT_TRANSMISSION) || (mat.flags & TB_MAT_NO_FRESNEL)) && NV > 0.0f) return brdfPdf;
    const float F = fresnel_dielectric(NV, etaI, etaO);
    const float bsdfPdf = pdfSpec * F;
    return tb_lerp(brdfPdf, bsdfPdf, mat.transmission);
}

// BSDFEval, disney.h:296-405 (Cdlum/Ctint/Cspec0 and the clearcoat alpha are per-material
// constants computed on the host with the reference's double intermediates, api.cu)
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV V3 bsdf_eval(const DMaterial& mat, float etaI, float etaO, V3 N, V3 V, V3 L)
{
    const float NDotL = dot(N, L);
    const float NDotV = dot(N, V);
    const V3 H = normalize(L + V);
    const float NDotH = dot(N, H);
    const float LDotH = dot(L, H);

    V3 bsdf = v3s(0.0f);
    V3 brdf = v3s(0.0f);

    if ((FEAT & TB_FEAT_TRANSMISSION) && mat.transmission > 0.0f) {
        if (NDotL <= 0) {
            const float F = fresnel_dielectric(NDotV, etaI, etaO);
            bsdf = v3s(mat.transmission * (1.0f - F) / tb_abs(NDotL) * (1.0f - mat.metallic));
        } else {
            const float a = mat.alpha;
            const float Ds = gtr2(NDotH, a);
            const float FH = fresnel_dielectric(LDotH, etaI, etaO);
            const V3 Fs = tb_lerp(mat.cspec0, v3s(1.0f), FH);
            const float Gs = smith_ggx(NDotV, a) * smith_ggx(NDotL, a);
            bsdf = Gs * Fs * Ds;
        }
    }

    if (!(FEAT & TB_FEAT_TRANSMISSION) || mat.transmission < 1.0f) {
        if (NDotL <= 0) {
            if ((FEAT & TB_FEAT_SUBSURFACE) && mat.subsurface > 0.0f) {
                const float FL = schlick_fresnel(tb_abs(NDotL)), FV = schlick_fresnel(NDotV);
                const float Fd = (1.0f - 0.5f * FL) * (1.0f - 0.5f * FV);
                brdf = TB_INV_PI * mat.sqrtColor * mat.subsurface * Fd * (1.0f - mat.metallic);
            }
        } else {
            const float a = mat.alpha;
            const float Ds = gtr2(NDotH, a);
            const float FH = schlick_fresnel(LDotH);
            const V3 Fs = tb_lerp(mat.cspec0, v3s(1.0f), FH);
            const float Gs = smith_ggx(NDotV, a) * smith_ggx(NDotL, a);

            const float FL = schlick_fresnel(NDotL), FV = schlick_fresnel(NDotV);
            // `0.5 + 2.0f*LDotH*LDotH*roughness`: the double add of two floats rounds like the fp32 add
            const float Fd90 = 0.5f + 2.0f * LDotH * LDotH * mat.roughness;
            const float Fd = tb_lerp(1.0f, Fd90, FL) * tb_lerp(1.0f, Fd90, FV);

            brdf = TB_INV_PI * Fd * mat.color * (1.0f - mat.metallic) * (1.0f - mat.subsurface) + Gs * Fs * Ds;
            // clearcoat lobe: `+ mat.clearcoat*Gr*Fc*Dr`.  With clearcoat == 0 and a finite GTR1 (TB_MAT_NO_CLEARCOAT,
            // tb_scene.cuh: make_material) the term is 0*finite = +-0 and adding it changes at most the sign of a
            // zero, which no branch or sum downstream can observe; skip the lobe then.
            if ((FEAT & TB_FEAT_CLEARCOAT) && !(mat.flags & TB_MAT_NO_CLEARCOAT)) {
                const float Dr = gtr1_clearcoat(mat, NDotH);
                const float Fc = tb_lerp(.04f, 1.0f, FH);
                const float Gr = smith_ggx(NDotL, .25f) * smith_ggx(NDotV, .25f);
                brdf = brdf + v3s(mat.clearcoat * Gr * Fc * Dr);
            }
        }
    }
    return tb_lerp(brdf, bsdf, mat.transmission);
}

// BSDFPdf + BSDFEval for the same (V, L): one out-of-line copy serves NEE and the BSDF sample
struct BsdfValue {
    V3 f;        // BSDFEval
    float pdf;   // BSDFPdf
};

template <uint32_t FEAT = TB_FEAT_ALL>
TB_NOINLINE BsdfValue bsdf_eval_pdf(const DMaterial& mat, float etaI, float etaO, V3 N, V3 V, V3 L)
{
    BsdfValue r;
    r.pdf = bsdf_pdf<FEAT>(mat, etaI, etaO, N, V, L);
    r.f = bsdf_eval<FEAT>(mat, etaI, etaO, N, V, L);
    return r;
}

// the GGX half-vector lobe shared by both branches of BSDFSample, disney.h:183-205 / 256-279;
// sinPhiHalf / cosPhiHalf = sinf / cosf(r1*k2Pi) are computed by the caller
TB_DEV V3 sample_ggx_reflection(const DMaterial& mat, float r2, float sinPhiHalf, float cosPhiHalf, V3 U, V3 Vt, V3 N, V3 view)
{
    const float a = mat.alpha;
    const float cosThetaHalf = sqrtf((1.0f - r2) / (1.0f + (tb_sqr(a) - 1.0f) * r2));
    const float sinThetaHalf = sqrtf(tb_max(0.0f, 1.0f - tb_sqr(cosThetaHalf)));
    V3 half = U * (sinThetaHalf * cosPhiHalf) + Vt * (sinThetaHalf * sinPhiHalf) + N * cosThetaHalf;
    if (dot(half, view) <= 0.0f) half = half * -1.0f;
    return 2.0f * dot(view, half) * half - view;
}

// BSDFSample, disney.h:170-293.  Draw order: Randf(transmission?) -> [Randf(F?) -> Sample2D | -]
// or Sample2D -> Randf(0.5) -> [Randf(subsurface?) -> (Randf,Randf) | -].
// The three lobes that need sinf/cosf of an angle (GGX: r1*k2Pi, cosine: k2Pi*r2, uniform
// hemisphere: k2Pi*Randf) first only pick their angle; one shared sincos call then serves all
// lanes of the warp instead of three divergent ones (same values: the product is commutative).
// Returns true when the pdf is BSDFPdf(light) (the caller evaluates it together with BSDFEval);
// false when `pdf` is already final (specular refraction, or 0 for total internal reflection).
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV bool bsdf_sample_dir(const DMaterial& mat, float etaI, float etaO, V3 U, V3 Vt, V3 N, V3 view, V3& light, float& pdf,
                            int& type, Rng& rng)
{
    enum { LOBE_GGX, LOBE_COSINE, LOBE_UNIFORM };
    int lobe;
    float angleArg, r1 = 0.0f, r2 = 0.0f, uz = 0.0f;
    // the draws are made whatever FEAT says; only the comparisons with a constant 0 fold (x < 0 is false for x >= 0)
    const float rt = rng_float(rng);
    if ((FEAT & TB_FEAT_TRANSMISSION) && rt < mat.transmission) {
        const float F = fresnel_dielectric(dot(N, view), etaI, etaO);
        if (rng_float(rng) < F) {
            r1 = rng_float(rng);
            r2 = rng_float(rng);
            type = TB_REFLECTED;
            lobe = LOBE_GGX;
            angleArg = r1;
        } else {
            const float eta = etaI / etaO;
            if (refract_dir(view, N, eta, light)) {
                type = TB_SPECULAR;
                pdf = (1.0f - F) * mat.transmission;
                return false;
            }
            pdf = 0.0f;
            return false;
        }
    } else {
        r1 = rng_float(rng);
        r2 = rng_float(rng);
        if (rng_float(rng) < 0.5f) {
            const float rs = rng_float(rng);
            if ((FEAT & TB_FEAT_SUBSURFACE) && rs < mat.subsurface) {
                // UniformSampleHemisphere(Random&), maths.h:1291-1302: z, then phi = k2Pi*Randf
                uz = rng_float(rng);
                angleArg = rng_float(rng);
                lobe = LOBE_UNIFORM;
                type = TB_TRANSMITTED;
            } else {
                lobe = LOBE_COSINE;
                angleArg = r2;
                type = TB_REFLECTED;
            }
        } else {
            lobe = LOBE_GGX;
            angleArg = r1;
            type = TB_REFLECTED;
        }
    }
    const float2 sca = tb_sincosf(angleArg * TB_2PI);
    const float sn = sca.x, cs = sca.y;
    if (lobe == LOBE_GGX) {
        light = sample_ggx_reflection(mat, r2, sn, cs, U, Vt, N, view);
    } else if (lobe == LOBE_COSINE) {
        // CosineSampleHemisphere, maths.h:1319-1325 via UniformSampleDisc, maths.h:1304-1310
        const float r = sqrtf(r1);
        const float sx = r * cs, sy = r * sn;
        const float z = sqrtf(tb_max(0.0f, 1.0f - sx * sx - sy * sy));
        light = U * sx + Vt * sy + N * z;
    } else {
        const float w = sqrtf(1.0f - uz * uz);
        const float dx = cs * w, dy = sn * w;
        light = U * dx + Vt * dy - N * uz;
    }
    return true;
}

// ---- probe / sky (probe.h, scene.h:161-181) -------------------------------------------------------

// ProbeDirToUV, probe.h:105-113 (out of line: the double-precision acos/atan2 are large); returns (u, v)
TB_NOINLINE float2 probe_dir_to_uv(V3 dir)
{
    const float theta = tbm_acosf(tb_clamp(dir.y, -1.0f, 1.0f));
    const float phi = (dir.x == 0.0f && dir.z == 0.0f) ? 0.0f : tbm_atan2f(dir.z, dir.x);
    return make_float2((TB_PI + phi) * TB_INV_PI * 0.5f, theta * TB_INV_PI);
}

// ProbeEval, probe.h:128-134
TB_DEV V3 probe_eval(const DProbe& pr, float u, float v)
{
    const int px = tb_clamp(int(u * pr.width), 0, pr.width - 1);
    const int py = tb_clamp(int(v * pr.height), 0, pr.height - 1);
    const float4 c = __ldg(&pr.data[py * pr.width + px]);
    return v3(c.x, c.y, c.z);
}

// ProbePdf, probe.h:136-160, given uv = ProbeDirToUV(d)
TB_DEV float probe_pdf(const DProbe& pr, float u, float v)
{
    const int col = tb_clamp(int(u * pr.width), 0, pr.width - 1);
    const int row = tb_clamp(int(v * pr.height), 0, pr.height - 1);
    float pdf = __ldg(&pr.pdfX[row * pr.width + col]) * __ldg(&pr.pdfY[row]);
    const float sinTheta = tbm_sinf(v * TB_PI);
    if (fabsf(sinTheta) < 0.0001f)
        pdf = 0.0f;
    else
        pdf *= float(pr.width) * float(pr.height) / (2.0f * TB_PI * TB_PI * sinTheta);
    return pdf;
}

// LowerBound(const float*, int, int, float), probe.h:186-203
TB_DEV int lower_bound_f(const float* arr, int lower, int upper, float value)
{
    while (lower < upper) {
        const int mid = lower + (upper - lower) / 2;
        if (__ldg(&arr[mid]) < value)
            lower = mid + 1;
        else
            upper = mid;
    }
    return lower;
}

// ProbeSample, probe.h:205-236
TB_DEV void probe_sample(const DProbe& pr, V3& dir, V3& color, float& pdf, Rng& rng)
{
    const float r1 = rng_float(rng);
    const float r2 = rng_float(rng);
    const int row = lower_bound_f(pr.cdfY, 0, pr.height, r1);
    const int col = lower_bound_f(pr.cdfX, row * pr.width, (row + 1) * pr.width, r2) - row * pr.width;
    const float4 c = __ldg(&pr.data[row * pr.width + col]);
    color = v3(c.x, c.y, c.z);
    pdf = __ldg(&pr.pdfX[row * pr.width + col]) * __ldg(&pr.pdfY[row]);
    const float u = col / float(pr.width);
    const float v = row / float(pr.height);
    const float sinTheta = tbm_sinf(v * TB_PI);
    if (sinTheta == 0.0f)
        pdf = 0.0f;
    else
        pdf *= (pr.width * pr.height) / (2.0f * TB_PI * TB_PI * sinTheta);
    // ProbeUVToDir, probe.h:115-125
    const float theta = v * TB_PI;
    const float phi = u * 2.0f * TB_PI;
    const float2 sct = tb_sincosf(theta), scp = tb_sincosf(phi);
    const float st = sct.x, ct = sct.y, sp = scp.x, cp = scp.y;
    dir = v3(-st * cp, ct, -st * sp);
}

// Sky::Eval, scene.h:168-178, given uv = ProbeDirToUV(dir) when the sky has a probe
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV V3 sky_eval(const DScene& sc, V3 dir, float u, float v)
{
    if ((FEAT & TB_FEAT_PROBE) && sc.probe.valid) return probe_eval(sc.probe, u, v);
    return tb_lerp(sc.horizon, sc.zenith, sqrtf(tb_abs(dir.y)));
}

// ---- light sampling (intersection.h:855-904) --------------------------------------------------

// PrimitiveSample
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV void prim_sample(const DScene& sc, const DPrim& p, float time, V3& pos, V3& normal, Rng& rng)
{
    const Xf xf = prim_transform<FEAT>(p, time);
    if (p.type == TB200_SPHERE) {
        const float u1 = rng_float(rng);
        const float u2 = rng_float(rng);
        pos = transform_point(xf, uniform_sample_sphere(u1, u2) * p.radius);
        normal = normalize(pos - xf.p);
        return;
    }
    if (p.type == TB200_MESH) {
        const DMesh& m = sc.meshes[p.mesh];
        const float r = rng_float(rng);
        // LowerBound(cdf, cdf+n, r) (probe.h:162-183) then Min(idx, n-1)
        const int tri = tb_min(lower_bound_f(m.cdf, 0, m.numTris, r), m.numTris - 1);
        // UniformSampleTriangle, maths.h:1312-1317
        const float sr = sqrtf(rng_float(rng));
        const float u = 1.0f - sr;
        const float v = rng_float(rng) * sr;
        const float4 q0 = __ldg(&m.triVerts[tri * 3 + 0]), q1 = __ldg(&m.triVerts[tri * 3 + 1]), q2 = __ldg(&m.triVerts[tri * 3 + 2]);
        const float4 m0 = __ldg(&m.triNormals[tri * 3 + 0]), m1 = __ldg(&m.triNormals[tri * 3 + 1]), m2 = __ldg(&m.triNormals[tri * 3 + 2]);
        const V3 a = v3(q0.x, q0.y, q0.z), b = v3(q0.w, q1.x, q1.y), c = v3(q1.z, q1.w, q2.x);
        const V3 n1 = v3(m0.x, m0.y, m0.z), n2 = v3(m0.w, m1.x, m1.y), n3 = v3(m1.z, m1.w, m2.x);
        pos = transform_point(xf, u * a + v * b + (1.0f - u - v) * c);
        normal = safe_normalize(transform_vector(xf, u * n1 + v * n2 + (1.0f - u - v) * n3), v3s(0.0f));
        return;
    }
    // planes cannot be lights (assert(0) in the reference)
    pos = v3s(0.0f);
    normal = v3s(0.0f);
}

// ---- path state and the PathTrace stages ------------------------------------------------------

struct PathState {
    V3 o, d;            // rayOrigin, rayDir
    float time;         // rayTime
    V3 T;               // pathThroughput
    V3 L;               // totalRadiance
    float eta;          // rayEta
    V3 absorb;          // rayAbsorption
    int rayType;        // BSDFType of the last bounce
    float bsdfPdf;
    Rng rng;
};

// what SampleLights / BSDFSample need to know about the surface point (render.cpp:255-278)
struct Surface {
    int prim;
    V3 p, n, wo;
    float etaI, etaO;
    V3 outAbsorb;
};

struct ShadowRay {
    V3 o, d;
    float dist;         // sqrtf(dSq); < 0 marks the probe sample
    V3 lightN;          // light normal, or the probe colour for the probe sample
    float skyPdf;
    int light;          // index of the sampled primitive
};

TB_DEV void path_init(PathState& ps, V3 origin, V3 dir, float time, Rng rng)
{
    ps.o = origin;
    ps.d = dir;
    ps.time = time;
    ps.T = v3s(1.0f);
    ps.L = v3s(0.0f);
    ps.eta = 1.0f;
    ps.absorb = v3s(0.0f);
    ps.rayType = TB_REFLECTED;
    ps.bsdfPdf = 1.0f;
    ps.rng = rng;
}

// Miss branch, render.cpp:365-384.  Always terminates the path.
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV void path_miss(const DScene& sc, PathState& ps, int bounce)
{
    float weight = 1.0f;
    float u = 0.0f, v = 0.0f;
    if ((FEAT & TB_FEAT_PROBE) && sc.probe.valid) {
        // shared by ProbePdf and Sky::Eval (both call ProbeDirToUV(rayDir))
        const float2 uv = probe_dir_to_uv(ps.d);
        u = uv.x;
        v = uv.y;
    }
    if ((FEAT & TB_FEAT_PROBE) && sc.probe.valid && bounce > 0 && ps.rayType != TB_SPECULAR) {
        const float skyPdf = probe_pdf(sc.probe, u, v);
        const float cbsdf = 0.5f, csky = 0.5f;   // kBsdfSamples/N, kProbeSamples/N with N = 2
        weight = cbsdf * ps.bsdfPdf / (cbsdf * ps.bsdfPdf + csky * skyPdf);
    }
    ps.L = ps.L + weight * sky_eval<FEAT>(sc, ps.d, u, v) * ps.T;
}

// Hit prologue, render.cpp:255-310: medium bookkeeping, Beer-Lambert, emission with MIS.
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV void path_hit(const DScene& sc, PathState& ps, const Hit& h, int bounce, Surface& sf)
{
    const DPrim& prim = sc.prims[h.prim];
    if (ps.eta == 1.0f) {
        sf.etaO = prim.mat.ior;
        sf.outAbsorb = prim.mat.absorption;
    } else {
        sf.etaO = 1.0f;
        sf.outAbsorb = v3s(0.0f);
    }
    // pathThroughput *= Exp(-rayAbsorption*t), render.cpp:272.  With zero absorption the argument is
    // -0*t = -0 and expf(-0) = 1 exactly, so the multiply is the identity and is skipped.
    // Without FEAT_ABSORPTION every material's absorption is 0, so ps.absorb only ever holds +-0.
    if ((FEAT & TB_FEAT_ABSORPTION) && !(ps.absorb.x == 0.0f && ps.absorb.y == 0.0f && ps.absorb.z == 0.0f)) {
        const V3 e = -ps.absorb * h.t;
        ps.T = ps.T * v3(tb_expf(e.x), tb_expf(e.y), tb_expf(e.z));
    }

    sf.prim = h.prim;
    sf.p = ps.o + ps.d * h.t;
    sf.n = h.n;
    sf.wo = -ps.d;
    sf.etaI = ps.eta;

    if (bounce == 0) {
        ps.L = ps.L + prim.mat.emission;
    } else {
        const float lightArea = prim.area;
        if (lightArea > 0.0f) {
            const float lightPdf = ((1.0f / lightArea) * h.t * h.t) / tb_clamp(dot(-ps.d, h.n), 1.e-3f, 1.0f);
            const int N = int(prim.lightSamples + 1.0f);
            const float cbsdf = 1.0f / N;
            const float clight = float(prim.lightSamples) / N;
            float weight = cbsdf * ps.bsdfPdf / (cbsdf * ps.bsdfPdf + clight * lightPdf);
            if (ps.rayType == TB_SPECULAR) weight = 1.0f;
            ps.L = ps.L + weight * ps.T * prim.mat.emission;
        }
    }
}

// SampleLights is unrolled into numNee slots processed in order: slot 0 is the probe sample
// (if the sky has a probe), then for every primitive with lightSamples>0, in scene order, one
// slot per sample (render.cpp:107-224).  nee_slot_light() maps a slot to its primitive.
struct NeeCursor {
    int slot;        // next slot (only compared with 0: the ring wavefront stores it as one bit)
    int prim;        // primitive scan position
    int sample;      // sample index within the current light
    V3 sum;          // running `sum`
    V3 Lacc;         // running `L` of the current light
};

// firstLight: no primitive before it has lightSamples > 0 (0 when not known)
TB_DEV void nee_begin(NeeCursor& c, int firstLight = 0)
{
    c.slot = 0;
    c.prim = firstLight;
    c.sample = 0;
    c.sum = v3s(0.0f);
    c.Lacc = v3s(0.0f);
}

// Generates the next shadow ray (drawing the RNG exactly as the reference does).  Returns
// false when all slots are exhausted.  lightEnd: no primitive from there on has lightSamples > 0
// (sc.numPrims when not known); the scan for the next light stops there.
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV bool nee_generate(const DScene& sc, const Surface& sf, float time, NeeCursor& c, Rng& rng, ShadowRay& sr, int lightEnd)
{
    if ((FEAT & TB_FEAT_PROBE) && c.slot == 0 && sc.probe.valid) {
        V3 wi, color;
        float pdf;
        probe_sample(sc.probe, wi, color, pdf, rng);
        sr.o = sf.p + face_forward(sf.n, wi) * TB_RAY_EPS;
        sr.d = wi;
        sr.dist = -1.0f;
        sr.lightN = color;
        sr.skyPdf = pdf;
        sr.light = -1;
        c.slot = 1;
        return true;
    }
    // advance to the next primitive that still has samples to take
    while (c.prim < lightEnd && c.sample >= sc.prims[c.prim].lightSamples) {
        c.prim++;
        c.sample = 0;
    }
    if (c.prim >= lightEnd) return false;
    const DPrim& light = sc.prims[c.prim];
    V3 lightPos, lightNormal;
    prim_sample<FEAT>(sc, light, time, lightPos, lightNormal, rng);
    V3 wi = lightPos - sf.p;
    const float dSq = length_sq(wi);
    wi = wi / sqrtf(dSq);
    sr.o = sf.p + face_forward(sf.n, wi) * TB_RAY_EPS;
    sr.d = wi;
    sr.dist = sqrtf(dSq);
    sr.lightN = lightNormal;
    sr.skyPdf = 0.0f;
    sr.light = c.prim;
    c.slot++;
    return true;
}

TB_DEV bool nee_generate(const DScene& sc, const Surface& sf, float time, NeeCursor& c, Rng& rng, ShadowRay& sr)
{
    return nee_generate<>(sc, sf, time, c, rng, sr, sc.numPrims);
}

// Consumes the traced shadow ray of the slot generated last; accumulates into the cursor in the
// reference's order (render.cpp:122-143 for the probe, :176-224 for area lights).
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV void nee_connect(const DScene& sc, const Surface& sf, const ShadowRay& sr, const Hit& sh, NeeCursor& c)
{
    const DMaterial& mat = sc.prims[sf.prim].mat;
    const bool isProbe = (FEAT & TB_FEAT_PROBE) && sr.light < 0;   // only the probe sample has no light
    // decide first whether BSDFPdf/BSDFEval are needed at all (both are pure), then evaluate them
    // once for whichever kind of sample this is
    float nl = 0.0f;
    bool need;
    if (isProbe) {
        need = sh.prim < 0;                                   // unoccluded probe direction, render.cpp:122
    } else {
        need = false;
        if (sh.prim >= 0 && fabsf(sh.t - sr.dist) <= 1.e-2f) {   // render.cpp:176-184
            nl = tb_abs(dot(sr.lightN, sr.d));
            need = !(tb_abs(nl) < 1.e-6f);                    // render.cpp:190-191 `continue`
        }
    }
    V3 f = v3s(0.0f);
    float bsdfPdf = 0.0f;
    if (need) {
        const BsdfValue b = bsdf_eval_pdf<FEAT>(mat, sf.etaI, sf.etaO, sf.n, sf.wo, sr.d);
        f = b.f;
        bsdfPdf = b.pdf;
    }

    if (isProbe) {
        if (need && bsdfPdf > 0.0f) {
            const float cbsdf = 0.5f, csky = 0.5f;
            const float skyPdf = sr.skyPdf;
            const float weight = csky * skyPdf / (cbsdf * bsdfPdf + csky * skyPdf);
            if (weight > 0.0f) c.sum = c.sum + weight * sr.lightN * f * tb_abs(dot(sr.d, sf.n)) / skyPdf;
        }
        // `sum /= float(kProbeSamples)` multiplies by 1.0: no-op
        return;
    }
    const DPrim& light = sc.prims[sr.light];
    if (need && bsdfPdf > 0.0f) {
        const float tSq = sh.t * sh.t;
        const float lightPdf = ((1.0f / light.area) * tSq) / nl;
        const int N = int(light.lightSamples + 1.0f);
        const float cbsdf = 1.0f / N;
        const float clight = float(light.lightSamples) / N;
        const float weight = clight * lightPdf / (cbsdf * bsdfPdf + clight * lightPdf);
        // emission of whatever the shadow ray hit, not of the sampled light (render.cpp:217)
        c.Lacc = c.Lacc + weight * f * sc.prims[sh.prim].mat.emission * (tb_abs(dot(sr.d, sf.n)) / tb_max(1.e-3f, lightPdf));
    }
    c.sample++;
    if (c.sample >= light.lightSamples) {
        c.sum = c.sum + c.Lacc * (1.0f / light.lightSamples);
        c.Lacc = v3s(0.0f);
    }
}

// After NEE: light-hit termination, BSDF sampling, throughput and medium update, next ray
// (render.cpp:314-363).  Returns false when the path ends here.
template <uint32_t FEAT = TB_FEAT_ALL>
TB_DEV bool path_scatter(const DScene& sc, PathState& ps, const Surface& sf, V3 neeSum)
{
    ps.L = ps.L + ps.T * neeSum;

    const DPrim& prim = sc.prims[sf.prim];
    if (prim.lightSamples) return false;

    V3 u, v;
    basis_from_vector(sf.n, &u, &v);
    V3 bsdfDir = v3s(0.0f);
    int bsdfType = TB_REFLECTED;
    float pdf = 0.0f;
    const bool pdfFromBsdf = bsdf_sample_dir<FEAT>(prim.mat, sf.etaI, sf.etaO, u, v, sf.n, sf.wo, bsdfDir, pdf, bsdfType, ps.rng);
    V3 f = v3s(0.0f);
    if (pdfFromBsdf || pdf > 0.0f) {
        // pdf = BSDFPdf(dir) (disney.h:291) and f = BSDFEval(dir) (render.cpp:341) share one call
        const BsdfValue b = bsdf_eval_pdf<FEAT>(prim.mat, sf.etaI, sf.etaO, sf.n, sf.wo, bsdfDir);
        f = b.f;
        if (pdfFromBsdf) pdf = b.pdf;
    }
    ps.bsdfPdf = pdf;
    if (pdf <= 0.0f) return false;

    if (dot(bsdfDir, sf.n) <= 0.0f) {
        ps.eta = sf.etaO;
        ps.absorb = sf.outAbsorb;
    }
    ps.T = ps.T * (f * tb_abs(dot(sf.n, bsdfDir)) / pdf);
    ps.rayType = bsdfType;
    ps.d = bsdfDir;
    ps.o = sf.p + face_forward(sf.n, bsdfDir) * TB_RAY_EPS;
    return true;
}
