// emitter_oracle.cpp -- TEST INFRASTRUCTURE: the CPU restatement's PrimitiveSample and ProbeSample over a batch, the
// arms the device's emitter and probe sample queries (tb200_sample_emitters, tb200_sample_probe) are checked against,
// and its SampleLights with a seed per slot, the arm a SampleLights built from those queries is checked against.  It
// compiles the restatement (oracle/tinsel_oracle.cpp) unchanged into the same translation unit and applies its
// prim_sample(), probe_sample() and sample_lights() arithmetic.  tests/emitteroracle.py builds it with
// oracle/Makefile's flags into a temporary directory and loads it.
#include "oracle/tinsel_oracle.cpp"

extern "C" {

// records: n tb200_emitter_query records; out[8k..8k+7] = pos, 0, normal, 0 of prim_sample(scene, primitives[prim],
// time, Random(seeds[k])).  A primitive without lightSamples or outside [0, numPrimitives) gives zeros.
void oracle_sample_emitters(const tb200_scene* scene, long long n, const tb200_emitter_query* records, const uint32_t* seeds,
                            float* out)
{
    for (long long k = 0; k < n; ++k) {
        const tb200_emitter_query& q = records[k];
        vec3 pos = splat(0.0f), nrm = splat(0.0f);
        if (q.prim >= 0 && q.prim < scene->numPrimitives && scene->primitives[q.prim].lightSamples > 0) {
            rng_t rng = rng_make(seeds[k]);
            prim_sample(*scene, scene->primitives[q.prim], q.time, pos, nrm, rng);
        }
        float* o = out + 8 * k;
        o[0] = pos.x; o[1] = pos.y; o[2] = pos.z; o[3] = 0.0f;
        o[4] = nrm.x; o[5] = nrm.y; o[6] = nrm.z; o[7] = 0.0f;
    }
}

// out[8k..8k+7] = dir, pdf, color, 0 of probe_sample(scene's sky, Random(seeds[k])); zeros without a probe.
void oracle_sample_probe(const tb200_scene* scene, long long n, const uint32_t* seeds, float* out)
{
    for (long long k = 0; k < n; ++k) {
        vec3 d = splat(0.0f), c = splat(0.0f);
        float pdf = 0.0f;
        if (scene->sky.probeValid) {
            rng_t rng = rng_make(seeds[k]);
            probe_sample(scene->sky, d, c, pdf, rng);
        }
        float* o = out + 8 * k;
        o[0] = d.x; o[1] = d.y; o[2] = d.z; o[3] = pdf;
        o[4] = c.x; o[5] = c.y; o[6] = c.z; o[7] = 0.0f;
    }
}

// sample_lights() of the restatement, line for line, for n tb200_light_query records, except that each slot draws
// from its own Random(seeds[k*numSlots + s]).  The slots are those of SampleLights: slot 0 is the probe sample when
// the sky has a probe, then every primitive with lightSamples > 0 in scene order, one slot per sample.  Writes
// radiance[3k..3k+2] and, per slot, slots[2(k*numSlots + s)] = the shadow ray's hit primitive (-1 on a miss, -2 when
// nothing was traced) and slots[2(k*numSlots + s) + 1] = 1 when the sample reached the BSDF evaluation (the probe
// ray missed; a light ray's hit passed the distance and light-normal tests), else 0.  A prim outside
// [0, numPrimitives) gives zeros and traces nothing.
void oracle_sample_lights_per_slot(const tb200_scene* scene, long long n, const tb200_light_query* records,
                                   const uint32_t* seeds, int numSlots, float* radiance, int32_t* slots)
{
    const tb200_scene& sc = *scene;
    for (long long k = 0; k < n; ++k) {
        const tb200_light_query& q = records[k];
        const uint32_t* sd = seeds + (size_t)k * numSlots;
        int32_t* so = slots + 2 * (size_t)k * numSlots;
        for (int s = 0; s < numSlots; ++s) {
            so[2 * s] = -2;
            so[2 * s + 1] = 0;
        }
        vec3 sum = splat(0.0f);
        if (q.prim >= 0 && q.prim < sc.numPrimitives) {
            const tb200_primitive& surf = sc.primitives[q.prim];
            const float etaI = q.etaI, etaO = q.etaO, time = q.time;
            const vec3 p = from(q.p), n = from(q.n), wo = from(q.wo);
            int slot = 0;
            if (sc.sky.probeValid) {
                rng_t rng = rng_make(sd[slot]);
                vec3 wi, skyColor;
                float skyPdf;
                probe_sample(sc.sky, wi, skyColor, skyPdf, rng);
                hit_t sh = closest_hit(sc, add(p, scale(face_fwd(n, wi), RAY_EPS)), wi, time);
                so[2 * slot] = sh.prim < 0 ? -1 : sh.prim;
                if (sh.prim < 0) {
                    so[2 * slot + 1] = 1;
                    float bp = bsdf_pdf(surf.material, etaI, etaO, n, wo, wi);
                    vec3 f = bsdf_eval(surf.material, etaI, etaO, n, wo, wi);
                    if (bp > 0.0f) {
                        float cbsdf = 1.0f / 2, csky = 1.0f / 2;
                        float weight = csky * skyPdf / (cbsdf * bp + csky * skyPdf);
                        if (weight > 0.0f) sum = add(sum, divs(scale(mul(scale(skyColor, weight), f), absf(dot3(wi, n))), skyPdf));
                    }
                }
                sum = scale(sum, 1.0f);
                ++slot;
            }
            for (int i = 0; i < sc.numPrimitives; ++i) {
                const tb200_primitive& light = sc.primitives[i];
                int numSamples = light.lightSamples;
                if (numSamples == 0) continue;
                vec3 L = splat(0.0f);
                for (int s = 0; s < numSamples; ++s, ++slot) {
                    rng_t rng = rng_make(sd[slot]);
                    vec3 lightPos, lightNormal;
                    prim_sample(sc, light, time, lightPos, lightNormal, rng);
                    vec3 wi = sub(lightPos, p);
                    float dSq = dot3(wi, wi);
                    wi = divs(wi, sqrtf(dSq));
                    hit_t sh = closest_hit(sc, add(p, scale(face_fwd(n, wi), RAY_EPS)), wi, time);
                    so[2 * slot] = sh.prim < 0 ? -1 : sh.prim;
                    if (sh.prim < 0) continue;
                    float t = sh.t, tSq = t * t;
                    if (!(fabsf(t - sqrtf(dSq)) <= 1.e-2f)) continue;
                    float nl = absf(dot3(lightNormal, wi));
                    if (absf(nl) < 1.e-6f) continue;
                    so[2 * slot + 1] = 1;
                    float lightPdf = ((1.0f / prim_area(sc, light)) * tSq) / nl;
                    float bp = bsdf_pdf(surf.material, etaI, etaO, n, wo, wi);
                    vec3 f = bsdf_eval(surf.material, etaI, etaO, n, wo, wi);
                    if (bp > 0.0f) {
                        int N = int(light.lightSamples + 1.0f);
                        float cbsdf = 1.0f / N, clight = float(light.lightSamples) / N;
                        float weight = clight * lightPdf / (cbsdf * bp + clight * lightPdf);
                        vec3 e = from(sc.primitives[sh.prim].material.emission);
                        L = add(L, scale(mul(scale(f, weight), e), absf(dot3(wi, n)) / fmax2(1.e-3f, lightPdf)));
                    }
                }
                sum = add(sum, scale(L, 1.0f / numSamples));
            }
        }
        radiance[3 * k + 0] = sum.x; radiance[3 * k + 1] = sum.y; radiance[3 * k + 2] = sum.z;
    }
}

}  // extern "C"
