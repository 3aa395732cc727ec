// light_oracle.cpp -- TEST INFRASTRUCTURE: the CPU restatement's SampleLights over a batch of surface records, the
// arm the device's next-event-estimation query (tb200_sample_lights) is checked against, and its PathTrace with the
// random-number stream cut at every call, the arm a path built from the queries is checked against.  It compiles
// the restatement (oracle/tinsel_oracle.cpp) unchanged into the same translation unit and applies its
// sample_lights(), whose results the restatement's own oracle_trace_frame golden vectors pin.  tests/lightoracle.py
// builds it with oracle/Makefile's flags into a temporary directory and loads it.
#include "oracle/tinsel_oracle.cpp"

extern "C" {

// records: n tb200_light_query records; out[3k..3k+2] = sample_lights(scene, primitives[prim], etaI, etaO, p, n, wo,
// time, Random(seeds[k])).  A prim outside [0, numPrimitives) gives zeros.
void oracle_sample_lights(const tb200_scene* scene, long long n, const tb200_light_query* records, const uint32_t* seeds,
                          float* out)
{
    for (long long k = 0; k < n; ++k) {
        const tb200_light_query& q = records[k];
        vec3 s = splat(0.0f);
        if (q.prim >= 0 && q.prim < scene->numPrimitives) {
            rng_t rng = rng_make(seeds[k]);
            s = sample_lights(*scene, scene->primitives[q.prim], q.etaI, q.etaO, from(q.p), from(q.n), from(q.wo), q.time, rng);
        }
        out[3 * k + 0] = s.x; out[3 * k + 1] = s.y; out[3 * k + 2] = s.z;
    }
}

// path_trace() of the restatement, line for line, for n rays (origin[3k..], dir[3k..], time[k]), except that each
// call that draws random numbers starts from its own seed: bounce b's sample_lights from Random(seeds[2(k*maxDepth+b)])
// and its bsdf_sample from Random(seeds[2(k*maxDepth+b)+1]).  Writes radiance[3k..3k+2], length[k] (the Trace calls
// the path made) and prims[k*maxDepth+b] (bounce b's hit primitive, -1 on a miss, -2 after the path ended).
void oracle_path_trace_reseeded(const tb200_scene* scene, long long n, const float* origin, const float* dir,
                                const float* time, int maxDepth, const uint32_t* seeds, float* radiance, int32_t* length,
                                int32_t* prims)
{
    const tb200_scene& sc = *scene;
    for (long long k = 0; k < n; ++k) {
        const uint32_t* sd = seeds + 2 * (size_t)k * maxDepth;
        int32_t* hp = prims + (size_t)k * maxDepth;
        for (int b = 0; b < maxDepth; ++b) hp[b] = -2;
        vec3 T = splat(1.0f), total = splat(0.0f);
        vec3 ro = from(origin + 3 * k), rd = from(dir + 3 * k);
        float rayEta = 1.0f;
        vec3 rayAbs = splat(0.0f);
        int rayType = REFLECTED;
        float bsdfPdf = 1.0f;
        int len = 0;
        for (int i = 0; i < maxDepth; ++i) {
            hit_t h = closest_hit(sc, ro, rd, time[k]);
            ++len;
            hp[i] = h.prim < 0 ? -1 : h.prim;
            if (h.prim >= 0) {
                const tb200_primitive& prim = sc.primitives[h.prim];
                float outEta;
                vec3 outAbs;
                if (rayEta == 1.0f) {
                    outEta = mat_ior(prim.material);
                    outAbs = from(prim.material.absorption);
                } else {
                    outEta = 1.0f;
                    outAbs = splat(0.0f);
                }
                vec3 e = scale(neg(rayAbs), h.t);
                T = mul(T, mk(tbm_expf(e.x), tbm_expf(e.y), tbm_expf(e.z)));
                vec3 p = add(ro, scale(rd, h.t));
                vec3 nn = h.n;
                vec3 emission = from(prim.material.emission);
                if (i == 0) {
                    total = add(total, emission);
                } else {
                    float area = prim_area(sc, prim);
                    if (area > 0.0f) {
                        float lightPdf = ((1.0f / area) * h.t * h.t) / clampf(dot3(neg(rd), nn), 1.e-3f, 1.0f);
                        int N = int(prim.lightSamples + 1.0f);
                        float cbsdf = 1.0f / N, clight = float(prim.lightSamples) / N;
                        float weight = cbsdf * bsdfPdf / (cbsdf * bsdfPdf + clight * lightPdf);
                        if (rayType == SPECULAR) weight = 1.0f;
                        total = add(total, mul(scale(T, weight), emission));
                    }
                }
                rng_t neeRng = rng_make(sd[2 * i]);
                total = add(total, mul(T, sample_lights(sc, prim, rayEta, outEta, p, nn, neg(rd), time[k], neeRng)));
                if (prim.lightSamples) break;
                vec3 u, v;
                basis(nn, u, v);
                vec3 bdir = splat(0.0f);
                int btype = REFLECTED;
                rng_t bsdfRng = rng_make(sd[2 * i + 1]);
                bsdf_sample(prim.material, rayEta, outEta, u, v, nn, neg(rd), bdir, bsdfPdf, btype, bsdfRng);
                if (bsdfPdf <= 0.0f) break;
                vec3 f = bsdf_eval(prim.material, rayEta, outEta, nn, neg(rd), bdir);
                if (dot3(bdir, nn) <= 0.0f) {
                    rayEta = outEta;
                    rayAbs = outAbs;
                }
                T = mul(T, divs(scale(f, absf(dot3(nn, bdir))), bsdfPdf));
                rayType = btype;
                rd = bdir;
                ro = add(p, scale(face_fwd(nn, bdir), RAY_EPS));
            } else {
                float weight = 1.0f;
                if (sc.sky.probeValid && i > 0 && rayType != SPECULAR) {
                    float skyPdf = probe_pdf(sc.sky, rd);
                    float cbsdf = 1.0f / 2, csky = 1.0f / 2;
                    weight = cbsdf * bsdfPdf / (cbsdf * bsdfPdf + csky * skyPdf);
                }
                total = add(total, mul(scale(sky_eval(sc.sky, rd), weight), T));
                break;
            }
        }
        radiance[3 * k + 0] = total.x; radiance[3 * k + 1] = total.y; radiance[3 * k + 2] = total.z;
        length[k] = len;
    }
}

}  // extern "C"
