// tb_film.cuh -- camera ray generation and filtered framebuffer accumulation.
#pragma once

#include "tb_shade.cuh"

// CameraSampler (util.h:45-83) after the host has built the two matrices (api.cu, camera_setup).
struct DCamera {
    float r2w[16];      // rasterToWorld, column major (cols[c][r] = r2w[c*4+r])
    V3 origin;          // cameraToWorld.GetCol(3)
    float shutterStart, shutterEnd;
};

struct DFilm {
    int width, height;
    int filterType;
    float filterWidth, filterFalloff, filterOffset;
    float clamp;
    int maxDepth;
    // arguments below this give expf(arg) < offset by a wide margin, i.e. Gaussian() == +0 exactly
    // (host: log(offset*(1-1e-3)); -inf disables the shortcut)
    float filterArgZero;
    // Owner-computes row slabs (multi-GPU): splats land only in pixel rows [rowLo, rowHi).  A device
    // that owns a slab also traces the samples of the rows within the filter's reach outside it, so
    // its rows receive exactly the contributions the whole image would give them.  Default: all rows.
    int rowLo, rowHi;
};

// GenerateRay, util.h:73-79 with TransformPoint(Mat44, Vec3(x,y,0)), maths.h:923-930
TB_DEV void generate_ray(const DCamera& cam, float rx, float ry, V3& origin, V3& dir)
{
    const float* m = cam.r2w;
    V3 p;
    p.x = m[0] * rx + m[4] * ry + m[8] * 0.0f + m[12];
    p.y = m[1] * rx + m[5] * ry + m[9] * 0.0f + m[13];
    p.z = m[2] * rx + m[6] * ry + m[10] * 0.0f + m[14];
    origin = cam.origin;
    dir = normalize(p - origin);
}

// The camera sample of pixel (px, py) in `frame` of a `width`-pixel-wide image (render.cpp:476-482, with the
// per-(pixel, frame) seed): Random(tb_sample_seed(pixel, frame)), the draws x, y, t in the oracle's order, the shutter
// time, and GenerateRay through the jittered raster position (rasterX, rasterY), which is also where the sample is
// splatted.  `rng` is left after the three draws.  The renderer (sample_begin) and tb200_camera_rays both call this.
TB_DEV void camera_sample(const DCamera& cam, int width, int px, int py, uint32_t frame, Rng& rng, V3& origin, V3& dir,
                          float& time, float& rasterX, float& rasterY)
{
    rng = rng_seed(tb_sample_seed((uint32_t)(py * width + px), frame));
    float x = rng_float(rng);
    float y = rng_float(rng);
    const float t = rng_float(rng);
    time = tb_lerp(cam.shutterStart, cam.shutterEnd, t);
    x += px;
    y += py;
    generate_ray(cam, x, y, origin, dir);
    rasterX = x;
    rasterY = y;
}

// DFilm::filterArgZero for a filter offset (host).  Gaussian() is exactly +0 wherever expf(arg) < offset; keep a
// 1e-3 relative margin so the shortcut never depends on the last bits of expf.  -inf (shortcut off) unless the
// offset lies in (0, 1) and tbm_expf confirms the cut-off.
inline float film_filter_arg_zero(float filterOffset)
{
    if (!(filterOffset > 0.0f && filterOffset < 1.0f)) return -INFINITY;
    const float a = (float)log((double)filterOffset * (1.0 - 1.0e-3));
    return tbm_expf(a) < filterOffset ? a : -INFINITY;
}

// Filter::Gaussian, render.h:29-32 (offset is taken as handed in, never recomputed)
TB_DEV float filter_gaussian(const DFilm& f, float x)
{
    const float arg = -f.filterFalloff * x * x;
    if (arg < f.filterArgZero) return 0.0f;   // Max(0, expf(arg) - offset) with expf(arg) < offset
    return tb_max(0.0f, tb_expf(arg) - f.filterOffset);
}

// one 16-byte vector REDUCTION per touched pixel: red.global.add.v4.f32 (REDG.E.ADD.F32x4).  CUDA's
// atomicAdd(float4*) compiles to the value-returning form (ATOMG), which makes the warp wait a round trip
// to L2 for a result nobody reads; the reduction is fire-and-forget.  Same adder, same rounding.  (The L2
// vector adder flushes denormal sums to zero -- ".FTZ" in the SASS mnemonic -- where the CPU's `+=` keeps
// them: the one place this renderer is not IEEE-exact; irrelevant at the 1e-4 image tolerance, and
// per-sample radiance never passes through it.)
TB_DEV void accum_add(float4* accum, int idx, float r, float g, float b, float w)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(accum + idx), "f"(r), "f"(g), "f"(b), "f"(w) : "memory");
}

// CpuRenderer::AddSample, render.cpp:401-445.  Pixels whose weight is exactly zero are skipped
// when the sample is finite (adding +0 changes nothing); a non-finite sample takes the literal
// path so that it poisons the same pixels as in the reference.
TB_DEV void add_sample(const DFilm& f, float4* accum, float rasterX, float rasterY, V3 sample)
{
    const int startX = tb_max(0, int(rasterX - f.filterWidth));
    const int startY = tb_max(f.rowLo, int(rasterY - f.filterWidth));
    const int endX = tb_min(int(rasterX + f.filterWidth), f.width - 1);
    const int endY = tb_min(int(rasterY + f.filterWidth), f.rowHi - 1);

    // ClampLength, maths.h:1577-1589
    V3 c = sample;
    const float l = length(sample);
    if (l > f.clamp) c = sample * (f.clamp / l);

    if (f.filterType == TB200_FILTER_BOX) {
        for (int x = startX; x <= endX; ++x)
            for (int y = startY; y <= endY; ++y) accum_add(accum, y * f.width + x, c.x, c.y, c.z, 1.0f);
        return;
    }
    const bool finite = isfinite(c.x) && isfinite(c.y) && isfinite(c.z);
    for (int x = startX; x <= endX; ++x) {
        const float gx = filter_gaussian(f, x - rasterX);
        if (gx == 0.0f && finite) continue;
        for (int y = startY; y <= endY; ++y) {
            const float w = gx * filter_gaussian(f, y - rasterY);
            if (w == 0.0f && finite) continue;
            accum_add(accum, y * f.width + x, c.x * w, c.y * w, c.z * w, w);
        }
    }
}

// add_sample out of line: add_sample_small's fallback, which a 3x3 Gaussian footprint and a finite sample never take,
// so that its ~350 instructions stay out of the splat that calls it
TB_NOINLINE void add_sample_cold(const DFilm& f, float4* accum, float rasterX, float rasterY, V3 sample)
{
    add_sample(f, accum, rasterX, rasterY, sample);
}

// add_sample with the Gaussian's weights evaluated once per column and once per row: for a finite sample whose
// footprint is at most 3x3 pixels, the six filter_gaussian values are independent, inline expf chains that run
// side by side (add_sample makes up to twelve out-of-line calls, one after the other).  Each pixel's weight is
// still gx * gy, and the pixels whose weight is zero are still skipped, so every reduction carries the same bits.
// Anything else takes add_sample (add_sample_cold).
TB_DEV void add_sample_small(const DFilm& f, float4* accum, float rasterX, float rasterY, V3 sample)
{
    const int startX = tb_max(0, int(rasterX - f.filterWidth));
    const int startY = tb_max(f.rowLo, int(rasterY - f.filterWidth));
    const int endX = tb_min(int(rasterX + f.filterWidth), f.width - 1);
    const int endY = tb_min(int(rasterY + f.filterWidth), f.rowHi - 1);
    V3 c = sample;
    const float l = length(sample);
    if (l > f.clamp) c = sample * (f.clamp / l);
    if (f.filterType != TB200_FILTER_GAUSSIAN || endX - startX > 2 || endY - startY > 2 || !(isfinite(c.x) && isfinite(c.y) && isfinite(c.z))) {
        add_sample_cold(f, accum, rasterX, rasterY, sample);
        return;
    }
    float gx[3], gy[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        // filter_gaussian, with tbm_expf inline
        const float dx = (float)(startX + k) - rasterX, dy = (float)(startY + k) - rasterY;
        const float ax = -f.filterFalloff * dx * dx, ay = -f.filterFalloff * dy * dy;
        gx[k] = ax < f.filterArgZero ? 0.0f : tb_max(0.0f, tbm_expf(ax) - f.filterOffset);
        gy[k] = ay < f.filterArgZero ? 0.0f : tb_max(0.0f, tbm_expf(ay) - f.filterOffset);
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (startX + i > endX || gx[i] == 0.0f) continue;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const float w = gx[i] * gy[j];
            if (startY + j > endY || w == 0.0f) continue;
            accum_add(accum, (startY + j) * f.width + startX + i, c.x * w, c.y * w, c.z * w, w);
        }
    }
}
