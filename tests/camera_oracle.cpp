// camera_oracle.cpp -- TEST INFRASTRUCTURE: the CPU restatement's camera samples over a batch of (pixel, frame)
// records, the arm the device's camera-ray query (tb200_camera_rays) is checked against.  It compiles the
// restatement (oracle/tinsel_oracle.cpp) unchanged into the same translation unit and applies its make_camera(),
// rng_make(), rng_f(), mixf() and generate_ray() in the order its trace_sample() does (render.cpp:476-482).
// tests/test_camera_splat.py checks the result against that library's own oracle_trace_frame() raster positions and
// oracle_generate_ray(), so the draws here are trace_sample's.  tests/cameraoracle.py builds it with oracle/Makefile's
// flags into a temporary directory and loads it.
#include "oracle/tinsel_oracle.cpp"

extern "C" {

// The camera samples of n (pixel, frame) records (pixelFrame[2k], pixelFrame[2k+1]) of a W x H image, drawn as
// trace_sample draws them: origin[3k..], dir[3k..], time[k], raster[2k..].  A pixel outside [0, W*H) gives a zero
// origin, direction and time and a NaN raster position.
void oracle_camera_samples(const tb200_camera* cam, int W, int H, long long n, const int32_t* pixelFrame, float* origin,
                           float* dir, float* time, float* raster)
{
    const camera_t cs = make_camera(*cam, W, H);
    for (long long k = 0; k < n; ++k) {
        const int p = pixelFrame[2 * k];
        vec3 o = splat(0.0f), d = splat(0.0f);
        float t = 0.0f, rx = NAN, ry = NAN;
        if (p >= 0 && (long long)p < (long long)W * H) {
            const int i = p % W, j = p / W;
            rng_t rng = rng_make(tb200_sample_seed((uint32_t)(j * W + i), (uint32_t)pixelFrame[2 * k + 1]));
            float x = rng_f(rng), y = rng_f(rng);
            const float u = rng_f(rng);
            t = mixf(cam->shutterStart, cam->shutterEnd, u);
            x += i;
            y += j;
            generate_ray(cs, x, y, o, d);
            rx = x;
            ry = y;
        }
        origin[3 * k + 0] = o.x; origin[3 * k + 1] = o.y; origin[3 * k + 2] = o.z;
        dir[3 * k + 0] = d.x; dir[3 * k + 1] = d.y; dir[3 * k + 2] = d.z;
        time[k] = t;
        raster[2 * k + 0] = rx; raster[2 * k + 1] = ry;
    }
}

}  // extern "C"
