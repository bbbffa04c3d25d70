// oracle_trace_rays.cpp — the CPU oracle's ray_color (oracle/rt_oracle.hpp, raytracer.rs:71-165) on caller-supplied primary
// rays: the reference answer of rtb200_scene_trace_rays[_device] (include/rtb200.h). Test infrastructure, built beside the
// tests by tests/oracle_trace_rays.py (and __graft_entry__.build()) with the oracle's own flags; the oracle's sources are
// only included.
#include "../oracle/rt_oracle.hpp"

using namespace rto;

extern "C" {

// For ray i and sample j < samples: ray_color(Ray{origin[3i..], direction[3i..]}, max_depth, max_depth) with the scene's seed
// and max_depth, on the stream of (pixel stream0 + i, sample sample0 + j) after its first two f64 draws (the render's pixel
// jitter, raytracer.rs:199-200). Outputs the render's resolve with spp = samples (render_pixel): linear = (1.0f / samples) *
// the f32 sum in sample order, rgb8 = quantise(sqrt(linear)); either may be NULL. *rays (may be NULL): hit_world calls.
// OpenMP over rays.
int oracle_trace_rays(const rt_scene* s, const double* origin, const double* direction, uint32_t n, uint32_t samples,
                      uint32_t sample0, uint32_t stream0, float* out_linear, uint8_t* out_rgb8, uint64_t* rays) {
    if (!s || samples == 0 || (n && (!origin || !direction))) return -1;
    const Scene sc(s);
    if (sc.lights.size() >= 10) return -4;   // the reference recursion does not terminate when n_lights * prob >= 1
    uint64_t total = 0;
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : total)
    for (int64_t k = 0; k < (int64_t)n; ++k) {
        const size_t i = (size_t)k;
        const Ray r{P3{origin[3 * i], origin[3 * i + 1], origin[3 * i + 2]}, P3{direction[3 * i], direction[3 * i + 1], direction[3 * i + 2]}};
        Stats st;
        float acc[3] = {0.0f, 0.0f, 0.0f};
        for (uint32_t j = 0; j < samples; ++j) {
            SampleRng rng(s->seed, stream0 + (uint32_t)i, sample0 + j);
            rng.gen_f64();
            rng.gen_f64();
            const Rgb c = ray_color(sc, r, s->max_depth, s->max_depth, rng, st, nullptr, nullptr);
            acc[0] += c.r; acc[1] += c.g; acc[2] += c.b;
        }
        const float scale = 1.0f / (float)samples;
        for (int c = 0; c < 3; ++c) {
            const float mean = scale * acc[c];
            if (out_linear) out_linear[3 * i + c] = mean;
            if (out_rgb8) out_rgb8[3 * i + c] = quantise_u8(std::sqrt(mean));
        }
        total += st.rays;
    }
    if (rays) *rays = total;
    return 0;
}

}  // extern "C"
