// oracle_aov.cpp — the CPU oracle's auxiliary buffers of a render's camera samples: the reference answer of
// rtb200_scene_aov[_device] (include/rtb200.h, DESIGN.md §4.14). Test infrastructure, built beside the tests by
// tests/oracle_aov.py (and __graft_entry__.build()) with the oracle's own flags; the oracle's sources are only included.
#include <cfloat>

#include "../oracle/rt_oracle.hpp"

using namespace rto;

// The attenuation Material::scatter (materials.rs:44-54) returns at h, taken without its random draws: the albedo as stored
// for Lambertian and Metal (also where a Metal's scatter would absorb), texture_get_albedo for Texture, white otherwise.
static Rgb albedo_at(const Scene& sc, const rt_sphere& sp, const Hit& h, Stats& st) {
    switch (sp.kind) {
    case RT_LAMBERTIAN:
    case RT_METAL: return Rgb{sp.albedo[0], sp.albedo[1], sp.albedo[2]};
    case RT_TEXTURE: return texture_get_albedo(sc.s->textures[sp.texture], sp.param, h.u, h.v, st);
    default: return Rgb{1.0f, 1.0f, 1.0f};   // Glass (materials.rs:184), Light (materials.rs:67)
    }
}

extern "C" {

// For every pixel (x, y) of the frame, top row first, and every sample s in [sample0, sample0 + samples): the render's primary
// ray (raytracer.rs:199-201 from the stream of (pixel y * width + x, sample s) under the scene's seed, camera.rs:79-84 with the
// scene's camera) and H = hit_world(world, ray, 0.001, f64::MAX). Per pixel, f32 sums in sample order times 1.0f / samples of
// the albedo at H (the sky of the ray on a miss) and of H's normal rounded to f32 (0 on a miss); the samples with a hit; the
// sphere (0xffffffff on a miss) and ray.at(t) (0 on a miss) of sample sample0. Every output may be NULL. OpenMP over pixels.
int oracle_aov(const rt_scene* s, uint32_t samples, uint32_t sample0, float* albedo, float* normal, uint32_t* hits, uint32_t* sphere,
               double* point) {
    if (!s || samples == 0 || (uint64_t)sample0 + samples > (1ull << 32)) return -1;
    const Scene sc(s);
    const uint64_t w = s->width, h = s->height;
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t k = 0; k < (int64_t)(w * h); ++k) {
        const uint64_t i = (uint64_t)k;
        const uint32_t x = (uint32_t)(i % w), y = (uint32_t)(i / w);
        Stats st;
        float a[3] = {0.0f, 0.0f, 0.0f}, n[3] = {0.0f, 0.0f, 0.0f};
        uint32_t nh = 0, sph = 0xffffffffu;
        P3 pt{0.0, 0.0, 0.0};
        for (uint32_t j = 0; j < samples; ++j) {
            SampleRng rng(s->seed, y * s->width + x, sample0 + j);
            const double u = ((double)x + rng.gen_f64()) / ((double)s->width - 1.0);
            const double v = ((double)s->height - ((double)y + rng.gen_f64())) / ((double)s->height - 1.0);
            const Ray r = get_ray(s->camera, u, v);
            Hit hit{};
            Rgb c;
            float hn[3] = {0.0f, 0.0f, 0.0f};
            if (hit_world(sc, r, 0.001, DBL_MAX, &hit, st)) {
                c = albedo_at(sc, s->spheres[hit.sphere], hit, st);
                hn[0] = (float)hit.normal.x; hn[1] = (float)hit.normal.y; hn[2] = (float)hit.normal.z;
                ++nh;
                if (j == 0) { sph = (uint32_t)hit.sphere; pt = hit.point; }
            } else {
                c = sky_color(sc, r);
            }
            a[0] += c.r; a[1] += c.g; a[2] += c.b;
            n[0] += hn[0]; n[1] += hn[1]; n[2] += hn[2];
        }
        const float scale = 1.0f / (float)samples;
        for (int q = 0; q < 3; ++q) {
            if (albedo) albedo[3 * i + q] = scale * a[q];
            if (normal) normal[3 * i + q] = scale * n[q];
        }
        if (hits) hits[i] = nh;
        if (sphere) sphere[i] = sph;
        if (point) { point[3 * i] = pt.x; point[3 * i + 1] = pt.y; point[3 * i + 2] = pt.z; }
    }
    return 0;
}

}  // extern "C"
