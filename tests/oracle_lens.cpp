// oracle_lens.cpp — the CPU oracle's thin-lens camera (include/rtb200.h, DESIGN.md §4.17): the reference answer of
// rtb200_camera_from_params_lens, rtb200_probe_lens_ray, lens renders (rtb200_render_frames_lens, rtb200_scene_set_lens) and
// the auxiliary buffers of a lens handle. Test infrastructure, built beside the tests by tests/oracle_lens.py (and
// __graft_entry__.build()) with the oracle's own flags; the oracle's sources are only included.
#include <cfloat>

#include "../oracle/rt_oracle.hpp"

using namespace rto;

// Camera::new's basis (camera.rs:52-58), then the image plane at focus distance fd, in the order the contract writes it.
static void lens_camera(const rt_camera_params& p, double aperture, double fd, rt_camera* out, rt_lens* lens) {
    const double PI = 3.14159265358979323846264338327950288;
    const double theta = p.vfov_deg * (PI / 180.0);
    const double half_height = std::tan(theta / 2.0);
    const double half_width = p.aspect * half_height;
    const P3 w = unit_vector(p3(p.look_from) - p3(p.look_at));
    const P3 u = unit_vector(cross(p3(p.vup), w));
    const P3 v = cross(w, u);
    const P3 origin = p3(p.look_from);
    const P3 llc = ((origin - u * (half_width * fd)) - v * (half_height * fd)) - w * fd;
    const P3 hor = ((u * 2.0) * half_width) * fd, ver = ((v * 2.0) * half_height) * fd;
    out->origin = rt_vec3{origin.x, origin.y, origin.z};
    out->lower_left_corner = rt_vec3{llc.x, llc.y, llc.z};
    out->horizontal = rt_vec3{hor.x, hor.y, hor.z};
    out->vertical = rt_vec3{ver.x, ver.y, ver.z};
    *lens = rt_lens{rt_vec3{u.x, u.y, u.z}, rt_vec3{v.x, v.y, v.z}, aperture / 2.0, 0};
}

// gen_range(-1.0..1.0) of one u64
static double m1_1(uint64_t u) {
    uint64_t bits = (u >> 12) | 0x3FF0000000000000ull;
    double v12; std::memcpy(&v12, &bits, 8);
    return (v12 - 1.0) * 2.0 + (-1.0);
}

// The lens disk: trial k reads Philox block (k, sample, pixel, 1), one trial at a time; returns the trials drawn.
static uint32_t lens_disk(uint64_t seed, uint32_t pixel, uint32_t sample, double& x, double& y) {
    const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    for (uint32_t k = 0;; ++k) {
        const uint32_t ctr[4] = {k, sample, pixel, 1u};
        uint32_t w[4];
        Philox::block(ctr, key, w);
        x = m1_1(((uint64_t)w[1] << 32) | w[0]);
        y = m1_1(((uint64_t)w[3] << 32) | w[2]);
        if (x * x + y * y < 1.0) return k + 1;
    }
}

static Ray lens_ray(const rt_camera& cam, const rt_lens& L, uint64_t seed, uint32_t pixel, uint32_t sample, double u, double v,
                    uint32_t* trials) {
    Ray r = get_ray(cam, u, v);
    if (trials) *trials = 0;
    if (L.radius != 0.0) {
        double x, y;
        const uint32_t t = lens_disk(seed, pixel, sample, x, y);
        if (trials) *trials = t;
        const double rdx = L.radius * x, rdy = L.radius * y;
        const P3 off = p3(L.u) * rdx + p3(L.v) * rdy;
        r = Ray{r.origin + off, r.direction - off};
    }
    return r;
}

// The primary ray of pixel (x, y) and sample smp of scene s through lens L; rng is left after the two jitter draws.
static Ray primary(const rt_scene& s, const rt_lens& L, uint32_t x, uint32_t y, uint32_t smp, SampleRng& rng) {
    const double u = ((double)x + rng.gen_f64()) / ((double)s.width - 1.0);
    const double v = ((double)s.height - ((double)y + rng.gen_f64())) / ((double)s.height - 1.0);
    return lens_ray(s.camera, L, s.seed, y * s.width + x, smp, u, v, nullptr);
}

extern "C" {

int oracle_camera_lens(const rt_camera_params* p, double aperture, double focus_dist, rt_camera* out, rt_lens* lens) {
    if (!p || !out || !lens) return -1;
    if (!std::isfinite(aperture) || aperture < 0.0 || !std::isfinite(focus_dist) || !(focus_dist > 0.0)) return -1;
    lens_camera(*p, aperture, focus_dist, out, lens);
    return 0;
}

// origin, direction (3 doubles each) and trials of the lens ray of (pixel, sample) at (u, v)
int oracle_lens_ray(const rt_camera* cam, const rt_lens* lens, uint64_t seed, uint32_t pixel, uint32_t sample, double u, double v,
                    double* out6, uint32_t* trials) {
    const Ray r = lens_ray(*cam, *lens, seed, pixel, sample, u, v, trials);
    const double o[6] = {r.origin.x, r.origin.y, r.origin.z, r.direction.x, r.direction.y, r.direction.z};
    std::memcpy(out6, o, sizeof o);
    return 0;
}

// The primary rays of sample `sample` of every pixel (top row first) through the lens: origin / direction [npix][3].
int oracle_lens_primary(const rt_scene* s, const rt_lens* lens, uint32_t sample, double* origin, double* direction) {
    const uint64_t npix = (uint64_t)s->width * s->height;
#pragma omp parallel for schedule(static)
    for (int64_t k = 0; k < (int64_t)npix; ++k) {
        const uint32_t x = (uint32_t)(k % s->width), y = (uint32_t)(k / s->width);
        SampleRng rng(s->seed, y * s->width + x, sample);
        const Ray r = primary(*s, *lens, x, y, sample, rng);
        origin[3 * k] = r.origin.x; origin[3 * k + 1] = r.origin.y; origin[3 * k + 2] = r.origin.z;
        direction[3 * k] = r.direction.x; direction[3 * k + 1] = r.direction.y; direction[3 * k + 2] = r.direction.z;
    }
    return 0;
}

// render_pixel (rt_oracle.hpp) of every pixel with the lens ray in place of get_ray's: linear and rgb8 [npix][3], *rays.
int oracle_lens_render(const rt_scene* s, const rt_lens* lens, float* out_linear, uint8_t* out_rgb8, uint64_t* rays) {
    const Scene sc(s);
    if (sc.lights.size() >= 10) return -4;
    const uint64_t npix = (uint64_t)s->width * s->height;
    uint64_t total = 0;
#pragma omp parallel for schedule(dynamic, 16) reduction(+ : total)
    for (int64_t k = 0; k < (int64_t)npix; ++k) {
        const uint32_t x = (uint32_t)(k % s->width), y = (uint32_t)(k / s->width);
        Stats st;
        float acc[3] = {0.0f, 0.0f, 0.0f};
        for (uint32_t smp = 0; smp < s->samples_per_pixel; ++smp) {
            SampleRng rng(s->seed, y * s->width + x, smp);
            const Ray r = primary(*s, *lens, x, y, smp, rng);
            const Rgb c = ray_color(sc, r, s->max_depth, s->max_depth, rng, st, nullptr, nullptr);
            acc[0] += c.r; acc[1] += c.g; acc[2] += c.b;
        }
        const float scale = 1.0f / (float)s->samples_per_pixel;
        for (int c = 0; c < 3; ++c) {
            const float mean = scale * acc[c];
            if (out_linear) out_linear[3 * k + c] = mean;
            if (out_rgb8) out_rgb8[3 * k + c] = quantise_u8(std::sqrt(mean));
        }
        total += st.rays;
    }
    if (rays) *rays = total;
    return 0;
}

// The first hit of sample sample0's lens ray and the count of samples in [sample0, sample0 + samples) that hit: sphere
// (0xffffffff on a miss), point [npix][3] (0 on a miss), hits [npix].
int oracle_lens_hits(const rt_scene* s, const rt_lens* lens, uint32_t samples, uint32_t sample0, uint32_t* sphere, double* point,
                     uint32_t* hits) {
    const Scene sc(s);
    const uint64_t npix = (uint64_t)s->width * s->height;
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t k = 0; k < (int64_t)npix; ++k) {
        const uint32_t x = (uint32_t)(k % s->width), y = (uint32_t)(k / s->width);
        Stats st;
        uint32_t nh = 0, sph = 0xffffffffu;
        P3 pt{0.0, 0.0, 0.0};
        for (uint32_t j = 0; j < samples; ++j) {
            SampleRng rng(s->seed, y * s->width + x, sample0 + j);
            const Ray r = primary(*s, *lens, x, y, sample0 + j, rng);
            Hit hit{};
            if (hit_world(sc, r, 0.001, DBL_MAX, &hit, st)) {
                ++nh;
                if (j == 0) { sph = (uint32_t)hit.sphere; pt = hit.point; }
            }
        }
        hits[k] = nh; sphere[k] = sph;
        point[3 * k] = pt.x; point[3 * k + 1] = pt.y; point[3 * k + 2] = pt.z;
    }
    return 0;
}

// The auxiliary buffers of the lens rays (tests/oracle_aov.cpp's, with the lens): per pixel the f32 means in sample order of
// the first-hit albedo (the sky on a miss) and of the normal rounded to f32 (0 on a miss), [npix][3] each.
int oracle_lens_aov(const rt_scene* s, const rt_lens* lens, uint32_t samples, uint32_t sample0, float* albedo, float* normal) {
    const Scene sc(s);
    const uint64_t npix = (uint64_t)s->width * s->height;
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t k = 0; k < (int64_t)npix; ++k) {
        const uint32_t x = (uint32_t)(k % s->width), y = (uint32_t)(k / s->width);
        Stats st;
        float a[3] = {0.0f, 0.0f, 0.0f}, n[3] = {0.0f, 0.0f, 0.0f};
        for (uint32_t j = 0; j < samples; ++j) {
            SampleRng rng(s->seed, y * s->width + x, sample0 + j);
            const Ray r = primary(*s, *lens, x, y, sample0 + j, rng);
            Hit hit{};
            Rgb c;
            float hn[3] = {0.0f, 0.0f, 0.0f};
            if (hit_world(sc, r, 0.001, DBL_MAX, &hit, st)) {
                const rt_sphere& sp = s->spheres[hit.sphere];
                if (sp.kind == RT_LAMBERTIAN || sp.kind == RT_METAL) c = Rgb{sp.albedo[0], sp.albedo[1], sp.albedo[2]};
                else if (sp.kind == RT_TEXTURE) c = texture_get_albedo(s->textures[sp.texture], sp.param, hit.u, hit.v, st);
                else c = Rgb{1.0f, 1.0f, 1.0f};
                hn[0] = (float)hit.normal.x; hn[1] = (float)hit.normal.y; hn[2] = (float)hit.normal.z;
            } else {
                c = sky_color(sc, r);
            }
            a[0] += c.r; a[1] += c.g; a[2] += c.b;
            n[0] += hn[0]; n[1] += hn[1]; n[2] += hn[2];
        }
        const float scale = 1.0f / (float)samples;
        for (int q = 0; q < 3; ++q) { albedo[3 * k + q] = scale * a[q]; normal[3 * k + q] = scale * n[q]; }
    }
    return 0;
}

}  // extern "C"
