// raytracer <config_file> <output_file> — the reference CLI (main.rs:7-20) on top of librtb200.so.
// Same argument contract, same two stdout lines ("\nRendering <file>", "Frame time: <ms>ms"); errors that make the
// reference panic print a message to stderr and exit with status 101 (Rust's panic exit code).
// Extra knobs, so the CLI stays identical: RTB200_SEED, RTB200_DEVICE, RTB200_GPUS=<n|0=all> (row bands dealt over n GPUs of
// this process, rtb200_render_rgb8_multi), RTB200_STATS=1 (prints rays / Mrays/s to stderr).
// RTB200_FRAMES=<frames.json> renders an animation over the scene (rtb200_render_frames): the file is a JSON array of
// {"camera": {<the config's camera schema>}, "seed"?: n, "max_depth"?: n}, omitted fields are the scene's, and <output_file> is a
// prefix: frame i is written to <prefix>_{i:03}.png (the reference's commented-out per-frame name, main.rs:17). Stdout gets
// "\nRendering <file>" per frame and one "Frames time: <ms>ms for <n> frames" line.
// RTB200_ADAPTIVE=<rel_tol>[,<abs_tol>[,<samples_per_round>[,<min_samples>]]] renders adaptively (rtb200_render_adaptive, defaults
// 0, 8, 16) with max_samples = the scene's samples_per_pixel: a pixel stops once its standard error is within
// abs_tol + rel_tol * mean in every channel (DESIGN.md §4.9). Same two stdout lines; RTB200_STATS also prints the samples
// traced out of samples_per_pixel * width * height.
// RTB200_AOV=<samples>[,<sample0>] also writes the auxiliary buffers of those camera samples of the frame (rtb200_scene_aov,
// DESIGN.md §4.14) next to <output_file>: <stem>_albedo.png, the mean first-hit albedo in the beauty image's encoding, and
// <stem>_normal.png, the mean normal n as 0.5 * n + 0.5 (no square root), where <stem> is <output_file> without its extension.
// RTB200_DENOISE=<iterations>[,<color_weight>[,<albedo_weight>[,<normal_weight>]]] also writes <stem>_denoised.png: the frame's
// linear image denoised (rtb200_denoise, DESIGN.md §4.15; omitted weights are the header's RTB200_DENOISE_DEFAULT_*) with the
// albedo and normal of the frame's own samples (samples_per_pixel samples from sample 0) as guides. The frame is rendered once,
// in linear f32, and out.png is its quantisation; the AOV pass uploads the scene once more.
// RTB200_TEMPORAL=<max_history>[,<iterations>[,<color_weight>[,<albedo_weight>[,<normal_weight>[,<clamp_gamma>]]]]], with
// RTB200_FRAMES only,
// also writes <prefix>_{i:03}_denoised.png per frame: the AOV pass of the frame's own samples (samples_per_pixel samples from
// sample 0, the frame's camera and seed), the temporal accumulation of its linear image over the frames before it
// (rtb200_temporal, DESIGN.md §4.16, without sphere motion: the frames move only the camera; depth_tol is the header's default),
// then the denoise with the frame's albedo and normal (iterations 0: the accumulated image alone; omitted values are the
// header's RTB200_DENOISE_DEFAULT_*). The frames are rendered once, in linear f32, and <prefix>_{i:03}.png is each one's
// quantisation, byte for byte the run's without the variable. With <clamp_gamma> the accumulation clamps each history to the
// frame's neighbourhood (rtb200_temporal_clamped, DESIGN.md §4.20, at the header's default radius); without it, the
// accumulation is rtb200_temporal's. Accumulation averages noise only across frames whose seeds
// differ: a frames file that omits "seed" renders every frame with the scene's seed, and the same noise accumulates.
// A camera (of the config or of a frame) may carry "aperture" and "focus_dist": the thin lens of DESIGN.md §4.17 (absent or 0
// aperture: the reference's pinhole camera; absent focus_dist: |look_from - look_at|, or the scene's for a frame). Plain renders
// and RTB200_FRAMES render lens cameras (rtb200_render_frames_lens). RTB200_GPUS, RTB200_ADAPTIVE, RTB200_AOV, RTB200_DENOISE
// and RTB200_TEMPORAL refuse a lens camera with status 101: none of them renders it as a pinhole.
// RTB200_DENOISE_VAR=<iterations>[,<color_weight>[,<albedo_weight>[,<normal_weight>[,<variance_floor>]]]] renders the frame with
// the variance of its pixel means (rtb200_render_frames_var) and writes <stem>_denoised.png: the variance-guided denoise
// (rtb200_denoise_var, DESIGN.md §4.18; omitted values are the header's RTB200_DENOISE_VAR_DEFAULT_*) with the AOVs of the
// frame's own samples. Not with RTB200_DENOISE, RTB200_GPUS, RTB200_FRAMES, RTB200_ADAPTIVE, RTB200_TEMPORAL or a lens camera.
// RTB200_TEMPORAL_VAR=<max_history>[,<iterations>[,<color_weight>[,<albedo_weight>[,<normal_weight>[,<variance_floor>[,<clamp_gamma>]]]]]],
// with RTB200_FRAMES only, is RTB200_TEMPORAL with each pixel's variance carried through the accumulation and the variance-guided
// denoise: the frames are rendered once with the variance of their pixel means (rtb200_render_frames_var), each frame is
// accumulated with its variance (rtb200_temporal_var, DESIGN.md §4.21; clamped at the header's default radius when <clamp_gamma>
// is given) and denoised by it (rtb200_denoise_var with the frame's albedo and normal) into <prefix>_{i:03}_denoised.png
// (iterations 0: the accumulated image alone; omitted values are the header's RTB200_DENOISE_VAR_DEFAULT_*). <prefix>_{i:03}.png
// is byte for byte the run's without the variable. Not with RTB200_TEMPORAL, RTB200_DENOISE, RTB200_DENOISE_VAR, RTB200_GPUS,
// RTB200_ADAPTIVE, RTB200_AOV or a lens camera.
#include <chrono>
#include <cmath>
#include <cstring>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/rtb200.h"
#include "png_writer.hpp"
#include "scene_json.hpp"

// RTB200_FRAMES: every frame of frames_path over `s`, written to <prefix>_000.png, <prefix>_001.png, ...
static int write_temporal(const rt_scene& s, const std::vector<rt_frame>& frames, const rt_options& opts, const float* linear,
                          const std::vector<std::string>& files, uint32_t max_history, const rt_denoise_params& dp,
                          const rt_temporal_clamp* clamp, const float* variance, const rt_denoise_var_params& vp);

// RTB200_TEMPORAL_VAR: the parameters of `spec` (101 and a message when it is malformed or out of range); *has_clamp tells
// whether it gives the clamp
static int parse_temporal_var(const rt_scene& s, const char* spec, uint32_t* max_history, rt_denoise_var_params* p,
                              rt_temporal_clamp* clamp, bool* has_clamp) {
    double v[7] = {0.0, RTB200_DENOISE_VAR_DEFAULT_ITERATIONS, RTB200_DENOISE_VAR_DEFAULT_COLOR_WEIGHT, RTB200_DENOISE_VAR_DEFAULT_ALBEDO_WEIGHT,
                   RTB200_DENOISE_VAR_DEFAULT_NORMAL_WEIGHT, RTB200_DENOISE_VAR_DEFAULT_VARIANCE_FLOOR, 0.0};
    int k = 0;
    for (const char* c = spec; k < 7; ++k) {
        char* end = nullptr;
        v[k] = strtod(c, &end);
        if (end == c || (*end != ',' && *end != 0) || (k == 6 && *end != 0)) {
            fprintf(stderr, "RTB200_TEMPORAL_VAR: expected <max_history>[,<iterations>[,<color_weight>[,<albedo_weight>[,<normal_weight>"
                            "[,<variance_floor>[,<clamp_gamma>]]]]]], got \"%s\"\n", spec);
            return 101;
        }
        if (*end == 0) break;
        c = end + 1;
    }
    *has_clamp = k == 6;
    if (!(v[0] >= 1 && v[0] <= 4294967295.0 && v[0] == std::floor(v[0]))) { fprintf(stderr, "RTB200_TEMPORAL_VAR: max_history must be an integer >= 1\n"); return 101; }
    if (!(v[1] >= 0 && v[1] <= 10 && v[1] == std::floor(v[1]))) { fprintf(stderr, "RTB200_TEMPORAL_VAR: iterations must be an integer in [0, 10]\n"); return 101; }
    for (int i = 2; i < 5; ++i)
        if (!(std::isfinite((float)v[i]) && v[i] >= 0)) { fprintf(stderr, "RTB200_TEMPORAL_VAR: the weights must be finite and >= 0\n"); return 101; }
    if (!(std::isfinite((float)v[5]) && (float)v[5] > 0.0f)) { fprintf(stderr, "RTB200_TEMPORAL_VAR: variance_floor must be finite and > 0\n"); return 101; }
    if (*has_clamp && !(std::isfinite((float)v[6]) && v[6] >= 0)) { fprintf(stderr, "RTB200_TEMPORAL_VAR: clamp_gamma must be finite and >= 0\n"); return 101; }
    if ((uint64_t)s.width * s.height >= (1ull << 31)) { fprintf(stderr, "RTB200_TEMPORAL_VAR: the frame must have fewer than 2^31 pixels\n"); return 101; }
    *max_history = (uint32_t)v[0];
    *p = rt_denoise_var_params{s.width, s.height, (uint32_t)v[1], 0u, (float)v[2], (float)v[3], (float)v[4], (float)v[5]};
    *clamp = rt_temporal_clamp{(float)v[6], RTB200_TEMPORAL_DEFAULT_CLAMP_RADIUS, {0u, 0u}};
    return 0;
}

// RTB200_TEMPORAL: the parameters of `spec` (101 and a message when it is malformed); *has_clamp tells whether it gives the clamp
static int parse_temporal(const rt_scene& s, const char* spec, uint32_t* max_history, rt_denoise_params* p, rt_temporal_clamp* clamp,
                          bool* has_clamp) {
    double v[6] = {0.0, RTB200_DENOISE_DEFAULT_ITERATIONS, RTB200_DENOISE_DEFAULT_COLOR_WEIGHT, RTB200_DENOISE_DEFAULT_ALBEDO_WEIGHT,
                   RTB200_DENOISE_DEFAULT_NORMAL_WEIGHT, 0.0};
    int k = 0;
    for (const char* c = spec; k < 6; ++k) {
        char* end = nullptr;
        v[k] = strtod(c, &end);
        if (end == c || (*end != ',' && *end != 0) || (k == 5 && *end != 0)) {
            fprintf(stderr, "RTB200_TEMPORAL: expected <max_history>[,<iterations>[,<color_weight>[,<albedo_weight>[,<normal_weight>[,<clamp_gamma>]]]]], got \"%s\"\n", spec);
            return 101;
        }
        if (*end == 0) break;
        c = end + 1;
    }
    *has_clamp = k == 5;
    if (*has_clamp && !(std::isfinite((float)v[5]) && v[5] >= 0)) { fprintf(stderr, "RTB200_TEMPORAL: clamp_gamma must be finite and >= 0\n"); return 101; }
    *clamp = rt_temporal_clamp{(float)v[5], RTB200_TEMPORAL_DEFAULT_CLAMP_RADIUS, {0u, 0u}};
    if (!(v[0] >= 1 && v[0] <= 4294967295.0 && v[0] == std::floor(v[0]))) { fprintf(stderr, "RTB200_TEMPORAL: max_history must be an integer >= 1\n"); return 101; }
    if (!(v[1] >= 0 && v[1] <= 10 && v[1] == std::floor(v[1]))) { fprintf(stderr, "RTB200_TEMPORAL: iterations must be an integer in [0, 10]\n"); return 101; }
    if ((uint64_t)s.width * s.height >= (1ull << 31)) { fprintf(stderr, "RTB200_TEMPORAL: the frame must have fewer than 2^31 pixels\n"); return 101; }
    *max_history = (uint32_t)v[0];
    *p = rt_denoise_params{s.width, s.height, (uint32_t)v[1], 0u, (float)v[2], (float)v[3], (float)v[4], 0.0f};
    return 0;
}

// The camera and lens of `spec` (rtb200_camera_from_params_lens) in place of Camera::new's `cam`; no lens: both unchanged.
static int apply_lens(const rthost::LensSpec& spec, rt_camera* cam, rt_lens* lens) {
    *lens = rt_lens{};
    if (spec.aperture == 0.0) return 0;
    if (rtb200_camera_from_params_lens(&spec.params, spec.aperture, spec.focus_dist, cam, lens) != 0) {
        fprintf(stderr, "invalid lens camera: %s\n", rtb200_last_error());
        return 101;
    }
    return 0;
}

static int render_animation(const rthost::SceneHolder& holder, const char* frames_path, const std::string& prefix, const char* temporal,
                            const char* temporal_var) {
    const rt_scene& s = holder.scene;
    if (getenv("RTB200_GPUS")) { fprintf(stderr, "RTB200_FRAMES with RTB200_GPUS is not supported: animations render on one GPU\n"); return 101; }
    std::ifstream f(frames_path, std::ios::binary);
    if (!f) { fprintf(stderr, "Unable to read frames file.: %s\n", frames_path); return 101; }
    std::stringstream ss; ss << f.rdbuf();
    std::vector<rt_frame> frames;
    std::vector<rthost::LensSpec> specs;
    try { frames = rthost::load_frames_json(ss.str(), holder, &specs); }
    catch (const std::exception& e) { fprintf(stderr, "Unable to parse frames json: %s\n", e.what()); return 101; }
    std::vector<rt_lens> lenses(frames.size());
    bool lensed = false;
    for (size_t i = 0; i < frames.size(); ++i) {
        if (apply_lens(specs[i], &frames[i].camera, &lenses[i]) != 0) return 101;
        lensed = lensed || lenses[i].radius != 0.0;
    }
    if (lensed && temporal) { fprintf(stderr, "RTB200_TEMPORAL with a lens camera (aperture > 0) is not supported\n"); return 101; }
    if (lensed && temporal_var) { fprintf(stderr, "RTB200_TEMPORAL_VAR with a lens camera (aperture > 0) is not supported\n"); return 101; }
    std::vector<std::string> files(frames.size());
    for (size_t i = 0; i < frames.size(); ++i) {
        char num[32];
        snprintf(num, sizeof num, "%03zu", i);   // Rust's {:0>3}: at least three digits
        files[i] = prefix + "_" + num + ".png";
        printf("\nRendering %s\n", files[i].c_str());
    }
    fflush(stdout);
    uint32_t max_history = 0;
    rt_denoise_params dp{};
    rt_temporal_clamp clamp{};
    bool has_clamp = false;
    if (temporal && parse_temporal(s, temporal, &max_history, &dp, &clamp, &has_clamp) != 0) return 101;
    rt_denoise_var_params vp{};
    if (temporal_var && parse_temporal_var(s, temporal_var, &max_history, &vp, &clamp, &has_clamp) != 0) return 101;
    const size_t frame_bytes = (size_t)s.width * s.height * 3;
    std::vector<uint8_t> pixels(frame_bytes * frames.size());
    std::vector<float> linear(temporal || temporal_var ? frame_bytes * frames.size() : 0), variance(temporal_var ? frame_bytes * frames.size() : 0);
    rt_options opts{};
    opts.device = getenv("RTB200_DEVICE") ? atoi(getenv("RTB200_DEVICE")) : -1; opts.rank = 0; opts.world = 1; opts.band_rows = 1;
    rt_stats st{};
    auto t0 = std::chrono::steady_clock::now();
    // the accumulation needs the linear frames: one render gives them, and each PNG is its frame's quantisation by the render's
    // own routine (rtb200_probe_quantise), byte for byte the RGB8 render's; RTB200_TEMPORAL_VAR's render adds the variance
    int rc = temporal     ? rtb200_render_frames(&s, &opts, frames.data(), (uint32_t)frames.size(), nullptr, linear.data(), &st)
           : temporal_var ? rtb200_render_frames_var(&s, &opts, frames.data(), nullptr, (uint32_t)frames.size(), nullptr, linear.data(),
                                                     variance.data(), &st)
           : lensed       ? rtb200_render_frames_lens(&s, &opts, frames.data(), lenses.data(), (uint32_t)frames.size(), pixels.data(), nullptr, &st)
                          : rtb200_render_frames(&s, &opts, frames.data(), (uint32_t)frames.size(), pixels.data(), nullptr, &st);
    for (size_t i = 0; rc == 0 && (temporal || temporal_var) && i < frames.size(); ++i)
        rc = rtb200_probe_quantise(linear.data() + i * frame_bytes, (uint32_t)frame_bytes, pixels.data() + i * frame_bytes);
    if (rc != 0) { fprintf(stderr, "render failed (%d): %s\n", rc, rtb200_last_error()); return 101; }
    long long ms = std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now() - t0).count();
    printf("Frames time: %lldms for %zu frames\n", ms, frames.size());
    if (getenv("RTB200_STATS"))
        fprintf(stderr, "rays=%llu samples=%llu device_ms=%.3f Mrays/s=%.1f launches=%u\n", (unsigned long long)st.rays, (unsigned long long)st.samples, st.device_ms,
                st.device_ms > 0 ? st.rays / st.device_ms / 1e3 : 0.0, st.kernel_launches);
    for (size_t i = 0; i < frames.size(); ++i) {
        std::string err;
        if (!rthost::write_png_rgb8(files[i].c_str(), pixels.data() + i * frame_bytes, s.width, s.height, &err)) { fprintf(stderr, "error writing image: %s\n", err.c_str()); return 101; }
    }
    if (!temporal && !temporal_var) return 0;
    return write_temporal(s, frames, opts, linear.data(), files, max_history, dp, has_clamp ? &clamp : nullptr,
                          temporal_var ? variance.data() : nullptr, vp);
}

// RTB200_TEMPORAL: frame i's AOVs, its accumulation over frames 0 .. i (the history ping-pongs between two buffers; clamped
// when clamp is given) and its denoise, written to <prefix>_{i:03}_denoised.png. RTB200_TEMPORAL_VAR (variance given: the
// frames' variances): the same with the variance accumulated beside the colour and the variance-guided denoise of vp.
static int write_temporal(const rt_scene& s, const std::vector<rt_frame>& frames, const rt_options& opts, const float* linear,
                          const std::vector<std::string>& files, uint32_t max_history, const rt_denoise_params& dp,
                          const rt_temporal_clamp* clamp, const float* variance, const rt_denoise_var_params& vp) {
    const size_t npix = (size_t)s.width * s.height;
    std::vector<float> acc_var[2] = {std::vector<float>(variance ? npix * 3 : 0), std::vector<float>(variance ? npix * 3 : 0)};
    std::vector<float> albedo(npix * 3), normal(npix * 3), color[2] = {std::vector<float>(npix * 3), std::vector<float>(npix * 3)};
    std::vector<uint32_t> sphere[2] = {std::vector<uint32_t>(npix), std::vector<uint32_t>(npix)}, length[2] = {std::vector<uint32_t>(npix), std::vector<uint32_t>(npix)};
    std::vector<double> point[2] = {std::vector<double>(npix * 3), std::vector<double>(npix * 3)};
    std::vector<uint8_t> rgb8(npix * 3);
    rtb200_scene_handle h = nullptr;
    int rc = rtb200_scene_upload(&s, &opts, &h);
    for (size_t i = 0, k = 0; rc == 0 && i < frames.size(); ++i, k ^= 1) {
        const rt_aov_params ap{s.samples_per_pixel, 0u, {0u, 0u}};
        const rt_aov_out ao{albedo.data(), normal.data(), nullptr, sphere[k].data(), point[k].data()};
        if ((rc = rtb200_scene_aov(h, &ap, &frames[i], &ao, nullptr)) != 0) break;
        rt_temporal_params tp{};
        tp.width = s.width; tp.height = s.height; tp.max_history = max_history; tp.n_motion = 0;
        tp.camera = frames[i].camera;
        if (i > 0) tp.prev_camera = frames[i - 1].camera;
        tp.depth_tol = RTB200_TEMPORAL_DEFAULT_DEPTH_TOL;
        const rt_temporal_frame cur{linear + i * npix * 3, sphere[k].data(), point[k].data()};
        const rt_temporal_history prev{color[k ^ 1].data(), length[k ^ 1].data(), sphere[k ^ 1].data(), point[k ^ 1].data()};
        const rt_temporal_out out{color[k].data(), length[k].data()};
        if (variance)
            rc = rtb200_temporal_var(opts.device, &tp, clamp, &cur, variance + i * npix * 3, i > 0 ? &prev : nullptr,
                                     i > 0 ? acc_var[k ^ 1].data() : nullptr, nullptr, &out, acc_var[k].data(), nullptr);
        else
            rc = clamp ? rtb200_temporal_clamped(opts.device, &tp, clamp, &cur, i > 0 ? &prev : nullptr, nullptr, &out, nullptr)
                       : rtb200_temporal(opts.device, &tp, &cur, i > 0 ? &prev : nullptr, nullptr, &out, nullptr);
        if (rc != 0) break;
        const uint32_t iterations = variance ? vp.iterations : dp.iterations;
        rc = !iterations ? rtb200_probe_quantise(color[k].data(), (uint32_t)(npix * 3), rgb8.data())
           : variance    ? rtb200_denoise_var(opts.device, &vp, color[k].data(), acc_var[k].data(), albedo.data(), normal.data(), nullptr,
                                              rgb8.data(), nullptr, nullptr)
                         : rtb200_denoise(opts.device, &dp, color[k].data(), albedo.data(), normal.data(), nullptr, rgb8.data(), nullptr);
        if (rc != 0) break;
        const std::string path = files[i].substr(0, files[i].size() - 4) + "_denoised.png";
        std::string err;
        if (!rthost::write_png_rgb8(path.c_str(), rgb8.data(), s.width, s.height, &err)) {
            fprintf(stderr, "error writing image: %s\n", err.c_str());
            if (h) rtb200_scene_release(h);
            return 101;
        }
    }
    if (h) rtb200_scene_release(h);
    if (rc != 0) { fprintf(stderr, "temporal accumulation failed (%d): %s\n", rc, rtb200_last_error()); return 101; }
    return 0;
}

// RTB200_ADAPTIVE: the scene rendered adaptively into `pixels`
static int render_adaptive(const rt_scene& s, const char* spec, const rt_options& opts, uint8_t* pixels, rt_stats* st) {
    rt_adaptive_params p{8u, 0u, 16u, 0u, 0.0f, 0.0f};
    double v[4] = {0.0, 0.0, 8.0, 16.0};
    int k = 0;
    for (const char* c = spec; k < 4; ++k) {
        char* end = nullptr;
        v[k] = strtod(c, &end);
        if (end == c || (*end != ',' && *end != 0)) { fprintf(stderr, "RTB200_ADAPTIVE: expected <rel_tol>[,<abs_tol>[,<samples_per_round>[,<min_samples>]]], got \"%s\"\n", spec); return 101; }
        if (*end == 0) { ++k; break; }
        c = end + 1;
    }
    if (v[2] < 1 || v[3] < 1 || v[2] > 4294967295.0 || v[3] > 4294967295.0) { fprintf(stderr, "RTB200_ADAPTIVE: samples_per_round and min_samples must be positive integers\n"); return 101; }
    p.rel_tol = (float)v[0]; p.abs_tol = (float)v[1]; p.samples_per_round = (uint32_t)v[2]; p.min_samples = (uint32_t)v[3];
    if (rtb200_render_adaptive(&s, &opts, &p, pixels, nullptr, nullptr, st) != 0) return -1;
    return 0;
}

// palette's f32 -> u8 (raytracer.rs:207-213 after its square root): min(x * 255, 255) plus 2^23, whose low mantissa bits
// are the value rounded half to even; 0 below 0 and 255 for NaN, like the kernel's quantise_u8
static uint8_t to_u8(float x) {
    const float scaled = std::fmin(x * 255.0f, 255.0f);
    const float f = scaled + 8388608.0f;
    uint32_t bits;
    memcpy(&bits, &f, 4);
    return bits >= 0x4B000000u ? (uint8_t)(bits - 0x4B000000u) : (uint8_t)0;
}

// <output_file> without its extension
static std::string stem_of(const std::string& out) {
    const size_t slash = out.find_last_of('/'), dot = out.find_last_of('.');
    return dot != std::string::npos && (slash == std::string::npos || dot > slash) ? out.substr(0, dot) : out;
}

// the mean albedo and normal of samples [sample0, sample0 + samples) of every pixel of `s` (rtb200_scene_aov)
static int aov_of(const rt_scene& s, const rt_options& opts, uint32_t samples, uint32_t sample0, float* albedo, float* normal) {
    rt_aov_params p{samples, sample0, {0u, 0u}};
    rt_aov_out o{albedo, normal, nullptr, nullptr, nullptr};
    rtb200_scene_handle h = nullptr;
    int rc = rtb200_scene_upload(&s, &opts, &h);
    if (rc == 0) rc = rtb200_scene_aov(h, &p, nullptr, &o, nullptr);
    if (h) rtb200_scene_release(h);
    if (rc != 0) fprintf(stderr, "aov failed (%d): %s\n", rc, rtb200_last_error());
    return rc;
}

// RTB200_AOV: the albedo and normal buffers of samples [sample0, sample0 + samples) of every pixel of `s`, written beside `out`
static int write_aov(const rt_scene& s, const char* spec, const rt_options& opts, const std::string& out) {
    char* end = nullptr;
    const unsigned long long samples = strtoull(spec, &end, 10);
    unsigned long long sample0 = 0;
    bool ok = end != spec && (*end == 0 || *end == ',');
    if (ok && *end == ',') { const char* c = end + 1; sample0 = strtoull(c, &end, 10); ok = end != c && *end == 0; }
    if (!ok || samples < 1 || samples > 4294967295ull || sample0 > 4294967295ull) {
        fprintf(stderr, "RTB200_AOV: expected <samples>[,<sample0>] with samples >= 1, got \"%s\"\n", spec);
        return 101;
    }
    const size_t npix = (size_t)s.width * s.height;
    std::vector<float> albedo(npix * 3), normal(npix * 3);
    if (aov_of(s, opts, (uint32_t)samples, (uint32_t)sample0, albedo.data(), normal.data()) != 0) return 101;
    std::vector<uint8_t> a8(npix * 3), n8(npix * 3);
    for (size_t i = 0; i < npix * 3; ++i) {
        a8[i] = to_u8(std::sqrt(albedo[i]));
        n8[i] = to_u8(0.5f * normal[i] + 0.5f);
    }
    const std::string stem = stem_of(out);
    std::string err;
    for (const auto& img : {std::make_pair(stem + "_albedo.png", &a8), std::make_pair(stem + "_normal.png", &n8)})
        if (!rthost::write_png_rgb8(img.first.c_str(), img.second->data(), s.width, s.height, &err)) { fprintf(stderr, "error writing image: %s\n", err.c_str()); return 101; }
    return 0;
}

// RTB200_DENOISE: the parameters of `spec` for the frame of `s` (101 and a message when it is malformed)
static int parse_denoise(const rt_scene& s, const char* spec, rt_denoise_params* p) {
    double v[4] = {RTB200_DENOISE_DEFAULT_ITERATIONS, RTB200_DENOISE_DEFAULT_COLOR_WEIGHT, RTB200_DENOISE_DEFAULT_ALBEDO_WEIGHT,
                   RTB200_DENOISE_DEFAULT_NORMAL_WEIGHT};
    int k = 0;
    for (const char* c = spec; k < 4; ++k) {
        char* end = nullptr;
        v[k] = strtod(c, &end);
        if (end == c || (*end != ',' && *end != 0)) {
            fprintf(stderr, "RTB200_DENOISE: expected <iterations>[,<color_weight>[,<albedo_weight>[,<normal_weight>]]], got \"%s\"\n", spec);
            return 101;
        }
        if (*end == 0) break;
        c = end + 1;
    }
    if (!(v[0] >= 1 && v[0] <= 10 && v[0] == std::floor(v[0]))) { fprintf(stderr, "RTB200_DENOISE: iterations must be an integer in [1, 10]\n"); return 101; }
    if ((uint64_t)s.width * s.height >= (1ull << 31)) { fprintf(stderr, "RTB200_DENOISE: the frame must have fewer than 2^31 pixels\n"); return 101; }
    *p = rt_denoise_params{s.width, s.height, (uint32_t)v[0], 0u, (float)v[1], (float)v[2], (float)v[3], 0.0f};
    return 0;
}

// RTB200_DENOISE: `linear`, the frame of `s`, denoised with the AOVs of its own samples, written to <stem>_denoised.png
static int write_denoised(const rt_scene& s, const rt_denoise_params& p, const rt_options& opts, const float* linear, const std::string& out) {
    const size_t npix = (size_t)s.width * s.height;
    std::vector<float> albedo(npix * 3), normal(npix * 3);
    std::vector<uint8_t> rgb8(npix * 3);
    if (aov_of(s, opts, s.samples_per_pixel, 0u, albedo.data(), normal.data()) != 0) return 101;
    if (rtb200_denoise(opts.device, &p, linear, albedo.data(), normal.data(), nullptr, rgb8.data(), nullptr) != 0) {
        fprintf(stderr, "denoise failed: %s\n", rtb200_last_error());
        return 101;
    }
    std::string err;
    if (!rthost::write_png_rgb8((stem_of(out) + "_denoised.png").c_str(), rgb8.data(), s.width, s.height, &err)) { fprintf(stderr, "error writing image: %s\n", err.c_str()); return 101; }
    return 0;
}

// RTB200_DENOISE_VAR: the parameters of `spec` for the frame of `s` (101 and a message when it is malformed); omitted values
// are the header's RTB200_DENOISE_VAR_DEFAULT_*
static int parse_denoise_var(const rt_scene& s, const char* spec, rt_denoise_var_params* p) {
    double v[5] = {RTB200_DENOISE_VAR_DEFAULT_ITERATIONS, RTB200_DENOISE_VAR_DEFAULT_COLOR_WEIGHT, RTB200_DENOISE_VAR_DEFAULT_ALBEDO_WEIGHT,
                   RTB200_DENOISE_VAR_DEFAULT_NORMAL_WEIGHT, RTB200_DENOISE_VAR_DEFAULT_VARIANCE_FLOOR};
    int k = 0;
    for (const char* c = spec; k < 5; ++k) {
        char* end = nullptr;
        v[k] = strtod(c, &end);
        if (end == c || (*end != ',' && *end != 0) || (k == 4 && *end != 0)) {
            fprintf(stderr, "RTB200_DENOISE_VAR: expected <iterations>[,<color_weight>[,<albedo_weight>[,<normal_weight>[,<variance_floor>]]]], got \"%s\"\n", spec);
            return 101;
        }
        if (*end == 0) break;
        c = end + 1;
    }
    if (!(v[0] >= 1 && v[0] <= 10 && v[0] == std::floor(v[0]))) { fprintf(stderr, "RTB200_DENOISE_VAR: iterations must be an integer in [1, 10]\n"); return 101; }
    for (int i = 1; i < 4; ++i)
        if (!(std::isfinite((float)v[i]) && v[i] >= 0)) { fprintf(stderr, "RTB200_DENOISE_VAR: the weights must be finite and >= 0\n"); return 101; }
    if (!(std::isfinite((float)v[4]) && (float)v[4] > 0.0f)) { fprintf(stderr, "RTB200_DENOISE_VAR: variance_floor must be finite and > 0\n"); return 101; }
    if ((uint64_t)s.width * s.height >= (1ull << 31)) { fprintf(stderr, "RTB200_DENOISE_VAR: the frame must have fewer than 2^31 pixels\n"); return 101; }
    *p = rt_denoise_var_params{s.width, s.height, (uint32_t)v[0], 0u, (float)v[1], (float)v[2], (float)v[3], (float)v[4]};
    return 0;
}

// RTB200_DENOISE_VAR: `linear` and `variance`, the frame of `s` and the variance of its pixel means, denoised with the AOVs of
// its own samples, written to <stem>_denoised.png
static int write_denoised_var(const rt_scene& s, const rt_denoise_var_params& p, const rt_options& opts, const float* linear,
                              const float* variance, const std::string& out) {
    const size_t npix = (size_t)s.width * s.height;
    std::vector<float> albedo(npix * 3), normal(npix * 3);
    std::vector<uint8_t> rgb8(npix * 3);
    if (aov_of(s, opts, s.samples_per_pixel, 0u, albedo.data(), normal.data()) != 0) return 101;
    if (rtb200_denoise_var(opts.device, &p, linear, variance, albedo.data(), normal.data(), nullptr, rgb8.data(), nullptr, nullptr) != 0) {
        fprintf(stderr, "denoise failed: %s\n", rtb200_last_error());
        return 101;
    }
    std::string err;
    if (!rthost::write_png_rgb8((stem_of(out) + "_denoised.png").c_str(), rgb8.data(), s.width, s.height, &err)) { fprintf(stderr, "error writing image: %s\n", err.c_str()); return 101; }
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 3) {                                                       // main.rs:9-12
        printf("Usage: %s <config_file> <output_file>\n", argc > 0 ? argv[0] : "raytracer");
        return 0;
    }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) { fprintf(stderr, "Unable to read config file.: %s\n", argv[1]); return 101; }              // main.rs:14
    std::stringstream ss; ss << f.rdbuf();
    rthost::SceneHolder holder;
    try {
        std::string path = argv[1];
        size_t slash = path.find_last_of('/');
        rthost::load_scene_json(ss.str(), slash == std::string::npos ? std::string(".") : path.substr(0, slash), &holder);
    } catch (const std::exception& e) { fprintf(stderr, "Unable to parse config json: %s\n", e.what()); return 101; }   // main.rs:15
    if (const char* sd = getenv("RTB200_SEED")) holder.scene.seed = strtoull(sd, nullptr, 0);
    const char* temporal = getenv("RTB200_TEMPORAL");
    const char* temporal_var = getenv("RTB200_TEMPORAL_VAR");
    if (temporal_var && (!getenv("RTB200_FRAMES") || temporal || getenv("RTB200_DENOISE") || getenv("RTB200_DENOISE_VAR") || getenv("RTB200_GPUS") ||
                         getenv("RTB200_ADAPTIVE") || getenv("RTB200_AOV"))) {
        fprintf(stderr, "RTB200_TEMPORAL_VAR needs RTB200_FRAMES, without RTB200_TEMPORAL, RTB200_DENOISE, RTB200_DENOISE_VAR, RTB200_GPUS, "
                        "RTB200_ADAPTIVE or RTB200_AOV: it accumulates the frames of one animation and their variance on one GPU and "
                        "denoises them itself\n");
        return 101;
    }
    if (temporal && (!getenv("RTB200_FRAMES") || getenv("RTB200_GPUS") || getenv("RTB200_ADAPTIVE") || getenv("RTB200_AOV") || getenv("RTB200_DENOISE"))) {
        fprintf(stderr, "RTB200_TEMPORAL needs RTB200_FRAMES, without RTB200_GPUS, RTB200_ADAPTIVE, RTB200_AOV or RTB200_DENOISE: it accumulates "
                        "the frames of one animation on one GPU and denoises them itself\n");
        return 101;
    }
    const char* adaptive = getenv("RTB200_ADAPTIVE");
    if (adaptive && (getenv("RTB200_GPUS") || getenv("RTB200_FRAMES"))) {
        fprintf(stderr, "RTB200_ADAPTIVE with RTB200_GPUS or RTB200_FRAMES is not supported: adaptive renders are one frame on one GPU\n");
        return 101;
    }
    const char* aov = getenv("RTB200_AOV");
    if (aov && (getenv("RTB200_GPUS") || getenv("RTB200_FRAMES") || adaptive)) {
        fprintf(stderr, "RTB200_AOV with RTB200_GPUS, RTB200_FRAMES or RTB200_ADAPTIVE is not supported: the buffers are of one frame's camera samples on one GPU\n");
        return 101;
    }
    const char* denoise = getenv("RTB200_DENOISE");
    if (denoise && (getenv("RTB200_GPUS") || getenv("RTB200_FRAMES") || adaptive)) {
        fprintf(stderr, "RTB200_DENOISE with RTB200_GPUS, RTB200_FRAMES or RTB200_ADAPTIVE is not supported: it denoises one frame on one GPU\n");
        return 101;
    }
    const char* denoise_var = getenv("RTB200_DENOISE_VAR");
    if (denoise_var && (denoise || getenv("RTB200_GPUS") || getenv("RTB200_FRAMES") || adaptive || temporal)) {
        fprintf(stderr, "RTB200_DENOISE_VAR with RTB200_DENOISE, RTB200_GPUS, RTB200_FRAMES, RTB200_ADAPTIVE or RTB200_TEMPORAL is not "
                        "supported: it denoises one frame on one GPU with its own variance\n");
        return 101;
    }
    rt_lens scene_lens{};
    if (apply_lens(holder.lens_spec, &holder.scene.camera, &scene_lens) != 0) return 101;
    const bool lens = scene_lens.radius != 0.0;
    if (lens && (getenv("RTB200_GPUS") || adaptive || aov || denoise || denoise_var || temporal || temporal_var)) {
        fprintf(stderr, "a lens camera (aperture > 0) with RTB200_GPUS, RTB200_ADAPTIVE, RTB200_AOV, RTB200_DENOISE, RTB200_DENOISE_VAR, RTB200_TEMPORAL "
                        "or RTB200_TEMPORAL_VAR is not supported: render it without them\n");
        return 101;
    }
    rt_denoise_params denoise_p{};
    if (denoise && parse_denoise(holder.scene, denoise, &denoise_p) != 0) return 101;
    rt_denoise_var_params denoise_var_p{};
    if (denoise_var && parse_denoise_var(holder.scene, denoise_var, &denoise_var_p) != 0) return 101;
    if (const char* fp = getenv("RTB200_FRAMES")) return render_animation(holder, fp, argv[2], temporal, temporal_var);
    printf("\nRendering %s\n", argv[2]);                                  // main.rs:18
    fflush(stdout);
    const rt_scene& s = holder.scene;
    std::vector<uint8_t> pixels((size_t)s.width * s.height * 3);          // raytracer.rs:254
    rt_options opts{};
    opts.device = getenv("RTB200_DEVICE") ? atoi(getenv("RTB200_DEVICE")) : -1; opts.rank = 0; opts.world = 1; opts.band_rows = 1;
    rt_stats st{};
    auto t0 = std::chrono::steady_clock::now();                           // raytracer.rs:259
    const char* gpus = getenv("RTB200_GPUS");
    std::vector<float> linear, variance;
    int rc = 0;
    if (adaptive) {
        rc = render_adaptive(s, adaptive, opts, pixels.data(), &st);
        if (rc == 101) return rc;
    } else if (denoise) {
        // the denoise needs the linear image: one render gives it, and out.png is its quantisation by the render's own routine
        // (rtb200_probe_quantise), byte for byte the RGB8 render's
        linear.resize(pixels.size());
        rc = rtb200_render_linear_f32(&s, &opts, linear.data(), &st);
        if (rc == 0) rc = rtb200_probe_quantise(linear.data(), (uint32_t)linear.size(), pixels.data());
    } else if (denoise_var) {
        // the frame with the variance of its pixel means; out.png is the linear image's quantisation, as for RTB200_DENOISE
        linear.resize(pixels.size());
        variance.resize(pixels.size());
        const rt_frame f{s.camera, s.seed, s.max_depth, 0};
        rc = rtb200_render_frames_var(&s, &opts, &f, nullptr, 1, nullptr, linear.data(), variance.data(), &st);
        if (rc == 0) rc = rtb200_probe_quantise(linear.data(), (uint32_t)linear.size(), pixels.data());
    } else if (lens) {
        const rt_frame f{s.camera, s.seed, s.max_depth, 0};   // one frame of the lens camera
        rc = rtb200_render_frames_lens(&s, &opts, &f, &scene_lens, 1, pixels.data(), nullptr, &st);
    } else {
        rc = gpus ? rtb200_render_rgb8_multi(&s, &opts, atoi(gpus), pixels.data(), &st)   // replaces raytracer.rs:260-262
                  : rtb200_render_rgb8(&s, &opts, pixels.data(), &st);
    }
    if (rc != 0) { fprintf(stderr, "render failed (%d): %s\n", rc, rtb200_last_error()); return 101; }
    long long ms = std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now() - t0).count();
    printf("Frame time: %lldms\n", ms);                                   // raytracer.rs:263
    if (getenv("RTB200_STATS"))
        fprintf(stderr, "rays=%llu samples=%llu device_ms=%.3f Mrays/s=%.1f gpus=%d\n", (unsigned long long)st.rays, (unsigned long long)st.samples, st.device_ms,
                st.device_ms > 0 ? st.rays / st.device_ms / 1e3 : 0.0, (int)st.gpus_used);
    if (adaptive && getenv("RTB200_STATS")) {
        const unsigned long long all = (unsigned long long)s.samples_per_pixel * s.width * s.height;
        fprintf(stderr, "adaptive: %llu of %llu samples traced (%.1f %%)\n", (unsigned long long)st.samples, all, all ? 100.0 * st.samples / all : 0.0);
    }
    std::string err;
    if (!rthost::write_png_rgb8(argv[2], pixels.data(), s.width, s.height, &err)) { fprintf(stderr, "error writing image: %s\n", err.c_str()); return 101; }   // raytracer.rs:265
    if (aov && (rc = write_aov(s, aov, opts, argv[2])) != 0) return rc;
    if (denoise) return write_denoised(s, denoise_p, opts, linear.data(), argv[2]);
    if (denoise_var) return write_denoised_var(s, denoise_var_p, opts, linear.data(), variance.data(), argv[2]);
    return 0;
}
