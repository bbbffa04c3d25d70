// rtb200_api_denoise.cu — denoising a frame with its auxiliary buffers through the C ABI (DESIGN.md §4.15), in both forms:
// device buffers on the caller's stream with the caller's scratch, or host buffers staged through the context's query block
// (HostStage). The kernels are in rtb200_denoise.cu; those of the variance-guided denoise (DESIGN.md §4.18), whose calls
// follow the same pattern, in rtb200_denoise_var.cu.

#include "rtb200_host.cuh"

using namespace rtk;

namespace {

// The argument checks of both forms (no device is touched); `scratch` is checked in the device form only.
int check_denoise(const rt_denoise_params* p, const float* color, const float* albedo, const float* normal, const void* scratch,
                  bool device_form, const float* out_linear, const uint8_t* out_rgb8) {
    if (!p) return fail(RT_ERR_INVALID, "params is null");
    if (!color) return fail(RT_ERR_INVALID, "color is null");
    if (!out_linear && !out_rgb8) return fail(RT_ERR_INVALID, "out_linear and out_rgb8 are both null");
    if (device_form && !scratch) return fail(RT_ERR_INVALID, "scratch is null");
    uint32_t bits2;
    memcpy(&bits2, &p->reserved2, 4);
    if (p->reserved != 0 || bits2 != 0) return fail(RT_ERR_INVALID, "rt_denoise_params.reserved and reserved2 must be 0");
    if (p->iterations < 1 || p->iterations > 10) return fail(RT_ERR_INVALID, "rt_denoise_params.iterations must be in [1, 10]");
    const std::pair<float, const char*> weights[3] = {{p->color_weight, "color_weight"}, {p->albedo_weight, "albedo_weight"},
                                                      {p->normal_weight, "normal_weight"}};
    for (const auto& w : weights)
        if (!(std::isfinite(w.first) && w.first >= 0.0f)) return fail(RT_ERR_INVALID, std::string("rt_denoise_params.") + w.second + " must be finite and >= 0");
    if (!std::isfinite(p->color_weight * (float)(1u << (2 * (p->iterations - 1)))))
        return fail(RT_ERR_INVALID, "rt_denoise_params.color_weight * 4^(iterations - 1) overflows f32");
    if (!albedo && p->albedo_weight != 0.0f) return fail(RT_ERR_INVALID, "albedo_weight is nonzero but albedo is null");
    if (!normal && p->normal_weight != 0.0f) return fail(RT_ERR_INVALID, "normal_weight is nonzero but normal is null");
    const uint64_t n = (uint64_t)p->width * p->height;
    if (n >= (1ull << 31)) return fail(RT_ERR_INVALID, "width * height must be below 2^31");
    const Range in[3] = {{color, n * 12, "color", 4}, {albedo, n * 12, "albedo", 4}, {normal, n * 12, "normal", 4}};
    const Range out[3] = {{out_linear, n * 12, "out_linear", 4}, {out_rgb8, n * 3, "out_rgb8", 1},
                          {scratch, device_form ? denoise_scratch_bytes(n) : 0, "scratch", 16}};
    if (device_form) {
        for (const Range* g : {in, out})
            for (int k = 0; k < 3; ++k)
                if ((uintptr_t)g[k].p % g[k].align) return fail(RT_ERR_INVALID, std::string(g[k].name) + " is not " + std::to_string(g[k].align) + "-byte aligned");
    }
    // an output or the scratch must not overlap an input or each other
    for (int i = 0; i < 3; ++i) {
        for (const Range& r : in)
            if (overlap(out[i], r)) return fail(RT_ERR_INVALID, std::string(out[i].name) + " overlaps " + r.name);
        for (int j = 0; j < i; ++j)
            if (overlap(out[i], out[j])) return fail(RT_ERR_INVALID, std::string(out[i].name) + " overlaps " + out[j].name);
    }
    return RT_OK;
}

DenoiseArgs denoise_args(const rt_denoise_params& p, const float* color, const float* albedo, const float* normal, void* scratch,
                         float* out_linear, uint8_t* out_rgb8) {
    return DenoiseArgs{p.width, p.height, p.iterations, p.color_weight, p.albedo_weight, p.normal_weight, color, albedo, normal,
                       scratch, out_linear, out_rgb8};
}

// The argument checks of both forms of the variance-guided denoise (no device is touched); `scratch` in the device form only.
int check_denoise_var(const rt_denoise_var_params* p, const float* color, const float* variance, const float* albedo,
                      const float* normal, const void* scratch, bool device_form, const float* out_linear, const uint8_t* out_rgb8,
                      const float* out_variance) {
    if (!p) return fail(RT_ERR_INVALID, "params is null");
    if (!color) return fail(RT_ERR_INVALID, "color is null");
    if (!variance) return fail(RT_ERR_INVALID, "variance is null");
    if (!out_linear && !out_rgb8 && !out_variance) return fail(RT_ERR_INVALID, "out_linear, out_rgb8 and out_variance are all null");
    if (device_form && !scratch) return fail(RT_ERR_INVALID, "scratch is null");
    if (p->reserved != 0) return fail(RT_ERR_INVALID, "rt_denoise_var_params.reserved must be 0");
    if (p->iterations < 1 || p->iterations > 10) return fail(RT_ERR_INVALID, "rt_denoise_var_params.iterations must be in [1, 10]");
    const std::pair<float, const char*> weights[3] = {{p->color_weight, "color_weight"}, {p->albedo_weight, "albedo_weight"},
                                                      {p->normal_weight, "normal_weight"}};
    for (const auto& w : weights)
        if (!(std::isfinite(w.first) && w.first >= 0.0f)) return fail(RT_ERR_INVALID, std::string("rt_denoise_var_params.") + w.second + " must be finite and >= 0");
    if (!(std::isfinite(p->variance_floor) && p->variance_floor > 0.0f))
        return fail(RT_ERR_INVALID, "rt_denoise_var_params.variance_floor must be finite and > 0");
    if (!albedo && p->albedo_weight != 0.0f) return fail(RT_ERR_INVALID, "albedo_weight is nonzero but albedo is null");
    if (!normal && p->normal_weight != 0.0f) return fail(RT_ERR_INVALID, "normal_weight is nonzero but normal is null");
    const uint64_t n = (uint64_t)p->width * p->height;
    if (n >= (1ull << 31)) return fail(RT_ERR_INVALID, "width * height must be below 2^31");
    const Range in[4] = {{color, n * 12, "color", 4}, {variance, n * 12, "variance", 4}, {albedo, n * 12, "albedo", 4},
                         {normal, n * 12, "normal", 4}};
    const Range out[4] = {{out_linear, n * 12, "out_linear", 4}, {out_rgb8, n * 3, "out_rgb8", 1},
                          {out_variance, n * 12, "out_variance", 4},
                          {scratch, device_form ? denoise_var_scratch_bytes(n) : 0, "scratch", 16}};
    if (device_form) {
        for (const Range* g : {in, out})
            for (int k = 0; k < 4; ++k)
                if ((uintptr_t)g[k].p % g[k].align) return fail(RT_ERR_INVALID, std::string(g[k].name) + " is not " + std::to_string(g[k].align) + "-byte aligned");
    }
    // an output or the scratch must not overlap an input or each other
    for (int i = 0; i < 4; ++i) {
        for (const Range& r : in)
            if (overlap(out[i], r)) return fail(RT_ERR_INVALID, std::string(out[i].name) + " overlaps " + r.name);
        for (int j = 0; j < i; ++j)
            if (overlap(out[i], out[j])) return fail(RT_ERR_INVALID, std::string(out[i].name) + " overlaps " + out[j].name);
    }
    return RT_OK;
}

DenoiseVarArgs denoise_var_args(const rt_denoise_var_params& p, const float* color, const float* variance, const float* albedo,
                                const float* normal, void* scratch, float* out_linear, uint8_t* out_rgb8, float* out_variance) {
    return DenoiseVarArgs{p.width, p.height, p.iterations, p.color_weight, p.albedo_weight, p.normal_weight, p.variance_floor,
                          color, variance, albedo, normal, scratch, out_linear, out_rgb8, out_variance};
}

}  // namespace

uint64_t rtb200_denoise_var_scratch_bytes(uint32_t width, uint32_t height) { return denoise_var_scratch_bytes((uint64_t)width * height); }

int rtb200_denoise_var_device(int32_t device, const rt_denoise_var_params* p, const float* color, const float* variance,
                              const float* albedo, const float* normal, void* scratch, float* out_linear, uint8_t* out_rgb8,
                              float* out_variance, void* stream_in) {
  return guarded([&]() -> int {
    int rc = check_denoise_var(p, color, variance, albedo, normal, scratch, true, out_linear, out_rgb8, out_variance);
    if (rc != RT_OK) return rc;
    if ((uint64_t)p->width * p->height == 0) return RT_OK;
    CTX_PROLOGUE(device, ctx);
    if ((rc = check_device_ptrs(ctx->device, {{color, "color"}, {variance, "variance"}, {albedo, "albedo"}, {normal, "normal"},
                                              {scratch, "scratch"}, {out_linear, "out_linear"}, {out_rgb8, "out_rgb8"},
                                              {out_variance, "out_variance"}})) != RT_OK)
        return rc;
    CU(launch_denoise_var(denoise_var_args(*p, color, variance, albedo, normal, scratch, out_linear, out_rgb8, out_variance),
                          call_stream(ctx, stream_in)));
    return RT_OK;
  });
}

int rtb200_denoise_var(int32_t device, const rt_denoise_var_params* p, const float* color, const float* variance,
                       const float* albedo, const float* normal, float* out_linear, uint8_t* out_rgb8, float* out_variance,
                       rt_stats* stats) {
  return guarded([&]() -> int {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_denoise_var(p, color, variance, albedo, normal, nullptr, false, out_linear, out_rgb8, out_variance);
    if (rc != RT_OK) return rc;
    const uint64_t N = (uint64_t)p->width * p->height;
    if (N == 0) return RT_OK;
    auto wall0 = std::chrono::steady_clock::now();
    CTX_PROLOGUE(device, ctx);
    // device image: the inputs, the scratch, the outputs
    HostStage io;
    io.add_in(color, N * 12); io.add_in(variance, N * 12);
    io.add_in(albedo, albedo ? N * 12 : 0); io.add_in(normal, normal ? N * 12 : 0);
    io.add_in(nullptr, denoise_var_scratch_bytes(N));
    io.add_out(out_linear, out_linear ? N * 12 : 0); io.add_out(out_rgb8, out_rgb8 ? N * 3 : 0);
    io.add_out(out_variance, out_variance ? N * 12 : 0);
    rc = host_call(ctx, ctx->stream, io, nullptr, nullptr, wall0, stats, [&](unsigned long long*) -> int {
        CU(launch_denoise_var(denoise_var_args(*p, (const float*)io.a[0].dev, (const float*)io.a[1].dev, (const float*)io.a[2].dev,
                                               (const float*)io.a[3].dev, io.a[4].dev, (float*)io.a[5].dev, (uint8_t*)io.a[6].dev,
                                               (float*)io.a[7].dev), ctx->stream));
        return RT_OK;
    });
    if (rc != RT_OK || !stats) return rc;
    stats->kernel_launches = 2 * p->iterations + 1;
    return RT_OK;
  });
}

uint64_t rtb200_denoise_scratch_bytes(uint32_t width, uint32_t height) { return denoise_scratch_bytes((uint64_t)width * height); }

int rtb200_denoise_device(int32_t device, const rt_denoise_params* p, const float* color, const float* albedo, const float* normal,
                          void* scratch, float* out_linear, uint8_t* out_rgb8, void* stream_in) {
  return guarded([&]() -> int {
    int rc = check_denoise(p, color, albedo, normal, scratch, true, out_linear, out_rgb8);
    if (rc != RT_OK) return rc;
    if ((uint64_t)p->width * p->height == 0) return RT_OK;
    CTX_PROLOGUE(device, ctx);
    if ((rc = check_device_ptrs(ctx->device, {{color, "color"}, {albedo, "albedo"}, {normal, "normal"}, {scratch, "scratch"},
                                              {out_linear, "out_linear"}, {out_rgb8, "out_rgb8"}})) != RT_OK)
        return rc;
    CU(launch_denoise(denoise_args(*p, color, albedo, normal, scratch, out_linear, out_rgb8), call_stream(ctx, stream_in)));
    return RT_OK;
  });
}

int rtb200_denoise(int32_t device, const rt_denoise_params* p, const float* color, const float* albedo, const float* normal,
                   float* out_linear, uint8_t* out_rgb8, rt_stats* stats) {
  return guarded([&]() -> int {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_denoise(p, color, albedo, normal, nullptr, false, out_linear, out_rgb8);
    if (rc != RT_OK) return rc;
    const uint64_t N = (uint64_t)p->width * p->height;
    if (N == 0) return RT_OK;
    auto wall0 = std::chrono::steady_clock::now();
    CTX_PROLOGUE(device, ctx);
    // device image: the inputs, the scratch, the outputs
    HostStage io;
    io.add_in(color, N * 12); io.add_in(albedo, albedo ? N * 12 : 0); io.add_in(normal, normal ? N * 12 : 0);
    io.add_in(nullptr, denoise_scratch_bytes(N));
    io.add_out(out_linear, out_linear ? N * 12 : 0); io.add_out(out_rgb8, out_rgb8 ? N * 3 : 0);
    rc = host_call(ctx, ctx->stream, io, nullptr, nullptr, wall0, stats, [&](unsigned long long*) -> int {
        CU(launch_denoise(denoise_args(*p, (const float*)io.a[0].dev, (const float*)io.a[1].dev, (const float*)io.a[2].dev, io.a[3].dev,
                                       (float*)io.a[4].dev, (uint8_t*)io.a[5].dev), ctx->stream));
        return RT_OK;
    });
    if (rc != RT_OK || !stats) return rc;
    stats->kernel_launches = p->iterations + 1;
    return RT_OK;
  });
}
