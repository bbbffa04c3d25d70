// rtb200_api_denoise.cu — denoising a frame with its auxiliary buffers through the C ABI (DESIGN.md §4.15), in both forms:
// device buffers on the caller's stream with the caller's scratch, or host buffers staged through the context's query block
// (HostStage). The kernels are in rtb200_denoise.cu.

#include "rtb200_host.cuh"

using namespace rtk;

namespace {

struct Range { const void* p; uint64_t bytes; const char* name; };

bool overlap(const Range& a, const Range& b) {
    if (!a.p || !b.p || !a.bytes || !b.bytes) return false;
    const uintptr_t a0 = (uintptr_t)a.p, b0 = (uintptr_t)b.p;
    return a0 < b0 + b.bytes && b0 < a0 + a.bytes;
}

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
    if (device_form) {
        for (const Range& r : {Range{color, 0, "color"}, Range{albedo, 0, "albedo"}, Range{normal, 0, "normal"}, Range{out_linear, 0, "out_linear"}})
            if ((uintptr_t)r.p % 4) return fail(RT_ERR_INVALID, std::string(r.name) + " is not 4-byte aligned");
        if ((uintptr_t)scratch % 16) return fail(RT_ERR_INVALID, "scratch is not 16-byte aligned");
    }
    // an output or the scratch must not overlap an input or each other
    const Range in[3] = {{color, n * 12, "color"}, {albedo, n * 12, "albedo"}, {normal, n * 12, "normal"}};
    const Range out[3] = {{out_linear, n * 12, "out_linear"}, {out_rgb8, n * 3, "out_rgb8"},
                          {scratch, device_form ? denoise_scratch_bytes(n) : 0, "scratch"}};
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

}  // namespace

uint64_t rtb200_denoise_scratch_bytes(uint32_t width, uint32_t height) { return denoise_scratch_bytes((uint64_t)width * height); }

int rtb200_denoise_device(int32_t device, const rt_denoise_params* p, const float* color, const float* albedo, const float* normal,
                          void* scratch, float* out_linear, uint8_t* out_rgb8, void* stream_in) {
  return guarded([&]() -> int {
    int rc = check_denoise(p, color, albedo, normal, scratch, true, out_linear, out_rgb8);
    if (rc != RT_OK) return rc;
    if ((uint64_t)p->width * p->height == 0) return RT_OK;
    DeviceRestore restore_;
    DeviceCtx* ctx = nullptr;
    if ((rc = get_ctx(device, &ctx)) != RT_OK) return rc;
    std::lock_guard<std::recursive_mutex> lock_(ctx->mu);
    if ((rc = check_device_ptrs(ctx->device, {{color, "color"}, {albedo, "albedo"}, {normal, "normal"}, {scratch, "scratch"},
                                              {out_linear, "out_linear"}, {out_rgb8, "out_rgb8"}})) != RT_OK)
        return rc;
    const cudaStream_t st = stream_in ? (cudaStream_t)stream_in : ctx->stream;
    CU(launch_denoise(denoise_args(*p, color, albedo, normal, scratch, out_linear, out_rgb8), st));
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
    DeviceRestore restore_;
    DeviceCtx* ctx = nullptr;
    if ((rc = get_ctx(device, &ctx)) != RT_OK) return rc;
    std::lock_guard<std::recursive_mutex> lock_(ctx->mu);
    for (auto& e : ctx->query_ev) if (!e) CU(cudaEventCreate(&e));
    // device image: the inputs, the scratch, the outputs
    HostStage io;
    io.add_in(color, N * 12); io.add_in(albedo, albedo ? N * 12 : 0); io.add_in(normal, normal ? N * 12 : 0);
    io.add_in(nullptr, denoise_scratch_bytes(N));
    io.add_out(out_linear, out_linear ? N * 12 : 0); io.add_out(out_rgb8, out_rgb8 ? N * 3 : 0);
    if ((rc = io.place(ctx, 0)) != RT_OK) return rc;
    const cudaStream_t st = ctx->stream;
    cudaEvent_t* ev = ctx->query_ev;
    CU(cudaEventRecord(ev[0], st));
    if ((rc = io.copy(st, false)) != RT_OK) return rc;
    CU(cudaEventRecord(ev[1], st));
    CU(launch_denoise(denoise_args(*p, (const float*)io.a[0].dev, (const float*)io.a[1].dev, (const float*)io.a[2].dev, io.a[3].dev,
                                   (float*)io.a[4].dev, (uint8_t*)io.a[5].dev), st));
    CU(cudaEventRecord(ev[2], st));
    if ((rc = io.copy(st, true)) != RT_OK) return rc;
    CU(cudaEventRecord(ev[3], st));
    CU(cudaStreamSynchronize(st));
    if (!stats) return RT_OK;
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, ev[0], ev[3])); stats->device_ms = ms;
    CU(cudaEventElapsedTime(&ms, ev[1], ev[2])); stats->trace_ms = ms;
    stats->kernel_launches = p->iterations + 1;
    stats->h2d_bytes = io.h2d; stats->d2h_bytes = io.d2h;
    stats->wall_ms = ms_since(wall0);
    return RT_OK;
  });
}
