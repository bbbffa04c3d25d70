// rtb200_api_temporal.cu — the temporal accumulation of animation frames through the C ABI (DESIGN.md §4.16), unclamped and
// with the history clamp (§4.20), with or without the variance of each pixel's mean (§4.21), in both forms:
// device buffers on the caller's stream, or host buffers staged through the context's query block (HostStage). The kernel is
// in rtb200_temporal.cu.

#include "rtb200_host.cuh"

using namespace rtk;

namespace {

// The argument checks of both forms (no device is touched); the alignment is checked in the device form only.
int check_temporal(const rt_temporal_params* p, const rt_temporal_frame* cur, const rt_temporal_history* prev, const double* motion,
                   const rt_temporal_out* out, bool device_form) {
    if (!p) return fail(RT_ERR_INVALID, "params is null");
    if (!cur || !cur->color || !cur->sphere || !cur->point) return fail(RT_ERR_INVALID, "cur or one of its arrays is null");
    if (!out || !out->color || !out->length) return fail(RT_ERR_INVALID, "out or one of its arrays is null");
    if (prev && !(prev->color && prev->length && prev->sphere && prev->point))
        return fail(RT_ERR_INVALID, "prev is a partial previous frame: give all four arrays or no prev");
    if (p->reserved[0] != 0 || p->reserved[1] != 0) return fail(RT_ERR_INVALID, "rt_temporal_params.reserved must be 0");
    if (p->max_history == 0) return fail(RT_ERR_INVALID, "rt_temporal_params.max_history must be >= 1");
    if (!(std::isfinite(p->depth_tol) && p->depth_tol >= 0.0)) return fail(RT_ERR_INVALID, "rt_temporal_params.depth_tol must be finite and >= 0");
    if (!motion && p->n_motion > 0) return fail(RT_ERR_INVALID, "motion is null but n_motion > 0");
    const uint64_t n = (uint64_t)p->width * p->height;
    if (n >= (1ull << 31)) return fail(RT_ERR_INVALID, "width * height must be below 2^31");
    const Range in[8] = {{cur->color, n * 12, "cur.color", 4}, {cur->sphere, n * 4, "cur.sphere", 4}, {cur->point, n * 24, "cur.point", 8},
                         {prev ? prev->color : nullptr, n * 12, "prev.color", 4}, {prev ? prev->length : nullptr, n * 4, "prev.length", 4},
                         {prev ? prev->sphere : nullptr, n * 4, "prev.sphere", 4}, {prev ? prev->point : nullptr, n * 24, "prev.point", 8},
                         {motion, (uint64_t)p->n_motion * 24, "motion", 8}};
    const Range outs[2] = {{out->color, n * 12, "out.color", 4}, {out->length, n * 4, "out.length", 4}};
    if (device_form) {
        for (const Range* g : {in, outs})
            for (int k = 0; k < (g == in ? 8 : 2); ++k)
                if ((uintptr_t)g[k].p % g[k].align) return fail(RT_ERR_INVALID, std::string(g[k].name) + " is not " + std::to_string(g[k].align) + "-byte aligned");
    }
    // an output must not overlap an input or the other output
    for (int i = 0; i < 2; ++i) {
        for (const Range& r : in)
            if (overlap(outs[i], r)) return fail(RT_ERR_INVALID, std::string(outs[i].name) + " overlaps " + r.name);
        if (i == 1 && overlap(outs[1], outs[0])) return fail(RT_ERR_INVALID, "out.length overlaps out.color");
    }
    return RT_OK;
}

// The clamp's checks (after check_temporal's, before any device work).
int check_clamp(const rt_temporal_clamp* c) {
    if (!c) return fail(RT_ERR_INVALID, "clamp is null");
    if (!(std::isfinite(c->gamma) && c->gamma >= 0.0f)) return fail(RT_ERR_INVALID, "rt_temporal_clamp.gamma must be finite and >= 0");
    if (c->radius < 1 || c->radius > 3) return fail(RT_ERR_INVALID, "rt_temporal_clamp.radius must be in [1, 3]");
    if (c->reserved[0] != 0 || c->reserved[1] != 0) return fail(RT_ERR_INVALID, "rt_temporal_clamp.reserved must be 0");
    return RT_OK;
}

// The variance's checks (after check_temporal's, before any device work): both variance arrays of this frame given, the
// history's exactly with prev, 4-byte alignment in the device form, and out_variance apart from every other array.
int check_var(const rt_temporal_params* p, const rt_temporal_frame* cur, const float* variance, const rt_temporal_history* prev,
              const float* prev_variance, const double* motion, const rt_temporal_out* out, const float* out_variance, bool device_form) {
    if (!variance) return fail(RT_ERR_INVALID, "variance is null");
    if (!out_variance) return fail(RT_ERR_INVALID, "out_variance is null");
    if (!prev != !prev_variance) return fail(RT_ERR_INVALID, prev ? "prev is given without prev_variance" : "prev_variance is given without prev");
    const uint64_t n = (uint64_t)p->width * p->height;
    const Range var[2] = {{variance, n * 12, "variance", 4}, {prev_variance, n * 12, "prev_variance", 4}};
    const Range ov{out_variance, n * 12, "out_variance", 4};
    if (device_form)
        for (const Range& r : {var[0], var[1], ov})
            if ((uintptr_t)r.p % r.align) return fail(RT_ERR_INVALID, std::string(r.name) + " is not 4-byte aligned");
    const Range others[10] = {{cur->color, n * 12, "cur.color", 4}, {cur->sphere, n * 4, "cur.sphere", 4}, {cur->point, n * 24, "cur.point", 8},
                              {prev ? prev->color : nullptr, n * 12, "prev.color", 4}, {prev ? prev->length : nullptr, n * 4, "prev.length", 4},
                              {prev ? prev->sphere : nullptr, n * 4, "prev.sphere", 4}, {prev ? prev->point : nullptr, n * 24, "prev.point", 8},
                              {motion, (uint64_t)p->n_motion * 24, "motion", 8},
                              {out->color, n * 12, "out.color", 4}, {out->length, n * 4, "out.length", 4}};
    for (const Range& r : var)
        if (overlap(ov, r)) return fail(RT_ERR_INVALID, std::string("out_variance overlaps ") + r.name);
    for (const Range& r : others)
        if (overlap(ov, r)) return fail(RT_ERR_INVALID, std::string("out_variance overlaps ") + r.name);
    for (int i = 8; i < 10; ++i)
        for (const Range& r : var)
            if (overlap(others[i], r)) return fail(RT_ERR_INVALID, std::string(others[i].name) + " overlaps " + r.name);
    return RT_OK;
}

TemporalArgs temporal_args(const rt_temporal_params& p, const float* color, const uint32_t* sphere, const double* point, const float* h_color,
                           const uint32_t* h_length, const uint32_t* h_sphere, const double* h_point, const double* motion,
                           float* out_color, uint32_t* out_length) {
    return TemporalArgs{p.width, p.height, p.max_history, p.n_motion, p.camera, p.prev_camera, p.depth_tol, color, sphere, point,
                        h_color, h_length, h_sphere, h_point, p.n_motion ? motion : nullptr, out_color, out_length};
}

// Every device form; clamp null: unclamped (rtb200_temporal_device), else checked by the caller; var null: no variance, else
// its three planes, checked by the caller.
int temporal_device(int32_t device, const rt_temporal_params* p, const TemporalClamp* clamp, const TemporalVar* var,
                    const rt_temporal_frame* cur, const rt_temporal_history* prev, const double* motion, const rt_temporal_out* out,
                    void* stream_in) {
    if ((uint64_t)p->width * p->height == 0) return RT_OK;
    CTX_PROLOGUE(device, ctx);
    const rt_temporal_history none{};
    const rt_temporal_history& h = prev ? *prev : none;
    int rc;
    if ((rc = check_device_ptrs(ctx->device, {{cur->color, "cur.color"}, {cur->sphere, "cur.sphere"}, {cur->point, "cur.point"},
                                              {h.color, "prev.color"}, {h.length, "prev.length"}, {h.sphere, "prev.sphere"},
                                              {h.point, "prev.point"}, {p->n_motion ? motion : nullptr, "motion"},
                                              {out->color, "out.color"}, {out->length, "out.length"}})) != RT_OK)
        return rc;
    if (var && (rc = check_device_ptrs(ctx->device, {{var->var, "variance"}, {var->h_var, "prev_variance"}, {var->out_var, "out_variance"}})) != RT_OK)
        return rc;
    CU(launch_temporal(temporal_args(*p, cur->color, cur->sphere, cur->point, h.color, h.length, h.sphere, h.point, motion, out->color,
                                     out->length), clamp, var, call_stream(ctx, stream_in)));
    return RT_OK;
}

// Every host form, after the checks; clamp and var as temporal_device (var's planes are host arrays here).
int temporal_host(int32_t device, const rt_temporal_params* p, const TemporalClamp* clamp, const TemporalVar* var,
                  const rt_temporal_frame* cur, const rt_temporal_history* prev, const double* motion, const rt_temporal_out* out,
                  rt_stats* stats) {
    const uint64_t N = (uint64_t)p->width * p->height;
    if (N == 0) return RT_OK;
    auto wall0 = std::chrono::steady_clock::now();
    CTX_PROLOGUE(device, ctx);
    // device image: this frame, the previous frame (absent: 0 bytes, a null dev), the motion, the outputs, then with var the
    // variance planes: this frame's, the previous frame's and the output's
    const uint64_t hb = prev ? N : 0;
    HostStage io;
    io.add_in(cur->color, N * 12); io.add_in(cur->sphere, N * 4); io.add_in(cur->point, N * 24);
    io.add_in(prev ? prev->color : nullptr, hb * 12); io.add_in(prev ? prev->length : nullptr, hb * 4);
    io.add_in(prev ? prev->sphere : nullptr, hb * 4); io.add_in(prev ? prev->point : nullptr, hb * 24);
    io.add_in(motion, (uint64_t)p->n_motion * 24);
    io.add_out(out->color, N * 12); io.add_out(out->length, N * 4);
    if (var) { io.add_in(var->var, N * 12); io.add_in(var->h_var, hb * 12); io.add_out(var->out_var, N * 12); }
    int rc = host_call(ctx, ctx->stream, io, nullptr, nullptr, wall0, stats, [&](unsigned long long*) -> int {
        auto dev = [&](int k) { return (const void*)io.a[k].dev; };
        const TemporalVar dv{(const float*)dev(10), (const float*)dev(11), (float*)io.a[12].dev};
        CU(launch_temporal(temporal_args(*p, (const float*)dev(0), (const uint32_t*)dev(1), (const double*)dev(2), (const float*)dev(3),
                                         (const uint32_t*)dev(4), (const uint32_t*)dev(5), (const double*)dev(6), (const double*)dev(7),
                                         (float*)io.a[8].dev, (uint32_t*)io.a[9].dev), clamp, var ? &dv : nullptr, ctx->stream));
        return RT_OK;
    });
    if (rc != RT_OK || !stats) return rc;
    stats->kernel_launches = 1;
    return RT_OK;
}

}  // namespace

int rtb200_temporal_device(int32_t device, const rt_temporal_params* p, const rt_temporal_frame* cur, const rt_temporal_history* prev,
                           const double* motion, const rt_temporal_out* out, void* stream_in) {
  return guarded([&]() -> int {
    const int rc = check_temporal(p, cur, prev, motion, out, true);
    return rc != RT_OK ? rc : temporal_device(device, p, nullptr, nullptr, cur, prev, motion, out, stream_in);
  });
}

int rtb200_temporal_clamped_device(int32_t device, const rt_temporal_params* p, const rt_temporal_clamp* clamp, const rt_temporal_frame* cur,
                                   const rt_temporal_history* prev, const double* motion, const rt_temporal_out* out, void* stream_in) {
  return guarded([&]() -> int {
    int rc = check_temporal(p, cur, prev, motion, out, true);
    if (rc != RT_OK || (rc = check_clamp(clamp)) != RT_OK) return rc;
    const TemporalClamp c{clamp->gamma, clamp->radius};
    return temporal_device(device, p, &c, nullptr, cur, prev, motion, out, stream_in);
  });
}

int rtb200_temporal(int32_t device, const rt_temporal_params* p, const rt_temporal_frame* cur, const rt_temporal_history* prev,
                    const double* motion, const rt_temporal_out* out, rt_stats* stats) {
  return guarded([&]() -> int {
    if (stats) memset(stats, 0, sizeof *stats);
    const int rc = check_temporal(p, cur, prev, motion, out, false);
    return rc != RT_OK ? rc : temporal_host(device, p, nullptr, nullptr, cur, prev, motion, out, stats);
  });
}

int rtb200_temporal_clamped(int32_t device, const rt_temporal_params* p, const rt_temporal_clamp* clamp, const rt_temporal_frame* cur,
                            const rt_temporal_history* prev, const double* motion, const rt_temporal_out* out, rt_stats* stats) {
  return guarded([&]() -> int {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_temporal(p, cur, prev, motion, out, false);
    if (rc != RT_OK || (rc = check_clamp(clamp)) != RT_OK) return rc;
    const TemporalClamp c{clamp->gamma, clamp->radius};
    return temporal_host(device, p, &c, nullptr, cur, prev, motion, out, stats);
  });
}

int rtb200_temporal_var_device(int32_t device, const rt_temporal_params* p, const rt_temporal_clamp* clamp, const rt_temporal_frame* cur,
                               const float* variance, const rt_temporal_history* prev, const float* prev_variance, const double* motion,
                               const rt_temporal_out* out, float* out_variance, void* stream_in) {
  return guarded([&]() -> int {
    int rc = check_temporal(p, cur, prev, motion, out, true);
    if (rc != RT_OK || (clamp && (rc = check_clamp(clamp)) != RT_OK) ||
        (rc = check_var(p, cur, variance, prev, prev_variance, motion, out, out_variance, true)) != RT_OK)
        return rc;
    const TemporalClamp c{clamp ? clamp->gamma : 0.0f, clamp ? clamp->radius : 0u};
    const TemporalVar v{variance, prev_variance, out_variance};
    return temporal_device(device, p, clamp ? &c : nullptr, &v, cur, prev, motion, out, stream_in);
  });
}

int rtb200_temporal_var(int32_t device, const rt_temporal_params* p, const rt_temporal_clamp* clamp, const rt_temporal_frame* cur,
                        const float* variance, const rt_temporal_history* prev, const float* prev_variance, const double* motion,
                        const rt_temporal_out* out, float* out_variance, rt_stats* stats) {
  return guarded([&]() -> int {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_temporal(p, cur, prev, motion, out, false);
    if (rc != RT_OK || (clamp && (rc = check_clamp(clamp)) != RT_OK) ||
        (rc = check_var(p, cur, variance, prev, prev_variance, motion, out, out_variance, false)) != RT_OK)
        return rc;
    const TemporalClamp c{clamp ? clamp->gamma : 0.0f, clamp ? clamp->radius : 0u};
    const TemporalVar v{variance, prev_variance, out_variance};
    return temporal_host(device, p, clamp ? &c : nullptr, &v, cur, prev, motion, out, stats);
  });
}
