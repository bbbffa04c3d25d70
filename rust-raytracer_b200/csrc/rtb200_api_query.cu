// rtb200_api_query.cu — closest-hit and occlusion queries of caller-supplied rays on a resident scene through the C ABI
// (DESIGN.md §4.10, §4.11), and the auxiliary buffers of its camera samples (§4.14), in both forms: device buffers on the
// caller's stream, or host buffers staged through the context's query block (HostStage, which the host form of
// rtb200_scene_trace_rays uses too).

#include "rtb200_host.cuh"

using namespace rtk;

int HostStage::place(DeviceCtx* ctx, size_t head) {
    Carver size;
    size.take(head);
    for (int k = 0; k < n; ++k) size.take(a[k].bytes);
    CU(ctx->query.ensure(size.off));
    Carver c(ctx->query.p);
    c.take(head);
    for (int k = 0; k < n; ++k) {
        char* d = (char*)c.take(a[k].bytes);
        a[k].dev = a[k].bytes ? d : nullptr;
    }
    return RT_OK;
}

int HostStage::copy(cudaStream_t st, bool back) {
    for (int k = 0; k < n; ++k) {
        const Array& x = a[k];
        if (!x.bytes || !(back ? x.out : x.in)) continue;
        CU(back ? cudaMemcpyAsync(x.out, x.dev, x.bytes, cudaMemcpyDeviceToHost, st) : cudaMemcpyAsync(x.dev, x.in, x.bytes, cudaMemcpyHostToDevice, st));
        (back ? d2h : h2d) += x.bytes;
    }
    return RT_OK;
}

// What a query writes: the outputs of rt_hits (closest-hit), or the occlusion bits. Output k is ptr[k], bytes[k] per ray.
struct QueryOut {
    bool any;             // occlusion
    rt_hits hits;         // closest-hit
    uint8_t* occluded;    // occlusion
    int count;
    void* ptr[6];
    uint32_t bytes[6];
    const char* name[6];
};
static QueryOut hits_out(const rt_hits& o) {
    QueryOut q{false, o, nullptr, 6, {o.t, o.sphere, o.point, o.normal, o.uv, o.front_face}, {8, 4, 24, 24, 16, 1},
               {"out->t", "out->sphere", "out->point", "out->normal", "out->uv", "out->front_face"}};
    return q;
}
static QueryOut occluded_out(uint8_t* o) {
    QueryOut q{true, rt_hits{}, o, 1, {o}, {1}, {"occluded"}};
    return q;
}
// the same outputs at other addresses (the host form's device image)
static QueryOut with_ptrs(const QueryOut& o, char* const* p) {
    if (o.any) return occluded_out((uint8_t*)p[0]);
    return hits_out(rt_hits{(double*)p[0], (uint32_t*)p[1], (double*)p[2], (double*)p[3], (double*)p[4], (uint8_t*)p[5]});
}

// The argument checks both forms of both kinds share (no device is touched).
static int check_query(rtb200_scene_handle h, const rt_rays* rays, const QueryOut* out) {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (!rays || !out) return fail(RT_ERR_INVALID, "rays or out is null");
    if (!rays->origin || !rays->direction) return fail(RT_ERR_INVALID, "rays->origin or rays->direction is null");
    bool any_out = false;
    for (int k = 0; k < out->count; ++k) any_out = any_out || out->ptr[k];
    if (!any_out) return fail(RT_ERR_INVALID, out->any ? "occluded is null" : "every output of out is null");
    return RT_OK;
}

// The one path of both forms: enqueue the query of the n rays `rays` into `out` (device buffers) on `st`, which the caller has
// ordered after the scene's last writer (scene_stream). Guard trips go to err[1], the counters to stat (null: not counted).
static int query_enqueue(rtb200_scene_handle h, const rt_rays& rays, uint32_t n, const QueryOut& out, unsigned long long* stat,
                         unsigned long long* err, cudaStream_t st) {
    int& occ = h->ctx->query_occ[out.any ? 1 : 0][h->mode];
    if (occ == 0) occ = query_max_ctas_per_sm(h->mode, out.any);
    if (occ <= 0) { occ = 0; return fail(RT_ERR_UNSUPPORTED, "no launch configuration of the query kernel fits shared memory"); }
    const int max_grid = h->ctx->sm_count * occ;
    auto common = [&](auto& q) {
        q.p = h->tp; q.p.stat = stat; q.p.err = err;
        q.origin = rays.origin; q.direction = rays.direction; q.t_max = rays.t_max;
        q.n = n;
    };
    if (out.any) {
        OcclusionParams q{};
        common(q);
        q.occluded = out.occluded;
        CU(launch_occluded(q, h->mode, max_grid, st));
        return RT_OK;
    }
    QueryParams q{};
    common(q);
    const rt_hits& o = out.hits;
    q.t = o.t; q.sphere = o.sphere; q.point = o.point; q.normal = o.normal; q.uv = o.uv; q.front_face = o.front_face;
    CU(launch_query(q, h->mode, max_grid, st));
    return RT_OK;
}

// After a stream-ordered reader of h's scene (a query, an AOV pass) enqueued on `st`: the next update, rebuild or edit and the
// release wait for the last one of each stream.
static int mark_query(rtb200_scene_handle h, cudaStream_t st) {
    uint32_t k = 0;
    while (k < h->n_queries && h->queries[k].stream != st) ++k;
    if (k == h->n_queries) {
        if (k == h->queries.size()) {
            cudaEvent_t e;
            CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            h->queries.push_back(rtb200_scene_t::QueryMark{st, e});
        }
        h->queries[k].stream = st;
        ++h->n_queries;
    }
    CU(cudaEventRecord(h->queries[k].done, st));
    return RT_OK;
}

// The device form of both kinds.
static int query_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const QueryOut* out, void* stream_in) {
    int rc = check_query(h, rays, out);
    if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    HANDLE_PROLOGUE(h);
    std::vector<std::pair<const void*, const char*>> ptrs = {{rays->origin, "rays->origin"}, {rays->direction, "rays->direction"},
                                                             {rays->t_max, "rays->t_max"}};
    for (int k = 0; k < out->count; ++k) ptrs.push_back({out->ptr[k], out->name[k]});
    if ((rc = check_device_ptrs(h, ptrs)) != RT_OK) return rc;
    cudaStream_t st;
    CU(scene_stream(h, stream_in, &st));
    if ((rc = query_enqueue(h, *rays, n, *out, nullptr, h->err, st)) != RT_OK) return rc;
    return mark_query(h, st);
}

// The host form of both kinds.
static int query_host(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const QueryOut* out, rt_stats* stats) {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_query(h, rays, out);
    if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    auto wall0 = std::chrono::steady_clock::now();
    HANDLE_PROLOGUE(h);
    // device image: counters, then rays and outputs
    const uint64_t N = n;
    HostStage io;
    io.add_in(rays->origin, N * 24); io.add_in(rays->direction, N * 24); io.add_in(rays->t_max, rays->t_max ? N * 8 : 0);
    for (int k = 0; k < out->count; ++k) io.add_out(out->ptr[k], out->ptr[k] ? N * out->bytes[k] : 0);
    cudaStream_t st;
    CU(scene_stream(h, nullptr, &st));
    unsigned long long hstat[kStatBytes / 8];
    rc = host_call(h->ctx, st, io, hstat, "internal error: the traversal guard tripped; the query results are not valid", wall0, stats,
                   [&](unsigned long long* stat) {
        char* dout[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
        for (int k = 0; k < out->count; ++k) dout[k] = io.a[3 + k].dev;
        const rt_rays drays{(const double*)io.a[0].dev, (const double*)io.a[1].dev, (const double*)io.a[2].dev};
        return query_enqueue(h, drays, n, with_ptrs(*out, dout), stat, stat + 30, st);
    });
    if (rc != RT_OK || !stats) return rc;
    stats->rays = hstat[0]; stats->candidates = hstat[1]; stats->clusters = hstat[4]; stats->nodes = hstat[6];
    stats->kernel_launches = 1; stats->batches = 1; stats->gpus_used = 1;
    return RT_OK;
}

int rtb200_scene_intersect_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_hits* out, void* stream_in) {
  return guarded([&]() -> int {
    const QueryOut o = hits_out(out ? *out : rt_hits{});
    return query_device(h, rays, n, out ? &o : nullptr, stream_in);
  });
}

int rtb200_scene_intersect(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_hits* out, rt_stats* stats) {
  return guarded([&]() -> int {
    const QueryOut o = hits_out(out ? *out : rt_hits{});
    return query_host(h, rays, n, out ? &o : nullptr, stats);
  });
}

int rtb200_scene_occluded_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, uint8_t* occluded, void* stream_in) {
  return guarded([&]() -> int {
    const QueryOut o = occluded_out(occluded);
    return query_device(h, rays, n, &o, stream_in);
  });
}

int rtb200_scene_occluded(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, uint8_t* occluded, rt_stats* stats) {
  return guarded([&]() -> int {
    const QueryOut o = occluded_out(occluded);
    return query_host(h, rays, n, &o, stats);
  });
}


// ---- auxiliary buffers of the camera samples (DESIGN.md §4.14) ----

// The outputs of rt_aov_out: output k is ptr[k], bytes[k] per pixel.
struct AovOut {
    void* ptr[5];
    const char* name[5];
};
static const uint32_t kAovBytes[5] = {12, 12, 4, 4, 24};
static AovOut aov_out(const rt_aov_out& o) {
    return AovOut{{o.albedo, o.normal, o.hits, o.sphere, o.point}, {"out->albedo", "out->normal", "out->hits", "out->sphere", "out->point"}};
}

// The argument checks of both forms (no device is touched).
static int check_aov(rtb200_scene_handle h, const rt_aov_params* p, const rt_frame* view, const rt_aov_out* out) {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (!p) return fail(RT_ERR_INVALID, "params is null");
    if (!out) return fail(RT_ERR_INVALID, "out is null");
    const AovOut o = aov_out(*out);
    if (std::none_of(o.ptr, o.ptr + 5, [](void* q) { return q != nullptr; })) return fail(RT_ERR_INVALID, "every output of out is null");
    if (p->samples == 0) return fail(RT_ERR_INVALID, "rt_aov_params.samples must be >= 1");
    if ((uint64_t)p->sample0 + p->samples > (1ull << 32)) return fail(RT_ERR_INVALID, "rt_aov_params.sample0 + samples exceeds 2^32");
    if (p->reserved[0] != 0 || p->reserved[1] != 0) return fail(RT_ERR_INVALID, "rt_aov_params.reserved must be 0");
    if (view && view->reserved != 0) return fail(RT_ERR_INVALID, "view->reserved must be 0");
    return RT_OK;
}

// The one path of both forms: enqueue the pass over every local pixel of h into `out` (device buffers) on `st`, which the caller
// has ordered after the scene's last writer (scene_stream). Guard trips go to err[1], the counters to stat (null: not counted).
static int aov_enqueue(rtb200_scene_handle h, const rt_aov_params& prm, const rt_frame* view, const AovOut& out,
                       unsigned long long* stat, unsigned long long* err, cudaStream_t st) {
    const bool lens = h->tp.lens.radius != 0.0;   // the handle's lens (rtb200_scene_set_lens)
    int& occ = h->ctx->query_occ[lens ? 3 : 2][h->mode];
    if (occ == 0) occ = aov_max_ctas_per_sm(h->mode, lens);
    if (occ <= 0) { occ = 0; return fail(RT_ERR_UNSUPPORTED, "no launch configuration of the aov kernel fits shared memory"); }
    AovParams q{};
    q.p = h->tp; q.p.stat = stat; q.p.err = err;
    if (view) { q.p.cam = view->camera; q.p.key0 = (uint32_t)view->seed; q.p.key1 = (uint32_t)(view->seed >> 32); }
    q.albedo = (float*)out.ptr[0]; q.normal = (float*)out.ptr[1]; q.hits = (uint32_t*)out.ptr[2]; q.sphere = (uint32_t*)out.ptr[3];
    q.point = (double*)out.ptr[4];
    q.samples = prm.samples; q.sample0 = prm.sample0;
    q.n = h->tp.npix_local;
    CU(launch_aov(q, h->mode, h->ctx->sm_count * occ, st));
    return RT_OK;
}

int rtb200_scene_aov_device(rtb200_scene_handle h, const rt_aov_params* p, const rt_frame* view, const rt_aov_out* out, void* stream_in) {
  return guarded([&]() -> int {
    int rc = check_aov(h, p, view, out);
    if (rc != RT_OK) return rc;
    HANDLE_PROLOGUE(h);
    const AovOut o = aov_out(*out);
    std::vector<std::pair<const void*, const char*>> ptrs;
    for (int k = 0; k < 5; ++k) ptrs.push_back({o.ptr[k], o.name[k]});
    if ((rc = check_device_ptrs(h, ptrs)) != RT_OK) return rc;
    if (h->tp.npix_local == 0) return RT_OK;
    cudaStream_t st;
    CU(scene_stream(h, stream_in, &st));
    if ((rc = aov_enqueue(h, *p, view, o, nullptr, h->err, st)) != RT_OK) return rc;
    return mark_query(h, st);
  });
}

int rtb200_scene_aov(rtb200_scene_handle h, const rt_aov_params* p, const rt_frame* view, const rt_aov_out* out, rt_stats* stats) {
  return guarded([&]() -> int {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_aov(h, p, view, out);
    if (rc != RT_OK) return rc;
    const uint64_t N = h->tp.npix_local;
    if (N == 0) return RT_OK;
    auto wall0 = std::chrono::steady_clock::now();
    HANDLE_PROLOGUE(h);
    // device image: counters, then the outputs
    const AovOut o = aov_out(*out);
    HostStage io;
    for (int k = 0; k < 5; ++k) io.add_out(o.ptr[k], o.ptr[k] ? N * kAovBytes[k] : 0);
    cudaStream_t st;
    CU(scene_stream(h, nullptr, &st));
    unsigned long long hstat[kStatBytes / 8];
    rc = host_call(h->ctx, st, io, hstat, "internal error: the traversal guard tripped; the aov results are not valid", wall0, stats,
                   [&](unsigned long long* stat) {
        AovOut dout = o;
        for (int k = 0; k < 5; ++k) dout.ptr[k] = io.a[k].dev;
        return aov_enqueue(h, *p, view, dout, stat, stat + 30, st);
    });
    if (rc != RT_OK || !stats) return rc;
    stats->rays = hstat[0]; stats->samples = hstat[3]; stats->candidates = hstat[1]; stats->clusters = hstat[4]; stats->nodes = hstat[6];
    stats->kernel_launches = 1; stats->batches = 1; stats->frames = 1; stats->gpus_used = 1;
    return RT_OK;
  });
}
