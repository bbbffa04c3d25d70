// rtb200_api_query.cu — closest-hit and occlusion queries of caller-supplied rays, nearest-sphere and overlap queries of
// caller-supplied points (DESIGN.md §4.10, §4.11, §4.19) on a resident scene through the C ABI, and the auxiliary buffers of
// its camera samples (§4.14), in both forms: device buffers on the caller's stream, or host buffers staged through the
// context's query block (HostStage, which the host form of rtb200_scene_trace_rays uses too).

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

// The four kinds of query: closest hits and occlusion of rays (§4.10, §4.11), nearest spheres and overlaps of points (§4.19).
enum QueryKind { QK_HITS, QK_OCCLUDED, QK_NEAREST, QK_OVERLAPS };

// What a query reads: input k is ptr[k], bytes[k] per ray or point (a null optional input: not read). The rays' origin,
// direction and t_max, or the points' point and bound; `given` is false when the caller passed no rt_rays or rt_points.
struct QueryIn {
    bool given;
    int count;
    const void* ptr[3];
    uint32_t bytes[3];
    const char* name[3];
};
static QueryIn rays_in(const rt_rays* p) {
    const rt_rays r = p ? *p : rt_rays{};
    return QueryIn{p != nullptr, 3, {r.origin, r.direction, r.t_max}, {24, 24, 8}, {"rays->origin", "rays->direction", "rays->t_max"}};
}
static QueryIn points_in(const rt_points* p) {
    const rt_points q = p ? *p : rt_points{};
    return QueryIn{p != nullptr, 2, {q.point, q.bound}, {24, 8}, {"q->point", "q->bound"}};
}

// What a query writes: the outputs of rt_hits (closest-hit), the occlusion bits, the outputs of rt_nearest, or the overlap bits.
// Output k is ptr[k], bytes[k] per ray or point; `given` is false when the caller passed no rt_hits or rt_nearest.
struct QueryOut {
    QueryKind kind;
    bool given;
    int count;
    void* ptr[6];
    uint32_t bytes[6];
    const char* name[6];
};
static QueryOut hits_out(const rt_hits* p) {
    const rt_hits o = p ? *p : rt_hits{};
    return QueryOut{QK_HITS, p != nullptr, 6, {o.t, o.sphere, o.point, o.normal, o.uv, o.front_face}, {8, 4, 24, 24, 16, 1},
                    {"out->t", "out->sphere", "out->point", "out->normal", "out->uv", "out->front_face"}};
}
static QueryOut occluded_out(uint8_t* o) { return QueryOut{QK_OCCLUDED, true, 1, {o}, {1}, {"occluded"}}; }
static QueryOut nearest_out(const rt_nearest* p) {
    const rt_nearest o = p ? *p : rt_nearest{};
    return QueryOut{QK_NEAREST, p != nullptr, 2, {o.distance, o.sphere}, {8, 4}, {"out->distance", "out->sphere"}};
}
static QueryOut overlaps_out(uint8_t* o) { return QueryOut{QK_OVERLAPS, true, 1, {o}, {1}, {"overlaps"}}; }

// The argument checks all forms of all kinds share (no device is touched).
static int check_query(rtb200_scene_handle h, const QueryIn* in, const QueryOut* out) {
    const bool rays = out->kind == QK_HITS || out->kind == QK_OCCLUDED;
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (!in->given || !out->given) return fail(RT_ERR_INVALID, rays ? "rays or out is null" : "q or out is null");
    if (rays && (!in->ptr[0] || !in->ptr[1])) return fail(RT_ERR_INVALID, "rays->origin or rays->direction is null");
    if (!rays && !in->ptr[0]) return fail(RT_ERR_INVALID, "q->point is null");
    if (out->kind == QK_OVERLAPS && !in->ptr[1]) return fail(RT_ERR_INVALID, "q->bound is null: overlaps needs the balls' radii");
    bool any_out = false;
    for (int k = 0; k < out->count; ++k) any_out = any_out || out->ptr[k];
    if (!any_out) return fail(RT_ERR_INVALID, out->count == 1 ? (out->kind == QK_OCCLUDED ? "occluded is null" : "overlaps is null")
                                                              : "every output of out is null");
    return RT_OK;
}

// The one path of both forms: enqueue the query of the n rays or points `in` into `out` (device buffers) on `st`, which the caller
// has ordered after the scene's last writer (scene_stream). Guard trips go to err[1], the counters to stat (null: not counted).
static int query_enqueue(rtb200_scene_handle h, const QueryIn& in, uint32_t n, const QueryOut& out, unsigned long long* stat,
                         unsigned long long* err, cudaStream_t st) {
    static const int kOccRow[4] = {0, 1, 4, 5};   // DeviceCtx::query_occ's row of each kind
    const bool pts = out.kind == QK_NEAREST || out.kind == QK_OVERLAPS;
    const bool any = out.kind == QK_OCCLUDED || out.kind == QK_OVERLAPS;
    int& occ = h->ctx->query_occ[kOccRow[out.kind]][h->mode];
    if (occ == 0) occ = pts ? distance_max_ctas_per_sm(h->mode, any) : query_max_ctas_per_sm(h->mode, any);
    if (occ <= 0) { occ = 0; return fail(RT_ERR_UNSUPPORTED, "no launch configuration of the query kernel fits shared memory"); }
    const int max_grid = h->ctx->sm_count * occ;
    if (pts) {
        DistanceParams q{};
        q.p = h->tp; q.p.stat = stat; q.p.err = err;
        q.point = (const double*)in.ptr[0]; q.bound = (const double*)in.ptr[1];
        q.distance = any ? nullptr : (double*)out.ptr[0]; q.sphere = any ? nullptr : (uint32_t*)out.ptr[1];
        q.overlaps = any ? (uint8_t*)out.ptr[0] : nullptr;
        q.n = n;
        CU(launch_distance(q, h->mode, any, max_grid, st));
        return RT_OK;
    }
    auto common = [&](auto& q) {
        q.p = h->tp; q.p.stat = stat; q.p.err = err;
        q.origin = (const double*)in.ptr[0]; q.direction = (const double*)in.ptr[1]; q.t_max = (const double*)in.ptr[2];
        q.n = n;
    };
    if (any) {
        OcclusionParams q{};
        common(q);
        q.occluded = (uint8_t*)out.ptr[0];
        CU(launch_occluded(q, h->mode, max_grid, st));
        return RT_OK;
    }
    QueryParams q{};
    common(q);
    q.t = (double*)out.ptr[0]; q.sphere = (uint32_t*)out.ptr[1]; q.point = (double*)out.ptr[2]; q.normal = (double*)out.ptr[3];
    q.uv = (double*)out.ptr[4]; q.front_face = (uint8_t*)out.ptr[5];
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

// The device form of every kind.
static int query_device(rtb200_scene_handle h, const QueryIn* in, uint32_t n, const QueryOut* out, void* stream_in) {
    int rc = check_query(h, in, out);
    if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    HANDLE_PROLOGUE(h);
    std::vector<std::pair<const void*, const char*>> ptrs;
    for (int k = 0; k < in->count; ++k) ptrs.push_back({in->ptr[k], in->name[k]});
    for (int k = 0; k < out->count; ++k) ptrs.push_back({out->ptr[k], out->name[k]});
    if ((rc = check_device_ptrs(h, ptrs)) != RT_OK) return rc;
    cudaStream_t st;
    CU(scene_stream(h, stream_in, &st));
    if ((rc = query_enqueue(h, *in, n, *out, nullptr, h->err, st)) != RT_OK) return rc;
    return mark_query(h, st);
}

// The host form of every kind.
static int query_host(rtb200_scene_handle h, const QueryIn* in, uint32_t n, const QueryOut* out, rt_stats* stats) {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_query(h, in, out);
    if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    auto wall0 = std::chrono::steady_clock::now();
    HANDLE_PROLOGUE(h);
    // device image: counters, then the inputs and outputs
    const uint64_t N = n;
    HostStage io;
    for (int k = 0; k < in->count; ++k) io.add_in(in->ptr[k], in->ptr[k] ? N * in->bytes[k] : 0);
    for (int k = 0; k < out->count; ++k) io.add_out(out->ptr[k], out->ptr[k] ? N * out->bytes[k] : 0);
    cudaStream_t st;
    CU(scene_stream(h, nullptr, &st));
    unsigned long long hstat[kStatBytes / 8];
    rc = host_call(h->ctx, st, io, hstat, "internal error: the traversal guard tripped; the query results are not valid", wall0, stats,
                   [&](unsigned long long* stat) {
        QueryIn din = *in;
        QueryOut dout = *out;
        for (int k = 0; k < in->count; ++k) din.ptr[k] = io.a[k].dev;
        for (int k = 0; k < out->count; ++k) dout.ptr[k] = io.a[in->count + k].dev;
        return query_enqueue(h, din, n, dout, stat, stat + 30, st);
    });
    if (rc != RT_OK || !stats) return rc;
    stats->rays = hstat[0]; stats->candidates = hstat[1]; stats->clusters = hstat[4]; stats->nodes = hstat[6];
    stats->kernel_launches = 1; stats->batches = 1; stats->gpus_used = 1;
    return RT_OK;
}

int rtb200_scene_intersect_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_hits* out, void* stream_in) {
  return guarded([&]() -> int {
    const QueryIn i = rays_in(rays);
    const QueryOut o = hits_out(out);
    return query_device(h, &i, n, &o, stream_in);
  });
}

int rtb200_scene_intersect(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_hits* out, rt_stats* stats) {
  return guarded([&]() -> int {
    const QueryIn i = rays_in(rays);
    const QueryOut o = hits_out(out);
    return query_host(h, &i, n, &o, stats);
  });
}

int rtb200_scene_occluded_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, uint8_t* occluded, void* stream_in) {
  return guarded([&]() -> int {
    const QueryIn i = rays_in(rays);
    const QueryOut o = occluded_out(occluded);
    return query_device(h, &i, n, &o, stream_in);
  });
}

int rtb200_scene_occluded(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, uint8_t* occluded, rt_stats* stats) {
  return guarded([&]() -> int {
    const QueryIn i = rays_in(rays);
    const QueryOut o = occluded_out(occluded);
    return query_host(h, &i, n, &o, stats);
  });
}

int rtb200_scene_nearest_device(rtb200_scene_handle h, const rt_points* q, uint32_t n, const rt_nearest* out, void* stream_in) {
  return guarded([&]() -> int {
    const QueryIn i = points_in(q);
    const QueryOut o = nearest_out(out);
    return query_device(h, &i, n, &o, stream_in);
  });
}

int rtb200_scene_nearest(rtb200_scene_handle h, const rt_points* q, uint32_t n, const rt_nearest* out, rt_stats* stats) {
  return guarded([&]() -> int {
    const QueryIn i = points_in(q);
    const QueryOut o = nearest_out(out);
    return query_host(h, &i, n, &o, stats);
  });
}

int rtb200_scene_overlaps_device(rtb200_scene_handle h, const rt_points* q, uint32_t n, uint8_t* overlaps, void* stream_in) {
  return guarded([&]() -> int {
    const QueryIn i = points_in(q);
    const QueryOut o = overlaps_out(overlaps);
    return query_device(h, &i, n, &o, stream_in);
  });
}

int rtb200_scene_overlaps(rtb200_scene_handle h, const rt_points* q, uint32_t n, uint8_t* overlaps, rt_stats* stats) {
  return guarded([&]() -> int {
    const QueryIn i = points_in(q);
    const QueryOut o = overlaps_out(overlaps);
    return query_host(h, &i, n, &o, stats);
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
