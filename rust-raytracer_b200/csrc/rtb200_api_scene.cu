// rtb200_api_scene.cu — the calls of the C ABI that write a resident scene: moving its spheres (refit, DESIGN.md §4.7),
// rebuilding its hierarchy (§4.8) and inserting and removing spheres (§4.13). Each one orders its stream after the scene's
// last writer and after the frames and queries in flight, and every frame enqueued later waits for it.

#include "rtb200_host.cuh"

using namespace rtk;

// The refit's scratch, built at the first update of a MODE_TREE handle on the update's stream `st`: exact boxes of the nodes
// and leaves, and the device copy of the builder's level order (an update never changes the topology).
static int refit_prepare(rtb200_scene_handle h, cudaStream_t st) {
    const uint32_t nn = h->tp.n_nodes, nl = h->tp.n_leaves;
    if (h->node_box || h->mode != MODE_TREE || nn == 0) return RT_OK;   // a rebuild brings its own scratch
    Carver c;
    const size_t node_off = c.offset((size_t)nn * 6 * sizeof(double)), leaf_off = c.offset((size_t)nl * 6 * sizeof(double)),
                 level_off = c.offset((size_t)nn * 4);
    char* p = nullptr;
    CU(cudaMalloc(&p, c.off));
    uint32_t* level_nodes = (uint32_t*)(p + level_off);
    const cudaError_t e = cudaMemcpyAsync(level_nodes, h->level_nodes.data(), (size_t)nn * 4, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { cudaFree(p); return fail_cuda(e, "cudaMemcpyAsync(level order)"); }
    // node_box marks the handle as prepared: set only once the level order is on its way
    h->refit = p; h->node_box = (double*)(p + node_off); h->leaf_box = (double*)(p + leaf_off); h->level_nodes_dev = level_nodes;
    return RT_OK;
}

// The start of a call that writes h's scene arrays, on `stream_in`: *st is ordered after the scene's last writer
// (scene_stream), and h->updated, which every later frame waits for, exists from here on.
static cudaError_t writer_begin(rtb200_scene_handle h, void* stream_in, cudaStream_t* st) {
    cudaError_t e = scene_stream(h, stream_in, st);
    if (e == cudaSuccess && !h->updated) e = cudaEventCreateWithFlags(&h->updated, cudaEventDisableTiming);
    return e;
}

// Order `st` after the frames and the queries of h in flight, on any stream: they read the arrays the update writes. Every
// later update or rebuild waits for this one (h->updated, scene_stream), so the queries waited for here are forgotten.
static int update_after_frames(rtb200_scene_handle h, cudaStream_t st) {
    for (const auto& p : h->pending) if (p.n_ev) CU(cudaStreamWaitEvent(st, h->ev[p.ev0 + 1], 0));
    for (uint32_t k = 0; k < h->n_queries; ++k) CU(cudaStreamWaitEvent(st, h->queries[k].done, 0));
    h->n_queries = 0;
    return RT_OK;
}

// Words of a writer's input at byte `off` of the staged block
struct StagedWords { const void* src; size_t off, bytes; };

// The input of a writer on st, in the pinned staging buffer and copied before this returns: the exact geo and the materials
// of the n spheres `sp` at geo_off and mat_off, and `words`. Bytes [0, in_bytes) go to h->upd_in, the tail_bytes after them to
// tail_dst. The copy is enqueued before the wait for the frames pending now (update_after_frames; DESIGN.md §4.7, Ordering).
// *nonfinite: a sphere has a non-finite albedo.
static int stage_input(rtb200_scene_handle h, cudaStream_t st, const rt_sphere* sp, uint32_t n, size_t geo_off, size_t mat_off,
                       std::initializer_list<StagedWords> words, size_t in_bytes, void* tail_dst, size_t tail_bytes, bool* nonfinite) {
    DeviceCtx* ctx = h->ctx;
    CU(cudaEventSynchronize(ctx->staging_free));   // the previous copy has left the staging buffer
    CU(ctx->staging.ensure(in_bytes + tail_bytes));
    char* S = (char*)ctx->staging.p;
    *nonfinite = false;
    for (uint32_t k = 0; k < n; ++k) {
        rtbvh::sphere_exact(sp[k], (double*)(S + geo_off) + 4 * (size_t)k, ((rtbvh::Mat32*)(S + mat_off))[k]);
        *nonfinite = *nonfinite || albedo_nonfinite(sp[k]);
    }
    for (const StagedWords& w : words) memcpy(S + w.off, w.src, w.bytes);
    CU(cudaMemcpyAsync(h->upd_in.p, S, in_bytes, cudaMemcpyHostToDevice, st));
    if (tail_bytes) CU(cudaMemcpyAsync(tail_dst, S + in_bytes, tail_bytes, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(ctx->staging_free, st));
    return update_after_frames(h, st);
}

// Enqueue the refit of the tree p describes: its leaf records and boxes, then one pass per level of the level order
// `level_nodes` (device) with level k at [level_off[k], level_off[k + 1]), deepest first.
static cudaError_t refit_tree(const RefitParams& p, const uint32_t* level_nodes, const std::vector<uint32_t>& level_off, cudaStream_t st) {
    cudaError_t e = launch_refit_spheres(p, st);
    for (size_t k = 0; e == cudaSuccess && k + 1 < level_off.size(); ++k)
        e = launch_refit_nodes(p, level_nodes + level_off[k], level_off[k + 1] - level_off[k], st);
    return e;
}

// Recompute the arrays of h's mode from its geo and record the end of the update: every frame enqueued later waits for it.
static int update_finish(rtb200_scene_handle h, cudaStream_t st) {
    RefitParams p{};
    p.geo = h->tp.geo; p.n = h->tp.n; p.g[0] = h->tp.gx; p.g[1] = h->tp.gy; p.g[2] = h->tp.gz;
    if (h->mode == MODE_BRUTE) {
        p.filt = (float*)h->tp.filt;
        CU(launch_refit_spheres(p, st));
    } else if (h->mode == MODE_TREE && h->node_box) {
        p.leaf_id = h->tp.leaf_id; p.leaf_rec = (float*)h->tp.leaf_rec; p.leaf_box = h->leaf_box; p.n_leaves = h->tp.n_leaves;
        p.nodes = (float*)h->tp.nodes; p.node_box = h->node_box;
        CU(refit_tree(p, h->level_nodes_dev, h->level_off, st));
    }
    CU(cudaEventRecord(h->updated, st));
    return RT_OK;
}

// The checks of one sphere a resident scene takes, sphere k of the caller's array `what` (updates and edits): a known kind, and
// a Texture index of an uploaded texture whose image was not empty.
static int check_sphere(rtb200_scene_handle h, const rt_sphere& sp, const char* what, uint32_t k) {
    if (sp.kind > RT_LIGHT) return fail(RT_ERR_INVALID, "unknown material kind (" + std::string(what) + "[" + std::to_string(k) + "])");
    if (sp.kind == RT_TEXTURE && (sp.texture < 0 || (size_t)sp.texture >= h->tex_ok.size() || !h->tex_ok[sp.texture]))
        return fail(RT_ERR_INVALID, "texture index out of range, or its image was empty at upload (" + std::string(what) + "[" + std::to_string(k) + "])");
    return RT_OK;
}

// The n sphere indices `index` sorted into *out, or a refusal when one is not a sphere of h or one repeats. The refusals name
// an index `name` and end a repeat's text with `twice`.
static int sorted_indices(rtb200_scene_handle h, const uint32_t* index, uint32_t n, const char* name, const char* twice,
                          std::vector<uint32_t>* out) {
    std::vector<uint32_t>& v = *out;
    v.assign(index, index + n);
    std::sort(v.begin(), v.end());
    if (n && v.back() >= h->tp.n)
        return fail(RT_ERR_INVALID, std::string(name) + " " + std::to_string(v.back()) + " is not a sphere of the scene (n_spheres = " + std::to_string(h->tp.n) + ")");
    for (uint32_t k = 1; k < n; ++k)
        if (v[k] == v[k - 1]) return fail(RT_ERR_INVALID, "sphere " + std::to_string(v[k]) + " is listed twice" + twice);
    return RT_OK;
}

int rtb200_scene_update_spheres(rtb200_scene_handle h, const uint32_t* index, const rt_sphere* spheres, uint32_t n, void* stream_in) {
  return guarded([&]() -> int {
    if (n && (!index || !spheres)) return fail(RT_ERR_INVALID, "index or spheres is null");
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (n == 0) return RT_OK;
    // everything is checked before anything is enqueued: on error the scene is unchanged
    std::vector<uint32_t> sorted;
    int rc = sorted_indices(h, index, n, "index", "", &sorted);
    if (rc != RT_OK) return rc;
    for (uint32_t k = 0; k < n; ++k) {
        const rt_sphere& sp = spheres[k];
        if ((rc = check_sphere(h, sp, "spheres", k)) != RT_OK) return rc;
        const bool was_light = std::binary_search(h->light_idx.begin(), h->light_idx.end(), index[k]);
        if (was_light != (sp.kind == RT_LIGHT))
            return fail(RT_ERR_UNSUPPORTED, "sphere " + std::to_string(index[k]) + ": the set of lights is fixed at upload (upload the scene again to change it)");
    }
    HANDLE_PROLOGUE(h);
    // the input (geo, materials, indices), after the last update, which read it
    const size_t geo_b = (size_t)n * 32, mat_b = (size_t)n * sizeof(DevMat), bytes = geo_b + mat_b + (size_t)n * 4;
    CU(h->upd_in.ensure(bytes, h->updated));
    ++h->updates;
    cudaStream_t st;
    CU(writer_begin(h, stream_in, &st));
    if ((rc = refit_prepare(h, st)) != RT_OK) return rc;
    bool nonfinite = false;
    if ((rc = stage_input(h, st, spheres, n, 0, geo_b, {{index, geo_b + mat_b, (size_t)n * 4}}, bytes, nullptr, 0, &nonfinite)) != RT_OK)
        return rc;
    // never cleared: the flag only selects the exact slow path, and frames already enqueued copied the old value
    if (nonfinite) h->tp.albedo_nonfinite = 1u;
    const char* D = (const char*)h->upd_in.p;
    CU(launch_update_scatter((const uint32_t*)(D + geo_b + mat_b), (const double4*)D, (const DevMat*)(D + geo_b), n,
                             (double4*)h->tp.geo, (DevMat*)h->tp.mat, st));
    return update_finish(h, st);
  });
}

int rtb200_scene_update_geometry_device(rtb200_scene_handle h, const void* dev_center_radius, void* stream_in) {
  return guarded([&]() -> int {
    if (!dev_center_radius) return fail(RT_ERR_INVALID, "dev_center_radius is null");
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    HANDLE_PROLOGUE(h);
    int rc = check_device_ptrs(h, {{dev_center_radius, "dev_center_radius"}});
    if (rc != RT_OK) return rc;
    if (h->tp.n == 0) return RT_OK;
    ++h->updates;
    cudaStream_t st;
    CU(writer_begin(h, stream_in, &st));
    if ((rc = refit_prepare(h, st)) == RT_OK) rc = update_after_frames(h, st);
    if (rc != RT_OK) return rc;
    CU(cudaMemcpyAsync((void*)h->tp.geo, dev_center_radius, (size_t)h->tp.n * 32, cudaMemcpyDeviceToDevice, st));
    return update_finish(h, st);
  });
}

// ---- rebuilding the hierarchy of a resident scene on the GPU (DESIGN.md §4.8) ----
// A device allocation a call makes before it enqueues anything, freed on return unless the call took it over (take).
struct FreshBlock {
    void* p = nullptr;
    uint32_t cap = 0;                    // spheres it is carved for
    ~FreshBlock() { if (p) cudaFree(p); }
    void* take() { void* q = p; p = nullptr; return q; }
};

// The rebuild block a hierarchy of n spheres needs: h->rebuild when it holds them, else a new block in *fresh, which
// rebuild_tree installs (frames in flight may still read the old one). The first block holds n spheres; a block that has to
// grow for an edit takes half as much again, so that a run of appends does not allocate on every call.
static int rebuild_reserve(rtb200_scene_handle h, uint32_t n, FreshBlock* fresh) {
    if (h->rebuild && n <= h->rebuild_n) return RT_OK;
    const uint32_t cap = h->rebuild ? (uint32_t)std::min<uint64_t>(std::max<uint64_t>(n, (uint64_t)h->rebuild_n * 3 / 2), (1u << 26) - 1) : n;
    const size_t bytes = rebuild_carve(nullptr, cap, nullptr);
    const cudaError_t e = cudaMalloc(&fresh->p, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        fresh->p = nullptr;
        return fail(RT_ERR_OOM, "rebuild: cannot allocate " + std::to_string(bytes) + " bytes of device memory for " + std::to_string(cap) + " spheres");
    }
    fresh->cap = cap;
    return RT_OK;
}

// A new hierarchy over tp.geo[0, n), n > 0, enqueued on st, which the caller has ordered after h's last writer and after the
// frames and queries of h in flight (update_after_frames), and installed in tp. The topology comes from rtb200_rebuild.cu, its
// values from the refit's kernels; the host reads back one header (counts, depth, level sizes, recentring offset) between the
// two, so st has passed those frames when this returns. The arrays live in the rebuild block (`fresh` when rebuild_reserve
// made one; the old block is freed once st has passed the frames that may read it).
static int rebuild_tree(rtb200_scene_handle h, uint32_t n, FreshBlock& fresh, cudaStream_t st) {
    RebuildBufs b;
    rebuild_carve(fresh.p ? fresh.p : h->rebuild, fresh.p ? fresh.cap : h->rebuild_n, &b);
    const char* ov = getenv("RTB200_REBUILD_OVERSIZE");   // benchmark hook: 0 keeps oversized spheres in the Morton order
    CU(launch_rebuild_topology(b, h->tp.geo, n, ov ? atof(ov) : kRebuildOversize, st));
    RebuildHeader H;
    CU(cudaMemcpyAsync(&H, b.header, sizeof H, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (H.overflow || H.depth > (uint32_t)rtbvh::kMaxDepth)   // unreachable by the depth bound (DESIGN.md §4.8)
        return fail(RT_ERR_CUDA, "internal error: the rebuilt hierarchy is deeper than the traversal stack reserve");
    // the level order, deepest level first (Records::level_off)
    std::vector<uint32_t> level_off(1, 0u);
    for (uint32_t k = H.depth; k-- > 0;) level_off.push_back(level_off.back() + H.level_count[k]);
    RefitParams p{};
    p.geo = h->tp.geo; p.n = n; p.g[0] = H.g[0]; p.g[1] = H.g[1]; p.g[2] = H.g[2];
    p.leaf_id = b.leaf_id; p.leaf_rec = b.leaf_rec; p.leaf_box = b.leaf_box; p.n_leaves = H.n_leaves;
    p.nodes = b.nodes; p.node_box = b.node_box;
    CU(refit_tree(p, b.level_nodes, level_off, st));
    CU(cudaEventRecord(h->updated, st));
    // every frame enqueued from here on traces the new tree, and every update refits it
    if (h->refit) { CU(cudaFree(h->refit)); h->refit = nullptr; }   // the stream synchronisation above covers the updates that used it
    if (fresh.p) {
        if (h->rebuild) CU(cudaFree(h->rebuild));   // and the frames that read the old block
        h->rebuild_n = fresh.cap;
        h->rebuild = fresh.take();
    }
    TraceParams& tp = h->tp;
    tp.nodes = (const float4*)b.nodes; tp.leaf_rec = (const float4*)b.leaf_rec; tp.leaf_id = b.leaf_id;
    tp.skip_pos = b.skip_pos; tp.always = b.always;
    tp.n_nodes = H.n_nodes; tp.n_leaves = H.n_leaves; tp.n_always = H.n_always; tp.depth = H.depth;
    tp.gx = H.g[0]; tp.gy = H.g[1]; tp.gz = H.g[2];
    h->level_off = level_off;
    h->level_nodes.clear();
    h->node_box = b.node_box; h->leaf_box = b.leaf_box; h->level_nodes_dev = b.level_nodes;
    return RT_OK;
}

int rtb200_scene_rebuild(rtb200_scene_handle h, void* stream_in) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (h->mode != MODE_TREE || h->tp.n == 0) return RT_OK;   // no hierarchy to rebuild
    if (h->tp.scene_in_smem & 1u)
        return fail(RT_ERR_UNSUPPORTED, "the handle stages its hierarchy in shared memory (RTB200_WF_SMEM bit 0), whose launch layout is fixed at upload");
    HANDLE_PROLOGUE(h);
    FreshBlock fresh;
    int rc = rebuild_reserve(h, h->tp.n, &fresh);
    if (rc != RT_OK) return rc;
    cudaStream_t st;   // the spheres stay as they are: an adaptive render may step across a rebuild
    CU(writer_begin(h, stream_in, &st));
    if ((rc = update_after_frames(h, st)) != RT_OK) return rc;
    return rebuild_tree(h, h->tp.n, fresh, st);
  });
}

// ---- inserting and removing spheres of a resident scene (DESIGN.md §4.13) ----
// The edit block of `cap` spheres carved out of `base` (null: only the size); returns the bytes. `flat`: the halves carry flat
// records (MODE_BRUTE).
static size_t edit_carve(void* base, uint32_t cap, bool flat, rtb200_scene_t::EditBlock* out) {
    Carver c(base);
    rtb200_scene_t::EditBlock b;
    b.mem = base; b.cap = cap;
    for (auto& H : b.half) {
        H.geo = (double4*)c.take((size_t)cap * 32);
        H.mat = (DevMat*)c.take((size_t)cap * sizeof(DevMat));
        H.filt = flat ? (float*)c.take((size_t)rtbvh::flat_pairs(cap) * 32) : nullptr;
        H.lights = (uint32_t*)c.take(16 * 4);   // at most 9 lights and the trailing 0 of the upload's list
    }
    b.skip_pos = (uint32_t*)c.take((size_t)cap * 4);
    b.keep = (uint32_t*)c.take(((size_t)cap + 1) * 4);
    b.pos = (uint32_t*)c.take(((size_t)cap + 1) * 4);
    b.temp_bytes = edit_scan_bytes(cap);
    b.temp = c.take(b.temp_bytes);
    if (out) *out = b;
    return c.off;
}

int rtb200_scene_edit_spheres(rtb200_scene_handle h, const uint32_t* remove, uint32_t n_remove, const uint32_t* at,
                                         const rt_sphere* insert, uint32_t n_insert, void* stream_in) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (n_remove && !remove) return fail(RT_ERR_INVALID, "remove is null");
    if (n_insert && !insert) return fail(RT_ERR_INVALID, "insert is null");
    if (n_remove == 0 && n_insert == 0) return RT_OK;
    // everything is checked before anything is enqueued: on error the scene is unchanged
    const uint32_t n_old = h->tp.n;
    std::vector<uint32_t> rem;
    int rc = sorted_indices(h, remove, n_remove, "remove index", " in remove", &rem);
    if (rc != RT_OK) return rc;
    std::vector<uint32_t> at_v(n_insert, n_old);   // at == NULL: every insert is appended
    for (uint32_t k = 0; k < n_insert; ++k) {
        if (at) {
            if (at[k] > n_old) return fail(RT_ERR_INVALID, "at[" + std::to_string(k) + "] = " + std::to_string(at[k]) + " exceeds n_spheres = " + std::to_string(n_old));
            if (k && at[k] < at[k - 1]) return fail(RT_ERR_INVALID, "at decreases at at[" + std::to_string(k) + "]");
            at_v[k] = at[k];
        }
        if ((rc = check_sphere(h, insert[k], "insert", k)) != RT_OK) return rc;
    }
    const uint64_t n_new64 = (uint64_t)n_old - n_remove + n_insert;
    if (n_new64 >= (1ull << 26)) return fail(RT_ERR_UNSUPPORTED, kErrSpheres);
    const uint32_t n_new = (uint32_t)n_new64;
    // the lights in the new list order: a kept old sphere i goes to kept(< i) + #{k : at[k] <= i}, insert k to kept(< at[k]) + k
    auto kept_below = [&](uint32_t j) { return j - (uint32_t)(std::lower_bound(rem.begin(), rem.end(), j) - rem.begin()); };
    std::vector<uint32_t> lights;
    for (uint32_t i : h->light_idx)
        if (!std::binary_search(rem.begin(), rem.end(), i))
            lights.push_back(kept_below(i) + (uint32_t)(std::upper_bound(at_v.begin(), at_v.end(), i) - at_v.begin()));
    for (uint32_t k = 0; k < n_insert; ++k)
        if (insert[k].kind == RT_LIGHT) lights.push_back(kept_below(at_v[k]) + k);
    std::sort(lights.begin(), lights.end());
    if (lights.size() >= 10) return fail(RT_ERR_UNSUPPORTED, kErrLights);
    if (h->tp.scene_in_smem)
        return fail(RT_ERR_UNSUPPORTED, "the handle stages the scene in shared memory (RTB200_WF_SMEM), whose launch layout is fixed at upload");

    HANDLE_PROLOGUE(h);
    TraceParams& tp = h->tp;
    // the single-frame kernel is another template with lights than without: its launch geometry follows n_lights > 0
    LaunchGeom g;
    if ((rc = launch_geometry(h, Q_SINGLE, !lights.empty(), &g)) != RT_OK) return rc;
    // device memory before anything is enqueued: a larger edit block, the rebuild block, the input
    const uint32_t need = std::max(std::max(n_old, n_new), 1u);
    FreshBlock fresh_ed, fresh_rb;
    rtb200_scene_t::EditBlock E = h->ed;
    if (need > E.cap) {   // grows geometrically: a run of single appends allocates once in a while, not on every call
        const uint32_t cap = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(std::max<uint64_t>(need + need / 2, 2ull * E.cap), 64), 1u << 26);
        const size_t bytes = edit_carve(nullptr, cap, h->mode == MODE_BRUTE, nullptr);
        if (cudaMalloc(&fresh_ed.p, bytes) != cudaSuccess) {
            cudaGetLastError();
            fresh_ed.p = nullptr;
            return fail(RT_ERR_OOM, "edit: cannot allocate " + std::to_string(bytes) + " bytes of device memory for " + std::to_string(cap) + " spheres");
        }
        edit_carve(fresh_ed.p, cap, h->mode == MODE_BRUTE, &E);
    }
    if (h->mode == MODE_TREE && n_new > 0 && (rc = rebuild_reserve(h, n_new, &fresh_rb)) != RT_OK) return rc;
    Carver in;   // the input: remove, at, the inserts' geo and materials; then the light list
    in.offset((size_t)n_remove * 4);
    const size_t at_off = in.offset((size_t)n_insert * 4), geo_off = in.offset((size_t)n_insert * 32),
                 mat_off = in.offset((size_t)n_insert * sizeof(DevMat)), in_bytes = in.off;
    CU(h->upd_in.ensure(in_bytes, h->updated));   // after the last update, which read it
    const int tgt = fresh_ed.p || h->ed_cur != 0 ? 0 : 1;   // the half that does not hold the current list
    const auto& T = E.half[tgt];

    ++h->updates;
    cudaStream_t st;   // after the previous update or edit too: it may still read upd_in and the target half
    CU(writer_begin(h, stream_in, &st));
    lights.push_back(0);
    bool nonfinite = false;
    if ((rc = stage_input(h, st, insert, n_insert, geo_off, mat_off,
                          {{rem.data(), 0, (size_t)n_remove * 4}, {at_v.data(), at_off, (size_t)n_insert * 4}, {lights.data(), in_bytes, lights.size() * 4}},
                          in_bytes, T.lights, lights.size() * 4, &nonfinite)) != RT_OK)
        return rc;
    if (fresh_ed.p) CU(cudaMemsetAsync(E.skip_pos, 0xff, (size_t)E.cap * 4, st));   // rtbvh::kNoSkip
    const char* D = (const char*)h->upd_in.p;
    EditParams p{};
    p.geo_old = tp.geo; p.mat_old = tp.mat; p.n_old = n_old;
    p.remove = (const uint32_t*)D; p.n_remove = n_remove;
    p.at = (const uint32_t*)(D + at_off); p.geo_in = (const double4*)(D + geo_off); p.mat_in = (const DevMat*)(D + mat_off); p.n_insert = n_insert;
    p.keep = E.keep; p.pos = E.pos; p.temp = E.temp; p.temp_bytes = E.temp_bytes;
    p.geo = T.geo; p.mat = T.mat;
    p.filt = T.filt; p.n_pairs = rtbvh::flat_pairs(n_new);
    CU(launch_edit_spheres(p, st));

    // every frame, query, update and rebuild enqueued from here on sees the new list
    void* retired = fresh_ed.p ? h->ed.mem : nullptr;   // freed once st has passed the frames that may read it
    if (fresh_ed.p) { h->ed = E; fresh_ed.take(); }
    h->ed_cur = tgt;
    lights.pop_back();
    tp.n = n_new; tp.n_pairs = p.n_pairs;
    tp.geo = T.geo; tp.mat = T.mat; tp.lights = T.lights; tp.n_lights = (uint32_t)lights.size();
    if (nonfinite) tp.albedo_nonfinite = 1u;   // never cleared, as in an update
    if (h->mode == MODE_BRUTE) tp.filt = (const float4*)T.filt;
    if (h->mode != MODE_TREE || n_new == 0) tp.skip_pos = E.skip_pos;
    h->light_idx = lights;
    h->ctas_per_sm = g.ctas_per_sm;
    h->grid = g.grid;
    if (h->mode == MODE_TREE && n_new > 0) {
        if ((rc = rebuild_tree(h, n_new, fresh_rb, st)) != RT_OK) return rc;   // returns when st has passed the frames
    } else {
        if (h->mode == MODE_TREE) {   // no spheres: the hierarchy of an empty upload
            tp.n_nodes = tp.n_leaves = tp.n_always = tp.depth = 0;
            tp.gx = tp.gy = tp.gz = 0.0;
            h->level_off.clear(); h->level_nodes.clear();
            h->node_box = h->leaf_box = nullptr; h->level_nodes_dev = nullptr;
        }
        if ((rc = update_finish(h, st)) != RT_OK) return rc;   // MODE_BRUTE: the flat records at the handle's recentring offset
        CU(cudaStreamSynchronize(st));
        if (h->refit) { CU(cudaFree(h->refit)); h->refit = nullptr; }
    }
    if (retired) CU(cudaFree(retired));
    return RT_OK;
  });
}
