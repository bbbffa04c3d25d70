// rtb200_api.cu — the C ABI of include/rtb200.h: error reporting, the per-device contexts, scene staging into HBM, the
// handle's diagnostics and the device probes. Rendering is in rtb200_api_render.cu, scene writes in rtb200_api_scene.cu and
// queries in rtb200_api_query.cu; rtb200_host.cuh is what they share. No CPU render path exists here.

#include "rtb200_host.cuh"

using namespace rtk;

static_assert(kCapIn >= 32 + 7 * rtbvh::kMaxDepth + 8, "the node stack must hold 32 roots plus a single-entry descent of the deepest tree (LIFO reserve, DESIGN.md 4.1)");

thread_local std::string rtk::g_last_error;

int rtk::fail(int code, const std::string& msg) { g_last_error = msg; return code; }
int rtk::fail_cuda(cudaError_t e, const char* what) {
    g_last_error = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? RT_ERR_NO_DEVICE
           : (e == cudaErrorMemoryAllocation ? RT_ERR_OOM : RT_ERR_CUDA);
}

static DeviceCtx g_ctx[64];
static std::mutex g_ctx_mu;

int rtk::get_ctx(int device, DeviceCtx** out) {
    if (device < 0) {
        cudaError_t e = cudaGetDevice(&device);
        if (e != cudaSuccess) return fail_cuda(e, "cudaGetDevice");
    }
    if (device >= 64) return fail(RT_ERR_INVALID, "device ordinal out of range");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess) return fail_cuda(e, "cudaGetDeviceCount");
    if (device >= count) return fail(RT_ERR_NO_DEVICE, "no such CUDA device");
    CU(cudaSetDevice(device));
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    DeviceCtx& c = g_ctx[device];
    if (!c.init) {
        cudaDeviceProp prop;
        CU(cudaGetDeviceProperties(&prop, device));
        if (prop.major != 9 || prop.minor != 0) {
            char buf[160];
            snprintf(buf, sizeof buf, "device %d is sm_%d%d; this library carries sm_90a code only", device, prop.major, prop.minor);
            return fail(RT_ERR_NO_DEVICE, buf);
        }
        c.device = device;
        c.sm_count = prop.multiProcessorCount;
        CU(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
        CU(cudaEventCreateWithFlags(&c.staging_free, cudaEventDisableTiming));
        for (auto& W : c.ws) CU(cudaEventCreateWithFlags(&W.done, cudaEventDisableTiming));
        c.init = true;
    }
    *out = &c;
    return RT_OK;
}

uint32_t rtk::mode_of(uint32_t variant) {
    return variant == RT_VARIANT_EXACT_F64 ? MODE_EXACT : (variant == RT_VARIANT_BRUTE_FORCE ? MODE_BRUTE : MODE_TREE);
}

uint32_t rtk::samples_per_batch(uint64_t cap, uint64_t items, uint32_t samples) {
    uint64_t spb = std::max<uint64_t>(1, cap / (std::max<uint64_t>(items, 1) * 16ull));
    spb = std::min<uint64_t>(spb, samples);
    while (spb > 1 && spb * items >= (1ull << 31)) spb /= 2;
    return (uint32_t)spb;
}

cudaError_t rtk::scene_stream(rtb200_scene_handle h, void* stream_in, cudaStream_t* out) {
    const cudaStream_t st = call_stream(h->ctx, stream_in);
    *out = st;
    if (st != h->ctx->stream) { cudaError_t e = cudaStreamWaitEvent(st, h->ctx->staging_free, 0); if (e != cudaSuccess) return e; }
    return h->updated ? cudaStreamWaitEvent(st, h->updated, 0) : cudaSuccess;
}

int rtk::check_device_ptrs(int device, const std::vector<std::pair<const void*, const char*>>& ptrs) {
    for (const auto& q : ptrs) {
        if (!q.first) continue;
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, q.first) != cudaSuccess) { cudaGetLastError(); a.type = cudaMemoryTypeUnregistered; }
        if (!((a.type == cudaMemoryTypeDevice && a.device == device) || a.type == cudaMemoryTypeManaged))
            return fail(RT_ERR_INVALID, std::string(q.second) + " is not device or managed memory of device " + std::to_string(device));
    }
    return RT_OK;
}
int rtk::check_device_ptrs(rtb200_scene_handle h, const std::vector<std::pair<const void*, const char*>>& ptrs) {
    return check_device_ptrs(h->device, ptrs);
}

struct V3 { double x, y, z; };
static inline V3 v3(const rt_vec3& a) { return V3{a.x, a.y, a.z}; }
static inline V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
static inline V3 operator*(V3 a, double s) { return V3{a.x * s, a.y * s, a.z * s}; }
static inline double vlen(V3 a) { return std::sqrt(a.x * a.x + a.y * a.y + a.z * a.z); }
static inline V3 vunit(V3 a) { double l = vlen(a); return V3{a.x / l, a.y / l, a.z / l}; }
static inline V3 vcross(V3 a, V3 b) { return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
static inline rt_vec3 rv(V3 a) { return rt_vec3{a.x, a.y, a.z}; }

int rtb200_abi_version(void) { return RTB200_ABI_VERSION; }
const char* rtb200_last_error(void) { return g_last_error.c_str(); }

int rtb200_device_count(void) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) { cudaGetLastError(); return 0; }
    return count;
}

// Camera::new — camera.rs:45-77. Host, once per frame, f64, same operation order as the reference.
// (Compiled with -ffp-contract=off: see the Makefile.)
int rtb200_camera_from_params(const rt_camera_params* p, rt_camera* out) {
    if (!p || !out) return fail(RT_ERR_INVALID, "null argument");
    const double PI = 3.14159265358979323846264338327950288;
    double theta = p->vfov_deg * (PI / 180.0);
    double half_height = std::tan(theta / 2.0);
    double half_width = p->aspect * half_height;
    V3 look_from = v3(p->look_from), look_at = v3(p->look_at), vup = v3(p->vup);
    V3 w = vunit(look_from - look_at);
    V3 u = vunit(vcross(vup, w));
    V3 v = vcross(w, u);
    V3 origin = look_from;
    V3 llc = origin - (u * half_width) - (v * half_height) - w;
    V3 horizontal = u * 2.0 * half_width;
    V3 vertical = v * 2.0 * half_height;
    out->origin = rv(origin); out->lower_left_corner = rv(llc); out->horizontal = rv(horizontal); out->vertical = rv(vertical);
    return RT_OK;
}

// The thin-lens camera (include/rtb200.h, DESIGN.md §4.17): Camera::new's basis, then the image plane at focus_dist.
int rtb200_camera_from_params_lens(const rt_camera_params* p, double aperture, double focus_dist, rt_camera* out, rt_lens* lens) {
    if (!p || !out || !lens) return fail(RT_ERR_INVALID, "null argument");
    if (!std::isfinite(aperture) || aperture < 0.0) return fail(RT_ERR_INVALID, "aperture must be finite and >= 0");
    if (!std::isfinite(focus_dist) || !(focus_dist > 0.0)) return fail(RT_ERR_INVALID, "focus_dist must be finite and > 0");
    const double PI = 3.14159265358979323846264338327950288, fd = focus_dist;
    double theta = p->vfov_deg * (PI / 180.0);
    double half_height = std::tan(theta / 2.0);
    double half_width = p->aspect * half_height;
    V3 look_from = v3(p->look_from), look_at = v3(p->look_at), vup = v3(p->vup);
    V3 w = vunit(look_from - look_at);
    V3 u = vunit(vcross(vup, w));
    V3 v = vcross(w, u);
    V3 origin = look_from;
    V3 llc = origin - (u * (half_width * fd)) - (v * (half_height * fd)) - w * fd;
    V3 horizontal = u * 2.0 * half_width * fd;
    V3 vertical = v * 2.0 * half_height * fd;
    out->origin = rv(origin); out->lower_left_corner = rv(llc); out->horizontal = rv(horizontal); out->vertical = rv(vertical);
    *lens = rt_lens{rv(u), rv(v), aperture / 2.0, 0};
    return RT_OK;
}

int rtk::check_lens(const rt_lens& L, const char* what) {
    const double f[7] = {L.u.x, L.u.y, L.u.z, L.v.x, L.v.y, L.v.z, L.radius};
    for (double x : f) if (!std::isfinite(x)) return fail(RT_ERR_INVALID, std::string(what) + ": u, v and radius must be finite");
    if (L.radius < 0.0) return fail(RT_ERR_INVALID, std::string(what) + ": radius must be >= 0");
    if (L.reserved != 0) return fail(RT_ERR_INVALID, std::string(what) + ": reserved must be 0");
    return RT_OK;
}

int rtb200_scene_set_lens(rtb200_scene_handle h, const rt_lens* lens) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    const rt_lens L = lens ? *lens : rt_lens{};
    int rc = check_lens(L, "lens");
    if (rc != RT_OK) return rc;
    HANDLE_PROLOGUE(h);
    if (L.radius == 0.0) h->tp.lens = rt_lens{};   // one pinhole: the lens of a fresh upload
    else h->tp.lens = L;
    ++h->updates;   // an adaptive render's sums would mix two cameras
    return RT_OK;
  });
}

uint32_t rtb200_shard_rows(uint32_t height, int32_t rank, int32_t world, uint32_t band_rows) {
    if (world <= 1) return height;
    if (band_rows == 0) band_rows = 1;
    const uint64_t bands = ((uint64_t)height + band_rows - 1) / band_rows;   // last band may be partial
    if ((uint64_t)rank >= bands) return 0;
    const uint64_t mine = (bands - 1 - (uint64_t)rank) / (uint64_t)world + 1;   // bands rank, rank+world, ...
    uint64_t rows = mine * band_rows;
    const uint64_t last = bands - 1;
    if (last % (uint64_t)world == (uint64_t)rank) rows -= bands * band_rows - height;   // the partial band is ours
    return (uint32_t)rows;
}

// info[8] of the diagnostics below
static void bvh_info(uint32_t info[8], uint32_t n_nodes, uint32_t n_leaves, uint32_t depth, uint32_t n_always, uint32_t n_pairs) {
    const uint32_t v[8] = {n_nodes, n_leaves, depth, (uint32_t)rtbvh::kLeafK, n_always, (uint32_t)rtbvh::kNodeFloats, n_pairs, 0u};
    memcpy(info, v, sizeof v);
}

// Diagnostic (host only, no GPU needed): the hierarchy rtb200_scene_upload would stage for `scene`.
// info = {n_nodes, n_leaves, depth, leaf_size, n_always, floats_per_node, n_pairs_flat, 0}; arrays are filled up to their capacities (elements).
int rtb200_debug_bvh(const rt_scene* s, double recentre[3], uint32_t info[8], float* nodes, uint64_t cap_nodes, float* leaf_rec,
                     uint64_t cap_leaf_rec, uint32_t* leaf_id, uint64_t cap_leaf_id, uint32_t* always, uint64_t cap_always,
                     float* flat, uint64_t cap_flat) {
  return guarded([&]() -> int {
    if (!s || !info) return fail(RT_ERR_INVALID, "null argument");
    if (s->n_spheres >= (1ull << 26)) return fail(RT_ERR_UNSUPPORTED, kErrSpheres);
    if (s->n_spheres && !s->spheres) return fail(RT_ERR_INVALID, "spheres is null");
    rtbvh::Records R;
    rtbvh::build_records(s, true, R);
    if (recentre) { recentre[0] = R.g[0]; recentre[1] = R.g[1]; recentre[2] = R.g[2]; }
    bvh_info(info, R.n_nodes, R.n_leaves, R.depth, (uint32_t)R.always.size(), R.n_pairs);
    if (nodes) memcpy(nodes, R.nodes.data(), std::min<uint64_t>(cap_nodes, R.nodes.size()) * 4);
    if (leaf_rec) memcpy(leaf_rec, R.leaf_rec.data(), std::min<uint64_t>(cap_leaf_rec, R.leaf_rec.size()) * 4);
    if (leaf_id) memcpy(leaf_id, R.leaf_id.data(), std::min<uint64_t>(cap_leaf_id, R.leaf_id.size()) * 4);
    if (always) memcpy(always, R.always.data(), std::min<uint64_t>(cap_always, R.always.size()) * 4);
    if (flat) memcpy(flat, R.flat.data(), std::min<uint64_t>(cap_flat, R.flat.size()) * 4);
    return RT_OK;
  });
}

int rtb200_scene_release(rtb200_scene_handle h) {
    if (!h) return RT_OK;
    DeviceRestore restore;
    if (h->ctx) {
        std::lock_guard<std::recursive_mutex> lk(h->ctx->mu);
        cudaSetDevice(h->device);
        if (!h->pending.empty()) render_collect(h, nullptr);   // frames still in flight read the scene arrays
        else if (h->ctx->stream) cudaStreamSynchronize(h->ctx->stream);
        if (h->updated) { cudaEventSynchronize(h->updated); cudaEventDestroy(h->updated); }   // an update in flight writes them
        for (const auto& q : h->queries) { cudaEventSynchronize(q.done); cudaEventDestroy(q.done); }   // queries in flight read them
        if (h->refit) cudaFree(h->refit);
        if (h->rebuild) cudaFree(h->rebuild);
        if (h->ed.mem) cudaFree(h->ed.mem);
        if (h->upd_in.p) cudaFree(h->upd_in.p);
        if (h->ad.mem) cudaFree(h->ad.mem);
        if (h->ad.active_host) cudaFreeHost(h->ad.active_host);
        for (cudaEvent_t e : h->ev) h->ctx->event_pool.push_back(e);
        if (h->arena) {
            auto& cache = h->ctx->arena_cache;
            if (h->arena_cap <= (64u << 20) && cache.size() < 4) cache.push_back(DeviceCtx::Arena{h->arena, h->arena_cap});
            else cudaFree(h->arena);
        }
    }
    delete h;
    return RT_OK;
}

// Scene arrays are collected first and then placed in ONE device arena filled by ONE host->device copy from pinned
// staging memory; arenas of released scenes are reused. `field` is patched with the device address.
static void upload_array(rtb200_scene_t* h, const void* src, size_t bytes, void** field) {
    *field = nullptr;
    if (bytes == 0) bytes = 16;
    h->uploads.push_back(rtb200_scene_t::Upload{src, bytes, field});
}

static int commit_uploads(rtb200_scene_t* h) {
    DeviceCtx* ctx = h->ctx;
    Carver size;
    for (auto& u : h->uploads) size.take(u.bytes);
    const size_t total = size.off ? size.off : 256;
    // smallest cached arena that is large enough, else a new allocation
    int pick = -1;
    for (int i = 0; i < (int)ctx->arena_cache.size(); ++i)
        if (ctx->arena_cache[i].cap >= total && (pick < 0 || ctx->arena_cache[i].cap < ctx->arena_cache[pick].cap)) pick = i;
    if (pick >= 0) {
        h->arena = ctx->arena_cache[pick].p; h->arena_cap = ctx->arena_cache[pick].cap;
        ctx->arena_cache.erase(ctx->arena_cache.begin() + pick);
    } else {
        size_t want = total + total / 4;
        cudaError_t e = cudaMalloc(&h->arena, want);
        if (e != cudaSuccess) { cudaGetLastError(); want = total; CU(cudaMalloc(&h->arena, want)); }
        h->arena_cap = want;
    }
    Carver arena(h->arena);
    for (auto& u : h->uploads) *u.field = arena.take(u.bytes);   // addresses first: tables may hold them
    CU(cudaEventSynchronize(ctx->staging_free));   // the previous upload's copy has left the staging buffer
    CU(ctx->staging.ensure(total));
    Carver staged(ctx->staging.p);
    for (auto& u : h->uploads) {
        void* d = staged.take(u.bytes);
        if (u.src) { memcpy(d, u.src, u.bytes); h->h2d_bytes += u.bytes; }
        else memset(d, 0, u.bytes);
    }
    CU(cudaMemcpyAsync(h->arena, ctx->staging.p, staged.off, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaEventRecord(ctx->staging_free, ctx->stream));
    h->uploads.clear();
    return RT_OK;
}

static bool image_ok(const rt_image& im) {
    if (!im.rgb8 || im.width == 0 || im.height == 0) return false;
    if (im.width > (1ull << 20) || im.height > (1ull << 20)) return false;
    return im.width * im.height * 3ull <= im.bytes;   // the callee reads width*height*3 bytes: the buffer must hold them
}

int rtk::validate_scene(const rt_scene* s, uint32_t* n_lights_out) {
    if (s->width < 2 || s->height < 2) return fail(RT_ERR_INVALID, "width and height must be >= 2 (u,v divide by w-1, h-1: raytracer.rs:199-200)");
    if (s->samples_per_pixel == 0) return fail(RT_ERR_INVALID, "samples_per_pixel must be > 0");
    if ((uint64_t)s->width * s->height >= (1ull << 31)) return fail(RT_ERR_INVALID, "image too large");
    if (s->n_spheres >= (1ull << 26)) return fail(RT_ERR_UNSUPPORTED, kErrSpheres);
    if (s->n_spheres && !s->spheres) return fail(RT_ERR_INVALID, "spheres is null");
    if (s->n_textures && !s->textures) return fail(RT_ERR_INVALID, "textures is null");
    uint32_t n_lights = 0;
    for (uint64_t i = 0; i < s->n_spheres; ++i) {
        const rt_sphere& sp = s->spheres[i];
        if (sp.kind > RT_LIGHT) return fail(RT_ERR_INVALID, "unknown material kind");
        if (sp.kind == RT_LIGHT) ++n_lights;
        if (sp.kind == RT_TEXTURE) {
            if (sp.texture < 0 || (uint64_t)sp.texture >= s->n_textures) return fail(RT_ERR_INVALID, "texture index out of range");
            if (!image_ok(s->textures[sp.texture])) return fail(RT_ERR_INVALID, "texture image is empty or smaller than width*height*3 bytes (rt_image.bytes)");
        }
    }
    if (n_lights >= 10) return fail(RT_ERR_UNSUPPORTED, kErrLights);
    if (s->sky.mode > RT_SKY_TEXTURE) return fail(RT_ERR_INVALID, "unknown sky mode");
    if (s->sky.mode == RT_SKY_TEXTURE && !image_ok(s->sky.tex)) return fail(RT_ERR_INVALID, "sky texture is empty or smaller than width*height*3 bytes (rt_image.bytes)");
    *n_lights_out = n_lights;
    return RT_OK;
}

int rtk::normalise_options(const rt_options* opts_in, rt_options* o) {
    memset(o, 0, sizeof *o);
    o->device = -1; o->rank = 0; o->world = 1; o->band_rows = 1; o->variant = RT_VARIANT_AUTO;
    if (opts_in) *o = *opts_in;
    if (o->world <= 0) o->world = 1;
    if (o->band_rows == 0) o->band_rows = 1;
    if (o->rank < 0 || o->rank >= o->world) return fail(RT_ERR_INVALID, "rank outside [0, world)");
    if (o->flags != 0) return fail(RT_ERR_INVALID, "flags must be 0");
    if (o->variant == RT_VARIANT_RETIRED_LANES) return fail(RT_ERR_UNSUPPORTED, "RT_VARIANT_LANES was retired in ABI 2");
    if (o->variant > RT_VARIANT_BRUTE_FORCE) return fail(RT_ERR_INVALID, "unknown variant");
    return RT_OK;
}

// TraceParams::albedo_nonfinite for a sphere: only Lambertian and Metal spheres carry their own albedo (Texture, Glass and
// Light albedos are finite)
bool rtk::albedo_nonfinite(const rt_sphere& sp) {
    return (sp.kind == RT_LAMBERTIAN || sp.kind == RT_METAL) &&
           !(std::isfinite(sp.albedo[0]) && std::isfinite(sp.albedo[1]) && std::isfinite(sp.albedo[2]));
}

void rtk::scene_records(const rt_scene* s, const rt_options& opts, rtbvh::Records& R) {
    rtbvh::build_records(s, mode_of(opts.variant) == MODE_TREE, R);
}

int rtk::scene_upload_records(const rt_scene* s, const rt_options& opts, uint32_t n_lights, const rtbvh::Records& R, rtb200_scene_handle* out) {
    *out = nullptr;
    DeviceCtx* ctx = nullptr;
    int rc = get_ctx(opts.device, &ctx);
    if (rc != RT_OK) return rc;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    if (R.depth > (uint32_t)rtbvh::kMaxDepth) return fail(RT_ERR_UNSUPPORTED, "hierarchy deeper than the traversal stack reserve");

    rtb200_scene_t* h = new rtb200_scene_t();
    struct Guard { rtb200_scene_t* h; bool ok = false; ~Guard() { if (!ok) rtb200_scene_release(h); } } guard{h};
    h->device = ctx->device; h->ctx = ctx; h->opts = opts;
    h->mode = mode_of(opts.variant);
    const uint32_t n = (uint32_t)s->n_spheres;

    TraceParams& tp = h->tp;
    tp.n = n; tp.n_pairs = R.n_pairs; tp.n_nodes = R.n_nodes; tp.n_leaves = R.n_leaves; tp.n_always = (uint32_t)R.always.size();
    tp.depth = R.depth; tp.n_lights = n_lights;
    upload_array(h, R.nodes.data(), R.nodes.size() * 4, (void**)&tp.nodes);
    upload_array(h, R.leaf_rec.data(), R.leaf_rec.size() * 4, (void**)&tp.leaf_rec);
    upload_array(h, R.leaf_id.data(), R.leaf_id.size() * 4, (void**)&tp.leaf_id);
    upload_array(h, R.skip_pos.data(), R.skip_pos.size() * 4, (void**)&tp.skip_pos);
    upload_array(h, R.always.data(), R.always.size() * 4, (void**)&tp.always);
    if (h->mode == MODE_BRUTE) upload_array(h, R.flat.data(), R.flat.size() * 4, (void**)&tp.filt);
    upload_array(h, R.geo.data(), R.geo.size() * 8, (void**)&tp.geo);
    upload_array(h, R.mat.data(), R.mat.size() * sizeof(DevMat), (void**)&tp.mat);

    std::vector<rtd::DevTex> texs(std::max<uint64_t>(s->n_textures, 1));
    for (uint64_t t = 0; t < s->n_textures; ++t) {
        const rt_image& im = s->textures[t];
        texs[t].rgb8 = nullptr; texs[t].width = im.width; texs[t].height = im.height;
        if (im.rgb8 && im.width && im.height && im.width * im.height * 3ull <= im.bytes)
            upload_array(h, im.rgb8, im.width * im.height * 3, (void**)&texs[t].rgb8);
    }
    upload_array(h, texs.data(), texs.size() * sizeof(rtd::DevTex), (void**)&tp.tex);
    tp.sky_mode = s->sky.mode;
    tp.sky.rgb8 = nullptr; tp.sky.width = 0; tp.sky.height = 0;
    if (s->sky.mode == RT_SKY_TEXTURE) {
        upload_array(h, s->sky.tex.rgb8, s->sky.tex.width * s->sky.tex.height * 3, (void**)&tp.sky.rgb8);
        tp.sky.width = s->sky.tex.width; tp.sky.height = s->sky.tex.height;
    }
    if (h->mode == MODE_TREE) { h->level_nodes = R.level_nodes; h->level_off = R.level_off; }
    std::vector<uint32_t> lights;
    for (uint32_t i = 0; i < n; ++i) {
        if (s->spheres[i].kind == RT_LIGHT) lights.push_back(i);
        if (albedo_nonfinite(s->spheres[i])) tp.albedo_nonfinite = 1u;
    }
    h->light_idx = lights;
    for (uint64_t t = 0; t < s->n_textures; ++t) h->tex_ok.push_back(image_ok(s->textures[t]));
    lights.push_back(0);
    upload_array(h, lights.data(), lights.size() * 4, (void**)&tp.lights);
    upload_array(h, nullptr, 16, (void**)&h->err);   // zero-filled error counters
    upload_array(h, nullptr, kMaxPending * kStatBytes, (void**)&h->stat_snap);
    tp.err = nullptr;                                // patched after commit
    tp.gx = R.g[0]; tp.gy = R.g[1]; tp.gz = R.g[2];
    tp.er_coef = 1.0f - (float)(96.0 * rtbvh::kU);
    tp.cam = s->camera;
    tp.width = s->width; tp.height = s->height; tp.spp = s->samples_per_pixel; tp.max_depth = s->max_depth;
    tp.key0 = (uint32_t)s->seed; tp.key1 = (uint32_t)(s->seed >> 32);
    tp.rank = opts.rank; tp.world = opts.world; tp.band_rows = opts.band_rows;
    tp.rows_local = rtb200_shard_rows(s->height, opts.rank, opts.world, opts.band_rows);
    tp.npix_local = tp.rows_local * s->width;

    // ---- launch geometry: persistent grid = SMs x resident CTAs of the mode's trace kernel ----
    // Nothing of the scene is staged into shared memory unless RTB200_WF_SMEM=<mask> asks for it (bit0 hierarchy / flat
    // records, bit1 geo, bit2 mat): for these small, hot arrays a larger L1 beats the staging (DESIGN.md §4.5).
    const char* es = getenv("RTB200_WF_SMEM");
    tp.scene_in_smem = es ? (uint32_t)atoi(es) : 0u;
    LaunchGeom g;
    if ((rc = launch_geometry(h, Q_SINGLE, n_lights > 0, &g)) != RT_OK) return rc;
    h->smem = g.smem; h->ctas_per_sm = g.ctas_per_sm; h->grid = g.grid;
    // ---- per-sample staging: samples per batch bounded by the buffer cap ----
    h->spp_batch = samples_per_batch(sample_buffer_cap(opts), tp.npix_local, s->samples_per_pixel);

    if ((rc = commit_uploads(h)) != RT_OK) return rc;
    h->tp.err = h->err;
    guard.ok = true;
    *out = h;
    return RT_OK;
}

// The first min(cap, count) elements of `elem` bytes of device array src into host array dst, enqueued on st (nothing when
// either array is null or either count is 0).
static cudaError_t copy_out(void* dst, const void* src, uint64_t cap, uint64_t count, size_t elem, cudaStream_t st) {
    if (!dst || !src || !cap || !count) return cudaSuccess;
    return cudaMemcpyAsync(dst, src, std::min(cap, count) * elem, cudaMemcpyDeviceToHost, st);
}

int rtb200_scene_upload(const rt_scene* s, const rt_options* opts_in, rtb200_scene_handle* out) {
  return guarded([&]() -> int {
    if (!s || !out) return fail(RT_ERR_INVALID, "null argument");
    *out = nullptr;
    rt_options opts;
    int rc = normalise_options(opts_in, &opts);
    if (rc != RT_OK) return rc;
    uint32_t n_lights = 0;
    if ((rc = validate_scene(s, &n_lights)) != RT_OK) return rc;
    DeviceRestore restore;
    rtbvh::Records R;
    scene_records(s, opts, R);
    return scene_upload_records(s, opts, n_lights, R, out);
  });
}

int rtb200_scene_kernel_info(rtb200_scene_handle h, rt_kernel_info* out) {
    if (!h || !out) return fail(RT_ERR_INVALID, "null argument");
    DeviceRestore restore;
    CU(cudaSetDevice(h->device));
    memset(out, 0, sizeof *out);
    KernelInfo ki{};
    CU(wavefront_info(h->mode, h->tp.n_lights > 0, Q_SINGLE, &ki));
    out->registers = ki.registers; out->local_bytes = ki.local_bytes; out->smem_bytes = (uint32_t)h->smem; out->grid = (uint32_t)h->grid;
    out->block = (uint32_t)kBlock; out->pool_slots = (uint32_t)kBlock;
    out->ctas_per_sm = (uint32_t)h->ctas_per_sm; out->smem_mask = h->tp.scene_in_smem;
    out->bvh_nodes = h->tp.n_nodes; out->bvh_leaves = h->tp.n_leaves; out->bvh_depth = h->tp.depth;
    snprintf(out->name, sizeof out->name, "%s", ki.name);
    return RT_OK;
}

// Diagnostic: the handle's current arrays, laid out as rtb200_debug_bvh's (flat records only in RT_VARIANT_BRUTE_FORCE)
int rtb200_scene_debug_records(rtb200_scene_handle h, uint32_t info[8], float* nodes, uint64_t cap_nodes, float* leaf_rec,
                               uint64_t cap_leaf_rec, float* flat, uint64_t cap_flat, double* geo, uint64_t cap_geo) {
  return guarded([&]() -> int {
    if (!h || !info) return fail(RT_ERR_INVALID, "null argument");
    const TraceParams& tp = h->tp;
    bvh_info(info, tp.n_nodes, tp.n_leaves, tp.depth, tp.n_always, tp.filt ? tp.n_pairs : 0u);
    HANDLE_PROLOGUE(h);
    cudaStream_t st;
    CU(scene_stream(h, nullptr, &st));
    CU(copy_out(nodes, tp.nodes, cap_nodes, (uint64_t)tp.n_nodes * rtbvh::kNodeFloats, 4, st));
    CU(copy_out(leaf_rec, tp.leaf_rec, cap_leaf_rec, (uint64_t)tp.n_leaves * rtbvh::kLeafK * 4, 4, st));
    CU(copy_out(flat, tp.filt, cap_flat, (uint64_t)info[6] * 8, 4, st));
    CU(copy_out(geo, tp.geo, cap_geo, (uint64_t)tp.n * 4, 8, st));
    CU(cudaStreamSynchronize(st));
    return RT_OK;
  });
}

// Diagnostic: the handle's current topology (the upload's, or the last rebuild's)
int rtb200_scene_debug_topology(rtb200_scene_handle h, double recentre[3], uint32_t info[8], uint32_t* leaf_id, uint64_t cap_leaf_id,
                                uint32_t* always, uint64_t cap_always, uint32_t* skip_pos, uint64_t cap_skip_pos,
                                uint32_t* level_nodes, uint64_t cap_level_nodes, uint32_t* level_off, uint64_t cap_level_off) {
  return guarded([&]() -> int {
    if (!h || !info) return fail(RT_ERR_INVALID, "null argument");
    const TraceParams& tp = h->tp;
    bvh_info(info, tp.n_nodes, tp.n_leaves, tp.depth, tp.n_always, tp.filt ? tp.n_pairs : 0u);
    if (recentre) { recentre[0] = tp.gx; recentre[1] = tp.gy; recentre[2] = tp.gz; }
    if (level_off && cap_level_off) memcpy(level_off, h->level_off.data(), std::min<uint64_t>(cap_level_off, h->level_off.size()) * 4);
    HANDLE_PROLOGUE(h);
    const bool tree = h->mode == MODE_TREE;
    cudaStream_t st;
    CU(scene_stream(h, nullptr, &st));
    CU(copy_out(leaf_id, tp.leaf_id, cap_leaf_id, (uint64_t)tp.n_leaves * rtbvh::kLeafK, 4, st));
    CU(copy_out(always, tp.always, cap_always, tp.n_always, 4, st));
    CU(copy_out(skip_pos, tp.skip_pos, cap_skip_pos, tree ? std::max<uint64_t>(tp.n, 1) : 0, 4, st));
    if (h->rebuild) CU(copy_out(level_nodes, h->level_nodes_dev, cap_level_nodes, tp.n_nodes, 4, st));
    if (level_nodes && cap_level_nodes && !h->rebuild)
        memcpy(level_nodes, h->level_nodes.data(), std::min<uint64_t>(cap_level_nodes, h->level_nodes.size()) * 4);
    CU(cudaStreamSynchronize(st));
    return RT_OK;
  });
}

// ---- probes ------------------------------------------------------------------------------------------
// One probe on the current device: in_bytes of `in` to the device, `launch(din, dout, stream)` enqueues the probe kernel,
// and the out_bytes it writes (zeroed first) come back into `out`. The probe buffer and the stream are the context's, so
// the context's lock is held until the result is on the host.
template <typename Launch>
static int probe_run(const void* in, size_t in_bytes, void* out, size_t out_bytes, Launch&& launch) {
    DeviceCtx* c = nullptr;
    int rc = get_ctx(-1, &c);
    if (rc != RT_OK) return rc;
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    CU(c->probe.ensure(in_bytes + out_bytes + 512));
    Carver block(c->probe.p);
    void* din = block.take(in_bytes);
    void* dout = block.take(out_bytes);
    CU(cudaMemsetAsync(dout, 0, out_bytes, c->stream));
    if (in_bytes) CU(cudaMemcpyAsync(din, in, in_bytes, cudaMemcpyHostToDevice, c->stream));
    CU(launch(din, dout, c->stream));
    CU(cudaMemcpyAsync(out, dout, out_bytes, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return RT_OK;
}

int rtb200_probe_sphere_hit(const rt_vec3* center, double radius, const rt_vec3* origin, const rt_vec3* dir, double t_min,
                            double t_max, int32_t* hit, double* t, rt_vec3* point, rt_vec3* normal, int32_t* front_face) {
    double in[12] = {center->x, center->y, center->z, radius, origin->x, origin->y, origin->z, dir->x, dir->y, dir->z, t_min, t_max};
    double out[9];
    int rc = probe_run(in, sizeof in, out, sizeof out, [](void* din, void* dout, cudaStream_t st) {
        return probe_sphere_hit((const double*)din, (double*)dout, st);
    });
    if (rc != RT_OK) return rc;
    *hit = out[0] != 0.0;
    if (*hit) {
        *t = out[1]; *point = rt_vec3{out[2], out[3], out[4]}; *normal = rt_vec3{out[5], out[6], out[7]};
        *front_face = out[8] != 0.0;
    }
    return RT_OK;
}
int rtb200_probe_refract(const rt_vec3* uv, const rt_vec3* n, double eta, rt_vec3* o) {
    double in[7] = {uv->x, uv->y, uv->z, n->x, n->y, n->z, eta}, out[3];
    int rc = probe_run(in, sizeof in, out, sizeof out, [](void* din, void* dout, cudaStream_t st) {
        return probe_refract((const double*)din, (double*)dout, st);
    });
    if (rc != RT_OK) return rc;
    *o = rt_vec3{out[0], out[1], out[2]};
    return RT_OK;
}
int rtb200_probe_reflectance(double cosine, double ref_idx, double* o) {
    double in[2] = {cosine, ref_idx};
    return probe_run(in, sizeof in, o, 8, [](void* din, void* dout, cudaStream_t st) {
        return probe_reflectance((const double*)din, (double*)dout, st);
    });
}
int rtb200_probe_sky(const rt_vec3* dir, uint32_t sky_mode, float out_rgb[3]) {
    if (sky_mode == RT_SKY_TEXTURE) return fail(RT_ERR_INVALID, "probe_sky supports none/gradient only");
    double in[3] = {dir->x, dir->y, dir->z};
    return probe_run(in, sizeof in, out_rgb, 12, [&](void* din, void* dout, cudaStream_t st) {
        return probe_sky((const double*)din, sky_mode, (float*)dout, st);
    });
}
int rtb200_probe_get_ray(const rt_camera* cam, double u, double v, rt_vec3* origin, rt_vec3* dir) {
    struct { rt_camera cam; double uv[2]; } in;
    in.cam = *cam; in.uv[0] = u; in.uv[1] = v;
    double out[6];
    int rc = probe_run(&in, sizeof in, out, sizeof out, [](void* din, void* dout, cudaStream_t st) {
        return probe_get_ray((const rt_camera*)din, (const double*)((char*)din + sizeof(rt_camera)), (double*)dout, st);
    });
    if (rc != RT_OK) return rc;
    *origin = rt_vec3{out[0], out[1], out[2]}; *dir = rt_vec3{out[3], out[4], out[5]};
    return RT_OK;
}
int rtb200_probe_lens_ray(const rt_camera* cam, const rt_lens* lens, uint64_t seed, uint32_t pixel, uint32_t sample, double u,
                          double v, rt_vec3* origin, rt_vec3* dir, uint32_t* trials) {
    if (!cam || !origin || !dir) return fail(RT_ERR_INVALID, "null argument");
    struct { rt_camera cam; rt_lens lens; double uv[2]; } in;
    in.cam = *cam; in.lens = lens ? *lens : rt_lens{}; in.uv[0] = u; in.uv[1] = v;
    int rc = check_lens(in.lens, "lens");
    if (rc != RT_OK) return rc;
    double out[7];
    rc = probe_run(&in, sizeof in, out, sizeof out, [&](void* din, void* dout, cudaStream_t st) {
        char* b = (char*)din;
        return probe_lens_ray((const rt_camera*)b, (const rt_lens*)(b + sizeof(rt_camera)), (const double*)(b + sizeof(rt_camera) + sizeof(rt_lens)),
                              seed, pixel, sample, (double*)dout, st);
    });
    if (rc != RT_OK) return rc;
    *origin = rt_vec3{out[0], out[1], out[2]}; *dir = rt_vec3{out[3], out[4], out[5]};
    if (trials) *trials = (uint32_t)out[6];
    return RT_OK;
}
int rtb200_probe_rng(uint64_t seed, uint32_t pixel, uint32_t sample, uint32_t kind, uint32_t n, double* o) {
    return probe_run(nullptr, 0, o, (size_t)n * 8, [&](void*, void* dout, cudaStream_t st) {
        return probe_rng(seed, pixel, sample, kind, n, (double*)dout, st);
    });
}
int rtb200_probe_sphere_uv(const double* hp_xyz, uint32_t n, double* out_uv) {
    return probe_run(hp_xyz, (size_t)n * 24, out_uv, (size_t)n * 16, [&](void* din, void* dout, cudaStream_t st) {
        return probe_sphere_uv((const double*)din, n, (double*)dout, st);
    });
}
int rtb200_probe_quantise(const float* mean_linear, uint32_t n, uint8_t* o) {
    return probe_run(mean_linear, (size_t)n * 4, o, n, [&](void* din, void* dout, cudaStream_t st) {
        return probe_quantise((const float*)din, n, (uint8_t*)dout, st);
    });
}

