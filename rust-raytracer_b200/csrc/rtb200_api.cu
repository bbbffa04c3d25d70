// rtb200_api.cu — the C ABI of include/rtb200.h: scene staging into HBM, scheduling of the trace / resolve kernels, multi-GPU
// frames, device<->host copies and error reporting. Every render entry point, one frame or many, blocking or asynchronous,
// enqueues its frames through render_enqueue and reports them through render_collect. No CPU render path exists here.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "rtb200_bvh.hpp"
#include "rtb200_kernels.cuh"

using namespace rtk;

static_assert(kCapIn >= 32 + 7 * rtbvh::kMaxDepth + 8, "the node stack must hold 32 roots plus a single-entry descent of the deepest tree (LIFO reserve, DESIGN.md 4.1)");

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) { g_last_error = msg; return code; }
int fail_cuda(cudaError_t e, const char* what) {
    g_last_error = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? RT_ERR_NO_DEVICE
           : (e == cudaErrorMemoryAllocation ? RT_ERR_OOM : RT_ERR_CUDA);
}
#define CU(call)                                              \
    do {                                                      \
        cudaError_t e__ = (call);                             \
        if (e__ != cudaSuccess) return fail_cuda(e__, #call); \
    } while (0)

struct GrowBuf {
    void* p = nullptr;
    size_t cap = 0;
    // `busy`: recorded after the last use of the buffer on the device; a growth waits for it on the host before the old
    // buffer is freed (cudaFree's own synchronisation is not relied on).
    cudaError_t ensure(size_t bytes, cudaEvent_t busy = nullptr) {
        if (bytes <= cap) return cudaSuccess;
        if (p && busy) { cudaError_t e = cudaEventSynchronize(busy); if (e != cudaSuccess) return e; }
        if (p) { cudaError_t e = cudaFree(p); if (e != cudaSuccess) return e; p = nullptr; cap = 0; }
        size_t want = bytes + bytes / 8;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { cudaGetLastError(); e = cudaMalloc(&p, bytes); want = bytes; }
        if (e != cudaSuccess) return e;
        cap = want;
        return cudaSuccess;
    }
};
constexpr size_t kStatBytes = 256;      // a work set's stat block (32 counters), followed by its queue counters
constexpr uint32_t kMaxPending = 64;    // submissions of one handle enqueued without a collect

struct PinnedBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) { cudaFreeHost(p); p = nullptr; cap = 0; }
        cudaError_t e = cudaHostAlloc(&p, bytes + bytes / 8, cudaHostAllocDefault);
        if (e != cudaSuccess) return e;
        cap = bytes + bytes / 8;
        return cudaSuccess;
    }
};

// Per-device execution context: one stream, grow-only work buffers. `mu` serialises the calls that use the context, so two
// host threads may render on two DIFFERENT devices concurrently; calls on the same device take turns.
struct DeviceCtx {
    std::recursive_mutex mu;
    bool init = false;
    int device = -1;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    // Two sets of per-frame work buffers, shared by every handle of the device: a frame loop that alternates two streams lets
    // frame k+1 start tracing while frame k drains its last paths and resolves (rtb200_render_device_async); blocking calls
    // use set 0 only. `done` is recorded after the last use of the set by the latest submission that took it, on that
    // submission's stream; the next submission's stream waits for it, so submissions that share a set run one after the other
    // whatever their streams and handles.
    struct WorkSet {
        GrowBuf samplebuf, accum, stack, small, frames, lterm, ftab;   // ftab: the multi-frame kernel's frame table
        cudaEvent_t done = nullptr;
    } ws[2];
    GrowBuf out_rgb8, out_lin, out_cnt, probe, frame;
    // scene arenas of released handles, kept for the next upload (a per-frame upload costs no cudaMalloc / cudaFree)
    struct Arena { void* p; size_t cap; };
    std::vector<Arena> arena_cache;
    std::vector<cudaEvent_t> event_pool;  // timing events of released handles (creating four events per one-shot render costs more than the upload)
    struct OccKey { uint32_t mode; bool lights; uint32_t queue; size_t smem; int occ; };
    std::vector<OccKey> occ_cache;        // cudaOccupancyMaxActiveBlocksPerMultiprocessor answers
    PinnedBuf staging;                    // host image of the arena being uploaded
    cudaEvent_t staging_free = nullptr;   // the last H2D copy out of `staging` has finished
    // the host form of rtb200_scene_intersect and rtb200_scene_occluded: rays, outputs and counters on the device, its timing
    // events (created at its first call), and the resident CTAs per SM of the query kernel of each kind and mode (0: not asked yet)
    GrowBuf query;
    cudaEvent_t query_ev[4] = {nullptr, nullptr, nullptr, nullptr};
    int query_occ[2][3] = {{0, 0, 0}, {0, 0, 0}};   // [closest-hit, occlusion][mode]
};
DeviceCtx g_ctx[64];
std::mutex g_ctx_mu;

int get_ctx(int device, DeviceCtx** out) {
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

// RAII: restores the caller's current device (the ABI must not leave cudaSetDevice changed behind the caller's back)
struct DeviceRestore {
    int prev = -1;
    DeviceRestore() { if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; } }
    ~DeviceRestore() { if (prev >= 0) cudaSetDevice(prev); }
};

struct V3 { double x, y, z; };
inline V3 v3(const rt_vec3& a) { return V3{a.x, a.y, a.z}; }
inline V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
inline V3 operator*(V3 a, double s) { return V3{a.x * s, a.y * s, a.z * s}; }
inline double vlen(V3 a) { return std::sqrt(a.x * a.x + a.y * a.y + a.z * a.z); }
inline V3 vunit(V3 a) { double l = vlen(a); return V3{a.x / l, a.y / l, a.z / l}; }
inline V3 vcross(V3 a, V3 b) { return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
inline rt_vec3 rv(V3 a) { return rt_vec3{a.x, a.y, a.z}; }

// No C++ exception may unwind through the C boundary (std::bad_alloc while building the hierarchy of a huge scene, ...).
template <typename F>
int guarded(F&& f) {
    try { return f(); }
    catch (const std::bad_alloc&) { return fail(RT_ERR_OOM, "host memory allocation failed"); }
    catch (const std::exception& e) { return fail(RT_ERR_INVALID, std::string("internal error: ") + e.what()); }
    catch (...) { return fail(RT_ERR_INVALID, "internal error: unknown exception"); }
}

uint32_t mode_of(uint32_t variant) {
    return variant == RT_VARIANT_EXACT_F64 ? MODE_EXACT : (variant == RT_VARIANT_BRUTE_FORCE ? MODE_BRUTE : MODE_TREE);
}

// resident CTAs per SM of one trace kernel with `smem` bytes of dynamic shared memory (cached per context)
int occupancy(DeviceCtx* ctx, uint32_t mode, bool lights, uint32_t queue, size_t smem) {
    for (auto& k : ctx->occ_cache) if (k.mode == mode && k.lights == lights && k.queue == queue && k.smem == smem) return k.occ;
    const int occ = wavefront_max_ctas_per_sm(mode, lights, queue, smem);
    ctx->occ_cache.push_back(DeviceCtx::OccKey{mode, lights, queue, smem, occ});
    return occ;
}

}  // namespace

struct rtb200_scene_t {
    int device = -1;
    DeviceCtx* ctx = nullptr;
    TraceParams tp{};
    rt_options opts{};
    uint32_t mode = MODE_TREE;
    int grid = 0;
    int ctas_per_sm = 0;
    size_t smem = 0;
    uint32_t spp_batch = 0;
    void* arena = nullptr;               // ONE device allocation holding every scene array (returned to the context's cache on release)
    size_t arena_cap = 0;
    unsigned long long* err = nullptr;   // device: [0] shadow-frame-stack overflows, [1] traversal guard trips; accumulated over frames, cleared by wait
    struct Upload { const void* src; size_t bytes; void** field; };
    std::vector<Upload> uploads;         // pending scene arrays (commit_uploads)
    std::vector<cudaEvent_t> ev;         // timing events of the pending submissions, each one's ev[ev0, ev0 + n_ev)
    // What one render_enqueue put on a stream. Events: begin, end, and a pair around each trace launch (or black memset).
    struct Submission {
        cudaStream_t stream;
        uint32_t ev0, n_ev;              // n_ev = 0: a shard with no rows, nothing was enqueued
        uint32_t frames, batches, launches;
        int grid;                        // of the widest launch (print_diagnostics)
        uint64_t black_samples;          // samples of max_depth 0 frames: black, no kernel counts them
        uint64_t ftab_bytes;             // frame table uploaded
    };
    std::vector<Submission> pending;     // enqueued since the last render_collect, oldest first
    // device: the stat block of pending[i], copied out of its work set at the end of the submission (the set may be taken by
    // another submission before the collect reads it)
    unsigned long long* stat_snap = nullptr;
    uint32_t frame_counter = 0;
    uint64_t h2d_bytes = 0;
    // ---- moving spheres (rtb200_scene_update_*): what the upload fixed, and the refit's scratch built at the first update ----
    std::vector<uint32_t> light_idx;     // the Light spheres, increasing
    std::vector<uint8_t> tex_ok;         // uploaded textures a Texture sphere may use
    cudaEvent_t updated = nullptr;       // recorded after the last update; every later frame waits for it
    std::vector<uint32_t> level_nodes, level_off;   // MODE_TREE: the builder's level order (rtbvh::Records::level_nodes)
    void* refit = nullptr;               // node_box, leaf_box, the device copy of level_nodes
    double* node_box = nullptr;          // n_nodes exact boxes {lo[3], hi[3]}
    double* leaf_box = nullptr;          // n_leaves exact boxes
    uint32_t* level_nodes_dev = nullptr;
    // ---- rebuilt hierarchy (rtb200_scene_rebuild): its arrays and the refit's scratch, allocated at the first rebuild ----
    void* rebuild = nullptr;             // RebuildBufs of rebuild_n spheres; once set, the tree arrays of tp and the refit scratch live here
    uint32_t rebuild_n = 0;
    GrowBuf upd_in;                      // host form's input: geo, materials, indices (an edit's: remove, at, geo, materials)
    // ---- edited list (rtb200_scene_edit_spheres, DESIGN.md §4.13): one device block for up to cap spheres, allocated at the
    // first edit and replaced by a larger one when an edit needs more. The list lives in half ed_cur (-1: still in the upload
    // arena) and the next edit writes the other half: frames enqueued before an edit keep reading the arrays they were
    // enqueued with ----
    struct EditBlock {
        void* mem = nullptr;
        uint32_t cap = 0;
        struct Half { double4* geo; DevMat* mat; float* filt; uint32_t* lights; } half[2] = {};   // filt: MODE_BRUTE only
        uint32_t* skip_pos = nullptr;    // cap x kNoSkip: the skip_pos of a list without a hierarchy
        uint32_t* keep = nullptr;        // cap + 1 words each: the keep flags of the old list and their scan
        uint32_t* pos = nullptr;
        void* temp = nullptr;            // cub's scan scratch
        size_t temp_bytes = 0;
    } ed;
    int ed_cur = -1;
    uint32_t updates = 0;                // rtb200_scene_update_* calls so far: an adaptive render refuses to step across one
    // ---- closest-hit queries (rtb200_scene_intersect_device): queries[0, n_queries) hold the last query of each stream enqueued
    // since the last update or rebuild, which the next update or rebuild waits for; the rest are spare events ----
    struct QueryMark { cudaStream_t stream; cudaEvent_t done; };
    std::vector<QueryMark> queries;
    uint32_t n_queries = 0;
    // ---- adaptive rendering (rtb200_adaptive_*, DESIGN.md §4.9): one device block allocated at the first begin ----
    struct Adaptive {
        void* mem = nullptr;             // sum, sq, count, keep, list[2], list_n[2], cub's scratch
        float* sum = nullptr;            // [npix_local][3] S_c
        float* sq = nullptr;             // [npix_local][3] Q_c
        uint32_t* count = nullptr;       // [npix_local] n
        uint32_t* keep = nullptr;        // [npix_local] by list position
        uint32_t* list[2] = {nullptr, nullptr};   // the list of the next round is list[cur], its length list_n[cur]
        uint32_t* list_n = nullptr;
        void* temp = nullptr;
        size_t temp_bytes = 0;
        uint32_t* active_host = nullptr; // pinned: list_n of the last step
        bool begun = false;              // false before the first begin and after a step that failed part-way
        rt_adaptive_params p{};
        uint32_t N = 0;                  // max_samples resolved
        uint32_t n = 0;                  // samples every listed pixel has
        uint32_t cur = 0;
        uint32_t active = 0;             // pixels on the list after the last step
        uint32_t updates = 0;            // `updates` at begin
    } ad;
};

// Releases a scene handle on scope exit; the error that made the scope return early survives the release.
struct ReleaseGuard {
    rtb200_scene_handle h;
    ~ReleaseGuard() { std::string keep = g_last_error; rtb200_scene_release(h); g_last_error = keep; }
};

extern "C" {

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

static int render_collect(rtb200_scene_handle h, rt_stats* stats);

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
    if (s->n_spheres >= (1ull << 26)) return fail(RT_ERR_UNSUPPORTED, "2^26 or more spheres (list entries carry 27-bit ids)");
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
    size_t total = 0;
    for (auto& u : h->uploads) total += (u.bytes + 255) & ~(size_t)255;
    if (total == 0) total = 256;
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
    char* base = (char*)h->arena;
    size_t off = 0;
    for (auto& u : h->uploads) { *u.field = base + off; off += (u.bytes + 255) & ~(size_t)255; }   // addresses first: tables may hold them
    CU(cudaEventSynchronize(ctx->staging_free));   // the previous upload's copy has left the staging buffer
    CU(ctx->staging.ensure(total));
    off = 0;
    for (auto& u : h->uploads) {
        if (u.src) { memcpy((char*)ctx->staging.p + off, u.src, u.bytes); h->h2d_bytes += u.bytes; }
        else memset((char*)ctx->staging.p + off, 0, u.bytes);
        off += (u.bytes + 255) & ~(size_t)255;
    }
    CU(cudaMemcpyAsync(base, ctx->staging.p, off, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaEventRecord(ctx->staging_free, ctx->stream));
    h->uploads.clear();
    return RT_OK;
}

static bool image_ok(const rt_image& im) {
    if (!im.rgb8 || im.width == 0 || im.height == 0) return false;
    if (im.width > (1ull << 20) || im.height > (1ull << 20)) return false;
    return im.width * im.height * 3ull <= im.bytes;   // the callee reads width*height*3 bytes: the buffer must hold them
}

static int validate_scene(const rt_scene* s, uint32_t* n_lights_out) {
    if (s->width < 2 || s->height < 2) return fail(RT_ERR_INVALID, "width and height must be >= 2 (u,v divide by w-1, h-1: raytracer.rs:199-200)");
    if (s->samples_per_pixel == 0) return fail(RT_ERR_INVALID, "samples_per_pixel must be > 0");
    if ((uint64_t)s->width * s->height >= (1ull << 31)) return fail(RT_ERR_INVALID, "image too large");
    if (s->n_spheres >= (1ull << 26)) return fail(RT_ERR_UNSUPPORTED, "2^26 or more spheres (list entries carry 27-bit ids)");
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
    if (n_lights >= 10) return fail(RT_ERR_UNSUPPORTED, "10 or more lights: the reference's light recursion (raytracer.rs:99-114) does not terminate when n_lights * 0.1 >= 1");
    if (s->sky.mode > RT_SKY_TEXTURE) return fail(RT_ERR_INVALID, "unknown sky mode");
    if (s->sky.mode == RT_SKY_TEXTURE && !image_ok(s->sky.tex)) return fail(RT_ERR_INVALID, "sky texture is empty or smaller than width*height*3 bytes (rt_image.bytes)");
    *n_lights_out = n_lights;
    return RT_OK;
}

static int normalise_options(const rt_options* opts_in, rt_options* o) {
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

// bytes of per-sample radiance one launch may stage (rt_options.sample_buffer_bytes, 0: 1 GiB)
static uint64_t sample_buffer_cap(const rt_options& o) { return o.sample_buffer_bytes ? o.sample_buffer_bytes : (1ull << 30); }

// TraceParams::albedo_nonfinite for a sphere: only Lambertian and Metal spheres carry their own albedo (Texture, Glass and
// Light albedos are finite)
static bool albedo_nonfinite(const rt_sphere& sp) {
    return (sp.kind == RT_LAMBERTIAN || sp.kind == RT_METAL) &&
           !(std::isfinite(sp.albedo[0]) && std::isfinite(sp.albedo[1]) && std::isfinite(sp.albedo[2]));
}

// `R` holds the host-side records (built once; the multi-GPU entry point shares them between its devices).
static int scene_upload_records(const rt_scene* s, const rt_options& opts, uint32_t n_lights, const rtbvh::Records& R, rtb200_scene_handle* out) {
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
    h->smem = wavefront_smem_bytes(tp, h->mode, tp.scene_in_smem, Q_SINGLE);
    const int occ = occupancy(ctx, h->mode, n_lights > 0, Q_SINGLE, h->smem);
    if (occ <= 0) return fail(RT_ERR_UNSUPPORTED, "no launch configuration fits shared memory");
    h->ctas_per_sm = occ;
    h->grid = ctx->sm_count * occ;

    // ---- per-sample staging: samples per batch bounded by the buffer cap ----
    uint64_t cap = sample_buffer_cap(opts);
    uint64_t per_spp = (uint64_t)std::max<uint32_t>(tp.npix_local, 1) * 16ull;
    uint64_t spb = std::max<uint64_t>(1, cap / per_spp);
    spb = std::min<uint64_t>(spb, s->samples_per_pixel);
    while (spb > 1 && spb * tp.npix_local >= (1ull << 31)) spb /= 2;
    h->spp_batch = (uint32_t)spb;

    if ((rc = commit_uploads(h)) != RT_OK) return rc;
    h->tp.err = h->err;
    guard.ok = true;
    *out = h;
    return RT_OK;
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
    rtbvh::build_records(s, mode_of(opts.variant) == MODE_TREE, R);
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

// Work buffers of W for launches of up to `threads_total` threads that trace paths up to `max_depth` deep, stage up to
// `samplebuf_bytes` of per-sample radiance and take `n_counters` queue counters; points tp at them (stack_stride excepted).
// A buffer that has to grow is freed only after the set's last submission has finished with it.
static int prepare_work(DeviceCtx::WorkSet& W, TraceParams& tp, uint32_t threads_total, uint32_t max_depth,
                        size_t samplebuf_bytes, uint32_t n_counters) {
    CU(W.samplebuf.ensure(samplebuf_bytes, W.done));
    CU(W.accum.ensure((size_t)tp.npix_local * 12, W.done));
    CU(W.stack.ensure((size_t)std::max<uint32_t>(max_depth, 1) * threads_total * 4, W.done));
    CU(W.small.ensure(kStatBytes + (size_t)n_counters * 4, W.done));
    if (tp.n_lights > 0) {
        // Nested light tests form a branching process: a vertex nests with probability 0.1 n and then spawns n shadow rays, so
        // depth d is reached with probability ~(0.1 n^2 P_hit)^d: harmless for 1-2 lights, near-critical for 3 (the reference
        // itself recurses hundreds of frames deep there) and super-critical beyond. Size the per-path frame stack accordingly;
        // an overflow is reported as an error, never rendered wrongly.
        tp.max_shadow = tp.n_lights == 1 ? 32u : tp.n_lights == 2 ? 96u : 384u;
        CU(W.frames.ensure((size_t)tp.max_shadow * threads_total * sizeof(ShadowFrame), W.done));
        CU(W.lterm.ensure((size_t)6 * threads_total * 4, W.done));
    }
    tp.frames = (ShadowFrame*)W.frames.p;
    tp.lterm = (float*)W.lterm.p;
    tp.samplebuf = (float4*)W.samplebuf.p;
    tp.stack = (uint32_t*)W.stack.p;
    tp.stat = (unsigned long long*)W.small.p;
    return RT_OK;
}

// Zero the stat block and the first n_counters queue counters of W.
static int clear_stats(DeviceCtx::WorkSet& W, uint32_t n_counters, cudaStream_t st) {
    CU(cudaMemsetAsync(W.small.p, 0, kStatBytes + (size_t)n_counters * 4, st));
    CU(cudaMemsetAsync((char*)W.small.p + 64, 0xff, 16, st));   // stat[8], stat[9]: minima (kernel start / first dry-queue time, ns)
    return RT_OK;
}

// ---- scheduling: frames of one resident scene in as few trace launches as the sample buffer allows ----
// A launch group is a run of consecutive frames with equal max_depth (a launch scalar) whose samples all fit the
// sample-buffer cap and the u32 work ids. A group of F >= 2 frames is ONE launch of the multi-frame trace kernel - the
// stragglers of frame i finish while frame i+1's work is handed out, so only the group's last frame pays the frame tail -
// followed by one resolve per frame. A frame that fits with no other, and every max_depth 0 frame, runs alone: per sample
// batch one launch of the single-frame trace kernel (a black memset at max_depth 0) and a resolve. So does a frame of more
// than kGroupMaxFrameWork samples: its own tail is a few per cent of its time at most, and the multi-frame kernel, which
// keeps the Philox key in registers instead of the parameter block, spills more and traced 800x600x128 frames 5 % slower
// than the single-frame kernel on an H100 (DESIGN.md §4.6).
struct FrameGroup { uint32_t first, count; };
constexpr uint64_t kGroupMaxFrameWork = 1ull << 24;   // samples per frame (spp * rows * width): ~8 ms of tracing on an H100

static std::vector<FrameGroup> frame_groups(const rt_frame* frames, uint32_t n, uint64_t frame_work, uint64_t cap) {
    std::vector<FrameGroup> groups;
    for (uint32_t i = 0; i < n;) {
        uint64_t F = 1;
        if (frames[i].max_depth != 0 && frame_work <= kGroupMaxFrameWork)
            while (i + F < n && frames[i + F].max_depth == frames[i].max_depth && (F + 1) * frame_work < (1ull << 31) && (F + 1) * frame_work * 16ull <= cap) ++F;
        groups.push_back(FrameGroup{i, (uint32_t)F});
        i += (uint32_t)F;
    }
    return groups;
}

// rt_frame checks shared by both frames entry points (no device is touched)
static int check_frames(const rt_frame* frames, uint32_t n, uint64_t rows, uint64_t width) {
    if (n == 0) return fail(RT_ERR_INVALID, "n_frames must be > 0");
    if (!frames) return fail(RT_ERR_INVALID, "frames is null");
    const uint64_t per_frame = rows * width * 3ull;   // < 2^33: width * height < 2^31 (validate_scene)
    if (per_frame != 0 && (uint64_t)n > ~0ull / per_frame) return fail(RT_ERR_INVALID, "n_frames * rows * width * 3 overflows 64 bits");
    for (uint32_t i = 0; i < n; ++i)
        if (frames[i].reserved != 0) return fail(RT_ERR_INVALID, "rt_frame.reserved must be 0 (frame " + std::to_string(i) + ")");
    return RT_OK;
}

// The handle's own view (the camera, seed and depth it was uploaded with) as a frame.
static rt_frame own_frame(rtb200_scene_handle h) { return rt_frame{h->tp.cam, h->tp.key0 | (uint64_t)h->tp.key1 << 32, h->tp.max_depth, 0}; }

// The stream of a call on h, `stream_in` (NULL: the context's stream), made to wait for what last wrote the scene arrays:
// the upload, which ran on the context's stream, and the last update or rebuild, on whichever stream it ran.
static cudaError_t scene_stream(rtb200_scene_handle h, void* stream_in, cudaStream_t* out) {
    const cudaStream_t st = stream_in ? (cudaStream_t)stream_in : h->ctx->stream;
    *out = st;
    if (st != h->ctx->stream) { cudaError_t e = cudaStreamWaitEvent(st, h->ctx->staging_free, 0); if (e != cudaSuccess) return e; }
    return h->updated ? cudaStreamWaitEvent(st, h->updated, 0) : cudaSuccess;
}

// ---- submissions: what one call enqueues on one stream with one work set, reported by render_collect ----
// A submission of h on `stream_in` (NULL: the context's stream) with work set `set` starts after the previous submission that
// took the same set, on any stream and of any handle, has finished with it; the caller holds the context's lock.
// submission_open picks the stream, submission_start sizes the set's buffers (prepare_work) and orders the stream after the
// set's last user, submission_events takes sub->n_ev timing events (begin, end, a pair per trace launch), clears the stat
// block and the sub->batches queue counters and records the begin event, submission_close records the end event, snapshots
// the stat block and appends the submission to h->pending. A submission that fails part-way is not recorded.
static int submission_open(rtb200_scene_handle h, void* stream_in, uint32_t frames, cudaStream_t* st, rtb200_scene_t::Submission* sub) {
    if (h->pending.size() >= kMaxPending) return fail(RT_ERR_INVALID, "more than 64 frames enqueued without rtb200_render_device_wait");
    CU(cudaSetDevice(h->device));
    CU(scene_stream(h, stream_in, st));
    const rtb200_scene_t::Submission* prev = h->pending.empty() ? nullptr : &h->pending.back();
    *sub = rtb200_scene_t::Submission{*st, prev ? prev->ev0 + prev->n_ev : 0u, 0, frames, 0, 0, h->grid, 0, 0};
    return RT_OK;
}

static int submission_start(DeviceCtx::WorkSet& W, cudaStream_t st, TraceParams& tp, const rtb200_scene_t::Submission& sub,
                            uint32_t max_depth, size_t samplebuf_bytes) {
    const uint32_t threads_total = (uint32_t)sub.grid * (uint32_t)kBlock;   // ray slots of the widest grid: columns of the per-slot global arrays
    int rc = prepare_work(W, tp, threads_total, max_depth, samplebuf_bytes, sub.batches);
    if (rc != RT_OK) return rc;
    CU(cudaStreamWaitEvent(st, W.done, 0));   // nothing below touches the set before its previous submission is done with it
    return RT_OK;
}

static int submission_events(rtb200_scene_handle h, DeviceCtx::WorkSet& W, cudaStream_t st, rtb200_scene_t::Submission& sub,
                             cudaEvent_t** ev_out) {
    DeviceCtx* ctx = h->ctx;
    sub.n_ev = 2 + 2 * sub.batches;
    while (h->ev.size() < (size_t)sub.ev0 + sub.n_ev) {
        cudaEvent_t e;
        if (!ctx->event_pool.empty()) { e = ctx->event_pool.back(); ctx->event_pool.pop_back(); }
        else CU(cudaEventCreate(&e));
        h->ev.push_back(e);
    }
    cudaEvent_t* ev = h->ev.data() + sub.ev0;
    int rc = clear_stats(W, sub.batches, st);
    if (rc != RT_OK) return rc;
    CU(cudaEventRecord(ev[0], st));
    *ev_out = ev;
    return RT_OK;
}

static int submission_close(rtb200_scene_handle h, DeviceCtx::WorkSet& W, cudaStream_t st, const rtb200_scene_t::Submission& sub) {
    CU(cudaEventRecord(h->ev[sub.ev0 + 1], st));
    CU(cudaMemcpyAsync(h->stat_snap + h->pending.size() * (kStatBytes / 8), W.small.p, kStatBytes, cudaMemcpyDeviceToDevice, st));
    CU(cudaEventRecord(W.done, st));
    h->pending.push_back(sub);
    return RT_OK;
}

// Enqueue frames[0, n) of h on `stream_in` (NULL: the context's stream) with work set `set`, without waiting, and append the
// submission to h->pending; the caller holds the context's lock. Frame i goes to output slice i (rows * width * 3 elements).
static int render_enqueue(rtb200_scene_handle h, const rt_frame* frames, uint32_t n, void* dev_rgb8, void* dev_linear_f32,
                          void* stream_in, int set) {
    DeviceCtx* ctx = h->ctx;
    DeviceCtx::WorkSet& W = ctx->ws[set];
    cudaStream_t st;
    rtb200_scene_t::Submission sub;
    int rc = submission_open(h, stream_in, n, &st, &sub);
    if (rc != RT_OK) return rc;
    TraceParams tp = h->tp;   // the handle's own view stays as uploaded
    const uint64_t npl = tp.npix_local;
    if (npl == 0) { h->pending.push_back(sub); return RT_OK; }   // a shard with no rows: nothing to trace
    const uint32_t spp = tp.spp, spb = h->spp_batch, n_batches = (spp + spb - 1) / spb;
    const uint64_t frame_work = (uint64_t)spp * npl;
    const std::vector<FrameGroup> groups = frame_groups(frames, n, frame_work, sample_buffer_cap(h->opts));
    // A batch of a group holds spb samples of each of its frames. A group of F >= 2 frames is one batch: frame_groups admits
    // it only when 2 * spp * npl * 16 bytes fit the cap and 2 * spp * npl < 2^31, and with these scene_upload_records made
    // spp_batch == spp.
    auto batches_of = [&](const FrameGroup& g) { return g.count > 1 ? 1u : n_batches; };

    // trace launches, work buffer sizes and the launch geometry of the multi-frame kernel (its pool also holds the slots' frames)
    size_t smem_f = 0;
    int grid_f = 0;
    uint32_t max_depth = 1;
    size_t sbuf = 0;
    for (const FrameGroup& g : groups) {
        sub.batches += batches_of(g);   // trace launches (or black memsets)
        sbuf = std::max(sbuf, (size_t)g.count * spb * npl * 16);
        max_depth = std::max(max_depth, frames[g.first].max_depth);
        if (g.count > 1 && grid_f == 0) {
            smem_f = wavefront_smem_bytes(tp, h->mode, tp.scene_in_smem, Q_FRAMES);
            const int occ = occupancy(ctx, h->mode, tp.n_lights > 0, Q_FRAMES, smem_f);
            if (occ <= 0) return fail(RT_ERR_UNSUPPORTED, "no launch configuration of the multi-frame trace kernel fits shared memory");
            grid_f = ctx->sm_count * occ;
        }
    }
    sub.grid = std::max(h->grid, grid_f);
    if ((rc = submission_start(W, st, tp, sub, max_depth, sbuf)) != RT_OK) return rc;
    if (grid_f) {   // the multi-frame kernel reads each frame's camera and key from this table
        std::vector<FrameRec> tab(n);
        for (uint32_t i = 0; i < n; ++i) {
            tab[i].cam = frames[i].camera; tab[i].key0 = (uint32_t)frames[i].seed; tab[i].key1 = (uint32_t)(frames[i].seed >> 32);
        }
        sub.ftab_bytes = (uint64_t)n * sizeof(FrameRec);
        CU(W.ftab.ensure(sub.ftab_bytes, W.done));
        CU(cudaMemcpyAsync(W.ftab.p, tab.data(), sub.ftab_bytes, cudaMemcpyHostToDevice, st));
    }
    cudaEvent_t* ev = nullptr;
    if ((rc = submission_events(h, W, st, sub, &ev)) != RT_OK) return rc;
    unsigned int* counters = (unsigned int*)((char*)W.small.p + kStatBytes);

    uint32_t b = 0;   // trace launch (or black memset) index: its queue counter and its event pair
    for (const FrameGroup& g : groups) {
        const rt_frame& f0 = frames[g.first];
        const bool multi = g.count > 1;   // the multi-frame trace kernel, which reads each frame's camera and key from ftab
        const uint32_t batches = batches_of(g);
        const int grid = multi ? grid_f : h->grid;
        const size_t smem = multi ? smem_f : h->smem;
        uint8_t* o8 = dev_rgb8 ? (uint8_t*)dev_rgb8 + (size_t)g.first * npl * 3 : nullptr;
        float* ol = dev_linear_f32 ? (float*)dev_linear_f32 + (size_t)g.first * npl * 3 : nullptr;
        TraceParams q = tp;
        q.max_depth = f0.max_depth;
        q.stack_stride = (uint32_t)grid * (uint32_t)kBlock;
        if (multi) { q.ftab = (const FrameRec*)W.ftab.p + g.first; q.frame_work = (uint32_t)frame_work; }
        else { q.cam = f0.camera; q.key0 = (uint32_t)f0.seed; q.key1 = (uint32_t)(f0.seed >> 32); }
        for (uint32_t k = 0; k < batches; ++k, ++b) {
            q.s0 = k * spb;
            q.s_count = std::min(spb, spp - q.s0);
            q.total_work = g.count * q.s_count * q.npix_local;
            q.work_counter = counters + b;
            CU(cudaEventRecord(ev[2 + 2 * b], st));
            if (q.max_depth == 0) {
                CU(cudaMemsetAsync(q.samplebuf, 0, (size_t)q.total_work * 16, st));   // ray_color(depth 0) = black, no ray (raytracer.rs:80-82)
            } else {
                CU(launch_wavefront(q, h->mode, multi ? Q_FRAMES : Q_SINGLE, grid, smem, st));
            }
            CU(cudaEventRecord(ev[3 + 2 * b], st));
            for (uint32_t j = 0; j < g.count; ++j) {   // samplebuf [frame][sample][pixel]
                ResolveParams r{};
                r.samplebuf = q.samplebuf + (size_t)j * q.s_count * npl; r.accum = (float*)W.accum.p; r.npix_local = q.npix_local;
                r.s_count = q.s_count; r.first = k == 0; r.last = k + 1 == batches; r.spp = spp;
                r.out_linear = ol ? ol + (size_t)j * npl * 3 : nullptr; r.out_rgb8 = o8 ? o8 + (size_t)j * npl * 3 : nullptr;
                CU(launch_resolve(r, st));
            }
        }
        sub.launches += batches * (1 + g.count);
        if (q.max_depth == 0) sub.black_samples += g.count * frame_work;
    }
    return submission_close(h, W, st, sub);
}

// RTB200_PRINT_TAIL / RTB200_PRINT_PHASES: the frame-tail and phase-clock counters of a stat block (stderr)
static void print_diagnostics(const unsigned long long* hstat, int grid) {
    if (getenv("RTB200_PRINT_TAIL") && hstat[8] != ~0ull) {   // when did the global queue run dry, when did the last CTA exit
        const double total = (double)(hstat[10] - hstat[8]) * 1e-6, tail = hstat[9] != ~0ull ? (double)(hstat[10] - hstat[9]) * 1e-6 : 0.0;
        fprintf(stderr, "[rtb200] trace kernel: first CTA start -> last CTA exit %.3f ms; queue dry -> last CTA exit (tail) %.3f ms; iterations after the queue ran dry: max %llu, mean %.1f per CTA\n",
                total, tail, hstat[11], (double)hstat[12] / std::max(1, grid));
    }
    if (getenv("RTB200_PRINT_PHASES")) {
        const unsigned long long* ph = hstat + kPhaseStat;
        if (ph[PH_ITERS] == 0) {
            fprintf(stderr, "[rtb200] fallbacks=%llu; no phase clocks: this library was built without RT_PHASE_CLOCKS (make -C rust-raytracer_b200 phase)\n", hstat[2]);
        } else {
            const double it = (double)ph[PH_ITERS];
            fprintf(stderr, "[rtb200] fallbacks=%llu phases (clock64 cycles per warp iteration): closest_hit=%.0f (node steps %.0f, leaf steps %.0f, exact steps %.0f) sort+waitA=%.0f shade=%.0f regen=%.0f waitC=%.0f; "
                    "warp_iters=%llu scatters=%llu deferred=%llu (%.4f of scatters); exact steps=%llu (%.2f per warp iteration) exact tests=%llu source-sphere skips=%llu rays=%llu\n",
                    hstat[2], ph[PH_HIT] / it, ph[PH_NODE] / it, ph[PH_LEAF] / it, ph[PH_EXACT] / it, ph[PH_SORT_WAIT_A] / it, ph[PH_SHADE] / it, ph[PH_REGEN] / it, ph[PH_WAIT_C] / it,
                    ph[PH_ITERS], ph[PH_SCATTERS], ph[PH_DEFERRED], (double)ph[PH_DEFERRED] / (double)std::max(1ull, ph[PH_SCATTERS]),
                    ph[PH_EXACT_STEPS], ph[PH_EXACT_STEPS] / it, ph[PH_EXACT_TESTS], ph[PH_SRC_SKIPS], hstat[0]);
        }
    }
}

// Wait for the pending submissions of h and report them (stats may be NULL). Counters, batches and the diagnostics are the
// last submission's (from its copy of the stat block); times, frames, kernel launches and frame-table bytes are summed over
// the submissions.
static int render_collect(rtb200_scene_handle h, rt_stats* stats) {
    if (stats) memset(stats, 0, sizeof *stats);
    if (h->pending.empty()) return RT_OK;
    CU(cudaSetDevice(h->device));
    const rtb200_scene_t::Submission last = h->pending.back();
    for (const auto& p : h->pending) if (p.stream != last.stream) CU(cudaStreamSynchronize(p.stream));
    unsigned long long hstat[kStatBytes / 8] = {0}, herr[2] = {0, 0};   // the whole stat block
    if (last.n_ev) {
        // error counters accumulate over every frame since the last collect (each frame adds to them; nothing clears them in between)
        const unsigned long long* snap = h->stat_snap + (h->pending.size() - 1) * (kStatBytes / 8);
        CU(cudaMemcpyAsync(hstat, snap, sizeof hstat, cudaMemcpyDeviceToHost, last.stream));
        CU(cudaMemcpyAsync(herr, h->err, sizeof herr, cudaMemcpyDeviceToHost, last.stream));
    }
    CU(cudaStreamSynchronize(last.stream));
    if (herr[0] | herr[1]) CU(cudaMemset(h->err, 0, sizeof herr));
    std::vector<rtb200_scene_t::Submission> subs;
    subs.swap(h->pending);
    if (herr[1] != 0) return fail(RT_ERR_CUDA, "internal error: the traversal guard tripped; the frames are not valid");
    if (herr[0] != 0) return fail(RT_ERR_UNSUPPORTED, "light-test recursion deeper than the shadow-frame stack occurred in one of the frames; it is not exact (the reference recursion is near-critical for this many lights)");
    if (!stats) return RT_OK;
    float ms = 0.f;
    for (const auto& p : subs) {
        const cudaEvent_t* ev = h->ev.data() + p.ev0;
        if (p.n_ev) { CU(cudaEventElapsedTime(&ms, ev[0], ev[1])); stats->device_ms += ms; }
        for (uint32_t b = 0; b < p.batches; ++b) { CU(cudaEventElapsedTime(&ms, ev[2 + 2 * b], ev[3 + 2 * b])); stats->trace_ms += ms; }
        stats->frames += p.frames; stats->kernel_launches += p.launches; stats->h2d_bytes += p.ftab_bytes;
    }
    stats->rays = hstat[0]; stats->candidates = hstat[1]; stats->samples = hstat[3] + last.black_samples; stats->clusters = hstat[4]; stats->nodes = hstat[6];
    stats->batches = last.batches; stats->gpus_used = 1;
    if (last.n_ev) print_diagnostics(hstat, last.grid);   // every launch of the last submission: the tail is one launch's when it made one
    return RT_OK;
}

// Drain the asynchronous frames of h, render `frames` on work set 0 and wait for them.
static int render_blocking(rtb200_scene_handle h, const rt_frame* frames, uint32_t n, void* dev_rgb8, void* dev_linear_f32,
                           void* stream_in, rt_stats* stats) {
    auto wall0 = std::chrono::steady_clock::now();
    DeviceRestore restore;
    std::lock_guard<std::recursive_mutex> lk(h->ctx->mu);
    int rc = render_collect(h, nullptr);
    if (rc == RT_OK) rc = render_enqueue(h, frames, n, dev_rgb8, dev_linear_f32, stream_in, 0);
    if (rc == RT_OK) rc = render_collect(h, stats);
    if (rc == RT_OK && stats) stats->wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    return rc;
}

int rtb200_render_device(rtb200_scene_handle h, void* dev_rgb8, void* dev_linear_f32, void* stream_in, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    const rt_frame f = own_frame(h);
    return render_blocking(h, &f, 1, dev_rgb8, dev_linear_f32, stream_in, stats);
  });
}

int rtb200_render_device_async(rtb200_scene_handle h, void* dev_rgb8, void* dev_linear_f32, void* stream_in) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    DeviceRestore restore;
    std::lock_guard<std::recursive_mutex> lk(h->ctx->mu);
    const rt_frame f = own_frame(h);
    return render_enqueue(h, &f, 1, dev_rgb8, dev_linear_f32, stream_in, (int)(h->frame_counter++ & 1u));
  });
}

int rtb200_render_device_wait(rtb200_scene_handle h, rt_stats* stats) {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    DeviceRestore restore;
    std::lock_guard<std::recursive_mutex> lk(h->ctx->mu);
    return render_collect(h, stats);
}

int rtb200_render_frames_device(rtb200_scene_handle h, const rt_frame* frames, uint32_t n_frames, void* dev_rgb8, void* dev_linear_f32,
                                void* stream_in, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    int rc = check_frames(frames, n_frames, h->tp.rows_local, h->tp.width);
    if (rc != RT_OK) return rc;
    if (!dev_rgb8 && !dev_linear_f32) return fail(RT_ERR_INVALID, "dev_rgb8 and dev_linear_f32 are both null");
    return render_blocking(h, frames, n_frames, dev_rgb8, dev_linear_f32, stream_in, stats);
  });
}

// ---- moving spheres of a resident scene: refit instead of rebuild (DESIGN.md §4.7) ----
// The refit's scratch, built at the first update of a MODE_TREE handle on the update's stream `st`: exact boxes of the nodes
// and leaves, and the device copy of the builder's level order (an update never changes the topology).
static int refit_prepare(rtb200_scene_handle h, cudaStream_t st) {
    const uint32_t nn = h->tp.n_nodes, nl = h->tp.n_leaves;
    if (h->node_box || h->mode != MODE_TREE || nn == 0) return RT_OK;   // a rebuild brings its own scratch
    void* p = nullptr;
    CU(cudaMalloc(&p, ((size_t)nn + nl) * 6 * sizeof(double) + (size_t)nn * 4));
    double* node_box = (double*)p;
    double* leaf_box = node_box + (size_t)nn * 6;
    uint32_t* level_nodes = (uint32_t*)(leaf_box + (size_t)nl * 6);
    const cudaError_t e = cudaMemcpyAsync(level_nodes, h->level_nodes.data(), (size_t)nn * 4, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { cudaFree(p); return fail_cuda(e, "cudaMemcpyAsync(level order)"); }
    // node_box marks the handle as prepared: set only once the level order is on its way
    h->refit = p; h->node_box = node_box; h->leaf_box = leaf_box; h->level_nodes_dev = level_nodes;
    return RT_OK;
}

// The event every later frame of h waits for, created by the first update or rebuild.
static cudaError_t update_begin(rtb200_scene_handle h) {
    return h->updated ? cudaSuccess : cudaEventCreateWithFlags(&h->updated, cudaEventDisableTiming);
}

// Order `st` after the frames and the queries of h in flight, on any stream: they read the arrays the update writes. Every
// later update or rebuild waits for this one (h->updated, scene_stream), so the queries waited for here are forgotten.
static int update_after_frames(rtb200_scene_handle h, cudaStream_t st) {
    for (const auto& p : h->pending) if (p.n_ev) CU(cudaStreamWaitEvent(st, h->ev[p.ev0 + 1], 0));
    for (uint32_t k = 0; k < h->n_queries; ++k) CU(cudaStreamWaitEvent(st, h->queries[k].done, 0));
    h->n_queries = 0;
    return RT_OK;
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

int rtb200_scene_update_spheres(rtb200_scene_handle h, const uint32_t* index, const rt_sphere* spheres, uint32_t n, void* stream_in) {
  return guarded([&]() -> int {
    if (n && (!index || !spheres)) return fail(RT_ERR_INVALID, "index or spheres is null");
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (n == 0) return RT_OK;
    // everything is checked before anything is enqueued: on error the scene is unchanged
    std::vector<uint32_t> sorted(index, index + n);
    std::sort(sorted.begin(), sorted.end());
    if (sorted.back() >= h->tp.n) return fail(RT_ERR_INVALID, "index " + std::to_string(sorted.back()) + " is not a sphere of the scene (n_spheres = " + std::to_string(h->tp.n) + ")");
    for (uint32_t k = 1; k < n; ++k)
        if (sorted[k] == sorted[k - 1]) return fail(RT_ERR_INVALID, "sphere " + std::to_string(sorted[k]) + " is listed twice");
    for (uint32_t k = 0; k < n; ++k) {
        const rt_sphere& sp = spheres[k];
        int rc = check_sphere(h, sp, "spheres", k);
        if (rc != RT_OK) return rc;
        const bool was_light = std::binary_search(h->light_idx.begin(), h->light_idx.end(), index[k]);
        if (was_light != (sp.kind == RT_LIGHT))
            return fail(RT_ERR_UNSUPPORTED, "sphere " + std::to_string(index[k]) + ": the set of lights is fixed at upload (upload the scene again to change it)");
    }
    DeviceRestore restore;
    DeviceCtx* ctx = h->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    CU(cudaSetDevice(h->device));
    ++h->updates;
    cudaStream_t st;   // after the previous update too: it may still read upd_in
    CU(scene_stream(h, stream_in, &st));
    CU(update_begin(h));
    int rc = refit_prepare(h, st);
    if (rc != RT_OK) return rc;
    // input in the pinned staging buffer (geo, materials, indices), copied before this call returns
    const size_t geo_b = (size_t)n * 32, mat_b = (size_t)n * sizeof(DevMat), bytes = geo_b + mat_b + (size_t)n * 4;
    CU(cudaEventSynchronize(ctx->staging_free));   // the previous copy has left the staging buffer
    CU(ctx->staging.ensure(bytes));
    char* S = (char*)ctx->staging.p;
    for (uint32_t k = 0; k < n; ++k) {
        rtbvh::sphere_exact(spheres[k], (double*)S + 4 * (size_t)k, ((rtbvh::Mat32*)(S + geo_b))[k]);
        // never cleared: the flag only selects the exact slow path, and frames already enqueued copied the old value
        if (albedo_nonfinite(spheres[k])) h->tp.albedo_nonfinite = 1u;
    }
    memcpy(S + geo_b + mat_b, index, (size_t)n * 4);
    CU(h->upd_in.ensure(bytes));
    char* D = (char*)h->upd_in.p;
    CU(cudaMemcpyAsync(D, S, bytes, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(ctx->staging_free, st));   // before the wait for the frames pending now (DESIGN.md §4.7, Ordering)
    if ((rc = update_after_frames(h, st)) != RT_OK) return rc;
    CU(launch_update_scatter((const uint32_t*)(D + geo_b + mat_b), (const double4*)D, (const DevMat*)(D + geo_b), n,
                             (double4*)h->tp.geo, (DevMat*)h->tp.mat, st));
    return update_finish(h, st);
  });
}

int rtb200_scene_update_geometry_device(rtb200_scene_handle h, const void* dev_center_radius, void* stream_in) {
  return guarded([&]() -> int {
    if (!dev_center_radius) return fail(RT_ERR_INVALID, "dev_center_radius is null");
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    DeviceRestore restore;
    DeviceCtx* ctx = h->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    CU(cudaSetDevice(h->device));
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, dev_center_radius) != cudaSuccess) { cudaGetLastError(); a.type = cudaMemoryTypeUnregistered; }
    if (!((a.type == cudaMemoryTypeDevice && a.device == h->device) || a.type == cudaMemoryTypeManaged))
        return fail(RT_ERR_INVALID, "dev_center_radius is not device or managed memory of device " + std::to_string(h->device));
    if (h->tp.n == 0) return RT_OK;
    ++h->updates;
    cudaStream_t st;
    CU(scene_stream(h, stream_in, &st));
    CU(update_begin(h));
    int rc = refit_prepare(h, st);
    if (rc == RT_OK) rc = update_after_frames(h, st);
    if (rc != RT_OK) return rc;
    CU(cudaMemcpyAsync((void*)h->tp.geo, dev_center_radius, (size_t)h->tp.n * 32, cudaMemcpyDeviceToDevice, st));
    return update_finish(h, st);
  });
}

// The first min(cap, count) elements of `elem` bytes of device array src into host array dst, enqueued on st (nothing when
// either array is null or either count is 0).
static cudaError_t copy_out(void* dst, const void* src, uint64_t cap, uint64_t count, size_t elem, cudaStream_t st) {
    if (!dst || !src || !cap || !count) return cudaSuccess;
    return cudaMemcpyAsync(dst, src, std::min(cap, count) * elem, cudaMemcpyDeviceToHost, st);
}

// Diagnostic: the handle's current arrays, laid out as rtb200_debug_bvh's (flat records only in RT_VARIANT_BRUTE_FORCE)
int rtb200_scene_debug_records(rtb200_scene_handle h, uint32_t info[8], float* nodes, uint64_t cap_nodes, float* leaf_rec,
                               uint64_t cap_leaf_rec, float* flat, uint64_t cap_flat, double* geo, uint64_t cap_geo) {
  return guarded([&]() -> int {
    if (!h || !info) return fail(RT_ERR_INVALID, "null argument");
    const TraceParams& tp = h->tp;
    bvh_info(info, tp.n_nodes, tp.n_leaves, tp.depth, tp.n_always, tp.filt ? tp.n_pairs : 0u);
    DeviceRestore restore;
    std::lock_guard<std::recursive_mutex> lk(h->ctx->mu);
    CU(cudaSetDevice(h->device));
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
    DeviceRestore restore;
    DeviceCtx* ctx = h->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    CU(cudaSetDevice(h->device));
    FreshBlock fresh;
    int rc = rebuild_reserve(h, h->tp.n, &fresh);
    if (rc != RT_OK) return rc;
    cudaStream_t st;
    CU(scene_stream(h, stream_in, &st));
    CU(update_begin(h));
    if ((rc = update_after_frames(h, st)) != RT_OK) return rc;
    return rebuild_tree(h, h->tp.n, fresh, st);
  });
}

// ---- inserting and removing spheres of a resident scene (DESIGN.md §4.13) ----
// The edit block of `cap` spheres carved out of `base` (null: only the size); returns the bytes. `flat`: the halves carry flat
// records (MODE_BRUTE).
static size_t edit_carve(void* base, uint32_t cap, bool flat, rtb200_scene_t::EditBlock* out) {
    size_t off = 0;
    char* p = (char*)base;
    auto take = [&](size_t bytes) -> void* { void* q = p ? p + off : nullptr; off += (bytes + 255) & ~(size_t)255; return q; };
    rtb200_scene_t::EditBlock b;
    b.mem = base; b.cap = cap;
    for (auto& H : b.half) {
        H.geo = (double4*)take((size_t)cap * 32);
        H.mat = (DevMat*)take((size_t)cap * sizeof(DevMat));
        H.filt = flat ? (float*)take((size_t)rtbvh::flat_pairs(cap) * 32) : nullptr;
        H.lights = (uint32_t*)take(16 * 4);   // at most 9 lights and the trailing 0 of the upload's list
    }
    b.skip_pos = (uint32_t*)take((size_t)cap * 4);
    b.keep = (uint32_t*)take(((size_t)cap + 1) * 4);
    b.pos = (uint32_t*)take(((size_t)cap + 1) * 4);
    b.temp_bytes = edit_scan_bytes(cap);
    b.temp = take(b.temp_bytes);
    if (out) *out = b;
    return off;
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
    std::vector<uint32_t> rem(remove, remove + n_remove);
    std::sort(rem.begin(), rem.end());
    if (n_remove && rem.back() >= n_old)
        return fail(RT_ERR_INVALID, "remove index " + std::to_string(rem.back()) + " is not a sphere of the scene (n_spheres = " + std::to_string(n_old) + ")");
    for (uint32_t k = 1; k < n_remove; ++k)
        if (rem[k] == rem[k - 1]) return fail(RT_ERR_INVALID, "sphere " + std::to_string(rem[k]) + " is listed twice in remove");
    std::vector<uint32_t> at_v(n_insert, n_old);   // at == NULL: every insert is appended
    for (uint32_t k = 0; k < n_insert; ++k) {
        if (at) {
            if (at[k] > n_old) return fail(RT_ERR_INVALID, "at[" + std::to_string(k) + "] = " + std::to_string(at[k]) + " exceeds n_spheres = " + std::to_string(n_old));
            if (k && at[k] < at[k - 1]) return fail(RT_ERR_INVALID, "at decreases at at[" + std::to_string(k) + "]");
            at_v[k] = at[k];
        }
        int rc = check_sphere(h, insert[k], "insert", k);
        if (rc != RT_OK) return rc;
    }
    const uint64_t n_new64 = (uint64_t)n_old - n_remove + n_insert;
    if (n_new64 >= (1ull << 26)) return fail(RT_ERR_UNSUPPORTED, "2^26 or more spheres (list entries carry 27-bit ids)");
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
    if (lights.size() >= 10) return fail(RT_ERR_UNSUPPORTED, "10 or more lights: the reference's light recursion (raytracer.rs:99-114) does not terminate when n_lights * 0.1 >= 1");
    if (h->tp.scene_in_smem)
        return fail(RT_ERR_UNSUPPORTED, "the handle stages the scene in shared memory (RTB200_WF_SMEM), whose launch layout is fixed at upload");

    DeviceRestore restore;
    DeviceCtx* ctx = h->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    CU(cudaSetDevice(h->device));
    TraceParams& tp = h->tp;
    // the single-frame kernel is another template with lights than without: its launch geometry follows n_lights > 0
    int occ = h->ctas_per_sm;
    if (lights.empty() != (tp.n_lights == 0)) {
        occ = occupancy(ctx, h->mode, !lights.empty(), Q_SINGLE, h->smem);
        if (occ <= 0) return fail(RT_ERR_UNSUPPORTED, "no launch configuration fits shared memory");
    }
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
    int rc = RT_OK;
    if (h->mode == MODE_TREE && n_new > 0 && (rc = rebuild_reserve(h, n_new, &fresh_rb)) != RT_OK) return rc;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t at_off = al((size_t)n_remove * 4), geo_off = at_off + al((size_t)n_insert * 4), mat_off = geo_off + al((size_t)n_insert * 32),
                 in_bytes = mat_off + al((size_t)n_insert * sizeof(DevMat));
    CU(h->upd_in.ensure(in_bytes, h->updated));   // after the last update, which read it
    const int tgt = fresh_ed.p || h->ed_cur != 0 ? 0 : 1;   // the half that does not hold the current list
    const auto& T = E.half[tgt];

    ++h->updates;
    cudaStream_t st;   // after the previous update or edit too: it may still read upd_in and the target half
    CU(scene_stream(h, stream_in, &st));
    CU(update_begin(h));
    // input in the pinned staging buffer (remove, at, the inserts' geo and materials; the light list), copied before this
    // call returns
    lights.push_back(0);
    CU(cudaEventSynchronize(ctx->staging_free));   // the previous copy has left the staging buffer
    CU(ctx->staging.ensure(in_bytes + lights.size() * 4));
    char* S = (char*)ctx->staging.p;
    memcpy(S, rem.data(), (size_t)n_remove * 4);
    memcpy(S + at_off, at_v.data(), (size_t)n_insert * 4);
    bool nonfinite = false;
    for (uint32_t k = 0; k < n_insert; ++k) {
        rtbvh::sphere_exact(insert[k], (double*)(S + geo_off) + 4 * (size_t)k, ((rtbvh::Mat32*)(S + mat_off))[k]);
        nonfinite = nonfinite || albedo_nonfinite(insert[k]);
    }
    memcpy(S + in_bytes, lights.data(), lights.size() * 4);
    char* D = (char*)h->upd_in.p;
    CU(cudaMemcpyAsync(D, S, in_bytes, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(T.lights, S + in_bytes, lights.size() * 4, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(ctx->staging_free, st));   // before the wait for the frames pending now (DESIGN.md §4.7, Ordering)
    if ((rc = update_after_frames(h, st)) != RT_OK) return rc;
    if (fresh_ed.p) CU(cudaMemsetAsync(E.skip_pos, 0xff, (size_t)E.cap * 4, st));   // rtbvh::kNoSkip
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
    h->ctas_per_sm = occ;
    h->grid = ctx->sm_count * occ;
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

// ---- closest-hit and occlusion queries on a resident scene (DESIGN.md §4.10, §4.11) ----
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
    if (out.any) {
        OcclusionParams q{};
        q.p = h->tp; q.p.stat = stat; q.p.err = err;
        q.origin = rays.origin; q.direction = rays.direction; q.t_max = rays.t_max;
        q.occluded = out.occluded;
        q.n = n;
        CU(launch_occluded(q, h->mode, max_grid, st));
        return RT_OK;
    }
    QueryParams q{};
    q.p = h->tp; q.p.stat = stat; q.p.err = err;
    q.origin = rays.origin; q.direction = rays.direction; q.t_max = rays.t_max;
    const rt_hits& o = out.hits;
    q.t = o.t; q.sphere = o.sphere; q.point = o.point; q.normal = o.normal; q.uv = o.uv; q.front_face = o.front_face;
    q.n = n;
    CU(launch_query(q, h->mode, max_grid, st));
    return RT_OK;
}

// RT_ERR_INVALID unless every non-null pointer of `ptrs` (pointer, name) is device memory of h's device or managed memory.
// The caller has made h's device current.
static int check_device_ptrs(rtb200_scene_handle h, const std::vector<std::pair<const void*, const char*>>& ptrs) {
    for (const auto& q : ptrs) {
        if (!q.first) continue;
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, q.first) != cudaSuccess) { cudaGetLastError(); a.type = cudaMemoryTypeUnregistered; }
        if (!((a.type == cudaMemoryTypeDevice && a.device == h->device) || a.type == cudaMemoryTypeManaged))
            return fail(RT_ERR_INVALID, std::string(q.second) + " is not device or managed memory of device " + std::to_string(h->device));
    }
    return RT_OK;
}

// The device form of both kinds.
static int query_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const QueryOut* out, void* stream_in) {
    int rc = check_query(h, rays, out);
    if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    DeviceRestore restore;
    std::lock_guard<std::recursive_mutex> lk(h->ctx->mu);
    CU(cudaSetDevice(h->device));
    std::vector<std::pair<const void*, const char*>> ptrs = {{rays->origin, "rays->origin"}, {rays->direction, "rays->direction"},
                                                             {rays->t_max, "rays->t_max"}};
    for (int k = 0; k < out->count; ++k) ptrs.push_back({out->ptr[k], out->name[k]});
    if ((rc = check_device_ptrs(h, ptrs)) != RT_OK) return rc;
    cudaStream_t st;
    CU(scene_stream(h, stream_in, &st));
    if ((rc = query_enqueue(h, *rays, n, *out, nullptr, h->err, st)) != RT_OK) return rc;
    // the next update or rebuild waits for the last query of each stream
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

// The host form of both kinds.
static int query_host(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const QueryOut* out, rt_stats* stats) {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_query(h, rays, out);
    if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    auto wall0 = std::chrono::steady_clock::now();
    DeviceRestore restore;
    DeviceCtx* ctx = h->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    CU(cudaSetDevice(h->device));
    for (auto& e : ctx->query_ev) if (!e) CU(cudaEventCreate(&e));
    // device image: counters (kStatBytes; the guard counters at stat[30..31]), then rays and outputs, 256-byte aligned
    const uint64_t N = n;
    const uint64_t in_b[3] = {N * 24, N * 24, rays->t_max ? N * 8 : 0};
    uint64_t out_b[6] = {0, 0, 0, 0, 0, 0};
    for (int k = 0; k < out->count; ++k) out_b[k] = out->ptr[k] ? N * out->bytes[k] : 0;
    auto al = [](uint64_t b) { return (b + 255) & ~(uint64_t)255; };
    uint64_t bytes = kStatBytes;
    for (uint64_t b : in_b) bytes += al(b);
    for (uint64_t b : out_b) bytes += al(b);
    CU(ctx->query.ensure(bytes));   // the last host-form query has finished: it waited for its stream
    char* D = (char*)ctx->query.p;
    unsigned long long* stat = (unsigned long long*)D;
    char* din[3]; char* dout[6];
    uint64_t off = kStatBytes;
    for (int k = 0; k < 3; ++k) { din[k] = in_b[k] ? D + off : nullptr; off += al(in_b[k]); }
    for (int k = 0; k < 6; ++k) { dout[k] = out_b[k] ? D + off : nullptr; off += al(out_b[k]); }
    cudaStream_t st;
    CU(scene_stream(h, nullptr, &st));
    cudaEvent_t* ev = ctx->query_ev;
    CU(cudaEventRecord(ev[0], st));
    CU(cudaMemsetAsync(stat, 0, kStatBytes, st));
    const void* src_in[3] = {rays->origin, rays->direction, rays->t_max};
    uint64_t h2d = 0, d2h = kStatBytes;
    for (int k = 0; k < 3; ++k) if (in_b[k]) { CU(cudaMemcpyAsync(din[k], src_in[k], in_b[k], cudaMemcpyHostToDevice, st)); h2d += in_b[k]; }
    const rt_rays drays{(const double*)din[0], (const double*)din[1], (const double*)din[2]};
    CU(cudaEventRecord(ev[1], st));
    if ((rc = query_enqueue(h, drays, n, with_ptrs(*out, dout), stat, stat + 30, st)) != RT_OK) return rc;
    CU(cudaEventRecord(ev[2], st));
    for (int k = 0; k < out->count; ++k) if (out_b[k]) { CU(cudaMemcpyAsync(out->ptr[k], dout[k], out_b[k], cudaMemcpyDeviceToHost, st)); d2h += out_b[k]; }
    unsigned long long hstat[kStatBytes / 8];
    CU(cudaMemcpyAsync(hstat, stat, kStatBytes, cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(ev[3], st));
    CU(cudaStreamSynchronize(st));
    if (hstat[31] != 0) return fail(RT_ERR_CUDA, "internal error: the traversal guard tripped; the query results are not valid");
    if (!stats) return RT_OK;
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, ev[0], ev[3])); stats->device_ms = ms;
    CU(cudaEventElapsedTime(&ms, ev[1], ev[2])); stats->trace_ms = ms;
    stats->rays = hstat[0]; stats->candidates = hstat[1]; stats->clusters = hstat[4]; stats->nodes = hstat[6];
    stats->kernel_launches = 1; stats->batches = 1; stats->gpus_used = 1;
    stats->h2d_bytes = h2d; stats->d2h_bytes = d2h;
    stats->wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count();
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

// ---- radiance of caller-supplied primary rays on a resident scene (DESIGN.md §4.12) ----
// The argument checks both forms share (no device is touched).
static int check_trace_rays(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_trace_params* p, const void* lin, const void* rgb) {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (!rays || !p) return fail(RT_ERR_INVALID, "rays or params is null");
    if (!rays->origin || !rays->direction) return fail(RT_ERR_INVALID, "rays->origin or rays->direction is null");
    if (rays->t_max) return fail(RT_ERR_INVALID, "rays->t_max must be null: ray_color traces its rays unbounded");
    if (!lin && !rgb) return fail(RT_ERR_INVALID, "the linear and rgb8 outputs are both null");
    if (p->samples == 0) return fail(RT_ERR_INVALID, "params->samples must be > 0");
    if (p->reserved[0] != 0 || p->reserved[1] != 0) return fail(RT_ERR_INVALID, "rt_trace_params.reserved must be 0");
    if ((uint64_t)p->stream0 + n > (1ull << 32)) return fail(RT_ERR_INVALID, "stream0 + n exceeds 2^32 (u32 RNG streams)");
    if ((uint64_t)p->sample0 + p->samples > (1ull << 32)) return fail(RT_ERR_INVALID, "sample0 + samples exceeds 2^32 (u32 sample indices)");
    if (n >= (1u << 31)) return fail(RT_ERR_INVALID, "n must be below 2^31 (u32 work ids of one sample of every ray)");
    if ((uint64_t)n * 16 > sample_buffer_cap(h->opts))
        return fail(RT_ERR_INVALID, "n * 16 bytes exceed the sample-buffer cap (rt_options.sample_buffer_bytes): one sample of every ray must fit");
    return RT_OK;
}

// Enqueue the samples of the n rays `rays` (device buffers) on work set 0 and append the submission to h->pending; the caller
// holds the context's lock and has collected h's asynchronous frames. Per batch of spb samples of every ray one launch of the
// Q_RAYS trace kernel (a black memset at max_depth 0) and one resolve, which carries the f32 sums across batches as
// render_enqueue's does. *st_out is the stream the submission runs on.
static int trace_rays_enqueue(rtb200_scene_handle h, const rt_rays& rays, uint32_t n, const rt_trace_params& tr, float* lin,
                              uint8_t* rgb, void* stream_in, cudaStream_t* st_out) {
    DeviceCtx* ctx = h->ctx;
    DeviceCtx::WorkSet& W = ctx->ws[0];
    cudaStream_t st;
    rtb200_scene_t::Submission sub;
    int rc = submission_open(h, stream_in, 1, &st, &sub);
    if (rc != RT_OK) return rc;
    *st_out = st;
    TraceParams tp = h->tp;
    tp.npix_local = n;   // Q_RAYS: the rays, which are also the resolve's pixels
    tp.max_depth = tr.max_depth;
    tp.key0 = (uint32_t)tr.seed; tp.key1 = (uint32_t)(tr.seed >> 32);
    tp.stream0 = tr.stream0;
    tp.ray_o = rays.origin; tp.ray_d = rays.direction;
    const uint32_t m = tr.samples;
    uint64_t spb = std::max<uint64_t>(1, sample_buffer_cap(h->opts) / ((uint64_t)n * 16));
    spb = std::min<uint64_t>(spb, m);
    while (spb > 1 && spb * n >= (1ull << 31)) spb /= 2;
    const uint32_t n_batches = (uint32_t)((m + spb - 1) / spb);
    const size_t smem = wavefront_smem_bytes(tp, h->mode, tp.scene_in_smem, Q_RAYS);
    const int occ = occupancy(ctx, h->mode, tp.n_lights > 0, Q_RAYS, smem);
    if (occ <= 0) return fail(RT_ERR_UNSUPPORTED, "no launch configuration of the rays trace kernel fits shared memory");
    const int grid = ctx->sm_count * occ;
    sub.grid = grid;
    sub.batches = n_batches;
    if ((rc = submission_start(W, st, tp, sub, tp.max_depth, (size_t)spb * n * 16)) != RT_OK) return rc;
    cudaEvent_t* ev = nullptr;
    if ((rc = submission_events(h, W, st, sub, &ev)) != RT_OK) return rc;
    unsigned int* counters = (unsigned int*)((char*)W.small.p + kStatBytes);
    for (uint32_t b = 0; b < n_batches; ++b) {
        TraceParams q = tp;
        const uint32_t first = b * (uint32_t)spb;
        q.s0 = tr.sample0 + first;
        q.s_count = (uint32_t)std::min<uint64_t>(spb, m - first);
        q.total_work = q.s_count * n;
        q.work_counter = counters + b;
        q.stack_stride = (uint32_t)grid * (uint32_t)kBlock;
        CU(cudaEventRecord(ev[2 + 2 * b], st));
        if (q.max_depth == 0) CU(cudaMemsetAsync(q.samplebuf, 0, (size_t)q.total_work * 16, st));   // ray_color(depth 0) = black, no ray
        else CU(launch_wavefront(q, h->mode, Q_RAYS, grid, smem, st));
        CU(cudaEventRecord(ev[3 + 2 * b], st));
        ResolveParams r{};
        r.samplebuf = q.samplebuf; r.accum = (float*)W.accum.p; r.npix_local = n;
        r.s_count = q.s_count; r.first = b == 0; r.last = b + 1 == n_batches; r.spp = m;
        r.out_linear = lin; r.out_rgb8 = rgb;
        CU(launch_resolve(r, st));
    }
    sub.launches = 2 * n_batches;
    if (tp.max_depth == 0) sub.black_samples = (uint64_t)n * m;
    return submission_close(h, W, st, sub);
}

// Both forms: the device form checks the memory kind of the caller's buffers and traces them on `stream_in`; the host form
// copies the rays into the context's query block, traces on the library's stream and copies the outputs back.
static int trace_rays_blocking(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_trace_params* p, float* lin,
                               uint8_t* rgb, void* stream_in, bool host, rt_stats* stats) {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_trace_rays(h, rays, n, p, lin, rgb);
    if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    auto wall0 = std::chrono::steady_clock::now();
    DeviceRestore restore;
    DeviceCtx* ctx = h->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    CU(cudaSetDevice(h->device));
    if (!host && (rc = check_device_ptrs(h, {{rays->origin, "rays->origin"}, {rays->direction, "rays->direction"},
                                             {lin, "dev_linear_f32"}, {rgb, "dev_rgb8"}})) != RT_OK)
        return rc;
    if ((rc = render_collect(h, nullptr)) != RT_OK) return rc;   // the handle's asynchronous frames first, like a blocking render
    rt_rays drays = *rays;
    float* dlin = lin;
    uint8_t* drgb = rgb;
    const uint64_t N = n;
    uint64_t h2d = 0, d2h = 0;
    if (host) {   // device image: origins, directions, linear, rgb8, 256-byte aligned (the last host-form user waited for it)
        auto al = [](uint64_t b) { return (b + 255) & ~(uint64_t)255; };
        CU(ctx->query.ensure(2 * al(N * 24) + (lin ? al(N * 12) : 0) + (rgb ? al(N * 3) : 0)));
        char* D = (char*)ctx->query.p;
        drays = rt_rays{(const double*)D, (const double*)(D + al(N * 24)), nullptr};
        char* o = D + 2 * al(N * 24);
        if (lin) { dlin = (float*)o; o += al(N * 12); }
        if (rgb) drgb = (uint8_t*)o;
        cudaStream_t st;
        CU(scene_stream(h, nullptr, &st));   // the stream the submission takes
        CU(cudaMemcpyAsync((void*)drays.origin, rays->origin, N * 24, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync((void*)drays.direction, rays->direction, N * 24, cudaMemcpyHostToDevice, st));
        h2d = N * 48;
    }
    cudaStream_t st = nullptr;
    if ((rc = trace_rays_enqueue(h, drays, n, *p, dlin, drgb, host ? nullptr : stream_in, &st)) != RT_OK) return rc;
    if (host) {
        if (lin) { CU(cudaMemcpyAsync(lin, dlin, N * 12, cudaMemcpyDeviceToHost, st)); d2h += N * 12; }
        if (rgb) { CU(cudaMemcpyAsync(rgb, drgb, N * 3, cudaMemcpyDeviceToHost, st)); d2h += N * 3; }
    }
    if ((rc = render_collect(h, stats)) != RT_OK) return rc;
    if (stats) {
        stats->h2d_bytes += h2d; stats->d2h_bytes += d2h;
        stats->wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    }
    return RT_OK;
}

int rtb200_scene_trace_rays_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_trace_params* params,
                                   float* dev_linear_f32, uint8_t* dev_rgb8, void* stream_in, rt_stats* stats) {
  return guarded([&]() -> int { return trace_rays_blocking(h, rays, n, params, dev_linear_f32, dev_rgb8, stream_in, false, stats); });
}

int rtb200_scene_trace_rays(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_trace_params* params,
                            float* out_linear_f32, uint8_t* out_rgb8, rt_stats* stats) {
  return guarded([&]() -> int { return trace_rays_blocking(h, rays, n, params, out_linear_f32, out_rgb8, nullptr, true, stats); });
}

// ---- adaptive rendering (DESIGN.md §4.9) ----
// The checks of rt_adaptive_params for a shard of npix_local pixels and a sample-buffer cap of `cap` bytes (no device is touched).
static int check_adaptive(const rt_adaptive_params* p, uint64_t npix_local, uint64_t cap) {
    if (!p) return fail(RT_ERR_INVALID, "null adaptive params");
    if (p->samples_per_round == 0) return fail(RT_ERR_INVALID, "samples_per_round must be > 0");
    if (p->min_samples == 0) return fail(RT_ERR_INVALID, "min_samples must be > 0");
    if (p->reserved != 0) return fail(RT_ERR_INVALID, "rt_adaptive_params.reserved must be 0");
    if (std::isnan(p->abs_tol) || std::isnan(p->rel_tol)) return fail(RT_ERR_INVALID, "abs_tol and rel_tol must not be NaN");
    const uint64_t work = (uint64_t)p->samples_per_round * npix_local;
    if (work >= (1ull << 31)) return fail(RT_ERR_INVALID, "samples_per_round * pixels must be below 2^31 (u32 work ids of a round)");
    if (work * 16 > cap) return fail(RT_ERR_INVALID, "samples_per_round * pixels * 16 bytes exceed the sample-buffer cap (rt_options.sample_buffer_bytes)");
    return RT_OK;
}

int rtb200_adaptive_begin(rtb200_scene_handle h, const rt_adaptive_params* p, void* stream_in) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    const uint32_t npl = h->tp.npix_local;
    int rc = check_adaptive(p, npl, sample_buffer_cap(h->opts));
    if (rc != RT_OK) return rc;
    DeviceRestore restore;
    std::lock_guard<std::recursive_mutex> lk(h->ctx->mu);
    CU(cudaSetDevice(h->device));
    auto& A = h->ad;
    A.begun = false;
    if (!A.mem && npl) {
        auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
        const size_t b3 = al((size_t)npl * 12), b1 = al((size_t)npl * 4), temp = adaptive_compact_bytes(npl);
        const size_t bytes = 2 * b3 + 4 * b1 + 256 + temp;
        void* m = nullptr;
        cudaError_t e = cudaMalloc(&m, bytes);
        if (e != cudaSuccess) { cudaGetLastError(); return fail(RT_ERR_OOM, "adaptive: cannot allocate " + std::to_string(bytes) + " bytes of device memory"); }
        e = cudaHostAlloc((void**)&A.active_host, 4, cudaHostAllocDefault);
        if (e != cudaSuccess) { cudaFree(m); A.active_host = nullptr; return fail_cuda(e, "cudaHostAlloc"); }
        char* c = (char*)m;
        A.mem = m;
        A.sum = (float*)c; c += b3;
        A.sq = (float*)c; c += b3;
        A.count = (uint32_t*)c; c += b1;   // sum, sq and count are contiguous: one memset clears them
        A.keep = (uint32_t*)c; c += b1;
        A.list[0] = (uint32_t*)c; c += b1;
        A.list[1] = (uint32_t*)c; c += b1;
        A.list_n = (uint32_t*)c; c += 256;
        A.temp = c; A.temp_bytes = temp;
    }
    cudaStream_t st;
    CU(scene_stream(h, stream_in, &st));
    if (npl) {
        CU(cudaMemsetAsync(A.sum, 0, (char*)A.keep - (char*)A.sum, st));
        CU(launch_adaptive_list(A.list[0], A.list_n, npl, st));
        CU(cudaStreamSynchronize(st));
    }
    A.p = *p;
    A.N = p->max_samples ? p->max_samples : h->tp.spp;
    A.n = 0; A.cur = 0; A.active = npl; A.updates = h->updates;
    A.begun = true;
    return RT_OK;
  });
}

// One submission of `rounds` rounds (DESIGN.md §4.9): per round a Q_LIST trace launch (a black memset at max_depth 0), the
// accumulate-and-test and the compaction into the other list buffer; then the active count is copied out and collected.
int rtb200_adaptive_step(rtb200_scene_handle h, uint32_t rounds, void* stream_in, uint32_t* active_out, rt_stats* stats) {
  return guarded([&]() -> int {
    if (stats) memset(stats, 0, sizeof *stats);
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    auto& A = h->ad;
    if (!A.begun) return fail(RT_ERR_INVALID, "no adaptive render on this handle: call rtb200_adaptive_begin");
    if (A.updates != h->updates) return fail(RT_ERR_INVALID, "the scene was updated since rtb200_adaptive_begin: the sums would mix two scenes (begin again)");
    auto wall0 = std::chrono::steady_clock::now();
    const uint32_t m = A.p.samples_per_round;
    const uint64_t left = A.active && A.n < A.N ? ((uint64_t)A.N - A.n + m - 1) / m : 0;   // rounds until every pixel has N
    rounds = (uint32_t)std::min<uint64_t>(rounds, left);
    if (active_out) *active_out = A.active;
    if (rounds == 0) return RT_OK;   // finished: nothing to do
    DeviceRestore restore;
    DeviceCtx* ctx = h->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    int rc = render_collect(h, nullptr);   // the handle's asynchronous frames first, like a blocking render
    if (rc != RT_OK) return rc;
    DeviceCtx::WorkSet& W = ctx->ws[0];
    cudaStream_t st;
    rtb200_scene_t::Submission sub;
    if ((rc = submission_open(h, stream_in, 1, &st, &sub)) != RT_OK) return rc;
    TraceParams tp = h->tp;
    const uint32_t npl = tp.npix_local;
    const size_t smem = wavefront_smem_bytes(tp, h->mode, tp.scene_in_smem, Q_LIST);
    const int occ = occupancy(ctx, h->mode, tp.n_lights > 0, Q_LIST, smem);
    if (occ <= 0) return fail(RT_ERR_UNSUPPORTED, "no launch configuration of the list trace kernel fits shared memory");
    const int grid = ctx->sm_count * occ;
    sub.grid = grid;
    sub.batches = rounds;
    if ((rc = submission_start(W, st, tp, sub, tp.max_depth, (size_t)m * npl * 16)) != RT_OK) return rc;
    cudaEvent_t* ev = nullptr;
    if ((rc = submission_events(h, W, st, sub, &ev)) != RT_OK) return rc;
    unsigned int* counters = (unsigned int*)((char*)W.small.p + kStatBytes);
    const bool black = tp.max_depth == 0;
    A.begun = false;   // until the rounds are enqueued: a step that fails part-way leaves the state unusable
    for (uint32_t r = 0; r < rounds; ++r) {
        TraceParams q = tp;
        q.s0 = A.n;
        q.s_count = std::min(m, A.N - A.n);
        q.total_work = 0;   // Q_LIST: n_list * s_count, n_list read on the device
        q.work_counter = counters + r;
        q.stack_stride = (uint32_t)grid * (uint32_t)kBlock;
        q.list = A.list[A.cur]; q.list_n = A.list_n + A.cur;
        CU(cudaEventRecord(ev[2 + 2 * r], st));
        if (black) CU(cudaMemsetAsync(q.samplebuf, 0, (size_t)q.s_count * npl * 16, st));   // ray_color(depth 0) = black, no ray
        else CU(launch_wavefront(q, h->mode, Q_LIST, grid, smem, st));
        CU(cudaEventRecord(ev[3 + 2 * r], st));
        AdaptiveParams a{};
        a.samplebuf = q.samplebuf; a.list = q.list; a.list_n = q.list_n;
        a.sum = A.sum; a.sq = A.sq; a.count = A.count; a.keep = A.keep;
        a.black_samples = black ? tp.stat + 3 : nullptr;
        a.npix_local = npl; a.s_count = q.s_count; a.n_after = A.n + q.s_count;
        a.max_samples = A.N; a.min_samples = A.p.min_samples; a.abs_tol = A.p.abs_tol; a.rel_tol = A.p.rel_tol;
        CU(launch_adaptive_accumulate(a, st));
        CU(launch_adaptive_compact(A.temp, A.temp_bytes, A.list[A.cur], A.keep, A.list[A.cur ^ 1u], A.list_n + (A.cur ^ 1u), npl, st));
        A.cur ^= 1u;
        A.n += q.s_count;
        sub.launches += 3;   // trace (or black memset), accumulate, compaction
    }
    CU(cudaMemcpyAsync(A.active_host, A.list_n + A.cur, 4, cudaMemcpyDeviceToHost, st));
    if ((rc = submission_close(h, W, st, sub)) != RT_OK) return rc;
    if ((rc = render_collect(h, stats)) != RT_OK) return rc;
    A.active = *A.active_host;
    A.begun = true;
    if (active_out) *active_out = A.active;
    if (stats) stats->wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    return RT_OK;
  });
}

int rtb200_adaptive_resolve(rtb200_scene_handle h, void* dev_rgb8, void* dev_linear_f32, void* dev_counts_u32, void* stream_in) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (!h->ad.begun) return fail(RT_ERR_INVALID, "no adaptive render on this handle: call rtb200_adaptive_begin");
    if (h->tp.npix_local == 0 || (!dev_rgb8 && !dev_linear_f32 && !dev_counts_u32)) return RT_OK;
    DeviceRestore restore;
    std::lock_guard<std::recursive_mutex> lk(h->ctx->mu);
    CU(cudaSetDevice(h->device));
    cudaStream_t st;
    CU(scene_stream(h, stream_in, &st));
    AdaptiveResolveParams r{};
    r.sum = h->ad.sum; r.count = h->ad.count; r.npix_local = h->tp.npix_local;
    r.out_linear = (float*)dev_linear_f32; r.out_rgb8 = (uint8_t*)dev_rgb8; r.out_count = (uint32_t*)dev_counts_u32;
    CU(launch_adaptive_resolve(r, st));
    CU(cudaStreamSynchronize(st));
    return RT_OK;
  });
}

int rtb200_render_adaptive(const rt_scene* s, const rt_options* opts_in, const rt_adaptive_params* p, uint8_t* out_rgb8,
                           float* out_lin, uint32_t* out_counts, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!s) return fail(RT_ERR_INVALID, "null argument");
    rt_options opts;
    int rc = normalise_options(opts_in, &opts);
    if (rc != RT_OK) return rc;
    uint32_t n_lights = 0;
    if ((rc = validate_scene(s, &n_lights)) != RT_OK) return rc;
    const uint64_t npl = (uint64_t)rtb200_shard_rows(s->height, opts.rank, opts.world, opts.band_rows) * s->width;
    if ((rc = check_adaptive(p, npl, sample_buffer_cap(opts))) != RT_OK) return rc;
    auto wall0 = std::chrono::steady_clock::now();
    DeviceRestore restore;
    rtb200_scene_handle h = nullptr;
    if ((rc = rtb200_scene_upload(s, &opts, &h)) != RT_OK) return rc;
    ReleaseGuard rel{h};
    DeviceCtx* ctx = h->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    CU(cudaSetDevice(h->device));
    rt_stats st{};
    uint32_t active = 0;
    if ((rc = rtb200_adaptive_begin(h, p, nullptr)) != RT_OK) return rc;
    if ((rc = rtb200_adaptive_step(h, 0xffffffffu, nullptr, &active, &st)) != RT_OK) return rc;
    void *d8 = nullptr, *dl = nullptr, *dc = nullptr;
    if (out_rgb8) { CU(ctx->out_rgb8.ensure(npl * 3 + 16)); d8 = ctx->out_rgb8.p; }
    if (out_lin) { CU(ctx->out_lin.ensure(npl * 12 + 16)); dl = ctx->out_lin.p; }
    if (out_counts) { CU(ctx->out_cnt.ensure(npl * 4 + 16)); dc = ctx->out_cnt.p; }
    if ((rc = rtb200_adaptive_resolve(h, d8, dl, dc, nullptr)) != RT_OK) return rc;
    if (npl) {
        if (out_rgb8) CU(cudaMemcpyAsync(out_rgb8, d8, npl * 3, cudaMemcpyDeviceToHost, ctx->stream));
        if (out_lin) CU(cudaMemcpyAsync(out_lin, dl, npl * 12, cudaMemcpyDeviceToHost, ctx->stream));
        if (out_counts) CU(cudaMemcpyAsync(out_counts, dc, npl * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    }
    st.frames = 1;
    st.h2d_bytes += h->h2d_bytes;
    st.d2h_bytes = (out_rgb8 ? npl * 3 : 0) + (out_lin ? npl * 12 : 0) + (out_counts ? npl * 4 : 0) + 128 + 16 + 4;
    st.wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    if (stats) *stats = st;
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
    DeviceRestore restore;
    std::lock_guard<std::recursive_mutex> lk(h->ctx->mu);
    CU(cudaSetDevice(h->device));
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

// Host buffers: upload the scene, render `frames` into the context's output buffers, copy them to the host and release the
// scene. The single-frame calls pass the scene's own view as one frame.
static int render_host(const rt_scene* s, const rt_options* opts_in, const rt_frame* frames, uint32_t n_frames, uint8_t* out_rgb8,
                       float* out_lin, rt_stats* stats) {
    rt_options opts;
    int rc = normalise_options(opts_in, &opts);
    if (rc != RT_OK) return rc;
    uint32_t n_lights = 0;
    if ((rc = validate_scene(s, &n_lights)) != RT_OK) return rc;
    if ((rc = check_frames(frames, n_frames, rtb200_shard_rows(s->height, opts.rank, opts.world, opts.band_rows), s->width)) != RT_OK) return rc;
    auto wall0 = std::chrono::steady_clock::now();
    DeviceRestore restore;
    rtb200_scene_handle h = nullptr;
    if ((rc = rtb200_scene_upload(s, &opts, &h)) != RT_OK) return rc;
    ReleaseGuard rel{h};
    DeviceCtx* ctx = h->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    CU(cudaSetDevice(h->device));
    const size_t total = (size_t)n_frames * h->tp.npix_local;   // pixels of all frames
    void *d8 = nullptr, *dl = nullptr;
    if (out_rgb8) { CU(ctx->out_rgb8.ensure(total * 3 + 16)); d8 = ctx->out_rgb8.p; }
    if (out_lin) { CU(ctx->out_lin.ensure(total * 12 + 16)); dl = ctx->out_lin.p; }
    rt_stats st{};
    if ((rc = render_blocking(h, frames, n_frames, d8, dl, nullptr, &st)) != RT_OK) return rc;
    if (total) {
        if (out_rgb8) CU(cudaMemcpyAsync(out_rgb8, d8, total * 3, cudaMemcpyDeviceToHost, ctx->stream));
        if (out_lin) CU(cudaMemcpyAsync(out_lin, dl, total * 12, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    }
    st.h2d_bytes += h->h2d_bytes;
    st.d2h_bytes = (out_rgb8 ? total * 3 : 0) + (out_lin ? total * 12 : 0) + 128 + 16;
    st.wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    if (stats) *stats = st;
    return RT_OK;
}

int rtb200_render_rgb8(const rt_scene* scene, const rt_options* opts, uint8_t* out_rgb8, rt_stats* stats) {
    if (!scene || !out_rgb8) return fail(RT_ERR_INVALID, "null argument");
    const rt_frame f{scene->camera, scene->seed, scene->max_depth, 0};
    return guarded([&]() -> int { return render_host(scene, opts, &f, 1, out_rgb8, nullptr, stats); });
}
int rtb200_render_linear_f32(const rt_scene* scene, const rt_options* opts, float* out_rgb, rt_stats* stats) {
    if (!scene || !out_rgb) return fail(RT_ERR_INVALID, "null argument");
    const rt_frame f{scene->camera, scene->seed, scene->max_depth, 0};
    return guarded([&]() -> int { return render_host(scene, opts, &f, 1, nullptr, out_rgb, stats); });
}

int rtb200_render_frames(const rt_scene* s, const rt_options* opts_in, const rt_frame* frames, uint32_t n_frames, uint8_t* out_rgb8,
                         float* out_lin, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!s) return fail(RT_ERR_INVALID, "null argument");
    if (!out_rgb8 && !out_lin) return fail(RT_ERR_INVALID, "out_rgb8 and out_linear_f32 are both null");
    return render_host(s, opts_in, frames, n_frames, out_rgb8, out_lin, stats);
  });
}

// One process, n_gpus devices: the reference's row bands (raytracer.rs:254-262) dealt round-robin to the devices (band b ->
// device b mod G, like the torchrun flavour in rtb200/dist.py). The hierarchy is built once; one host thread per device
// uploads the scene, enqueues trace + resolve, copies its compact shard peer-to-peer over NVLink straight into its interleaved
// rows of the frame on the first device and waits for its stream; then ONE device->host copy.
static std::mutex g_multi_mu;   // multi-GPU calls take turns (they share the frame buffer of the first device)

int rtb200_render_rgb8_multi(const rt_scene* s, const rt_options* opts_in, int32_t n_gpus, uint8_t* out_rgb8, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!s || !out_rgb8) return fail(RT_ERR_INVALID, "null argument");
    auto wall0 = std::chrono::steady_clock::now();
    rt_options base;
    int rc = normalise_options(opts_in, &base);
    if (rc != RT_OK) return rc;
    if (base.world != 1 || base.rank != 0) return fail(RT_ERR_INVALID, "rtb200_render_rgb8_multi shards the frame itself: opts->rank/world must be 0/1");
    uint32_t n_lights = 0;
    if ((rc = validate_scene(s, &n_lights)) != RT_OK) return rc;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess) return fail_cuda(e, "cudaGetDeviceCount");
    if (count <= 0) return fail(RT_ERR_NO_DEVICE, "no CUDA device");
    const int first = base.device < 0 ? 0 : base.device;
    if (first >= count) return fail(RT_ERR_NO_DEVICE, "no such CUDA device");
    int G = n_gpus <= 0 ? count - first : std::min(n_gpus, count - first);
    G = std::min(G, 64 - first);   // device contexts exist for ordinals below 64
    const uint32_t bands = (s->height + base.band_rows - 1) / base.band_rows;
    G = (int)std::min<uint32_t>((uint32_t)G, bands);   // a device needs at least one band
    if (G <= 1) {
        base.device = first;
        const rt_frame f{s->camera, s->seed, s->max_depth, 0};
        return render_host(s, &base, &f, 1, out_rgb8, nullptr, stats);
    }

    DeviceRestore restore;
    std::lock_guard<std::mutex> multi_lock(g_multi_mu);
    rtbvh::Records R;
    rtbvh::build_records(s, mode_of(base.variant) == MODE_TREE, R);
    const size_t row_bytes = (size_t)s->width * 3;
    // the frame lives on the first device; peers get access both ways once per process (without it the copies stage through the host)
    DeviceCtx* c0 = nullptr;
    if ((rc = get_ctx(first, &c0)) != RT_OK) return rc;
    uint8_t* frame = nullptr;
    {
        std::lock_guard<std::recursive_mutex> lk(c0->mu);
        CU(c0->frame.ensure((size_t)s->height * row_bytes + 16));
        frame = (uint8_t*)c0->frame.p;
        static bool peered[64] = {false};
        for (int g = 1; g < G; ++g) {
            if (peered[first + g]) continue;
            cudaSetDevice(first); if (cudaDeviceEnablePeerAccess(first + g, 0) != cudaSuccess) cudaGetLastError();
            cudaSetDevice(first + g); if (cudaDeviceEnablePeerAccess(first, 0) != cudaSuccess) cudaGetLastError();
            peered[first + g] = true;
        }
    }
    struct Result { int rc = RT_OK; std::string err; rt_stats st{}; uint64_t h2d = 0; };
    std::vector<Result> res((size_t)G);
    auto worker = [&](int g) {
        Result& r = res[(size_t)g];
        auto body = [&]() -> int {
            rt_options o = base; o.device = first + g; o.rank = g; o.world = G;
            rtb200_scene_handle h = nullptr;
            int rcw = scene_upload_records(s, o, n_lights, R, &h);
            if (rcw != RT_OK) return rcw;
            ReleaseGuard rel{h};
            DeviceCtx* c = h->ctx;
            std::lock_guard<std::recursive_mutex> lk(c->mu);
            CU(cudaSetDevice(first + g));
            const size_t rows = h->tp.rows_local;
            CU(c->out_rgb8.ensure(rows * row_bytes + 16));
            const rt_frame f = own_frame(h);
            if ((rcw = render_enqueue(h, &f, 1, c->out_rgb8.p, nullptr, nullptr, 0)) != RT_OK) return rcw;
            // shard -> frame: full bands as one strided 2-D copy (a "row" of the copy = one band), then the partial last band
            const size_t band_bytes = (size_t)base.band_rows * row_bytes;
            const size_t full = rows / base.band_rows, rem = rows - full * base.band_rows;
            if (full) CU(cudaMemcpy2DAsync(frame + (size_t)g * band_bytes, (size_t)G * band_bytes, c->out_rgb8.p, band_bytes, band_bytes, full, cudaMemcpyDefault, c->stream));
            if (rem) CU(cudaMemcpyAsync(frame + ((size_t)full * G + g) * band_bytes, (uint8_t*)c->out_rgb8.p + full * band_bytes, rem * row_bytes, cudaMemcpyDefault, c->stream));
            if ((rcw = render_collect(h, &r.st)) != RT_OK) return rcw;   // waits for the stream: the shard is in the frame
            r.h2d = h->h2d_bytes;
            return RT_OK;
        };
        r.rc = guarded(body);
        if (r.rc != RT_OK) r.err = g_last_error;
    };
    std::vector<std::thread> threads;
    threads.reserve((size_t)G);
    struct Joiner { std::vector<std::thread>& ts; ~Joiner() { for (auto& t : ts) if (t.joinable()) t.join(); } };
    {
        Joiner joiner{threads};   // also on the exceptional path (thread creation can throw): never destroy a joinable thread
        for (int g = 1; g < G; ++g) threads.emplace_back(worker, g);
        worker(0);
    }
    for (int g = 0; g < G; ++g) if (res[(size_t)g].rc != RT_OK) return fail(res[(size_t)g].rc, "device " + std::to_string(first + g) + ": " + res[(size_t)g].err);
    rt_stats total{};
    for (int g = 0; g < G; ++g) {
        const rt_stats& st = res[(size_t)g].st;
        total.rays += st.rays; total.samples += st.samples; total.candidates += st.candidates; total.clusters += st.clusters; total.nodes += st.nodes;
        total.device_ms = std::max(total.device_ms, st.device_ms); total.trace_ms = std::max(total.trace_ms, st.trace_ms);
        total.kernel_launches += st.kernel_launches; total.batches = std::max(total.batches, st.batches);
        total.h2d_bytes += res[(size_t)g].h2d;
    }
    {
        std::lock_guard<std::recursive_mutex> lk(c0->mu);
        CU(cudaSetDevice(first));
        CU(cudaMemcpyAsync(out_rgb8, frame, (size_t)s->height * row_bytes, cudaMemcpyDeviceToHost, c0->stream));
        CU(cudaStreamSynchronize(c0->stream));
    }
    total.frames = 1; total.gpus_used = G;
    total.d2h_bytes = (size_t)s->height * row_bytes + (size_t)G * (128 + 16);
    total.wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    if (stats) *stats = total;
    return RT_OK;
  });
}

}  // extern "C"

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
    void* din = c->probe.p;
    void* dout = (char*)c->probe.p + ((in_bytes + 255) / 256) * 256;
    CU(cudaMemsetAsync(dout, 0, out_bytes, c->stream));
    if (in_bytes) CU(cudaMemcpyAsync(din, in, in_bytes, cudaMemcpyHostToDevice, c->stream));
    CU(launch(din, dout, c->stream));
    CU(cudaMemcpyAsync(out, dout, out_bytes, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return RT_OK;
}

extern "C" {

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

}  // extern "C"
