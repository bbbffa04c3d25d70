// rtb200_host.cuh — what the host translation units of the C ABI share (rtb200_api.cu, rtb200_api_render.cu,
// rtb200_api_scene.cu, rtb200_api_query.cu, rtb200_api_denoise.cu, rtb200_api_temporal.cu): error reporting, the per-device contexts, the scene
// handle and the helpers more than one of them calls. Not installed.
#pragma once
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "rtb200_bvh.hpp"
#include "rtb200_kernels.cuh"

namespace rtk {

extern thread_local std::string g_last_error;

int fail(int code, const std::string& msg);
int fail_cuda(cudaError_t e, const char* what);
#define CU(call)                                              \
    do {                                                      \
        cudaError_t e__ = (call);                             \
        if (e__ != cudaSuccess) return fail_cuda(e__, #call); \
    } while (0)

// refusal texts that more than one check gives
constexpr const char* kErrSpheres = "2^26 or more spheres (list entries carry 27-bit ids)";
constexpr const char* kErrLights = "10 or more lights: the reference's light recursion (raytracer.rs:99-114) does not terminate when n_lights * 0.1 >= 1";

// No C++ exception may unwind through the C boundary (std::bad_alloc while building the hierarchy of a huge scene, ...).
template <typename F>
int guarded(F&& f) {
    try { return f(); }
    catch (const std::bad_alloc&) { return fail(RT_ERR_OOM, "host memory allocation failed"); }
    catch (const std::exception& e) { return fail(RT_ERR_INVALID, std::string("internal error: ") + e.what()); }
    catch (...) { return fail(RT_ERR_INVALID, "internal error: unknown exception"); }
}

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
        GrowBuf samplebuf, accum, stack, small, frames, lterm, ftab, ltab;   // ftab / ltab: the multi-frame kernel's frame and lens tables
        GrowBuf accum_sq;   // the resolve's sums of squares, grown only by a render with a variance output
        cudaEvent_t done = nullptr;
    } ws[2];
    GrowBuf out_rgb8, out_lin, out_cnt, out_var, probe, frame;
    // scene arenas of released handles, kept for the next upload (a per-frame upload costs no cudaMalloc / cudaFree)
    struct Arena { void* p; size_t cap; };
    std::vector<Arena> arena_cache;
    std::vector<cudaEvent_t> event_pool;  // timing events of released handles (creating four events per one-shot render costs more than the upload)
    struct OccKey { uint32_t mode; bool lights; uint32_t queue; size_t smem; int occ; };
    std::vector<OccKey> occ_cache;        // cudaOccupancyMaxActiveBlocksPerMultiprocessor answers
    PinnedBuf staging;                    // host image of the arena being uploaded
    cudaEvent_t staging_free = nullptr;   // the last H2D copy out of `staging` has finished
    // the host forms of rtb200_scene_intersect, _occluded, _nearest, _overlaps, _trace_rays, _aov, rtb200_denoise and rtb200_temporal:
    // their arrays on the device (HostStage), host_call's timing events (created at its first call), and the resident CTAs per SM of
    // the query kernel of each kind and mode (0: not asked yet)
    GrowBuf query;
    cudaEvent_t query_ev[4] = {nullptr, nullptr, nullptr, nullptr};
    int query_occ[6][3] = {};   // [closest-hit, occlusion, auxiliary buffers, lens ones, nearest, overlaps][mode]
};
// the context of a device ordinal below 64, created at its first use
int get_ctx(int device, DeviceCtx** out);

// RAII: restores the caller's current device (the ABI must not leave cudaSetDevice changed behind the caller's back)
struct DeviceRestore {
    int prev = -1;
    DeviceRestore() { if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; } }
    ~DeviceRestore() { if (prev >= 0) cudaSetDevice(prev); }
};

// The prologue of an entry point on handle h, after its argument checks (a refusal never waits for a CUDA call): the
// caller's current device is restored on return, the context's lock is held until then, and h's device is made current.
#define HANDLE_PROLOGUE(h)                                           \
    DeviceRestore restore_;                                          \
    std::lock_guard<std::recursive_mutex> lock_((h)->ctx->mu);       \
    CU(cudaSetDevice(h->device))

// The same for an entry point on a device ordinal (-1: the current device): declares `ctx`, the device's context, which
// get_ctx has made current.
#define CTX_PROLOGUE(device, ctx)                                    \
    DeviceRestore restore_;                                          \
    DeviceCtx* ctx = nullptr;                                        \
    if (int rc_ = get_ctx(device, &ctx); rc_ != RT_OK) return rc_;   \
    std::lock_guard<std::recursive_mutex> lock_(ctx->mu)

// The stream of a call on ctx's device: `stream_in`, or the context's stream for NULL
inline cudaStream_t call_stream(const DeviceCtx* ctx, void* stream_in) { return stream_in ? (cudaStream_t)stream_in : ctx->stream; }

// A caller's array in an argument check: its bytes, its name in a refusal and the alignment the device form needs
struct Range { const void* p; uint64_t bytes; const char* name; uintptr_t align; };
inline bool overlap(const Range& a, const Range& b) {
    if (!a.p || !b.p || !a.bytes || !b.bytes) return false;
    const uintptr_t a0 = (uintptr_t)a.p, b0 = (uintptr_t)b.p;
    return a0 < b0 + b.bytes && b0 < a0 + a.bytes;
}

inline double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace rtk

struct rtb200_scene_t {
    int device = -1;
    rtk::DeviceCtx* ctx = nullptr;
    rtk::TraceParams tp{};
    rt_options opts{};
    uint32_t mode = rtk::MODE_TREE;
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
    // What one submission put on a stream. Events: begin, end, and a pair around each trace launch (or black memset).
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
    rtk::GrowBuf upd_in;                 // host form's input: geo, materials, indices (an edit's: remove, at, geo, materials)
    // ---- edited list (rtb200_scene_edit_spheres, DESIGN.md §4.13): one device block for up to cap spheres, allocated at the
    // first edit and replaced by a larger one when an edit needs more. The list lives in half ed_cur (-1: still in the upload
    // arena) and the next edit writes the other half: frames enqueued before an edit keep reading the arrays they were
    // enqueued with ----
    struct EditBlock {
        void* mem = nullptr;
        uint32_t cap = 0;
        struct Half { double4* geo; rtk::DevMat* mat; float* filt; uint32_t* lights; } half[2] = {};   // filt: MODE_BRUTE only
        uint32_t* skip_pos = nullptr;    // cap x kNoSkip: the skip_pos of a list without a hierarchy
        uint32_t* keep = nullptr;        // cap + 1 words each: the keep flags of the old list and their scan
        uint32_t* pos = nullptr;
        void* temp = nullptr;            // cub's scan scratch
        size_t temp_bytes = 0;
    } ed;
    int ed_cur = -1;
    uint32_t updates = 0;                // rtb200_scene_update_* and _edit_spheres calls so far: an adaptive render refuses to step across one
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

namespace rtk {

// ---- rtb200_api.cu ----
// bytes of per-sample radiance one launch may stage (rt_options.sample_buffer_bytes, 0: 1 GiB)
inline uint64_t sample_buffer_cap(const rt_options& o) { return o.sample_buffer_bytes ? o.sample_buffer_bytes : (1ull << 30); }
// Samples per batch when `samples` samples of each of `items` pixels or rays are due: as many as the sample buffer (`cap`
// bytes) holds, and fewer than 2^31 work ids in a batch.
uint32_t samples_per_batch(uint64_t cap, uint64_t items, uint32_t samples);
int normalise_options(const rt_options* opts_in, rt_options* o);
// RT_ERR_INVALID (message prefixed by `what`) unless the lens's u, v and radius are finite, radius >= 0 and reserved is 0
int check_lens(const rt_lens& L, const char* what);
int validate_scene(const rt_scene* s, uint32_t* n_lights_out);
uint32_t mode_of(uint32_t variant);
bool albedo_nonfinite(const rt_sphere& sp);
// The host-side records of s for the variant of opts (a hierarchy in MODE_TREE only)
void scene_records(const rt_scene* s, const rt_options& opts, rtbvh::Records& R);
// `R` holds the host-side records (built once; the multi-GPU entry point shares them between its devices)
int scene_upload_records(const rt_scene* s, const rt_options& opts, uint32_t n_lights, const rtbvh::Records& R, rtb200_scene_t** out);
// The stream of a call on h, `stream_in` (NULL: the context's stream), made to wait for what last wrote the scene arrays:
// the upload, which ran on the context's stream, and the last update or rebuild, on whichever stream it ran.
cudaError_t scene_stream(rtb200_scene_t* h, void* stream_in, cudaStream_t* out);
// RT_ERR_INVALID unless every non-null pointer of `ptrs` (pointer, name) is device memory of `device` or managed memory.
// The caller has made that device current.
int check_device_ptrs(int device, const std::vector<std::pair<const void*, const char*>>& ptrs);
// the same for h's device
int check_device_ptrs(rtb200_scene_t* h, const std::vector<std::pair<const void*, const char*>>& ptrs);

// ---- rtb200_api_render.cu ----
// The launch geometry of h's trace kernel on `queue`, with or without lights: its dynamic shared memory, and the persistent
// grid of every SM's resident CTAs.
struct LaunchGeom { size_t smem; int ctas_per_sm, grid; };
int launch_geometry(rtb200_scene_t* h, uint32_t queue, bool lights, LaunchGeom* g);
// Wait for the pending submissions of h and report them (stats may be NULL).
int render_collect(rtb200_scene_t* h, rt_stats* stats);

// The host form of a call on caller-supplied arrays (closest-hit, occlusion, trace_rays, aov, denoise, temporal): the device
// images of the caller's host arrays in the context's query block, after `head` bytes the call keeps for itself, in the order
// they were added, each at a 256-byte boundary (an array of 0 bytes has none: a null dev). The last host-form call waited for
// its stream, so the block is free. copy enqueues the inputs' copies to the device, or with `back` the outputs' to the host;
// h2d and d2h count them.
struct HostStage {
    struct Array { const void* in; void* out; uint64_t bytes; char* dev; };
    Array a[13];
    int n = 0;
    uint64_t h2d = 0, d2h = 0;
    void add_in(const void* host, uint64_t bytes) { a[n++] = Array{host, nullptr, bytes, nullptr}; }
    void add_out(void* host, uint64_t bytes) { a[n++] = Array{nullptr, host, bytes, nullptr}; }
    int place(DeviceCtx* ctx, size_t head);
    int copy(cudaStream_t st, bool back);
};

// The blocking host form of a call whose wall clock started at wall0, on `st` of ctx's device (made current, ctx->mu held): io's
// arrays are staged through the query block, `launch(stat)` enqueues the call on their device images, the outputs are copied
// back and the stream is waited for. With `hstat`, the image starts with a counter block (kStatBytes; the guard counters at
// [30..31]), cleared before the inputs are copied in and read back into hstat after the outputs; `stat` is its device image
// (else NULL), and a trip of the traversal guard refuses with `guard_trip`. Fills the times and byte counts of stats (may be
// NULL); the caller adds its own counters.
template <typename Launch>
int host_call(DeviceCtx* ctx, cudaStream_t st, HostStage& io, unsigned long long* hstat, const char* guard_trip,
              std::chrono::steady_clock::time_point wall0, rt_stats* stats, Launch&& launch) {
    for (auto& e : ctx->query_ev) if (!e) CU(cudaEventCreate(&e));
    int rc = io.place(ctx, hstat ? kStatBytes : 0);
    if (rc != RT_OK) return rc;
    unsigned long long* stat = hstat ? (unsigned long long*)ctx->query.p : nullptr;
    cudaEvent_t* ev = ctx->query_ev;
    CU(cudaEventRecord(ev[0], st));
    if (stat) CU(cudaMemsetAsync(stat, 0, kStatBytes, st));
    if ((rc = io.copy(st, false)) != RT_OK) return rc;
    CU(cudaEventRecord(ev[1], st));
    if ((rc = launch(stat)) != RT_OK) return rc;
    CU(cudaEventRecord(ev[2], st));
    if ((rc = io.copy(st, true)) != RT_OK) return rc;
    if (stat) CU(cudaMemcpyAsync(hstat, stat, kStatBytes, cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(ev[3], st));
    CU(cudaStreamSynchronize(st));
    if (hstat && hstat[31] != 0) return fail(RT_ERR_CUDA, guard_trip);
    if (!stats) return RT_OK;
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, ev[0], ev[3])); stats->device_ms = ms;
    CU(cudaEventElapsedTime(&ms, ev[1], ev[2])); stats->trace_ms = ms;
    stats->h2d_bytes = io.h2d; stats->d2h_bytes = (stat ? kStatBytes : 0) + io.d2h;
    stats->wall_ms = ms_since(wall0);
    return RT_OK;
}

}  // namespace rtk
