// rtb200_kernels.cuh — parameter blocks and launch wrappers shared by the kernels and the host code of the C ABI
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/rtb200.h"
#include "rtb200_bvh.hpp"
#include "rtb200_device.cuh"

namespace rtk {

// the scene's layout is rtbvh's (rtb200_bvh.hpp)
using rtbvh::kLeafK;                                // sphere slots per BVH leaf
constexpr int kNodeVec = rtbvh::kNodeFloats / 4;    // float4 per 8-wide BVH node
constexpr int kChildVec = rtbvh::kChildOff / 4;     // float4 offset of a node's child words
using DevMat = rtbvh::Mat32;                         // 32-byte material record

#ifndef RT_BLOCK
#define RT_BLOCK 256
#endif
constexpr int kBlock = RT_BLOCK;   // threads (= ray slots) per CTA of the trace kernel
#ifndef RT_PHASE_CLOCKS
#define RT_PHASE_CLOCKS 0          // 1: the trace kernel accounts its stages per warp (Makefile target `phase`, RTB200_PRINT_PHASES)
#endif
// stat[kPhaseStat + k] of an RT_PHASE_CLOCKS build: clock64() cycles of each stage summed over warps (k < PH_ITERS), warp
// iterations, diffuse / metal vertices shaded (scatter attempts), and those of them whose scatter sample was deferred; then
// the cycles of closest-hit's node, leaf and exact steps (part of PH_HIT), the exact steps, the (ray, sphere) tests they
// ran, and the source spheres the node and leaf steps left out because the certificate proved the exact test rejects them
enum : uint32_t { PH_HIT, PH_SORT_WAIT_A, PH_SHADE, PH_REGEN, PH_WAIT_C, PH_ITERS, PH_SCATTERS, PH_DEFERRED,
                  PH_NODE, PH_LEAF, PH_EXACT, PH_EXACT_STEPS, PH_EXACT_TESTS, PH_SRC_SKIPS, kPhaseN };
constexpr uint32_t kPhaseStat = 13;
// per-warp work lists of the closest-hit stage (entries: id << 5 | ray lane)
#ifndef RT_CAP_IN
#define RT_CAP_IN 192
#endif
#ifndef RT_CAP_LF
#define RT_CAP_LF 160
#endif
#ifndef RT_CAP_CD
#define RT_CAP_CD 96
#endif
constexpr int kCapIn = RT_CAP_IN;   // (ray, inner node) pairs: LIFO stack; 7*depth+8 entries are reserved for single-entry descents
constexpr int kCapLf = RT_CAP_LF;   // (ray, leaf) pairs
constexpr int kCapCd = RT_CAP_CD;   // (ray, sphere) pairs awaiting the exact f64 test

// One pending light test (raytracer.rs:99-114): the vertex it belongs to and the partial sum over the lights.
struct ShadowFrame {
    double px, py, pz;      // hit point = origin of the shadow rays and of the scattered ray
    double ndx, ndy, ndz;   // scattered direction (continuation of the main path)
    float ar, ag, ab;       // albedo of the vertex
    float sr, sg, sb;       // sum over lights of albedo * ray_color(light_ray, 2, 1)
    uint32_t li, code, is_light, pad;
};
static_assert(sizeof(ShadowFrame) == 88, "ShadowFrame layout");

enum TraceMode : uint32_t { MODE_TREE = 0, MODE_BRUTE = 1, MODE_EXACT = 2 };
// The work queue of a trace launch: every pixel of one frame, every pixel of several frames (TraceParams::ftab), the
// pixels of an adaptive render's list (TraceParams::list, DESIGN.md §4.9), or caller-supplied primary rays
// (TraceParams::ray_o / ray_d, rtb200_scene_trace_rays, DESIGN.md §4.12)
// Q_FRAMES_LENS and Q_LIST_LENS are Q_FRAMES and Q_LIST with a thin lens (DESIGN.md §4.17): the lens is a compile-time choice,
// so that the pinhole kernels carry no lens code.
enum TraceQueue : uint32_t { Q_SINGLE = 0, Q_FRAMES = 1, Q_LIST = 2, Q_RAYS = 3, Q_FRAMES_LENS = 4, Q_LIST_LENS = 5 };
__host__ __device__ constexpr uint32_t base_queue(uint32_t q) { return q == Q_FRAMES_LENS ? Q_FRAMES : q == Q_LIST_LENS ? Q_LIST : q; }

// One frame of a multi-frame launch (rt_wavefront_kernel<.., Q_FRAMES>): the view and the Philox key that replace
// TraceParams::cam / key0 / key1 for the work ids of that frame.
struct FrameRec { rt_camera cam; uint32_t key0, key1; };
static_assert(sizeof(FrameRec) == 104, "FrameRec layout");

struct TraceParams {
    // ---- scene, resident in HBM (built by rtbvh::build_records) ----
    const float4*   nodes;       // n_nodes * kNodeVec: lo_x[8] lo_y[8] lo_z[8] hi_x[8] hi_y[8] hi_z[8] child[8], f32 boxes rounded outwards
    const float4*   leaf_rec;    // n_leaves * kLeafK float4: kLeafK/2 pair-packed sphere records {cx0,cx1,cy0,cy1},{cz0,cz1,nk0,nk1}
    const uint32_t* leaf_id;     // n_leaves * kLeafK: slot -> ORIGINAL sphere index (rtbvh::kPadId = padding)
    const uint32_t* skip_pos;    // n: where the traversal can leave the sphere out (rtbvh::Records::skip_pos)
    const uint32_t* always;      // n_always sphere indices tested in f64 for every ray (not representable in the f32 frame)
    const float4*   filt;        // n_pairs * 2 float4: every sphere in list order, pair-packed (MODE_BRUTE)
    const double4*  geo;         // n: {cx,cy,cz,radius} exact f64
    const DevMat*   mat;         // n
    const rtd::DevTex* tex;      // n_tex
    uint32_t n, n_pairs, n_nodes, n_leaves, n_always, depth;
    uint32_t n_lights;
    uint32_t scene_in_smem;      // bit0: nodes + leaves (MODE_TREE) / flat records (MODE_BRUTE), bit1: geo, bit2: mat staged into shared memory
    double gx, gy, gz;           // recentring offset of the f32 frame
    float  er_coef;              // per-ray error coefficient of the sphere test (DESIGN.md "filter soundness")
    rt_camera cam;
    uint32_t width, height, spp, max_depth;
    uint32_t sky_mode;
    rtd::DevTex sky;
    uint32_t key0, key1;         // Philox key = seed
    // ---- work of this launch: samples [s0, s0+s_count) of every pixel of the shard ----
    uint32_t s0, s_count;
    uint32_t npix_local, rows_local;
    int32_t  rank, world;
    uint32_t band_rows;
    uint32_t total_work;         // npix_local * s_count
    unsigned int* work_counter;
    float4*  samplebuf;          // [s_count][npix_local] per-sample radiance (w = rays of the sample)
    uint32_t* stack;             // [max_depth][stack_stride] per-slot albedo codes (levels beyond the shared-memory part)
    uint32_t stack_stride;
    const uint32_t* lights;      // sphere indices of the Light spheres in list order (find_lights, raytracer.rs:220-229)
    ShadowFrame* frames;         // [max_shadow][stack_stride], only when n_lights > 0
    uint32_t max_shadow;         // nested light-test frames per path (a level nests with probability <= n_lights*0.1)
    float* lterm;                // [2 levels][3][stack_stride] light terms of the first two path levels
    unsigned long long* stat;    // per frame: [0]=rays [1]=f64 tests [2]=all-spheres fallbacks [3]=samples [4]=leaf visits [6]=node visits, [8..12] frame tail, [kPhaseStat..] phase clocks
    unsigned long long* err;     // per scene handle, accumulated over frames: [0]=shadow-frame-stack overflows [1]=traversal guard trips (must stay 0)
    // ---- multi-frame launches only (appended, so that the fields above keep their offsets) ----
    const FrameRec* ftab;        // [frames of the launch]: work id w belongs to frame w / frame_work
    union {
        uint32_t frame_work;     // Q_FRAMES: work ids per frame = s_count * npix_local; total_work = frames * frame_work
        uint32_t stream0;        // Q_RAYS: ray i draws from the RNG stream of pixel stream0 + i
    };
    // ---- appended after the multi-frame fields ----
    // 1: a Lambertian or Metal sphere has, or once had, an infinite or NaN albedo component. A black path then has to unwind
    // its albedo stack, and a nested shadow vertex has to read its albedo, because albedo * 0 is NaN for such an albedo.
    uint32_t albedo_nonfinite;
    // ---- Q_LIST launches only (appended after albedo_nonfinite) ----
    // Q_RAYS launches share these slots (a queue reads only its own member): appending the ray arrays instead would move the
    // fields that QueryParams and OcclusionParams place after their TraceParams, and with them the query kernels' code.
    // Q_RAYS: npix_local is the number of rays n; work id w is ray w % n, sample s0 + w / n, samplebuf index w.
    union {
        const uint32_t* list;    // Q_LIST: local pixel indices, increasing; samplebuf is [s_count][n_list]
        const double* ray_o;     // Q_RAYS: [n][3] ray origins
    };
    union {
        const uint32_t* list_n;  // Q_LIST: device: n_list, read once at kernel start; total_work = n_list * s_count
        const double* ray_d;     // Q_RAYS: [n][3] ray directions
    };
    // ---- the thin lens (DESIGN.md §4.17), appended after the Q_LIST fields ----
    rt_lens lens;                // the handle's lens (radius 0: pinhole); read by Q_LIST_LENS and the lens AOV kernel only
    const rt_lens* ltab;         // Q_FRAMES_LENS: [frames of the launch] each frame's lens (radius 0: pinhole)
};

// An adaptive round's accumulate-and-test (rtb200_adaptive.cu, DESIGN.md §4.9): one thread per list position.
struct AdaptiveParams {
    const float4* samplebuf;     // [s_count][n_list] the round's samples
    const uint32_t* list;        // [n_list] local pixel indices
    const uint32_t* list_n;      // device: n_list
    float* sum;                  // [npix_local][3] S_c, f32 in sample order
    float* sq;                   // [npix_local][3] Q_c
    uint32_t* count;             // [npix_local] n
    uint32_t* keep;              // [npix_local] by list position: 1 = the pixel stays on the list (0 past n_list)
    unsigned long long* black_samples;   // max_depth 0 rounds: stat[3], which no trace kernel counts; else null
    uint32_t npix_local, s_count;
    uint32_t n_after;            // samples of every listed pixel after the round
    uint32_t max_samples, min_samples;
    float abs_tol, rel_tol;
};
struct AdaptiveResolveParams {
    const float* sum; const uint32_t* count;
    uint32_t npix_local;
    float* out_linear; uint8_t* out_rgb8; uint32_t* out_count;   // each may be null
};

// The edge-avoiding à-trous filter (rtb200_denoise.cu, DESIGN.md §4.15) of a width x height image: the caller's buffers and
// the scratch of denoise_scratch_bytes, which the library lays out (denoise_carve).
struct DenoiseArgs {
    uint32_t width, height, iterations;
    float color_weight, albedo_weight, normal_weight;
    const float* color; const float* albedo; const float* normal;   // [npix][3]; a guide may be null (its weight is then 0)
    void* scratch;
    float* out_linear; uint8_t* out_rgb8;                            // [npix][3]; either may be null, not both
};

// The variance-guided à-trous filter (rtb200_denoise_var.cu, DESIGN.md §4.18): the caller's buffers and the scratch of
// denoise_var_scratch_bytes.
struct DenoiseVarArgs {
    uint32_t width, height, iterations;
    float color_weight, albedo_weight, normal_weight, variance_floor;
    const float* color; const float* variance; const float* albedo; const float* normal;   // [npix][3]; a guide may be null
    void* scratch;
    float* out_linear; uint8_t* out_rgb8; float* out_variance;                             // [npix][3]; each may be null, not all
};

// The 1-D grid of one à-trous step of both filters (rt_denoise_step_kernel, rt_denoise_var_step_kernel; DESIGN.md §4.15). Step h
// splits a width x height image into the residue classes (rx, ry) = (x mod h, y mod h), each a dense sub-grid of at most
// ceil(W/h) x ceil(H/h) pixels cut into bx x by tiles. Only the classes that hold a pixel are launched, rx < min(h, W) and
// ry < min(h, H), so the grid is at most W * H CTAs and stays under gridDim.x's 2^31 - 1 for every image the filters accept.
// CTA b is tile x fastest, then tile y, then rx, then ry; when h <= min(W, H) that is the grid of all h * h classes. The host
// computes it once per step and passes it to the kernel, which only decodes.
struct AtrousTiles {
    uint32_t tiles_x, tiles_y, res_x, res_y;
    AtrousTiles() = default;
    AtrousTiles(uint32_t width, uint32_t height, uint32_t h, uint32_t bx, uint32_t by)
        : tiles_x(((width + h - 1) / h + bx - 1) / bx), tiles_y(((height + h - 1) / h + by - 1) / by),
          res_x(h < width ? h : width), res_y(h < height ? h : height) {}
    uint64_t ctas() const { return (uint64_t)tiles_x * tiles_y * res_x * res_y; }
    // CTA b's tile (tix, tiy) and residue class (rx, ry)
    __device__ void decode(uint32_t b, uint32_t& tix, uint32_t& tiy, uint32_t& rx, uint32_t& ry) const {
        tix = b % tiles_x; b /= tiles_x;
        tiy = b % tiles_y; b /= tiles_y;
        rx = b % res_x; ry = b / res_x;
    }
};

// The temporal accumulation (rtb200_temporal.cu, DESIGN.md §4.16) of a width x height frame: the caller's buffers.
struct TemporalArgs {
    uint32_t width, height, max_history, n_motion;
    rt_camera cam, prev_cam;
    double depth_tol;
    const float* color; const uint32_t* sphere; const double* point;                  // this frame
    const float* h_color; const uint32_t* h_length; const uint32_t* h_sphere; const double* h_point;   // all null: no history
    const double* motion;                                                             // [n_motion][3], null when n_motion is 0
    float* out_color; uint32_t* out_length;
};
// The history clamp of rtb200_temporal_clamped (DESIGN.md §4.20): gamma finite and >= 0, radius in [1, 3].
struct TemporalClamp { float gamma; uint32_t radius; };
// The variance planes of rtb200_temporal_var (DESIGN.md §4.21), 3 x f32 per pixel: this frame's, the history's (null without a
// history) and the output's. A kernel parameter beside TemporalArgs, which the kernels without them keep as it is.
struct TemporalVar { const float* var; const float* h_var; float* out_var; };

struct ResolveParams {
    const float4* samplebuf;
    float*   accum;        // [npix_local][3] running f32 sums in sample order
    uint32_t npix_local, s_count;
    uint32_t first, last;  // first batch zeroes accum, last batch writes outputs
    uint32_t spp;
    float*   out_linear;   // [npix_local][3] or null
    uint8_t* out_rgb8;     // [npix_local][3] or null
};
// The resolve with the variance of each pixel's mean (rt_resolve_var_kernel, DESIGN.md §4.18): `r`'s sums and outputs, plus
// the running f32 sums of x_c * x_c in sample order and the variance output.
struct ResolveVarParams {
    ResolveParams r;
    float* accum_sq;       // [npix_local][3] Q_c, carried across batches like r.accum
    float* out_variance;   // [npix_local][3]
};
struct AdaptiveResolveVarParams {
    AdaptiveResolveParams r;
    const float* sq;       // [npix_local][3] Q_c
    float* out_variance;   // [npix_local][3]
};


// Refit of a resident scene after its spheres moved (rtb200_refit.cu, DESIGN.md §4.7): the records and f32 boxes are
// recomputed from `geo` on the upload's topology and recentring offset. Exact boxes are {lo[3], hi[3]} f64.
struct RefitParams {
    const double4* geo;
    uint32_t n;
    double g[3];                 // recentring offset
    float* filt;                 // MODE_BRUTE: n_pairs * 8 flat records, else null
    const uint32_t* leaf_id;     // MODE_TREE from here on
    float* leaf_rec;
    double* leaf_box;            // n_leaves exact boxes
    uint32_t n_leaves;
    float* nodes;
    double* node_box;            // n_nodes exact boxes (the union of the node's children)
};

// Rebuild of a resident scene's hierarchy on the GPU (rtb200_rebuild.cu, DESIGN.md §4.8). The header is what the host reads
// back: the counts, the recentring offset and the level sizes it needs for TraceParams and for later refits.
constexpr uint32_t kRebuildIdBits = 26;   // sphere index bits of a sort key (n < 2^26, validate_scene)
struct RebuildHeader {
    double g[3];                                     // recentring offset
    double r_big;                                    // |radius| above which a sphere is oversized
    unsigned long long box_lo[3], box_hi[3];         // Morton box of the centres (order-preserving integer form)
    uint32_t n_in, n_always, n_nodes, n_leaves, depth, overflow;
    uint32_t level_count[rtbvh::kMaxDepth + 1];      // nodes per wide level, root level first
    uint32_t level_base[rtbvh::kMaxDepth + 2];       // the first node of each level: nodes are numbered level by level
};
struct RebuildBufs {
    RebuildHeader* header;
    // the new hierarchy (TraceParams) and the refit's scratch of its topology
    float* nodes; float* leaf_rec; uint32_t* leaf_id; uint32_t* skip_pos; uint32_t* always;
    double* node_box; double* leaf_box; uint32_t* level_nodes;
    // scratch of the build
    double* col; double* sorted; unsigned long long* keys; unsigned long long* keys_sorted;
    uint32_t *out_flag, *always_pos, *leaf_start, *leaf_scan, *leaf_cnt;
    uint2* tasks[2]; uint2* kids; uint32_t *n_inner, *off;
    uint32_t cap;                                    // nodes per level at most
    void* temp; size_t temp_bytes;                   // cub's temporary storage
};

// Insert and remove spheres of a resident scene (rtb200_edit.cu, DESIGN.md §4.13): the old list without remove[0, n_remove),
// with insert k placed just before old sphere at[k] (at non-decreasing, at most n_old), written to geo / mat, which are not the
// old arrays. keep and pos hold n_old + 1 words.
struct EditParams {
    const double4* geo_old; const DevMat* mat_old;
    uint32_t n_old;
    const uint32_t* remove;      // [n_remove] distinct, below n_old
    uint32_t n_remove;
    const uint32_t* at;          // [n_insert]
    const double4* geo_in; const DevMat* mat_in;
    uint32_t n_insert;
    uint32_t* keep; uint32_t* pos;   // keep[i]: old sphere i stays; pos[j] = kept(< j), the exclusive scan of keep
    void* temp; size_t temp_bytes;   // cub's scan scratch (edit_scan_bytes)
    double4* geo; DevMat* mat;
    float* filt;                 // MODE_BRUTE: the new flat records, whose slots [n_old - n_remove + n_insert, 2 * n_pairs) get
    uint32_t n_pairs;            // the builder's padding; else null
};

// Closest-hit queries on caller-supplied rays (rtb200_query.cu, DESIGN.md §4.10). `p` is the handle's TraceParams: closest_hit
// reads the scene fields of it, err (guard trips) and stat (the counters; null: not counted). The outputs of rt_hits may be null.
struct QueryParams {
    TraceParams p;
    const double* origin;        // [n][3]
    const double* direction;     // [n][3]
    const double* t_max;         // [n] or null: DBL_MAX
    double* t; uint32_t* sphere; double* point; double* normal; double* uv; uint8_t* front_face;
    uint32_t n;
};

// Occlusion queries on caller-supplied rays (rtb200_query.cu, DESIGN.md §4.11): `p`, the rays and n as in QueryParams.
struct OcclusionParams {
    TraceParams p;
    const double* origin;        // [n][3]
    const double* direction;     // [n][3]
    const double* t_max;         // [n] or null: DBL_MAX
    uint8_t* occluded;           // [n]
    uint32_t n;
};

// Auxiliary buffers of the camera samples [sample0, sample0 + samples) of every pixel of the handle's rows (rtb200_aov.cu,
// DESIGN.md §4.14). `p` is the handle's TraceParams with the view's camera and key in cam / key0 / key1: closest_hit reads its
// scene fields, err (guard trips) and stat (the counters; null: not counted). Outputs are compact, per local pixel; each may be null.
struct AovParams {
    TraceParams p;
    float* albedo; float* normal;     // [n][3] the means of the samples' albedo and f32 normal
    uint32_t* hits;                   // [n] samples with a hit
    uint32_t* sphere; double* point;  // [n], [n][3] the hit of sample sample0
    uint32_t samples, sample0;
    uint32_t n;                       // local pixels = npix_local
};

// Point queries (rtb200_distance.cu, DESIGN.md §4.19): `p` is the handle's TraceParams, of which the kernel reads the scene
// fields, err (guard trips) and stat (the counters; null: not counted). The nearest kind writes distance and sphere (either may be
// null), the overlaps kind (bound = the balls' radii, never null) writes overlaps.
struct DistanceParams {
    TraceParams p;
    const double* point;         // [n][3]
    const double* bound;         // [n] or null: +inf
    double* distance; uint32_t* sphere;
    uint8_t* overlaps;
    uint32_t n;
};

struct KernelInfo { int registers, max_threads, const_bytes, local_bytes; char name[96]; };

// `queue` (TraceQueue): Q_FRAMES is the multi-frame kernel (work ids span p.ftab's frames), Q_LIST the adaptive round's,
// Q_RAYS the caller-supplied rays' (work ids span samples x rays)
size_t wavefront_smem_bytes(const TraceParams& p, uint32_t mode, uint32_t smem_mask, uint32_t queue);
cudaError_t launch_wavefront(const TraceParams& p, uint32_t mode, uint32_t queue, int grid, size_t smem, cudaStream_t st);
int wavefront_max_ctas_per_sm(uint32_t mode, bool lights, uint32_t queue, size_t smem);   // 0 when the kernel cannot run on the current device
cudaError_t wavefront_info(uint32_t mode, bool lights, uint32_t queue, KernelInfo* out);
cudaError_t launch_resolve(const ResolveParams& p, cudaStream_t st);
cudaError_t launch_resolve_var(const ResolveVarParams& p, cudaStream_t st);
// closest-hit (any = false) and occlusion (any = true) queries: resident CTAs per SM of the query kernel of that kind and
// `mode` (0 when it cannot run on the current device), and a launch of at most `max_grid` CTAs (no more than the rays need)
int query_max_ctas_per_sm(uint32_t mode, bool any);
cudaError_t launch_query(const QueryParams& q, uint32_t mode, int max_grid, cudaStream_t st);
cudaError_t launch_occluded(const OcclusionParams& q, uint32_t mode, int max_grid, cudaStream_t st);
// point queries, nearest (any = false) and overlaps (any = true): resident CTAs per SM of the kernel of that kind and `mode` (0
// when it cannot run on the current device), and a launch of at most `max_grid` CTAs (no more than the points need)
int distance_max_ctas_per_sm(uint32_t mode, bool any);
cudaError_t launch_distance(const DistanceParams& q, uint32_t mode, bool any, int max_grid, cudaStream_t st);
// the auxiliary buffers: resident CTAs per SM of the kernel of `mode` (0 when it cannot run on the current device), and a launch
// of at most `max_grid` CTAs (through the lens kernel when q.p.lens.radius is not 0)
int aov_max_ctas_per_sm(uint32_t mode, bool lens);   // lens: the kernel whose camera rays go through p.lens
cudaError_t launch_aov(const AovParams& q, uint32_t mode, int max_grid, cudaStream_t st);
// adaptive rendering (rtb200_adaptive.cu): the round's accumulate-and-test, the list compaction (cub::DeviceSelect::Flagged,
// keep[0, npix_local) over list_in, the count to *list_n_out), and the resolve
cudaError_t launch_adaptive_list(uint32_t* list, uint32_t* list_n, uint32_t npix_local, cudaStream_t st);   // list = 0, 1, .., npix_local - 1
cudaError_t launch_adaptive_accumulate(const AdaptiveParams& p, cudaStream_t st);
size_t adaptive_compact_bytes(uint32_t npix_local);   // cub's temporary storage
cudaError_t launch_adaptive_compact(void* temp, size_t temp_bytes, const uint32_t* list_in, const uint32_t* keep, uint32_t* list_out,
                                    uint32_t* list_n_out, uint32_t npix_local, cudaStream_t st);
cudaError_t launch_adaptive_resolve(const AdaptiveResolveParams& p, cudaStream_t st);
cudaError_t launch_adaptive_resolve_var(const AdaptiveResolveVarParams& p, cudaStream_t st);
// the denoise (rtb200_denoise.cu): its scratch for npix pixels, and its iterations + 1 launches (the guides' packing, then one
// per iteration)
uint64_t denoise_scratch_bytes(uint64_t npix);
cudaError_t launch_denoise(const DenoiseArgs& a, cudaStream_t st);
// the variance-guided denoise (rtb200_denoise_var.cu): its scratch, and its 2 * iterations + 1 launches (the packing, then a
// prefilter and a step per iteration)
uint64_t denoise_var_scratch_bytes(uint64_t npix);
cudaError_t launch_denoise_var(const DenoiseVarArgs& a, cudaStream_t st);
// the temporal accumulation (rtb200_temporal.cu): one launch, one thread per pixel, with the history clamp when it is given
cudaError_t launch_temporal(const TemporalArgs& a, const TemporalClamp* clamp, const TemporalVar* var,   // clamp null: unclamped;
                            cudaStream_t st);                                                       // var null: no variance
// geo[idx[k]] = geo_in[k], mat[idx[k]] = mat_in[k] for k < n (idx has no repeats)
cudaError_t launch_update_scatter(const uint32_t* idx, const double4* geo_in, const DevMat* mat_in, uint32_t n, double4* geo, DevMat* mat,
                                  cudaStream_t st);
// flat records (p.filt) or leaf records and leaf boxes (p.leaf_rec), whichever p carries
cudaError_t launch_refit_spheres(const RefitParams& p, cudaStream_t st);
// the `count` nodes level_nodes[0, count) of one tree level; their children's exact boxes are final
cudaError_t launch_refit_nodes(const RefitParams& p, const uint32_t* level_nodes, uint32_t count, cudaStream_t st);
// Lays out arrays one after another in a block, each at a 256-byte boundary, in the order they are taken. With a null base
// take returns null and `off` ends as the block's size.
struct Carver {
    char* base;
    size_t off = 0;
    explicit Carver(void* b = nullptr) : base((char*)b) {}
    size_t offset(size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; }
    void* take(size_t bytes) { const size_t o = offset(bytes); return base ? base + o : nullptr; }
};
// the rebuild's arrays for n spheres carved out of `base` (null: only the size); returns the bytes they take
size_t rebuild_carve(void* base, uint32_t n, RebuildBufs* b);
// the topology of a new hierarchy over geo[0, n): header, child words, leaf members and padding, always-list, skip_pos and the
// level order; the position-dependent values are then the refit's (launch_refit_spheres / launch_refit_nodes). A sphere whose
// |radius| exceeds `oversize` times the median |radius| gets its own subtree near the root (oversize <= 0: none does).
constexpr double kRebuildOversize = 16.0;
cudaError_t launch_rebuild_topology(const RebuildBufs& b, const double4* geo, uint32_t n, double oversize, cudaStream_t st);
// the edited list (EditParams): keep flags, their scan, every kept and inserted record at its new position, flat padding
size_t edit_scan_bytes(uint32_t n_old);   // cub's scan scratch for n_old + 1 flags
cudaError_t launch_edit_spheres(const EditParams& p, cudaStream_t st);

// single-thread probes of the device routines (known-answer tests)
cudaError_t probe_sphere_hit(const double* in /*12*/, double* out /*9*/, cudaStream_t st);
cudaError_t probe_refract(const double* in /*7*/, double* out /*3*/, cudaStream_t st);
cudaError_t probe_reflectance(const double* in /*2*/, double* out /*1*/, cudaStream_t st);
cudaError_t probe_sky(const double* in /*3*/, uint32_t mode, float* out /*3*/, cudaStream_t st);
cudaError_t probe_get_ray(const rt_camera* cam_dev, const double* in /*2*/, double* out /*6*/, cudaStream_t st);
cudaError_t probe_lens_ray(const rt_camera* cam_dev, const rt_lens* lens_dev, const double* in /*2*/, uint64_t seed, uint32_t pixel,
                           uint32_t sample, double* out /*7*/, cudaStream_t st);
cudaError_t probe_rng(uint64_t seed, uint32_t pixel, uint32_t sample, uint32_t kind, uint32_t n, double* out, cudaStream_t st);
cudaError_t probe_quantise(const float* in, uint32_t n, uint8_t* out, cudaStream_t st);
cudaError_t probe_sphere_uv(const double* in /*3n*/, uint32_t n, double* out /*2n*/, cudaStream_t st);

}  // namespace rtk
