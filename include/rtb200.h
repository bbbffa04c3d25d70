/* rtb200.h — C ABI of the H100-native render path.
 *
 * This is the drop-in boundary for ONE hot path of dps/rust-raytracer: the timed
 * region of `pub fn render(filename, scene)` (reference raytracer/src/raytracer.rs:250-266,
 * precisely lines 259-263: the rayon `into_par_iter().for_each(render_line)` over row bands).
 * The reference has no FFI; the contract of that region is
 *     "given an immutable parsed scene, fill a caller-owned w*h*3 RGB8 row-major buffer, top row first".
 * A Rust maintainer binds these entry points with an `extern "C"` block and calls
 * rtb200_render_rgb8() in place of raytracer.rs:259-263 (see INTEGRATION.md).
 *
 * Conventions
 *   - every struct is POD, little-endian, caller-owned and read-only for the callee;
 *   - the callee copies what it needs before returning; no callee allocation escapes
 *     except opaque handles released with the matching *_release call;
 *   - every function returns 0 on success, a negative rt_status otherwise, and
 *     rtb200_last_error() then returns a thread-local message (the reference panics instead); no C++
 *     exception leaves the library (host out-of-memory while building the hierarchy is RT_ERR_OOM);
 *   - calls are blocking unless stated otherwise. Thread safety: every device has its own execution context guarded
 *     by a mutex, so two host threads may render on two DIFFERENT devices concurrently; calls that use the same
 *     device are serialised. A scene handle must not be used from two threads at once. The caller's current CUDA
 *     device is restored before every entry point returns;
 *   - there is NO CPU fallback: without a CUDA device / the sm_90a kernels every render call fails.
 */
#ifndef RTB200_H
#define RTB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RTB200_ABI_VERSION 2   /* 2: rt_image.bytes, rt_stats.nodes/gpus_used, multi-GPU entry point, BVH diagnostics, RT_VARIANT_LANES retired */

/* ---- scene records (reference types flattened) --------------------------------------------- */

/* Point3D {x,y,z: f64} — raytracer/src/point3d.rs:10-15 */
typedef struct { double x, y, z; } rt_vec3;

/* The four computed fields of Camera that get_ray uses — raytracer/src/camera.rs:12-21,79-84.
 * Fill with rtb200_camera_from_params() (= Camera::new, camera.rs:45-77). */
typedef struct { rt_vec3 origin, lower_left_corner, horizontal, vertical; } rt_camera;

/* CameraParams — raytracer/src/camera.rs:29-36 (the JSON form of the camera) */
typedef struct { rt_vec3 look_from, look_at, vup; double vfov_deg, aspect; } rt_camera_params;

/* Material variants — raytracer/src/materials.rs:35-42 */
enum rt_material_kind {
    RT_LAMBERTIAN = 0, /* materials.rs:73-95   albedo                              */
    RT_METAL      = 1, /* materials.rs:99-129  albedo, param = fuzz                */
    RT_GLASS      = 2, /* materials.rs:132-199 param = index_of_refraction         */
    RT_TEXTURE    = 3, /* materials.rs:203-267 texture index, param = h_offset     */
    RT_LIGHT      = 4  /* materials.rs:57-69                                       */
};

/* Sphere {center, radius, material} — raytracer/src/sphere.rs:18-23. radius may be negative
 * (hollow glass shell, data/test_scene.json:137). List ORDER is semantic: hit_world keeps the
 * first sphere on equal t (raytracer.rs:52-56) and lights are visited in list order (raytracer.rs:103). */
typedef struct {
    rt_vec3  center;
    double   radius;
    uint32_t kind;        /* enum rt_material_kind */
    float    albedo[3];   /* Srgb<f32>; ignored for Glass/Light; ignored for Texture (materials.rs:264) */
    double   param;       /* fuzz | index_of_refraction | h_offset */
    int32_t  texture;     /* index into rt_scene.textures for RT_TEXTURE, else -1 */
    int32_t  reserved;
} rt_sphere;

/* Decoded RGB8 image, row-major, 3 B/texel. For Texture materials width/height are the values
 * written in the JSON, NOT the decoded file's (materials.rs:208-209 with loader result .0 only, :32). */
typedef struct {
    const uint8_t* rgb8;
    uint64_t width, height;
    uint64_t bytes;       /* size of the buffer rgb8 points to; the callee reads width*height*3 bytes and rejects bytes < that */
} rt_image;

/* Sky — raytracer/src/config.rs:22-28 and the miss branch raytracer.rs:134-163 */
enum rt_sky_mode { RT_SKY_NONE = 0 /* black */, RT_SKY_GRADIENT = 1, RT_SKY_TEXTURE = 2 };
typedef struct { uint32_t mode; uint32_t reserved; rt_image tex; } rt_sky;

/* Config — raytracer/src/config.rs:66-75, plus the seed (the reference draws from an OS-seeded
 * thread_rng and is not reproducible; see DESIGN.md "RNG contract"). */
typedef struct {
    uint32_t width, height, samples_per_pixel, max_depth;
    rt_camera camera;
    rt_sky    sky;
    const rt_sphere* spheres;  uint64_t n_spheres;
    const rt_image*  textures; uint64_t n_textures;
    uint64_t seed;
} rt_scene;

/* ---- execution options and results ---------------------------------------------------------- */

enum rt_trace_variant {
    RT_VARIANT_AUTO      = 0,
    RT_VARIANT_FILTERED  = 1, /* CTA-wavefront kernel: warp-cooperative traversal of an 8-wide BVH with conservative f32 tests + exact f64 confirmation (default) */
    RT_VARIANT_EXACT_F64 = 2, /* every sphere tested in f64 (validation of the conservative tests) */
    RT_VARIANT_RETIRED_LANES = 3, /* ABI 1's lane-autonomous kernel; retired: RT_ERR_UNSUPPORTED */
    RT_VARIANT_BRUTE_FORCE = 4 /* CTA-wavefront kernel scanning every sphere in list order (no hierarchy), like the reference's hit_world */
};

/* Which rows this call renders. Row-band b (band_rows consecutive rows) belongs to shard
 * (b mod world). world=1 renders everything. Output buffers of a shard call are COMPACT: the
 * shard's rows in increasing y, see rtb200_shard_rows(). */
typedef struct {
    int32_t  device;      /* CUDA ordinal; -1 = current device */
    int32_t  rank, world; /* shard of the image rendered by this call */
    uint32_t band_rows;   /* rows per interleaved band; 0 = default (1) */
    uint32_t variant;     /* enum rt_trace_variant */
    uint32_t flags;       /* reserved, must be 0 */
    uint64_t sample_buffer_bytes; /* cap for the per-sample radiance staging buffer; 0 = default */
} rt_options;

typedef struct {
    uint64_t rays;          /* hit_world invocations (primary + scattered + shadow), raytracer.rs:83 */
    uint64_t samples;       /* camera samples traced */
    uint64_t candidates;    /* f64-confirmed sphere tests (diagnostic) */
    double   device_ms;     /* CUDA-event time of all kernels of this call on the launching stream */
    double   trace_ms;      /* the trace kernel(s) alone */
    double   wall_ms;       /* host wall time of the call, copies included */
    uint32_t kernel_launches;
    uint32_t batches;
    uint64_t h2d_bytes, d2h_bytes;
    uint64_t clusters;      /* BVH leaves visited (diagnostic) */
    uint64_t frames;        /* frames covered by device_ms / trace_ms / kernel_launches (1 for the blocking one-frame calls,
                               n_frames for the frames calls, also on a shard with no rows) */
    uint64_t nodes;         /* BVH nodes visited (diagnostic) */
    int32_t  gpus_used;     /* devices that rendered this frame (1 on a shard with no rows) */
    int32_t  reserved;
} rt_stats;

/* The trace kernel a scene handle launches (cudaFuncGetAttributes + the launch geometry chosen at upload). */
typedef struct {
    int32_t  registers, local_bytes;       /* per thread */
    uint32_t smem_bytes, grid, block, ctas_per_sm;
    uint32_t smem_mask;                    /* bit0 hierarchy, bit1 exact geometry, bit2 materials staged into shared memory */
    uint32_t bvh_nodes, bvh_leaves, bvh_depth;
    uint32_t pool_slots;                   /* ray slots per CTA */
    char     name[96];
} rt_kernel_info;

enum rt_status {
    RT_OK = 0,
    RT_ERR_INVALID = -1,     /* bad argument / inconsistent scene */
    RT_ERR_NO_DEVICE = -2,   /* no CUDA device or not sm_90 */
    RT_ERR_CUDA = -3,        /* CUDA runtime failure (message has the detail) */
    RT_ERR_UNSUPPORTED = -4, /* scene needs a feature this build lacks */
    RT_ERR_OOM = -5
};

/* ---- entry points ---------------------------------------------------------------------------- */

int rtb200_abi_version(void);
const char* rtb200_last_error(void);

/* Camera::new — camera.rs:45-77 (host, f64, once per frame). */
int rtb200_camera_from_params(const rt_camera_params* p, rt_camera* out);

/* Number of rows of `height` that shard `rank` of `world` owns with the given band size. */
uint32_t rtb200_shard_rows(uint32_t height, int32_t rank, int32_t world, uint32_t band_rows);

/* Replaces raytracer.rs:259-263 (+ the Vec<u8> it fills, :254): host scene in, host RGB8 out.
 * Uploads the scene, renders on one GPU (opts==NULL) or the shard opts describes, copies back.
 * out_rgb8: width*height*3 bytes (or shard_rows*width*3 when opts->world > 1). */
int rtb200_render_rgb8(const rt_scene* scene, const rt_options* opts, uint8_t* out_rgb8, rt_stats* stats);

/* The same frame on n_gpus devices of this process (0 = all; devices opts->device.. when opts->device >= 0, else 0..):
 * the reference's row bands (raytracer.rs:254-262) are dealt round-robin to the devices (band b -> device b mod G), the
 * scene is replicated, every device renders its shard, the shards are copied peer-to-peer into the frame on the first
 * device and ONE device->host copy fills out_rgb8 (width*height*3 bytes). Bit-identical to rtb200_render_rgb8.
 * opts->rank/world must be 0/1 (or opts NULL). */
int rtb200_device_count(void);
int rtb200_render_rgb8_multi(const rt_scene* scene, const rt_options* opts, int32_t n_gpus, uint8_t* out_rgb8, rt_stats* stats);

/* Same path, but returns the per-pixel mean radiance BEFORE sqrt/quantisation (raytracer.rs:207-212
 * computes sqrt(scale*sum)); used by parity tests. out_rgb: width*height*3 floats (or the shard's). */
int rtb200_render_linear_f32(const rt_scene* scene, const rt_options* opts, float* out_rgb, rt_stats* stats);

/* Resident form (scene stays in HBM between frames; output stays on the device). */
typedef struct rtb200_scene_t* rtb200_scene_handle;
int rtb200_scene_upload(const rt_scene* scene, const rt_options* opts, rtb200_scene_handle* out);
/* dev_rgb8 / dev_linear_f32 are DEVICE pointers (either may be NULL); stream is a cudaStream_t, or NULL for the library's
 * own non-blocking stream (pass cudaStreamLegacy / cudaStreamPerThread explicitly to order against the default stream). */
int rtb200_render_device(rtb200_scene_handle h, void* dev_rgb8, void* dev_linear_f32, void* stream, rt_stats* stats);
/* Non-blocking form for frame loops: enqueue a frame on `stream` and return; rtb200_render_device_wait() blocks until the
 * frames enqueued so far are done and returns statistics: rays, samples and the other counters are those of the last frame
 * enqueued, times and frames are summed. A device has two sets of work buffers, shared by all its scenes: successive
 * asynchronous frames of a scene alternate between them and every blocking render uses the first. A frame starts only after
 * the previous frame that used the same set has finished with it, whatever its stream and scene, so any number of scenes may
 * have frames in flight on any streams; a caller that alternates two streams (and two output buffers) lets frame k+1 start
 * while frame k drains its last paths. */
int rtb200_render_device_async(rtb200_scene_handle h, void* dev_rgb8, void* dev_linear_f32, void* stream);
int rtb200_render_device_wait(rtb200_scene_handle h, rt_stats* stats);
int rtb200_scene_release(rtb200_scene_handle h);
int rtb200_scene_kernel_info(rtb200_scene_handle h, rt_kernel_info* out);

/* ---- animations: many frames of one scene ------------------------------------------------------------------------------
 * One frame of an animation over a resident scene: the view, the RNG key and the depth that replace the scene's own. */
typedef struct {
    rt_camera camera;     /* Camera::new of this frame's CameraParams (rtb200_camera_from_params) */
    uint64_t  seed;       /* Philox key of this frame, as rt_scene.seed */
    uint32_t  max_depth;  /* as rt_scene.max_depth (0 = black frame, no ray) */
    uint32_t  reserved;   /* must be 0 */
} rt_frame;               /* 112 bytes */

/* Render n_frames frames of one scene. Frame i is bit-identical, in linear f32 and RGB8, to rtb200_render_rgb8 /
 * rtb200_render_linear_f32 of the scene with camera, seed and max_depth taken from frames[i]; the scene's own camera, seed
 * and max_depth are ignored, its size, samples_per_pixel, sky, spheres and textures are shared by all frames. Shards
 * (opts->rank/world/band_rows) and every variant work as for one frame.
 * Outputs are frame-major and contiguous: n_frames * rows * width * 3 (rows = rtb200_shard_rows(...) for a shard); either may
 * be NULL, not both. Consecutive frames with equal max_depth whose samples fit the sample-buffer cap together
 * (F * samples_per_pixel * rows * width * 16 bytes <= opts->sample_buffer_bytes) are traced by ONE persistent launch whose work
 * queue spans all of them, so that only the last frame of a launch waits for its slowest paths; frames of more than 2^24
 * samples (samples_per_pixel * rows * width) are long enough to hide their own tail and are traced one launch each.
 * stats: rays and samples are sums over the frames; frames = n_frames; batches = trace launches (or black max_depth 0 batches);
 * kernel_launches = trace + resolve launches. RT_ERR_INVALID, before any device is touched, for n_frames == 0, a NULL frames,
 * a nonzero rt_frame.reserved or n_frames * rows * width * 3 overflowing 64 bits.
 * rtb200_render_frames uploads the scene, renders, copies back and releases, like rtb200_render_rgb8. */
int rtb200_render_frames(const rt_scene* scene, const rt_options* opts, const rt_frame* frames, uint32_t n_frames,
                         uint8_t* out_rgb8, float* out_linear_f32, rt_stats* stats);
/* The same on a resident scene into DEVICE buffers. Blocking: drains the handle's asynchronous frames first, uploads the frame
 * table of the frames that share a launch (counted in h2d_bytes) on `stream` (NULL: the library's stream) and returns when
 * the frames are done. The handle's own view is unchanged:
 * a later rtb200_render_device renders the camera it was uploaded with. */
int rtb200_render_frames_device(rtb200_scene_handle h, const rt_frame* frames, uint32_t n_frames,
                                void* dev_rgb8, void* dev_linear_f32, void* stream, rt_stats* stats);

/* ---- depth of field: a thin-lens camera (DESIGN.md §4.17) ---------------------------------------------------------------
 * The reference's camera is a pinhole. This is the lens of Ray Tracing in One Weekend's camera (random_in_unit_disk), with this
 * library's own contract; every f64 operation is rounded to nearest, never contracted, and runs in the order written.
 * Camera: rtb200_camera_from_params_lens takes p, aperture >= 0 and focus_dist fd > 0 (both finite), computes half_height,
 * half_width, w, u and v as rtb200_camera_from_params (Camera::new, camera.rs:52-58), then
 *     origin = look_from    lower_left_corner = ((origin - u*(half_width*fd)) - v*(half_height*fd)) - w*fd
 *     horizontal = ((u*2.0)*half_width)*fd    vertical = ((v*2.0)*half_height)*fd    lens = {u, v, radius = aperture / 2}.
 * At fd = 1.0 every product by fd is exact: the camera is rtb200_camera_from_params' bit for bit.
 * Lens draws, a separate RNG domain: trial k = 0, 1, .. of sample (pixel, sample) reads Philox block (k, sample, pixel, 1) under
 * the frame's key (the path's draws are blocks (b, sample, pixel, 0)); x = gen_range(-1.0..1.0) of the u64 (w1 << 32) | w0 and
 * y of (w3 << 32) | w2 (the mapping of rtb200_probe_rng kind 1). The first trial with x*x + y*y < 1.0 is accepted; the loop is
 * unbounded, like random_in_unit_sphere. The two jitter draws and every path draw therefore stay where the pinhole render has
 * them, and a lens render equals rtb200_scene_trace_rays of its own lens primary rays, sample by sample.
 * Ray: (o0, d0) = Camera::get_ray(camera, u, v) of the pixel's jittered (u, v) (raytracer.rs:199-201); with radius r > 0
 *     rdx = r*x   rdy = r*y   offset = lens.u*rdx + lens.v*rdy (per component)   origin = o0 + offset   direction = d0 - offset.
 * With r == 0 no lens block is drawn and the ray is (o0, d0): a pinhole render is bit for bit today's. */
typedef struct {
    rt_vec3  u, v;        /* the camera's unit right and up vectors */
    double   radius;      /* aperture / 2; 0 = pinhole */
    uint64_t reserved;    /* must be 0 */
} rt_lens;                /* 64 bytes */

/* RT_ERR_INVALID for a NULL p / out / lens, a negative or non-finite aperture, or a focus_dist that is not finite and > 0. */
int rtb200_camera_from_params_lens(const rt_camera_params* p, double aperture, double focus_dist, rt_camera* out, rt_lens* lens);
/* The lens of a resident scene (NULL or radius 0: pinhole, as uploaded). Host-side handle state, copied: it applies to every call
 * enqueued after this returns that makes camera rays from a view without its own lens - rtb200_render_device[_async],
 * rtb200_render_frames[_device] (every frame), the adaptive rounds and rtb200_scene_aov[_device] with or without a view.
 * rtb200_scene_trace_rays and the queries take the caller's rays and ignore it. It counts as an update for adaptive rendering
 * (rtb200_adaptive_step refuses until the next begin); updates, rebuilds and edits keep it. RT_ERR_INVALID for a NULL handle,
 * a non-finite u, v or radius, a negative radius or a nonzero reserved (the handle's lens is then unchanged). */
int rtb200_scene_set_lens(rtb200_scene_handle h, const rt_lens* lens);
/* rtb200_render_frames[_device] with a lens per frame: frame i is rendered with lenses[i] (radius 0: pinhole) instead of the
 * handle's lens. The lens table of the frames that share a launch is a separate device array, uploaded on `stream` and counted in
 * h2d_bytes. lenses == NULL: exactly rtb200_render_frames[_device]. The host form with n_frames = 1 is the one-shot render of a
 * lens camera. RT_ERR_INVALID, before any device is touched, for a lens that rtb200_scene_set_lens would refuse, and for every
 * reason rtb200_render_frames[_device] refuses. rtb200_render_rgb8_multi takes no lens. */
int rtb200_render_frames_lens(const rt_scene* scene, const rt_options* opts, const rt_frame* frames, const rt_lens* lenses,
                              uint32_t n_frames, uint8_t* out_rgb8, float* out_linear_f32, rt_stats* stats);
int rtb200_render_frames_lens_device(rtb200_scene_handle h, const rt_frame* frames, const rt_lens* lenses, uint32_t n_frames,
                                     void* dev_rgb8, void* dev_linear_f32, void* stream, rt_stats* stats);
/* The variance of the pixel means (DESIGN.md §4.18): rtb200_render_frames_lens[_device] plus dev_variance_f32 / out_variance
 * (n_frames * rows * width * 3 floats, not NULL). Per pixel and channel, with S_c the f32 sum of the n = samples_per_pixel
 * samples in sample order (the render's) and Q_c the f32 sum of x_c * x_c in the same order, every op rounded and never
 * contracted: inv = 1.0f / n, mean_c = inv * S_c, d_c = inv * Q_c - mean_c * mean_c, var_c = (d_c < 0 ? 0 : d_c) * inv - the
 * adaptive rule's err_c^2 without its max; a NaN d_c stays NaN; max_depth 0 gives 0. Q carries across sample batches in a
 * second plane of the work set, grown only by these calls. lenses may be NULL; shards, every variant, multi-frame groups and
 * batches work as in the frames call; the rgb8 and linear outputs (each may be NULL) equal that call's bit for bit. The resolve
 * is a kernel of its own, so a render without a variance output launches exactly what it did. */
int rtb200_render_frames_var_device(rtb200_scene_handle h, const rt_frame* frames, const rt_lens* lenses, uint32_t n_frames,
                                    void* dev_rgb8, void* dev_linear_f32, float* dev_variance_f32, void* stream, rt_stats* stats);
int rtb200_render_frames_var(const rt_scene* scene, const rt_options* opts, const rt_frame* frames, const rt_lens* lenses,
                             uint32_t n_frames, uint8_t* out_rgb8, float* out_linear_f32, float* out_variance, rt_stats* stats);

/* ---- moving spheres of a resident scene ---------------------------------------------------------------------------------
 * The hierarchy is refitted on the GPU (its topology and recentring stay as uploaded, DESIGN.md §4.7) instead of rebuilt.
 * Contract: after an update every render of h is bit-identical, in linear f32, RGB8 and ray count, to the same render of a
 * fresh upload of the edited scene (the diagnostic candidates / clusters / nodes counters may differ: the tree differs).
 * Stream-ordered, without waiting for the GPU: the update runs on `stream` (NULL: the library's stream) after every frame of
 * h already enqueued, on any stream, and before every frame enqueued later; rtb200_scene_release waits for it. The first
 * update of a handle builds the refit's scratch and waits for the library's stream once.
 * Spheres that no longer fit the f32 frame (non-finite, or max|c - recentre| + |radius| >= 1e15) are tested in f64 by every
 * ray; the tree gets slower as spheres wander from where they were uploaded: rtb200_scene_rebuild gives it a new topology. */
/* Replace spheres index[k] (k < n) of a resident scene by spheres[k]: centre, radius and material. Everything is checked on
 * the host before anything is enqueued (on error the scene is unchanged); n == 0 is a no-op. RT_ERR_INVALID: NULL arrays, an
 * index >= n_spheres, a repeated index, an unknown kind, a texture index outside the uploaded textures (or one whose image was
 * empty). RT_ERR_UNSUPPORTED: making a sphere a light or a light something else (a light may move; to change the set of lights,
 * remove and insert the spheres with rtb200_scene_edit_spheres). The input is copied into pinned staging memory before the
 * call returns. */
int rtb200_scene_update_spheres(rtb200_scene_handle h, const uint32_t* index, const rt_sphere* spheres, uint32_t n, void* stream);
/* Replace the centre and radius of EVERY sphere from device memory: n_spheres x {cx, cy, cz, radius} f64 (the layout of the geo
 * array); materials stay. Any values are accepted. RT_ERR_INVALID for a NULL pointer or one that is not device memory of h's
 * device or managed memory. The caller keeps the buffer unchanged until the update has run on `stream`. */
int rtb200_scene_update_geometry_device(rtb200_scene_handle h, const void* dev_center_radius, void* stream);
/* Diagnostic: D2H copy of the handle's current nodes / leaf records / flat records (RT_VARIANT_BRUTE_FORCE only) / exact geometry
 * {cx,cy,cz,radius}, laid out as rtb200_debug_bvh's (same info[]); arrays are filled up to their capacities (elements). */
int rtb200_scene_debug_records(rtb200_scene_handle h, uint32_t info[8], float* nodes, uint64_t cap_nodes, float* leaf_rec,
                               uint64_t cap_leaf_rec, float* flat, uint64_t cap_flat, double* geo, uint64_t cap_geo);

/* Rebuild the hierarchy of a resident RT_VARIANT_FILTERED / RT_VARIANT_AUTO scene from its current spheres, on the GPU
 * (DESIGN.md §4.8): a refit keeps the upload's topology, which loosens as spheres wander; a rebuild gives a new one without a
 * host build or a copy through host memory. Contract, the update's: after a rebuild every render of h is bit-identical, in
 * linear f32, RGB8 and ray count, to the same render of a fresh upload of the current spheres (the diagnostic candidates /
 * clusters / nodes counters may differ: the tree differs). The recentring offset (element n/2 of each sorted centre
 * coordinate, 0 when not finite) and the always-list (the spheres outside the f32 frame, in increasing index order) equal a
 * fresh upload's.
 * Ordering: enqueued on `stream` (NULL: the library's stream) after the handle's last update and after every frame of h
 * already enqueued, on any stream; every frame enqueued later traces the new tree, and later rtb200_scene_update_* calls refit
 * it. Blocking: the call waits for those frames and for the new topology, reads back one small header (counts, depth, level
 * sizes, recentring offset) and returns; the values of the new tree are computed on `stream` after it returns.
 * Memory: one device block for n spheres, allocated at the first rebuild and kept until release: 576 * n + 88 * (n / 9 + 1)
 * bytes (the tree bound is n leaves and n nodes, DESIGN.md §4.8) plus cub's sort and scan scratch; RT_ERR_OOM, with the scene
 * unchanged, when it cannot be allocated. A no-op returning RT_OK for RT_VARIANT_EXACT_F64 / RT_VARIANT_BRUTE_FORCE handles (no hierarchy) and for
 * n_spheres == 0. RT_ERR_INVALID for a NULL handle, before any device is touched. RT_ERR_UNSUPPORTED for a handle that stages
 * its hierarchy in shared memory (RTB200_WF_SMEM bit 0 at upload): its launch layout is fixed by the upload's tree size. */
int rtb200_scene_rebuild(rtb200_scene_handle h, void* stream);
/* Diagnostic: the handle's current topology, the upload's or the last rebuild's: recentring offset, info[] as
 * rtb200_debug_bvh's, leaf slot -> sphere index (n_leaves * leaf_size), the always-list (n_always), skip_pos (max(n, 1) entries
 * of a hierarchy handle: kSkipNodeBit | node * 8 + child, leaf * leaf_size + slot, or 0xffffffff), the level order of the
 * nodes, deepest level first (n_nodes) and its offsets (depth + 1). Arrays are filled up to their capacities (elements). */
int rtb200_scene_debug_topology(rtb200_scene_handle h, double recentre[3], uint32_t info[8], uint32_t* leaf_id, uint64_t cap_leaf_id,
                                uint32_t* always, uint64_t cap_always, uint32_t* skip_pos, uint64_t cap_skip_pos,
                                uint32_t* level_nodes, uint64_t cap_level_nodes, uint32_t* level_off, uint64_t cap_level_off);

/* Insert and remove spheres of a resident scene, on the GPU (DESIGN.md §4.13). The edited list is the old list without the
 * spheres remove[0, n_remove) (indices into the old list, distinct, < n_spheres), with insert[k] placed just before old sphere
 * at[k] for every k < n_insert. at is non-decreasing with values in [0, n_spheres]; n_spheres appends, and at == NULL appends
 * every insert; inserts with equal at keep their order. So a kept old sphere i lands at kept(< i) + #{k : at[k] <= i} and
 * insert k at kept(< at[k]) + k, where kept(< j) counts the kept old spheres below j (also when at[k] names a removed sphere).
 * Lights are the Light spheres of the new list in its order, so an edit may change them.
 * Contract, the update's: after an edit every call on h is bit-identical to the same call on a fresh upload of the edited list
 * with the same textures, sky, camera, seed and options: renders, frames, adaptive renders and trace_rays (linear f32, RGB8,
 * rays) and every output of the queries, with the new sphere indices (the diagnostic candidates / clusters / nodes counters
 * may differ: a RT_VARIANT_FILTERED / AUTO handle gets the rebuild's hierarchy of the new list, as rtb200_scene_rebuild).
 * Everything is checked on the host before anything is enqueued; on error the scene is unchanged. RT_ERR_INVALID: a NULL
 * handle, a NULL remove with n_remove > 0 or insert with n_insert > 0, a remove index >= n_spheres or repeated, an at that
 * decreases or exceeds n_spheres, an insert that rtb200_scene_update_spheres would refuse as INVALID. RT_ERR_UNSUPPORTED: a
 * list of 2^26 spheres or more, 10 or more lights, a handle that stages the scene in shared memory (any RTB200_WF_SMEM bit at
 * upload). RT_ERR_OOM: device memory for the new arrays cannot be allocated. n_remove == n_insert == 0 is a no-op.
 * Ordering and blocking, like rtb200_scene_rebuild: on `stream` (NULL: the library's stream) after the handle's last update,
 * rebuild or edit and after every frame and query of h already enqueued, on any stream; every frame, query, update and rebuild
 * enqueued later sees the new list. The call returns when the new list and its topology exist. It counts as an update (an
 * adaptive render begun before it refuses to step). Host work and copies are O(n_remove + n_insert): the indices and the
 * inserted records go through pinned staging memory.
 * Memory: the new list lives in a per-handle block of two halves (the list and the next edit's target) for up to cap spheres,
 * about 2 * 64 B per sphere (+ 2 * 16 B in RT_VARIANT_BRUTE_FORCE) plus 12 B of skip and scan arrays, allocated at the first
 * edit and replaced by one of at least twice the size when an edit needs more; a hierarchy handle grows its rebuild block
 * by half when the new list needs more. Both are freed at release; the upload's arrays stay as they are. */
int rtb200_scene_edit_spheres(rtb200_scene_handle h, const uint32_t* remove, uint32_t n_remove, const uint32_t* at,
                              const rt_sphere* insert, uint32_t n_insert, void* stream);

/* ---- adaptive rendering: stop sampling the pixels that have converged (DESIGN.md §4.9) -----------------------------------
 * Parameters: m = samples_per_round >= 1, N = max_samples (0: the scene's samples_per_pixel), min_samples >= 1, and the f32
 * tolerances abs_tol and rel_tol. Per pixel the state is n (samples taken) and, per channel c, the f32 sums in sample order
 * S_c = sum of the sample radiances (the sum the one-shot render forms) and Q_c = sum of x_c * x_c.
 * Round: every pixel still on the list traces samples [n, min(n + m, N)) (all listed pixels have the same n).
 * Test after the round, every f32 operation rounded to nearest and never contracted: inv = 1/n and per channel
 *     mean_c = inv*S_c   var_c = inv*Q_c - mean_c*mean_c   err_c = sqrt(max(var_c, 0)*inv)   tol_c = abs_tol + rel_tol*mean_c
 * The pixel leaves the list if n == N, or if n >= min_samples, every S_c and Q_c is finite and err_c <= tol_c for all three
 * channels. A pixel with a NaN or infinite sum therefore runs to N, and negative tolerances never stop a pixel early.
 * Resolve: linear = mean_c, RGB8 = the one-shot quantisation of mean_c; a pixel with n == 0 is 0.
 * Contract: a pixel that received n samples has exactly the linear f32 value, RGB8 value and rays of the one-shot render of the
 * same scene at samples_per_pixel = n. */
typedef struct {
    uint32_t samples_per_round, max_samples, min_samples, reserved;   /* reserved must be 0 */
    float    abs_tol, rel_tol;
} rt_adaptive_params;     /* 24 bytes */

/* Resident form: the state (about 40 bytes per pixel of the shard plus cub's scan scratch) lives in the scene handle; it is
 * allocated at the first begin and freed with the handle. A shard handle (rank/world/band_rows) works on its own rows, every
 * variant is supported. Outputs are compact like the other calls' (shard rows * width). All three calls are blocking.
 * begin (re)starts: n = 0 everywhere, every pixel on the list. RT_ERR_INVALID, before any device work, for a NULL handle or
 * params, samples_per_round or min_samples of 0, a NaN tolerance, a nonzero reserved, samples_per_round * pixels * 16 above the
 * handle's sample-buffer cap (rt_options.sample_buffer_bytes) or samples_per_round * pixels >= 2^31.
 * step enqueues `rounds` rounds with no host wait between them, then waits once, and reports the pixels still active and
 * rt_stats summed over the rounds (rays, samples, device and trace time, kernel launches; batches = trace launches). Once no
 * pixel is active a step is a no-op. It drains the handle's asynchronous frames first, takes work set 0 and orders its rounds
 * after the previous user of that set like a blocking render (rtb200_render_device). RT_ERR_INVALID before any begin and after an
 * rtb200_scene_update_* since the last begin (the sums would mix two scenes); a rebuild does not change renders and is allowed.
 * resolve writes, for every pixel of the handle, the mean (dev_linear_f32, rows * width * 3 floats), its RGB8 value (dev_rgb8)
 * and n (dev_counts_u32, rows * width); each output may be NULL. stream: as rtb200_render_device's. */
int rtb200_adaptive_begin(rtb200_scene_handle h, const rt_adaptive_params* p, void* stream);
int rtb200_adaptive_step(rtb200_scene_handle h, uint32_t rounds, void* stream, uint32_t* active_out, rt_stats* stats);
int rtb200_adaptive_resolve(rtb200_scene_handle h, void* dev_rgb8, void* dev_linear_f32, void* dev_counts_u32, void* stream);
/* rtb200_adaptive_resolve plus the variance of each pixel's mean (DESIGN.md §4.18) from the adaptive state's own sums S_c, Q_c
 * and count n: inv = 1/n, mean_c = inv * S_c, d_c = inv * Q_c - mean_c * mean_c, var_c = (d_c < 0 ? 0 : d_c) * inv, every op
 * rounded and never contracted (a NaN d_c stays NaN; n = 0 gives 0), into dev_variance_f32 (rows * width * 3 floats, not NULL).
 * The other outputs equal rtb200_adaptive_resolve's bit for bit; it runs its own kernel, so that call launches what it did. */
int rtb200_adaptive_resolve_var(rtb200_scene_handle h, void* dev_rgb8, void* dev_linear_f32, void* dev_counts_u32,
                                float* dev_variance_f32, void* stream);
/* Host form, like rtb200_render_frames: upload, run rounds until no pixel is active, copy back, release. Outputs are host
 * buffers of rows * width * 3 bytes / floats and rows * width counts; each may be NULL. Same checks as begin. */
int rtb200_render_adaptive(const rt_scene* scene, const rt_options* opts, const rt_adaptive_params* p,
                           uint8_t* out_rgb8, float* out_linear_f32, uint32_t* out_counts, rt_stats* stats);
/* rtb200_render_adaptive plus out_variance (rows * width * 3 floats, not NULL): rtb200_adaptive_resolve_var's variance of
 * each pixel's mean; the other outputs equal rtb200_render_adaptive's bit for bit. */
int rtb200_render_adaptive_var(const rt_scene* scene, const rt_options* opts, const rt_adaptive_params* p, uint8_t* out_rgb8,
                               float* out_linear_f32, uint32_t* out_counts, float* out_variance, rt_stats* stats);

/* ---- closest-hit queries on a resident scene (DESIGN.md §4.10) -----------------------------------------------------------
 * Contract: for ray i with origin o = origin[3i..3i+2], direction d = direction[3i..3i+2] (any f64 values, not necessarily
 * normalised) and bound t_max_i = t_max[i] (f64::MAX when t_max is NULL; a bound above f64::MAX, i.e. +inf, counts as
 * f64::MAX), the result is hit_world(world, Ray{o, d}, 0.001, t_max_i) (raytracer.rs:44-59) over the handle's CURRENT spheres:
 * the upload's, or those of the last update or rebuild enqueued before the query. Every output equals the reference's bit for
 * bit, for every variant:
 *   sphere      index of the hit sphere (on equal t the first in list order), 0xffffffff for a miss;
 *   t           the accepted root;
 *   point       ray.at(t) (ray.rs:18-20);
 *   normal      (point - centre) / radius, flipped against the ray, as HitRecord.normal (sphere.rs:59-76);
 *   front_face  1 when the ray hits the outside, else 0;
 *   uv          u_v_from_sphere_hit_point (sphere.rs:35-43), whose f64::atan2 is the explicit algorithm the texture path and
 *               the oracle share (DESIGN.md §3), not the platform's: the last bit of u may differ from a host libm's.
 * A miss writes sphere = 0xffffffff, t = +inf, zeros in point, normal and uv, and front_face = 0. t_min is always 0.001. */
typedef struct {
    const double* origin;     /* n x 3 */
    const double* direction;  /* n x 3 */
    const double* t_max;      /* n, or NULL: f64::MAX for every ray */
} rt_rays;                    /* 24 bytes */
typedef struct {              /* every pointer may be NULL: that output is not written */
    double* t; uint32_t* sphere; double* point /* n x 3 */; double* normal /* n x 3 */; double* uv /* n x 2 */; uint8_t* front_face;
} rt_hits;                    /* 48 bytes */
/* Device buffers (of h's device, or managed memory), stream-ordered, without waiting for the GPU. The query runs on `stream`
 * (NULL: the library's stream) after the upload and after the last update or rebuild of h enqueued before it, on any stream;
 * every rtb200_scene_update_* and rtb200_scene_rebuild enqueued after it waits for it, and rtb200_scene_release waits for it.
 * Queries only read the scene and take no work set: they neither wait for frames nor make frames wait, and queries on any
 * streams may overlap each other and frames. The buffers must stay valid until the query has run on `stream`. A traversal-guard
 * trip is counted with the handle's frames' and reported when its next frames are collected (rtb200_render_device_wait or a
 * blocking render).
 * RT_ERR_INVALID, before any device work, for a NULL handle, NULL rays, out, origin or direction, an out with every output NULL,
 * or a pointer that is not device memory of h's device or managed memory. n == 0 is a no-op. */
int rtb200_scene_intersect_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_hits* out, void* stream);
/* Host buffers, blocking: the same query, through the same kernel, on the library's stream with copies in and out. stats (may
 * be NULL): rays = n, candidates (f64 sphere tests), clusters (leaves visited), nodes (nodes visited), device_ms (copies and
 * kernel), trace_ms (the kernel), wall_ms, h2d_bytes, d2h_bytes and kernel_launches. Same checks as the device form, bar the
 * memory kind; a traversal-guard trip fails the call with RT_ERR_CUDA. */
int rtb200_scene_intersect(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_hits* out, rt_stats* stats);

/* Occlusion queries on a resident scene (DESIGN.md §4.11). For ray i (origin, direction, t_max as in rt_rays; a NULL t_max is
 * f64::MAX, a bound above f64::MAX counts as f64::MAX) occluded[i] = 1 if hit_world(world, Ray{o, d}, 0.001, t_max_i) is Some
 * over the handle's CURRENT spheres, else 0, in every variant. Same ordering, memory-kind checks and guard-trip reporting as
 * rtb200_scene_intersect[_device]; n == 0 is a no-op. */
int rtb200_scene_occluded_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, uint8_t* occluded, void* stream);
int rtb200_scene_occluded(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, uint8_t* occluded, rt_stats* stats);

/* ---- point queries on a resident scene (DESIGN.md §4.19) ------------------------------------------------------------------
 * Contract: for point p = point[3i..3i+2] (any f64 values) and sphere j of the handle's CURRENT list (centre c, radius R, any
 * material, lights included), the distance is computed with round-to-nearest and no contraction:
 *   x = fl(p.x - c.x),  y = fl(p.y - c.y),  z = fl(p.z - c.z)
 *   s = fl(sqrt(fl(fl(fl(x*x) + fl(y*y)) + fl(z*z))))
 *   dist_j = fl(s - |R|)
 * the signed distance to the sphere's surface: negative inside, and |R| because a negative radius has the same surface. numpy
 * float64 reproduces it bit for bit.
 * Nearest: point i has the bound b_i = bound[i] (+inf when bound is NULL). The answer is the sphere j with dist_j < b_i and the
 * least dist_j, the lowest index among equal distances: sphere = j, distance = dist_j. With no such sphere, sphere = 0xffffffff
 * and distance = +inf. So a NaN distance never qualifies, and neither does +inf; a NaN point, or a NaN or -inf bound, gives
 * none; a scene with no spheres gives none everywhere.
 * Overlaps: ball i has centre point i and radius bound[i] (required). overlaps[i] = 1 iff some sphere has dist_j < bound[i],
 * else 0: bit for bit nearest(point i, bound[i]).sphere != 0xffffffff. Touching (dist_j = r) does not count; r = 0 asks whether
 * the point lies strictly inside a sphere.
 * Every variant gives the same answers. */
typedef struct {
    const double* point;      /* n x 3 */
    const double* bound;      /* n, or NULL (nearest only): +inf for every point */
} rt_points;                  /* 16 bytes */
typedef struct {              /* either may be NULL, not both */
    double* distance; uint32_t* sphere;
} rt_nearest;                 /* 16 bytes */
/* Device buffers, stream-ordered, with the ordering, memory-kind checks and guard-trip reporting of
 * rtb200_scene_intersect_device: after the last update, rebuild or edit of h enqueued before, on any stream; later updates,
 * rebuilds, edits and the release wait for it; no work set. The host forms are blocking, through the same kernels; their stats
 * (may be NULL): rays = n, candidates (exact distance evaluations), clusters (leaves visited), nodes (nodes visited), the times,
 * byte counts and kernel_launches; a traversal-guard trip fails the call with RT_ERR_CUDA.
 * RT_ERR_INVALID, before any device work, for a NULL handle, q, q->point or output, an rt_nearest with both outputs NULL, or an
 * overlaps call with a NULL q->bound. n == 0 is a no-op. */
int rtb200_scene_nearest_device(rtb200_scene_handle h, const rt_points* q, uint32_t n, const rt_nearest* out, void* stream);
int rtb200_scene_nearest(rtb200_scene_handle h, const rt_points* q, uint32_t n, const rt_nearest* out, rt_stats* stats);
int rtb200_scene_overlaps_device(rtb200_scene_handle h, const rt_points* q, uint32_t n, uint8_t* overlaps, void* stream);
int rtb200_scene_overlaps(rtb200_scene_handle h, const rt_points* q, uint32_t n, uint8_t* overlaps, rt_stats* stats);

/* ---- radiance of caller-supplied primary rays on a resident scene (DESIGN.md §4.12) --------------------------------------
 * Contract: for ray i (origin, direction as in rt_rays, any f64 values; rays->t_max must be NULL) and sample j < samples, the
 * sample's radiance is ray_color(Ray{o, d}, max_depth, max_depth) (raytracer.rs:71-165) over the handle's CURRENT spheres. It
 * draws from the Philox stream of (pixel = stream0 + i, sample = sample0 + j) under the key `seed`, starting at the stream's
 * third f64 draw: the two draws a render spends on the pixel jitter (raytracer.rs:199-200) are skipped. The outputs are the
 * render's resolve with spp = samples: S_c the f32 sum of the samples in sample order, linear = (1.0f / samples) * S_c,
 * rgb8 = the render's quantisation of sqrt(linear). Bit for bit in every variant, with or without lights, every sky, textures,
 * shard handles (rank / world do not affect rays) and shared-memory-staged handles. So when ray p of a call with sample0 = s
 * and samples = 1 is the render's primary ray of (pixel p, sample s), its output is that sample's radiance, and the f32 sum of
 * such calls in sample order times 1.0f / spp is the render's linear image. */
typedef struct {
    uint64_t seed;        /* Philox key, as rt_scene.seed */
    uint32_t samples;     /* samples of every ray, >= 1 */
    uint32_t sample0;     /* sample index of the first sample */
    uint32_t stream0;     /* ray i draws from the stream of pixel stream0 + i */
    uint32_t max_depth;   /* as rt_scene.max_depth; 0: black, no ray */
    uint32_t reserved[2]; /* must be 0 */
} rt_trace_params;        /* 32 bytes */
/* Device buffers (of h's device, or managed memory): dev_linear_f32 and dev_rgb8 hold n x 3 floats / bytes, either may be NULL,
 * not both. Blocking, like rtb200_render_device: drains the handle's asynchronous frames, takes work set 0 like a blocking render,
 * runs on `stream` (NULL: the library's stream) after the last update or rebuild of h, and returns when the outputs are
 * written. The samples are traced in batches of spb samples of every ray with n * spb * 16 bytes <= the handle's sample-buffer
 * cap (rt_options.sample_buffer_bytes) and n * spb < 2^31; the sums carry across batches. stats (may be NULL): rays (hit_world
 * calls), samples = n * samples, candidates, clusters, nodes, device_ms, trace_ms, wall_ms, kernel_launches, batches (trace
 * launches, or black batches at max_depth 0) and frames = 1. Shadow-frame-stack overflows (RT_ERR_UNSUPPORTED) and
 * traversal-guard trips (RT_ERR_CUDA) fail the call as they fail a render.
 * RT_ERR_INVALID, before any device work, for a NULL handle, rays, params, origin or direction, a non-NULL rays->t_max, both
 * outputs NULL, samples == 0, a nonzero reserved, stream0 + n or sample0 + samples above 2^32, n >= 2^31, n * 16 above the
 * sample-buffer cap (one sample of every ray must fit), or a pointer that is not device memory of h's device or managed
 * memory. n == 0 is a no-op. */
int rtb200_scene_trace_rays_device(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_trace_params* params,
                                   float* dev_linear_f32, uint8_t* dev_rgb8, void* stream, rt_stats* stats);
/* Host buffers: the same through the same path on the library's stream, with the rays copied in and the outputs copied out
 * (h2d_bytes = 48 n, d2h_bytes = 12 n with linear + 3 n with rgb8). Same checks, bar the memory kind. */
int rtb200_scene_trace_rays(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_trace_params* params,
                            float* out_linear_f32, uint8_t* out_rgb8, rt_stats* stats);

/* ---- auxiliary buffers of a resident scene's camera samples (DESIGN.md §4.14) ---------------------------------------------
 * Denoiser guides (albedo, normal), coverage, object ids and hit points of the render's own samples. Contract: for every pixel
 * (x, y) of the handle's rows and every sample s in [sample0, sample0 + samples):
 *   ray      the render's primary ray of (pixel y * width + x, sample s) under the view's camera and seed: the two jitter
 *            draws of raytracer.rs:199-200 from that Philox stream, then Camera::get_ray (camera.rs:79-84);
 *   H        hit_world(world, ray, 0.001, f64::MAX) over the handle's CURRENT spheres (those after the last update, rebuild or
 *            edit enqueued before the call);
 *   albedo_s the attenuation Material::scatter returns at H, without drawing a random number: a Lambertian's or Metal's albedo
 *            as stored (non-finite values included, also where a Metal's scatter would absorb), a Texture's
 *            texture_get_albedo at H's (u, v) with its h_offset (materials.rs:236-253), (1, 1, 1) for Glass and Light; on a
 *            miss the sky of the ray (raytracer.rs:134-163; black for RT_SKY_NONE);
 *   normal_s HitRecord.normal (flipped against the ray, sphere.rs:59-76) with each component rounded to f32; 0 on a miss.
 * Outputs per pixel, compact rows * width and top row first like every output (a shard handle writes its own rows), with the
 * render's resolve arithmetic (f32 sums in sample order, every operation rounded, never contracted):
 *   albedo   3 x f32: (1.0f / samples) * S_c, S_c the f32 sum of albedo_s in sample order;
 *   normal   3 x f32: the same mean of normal_s, not renormalised (mixed surfaces or misses give a shorter vector);
 *   hits     u32: the samples whose H is Some (coverage = hits / samples);
 *   sphere   u32: the hit sphere of sample sample0 (first in list order on equal t), 0xffffffff on a miss;
 *   point    3 x f64: ray.at(t) of sample sample0, 0 on a miss (its distance from the camera origin is the depth).
 * sphere and point equal rtb200_scene_intersect of sample sample0's primary ray bit for bit. Every output is bit for bit the
 * same in every variant, on shard and shared-memory-staged handles, and after updates, rebuilds and edits equals a fresh
 * upload of the same spheres. max_depth plays no part (a handle uploaded with max_depth 0 has AOVs too).
 * view: NULL for the handle's own camera and seed; else view->camera and view->seed, so that the buffers of an animation frame
 * match that frame of rtb200_render_frames[_device]; view->max_depth is ignored. */
typedef struct { uint32_t samples, sample0; uint32_t reserved[2]; } rt_aov_params;   /* 16 bytes; samples >= 1, reserved must be 0 */
typedef struct {              /* every pointer may be NULL: that output is not written */
    float* albedo /* rows x width x 3 */; float* normal /* rows x width x 3 */; uint32_t* hits; uint32_t* sphere;
    double* point /* rows x width x 3 */;
} rt_aov_out;                 /* 40 bytes */
/* Device buffers (of h's device, or managed memory), stream-ordered like rtb200_scene_intersect_device: runs on `stream` (NULL:
 * the library's stream) after the upload and the last update, rebuild or edit of h enqueued before it, without waiting for the
 * GPU; every later update, rebuild and edit and rtb200_scene_release wait for it. It takes no work set and no sample buffer (the
 * sums live in registers). A traversal-guard trip is reported with the handle's next collected frames.
 * RT_ERR_INVALID, before any device work, for a NULL handle, params or out, an out with every output NULL, samples == 0,
 * sample0 + samples above 2^32, a nonzero params->reserved or view->reserved, or a pointer that is not device memory of h's
 * device or managed memory. A shard with no rows is a no-op. */
int rtb200_scene_aov_device(rtb200_scene_handle h, const rt_aov_params* p, const rt_frame* view, const rt_aov_out* out, void* stream);
/* Host buffers, blocking: the same through the same kernel on the library's stream, copied back. stats (may be NULL): rays =
 * samples = pixels * samples, candidates, clusters, nodes, device_ms, trace_ms, wall_ms, d2h_bytes (the outputs asked for plus a
 * 256-byte counter block), kernel_launches = batches = frames = gpus_used = 1. Same checks, bar the memory kind; a
 * traversal-guard trip fails the call with RT_ERR_CUDA. */
int rtb200_scene_aov(rtb200_scene_handle h, const rt_aov_params* p, const rt_frame* view, const rt_aov_out* out, rt_stats* stats);

/* ---- denoising a frame with its auxiliary buffers (DESIGN.md §4.15) -------------------------------------------------------
 * The edge-avoiding à-trous wavelet filter (Dammertz et al. 2010) with rational edge-stopping weights, every f32 operation
 * rounded to nearest and never contracted. Inputs, width x height pixels of 3 x f32, row-major, top row first: color (normally a
 * render's linear mean) and the optional guides albedo and normal (normally rtb200_scene_aov's). A guide is on when it is given
 * and its weight is not 0. Iteration i = 0 .. L-1 reads image c (color for i = 0, else the previous output) with step h = 2^i.
 * Pixel p keeps c_p if any value of p (its colour, and every guide given) is not finite. Otherwise num_k = den = 0 and for
 * dy = -2..2 (outer), dx = -2..2 (inner), q = p + h * (dx, dy), skipping q outside the image or with a non-finite value:
 *   k = B[dx] * B[dy] with B = {1/16, 1/4, 3/8, 1/4, 1/16};
 *   d_g = ((q0 - p0)^2 + (q1 - p1)^2) + (q2 - p2)^2 for each guide on (colour from c, albedo and normal as given);
 *   w = k / ((1 + lc_i * d_c) * (1 + la * d_a) * (1 + ln * d_n)), lc_i = color_weight * 4^i, factors left to right, an off
 *       guide's left out (an overflowing factor gives w = 0);
 *   num_k += w * c_q,k, then den += w.
 * The output is num_k / den (the centre tap alone gives den >= 9/64). Whole frames only: gather a sharded render first.
 * Outputs: out_linear (3 x f32) and/or out_rgb8, the render's quantisation of sqrt(linear) (rtb200_probe_quantise). */
typedef struct {
    uint32_t width, height;
    uint32_t iterations;          /* L, in [1, 10] */
    uint32_t reserved;            /* must be 0 */
    float    color_weight, albedo_weight, normal_weight;   /* finite, >= 0; 0 turns that guide off */
    float    reserved2;           /* must be 0 */
} rt_denoise_params;              /* 32 bytes */
/* Defaults of the Python binding and the CLI (DESIGN.md §4.15: chosen on the 2-spp cover render at 64 x 48) */
#define RTB200_DENOISE_DEFAULT_ITERATIONS    3
#define RTB200_DENOISE_DEFAULT_COLOR_WEIGHT  16.0f
#define RTB200_DENOISE_DEFAULT_ALBEDO_WEIGHT 4.0f
#define RTB200_DENOISE_DEFAULT_NORMAL_WEIGHT 1.0f
/* Bytes of device scratch rtb200_denoise_device needs for width x height pixels (the library owns its layout). */
uint64_t rtb200_denoise_scratch_bytes(uint32_t width, uint32_t height);
/* Device buffers of `device` (-1: the current device) or managed memory; scratch holds rtb200_denoise_scratch_bytes and is
 * 16-byte aligned. Stream-ordered, without waiting for the GPU: runs on `stream` (NULL: the library's stream of that device);
 * the caller keeps every buffer valid until it has run. It touches no scene handle and no work set, so any number of calls
 * with separate scratch may overlap on different streams.
 * RT_ERR_INVALID, before any device work, for a NULL params, color or scratch, both outputs NULL, a nonzero reserved or
 * reserved2, iterations outside [1, 10], a weight that is NaN, negative or infinite, color_weight * 4^(iterations - 1) not
 * finite, a nonzero weight for a NULL guide, width * height >= 2^31, an output or the scratch overlapping an input or each
 * other, or a pointer that is not device memory of `device` nor managed memory. A 0-pixel image is a no-op. */
int rtb200_denoise_device(int32_t device, const rt_denoise_params* p, const float* color, const float* albedo, const float* normal,
                          void* scratch, float* out_linear, uint8_t* out_rgb8, void* stream);
/* Host buffers, blocking: the same through the same kernels on the library's stream, with the inputs copied in and the outputs
 * copied out. stats (may be NULL): device_ms (copies and kernels), trace_ms (the kernels), wall_ms, h2d_bytes, d2h_bytes and
 * kernel_launches (iterations + 1). Same checks, bar the scratch and the memory kind. */
int rtb200_denoise(int32_t device, const rt_denoise_params* p, const float* color, const float* albedo, const float* normal,
                   float* out_linear, uint8_t* out_rgb8, rt_stats* stats);

/* ---- the variance-guided denoise (DESIGN.md §4.18) -------------------------------------------------------------------------
 * The à-trous filter of rtb200_denoise with the colour distance divided by each pixel's prefiltered variance, which is filtered
 * beside the colour (SVGF), every f32 operation rounded to nearest and never contracted. Inputs, width x height pixels of 3 x f32,
 * row-major, top row first: color (normally a render's linear mean), variance (normally the variance of that mean) and the
 * optional guides albedo and normal; a guide is on when it is given and its weight is not 0. eps = variance_floor.
 * Pixel p is ok when its colour, its variance and every guide given are finite and its variance is >= 0 (-0 is). A pixel that
 * is not ok keeps its colour and variance in every iteration. Iteration i = 0 .. L-1 reads colour c and variance var (the inputs
 * for i = 0, else the previous outputs) with step h = 2^i. For each ok p:
 *   v_q = (var_q0 + var_q1) + var_q2;
 *   vbar_p = (sum of g[dx] * g[dy] * v_q) / (sum of g[dx] * g[dy]) over the ok q = p + (dx, dy) inside the image, dx, dy in
 *       -1..1, dy outer, dx inner, g = {1/4, 1/2, 1/4} (step 1 in every iteration), each sum in that order;
 *   num_k = den = nv_k = 0 and for dy = -2..2 (outer), dx = -2..2 (inner), q = p + h * (dx, dy), skipping q outside the image
 *   or not ok:
 *     k = B[dx] * B[dy] with B = {1/16, 1/4, 3/8, 1/4, 1/16};
 *     d_g = ((q0 - p0)^2 + (q1 - p1)^2) + (q2 - p2)^2 for each guide on (colour from c, albedo and normal as given);
 *     f = (1 + lc * (d_c / (eps + vbar_p))) * (1 + la * d_a) * (1 + ln * d_n), factors left to right, the colour factor left
 *         out when lc = 0 and an off guide's left out (f = 1 when none is on); lc is not scaled by 4^i;
 *     w = k / f; num_k += w * c_q,k; den += w; nv_k += (w * w) * var_q,k.
 *   The outputs are num_k / den and nv_k / (den * den); p stays ok when all six are finite.
 * Outputs (each may be NULL, not all three): out_linear (3 x f32), out_rgb8 (the render's quantisation of sqrt(linear), as
 * rtb200_probe_quantise) and out_variance (3 x f32). Whole frames only: gather a sharded render first. */
typedef struct {
    uint32_t width, height;
    uint32_t iterations;          /* L, in [1, 10] */
    uint32_t reserved;            /* must be 0 */
    float    color_weight, albedo_weight, normal_weight;   /* finite, >= 0; 0 turns that guide off */
    float    variance_floor;      /* eps: finite, > 0 */
} rt_denoise_var_params;          /* 32 bytes */
/* Defaults of the Python binding and the CLI (DESIGN.md §4.18: chosen on the cover render at 64 x 48, 2 to 32 spp). On frames of
 * 800 x 600 and 1920 x 1080 they lose to rtb200_denoise's defaults at 4 and 8 spp and win from 16 spp up. */
#define RTB200_DENOISE_VAR_DEFAULT_ITERATIONS     3
#define RTB200_DENOISE_VAR_DEFAULT_COLOR_WEIGHT   1.0f
#define RTB200_DENOISE_VAR_DEFAULT_ALBEDO_WEIGHT  4.0f
#define RTB200_DENOISE_VAR_DEFAULT_NORMAL_WEIGHT  1.0f
#define RTB200_DENOISE_VAR_DEFAULT_VARIANCE_FLOOR 1e-4f
/* Bytes of device scratch rtb200_denoise_var_device needs for width x height pixels (the library owns its layout). */
uint64_t rtb200_denoise_var_scratch_bytes(uint32_t width, uint32_t height);
/* Device buffers of `device` (-1: the current device) or managed memory; scratch holds rtb200_denoise_var_scratch_bytes and is
 * 16-byte aligned. Stream-ordered as rtb200_denoise_device: runs on `stream` (NULL: the library's stream of that device)
 * without waiting, touches no scene handle and no work set.
 * RT_ERR_INVALID, before any device work, for a NULL params, color, variance or scratch, all three outputs NULL, a nonzero
 * reserved, iterations outside [1, 10], a weight that is NaN, negative or infinite, a variance_floor that is not finite or not
 * > 0, a nonzero weight for a NULL guide, width * height >= 2^31, a buffer that is not 4-byte aligned, an output or the scratch
 * overlapping an input or each other, or a pointer that is not device memory of `device` nor managed memory. A 0-pixel image
 * is a no-op. */
int rtb200_denoise_var_device(int32_t device, const rt_denoise_var_params* p, const float* color, const float* variance,
                              const float* albedo, const float* normal, void* scratch, float* out_linear, uint8_t* out_rgb8,
                              float* out_variance, void* stream);
/* Host buffers, blocking: the same through the same kernels on the library's stream, with the inputs copied in and the outputs
 * copied out. stats (may be NULL): device_ms, trace_ms (the kernels), wall_ms, h2d_bytes, d2h_bytes and kernel_launches
 * (2 * iterations + 1). Same checks, bar the scratch and the memory kind. */
int rtb200_denoise_var(int32_t device, const rt_denoise_var_params* p, const float* color, const float* variance,
                       const float* albedo, const float* normal, float* out_linear, uint8_t* out_rgb8, float* out_variance,
                       rt_stats* stats);

/* ---- temporal accumulation of animation frames (DESIGN.md §4.16; the history clamp below, §4.20) --------------------------
 * Blends each pixel of a frame with the history of the previous frame where its first hit was, the reprojection and blend of
 * SVGF's first stage. Every f64 and f32 operation is rounded to nearest and never contracted; sums and products run in the
 * order written. Whole frames only (width x height pixels, row-major, top row first): a shard's compact rows are not image
 * neighbours. Inputs of this frame (rt_temporal_frame): color 3 x f32 (normally a render's linear mean), sphere u32 and
 * point 3 x f64 (rtb200_scene_aov's sphere and point of the same camera; 0xffffffff is a miss), camera = p->camera. The previous
 * frame (rt_temporal_history, or NULL for none): the previous call's output color and length, the previous frame's AOV sphere
 * and point, and p->prev_camera. motion (may be NULL when n_motion is 0): n_motion x 3 f64, the displacement of sphere j since
 * the previous frame (its current centre minus its previous one); spheres j >= n_motion did not move. N = p->max_history.
 * Per pixel p = (x, y), with c = color[p]:
 *  1. if c has a non-finite value or there is no previous frame: the output is c, length 1. Otherwise:
 *  2. a hit (j = sphere[p] != 0xffffffff): P = point[p], P' = P - motion[j] (P when j >= n_motion), D_cur = P - camera.origin,
 *     D_prev = P' - prev_camera.origin. A miss: D_cur = D_prev = Camera::get_ray's direction under camera at the pixel centre,
 *     u = (x + 0.5) / (W - 1), v = (H - (y + 0.5)) / (H - 1) (camera.rs:79-84, raytracer.rs:199-200 with both draws 0.5).
 *  3. the projection of D into a camera {origin, llc, h, vt}: a = llc - origin; cn = h x vt, cu = vt x a, cv = a x h (cross
 *     products (y1 z2 - z1 y2, z1 x2 - x1 z2, x1 y2 - y1 x2), dot products (x + y) + z); den = cn . D; u = (cu . D) / den,
 *     v = (cv . D) / den. It is valid when den != 0, (cn . a) / den > 0 (in front of the camera), and u and v are finite.
 *  4. (u_c, v_c) of D_cur under camera, (u_p, v_p) of D_prev under prev_camera; fx = x + (u_p - u_c) * (W - 1),
 *     fy = y - (v_p - v_c) * (H - 1). No history if a projection is invalid or fx or fy is not finite. A static camera with no
 *     motion gives fx = x, fy = y exactly: the motion is measured at the sample's own point and applied to the pixel centre.
 *  5. x0 = floor(fx), y0 = floor(fy), ax = f32(fx - x0), ay = f32(fy - y0); taps (x0, y0), (x0+1, y0), (x0, y0+1),
 *     (x0+1, y0+1) in that order with f32 weights (1-ax)(1-ay), ax(1-ay), (1-ax)ay, ax ay. Tap q is valid when its weight is
 *     > 0, it is inside the image, length[q] >= 1, the history colour of q is finite, the previous sphere of q is sphere[p] and,
 *     for a hit, |prev_point[q] - P'|^2 <= (depth_tol * depth_tol) * |D_prev|^2 (|v|^2 = v . v, f64).
 *  6. s = the f32 sum of the valid taps' weights in tap order; s = 0 is no history. Else h_k = (sum of w * hist_k in tap
 *     order) / s, L = the least length of the valid taps, n = min(L, N - 1) + 1 (no overflow at L = 2^32 - 1), and for n >= 2
 *     the output is h_k + (1.0f / f32(n)) * (c_k - h_k) with length n. No history (or n = 1) is c with length 1.
 * A history must ping-pong between two buffers: an output may not overlap any input. After an edit that renumbers spheres
 * (rtb200_scene_edit_spheres), pass no previous frame. */
typedef struct {
    uint32_t  width, height;
    uint32_t  max_history;        /* N >= 1: a pixel's history is the mean of at most its last N frames */
    uint32_t  n_motion;           /* rows of motion */
    rt_camera camera, prev_camera;   /* this frame's and the previous frame's (prev_camera is ignored without a previous frame) */
    double    depth_tol;          /* finite, >= 0: a relative depth tolerance */
    uint32_t  reserved[2];        /* must be 0 */
} rt_temporal_params;             /* 224 bytes */
typedef struct { const float* color; const uint32_t* sphere; const double* point; } rt_temporal_frame;   /* 24 bytes */
typedef struct { const float* color; const uint32_t* length; const uint32_t* sphere; const double* point; } rt_temporal_history;   /* 32 bytes */
typedef struct { float* color; uint32_t* length; } rt_temporal_out;   /* 16 bytes: the new history */
/* Defaults of the Python binding and the CLI (DESIGN.md §4.16: chosen on an orbit of the 2-spp cover render at 64 x 48) */
#define RTB200_TEMPORAL_DEFAULT_MAX_HISTORY 2
#define RTB200_TEMPORAL_DEFAULT_DEPTH_TOL   0.03
/* Device buffers of `device` (-1: the current device) or managed memory. Stream-ordered, without waiting for the GPU: runs on
 * `stream` (NULL: the library's stream of that device); the caller keeps every buffer valid until it has run. It needs no
 * scratch and touches no scene handle and no work set.
 * RT_ERR_INVALID, before any device work, for a NULL params, cur, cur->color, cur->sphere, cur->point, out, out->color or
 * out->length, a prev with a NULL member, a nonzero reserved, max_history 0, a depth_tol that is NaN, negative or infinite, a
 * NULL motion with n_motion > 0, width * height >= 2^31, a misaligned pointer (4 bytes for f32 and u32 arrays, 8 for f64), an
 * output overlapping an input or the other output, or a pointer that is not device memory of `device` nor managed memory.
 * A 0-pixel image is a no-op. */
int rtb200_temporal_device(int32_t device, const rt_temporal_params* p, const rt_temporal_frame* cur, const rt_temporal_history* prev,
                           const double* motion, const rt_temporal_out* out, void* stream);
/* Host buffers, blocking: the same through the same kernel on the library's stream, with the inputs copied in and the outputs
 * copied out. stats (may be NULL): device_ms (copies and kernel), trace_ms (the kernel), wall_ms, h2d_bytes, d2h_bytes and
 * kernel_launches (1). Same checks, bar the alignment and the memory kind. */
int rtb200_temporal(int32_t device, const rt_temporal_params* p, const rt_temporal_frame* cur, const rt_temporal_history* prev,
                    const double* motion, const rt_temporal_out* out, rt_stats* stats);

/* ---- the history clamp of the temporal accumulation (DESIGN.md §4.20) -----------------------------------------------------
 * rtb200_temporal with one more step between step 6's h and the blend; steps 1-5, the tap rules, L, n and every no-history case
 * are unchanged. Where n >= 2, for pixel p, window radius r and clamp width gamma:
 *  7. the window is q = p + (dx, dy), dy = -r..r (outer), dx = -r..r (inner); the q inside the image whose colour color[q] is
 *     finite in all three channels are kept, m of them (p itself always is: m >= 1). Per channel k, in f32 from 0.0f and in
 *     window order: S_k += c_q,k and Q_k += c_q,k * c_q,k (the product rounded before the add). mean = S_k / f32(m),
 *     var = Q_k / f32(m) - mean * mean, sd = sqrt(var < 0 ? 0 : var) (a NaN var stays NaN), lo = mean - gamma * sd,
 *     hi = mean + gamma * sd, and h'_k = h_k < lo ? lo : (h_k > hi ? hi : h_k), so a NaN lo, hi or h_k leaves h_k as it is.
 *     The output is h'_k + (1.0f / f32(n)) * (c_k - h'_k) with length n: the clamp does not shorten the history.
 * Every operation is rounded to nearest and never contracted. The clamp rejects a history whose colour the current frame's
 * neighbourhood does not show, such as a reflection that moved across the surface the reprojection follows. */
typedef struct {
    float    gamma;               /* finite, >= 0: the clamp's width in standard deviations (0: the window mean) */
    uint32_t radius;              /* r in [1, 3]: a (2r + 1) x (2r + 1) window */
    uint32_t reserved[2];         /* must be 0 */
} rt_temporal_clamp;              /* 16 bytes */
/* Defaults of the Python binding and the CLI's clamp (DESIGN.md §4.20: chosen on 16 frames of C2 at 4 spp and of C2 with its metal
 * and glass Lambertian, under a one-degree orbit and a still camera, against 1024-spp frames; at N = 2 they beat the denoise
 * alone on C2's orbit, where the unclamped accumulation loses to it) */
#define RTB200_TEMPORAL_DEFAULT_CLAMP_GAMMA  0.5f
#define RTB200_TEMPORAL_DEFAULT_CLAMP_RADIUS 1
/* rtb200_temporal_device with the history clamp: the same buffers, stream order and checks, and RT_ERR_INVALID, before any
 * device work, for a NULL clamp, a gamma that is NaN, negative or infinite, a radius outside [1, 3] or a nonzero reserved. */
int rtb200_temporal_clamped_device(int32_t device, const rt_temporal_params* p, const rt_temporal_clamp* clamp, const rt_temporal_frame* cur,
                                   const rt_temporal_history* prev, const double* motion, const rt_temporal_out* out, void* stream);
/* rtb200_temporal with the history clamp: host buffers, blocking, the same stats and checks, and the clamp's checks above. */
int rtb200_temporal_clamped(int32_t device, const rt_temporal_params* p, const rt_temporal_clamp* clamp, const rt_temporal_frame* cur,
                            const rt_temporal_history* prev, const double* motion, const rt_temporal_out* out, rt_stats* stats);

/* ---- the variance of each pixel's mean through the temporal accumulation (DESIGN.md §4.21) ---------------------------------
 * rtb200_temporal (clamp NULL) or rtb200_temporal_clamped (clamp given) with one more output; steps 1-7, the tap rules, L, n and
 * the clamp are unchanged and never read a variance, so out->color and out->length are those calls' outputs bit for bit. New
 * arrays, 3 x f32 per pixel, row-major like color: variance, this frame's variance of its pixel mean (normally from
 * rtb200_render_frames_var[_device]); prev_variance, the previous call's out_variance, given exactly when prev is; and
 * out_variance, the new history's. Per pixel p with this frame's variance v:
 *  8. with no history (a non-finite c, no previous frame, an invalid projection, s = 0 or n = 1) out_variance = v as given
 *     (NaN, infinities, negative values and -0 included). For n >= 2: Vh_k = (sum of w * prev_variance_q,k over step 5's valid
 *     taps, in tap order, from 0.0f) / s, with step 5's weights w and step 6's s (a non-finite tap variance does not make a tap
 *     invalid: it propagates); a = 1.0f / f32(n), b = 1.0f - a, and out_variance_k = (b * b) * Vh_k + (a * a) * v_k. The clamp
 *     moves the history's colour only, not Vh.
 * Every f32 operation is rounded to nearest and never contracted. The blend b h + a c of a history and a frame of another seed has
 * variance b^2 Var(h) + a^2 v; the linear weights give an upper bound on the variance of the correlated taps' resample. A static
 * camera with a constant v gives v / k after k <= N frames and a v / (2 - a) past N. */
/* Device buffers of `device` (-1: the current device) or managed memory, stream-ordered as rtb200_temporal_device. The checks of
 * rtb200_temporal_device, the clamp's of rtb200_temporal_clamped_device when clamp is given, and RT_ERR_INVALID, before any
 * device work, for a NULL variance or out_variance, a prev without prev_variance or a prev_variance without prev, a variance
 * array that is not 4-byte aligned, an out_variance overlapping an input or another output, an out->color or out->length
 * overlapping variance or prev_variance, or a variance pointer that is not device memory of `device` nor managed memory.
 * A 0-pixel image is a no-op. */
int rtb200_temporal_var_device(int32_t device, const rt_temporal_params* p, const rt_temporal_clamp* clamp, const rt_temporal_frame* cur,
                               const float* variance, const rt_temporal_history* prev, const float* prev_variance, const double* motion,
                               const rt_temporal_out* out, float* out_variance, void* stream);
/* Host buffers, blocking: the same through the same kernel on the library's stream, with the inputs copied in and the outputs
 * copied out; stats as rtb200_temporal's (kernel_launches 1). Same checks, bar the alignment and the memory kind. */
int rtb200_temporal_var(int32_t device, const rt_temporal_params* p, const rt_temporal_clamp* clamp, const rt_temporal_frame* cur,
                        const float* variance, const rt_temporal_history* prev, const float* prev_variance, const double* motion,
                        const rt_temporal_out* out, float* out_variance, rt_stats* stats);

/* load_texture_image — materials.rs:213-219, config.rs:36-47: decode a baseline JPEG file to RGB8 (host-side scene staging
 * helper for hosts without their own decoder; the reference uses the jpeg-decoder crate). *out_rgb8 is released with rtb200_free(). */
int  rtb200_decode_jpeg_file(const char* path, uint8_t** out_rgb8, uint64_t* width, uint64_t* height);
void rtb200_free(void* p);

/* Diagnostic, host only (no GPU needed): what the closest-hit stage of hit_world (raytracer.rs:44-59) would read for `scene`:
 * recentring offset; the 8-wide BVH nodes (floats_per_node floats each: lo_x[8] lo_y[8] lo_z[8] hi_x[8] hi_y[8] hi_z[8]
 * child[8], child = 0xffffffff empty | 0x80000000+leaf | node); the leaves (leaf_size pair-packed sphere records
 * {cx0,cx1,cy0,cy1},{cz0,cz1,nk0,nk1} + slot -> sphere index, 0xffffffff = padding); the spheres tested for every ray; the
 * flat records of RT_VARIANT_BRUTE_FORCE. info = {n_nodes, n_leaves, depth, leaf_size, n_always, floats_per_node, flat_pairs, 0}.
 * Arrays are filled up to their capacities (elements). */
int rtb200_debug_bvh(const rt_scene* scene, double recentre[3], uint32_t info[8], float* nodes, uint64_t cap_nodes,
                     float* leaf_rec, uint64_t cap_leaf_rec, uint32_t* leaf_id, uint64_t cap_leaf_id,
                     uint32_t* always, uint64_t cap_always, float* flat, uint64_t cap_flat);

/* Device-function probes: run the kernel's own device routines on one thread and return the result,
 * so the reference's known-answer tests can be asserted against the GPU code itself.
 *   sphere.rs:81-88, materials.rs:157-174, raytracer.rs:167-189, camera.rs:105-122 */
int rtb200_probe_sphere_hit(const rt_vec3* center, double radius, const rt_vec3* origin, const rt_vec3* dir,
                            double t_min, double t_max, int32_t* hit, double* t, rt_vec3* point, rt_vec3* normal,
                            int32_t* front_face);
int rtb200_probe_refract(const rt_vec3* uv, const rt_vec3* n, double etai_over_etat, rt_vec3* out);
int rtb200_probe_reflectance(double cosine, double ref_idx, double* out);
int rtb200_probe_sky(const rt_vec3* dir, uint32_t sky_mode, float out_rgb[3]);
int rtb200_probe_get_ray(const rt_camera* cam, double u, double v, rt_vec3* origin, rt_vec3* dir);
/* The lens ray of (pixel, sample) under `seed` at the jittered (u, v) (DESIGN.md §4.17), by the kernel's own lens routine;
 * *trials (may be NULL) = lens trials drawn (0 for a pinhole lens). lens NULL: pinhole. Same lens checks as rtb200_scene_set_lens. */
int rtb200_probe_lens_ray(const rt_camera* cam, const rt_lens* lens, uint64_t seed, uint32_t pixel, uint32_t sample, double u,
                          double v, rt_vec3* origin, rt_vec3* dir, uint32_t* trials);
/* n uniform draws of the per-(pixel,sample) stream: kind 0 = gen::<f64>() in [0,1), 1 = gen_range(-1.0..1.0) */
int rtb200_probe_rng(uint64_t seed, uint32_t pixel, uint32_t sample, uint32_t kind, uint32_t n, double* out);
/* u_v_from_sphere_hit_point (sphere.rs:35-43) of n vectors hp = hit point - centre (3 doubles each); out = n {u, v} pairs */
int rtb200_probe_sphere_uv(const double* hp_xyz, uint32_t n, double* out_uv);
/* u8 quantisation of raytracer.rs:207-213 for n linear means */
int rtb200_probe_quantise(const float* mean_linear, uint32_t n, uint8_t* out);

#ifdef __cplusplus
}
#endif
#endif /* RTB200_H */
