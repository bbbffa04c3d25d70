// rtb200_api_render.cu — rendering through the C ABI: work sets and submissions, the trace step every submission's batches
// go through, the frame scheduler (render_enqueue / render_collect), every render entry point (resident, one-shot and
// multi-GPU), the radiance of caller-supplied rays and adaptive rendering.

#include "rtb200_host.cuh"

using namespace rtk;

// resident CTAs per SM of one trace kernel with `smem` bytes of dynamic shared memory (cached per context)
static int occupancy(DeviceCtx* ctx, uint32_t mode, bool lights, uint32_t queue, size_t smem) {
    for (auto& k : ctx->occ_cache) if (k.mode == mode && k.lights == lights && k.queue == queue && k.smem == smem) return k.occ;
    const int occ = wavefront_max_ctas_per_sm(mode, lights, queue, smem);
    ctx->occ_cache.push_back(DeviceCtx::OccKey{mode, lights, queue, smem, occ});
    return occ;
}

int rtk::launch_geometry(rtb200_scene_handle h, uint32_t queue, bool lights, LaunchGeom* g) {
    static const char* const kernel[4] = {"", " of the multi-frame trace kernel", " of the list trace kernel", " of the rays trace kernel"};
    g->smem = wavefront_smem_bytes(h->tp, h->mode, h->tp.scene_in_smem, queue);
    g->ctas_per_sm = occupancy(h->ctx, h->mode, lights, queue, g->smem);
    if (g->ctas_per_sm <= 0) return fail(RT_ERR_UNSUPPORTED, std::string("no launch configuration") + kernel[base_queue(queue)] + " fits shared memory");
    g->grid = h->ctx->sm_count * g->ctas_per_sm;
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

// ---- submissions: what one call enqueues on one stream with one work set, reported by render_collect ----
// A submission of h on `stream_in` (NULL: the context's stream) with work set `set` starts after the previous submission that
// took the same set, on any stream and of any handle, has finished with it; the caller holds the context's lock.
// submission_open picks the stream (scene_stream); submission_begin sizes the set's buffers
// (prepare_work), orders the stream after the set's last user, uploads the frame table, takes the timing events (begin, end,
// a pair per batch), clears the stat block and the queue counters and records the begin event; trace_step enqueues one batch;
// submission_close records the end event, snapshots the stat block and appends the submission to h->pending. A submission
// that fails part-way is not recorded.
// An open submission: its record, stream and work set, its timing events and the queue counters of its batches.
struct Submit {
    rtb200_scene_t::Submission sub;
    cudaStream_t st;
    DeviceCtx::WorkSet* W;
    cudaEvent_t* ev;                     // ev[0] begin, ev[1] end, ev[2 + 2b] and ev[3 + 2b] around batch b
    unsigned int* counters;
};

static int submission_open(rtb200_scene_handle h, void* stream_in, uint32_t frames, Submit* s) {
    if (h->pending.size() >= kMaxPending) return fail(RT_ERR_INVALID, "more than 64 frames enqueued without rtb200_render_device_wait");
    CU(cudaSetDevice(h->device));
    CU(scene_stream(h, stream_in, &s->st));
    const rtb200_scene_t::Submission* prev = h->pending.empty() ? nullptr : &h->pending.back();
    s->sub = rtb200_scene_t::Submission{s->st, prev ? prev->ev0 + prev->n_ev : 0u, 0, frames, 0, 0, h->grid, 0, 0};
    return RT_OK;
}

// The opened submission s in `batches` batches, whose widest trace launch has `grid` CTAs, for paths up to max_depth deep that
// stage up to samplebuf_bytes of samples; points tp at the set's buffers. The multi-frame kernel reads each frame's camera and
// key from the n_ftab records of `ftab` (and, when ltab is not null, its lens from n_ftab lenses of `ltab`), copied here
// because the copy has to come after the wait for the set's last user and before the stat block is cleared.
static int submission_begin(rtb200_scene_handle h, int set, uint32_t batches, int grid, TraceParams& tp, uint32_t max_depth,
                            size_t samplebuf_bytes, const FrameRec* ftab, uint32_t n_ftab, Submit* s, const rt_lens* ltab = nullptr) {
    DeviceCtx* ctx = h->ctx;
    DeviceCtx::WorkSet& W = ctx->ws[set];
    rtb200_scene_t::Submission& sub = s->sub;
    const cudaStream_t st = s->st;
    s->W = &W;
    sub.batches = batches;
    sub.grid = grid;
    const uint32_t threads_total = (uint32_t)grid * (uint32_t)kBlock;   // ray slots of the widest grid: columns of the per-slot global arrays
    const int rc = prepare_work(W, tp, threads_total, max_depth, samplebuf_bytes, batches);
    if (rc != RT_OK) return rc;
    CU(cudaStreamWaitEvent(st, W.done, 0));   // nothing below touches the set before its previous submission is done with it
    if (n_ftab) {
        sub.ftab_bytes = (uint64_t)n_ftab * sizeof(FrameRec);
        CU(W.ftab.ensure(sub.ftab_bytes, W.done));
        CU(cudaMemcpyAsync(W.ftab.p, ftab, sub.ftab_bytes, cudaMemcpyHostToDevice, st));
        if (ltab) {
            const uint64_t lbytes = (uint64_t)n_ftab * sizeof(rt_lens);
            CU(W.ltab.ensure(lbytes, W.done));
            CU(cudaMemcpyAsync(W.ltab.p, ltab, lbytes, cudaMemcpyHostToDevice, st));
            sub.ftab_bytes += lbytes;
        }
    }
    sub.n_ev = 2 + 2 * batches;
    while (h->ev.size() < (size_t)sub.ev0 + sub.n_ev) {
        cudaEvent_t e;
        if (!ctx->event_pool.empty()) { e = ctx->event_pool.back(); ctx->event_pool.pop_back(); }
        else CU(cudaEventCreate(&e));
        h->ev.push_back(e);
    }
    s->ev = h->ev.data() + sub.ev0;
    CU(cudaMemsetAsync(W.small.p, 0, kStatBytes + (size_t)batches * 4, st));
    CU(cudaMemsetAsync((char*)W.small.p + 64, 0xff, 16, st));   // stat[8], stat[9]: minima (kernel start / first dry-queue time, ns)
    CU(cudaEventRecord(s->ev[0], st));
    s->counters = (unsigned int*)((char*)W.small.p + kStatBytes);
    return RT_OK;
}

// Batch b of submission s between its event pair: the trace launch of q on `queue` with launch geometry g (q takes the
// batch's queue counter and the grid's stack stride), or at max_depth 0 a zero fill of black_bytes of q.samplebuf, since
// ray_color(depth 0) is black and traces no ray (raytracer.rs:80-82).
static int trace_step(rtb200_scene_handle h, const Submit& s, uint32_t b, TraceParams& q, uint32_t queue, const LaunchGeom& g, size_t black_bytes) {
    q.work_counter = s.counters + b;
    q.stack_stride = (uint32_t)g.grid * (uint32_t)kBlock;
    CU(cudaEventRecord(s.ev[2 + 2 * b], s.st));
    if (q.max_depth == 0) CU(cudaMemsetAsync(q.samplebuf, 0, black_bytes, s.st));
    else CU(launch_wavefront(q, h->mode, queue, g.grid, g.smem, s.st));
    CU(cudaEventRecord(s.ev[3 + 2 * b], s.st));
    return RT_OK;
}

static int submission_close(rtb200_scene_handle h, const Submit& s) {
    CU(cudaEventRecord(s.ev[1], s.st));
    CU(cudaMemcpyAsync(h->stat_snap + h->pending.size() * (kStatBytes / 8), s.W->small.p, kStatBytes, cudaMemcpyDeviceToDevice, s.st));
    CU(cudaEventRecord(s.W->done, s.st));
    h->pending.push_back(s.sub);
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

// rt_frame checks (and of the per-frame lenses, when not null) shared by the frames entry points (no device is touched)
static int check_frames(const rt_frame* frames, uint32_t n, uint64_t rows, uint64_t width, const rt_lens* lenses) {
    if (n == 0) return fail(RT_ERR_INVALID, "n_frames must be > 0");
    if (!frames) return fail(RT_ERR_INVALID, "frames is null");
    const uint64_t per_frame = rows * width * 3ull;   // < 2^33: width * height < 2^31 (validate_scene)
    if (per_frame != 0 && (uint64_t)n > ~0ull / per_frame) return fail(RT_ERR_INVALID, "n_frames * rows * width * 3 overflows 64 bits");
    for (uint32_t i = 0; i < n; ++i)
        if (frames[i].reserved != 0) return fail(RT_ERR_INVALID, "rt_frame.reserved must be 0 (frame " + std::to_string(i) + ")");
    if (lenses)
        for (uint32_t i = 0; i < n; ++i) {
            const int rc = check_lens(lenses[i], ("lens of frame " + std::to_string(i)).c_str());
            if (rc != RT_OK) return rc;
        }
    return RT_OK;
}

// The handle's own view (the camera, seed and depth it was uploaded with) as a frame.
static rt_frame own_frame(rtb200_scene_handle h) { return rt_frame{h->tp.cam, h->tp.key0 | (uint64_t)h->tp.key1 << 32, h->tp.max_depth, 0}; }

// Enqueue frames[0, n) of h on `stream_in` (NULL: the context's stream) with work set `set`, without waiting, and append the
// submission to h->pending; the caller holds the context's lock and has made h's device current. Frame i goes to output
// slice i (rows * width * 3 elements). Frame i's lens is lenses[i], or the handle's (h->tp.lens) when lenses is null. When no
// frame has a lens the launches are the pinhole ones; else every group, one frame or many, runs the multi-frame kernel with
// the lens (Q_FRAMES_LENS), which reads each frame's camera, key and lens from the frame and lens tables.
// With dev_var (n * rows * width * 3 f32), the resolve is rt_resolve_var_kernel, which also writes each frame's variance of
// the pixel means and carries the sums of squares across batches in the set's accum_sq.
static int render_enqueue(rtb200_scene_handle h, const rt_frame* frames, uint32_t n, void* dev_rgb8, void* dev_linear_f32,
                          void* stream_in, int set, const rt_lens* lenses = nullptr, float* dev_var = nullptr) {
    Submit s;
    int rc = submission_open(h, stream_in, n, &s);
    if (rc != RT_OK) return rc;
    TraceParams tp = h->tp;   // the handle's own view stays as uploaded
    const uint64_t npl = tp.npix_local;
    if (npl == 0) { h->pending.push_back(s.sub); return RT_OK; }   // a shard with no rows: nothing to trace
    const uint32_t spp = tp.spp, spb = h->spp_batch, n_batches = (spp + spb - 1) / spb;
    const uint64_t frame_work = (uint64_t)spp * npl;
    const std::vector<FrameGroup> groups = frame_groups(frames, n, frame_work, sample_buffer_cap(h->opts));
    // A batch of a group holds spb samples of each of its frames. A group of F >= 2 frames is one batch: frame_groups admits
    // it only when 2 * spp * npl * 16 bytes fit the cap and 2 * spp * npl < 2^31, and with these samples_per_batch gave
    // spp_batch == spp.
    auto batches_of = [&](const FrameGroup& g) { return g.count > 1 ? 1u : n_batches; };
    std::vector<rt_lens> ltab;   // each frame's lens, when one of them has a lens
    for (uint32_t i = 0; i < n && ltab.empty(); ++i)
        if ((lenses ? lenses[i] : tp.lens).radius != 0.0) ltab.resize(n);
    for (uint32_t i = 0; i < ltab.size(); ++i) {
        const rt_lens& L = lenses ? lenses[i] : tp.lens;
        ltab[i] = L.radius != 0.0 ? L : rt_lens{};
    }
    const bool lensed = !ltab.empty();

    // trace launches, work buffer sizes and the launch geometry of the multi-frame kernel (its pool also holds the slots' frames)
    const LaunchGeom single{h->smem, h->ctas_per_sm, h->grid};
    LaunchGeom multi{0, 0, 0};
    uint32_t all_batches = 0, max_depth = 1;
    size_t sbuf = 0;
    for (const FrameGroup& g : groups) {
        all_batches += batches_of(g);   // trace launches (or black memsets)
        sbuf = std::max(sbuf, (size_t)g.count * spb * npl * 16);
        max_depth = std::max(max_depth, frames[g.first].max_depth);
        if ((g.count > 1 || lensed) && multi.grid == 0 && (rc = launch_geometry(h, lensed ? Q_FRAMES_LENS : Q_FRAMES, tp.n_lights > 0, &multi)) != RT_OK)
            return rc;
    }
    std::vector<FrameRec> tab(multi.grid ? n : 0);
    for (uint32_t i = 0; i < tab.size(); ++i) {
        tab[i].cam = frames[i].camera; tab[i].key0 = (uint32_t)frames[i].seed; tab[i].key1 = (uint32_t)(frames[i].seed >> 32);
    }
    if (dev_var) CU(h->ctx->ws[set].accum_sq.ensure((size_t)npl * 12, h->ctx->ws[set].done));
    if ((rc = submission_begin(h, set, all_batches, std::max(h->grid, multi.grid), tp, max_depth, sbuf, tab.data(),
                               (uint32_t)tab.size(), &s, lensed ? ltab.data() : nullptr)) != RT_OK)
        return rc;

    uint32_t b = 0;   // trace launch (or black memset) index: its queue counter and its event pair
    for (const FrameGroup& g : groups) {
        const rt_frame& f0 = frames[g.first];
        const bool is_multi = g.count > 1 || lensed;   // the multi-frame trace kernel, which reads each frame's camera and key from ftab
        const uint32_t batches = batches_of(g);
        uint8_t* o8 = dev_rgb8 ? (uint8_t*)dev_rgb8 + (size_t)g.first * npl * 3 : nullptr;
        float* ol = dev_linear_f32 ? (float*)dev_linear_f32 + (size_t)g.first * npl * 3 : nullptr;
        TraceParams q = tp;
        q.max_depth = f0.max_depth;
        if (is_multi) {
            q.ftab = (const FrameRec*)s.W->ftab.p + g.first;
            if (lensed) q.ltab = (const rt_lens*)s.W->ltab.p + g.first;
        } else {
            q.cam = f0.camera; q.key0 = (uint32_t)f0.seed; q.key1 = (uint32_t)(f0.seed >> 32);
        }
        for (uint32_t k = 0; k < batches; ++k, ++b) {
            q.s0 = k * spb;
            q.s_count = std::min(spb, spp - q.s0);
            q.total_work = g.count * q.s_count * q.npix_local;
            if (is_multi) q.frame_work = q.s_count * q.npix_local;   // frame_work of a group of several frames (one batch of spp)
            const uint32_t queue = !is_multi ? Q_SINGLE : lensed ? Q_FRAMES_LENS : Q_FRAMES;
            if ((rc = trace_step(h, s, b, q, queue, is_multi ? multi : single, (size_t)q.total_work * 16)) != RT_OK) return rc;
            for (uint32_t j = 0; j < g.count; ++j) {   // samplebuf [frame][sample][pixel]
                ResolveParams r{};
                r.samplebuf = q.samplebuf + (size_t)j * q.s_count * npl; r.accum = (float*)s.W->accum.p; r.npix_local = q.npix_local;
                r.s_count = q.s_count; r.first = k == 0; r.last = k + 1 == batches; r.spp = spp;
                r.out_linear = ol ? ol + (size_t)j * npl * 3 : nullptr; r.out_rgb8 = o8 ? o8 + (size_t)j * npl * 3 : nullptr;
                if (dev_var) {
                    const ResolveVarParams v{r, (float*)s.W->accum_sq.p, dev_var + ((size_t)g.first + j) * npl * 3};
                    CU(launch_resolve_var(v, s.st));
                } else {
                    CU(launch_resolve(r, s.st));
                }
            }
        }
        s.sub.launches += batches * (1 + g.count);
        if (q.max_depth == 0) s.sub.black_samples += g.count * frame_work;
    }
    return submission_close(h, s);
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

// Counters, batches and the diagnostics are the last submission's (from its copy of the stat block); times, frames, kernel
// launches and frame-table bytes are summed over the submissions.
int rtk::render_collect(rtb200_scene_handle h, rt_stats* stats) {
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

// A blocking call on h: drain its asynchronous frames, enqueue one submission on work set 0 (`enqueue`), wait for it and
// report it in stats (may be NULL) with the wall time of the three. The caller holds the context's lock.
template <typename Enqueue>
static int blocking(rtb200_scene_handle h, rt_stats* stats, Enqueue&& enqueue) {
    const auto wall0 = std::chrono::steady_clock::now();
    int rc = render_collect(h, nullptr);
    if (rc == RT_OK) rc = enqueue();
    if (rc == RT_OK) rc = render_collect(h, stats);
    if (rc == RT_OK && stats) stats->wall_ms = ms_since(wall0);
    return rc;
}

static int render_blocking(rtb200_scene_handle h, const rt_frame* frames, uint32_t n, void* dev_rgb8, void* dev_linear_f32,
                           void* stream_in, rt_stats* stats, const rt_lens* lenses = nullptr, float* dev_var = nullptr) {
    HANDLE_PROLOGUE(h);
    return blocking(h, stats, [&] { return render_enqueue(h, frames, n, dev_rgb8, dev_linear_f32, stream_in, 0, lenses, dev_var); });
}

// Releases a scene handle on scope exit; the error that made the scope return early survives the release.
struct ReleaseGuard {
    rtb200_scene_handle h;
    ~ReleaseGuard() { std::string keep = g_last_error; rtb200_scene_release(h); g_last_error = keep; }
};

// A call on host buffers: upload s, run `body(h, dev, &stats)` with the context's output buffers dev[k] for `frames` frames
// of the shard (rgb8, linear f32, u32 counts, f32 variance, each only when out[k] asks for it), copy them to out[k] and release
// the scene.
// The stats are body's with the upload's bytes, the copies' bytes plus `d2h` bytes the body read back, and the wall time.
template <typename Body>
static int one_shot(const rt_scene* s, const rt_options& opts, uint64_t frames, void* const out[4], uint64_t d2h, rt_stats* stats,
                    Body&& body) {
    const auto wall0 = std::chrono::steady_clock::now();
    rtb200_scene_handle h = nullptr;
    int rc = rtb200_scene_upload(s, &opts, &h);
    if (rc != RT_OK) return rc;
    ReleaseGuard rel{h};
    HANDLE_PROLOGUE(h);
    DeviceCtx* ctx = h->ctx;
    GrowBuf* buf[4] = {&ctx->out_rgb8, &ctx->out_lin, &ctx->out_cnt, &ctx->out_var};
    const size_t pixels = frames * h->tp.npix_local, elem[4] = {3, 12, 4, 12};
    void* dev[4] = {nullptr, nullptr, nullptr, nullptr};
    for (int k = 0; k < 4; ++k) if (out[k]) { CU(buf[k]->ensure(pixels * elem[k] + 16)); dev[k] = buf[k]->p; }
    rt_stats st{};
    if ((rc = body(h, dev, &st)) != RT_OK) return rc;
    for (int k = 0; k < 4; ++k) {
        if (out[k] && pixels) CU(cudaMemcpyAsync(out[k], dev[k], pixels * elem[k], cudaMemcpyDeviceToHost, ctx->stream));
        if (out[k]) d2h += pixels * elem[k];
    }
    if (pixels) CU(cudaStreamSynchronize(ctx->stream));
    st.h2d_bytes += h->h2d_bytes;
    st.d2h_bytes = d2h;
    st.wall_ms = ms_since(wall0);
    if (stats) *stats = st;
    return RT_OK;
}

// Host buffers: render `frames` of s. The single-frame calls pass the scene's own view as one frame.
static int render_host(const rt_scene* s, const rt_options* opts_in, const rt_frame* frames, uint32_t n_frames, uint8_t* out_rgb8,
                       float* out_lin, rt_stats* stats, const rt_lens* lenses = nullptr, float* out_var = nullptr) {
    rt_options opts;
    int rc = normalise_options(opts_in, &opts);
    if (rc != RT_OK) return rc;
    uint32_t n_lights = 0;
    if ((rc = validate_scene(s, &n_lights)) != RT_OK) return rc;
    if ((rc = check_frames(frames, n_frames, rtb200_shard_rows(s->height, opts.rank, opts.world, opts.band_rows), s->width, lenses)) != RT_OK) return rc;
    void* const out[4] = {out_rgb8, out_lin, nullptr, out_var};
    return one_shot(s, opts, n_frames, out, 128 + 16, stats, [&](rtb200_scene_handle h, void* const* dev, rt_stats* st) {
        return render_blocking(h, frames, n_frames, dev[0], dev[1], nullptr, st, lenses, (float*)dev[3]);
    });
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
    HANDLE_PROLOGUE(h);
    const rt_frame f = own_frame(h);
    return render_enqueue(h, &f, 1, dev_rgb8, dev_linear_f32, stream_in, (int)(h->frame_counter++ & 1u));
  });
}

int rtb200_render_device_wait(rtb200_scene_handle h, rt_stats* stats) {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    HANDLE_PROLOGUE(h);
    return render_collect(h, stats);
}

int rtb200_render_frames_lens_device(rtb200_scene_handle h, const rt_frame* frames, const rt_lens* lenses, uint32_t n_frames,
                                     void* dev_rgb8, void* dev_linear_f32, void* stream_in, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    int rc = check_frames(frames, n_frames, h->tp.rows_local, h->tp.width, lenses);
    if (rc != RT_OK) return rc;
    if (!dev_rgb8 && !dev_linear_f32) return fail(RT_ERR_INVALID, "dev_rgb8 and dev_linear_f32 are both null");
    return render_blocking(h, frames, n_frames, dev_rgb8, dev_linear_f32, stream_in, stats, lenses);
  });
}

int rtb200_render_frames_device(rtb200_scene_handle h, const rt_frame* frames, uint32_t n_frames, void* dev_rgb8, void* dev_linear_f32,
                                void* stream_in, rt_stats* stats) {
    return rtb200_render_frames_lens_device(h, frames, nullptr, n_frames, dev_rgb8, dev_linear_f32, stream_in, stats);
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

int rtb200_render_frames_lens(const rt_scene* s, const rt_options* opts_in, const rt_frame* frames, const rt_lens* lenses,
                              uint32_t n_frames, uint8_t* out_rgb8, float* out_lin, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!s) return fail(RT_ERR_INVALID, "null argument");
    if (!out_rgb8 && !out_lin) return fail(RT_ERR_INVALID, "out_rgb8 and out_linear_f32 are both null");
    return render_host(s, opts_in, frames, n_frames, out_rgb8, out_lin, stats, lenses);
  });
}

int rtb200_render_frames(const rt_scene* s, const rt_options* opts_in, const rt_frame* frames, uint32_t n_frames, uint8_t* out_rgb8,
                         float* out_lin, rt_stats* stats) {
    return rtb200_render_frames_lens(s, opts_in, frames, nullptr, n_frames, out_rgb8, out_lin, stats);
}

// ---- the variance of the pixel means (DESIGN.md §4.18) ----
int rtb200_render_frames_var_device(rtb200_scene_handle h, const rt_frame* frames, const rt_lens* lenses, uint32_t n_frames,
                                    void* dev_rgb8, void* dev_linear_f32, float* dev_variance_f32, void* stream_in, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    int rc = check_frames(frames, n_frames, h->tp.rows_local, h->tp.width, lenses);
    if (rc != RT_OK) return rc;
    if (!dev_variance_f32) return fail(RT_ERR_INVALID, "dev_variance_f32 is null");
    return render_blocking(h, frames, n_frames, dev_rgb8, dev_linear_f32, stream_in, stats, lenses, dev_variance_f32);
  });
}

int rtb200_render_frames_var(const rt_scene* s, const rt_options* opts_in, const rt_frame* frames, const rt_lens* lenses,
                             uint32_t n_frames, uint8_t* out_rgb8, float* out_lin, float* out_variance, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!s) return fail(RT_ERR_INVALID, "null argument");
    if (!out_variance) return fail(RT_ERR_INVALID, "out_variance is null");
    return render_host(s, opts_in, frames, n_frames, out_rgb8, out_lin, stats, lenses, out_variance);
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
    Submit s;
    int rc = submission_open(h, stream_in, 1, &s);
    if (rc != RT_OK) return rc;
    TraceParams tp = h->tp;
    tp.npix_local = n;   // Q_RAYS: the rays, which are also the resolve's pixels
    tp.max_depth = tr.max_depth;
    tp.key0 = (uint32_t)tr.seed; tp.key1 = (uint32_t)(tr.seed >> 32);
    tp.stream0 = tr.stream0;
    tp.ray_o = rays.origin; tp.ray_d = rays.direction;
    const uint32_t m = tr.samples;
    const uint32_t spb = samples_per_batch(sample_buffer_cap(h->opts), n, m);
    const uint32_t n_batches = (uint32_t)(((uint64_t)m + spb - 1) / spb);
    LaunchGeom g;
    if ((rc = launch_geometry(h, Q_RAYS, tp.n_lights > 0, &g)) != RT_OK) return rc;
    if ((rc = submission_begin(h, 0, n_batches, g.grid, tp, tp.max_depth, (size_t)spb * n * 16, nullptr, 0, &s)) != RT_OK) return rc;
    *st_out = s.st;
    for (uint32_t b = 0; b < n_batches; ++b) {
        TraceParams q = tp;
        const uint32_t first = b * spb;
        q.s0 = tr.sample0 + first;
        q.s_count = std::min(spb, m - first);
        q.total_work = q.s_count * n;
        if ((rc = trace_step(h, s, b, q, Q_RAYS, g, (size_t)q.total_work * 16)) != RT_OK) return rc;
        ResolveParams r{};
        r.samplebuf = q.samplebuf; r.accum = (float*)s.W->accum.p; r.npix_local = n;
        r.s_count = q.s_count; r.first = b == 0; r.last = b + 1 == n_batches; r.spp = m;
        r.out_linear = lin; r.out_rgb8 = rgb;
        CU(launch_resolve(r, s.st));
    }
    s.sub.launches = 2 * n_batches;
    if (tp.max_depth == 0) s.sub.black_samples = (uint64_t)n * m;
    return submission_close(h, s);
}

// Both forms: the device form checks the memory kind of the caller's buffers and traces them on `stream_in`; the host form
// copies the rays into the context's query block, traces on the library's stream and copies the outputs back.
static int trace_rays_blocking(rtb200_scene_handle h, const rt_rays* rays, uint32_t n, const rt_trace_params* p, float* lin,
                               uint8_t* rgb, void* stream_in, bool host, rt_stats* stats) {
    if (stats) memset(stats, 0, sizeof *stats);
    int rc = check_trace_rays(h, rays, n, p, lin, rgb);
    if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    HANDLE_PROLOGUE(h);
    if (!host && (rc = check_device_ptrs(h, {{rays->origin, "rays->origin"}, {rays->direction, "rays->direction"},
                                             {lin, "dev_linear_f32"}, {rgb, "dev_rgb8"}})) != RT_OK)
        return rc;
    HostStage io;
    rc = blocking(h, stats, [&]() -> int {
        rt_rays drays = *rays;
        float* dlin = lin;
        uint8_t* drgb = rgb;
        int rcq = RT_OK;
        if (host) {   // device image: origins, directions, linear, rgb8
            const uint64_t N = n;
            io.add_in(rays->origin, N * 24); io.add_in(rays->direction, N * 24);
            io.add_out(lin, lin ? N * 12 : 0); io.add_out(rgb, rgb ? N * 3 : 0);
            if ((rcq = io.place(h->ctx, 0)) != RT_OK) return rcq;
            drays = rt_rays{(const double*)io.a[0].dev, (const double*)io.a[1].dev, nullptr};
            dlin = (float*)io.a[2].dev;
            drgb = (uint8_t*)io.a[3].dev;
            cudaStream_t st;
            CU(scene_stream(h, nullptr, &st));   // the stream the submission takes
            if ((rcq = io.copy(st, false)) != RT_OK) return rcq;
        }
        cudaStream_t st = nullptr;
        if ((rcq = trace_rays_enqueue(h, drays, n, *p, dlin, drgb, host ? nullptr : stream_in, &st)) != RT_OK) return rcq;
        return host ? io.copy(st, true) : RT_OK;
    });
    if (rc == RT_OK && stats) { stats->h2d_bytes += io.h2d; stats->d2h_bytes += io.d2h; }
    return rc;
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

// The adaptive block of a shard of npl pixels carved out of `base` (null: only the size); returns the bytes.
static size_t adaptive_carve(void* base, uint32_t npl, rtb200_scene_t::Adaptive* A) {
    Carver c(base);
    A->sum = (float*)c.take((size_t)npl * 12);
    A->sq = (float*)c.take((size_t)npl * 12);
    A->count = (uint32_t*)c.take((size_t)npl * 4);   // sum, sq and count are contiguous: one memset clears them
    A->keep = (uint32_t*)c.take((size_t)npl * 4);
    A->list[0] = (uint32_t*)c.take((size_t)npl * 4);
    A->list[1] = (uint32_t*)c.take((size_t)npl * 4);
    A->list_n = (uint32_t*)c.take(2 * 4);
    A->temp_bytes = adaptive_compact_bytes(npl);
    A->temp = c.take(A->temp_bytes);
    return c.off;
}

int rtb200_adaptive_begin(rtb200_scene_handle h, const rt_adaptive_params* p, void* stream_in) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    const uint32_t npl = h->tp.npix_local;
    int rc = check_adaptive(p, npl, sample_buffer_cap(h->opts));
    if (rc != RT_OK) return rc;
    HANDLE_PROLOGUE(h);
    auto& A = h->ad;
    A.begun = false;
    if (!A.mem && npl) {
        const size_t bytes = adaptive_carve(nullptr, npl, &A);
        void* m = nullptr;
        cudaError_t e = cudaMalloc(&m, bytes);
        if (e != cudaSuccess) { cudaGetLastError(); return fail(RT_ERR_OOM, "adaptive: cannot allocate " + std::to_string(bytes) + " bytes of device memory"); }
        e = cudaHostAlloc((void**)&A.active_host, 4, cudaHostAllocDefault);
        if (e != cudaSuccess) { cudaFree(m); A.active_host = nullptr; return fail_cuda(e, "cudaHostAlloc"); }
        A.mem = m;
        adaptive_carve(m, npl, &A);
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
    const uint32_t m = A.p.samples_per_round;
    const uint64_t left = A.active && A.n < A.N ? ((uint64_t)A.N - A.n + m - 1) / m : 0;   // rounds until every pixel has N
    rounds = (uint32_t)std::min<uint64_t>(rounds, left);
    if (active_out) *active_out = A.active;
    if (rounds == 0) return RT_OK;   // finished: nothing to do
    HANDLE_PROLOGUE(h);
    int rc = blocking(h, stats, [&]() -> int {
        Submit s;
        int rcs = submission_open(h, stream_in, 1, &s);
        if (rcs != RT_OK) return rcs;
        TraceParams tp = h->tp;
        const uint32_t npl = tp.npix_local;
        LaunchGeom g;
        const uint32_t queue = tp.lens.radius != 0.0 ? Q_LIST_LENS : Q_LIST;   // the handle's lens (rtb200_scene_set_lens)
        if ((rcs = launch_geometry(h, queue, tp.n_lights > 0, &g)) != RT_OK) return rcs;
        if ((rcs = submission_begin(h, 0, rounds, g.grid, tp, tp.max_depth, (size_t)m * npl * 16, nullptr, 0, &s)) != RT_OK) return rcs;
        const bool black = tp.max_depth == 0;
        A.begun = false;   // until the rounds are enqueued: a step that fails part-way leaves the state unusable
        for (uint32_t r = 0; r < rounds; ++r) {
            TraceParams q = tp;
            q.s0 = A.n;
            q.s_count = std::min(m, A.N - A.n);
            q.total_work = 0;   // Q_LIST: n_list * s_count, n_list read on the device
            q.list = A.list[A.cur]; q.list_n = A.list_n + A.cur;
            if ((rcs = trace_step(h, s, r, q, queue, g, (size_t)q.s_count * npl * 16)) != RT_OK) return rcs;
            AdaptiveParams a{};
            a.samplebuf = q.samplebuf; a.list = q.list; a.list_n = q.list_n;
            a.sum = A.sum; a.sq = A.sq; a.count = A.count; a.keep = A.keep;
            a.black_samples = black ? tp.stat + 3 : nullptr;
            a.npix_local = npl; a.s_count = q.s_count; a.n_after = A.n + q.s_count;
            a.max_samples = A.N; a.min_samples = A.p.min_samples; a.abs_tol = A.p.abs_tol; a.rel_tol = A.p.rel_tol;
            CU(launch_adaptive_accumulate(a, s.st));
            CU(launch_adaptive_compact(A.temp, A.temp_bytes, A.list[A.cur], A.keep, A.list[A.cur ^ 1u], A.list_n + (A.cur ^ 1u), npl, s.st));
            A.cur ^= 1u;
            A.n += q.s_count;
            s.sub.launches += 3;   // trace (or black memset), accumulate, compaction
        }
        CU(cudaMemcpyAsync(A.active_host, A.list_n + A.cur, 4, cudaMemcpyDeviceToHost, s.st));
        return submission_close(h, s);
    });
    if (rc != RT_OK) return rc;
    A.active = *A.active_host;
    A.begun = true;
    if (active_out) *active_out = A.active;
    return RT_OK;
  });
}

int rtb200_adaptive_resolve_var(rtb200_scene_handle h, void* dev_rgb8, void* dev_linear_f32, void* dev_counts_u32,
                                float* dev_variance_f32, void* stream_in) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (!h->ad.begun) return fail(RT_ERR_INVALID, "no adaptive render on this handle: call rtb200_adaptive_begin");
    if (!dev_variance_f32) return fail(RT_ERR_INVALID, "dev_variance_f32 is null");
    if (h->tp.npix_local == 0) return RT_OK;
    HANDLE_PROLOGUE(h);
    cudaStream_t st;
    CU(scene_stream(h, stream_in, &st));
    AdaptiveResolveVarParams v{};
    v.r.sum = h->ad.sum; v.r.count = h->ad.count; v.r.npix_local = h->tp.npix_local;
    v.r.out_linear = (float*)dev_linear_f32; v.r.out_rgb8 = (uint8_t*)dev_rgb8; v.r.out_count = (uint32_t*)dev_counts_u32;
    v.sq = h->ad.sq; v.out_variance = dev_variance_f32;
    CU(launch_adaptive_resolve_var(v, st));
    CU(cudaStreamSynchronize(st));
    return RT_OK;
  });
}

int rtb200_adaptive_resolve(rtb200_scene_handle h, void* dev_rgb8, void* dev_linear_f32, void* dev_counts_u32, void* stream_in) {
  return guarded([&]() -> int {
    if (!h) return fail(RT_ERR_INVALID, "null scene handle");
    if (!h->ad.begun) return fail(RT_ERR_INVALID, "no adaptive render on this handle: call rtb200_adaptive_begin");
    if (h->tp.npix_local == 0 || (!dev_rgb8 && !dev_linear_f32 && !dev_counts_u32)) return RT_OK;
    HANDLE_PROLOGUE(h);
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

// The host form of an adaptive render, with the variance of the pixel means when out_var is not null.
static int render_adaptive_host(const rt_scene* s, const rt_options* opts_in, const rt_adaptive_params* p, uint8_t* out_rgb8,
                                float* out_lin, uint32_t* out_counts, float* out_var, rt_stats* stats) {
    if (!s) return fail(RT_ERR_INVALID, "null argument");
    rt_options opts;
    int rc = normalise_options(opts_in, &opts);
    if (rc != RT_OK) return rc;
    uint32_t n_lights = 0;
    if ((rc = validate_scene(s, &n_lights)) != RT_OK) return rc;
    const uint64_t npl = (uint64_t)rtb200_shard_rows(s->height, opts.rank, opts.world, opts.band_rows) * s->width;
    if ((rc = check_adaptive(p, npl, sample_buffer_cap(opts))) != RT_OK) return rc;
    void* const out[4] = {out_rgb8, out_lin, out_counts, out_var};
    return one_shot(s, opts, 1, out, 128 + 16 + 4, stats, [&](rtb200_scene_handle h, void* const* dev, rt_stats* st) {
        uint32_t active = 0;
        int rcb = rtb200_adaptive_begin(h, p, nullptr);
        if (rcb == RT_OK) rcb = rtb200_adaptive_step(h, 0xffffffffu, nullptr, &active, st);
        if (rcb == RT_OK) rcb = out_var ? rtb200_adaptive_resolve_var(h, dev[0], dev[1], dev[2], (float*)dev[3], nullptr)
                                        : rtb200_adaptive_resolve(h, dev[0], dev[1], dev[2], nullptr);
        st->frames = 1;
        return rcb;
    });
}

int rtb200_render_adaptive(const rt_scene* s, const rt_options* opts_in, const rt_adaptive_params* p, uint8_t* out_rgb8,
                           float* out_lin, uint32_t* out_counts, rt_stats* stats) {
    return guarded([&]() -> int { return render_adaptive_host(s, opts_in, p, out_rgb8, out_lin, out_counts, nullptr, stats); });
}

int rtb200_render_adaptive_var(const rt_scene* s, const rt_options* opts_in, const rt_adaptive_params* p, uint8_t* out_rgb8,
                               float* out_lin, uint32_t* out_counts, float* out_variance, rt_stats* stats) {
  return guarded([&]() -> int {
    if (!out_variance) return fail(RT_ERR_INVALID, "out_variance is null");
    return render_adaptive_host(s, opts_in, p, out_rgb8, out_lin, out_counts, out_variance, stats);
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
    scene_records(s, base, R);
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
            HANDLE_PROLOGUE(h);
            DeviceCtx* c = h->ctx;
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
    total.wall_ms = ms_since(wall0);
    if (stats) *stats = total;
    return RT_OK;
  });
}
