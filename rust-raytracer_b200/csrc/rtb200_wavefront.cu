// rtb200_wavefront.cu — the barrier-synchronised wavefront trace kernel (round 1's structure with round 2's stages).
//
// One persistent CTA (256 threads) per resident slot of every SM owns a pool of 256 ray slots in shared memory. Until the
// global (pixel,sample) queue is drained and the pool is empty, the CTA repeats three stages (two barriers per iteration)
// (rtb200_trace.cuh): closest-hit (thread t <-> slot t; warp-cooperative BVH traversal, or the linear scans of the
// validation modes), a sort that compacts the live slots class by class with warp ballots (perm[]), and shade + ray-gen
// (thread i <-> slot perm[i], so a warp shades one material).
//
// The three template modes share everything but the closest-hit stage: MODE_TREE (production: BVH traversal), MODE_BRUTE
// (RT_VARIANT_BRUTE_FORCE: linear scan with the conservative sphere test) and MODE_EXACT (RT_VARIANT_EXACT_F64: every
// sphere in f64) - the last two validate the first. Each mode has a single-frame kernel, a multi-frame one (Q_FRAMES: the
// queue spans several frames of the scene, each with its own camera and key; rtb200_render_frames, DESIGN.md §4.6), a list
// one (Q_LIST: the queue spans the pixels still on an adaptive render's list; rtb200_adaptive_step, DESIGN.md §4.9) and a rays
// one (Q_RAYS: the queue spans samples of caller-supplied primary rays; rtb200_scene_trace_rays, DESIGN.md §4.12).
#include <cstdio>
#include <cstdlib>

#include "rtb200_trace.cuh"

namespace rtk {

namespace {

struct WfSmem {
    uint32_t nodes_off, leafrec_off, leafid_off, filt_off, geo_off, mat_off;
    uint32_t warpctx;   // kWarpCtxBytes per warp (MODE_TREE)
    uint32_t pool;      // kSlotBytes * kBlock
    uint32_t perm;      // uint16[5 classes][kBlock]: every class has its own segment, so a slot's position needs no other class's count
    uint32_t cnt;       // uint32[2][8]
    uint32_t phase;     // RT_PHASE_CLOCKS: u64[8 warps][kPhaseN]
    uint32_t total;
};

// A staged segment is copied with one cp.async.bulk, whose shared and global addresses must be 16-byte aligned and whose
// size must be a multiple of 16. Every segment therefore starts at a multiple of 16 and is copied (and counted by the
// mbarrier) at its size rounded up to 16: stage_bytes of `count` elements of UNIT bytes. The nodes (224 B), leaf records
// (kLeafK * 16 B), flat record pairs, geometry and materials (32 B) are whole 16 B blocks already. Only the leaf-id block can
// be short (UNIT = kLeafK * 4 with kLeafK / 2 odd, and an odd leaf count: 8 B short); its copy then reads 8 B past the
// array, inside the array's 256 B upload block (commit_uploads). A UNIT that is a multiple of 16 compiles to no rounding:
// the default build's leaves of 8 keep their code.
template <uint32_t UNIT>
__host__ __device__ constexpr uint32_t stage_bytes(uint32_t count) { return UNIT % 16u == 0u ? count * UNIT : (count * UNIT + 15u) & ~15u; }

// mask: bit0 hierarchy (MODE_TREE) / flat records (MODE_BRUTE), bit1 exact geometry, bit2 materials in shared memory
// frames: the multi-frame kernel's pool also holds Pool.frm
__host__ __device__ constexpr WfSmem wf_layout(uint32_t n, uint32_t n_pairs, uint32_t n_nodes, uint32_t n_leaves, uint32_t mode, uint32_t mask, bool frames) {
    WfSmem L{};
    uint32_t off = 16;   // mbarrier
    L.nodes_off = off;   if (mode == MODE_TREE && (mask & 1u)) off += n_nodes * (uint32_t)(kNodeVec * 16);
    L.leafrec_off = off; if (mode == MODE_TREE && (mask & 1u)) off += n_leaves * (uint32_t)(kLeafK * 16);
    L.leafid_off = off;  if (mode == MODE_TREE && (mask & 1u)) off += stage_bytes<kLeafK * 4>(n_leaves);
    L.filt_off = off;    if (mode == MODE_BRUTE && (mask & 1u)) off += n_pairs * 32u;
    L.geo_off = off; if (mask & 2u) off += n * 32u;
    L.mat_off = off; if (mask & 4u) off += n * 32u;
    off = (off + 15u) & ~15u;
    L.warpctx = off; if (mode == MODE_TREE) off += (uint32_t)(kBlock / 32) * kWarpCtxBytes;
    L.pool = off; off += (kSlotBytes + (frames ? kFrameSlotBytes : 0u)) * (uint32_t)kBlock;
    L.perm = off; off += 5u * kBlock * 2u;
    L.cnt = off; off += 2u * 8u * 4u;
    L.phase = off; if (RT_PHASE_CLOCKS) off += (uint32_t)(kBlock / 32) * kPhaseN * 8u;
    L.total = off;
    return L;
}

}  // namespace

size_t wavefront_smem_bytes(const TraceParams& p, uint32_t mode, uint32_t smem_mask, uint32_t queue) {
    return wf_layout(p.n, p.n_pairs, p.n_nodes, p.n_leaves, mode, smem_mask, base_queue(queue) == Q_FRAMES).total;
}

// CTAs per SM each kernel's register budget is built for: 3 of 256 threads for the BVH path (80 registers), 2 for the
// validation modes
constexpr int wf_min_blocks(uint32_t mode) {
    const int n = (mode == MODE_TREE ? 3 : 2) * 256 / kBlock;
    return n > 0 ? n : 1;
}

// Shared memory and L1 share the SM's 256 KiB, and every scene load and local-memory spill of the trace kernel goes through
// L1. The H100 sets the shared-memory side in steps (..., 164, 196, 228 KiB), allocates a CTA's shared memory in 128 B units
// and reserves 1 KiB per CTA. Three tree CTAs therefore leave 60 KiB of L1 when each takes at most 65,792 B of dynamic shared
// memory, and 28 KiB when it takes more; on C2 the same kernel ran 3.3 % faster with 60 KiB (DESIGN.md §4.5). (The
// stage-clock build's per-warp table does not fit.)
constexpr uint32_t smem_alloc(uint32_t bytes) { return (bytes + 127u) / 128u * 128u + 1024u; }
static_assert(RT_PHASE_CLOCKS || 3u * smem_alloc(wf_layout(0, 0, 0, 0, MODE_TREE, 0u, false).total) <= 196u * 1024u,
              "three single-frame tree CTAs per SM must fit the 196 KiB carveout");

// Give the kernel the smallest carveout that holds the CTAs per SM its register budget is built for (wf_min_blocks), so that
// L1 keeps the rest whatever the driver would pick. A percentage is rounded up to the next carveout step, so the rounded-down
// percentage of what the CTAs need is tried first, and one percent more only when the occupancy says that step is too small.
// RTB200_WF_CARVEOUT=<percent> sets the preference instead (experiments: tools/l1_probe.py). Needs the kernel's
// cudaFuncAttributeMaxDynamicSharedMemorySize set to `smem`.
template <typename K>
static cudaError_t set_carveout(K kern, uint32_t mode, size_t smem) {
    static const char* forced = getenv("RTB200_WF_CARVEOUT");
    if (forced) return cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(forced));
    int dev = 0, max_sm = 0, reserved = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&max_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev);
    if (e != cudaSuccess) return e;
    const size_t need = (size_t)wf_min_blocks(mode) * ((smem + 127u) / 128u * 128u + (size_t)reserved);
    const int pct = need >= (size_t)max_sm ? 100 : (int)(need * 100u / (size_t)max_sm);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
    if (e != cudaSuccess || pct == 100) return e;
    int nb = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kBlock, smem);
    if (e != cudaSuccess || nb >= wf_min_blocks(mode)) return e;
    return cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, pct + 1);
}

// Q_FRAMES: one launch renders several frames of the scene (TraceParams::ftab / frame_work, rtb200_render_frames)
// Q_LIST: one launch traces a round of an adaptive render (TraceParams::list / list_n, rtb200_adaptive_step)
// Q_RAYS: one launch traces a batch of samples of caller-supplied rays (TraceParams::ray_o / ray_d, rtb200_scene_trace_rays)
// Q_FRAMES_LENS / Q_LIST_LENS: Q_FRAMES / Q_LIST whose camera rays go through a thin lens (TraceParams::ltab / lens, DESIGN.md §4.17)
template <uint32_t MODE, bool LIGHTS, uint32_t QUEUE_>
__global__ void __launch_bounds__(kBlock, wf_min_blocks(MODE)) rt_wavefront_kernel(const __grid_constant__ TraceParams p) {
    constexpr uint32_t QUEUE = base_queue(QUEUE_);
    constexpr bool LENS = QUEUE != QUEUE_;
    constexpr bool FRAMES = QUEUE == Q_FRAMES;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const WfSmem L = wf_layout(p.n, p.n_pairs, p.n_nodes, p.n_leaves, MODE, p.scene_in_smem, FRAMES);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
    const bool tree_smem = (p.scene_in_smem & 1u) != 0u;
    SceneRefs sc;
    sc.nodes = (MODE == MODE_TREE && tree_smem) ? reinterpret_cast<const float4*>(smem_raw + L.nodes_off) : p.nodes;
    sc.leaf_rec = (MODE == MODE_TREE && tree_smem) ? reinterpret_cast<const float4*>(smem_raw + L.leafrec_off) : p.leaf_rec;
    sc.leaf_id = (MODE == MODE_TREE && tree_smem) ? reinterpret_cast<const uint32_t*>(smem_raw + L.leafid_off) : p.leaf_id;
    sc.filt = (MODE == MODE_BRUTE && tree_smem) ? reinterpret_cast<const float4*>(smem_raw + L.filt_off) : p.filt;
    sc.geo = (p.scene_in_smem & 2u) ? reinterpret_cast<const double4*>(smem_raw + L.geo_off) : p.geo;
    sc.mat = (p.scene_in_smem & 4u) ? reinterpret_cast<const DevMat*>(smem_raw + L.mat_off) : p.mat;
    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const unsigned FULL = 0xffffffffu;
    const Pool P = pool_at(smem_raw + L.pool, (uint32_t)kBlock, blockIdx.x * (uint32_t)kBlock);
    const WarpCtx W = warpctx_at(smem_raw + L.warpctx + (uint32_t)(tid >> 5) * kWarpCtxBytes);
    uint16_t* s_perm = reinterpret_cast<uint16_t*>(smem_raw + L.perm);
    uint32_t* s_cnt = reinterpret_cast<uint32_t*>(smem_raw + L.cnt);

    // ---- stage the scene into shared memory (TMA bulk copies, one mbarrier) ----
    if (tid == 0) mbar_init(bar, 1);
    if (tid < 16) s_cnt[tid] = 0;
    P.lvl[tid] = kDeadLevel;
    __syncthreads();
    if (tid == 0) {   // the segment sizes of wf_layout, which the mbarrier counts
        const uint32_t b_nodes = (MODE == MODE_TREE && tree_smem) ? p.n_nodes * (uint32_t)(kNodeVec * 16) : 0u;
        const uint32_t b_lrec = (MODE == MODE_TREE && tree_smem) ? p.n_leaves * (uint32_t)(kLeafK * 16) : 0u;
        const uint32_t b_lid = (MODE == MODE_TREE && tree_smem) ? stage_bytes<kLeafK * 4>(p.n_leaves) : 0u;
        const uint32_t b_filt = (MODE == MODE_BRUTE && tree_smem) ? p.n_pairs * 32u : 0u;
        const uint32_t b_geo = (p.scene_in_smem & 2u) ? p.n * 32u : 0u, b_mat = (p.scene_in_smem & 4u) ? p.n * 32u : 0u;
        mbar_arrive_expect_tx(bar, b_nodes + b_lrec + b_lid + b_filt + b_geo + b_mat);
        if (b_nodes) bulk_stage(smem_raw + L.nodes_off, p.nodes, b_nodes, bar);
        if (b_lrec) bulk_stage(smem_raw + L.leafrec_off, p.leaf_rec, b_lrec, bar);
        if (b_lid) bulk_stage(smem_raw + L.leafid_off, p.leaf_id, b_lid, bar);
        if (b_filt) bulk_stage(smem_raw + L.filt_off, p.filt, b_filt, bar);
        if (b_geo) bulk_stage(smem_raw + L.geo_off, p.geo, b_geo, bar);
        if (b_mat) bulk_stage(smem_raw + L.mat_off, p.mat, b_mat, bar);
    }
    mbar_wait(bar, 0);

    // frame-tail diagnostics (stat[8..10]): first CTA start, first moment a warp found the global queue dry, last CTA exit (ns)
    auto now_ns = []() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; };
    if (tid == 0) atomicMin(&p.stat[8], now_ns());
    Stats st;
    bool exhausted = false;   // warp-uniform: this warp has seen the end of the queue
    bool stamped = false;
    uint32_t dry_iters = 0;   // iterations of this CTA after it first found the global queue dry
    uint32_t n_list = 0u;   // Q_LIST: the pixels on the list, fixed for the launch
    if constexpr (QUEUE == Q_LIST) n_list = *p.list_n;
    regenerate_slot<LIGHTS, QUEUE, LENS>(p, P, true, (uint32_t)tid, lane, exhausted, st, n_list);   // initial fill of the pool
    __syncthreads();

#if RT_PHASE_CLOCKS
    // lane 0 of each warp adds the warp's clock64() time of each stage to the warp's own row of ph[]
    static_assert(kPhaseStat + kPhaseN <= 32, "the per-launch stat block holds 32 counters");
    unsigned long long* ph = reinterpret_cast<unsigned long long*>(smem_raw + L.phase) + (uint32_t)(tid >> 5) * kPhaseN;
    if (lane < (int)kPhaseN) ph[lane] = 0ull;
    unsigned long long t_mark = clock64();
    auto tick = [&](uint32_t k) { __syncwarp(); const unsigned long long t = clock64(); if (lane == 0) ph[k] += t - t_mark; t_mark = t; };
#endif
    const uint32_t lt_mask = (1u << lane) - 1u;
    uint32_t it = 0;
    for (;; ++it) {
        uint32_t* cnt = s_cnt + (it & 1u) * 8u;
        // =========================== closest-hit: thread t <-> slot t ===========================
        // A slot whose scatter sample is pending is not traced: it keeps its hit (and its ray count) and takes the class of
        // the sphere it hit, so the sort puts it back among the fresh hits of its material.
        const bool alive = P.lvl[tid] != kDeadLevel;
        const bool pending = alive && (P.shd[tid] & kScatterPending) != 0u;
        uint32_t cls = closest_hit<MODE>(p, sc, P, W, alive && !pending, (uint32_t)tid, lane, st);
        if (pending) cls = class_of(sc.mat[P.bi[tid]].kind);
#if RT_PHASE_CLOCKS
        tick(PH_HIT);
#endif

        // =========================== sort: compact the live slots class by class ===========================
        // warp ballot + one shared-memory atomic per (warp, class) reserve positions in the class's own segment of perm[]
#pragma unroll
        for (uint32_t c = 0; c < CLS_DEAD; ++c) {
            unsigned b = __ballot_sync(FULL, cls == c);
            if (b) {
                uint32_t base = 0;
                if (lane == 0) base = atomicAdd(&cnt[c], (uint32_t)__popc(b));
                base = __shfl_sync(FULL, base, 0);
                if (cls == c) s_perm[c * (uint32_t)kBlock + base + (uint32_t)__popc(b & lt_mask)] = (uint16_t)tid;
            }
        }
        __syncthreads();   // A: class counts and perm complete (and every warp's closest-hit results are in the pool)
#if RT_PHASE_CLOCKS
        tick(PH_SORT_WAIT_A);
#endif
        uint32_t c0 = cnt[0], c1 = cnt[1], c2 = cnt[2], c3 = cnt[3], c4 = cnt[4];
        const uint32_t e0 = c0, e1 = e0 + c1, e2 = e1 + c2, e3 = e2 + c3, n_live = e3 + c4;   // class end offsets
        if (tid < 8) s_cnt[((it + 1u) & 1u) * 8u + tid] = 0u;   // reset the other counter set for the next iteration

        // =========================== shade + regenerate: thread i <-> slot perm[i] ===========================
        const bool active = (uint32_t)tid < n_live;
        const uint32_t c = !active ? CLS_DEAD : ((uint32_t)tid < e0 ? CLS_MISS : (uint32_t)tid < e1 ? CLS_DIFFUSE : (uint32_t)tid < e2 ? CLS_METAL : (uint32_t)tid < e3 ? CLS_GLASS : CLS_LIGHT);
        const uint32_t cstart = c == CLS_MISS ? 0u : c == CLS_DIFFUSE ? e0 : c == CLS_METAL ? e1 : c == CLS_GLASS ? e2 : e3;
        const uint32_t s = active ? (uint32_t)s_perm[c * (uint32_t)kBlock + ((uint32_t)tid - cstart)] : 0u;
        bool done = false;
        if (active) done = shade_slot<LIGHTS, FRAMES>(p, sc, P, s, c);
#if RT_PHASE_CLOCKS
        tick(PH_SHADE);
        {
            const bool scatter = active && (c == CLS_DIFFUSE || c == CLS_METAL);
            const unsigned sm = __ballot_sync(FULL, scatter), dm = __ballot_sync(FULL, scatter && !done && (P.shd[s] & kScatterPending) != 0u);
            if (lane == 0) { ph[PH_ITERS] += 1ull; ph[PH_SCATTERS] += (unsigned)__popc(sm); ph[PH_DEFERRED] += (unsigned)__popc(dm); }
        }
#endif
        regenerate_slot<LIGHTS, QUEUE, LENS>(p, P, active && done, s, lane, exhausted, st, n_list);
        if (exhausted && !stamped) { stamped = true; if (lane == 0) atomicMin(&p.stat[9], now_ns()); }
        if (stamped) ++dry_iters;
        const bool still_alive = active && (P.lvl[s] != kDeadLevel);
#if RT_PHASE_CLOCKS
        tick(PH_REGEN);
#endif
        const int more = __syncthreads_or(still_alive ? 1 : 0);   // C: pool written back; exit when the CTA has no ray left
#if RT_PHASE_CLOCKS
        tick(PH_WAIT_C);
#endif
        if (!more) break;
    }
    flush_stats(p, st, lane);
#if RT_PHASE_CLOCKS
    __syncwarp();
    if (lane < (int)kPhaseN) atomicAdd(&p.stat[kPhaseStat + lane], ph[lane]);
#endif
    if (tid == 0) { atomicMax(&p.stat[10], now_ns()); atomicMax(&p.stat[11], (unsigned long long)dry_iters); atomicAdd(&p.stat[12], (unsigned long long)dry_iters); }
}

template <uint32_t QUEUE, typename F>
static auto dispatch_mode(uint32_t mode, bool lights, F&& f) {
    if (mode == MODE_EXACT) return lights ? f(rt_wavefront_kernel<MODE_EXACT, true, QUEUE>) : f(rt_wavefront_kernel<MODE_EXACT, false, QUEUE>);
    if (mode == MODE_BRUTE) return lights ? f(rt_wavefront_kernel<MODE_BRUTE, true, QUEUE>) : f(rt_wavefront_kernel<MODE_BRUTE, false, QUEUE>);
    return lights ? f(rt_wavefront_kernel<MODE_TREE, true, QUEUE>) : f(rt_wavefront_kernel<MODE_TREE, false, QUEUE>);
}
template <typename F>
static auto dispatch(uint32_t mode, bool lights, uint32_t queue, F&& f) {
    if (queue == Q_RAYS) return dispatch_mode<Q_RAYS>(mode, lights, f);
    if (queue == Q_LIST) return dispatch_mode<Q_LIST>(mode, lights, f);
    if (queue == Q_FRAMES_LENS) return dispatch_mode<Q_FRAMES_LENS>(mode, lights, f);
    if (queue == Q_LIST_LENS) return dispatch_mode<Q_LIST_LENS>(mode, lights, f);
    return queue == Q_FRAMES ? dispatch_mode<Q_FRAMES>(mode, lights, f) : dispatch_mode<Q_SINGLE>(mode, lights, f);
}

cudaError_t launch_wavefront(const TraceParams& p, uint32_t mode, uint32_t queue, int grid, size_t smem, cudaStream_t st) {
    return dispatch(mode, p.n_lights > 0, queue, [&](auto kern) -> cudaError_t {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) e = set_carveout(kern, mode, smem);
        if (e != cudaSuccess) return e;
        kern<<<grid, kBlock, smem, st>>>(p);
        return cudaGetLastError();
    });
}

int wavefront_max_ctas_per_sm(uint32_t mode, bool lights, uint32_t queue, size_t smem) {
    return dispatch(mode, lights, queue, [&](auto kern) -> int {
        int nb = 0;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { cudaGetLastError(); return 0; }
        if (set_carveout(kern, mode, smem) != cudaSuccess) { cudaGetLastError(); return 0; }
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kBlock, smem) != cudaSuccess) { cudaGetLastError(); return 0; }
        return nb;
    });
}

cudaError_t wavefront_info(uint32_t mode, bool lights, uint32_t queue, KernelInfo* out) {
    return dispatch(mode, lights, queue, [&](auto kern) -> cudaError_t {
        cudaFuncAttributes a;
        cudaError_t e = cudaFuncGetAttributes(&a, kern);
        if (e != cudaSuccess) return e;
        out->registers = a.numRegs; out->max_threads = a.maxThreadsPerBlock; out->const_bytes = (int)a.constSizeBytes; out->local_bytes = (int)a.localSizeBytes;
        const uint32_t bq = base_queue(queue);
        snprintf(out->name, sizeof out->name, "rt_wavefront_kernel<%s,%s%s%s>",
                 mode == MODE_TREE ? "MODE_TREE" : mode == MODE_BRUTE ? "MODE_BRUTE" : "MODE_EXACT", lights ? "LIGHTS" : "NO_LIGHTS",
                 bq == Q_FRAMES ? ",FRAMES" : bq == Q_LIST ? ",LIST" : bq == Q_RAYS ? ",RAYS" : "", bq != queue ? ",LENS" : "");
        return cudaSuccess;
    });
}

}  // namespace rtk
