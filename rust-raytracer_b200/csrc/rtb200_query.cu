// rtb200_query.cu — closest-hit queries on caller-supplied rays (rtb200_scene_intersect[_device], DESIGN.md §4.10).
//
// The trace kernel's closest-hit stage, closest_hit<MODE> (rtb200_trace.cuh), is hit_world (raytracer.rs:44-59) bit for bit
// for the 32 rays a warp holds in its pool slots. This kernel feeds it the caller's rays instead of camera and scattered
// ones: each warp owns 32 slots and, for MODE_TREE, its own traversal context in shared memory, loads 32 consecutive rays
// (a query ray starts on no known sphere), calls closest_hit unchanged, and writes what the caller asked for. The warps of a
// CTA share nothing, so there is no CTA barrier; the warps take chunks of 32 rays in grid-stride order.
//
// t_max costs nothing in the traversal: closest_hit finds the unbounded closest hit (r*, j*) under f64::MAX and the kernel
// reports it only when r* < t_max (Sphere::hit's strict bound). That equals hit_world under t_max (DESIGN.md §4.10).
//
// rt_occluded_kernel<MODE> answers occlusion queries (rtb200_scene_occluded[_device], DESIGN.md §4.11) with the same CTA, chunks
// and slots: it calls the any-hit kind of the same stage, closest_hit<MODE, true>, under each ray's own bound
// T = min(t_max, f64::MAX), which prunes boxes beyond T and stops at the first sphere that accepts a root below T. A ray with
// !(T > 0.001) cannot be occluded (an accepted root is > 0.001 and < T) and does not enter the stage.
#include "rtb200_query.cuh"

namespace rtk {

namespace {

// occlusion queries: the traversal context is followed by the 32 rays' f32 bounds T~ (MODE_TREE), then the slots
constexpr uint32_t kTcapBytes = 32u * 4u;
__host__ __device__ constexpr uint32_t occluded_warp_bytes(uint32_t mode) {
    return query_warp_bytes(mode) + (mode == MODE_TREE ? kTcapBytes : 0u);
}
constexpr size_t occluded_smem_bytes(uint32_t mode) { return (size_t)kQueryWarps * occluded_warp_bytes(mode); }

template <uint32_t MODE>
__global__ void __launch_bounds__(kQueryBlock) rt_query_kernel(const __grid_constant__ QueryParams q) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const uint32_t warp = threadIdx.x >> 5;
    unsigned char* base = smem_raw + warp * query_warp_bytes(MODE);
    const WarpCtx W = warpctx_at(base);   // read by MODE_TREE only
    const Pool P = query_pool_at(base + (MODE == MODE_TREE ? kWarpCtxBytes : 0u));
    const SceneRefs sc = scene_refs(q.p);
    Stats st;
    const uint64_t chunks = ((uint64_t)q.n + 31u) / 32u;
    for (uint64_t c = (uint64_t)blockIdx.x * kQueryWarps + warp; c < chunks; c += (uint64_t)gridDim.x * kQueryWarps) {
        const uint64_t i = c * 32u + (uint64_t)lane;
        const bool alive = i < q.n;   // the last chunk has dead lanes
        D3 o = mk(0, 0, 0), d = mk(0, 0, 0);
        if (alive) {
            o = mk(q.origin[3 * i], q.origin[3 * i + 1], q.origin[3 * i + 2]);
            d = mk(q.direction[3 * i], q.direction[3 * i + 1], q.direction[3 * i + 2]);
            P.ox[lane] = o.x; P.oy[lane] = o.y; P.oz[lane] = o.z; P.dx[lane] = d.x; P.dy[lane] = d.y; P.dz[lane] = d.z;
            P.src[lane] = kNoSphere;
        }
        __syncwarp();   // the exact step reads the other lanes' rays
        closest_hit<MODE>(q.p, sc, P, W, alive, (uint32_t)lane, lane, st);
        if (alive) {
            const uint32_t j = P.bi[lane];
            const double r = P.bt[lane];
            const double tm = q.t_max ? q.t_max[i] : DBL_MAX;
            const bool hit = j != kNoSphere && r < tm;   // r < DBL_MAX always, so tm = +inf is tm = DBL_MAX
            D3 pt = mk(0, 0, 0), nrm = mk(0, 0, 0);
            bool front = false;
            double u = 0.0, v = 0.0;
            if (hit && (q.point || q.normal || q.front_face || q.uv)) {
                const double4 g = sc.geo[j];
                const D3 center = mk(g.x, g.y, g.z);
                const HitRec h = hit_record(center, g.w, o, d, r);
                pt = h.point; nrm = h.normal; front = h.front_face;
                if (q.uv) sphere_uv(sub(h.point, center), u, v);
            }
            if (q.t) q.t[i] = hit ? r : __longlong_as_double(0x7ff0000000000000ll);
            if (q.sphere) q.sphere[i] = hit ? j : kNoSphere;
            if (q.point) { q.point[3 * i] = pt.x; q.point[3 * i + 1] = pt.y; q.point[3 * i + 2] = pt.z; }
            if (q.normal) { q.normal[3 * i] = nrm.x; q.normal[3 * i + 1] = nrm.y; q.normal[3 * i + 2] = nrm.z; }
            if (q.uv) { q.uv[2 * i] = u; q.uv[2 * i + 1] = v; }
            if (q.front_face) q.front_face[i] = front ? 1u : 0u;
        }
        __syncwarp();   // every lane is done with the slots before the next chunk overwrites them
    }
    if (q.p.stat) flush_stats(q.p, st, lane);
}

template <uint32_t MODE>
__global__ void __launch_bounds__(kQueryBlock) rt_occluded_kernel(const __grid_constant__ OcclusionParams q) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const uint32_t warp = threadIdx.x >> 5;
    unsigned char* base = smem_raw + warp * occluded_warp_bytes(MODE);
    const WarpCtx W = warpctx_at(base);   // read by MODE_TREE only
    float* tcap = reinterpret_cast<float*>(base + kWarpCtxBytes);   // MODE_TREE only
    const Pool P = query_pool_at(base + (MODE == MODE_TREE ? kWarpCtxBytes + kTcapBytes : 0u));
    const SceneRefs sc = scene_refs(q.p);
    Stats st;
    const uint64_t chunks = ((uint64_t)q.n + 31u) / 32u;
    for (uint64_t c = (uint64_t)blockIdx.x * kQueryWarps + warp; c < chunks; c += (uint64_t)gridDim.x * kQueryWarps) {
        const uint64_t i = c * 32u + (uint64_t)lane;
        const bool alive = i < q.n;   // the last chunk has dead lanes
        double tb = DBL_MAX;   // T
        if (alive) {
            P.ox[lane] = q.origin[3 * i]; P.oy[lane] = q.origin[3 * i + 1]; P.oz[lane] = q.origin[3 * i + 2];
            P.dx[lane] = q.direction[3 * i]; P.dy[lane] = q.direction[3 * i + 1]; P.dz[lane] = q.direction[3 * i + 2];
            P.src[lane] = kNoSphere;
            if (q.t_max) { const double t = q.t_max[i]; tb = t > DBL_MAX ? DBL_MAX : t; }   // +inf counts as f64::MAX; NaN stays NaN
        }
        const bool live = alive && tb > 0.001;   // else no root can be accepted: 0 without a traversal
        __syncwarp();   // the exact step reads the other lanes' rays
        closest_hit<MODE, true>(q.p, sc, P, W, live, (uint32_t)lane, lane, st, live ? tb : DBL_MAX, tcap);
        if (alive) {
            q.occluded[i] = live && P.bi[lane] != kNoSphere ? 1u : 0u;
            if (!live) ++st.rays;
        }
        __syncwarp();   // every lane is done with the slots before the next chunk overwrites them
    }
    if (q.p.stat) flush_stats(q.p, st, lane);
}

template <typename F>
static auto dispatch_query(uint32_t mode, F&& f) {
    if (mode == MODE_EXACT) return f(rt_query_kernel<MODE_EXACT>);
    if (mode == MODE_BRUTE) return f(rt_query_kernel<MODE_BRUTE>);
    return f(rt_query_kernel<MODE_TREE>);
}
template <typename F>
static auto dispatch_occluded(uint32_t mode, F&& f) {
    if (mode == MODE_EXACT) return f(rt_occluded_kernel<MODE_EXACT>);
    if (mode == MODE_BRUTE) return f(rt_occluded_kernel<MODE_BRUTE>);
    return f(rt_occluded_kernel<MODE_TREE>);
}

// one query kind's kernel of `mode` and its dynamic shared memory
template <typename F>
static auto dispatch_kind(bool any, uint32_t mode, F&& f) {
    if (any) return dispatch_occluded(mode, [&](auto kern) { return f(kern, occluded_smem_bytes(mode)); });
    return dispatch_query(mode, [&](auto kern) { return f(kern, query_smem_bytes(mode)); });
}

}  // namespace

int query_max_ctas_per_sm(uint32_t mode, bool any) {
    return dispatch_kind(any, mode, [&](auto kern, size_t smem) -> int { return query_ctas_per_sm(kern, smem); });
}

cudaError_t launch_query(const QueryParams& q, uint32_t mode, int max_grid, cudaStream_t st) {
    return dispatch_query(mode, [&](auto kern) { return query_launch(kern, query_smem_bytes(mode), q, max_grid, st); });
}

cudaError_t launch_occluded(const OcclusionParams& q, uint32_t mode, int max_grid, cudaStream_t st) {
    return dispatch_occluded(mode, [&](auto kern) { return query_launch(kern, occluded_smem_bytes(mode), q, max_grid, st); });
}

}  // namespace rtk
