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
#include <algorithm>

#include "rtb200_trace.cuh"

namespace rtk {

namespace {

constexpr int kQueryBlock = 128;
constexpr uint32_t kQueryWarps = kQueryBlock / 32;
constexpr uint32_t kQuerySlotBytes = 7 * 8 + 2 * 4;   // Pool.ox .. Pool.bt, Pool.bi, Pool.src

// shared memory of one warp: its traversal context (MODE_TREE), then its 32 pool slots
__host__ __device__ constexpr uint32_t query_warp_bytes(uint32_t mode) {
    return (mode == MODE_TREE ? kWarpCtxBytes : 0u) + 32u * kQuerySlotBytes;
}
constexpr size_t query_smem_bytes(uint32_t mode) { return (size_t)kQueryWarps * query_warp_bytes(mode); }

template <uint32_t MODE>
__global__ void __launch_bounds__(kQueryBlock) rt_query_kernel(const __grid_constant__ QueryParams q) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const uint32_t warp = threadIdx.x >> 5;
    unsigned char* base = smem_raw + warp * query_warp_bytes(MODE);
    const WarpCtx W = warpctx_at(base);   // read by MODE_TREE only
    double* dbl = reinterpret_cast<double*>(base + (MODE == MODE_TREE ? kWarpCtxBytes : 0u));
    uint32_t* u32 = reinterpret_cast<uint32_t*>(dbl + 7 * 32);
    Pool P{};   // closest_hit touches the ray, the best root and index, and the source sphere of a slot
    P.ox = dbl; P.oy = dbl + 32; P.oz = dbl + 64; P.dx = dbl + 96; P.dy = dbl + 128; P.dz = dbl + 160; P.bt = dbl + 192;
    P.bi = u32; P.src = u32 + 32;
    P.n_slots = 32u;
    SceneRefs sc;
    sc.nodes = q.p.nodes; sc.leaf_rec = q.p.leaf_rec; sc.leaf_id = q.p.leaf_id; sc.filt = q.p.filt; sc.geo = q.p.geo; sc.mat = q.p.mat;
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

template <typename F>
static auto dispatch_query(uint32_t mode, F&& f) {
    if (mode == MODE_EXACT) return f(rt_query_kernel<MODE_EXACT>);
    if (mode == MODE_BRUTE) return f(rt_query_kernel<MODE_BRUTE>);
    return f(rt_query_kernel<MODE_TREE>);
}

}  // namespace

int query_max_ctas_per_sm(uint32_t mode) {
    return dispatch_query(mode, [&](auto kern) -> int {
        const size_t smem = query_smem_bytes(mode);
        int nb = 0;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { cudaGetLastError(); return 0; }
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kQueryBlock, smem) != cudaSuccess) { cudaGetLastError(); return 0; }
        return nb;
    });
}

cudaError_t launch_query(const QueryParams& q, uint32_t mode, int max_grid, cudaStream_t st) {
    if (q.n == 0) return cudaSuccess;
    const uint64_t ctas = ((uint64_t)q.n + 32u * kQueryWarps - 1u) / (32u * kQueryWarps);
    const int grid = (int)std::min<uint64_t>(ctas, (uint64_t)std::max(max_grid, 1));
    return dispatch_query(mode, [&](auto kern) -> cudaError_t {
        const size_t smem = query_smem_bytes(mode);
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        kern<<<grid, kQueryBlock, smem, st>>>(q);
        return cudaGetLastError();
    });
}

}  // namespace rtk
