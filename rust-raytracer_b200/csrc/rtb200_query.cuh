// rtb200_query.cuh — the CTA of the kernels that run the trace kernel's closest-hit stage on rays they load or make
// themselves: the queries (rtb200_query.cu, DESIGN.md §4.10, §4.11) and the auxiliary buffers (rtb200_aov.cu, §4.14).
// 128 threads; per warp its traversal context (MODE_TREE) and 32 pool slots holding only what closest_hit touches. The warps
// of a CTA share nothing, so there is no CTA barrier.
#pragma once
#include <algorithm>

#include "rtb200_trace.cuh"

namespace rtk {

constexpr int kQueryBlock = 128;
constexpr uint32_t kQueryWarps = kQueryBlock / 32;
constexpr uint32_t kQuerySlotBytes = 7 * 8 + 2 * 4;   // Pool.ox .. Pool.bt, Pool.bi, Pool.src

// shared memory of one warp: its traversal context (MODE_TREE), then its 32 pool slots
__host__ __device__ constexpr uint32_t query_warp_bytes(uint32_t mode) {
    return (mode == MODE_TREE ? kWarpCtxBytes : 0u) + 32u * kQuerySlotBytes;
}
constexpr size_t query_smem_bytes(uint32_t mode) { return (size_t)kQueryWarps * query_warp_bytes(mode); }

// the 32 pool slots of a warp at `slots`: closest_hit touches the ray, the best root and index, and the source sphere of a slot
RT_DEV Pool query_pool_at(unsigned char* slots) {
    double* dbl = reinterpret_cast<double*>(slots);
    uint32_t* u32 = reinterpret_cast<uint32_t*>(dbl + 7 * 32);
    Pool P{};
    P.ox = dbl; P.oy = dbl + 32; P.oz = dbl + 64; P.dx = dbl + 96; P.dy = dbl + 128; P.dz = dbl + 160; P.bt = dbl + 192;
    P.bi = u32; P.src = u32 + 32;
    P.n_slots = 32u;
    return P;
}

RT_DEV SceneRefs scene_refs(const TraceParams& p) {
    SceneRefs sc;
    sc.nodes = p.nodes; sc.leaf_rec = p.leaf_rec; sc.leaf_id = p.leaf_id; sc.filt = p.filt; sc.geo = p.geo; sc.mat = p.mat;
    return sc;
}

// resident CTAs per SM of `kern` with `smem` bytes of dynamic shared memory (0 when it cannot run on the current device)
template <typename K>
int query_ctas_per_sm(K kern, size_t smem) {
    int nb = 0;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { cudaGetLastError(); return 0; }
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kQueryBlock, smem) != cudaSuccess) { cudaGetLastError(); return 0; }
    return nb;
}

// a launch over q.n items in chunks of 32, of at most max_grid CTAs (no more than the chunks need)
template <typename K, typename Q>
cudaError_t query_launch(K kern, size_t smem, const Q& q, int max_grid, cudaStream_t st) {
    if (q.n == 0) return cudaSuccess;
    const uint64_t ctas = ((uint64_t)q.n + 32u * kQueryWarps - 1u) / (32u * kQueryWarps);
    const int grid = (int)std::min<uint64_t>(ctas, (uint64_t)std::max(max_grid, 1));
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, kQueryBlock, smem, st>>>(q);
    return cudaGetLastError();
}

}  // namespace rtk
