// rtb200_edit.cu — insert and remove spheres of a resident scene (rtb200_scene_edit_spheres, DESIGN.md §4.13).
//
// The edited list is the old list without the removed spheres, with insert k placed just before old sphere at[k]. With
// kept(< j) the number of kept old spheres below j, a kept old sphere i goes to kept(< i) + #{k : at[k] <= i} and insert k to
// kept(< at[k]) + k. Steps, each a launch on one stream:
//   1. keep[i] = 1 for every old sphere, keep[n_old] = 0; then keep[remove[k]] = 0;
//   2. pos = exclusive scan of keep[0, n_old] (cub), so pos[j] = kept(< j) for every j <= n_old;
//   3. one thread per old sphere and per insert writes its geo and mat record at its new position, into arrays that are not
//      the old ones (frames enqueued before the edit still read those);
//   4. MODE_BRUTE: the flat-record slots past the new list get the builder's padding. The records of the spheres themselves are
//      the refit's (launch_refit_spheres), and the tree is the rebuild's (rtb200_rebuild.cu).
#include <cub/cub.cuh>

#include "rtb200_kernels.cuh"

namespace rtk {

namespace {

inline int blocks_of(uint32_t n) { return (int)((n + 255u) / 256u); }

__global__ void __launch_bounds__(256) rt_edit_keep_kernel(uint32_t* keep, uint32_t n_old) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n_old) keep[i] = i < n_old ? 1u : 0u;
}

__global__ void __launch_bounds__(256) rt_edit_remove_kernel(uint32_t* keep, const uint32_t* remove, uint32_t n_remove) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n_remove) keep[remove[k]] = 0u;
}

// threads [0, n_old): the old spheres; [n_old, n_old + n_insert): the inserts
__global__ void __launch_bounds__(256) rt_edit_scatter_kernel(const EditParams p) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < p.n_old) {
        if (!p.keep[t]) return;
        uint32_t lo = 0, hi = p.n_insert;   // #{k : at[k] <= t}: at is non-decreasing
        while (lo < hi) {
            const uint32_t mid = (lo + hi) / 2;
            if (p.at[mid] <= t) lo = mid + 1;
            else hi = mid;
        }
        const uint32_t dst = p.pos[t] + lo;
        p.geo[dst] = p.geo_old[t];
        p.mat[dst] = p.mat_old[t];
    } else if (t - p.n_old < p.n_insert) {
        const uint32_t k = t - p.n_old, dst = p.pos[p.at[k]] + k;
        p.geo[dst] = p.geo_in[k];
        p.mat[dst] = p.mat_in[k];
    }
}

// flat-record slots [first, slots): padding that never hits (Builder::flat_and_exact)
__global__ void __launch_bounds__(256) rt_edit_pad_kernel(float* filt, uint32_t first, uint32_t slots) {
    const uint32_t s = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= slots) return;
    const float pad[4] = {0.f, 0.f, 0.f, -INFINITY};
    rtbvh::put_record(filt, s, pad);
}

}  // namespace

size_t edit_scan_bytes(uint32_t n_old) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n_old + 1);
    return bytes;
}

cudaError_t launch_edit_spheres(const EditParams& p, cudaStream_t st) {
    rt_edit_keep_kernel<<<blocks_of(p.n_old + 1), 256, 0, st>>>(p.keep, p.n_old);
    if (p.n_remove) rt_edit_remove_kernel<<<blocks_of(p.n_remove), 256, 0, st>>>(p.keep, p.remove, p.n_remove);
    size_t tb = p.temp_bytes;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(p.temp, tb, p.keep, p.pos, (int)p.n_old + 1, st);
    if (e != cudaSuccess) return e;
    if (p.n_old + p.n_insert) rt_edit_scatter_kernel<<<blocks_of(p.n_old + p.n_insert), 256, 0, st>>>(p);
    const uint32_t n_new = p.n_old - p.n_remove + p.n_insert;
    if (p.filt && 2 * p.n_pairs > n_new) rt_edit_pad_kernel<<<blocks_of(2 * p.n_pairs - n_new), 256, 0, st>>>(p.filt, n_new, 2 * p.n_pairs);
    return cudaGetLastError();
}

}  // namespace rtk
