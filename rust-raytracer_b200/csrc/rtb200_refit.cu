// rtb200_refit.cu — refit of a resident scene after its spheres moved (rtb200_scene_update_spheres / _geometry_device).
//
// Every position-dependent array is recomputed from the exact geometry `geo`, on the upload's topology (child words, leaf
// members) and recentring offset g, by the same functions rtbvh::Builder uses on the host (sphere_record, sphere_box,
// set_child_box, put_record in rtb200_bvh.hpp, compiled for both): the arrays are what the host build emits for the same
// spheres on that topology and g. Why the refit boxes keep the traversal sound: DESIGN.md §4.7.
#include "rtb200_kernels.cuh"

namespace rtk {

namespace {

using rtbvh::kWide;

__device__ __forceinline__ void load_geo(const double4* geo, uint32_t i, double G[4]) { const double4 v = geo[i]; G[0] = v.x; G[1] = v.y; G[2] = v.z; G[3] = v.w; }

__global__ void __launch_bounds__(256) rt_update_scatter_kernel(const uint32_t* idx, const double4* geo_in, const DevMat* mat_in,
                                                                uint32_t n, double4* geo, DevMat* mat) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint32_t i = idx[k];
    geo[i] = geo_in[k];
    mat[i] = mat_in[k];
}

// one thread per sphere: its slot of the pair-packed flat records (MODE_BRUTE)
__global__ void __launch_bounds__(256) rt_refit_flat_kernel(const RefitParams p) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    double G[4];
    float rec[4];
    load_geo(p.geo, i, G);
    rtbvh::sphere_record(G, p.g, rec);
    rtbvh::put_record(p.filt, i, rec);
}

// one thread per leaf: the records of its members and its exact box, the union of their sphere_box. A member the host builder
// would send to the always-list gets an infinite box: the slab test passes it to the sphere test, whose record makes it a
// candidate, so every ray tests it in f64. Padding slots stay as uploaded.
__global__ void __launch_bounds__(256) rt_refit_leaf_kernel(const RefitParams p) {
    const uint32_t leaf = blockIdx.x * blockDim.x + threadIdx.x;
    if (leaf >= p.n_leaves) return;
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int j = 0; j < kLeafK; ++j) {
        const uint32_t id = p.leaf_id[(size_t)leaf * kLeafK + j];
        if (id == rtbvh::kPadId) continue;
        double G[4], blo[3], bhi[3];
        float rec[4];
        load_geo(p.geo, id, G);
        rtbvh::sphere_record(G, p.g, rec);
        rtbvh::put_record(p.leaf_rec + (size_t)leaf * kLeafK * 4, j, rec);
        rtbvh::sphere_box(G, p.g, blo, bhi);
        for (int a = 0; a < 3; ++a) { lo[a] = fmin(lo[a], blo[a]); hi[a] = fmax(hi[a], bhi[a]); }
    }
    double* B = p.leaf_box + (size_t)leaf * 6;
    for (int a = 0; a < 3; ++a) { B[a] = lo[a]; B[3 + a] = hi[a]; }
}

// one thread per node of one level: each child slot gets its child's exact box through set_child_box, as in
// Builder::emit_wide; the node keeps the union for its parent
__global__ void __launch_bounds__(256) rt_refit_node_kernel(const RefitParams p, const uint32_t* level_nodes, uint32_t count) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const uint32_t node = level_nodes[t];
    float* N = p.nodes + (size_t)node * rtbvh::kNodeFloats;
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = 0; i < kWide; ++i) {
        const uint32_t ref = rtbvh::child_of(N, i);
        if (ref == rtbvh::kEmptyChild) continue;   // empty slot: (+inf, -inf) as uploaded
        const double* B = (ref & rtbvh::kLeafBit) ? p.leaf_box + (size_t)(ref & ~rtbvh::kLeafBit) * 6 : p.node_box + (size_t)ref * 6;
        const double blo[3] = {B[0], B[1], B[2]}, bhi[3] = {B[3], B[4], B[5]};   // read once: the stores to N may alias B
        rtbvh::set_child_box(N, i, blo, bhi);
        for (int a = 0; a < 3; ++a) { lo[a] = fmin(lo[a], blo[a]); hi[a] = fmax(hi[a], bhi[a]); }
    }
    double* D = p.node_box + (size_t)node * 6;
    for (int a = 0; a < 3; ++a) { D[a] = lo[a]; D[3 + a] = hi[a]; }
}

inline int blocks_of(uint32_t n) { return (int)((n + 255u) / 256u); }

}  // namespace

cudaError_t launch_update_scatter(const uint32_t* idx, const double4* geo_in, const DevMat* mat_in, uint32_t n, double4* geo, DevMat* mat,
                                  cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    rt_update_scatter_kernel<<<blocks_of(n), 256, 0, st>>>(idx, geo_in, mat_in, n, geo, mat);
    return cudaGetLastError();
}

cudaError_t launch_refit_spheres(const RefitParams& p, cudaStream_t st) {
    if (p.filt && p.n) rt_refit_flat_kernel<<<blocks_of(p.n), 256, 0, st>>>(p);
    if (p.leaf_rec && p.n_leaves) rt_refit_leaf_kernel<<<blocks_of(p.n_leaves), 256, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_refit_nodes(const RefitParams& p, const uint32_t* level_nodes, uint32_t count, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    rt_refit_node_kernel<<<blocks_of(count), 256, 0, st>>>(p, level_nodes, count);
    return cudaGetLastError();
}

}  // namespace rtk
