// rtb200_refit.cu — refit of a resident scene after its spheres moved (rtb200_scene_update_spheres / _geometry_device).
//
// Every position-dependent array is recomputed from the exact geometry `geo`, on the upload's topology (child words, leaf
// members) and recentring offset g, and comes out bit-identical to what rtbvh::Builder emits for the same spheres on that
// topology and g. The host builder is compiled with -ffp-contract=off, so every f64 operation below is an explicit
// __dadd_rn / __dsub_rn / __dmul_rn (nvcc would contract a*b+c into an FMA); (float)x is __double2float_rn, f32_up and
// f32_down are __double2float_ru and __double2float_rd. Why the refit boxes keep the traversal sound: DESIGN.md §4.7.
#include "rtb200_bvh.hpp"
#include "rtb200_kernels.cuh"

namespace rtk {

namespace {

using rtbvh::kU;
using rtbvh::kWide;

// rtbvh::sphere_record; a sphere outside the f32 frame becomes an always-candidate (0, 0, 0, +inf)
__device__ __forceinline__ void refit_record(const double4 G, double gx, double gy, double gz, float rec[4]) {
    const double x = __dsub_rn(G.x, gx), y = __dsub_rn(G.y, gy), z = __dsub_rn(G.z, gz), r2 = __dmul_rn(G.w, G.w);
    const double c2 = __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
    const double Es = __dadd_rn(__dadd_rn(__dmul_rn(96.0 * kU, c2), __dmul_rn(16.0 * kU, r2)), 1e-30);
    const double nkd = __dadd_rn(-__dsub_rn(c2, r2), Es);
    rec[0] = __double2float_rn(x); rec[1] = __double2float_rn(y); rec[2] = __double2float_rn(z);
    rec[3] = isfinite(nkd) ? __double2float_ru(nkd) : INFINITY;
    if (!(isfinite(rec[0]) && isfinite(rec[1]) && isfinite(rec[2]) && isfinite(nkd) && c2 < 1e30)) {
        rec[0] = rec[1] = rec[2] = 0.f; rec[3] = INFINITY;
    }
}

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
    float rec[4];
    refit_record(p.geo[i], p.gx, p.gy, p.gz, rec);
    float* A = p.filt + (size_t)(i / 2) * 8;
    const uint32_t k = i & 1u;
    A[0 + k] = rec[0]; A[2 + k] = rec[1]; A[4 + k] = rec[2]; A[6 + k] = rec[3];
}

// one thread per leaf: the records of its members and its exact box, the union of (c - g) +- |r|. A member the host builder
// would send to the always-list (non-finite, or max|c - g| + |r| >= 1e15) gets an infinite box: the slab test passes it to
// the sphere test, whose record makes it a candidate, so every ray tests it in f64. Padding slots stay as uploaded.
__global__ void __launch_bounds__(256) rt_refit_leaf_kernel(const RefitParams p) {
    const uint32_t leaf = blockIdx.x * blockDim.x + threadIdx.x;
    if (leaf >= p.n_leaves) return;
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int j = 0; j < kLeafK; ++j) {
        const uint32_t id = p.leaf_id[(size_t)leaf * kLeafK + j];
        if (id == rtbvh::kEmptyChild) continue;
        const double4 G = p.geo[id];
        float rec[4];
        refit_record(G, p.gx, p.gy, p.gz, rec);
        float* A = p.leaf_rec + ((size_t)leaf * kLeafK + (size_t)(j / 2) * 2) * 4;
        const int kk = j & 1;
        A[0 + kk] = rec[0]; A[2 + kk] = rec[1]; A[4 + kk] = rec[2]; A[6 + kk] = rec[3];
        const double c[3] = {__dsub_rn(G.x, p.gx), __dsub_rn(G.y, p.gy), __dsub_rn(G.z, p.gz)};
        const double r = fabs(G.w);
        const bool fin = isfinite(c[0]) && isfinite(c[1]) && isfinite(c[2]) && isfinite(r);   // before any max: NaN
        const double ext = fin ? __dadd_rn(fmax(fmax(fabs(c[0]), fabs(c[1])), fabs(c[2])), r) : INFINITY;
        const bool inside = fin && ext < 1e15;
        for (int a = 0; a < 3; ++a) {
            lo[a] = fmin(lo[a], inside ? __dsub_rn(c[a], r) : -INFINITY);
            hi[a] = fmax(hi[a], inside ? __dadd_rn(c[a], r) : INFINITY);
        }
    }
    double* B = p.leaf_box + (size_t)leaf * 6;
    for (int a = 0; a < 3; ++a) { B[a] = lo[a]; B[3 + a] = hi[a]; }
}

// one thread per node of one level: each child slot gets its child's exact box inflated and rounded as Builder::emit_wide
// does (m = 32u * max|coordinate| + 1e-30, lo = f32_down(lo - m), hi = f32_up(hi + m)); the node keeps the union for its parent
__global__ void __launch_bounds__(256) rt_refit_node_kernel(const RefitParams p, const uint32_t* level_nodes, uint32_t count) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const uint32_t node = level_nodes[t];
    float* N = p.nodes + (size_t)node * kNodeVec * 4;
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = 0; i < kWide; ++i) {
        const uint32_t ref = __float_as_uint(N[6 * kWide + i]);
        if (ref == rtbvh::kEmptyChild) continue;   // empty slot: (+inf, -inf) as uploaded
        const double* B = (ref & rtbvh::kLeafBit) ? p.leaf_box + (size_t)(ref & ~rtbvh::kLeafBit) * 6 : p.node_box + (size_t)ref * 6;
        double bmax = 0.0;
        for (int a = 0; a < 3; ++a) bmax = fmax(bmax, fmax(fabs(B[a]), fabs(B[3 + a])));
        const double m = __dadd_rn(__dmul_rn(32.0 * kU, bmax), 1e-30);
        for (int a = 0; a < 3; ++a) {
            N[a * kWide + i] = __double2float_rd(__dsub_rn(B[a], m));
            N[3 * kWide + a * kWide + i] = __double2float_ru(__dadd_rn(B[3 + a], m));
            lo[a] = fmin(lo[a], B[a]);
            hi[a] = fmax(hi[a], B[3 + a]);
        }
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
