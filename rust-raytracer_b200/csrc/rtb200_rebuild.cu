// rtb200_rebuild.cu — rebuild of a resident scene's hierarchy on the GPU (rtb200_scene_rebuild, DESIGN.md §4.8).
//
// Only the topology is new here: the recentring offset g (the host's rule), the always-list, and which spheres share a leaf
// and which nodes share a parent. The position-dependent arrays of that topology are then computed by the refit's kernels
// (rtb200_refit.cu), so they are what the refit computes on it by construction. Steps, each a launch on one stream:
//   1. g: element n/2 of each sorted centre coordinate (cub radix sorts); the median |radius| sets which spheres are oversized;
//   2. sphere_box puts each sphere in the f32 frame or on the always-list (a scan keeps the list in increasing index order);
//   3. 64-bit keys of the in-frame spheres: oversized bit | 30-bit Morton code of the centre | sphere index, radix-sorted;
//   4. top down, one launch pair per wide level: a node owns a contiguous range of the sorted keys and splits it into up to 8
//      children, at the radix split points of the keys on the first kRadixLevels levels, into equal halves below (bounded depth);
//      inner children are numbered by a scan over the level's nodes, leaves by a scan over their first positions: no atomic
//      order reaches the arrays, so the same positions give the same bytes;
//   5. leaf members in increasing index, padding records, skip_pos and the level order (deepest first).
#include <cub/cub.cuh>

#include "rtb200_kernels.cuh"

namespace rtk {

namespace {

using rtbvh::kWide;
constexpr uint32_t kIdMask = (1u << kRebuildIdBits) - 1u;   // sphere index bits of a key
constexpr uint32_t kRadixLevels = 13;   // wide levels split at radix split points; equal-count splits below (DESIGN.md §4.8, depth bound)

inline int blocks_of(uint32_t n) { return (int)((n + 255u) / 256u); }

// order-preserving map of a double onto an unsigned 64-bit integer (for atomicMin / atomicMax)
__device__ __forceinline__ unsigned long long ordered(double x) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(x);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double unordered(unsigned long long u) {
    return __longlong_as_double((long long)((u >> 63) ? (u & 0x7fffffffffffffffull) : ~u));
}

__device__ __forceinline__ void load_geo(const double4* geo, uint32_t i, double G[4]) { const double4 v = geo[i]; G[0] = v.x; G[1] = v.y; G[2] = v.z; G[3] = v.w; }

// the four columns cx, cy, cz, |radius| to be sorted
__global__ void __launch_bounds__(256) rt_rebuild_columns_kernel(const double4* geo, uint32_t n, double* col) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double4 v = geo[i];
    col[i] = v.x; col[(size_t)n + i] = v.y; col[2 * (size_t)n + i] = v.z; col[3 * (size_t)n + i] = fabs(v.w);
}

// g = element n/2 of each sorted coordinate, 0 when it is not finite (Builder::recentre); resets the header
__global__ void rt_rebuild_median_kernel(const double* sorted, uint32_t n, double oversize, RebuildHeader* H) {
    for (int a = 0; a < 3; ++a) {
        const double v = sorted[(size_t)a * n + n / 2];
        H->g[a] = isfinite(v) ? v : 0.0;
    }
    H->r_big = oversize > 0.0 ? oversize * sorted[3 * (size_t)n + n / 2] : INFINITY;
    for (int a = 0; a < 3; ++a) { H->box_lo[a] = ~0ull; H->box_hi[a] = 0ull; }
    H->n_in = H->n_always = H->n_nodes = H->n_leaves = H->depth = H->overflow = 0;
    for (int k = 0; k <= rtbvh::kMaxDepth; ++k) H->level_count[k] = 0;
    for (int k = 0; k <= rtbvh::kMaxDepth + 1; ++k) H->level_base[k] = 0;
}

// sphere_box decides frame membership, as in Builder::run; the Morton box is that of the in-frame, not oversized centres
__global__ void __launch_bounds__(256) rt_rebuild_classify_kernel(const double4* geo, uint32_t n, RebuildHeader* H, uint32_t* out_flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    if (i < n) {
        double G[4], blo[3], bhi[3];
        load_geo(geo, i, G);
        const double g[3] = {H->g[0], H->g[1], H->g[2]};
        const bool inside = rtbvh::sphere_box(G, g, blo, bhi);
        out_flag[i] = !inside;
        if (inside && !(fabs(G[3]) > H->r_big))
            for (int a = 0; a < 3; ++a) lo[a] = hi[a] = rtbvh::sub_rn(G[a], g[a]);
    }
    for (int a = 0; a < 3; ++a)
        for (int o = 16; o > 0; o >>= 1) { lo[a] = fmin(lo[a], __shfl_xor_sync(~0u, lo[a], o)); hi[a] = fmax(hi[a], __shfl_xor_sync(~0u, hi[a], o)); }
    if ((threadIdx.x & 31) == 0 && lo[0] <= hi[0])
        for (int a = 0; a < 3; ++a) { atomicMin(&H->box_lo[a], ordered(lo[a])); atomicMax(&H->box_hi[a], ordered(hi[a])); }
}

__device__ __forceinline__ uint32_t spread3(uint32_t v) {   // 10 bits -> every third bit of 30
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}

// the always-list (increasing index) and the key of every in-frame sphere; out-of-frame spheres get ~0 and sort last
__global__ void __launch_bounds__(256) rt_rebuild_keys_kernel(const double4* geo, uint32_t n, RebuildHeader* H, const uint32_t* out_flag,
                                                             const uint32_t* always_pos, uint32_t* always, unsigned long long* keys, uint2* tasks) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (i == n - 1) {
        const uint32_t n_always = always_pos[i] + out_flag[i];
        H->n_always = n_always; H->n_in = n - n_always;
        H->level_count[0] = n - n_always > 0 ? 1u : 0u;
        tasks[0] = make_uint2(0u, n - n_always);   // the root owns every in-frame sphere
    }
    if (out_flag[i]) { always[always_pos[i]] = i; keys[i] = ~0ull; return; }
    double G[4];
    load_geo(geo, i, G);
    double lo[3], ext = 0.0;
    for (int a = 0; a < 3; ++a) { lo[a] = unordered(H->box_lo[a]); ext = fmax(ext, unordered(H->box_hi[a]) - lo[a]); }
    const bool empty = H->box_lo[0] > H->box_hi[0];   // no in-frame sphere that is not oversized
    uint32_t code = 0;
    for (int a = 0; a < 3; ++a) {
        double t = empty || !(ext > 0.0) ? 0.0 : (rtbvh::sub_rn(G[a], H->g[a]) - lo[a]) / ext * 1024.0;   // one cube: flat scenes split their wide axes
        t = fmin(fmax(t, 0.0), 1023.0);
        code |= spread3((uint32_t)t) << (2 - a);
    }
    const unsigned long long big = fabs(G[3]) > H->r_big ? 1ull : 0ull;
    keys[i] = big << 63 | (unsigned long long)code << kRebuildIdBits | i;
}

// Karras's findSplit: the size of the left part of keys[f, l], cut where the highest differing bit of the range changes
__device__ __forceinline__ uint32_t find_split(const unsigned long long* keys, uint32_t f, uint32_t l) {
    const unsigned long long kf = keys[f];
    const int p = __clzll(kf ^ keys[l]);   // keys are distinct: p < 64
    uint32_t split = f, step = l - f;
    do {
        step = (step + 1) >> 1;
        const uint32_t ns = split + step;
        if (ns < l && __clzll(kf ^ keys[ns]) > p) split = ns;
    } while (step > 1);
    return split - f + 1;
}

// One thread per node of `level`: its children, in key order, and how many of them are inner nodes. Radix levels expand the
// child with the largest Morton cell (shortest common key prefix) first, larger ranges first among equals, until 8 children
// or no child has more than kLeafK spheres; the levels below halve every such child three times.
__global__ void __launch_bounds__(256) rt_rebuild_split_kernel(const unsigned long long* keys, const RebuildHeader* H, uint32_t level,
                                                              const uint2* tasks, uint2* kids, uint32_t* n_inner, uint32_t cap) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= cap) return;
    if (t >= H->level_count[level]) { n_inner[t] = 0; return; }
    uint2 ch[kWide];
    int m = 1;
    ch[0] = tasks[t];
    if (level < kRadixLevels) {
        while (m < kWide) {
            int pick = -1, best_p = 65;
            uint32_t best_c = 0;
            for (int i = 0; i < m; ++i) {
                if (ch[i].y <= (uint32_t)kLeafK) continue;
                const int p = __clzll(keys[ch[i].x] ^ keys[ch[i].x + ch[i].y - 1]);
                if (p < best_p || (p == best_p && ch[i].y > best_c)) { pick = i; best_p = p; best_c = ch[i].y; }
            }
            if (pick < 0) break;
            const uint2 c = ch[pick];
            const uint32_t left = find_split(keys, c.x, c.x + c.y - 1);
            for (int i = m; i > pick + 1; --i) ch[i] = ch[i - 1];
            ch[pick] = make_uint2(c.x, left);
            ch[pick + 1] = make_uint2(c.x + left, c.y - left);
            ++m;
        }
    } else {
        for (int round = 0; round < 3; ++round)
            for (int i = m - 1; i >= 0; --i) {
                const uint2 c = ch[i];
                if (c.y <= (uint32_t)kLeafK) continue;
                const uint32_t left = c.y - c.y / 2;
                for (int j = m; j > i + 1; --j) ch[j] = ch[j - 1];
                ch[i] = make_uint2(c.x, left);
                ch[i + 1] = make_uint2(c.x + left, c.y - left);
                ++m;
            }
    }
    uint32_t inner = 0;
    for (int i = 0; i < kWide; ++i) {
        const uint2 c = i < m ? ch[i] : make_uint2(0u, 0u);
        kids[(size_t)t * kWide + i] = c;
        inner += c.y > (uint32_t)kLeafK;
    }
    n_inner[t] = inner;
}

// One thread per node of `level`: its child words. Inner children become the next level's nodes (numbered by the scan `off`);
// a leaf child is written as kLeafBit | its first key position until the leaves are numbered. Empty slots get (+inf, -inf).
__global__ void __launch_bounds__(256) rt_rebuild_emit_kernel(RebuildHeader* H, uint32_t level, const uint2* kids, const uint32_t* n_inner,
                                                             const uint32_t* off, uint2* next, float* nodes, uint32_t* leaf_start,
                                                             uint32_t* leaf_cnt) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t T = H->level_count[level], base = H->level_base[level];
    if (T == 0) {
        if (t == 0) { H->level_count[level + 1] = 0; H->level_base[level + 1] = base; }
        return;
    }
    if (t >= T) return;
    if (t == T - 1) { H->level_count[level + 1] = off[t] + n_inner[t]; H->level_base[level + 1] = base + T; }
    float* N = nodes + (size_t)(base + t) * rtbvh::kNodeFloats;
    uint32_t k = off[t];
    for (int i = 0; i < kWide; ++i) {
        const uint2 c = kids[(size_t)t * kWide + i];
        uint32_t ref;
        if (c.y == 0) {
            ref = rtbvh::kEmptyChild;
            for (int a = 0; a < 3; ++a) { N[a * kWide + i] = INFINITY; N[3 * kWide + a * kWide + i] = -INFINITY; }   // never hit
        } else if (c.y > (uint32_t)kLeafK) {
            ref = base + T + k;
            next[k++] = c;
        } else {
            ref = rtbvh::kLeafBit | c.x;
            leaf_start[c.x] = 1u;
            leaf_cnt[c.x] = c.y;
        }
        memcpy(N + rtbvh::kChildOff + i, &ref, 4);
    }
}

__global__ void rt_rebuild_counts_kernel(RebuildHeader* H, const uint32_t* leaf_start, const uint32_t* leaf_scan, uint32_t n) {
    uint32_t depth = 0;
    while (depth < (uint32_t)rtbvh::kMaxDepth && H->level_count[depth] > 0) ++depth;
    H->depth = depth;
    H->n_nodes = H->level_base[depth];
    H->overflow = H->level_count[rtbvh::kMaxDepth] > 0;   // nodes below kMaxDepth levels: never, by the depth bound
    H->n_leaves = leaf_scan[n - 1] + leaf_start[n - 1];
}

// One thread per key position that starts a leaf: its members in increasing index, padding slots, and skip_pos of the members.
__global__ void __launch_bounds__(256) rt_rebuild_leaf_kernel(const unsigned long long* keys, uint32_t n, const uint32_t* leaf_start,
                                                             const uint32_t* leaf_scan, const uint32_t* leaf_cnt, uint32_t* leaf_id,
                                                             float* leaf_rec, uint32_t* skip_pos) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n || !leaf_start[p]) return;
    const uint32_t leaf = leaf_scan[p], c = leaf_cnt[p];
    uint32_t mem[kLeafK];
    for (uint32_t j = 0; j < c; ++j) {   // insertion sort of at most kLeafK indices
        const uint32_t id = (uint32_t)keys[p + j] & kIdMask;
        uint32_t s = j;
        for (; s > 0 && mem[s - 1] > id; --s) mem[s] = mem[s - 1];
        mem[s] = id;
    }
    const float pad[4] = {0.f, 0.f, 0.f, -INFINITY};   // padding slot: never hit
    for (uint32_t j = 0; j < (uint32_t)kLeafK; ++j) {
        const size_t slot = (size_t)leaf * kLeafK + j;
        if (j < c) { leaf_id[slot] = mem[j]; skip_pos[mem[j]] = (uint32_t)slot; }
        else { leaf_id[slot] = rtbvh::kPadId; rtbvh::put_record(leaf_rec + (size_t)leaf * kLeafK * 4, j, pad); }
    }
}

// One thread per node: leaf child words get the leaf's number, a single-member leaf is left out by its parent slot
// (build_records' skip_pos rule), and the node takes its place in the level order, deepest level first.
__global__ void __launch_bounds__(256) rt_rebuild_nodes_kernel(const unsigned long long* keys, const RebuildHeader* H, const uint32_t* leaf_scan,
                                                              const uint32_t* leaf_cnt, float* nodes, uint32_t* skip_pos, uint32_t* level_nodes,
                                                              uint32_t cap) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    const uint32_t nn = H->n_nodes;
    if (i >= nn) return;
    float* N = nodes + (size_t)i * rtbvh::kNodeFloats;
    for (int c = 0; c < kWide; ++c) {
        const uint32_t ref = rtbvh::child_of(N, c);
        if (ref == rtbvh::kEmptyChild || !(ref & rtbvh::kLeafBit)) continue;
        const uint32_t p = ref & ~rtbvh::kLeafBit, leaf = rtbvh::kLeafBit | leaf_scan[p];
        memcpy(N + rtbvh::kChildOff + c, &leaf, 4);
        if (leaf_cnt[p] == 1) skip_pos[(uint32_t)keys[p] & kIdMask] = rtbvh::kSkipNodeBit | (i * (uint32_t)kWide + (uint32_t)c);
    }
    uint32_t l = 0;
    while (i >= H->level_base[l + 1]) ++l;
    level_nodes[(nn - H->level_base[l + 1]) + (i - H->level_base[l])] = i;
}

// cub's temporary storage for the sorts and scans of n spheres and `cap` nodes per level
size_t cub_bytes(uint32_t n, uint32_t cap) {
    size_t a = 0, b = 0, c = 0, d = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, a, (const double*)nullptr, (double*)nullptr, (int)n);
    cub::DeviceRadixSort::SortKeys(nullptr, b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n);
    cub::DeviceScan::ExclusiveSum(nullptr, c, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
    cub::DeviceScan::ExclusiveSum(nullptr, d, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)cap);
    return std::max(std::max(a, b), std::max(c, d));
}

}  // namespace

// Carve the rebuild's arrays for n spheres out of `base` (null: only the size); returns the bytes. Bounds: every leaf holds a
// sphere, every inner node two children (but a root over at most kLeafK spheres): n_leaves <= n, n_nodes <= max(n, 1); the
// inner nodes of one level own disjoint ranges of more than kLeafK spheres: at most n / (kLeafK + 1) + 1 per level.
size_t rebuild_carve(void* base, uint32_t n, RebuildBufs* b) {
    const size_t n1 = std::max<uint32_t>(n, 1), cap = n / (kLeafK + 1) + 1;
    Carver c(base);
    RebuildBufs r{};
    r.cap = (uint32_t)cap;
    r.header = (RebuildHeader*)c.take(sizeof(RebuildHeader));
    r.nodes = (float*)c.take(n1 * rtbvh::kNodeFloats * 4);
    r.leaf_rec = (float*)c.take(n1 * kLeafK * 16);
    r.leaf_id = (uint32_t*)c.take(n1 * kLeafK * 4);
    r.skip_pos = (uint32_t*)c.take(n1 * 4);
    r.always = (uint32_t*)c.take(n1 * 4);
    r.node_box = (double*)c.take(n1 * 48);
    r.leaf_box = (double*)c.take(n1 * 48);
    r.level_nodes = (uint32_t*)c.take(n1 * 4);
    r.col = (double*)c.take(n1 * 32);            // the four columns; then the keys and the sorted keys
    r.sorted = (double*)c.take(n1 * 32);
    r.keys = (unsigned long long*)r.col;
    r.keys_sorted = (unsigned long long*)r.col + n1;
    r.out_flag = (uint32_t*)c.take(n1 * 4);
    r.always_pos = (uint32_t*)c.take(n1 * 4);
    r.leaf_start = (uint32_t*)c.take(n1 * 4);
    r.leaf_scan = (uint32_t*)c.take(n1 * 4);
    r.leaf_cnt = (uint32_t*)c.take(n1 * 4);
    r.tasks[0] = (uint2*)c.take(cap * 8);
    r.tasks[1] = (uint2*)c.take(cap * 8);
    r.kids = (uint2*)c.take(cap * kWide * 8);
    r.n_inner = (uint32_t*)c.take(cap * 4);
    r.off = (uint32_t*)c.take(cap * 4);
    r.temp_bytes = cub_bytes(n, (uint32_t)cap);
    r.temp = c.take(r.temp_bytes);
    if (b) *b = r;
    return c.off;
}

cudaError_t launch_rebuild_topology(const RebuildBufs& b, const double4* geo, uint32_t n, double oversize, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    cudaError_t e;
    size_t tb = b.temp_bytes;
    rt_rebuild_columns_kernel<<<blocks_of(n), 256, 0, st>>>(geo, n, b.col);
    for (int a = 0; a < 4; ++a)
        if ((e = cub::DeviceRadixSort::SortKeys(b.temp, tb, b.col + (size_t)a * n, b.sorted + (size_t)a * n, (int)n, 0, 64, st)) != cudaSuccess) return e;
    rt_rebuild_median_kernel<<<1, 1, 0, st>>>(b.sorted, n, oversize, b.header);
    rt_rebuild_classify_kernel<<<blocks_of(n), 256, 0, st>>>(geo, n, b.header, b.out_flag);
    if ((e = cub::DeviceScan::ExclusiveSum(b.temp, tb, b.out_flag, b.always_pos, (int)n, st)) != cudaSuccess) return e;
    rt_rebuild_keys_kernel<<<blocks_of(n), 256, 0, st>>>(geo, n, b.header, b.out_flag, b.always_pos, b.always, b.keys, b.tasks[0]);
    if ((e = cub::DeviceRadixSort::SortKeys(b.temp, tb, b.keys, b.keys_sorted, (int)n, 0, 64, st)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(b.leaf_start, 0, (size_t)n * 4, st)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(b.skip_pos, 0xff, (size_t)n * 4, st)) != cudaSuccess) return e;
    for (uint32_t level = 0; level < (uint32_t)rtbvh::kMaxDepth; ++level) {   // the host never waits between levels
        const uint2* tasks = b.tasks[level & 1];
        rt_rebuild_split_kernel<<<blocks_of(b.cap), 256, 0, st>>>(b.keys_sorted, b.header, level, tasks, b.kids, b.n_inner, b.cap);
        if ((e = cub::DeviceScan::ExclusiveSum(b.temp, tb, b.n_inner, b.off, (int)b.cap, st)) != cudaSuccess) return e;
        rt_rebuild_emit_kernel<<<blocks_of(b.cap), 256, 0, st>>>(b.header, level, b.kids, b.n_inner, b.off, b.tasks[(level + 1) & 1], b.nodes,
                                                                 b.leaf_start, b.leaf_cnt);
    }
    if ((e = cub::DeviceScan::ExclusiveSum(b.temp, tb, b.leaf_start, b.leaf_scan, (int)n, st)) != cudaSuccess) return e;
    rt_rebuild_counts_kernel<<<1, 1, 0, st>>>(b.header, b.leaf_start, b.leaf_scan, n);
    rt_rebuild_leaf_kernel<<<blocks_of(n), 256, 0, st>>>(b.keys_sorted, n, b.leaf_start, b.leaf_scan, b.leaf_cnt, b.leaf_id, b.leaf_rec, b.skip_pos);
    rt_rebuild_nodes_kernel<<<blocks_of(n), 256, 0, st>>>(b.keys_sorted, b.header, b.leaf_scan, b.leaf_cnt, b.nodes, b.skip_pos, b.level_nodes, n);
    return cudaGetLastError();
}

}  // namespace rtk
