// rtb200_distance.cu — point queries on a resident scene (rtb200_scene_nearest[_device], rtb200_scene_overlaps[_device],
// DESIGN.md §4.19): the nearest sphere to each point under a bound, and whether a ball overlaps any sphere.
//
// One point per thread, in the 128-thread CTA of the query kernels (rtb200_query.cuh) without its shared memory: the warps share
// nothing. dist_j = fl(sqrt(x*x + y*y + z*z)) - |R| in f64 round-to-nearest, never contracted (include/rtb200.h).
//
// MODE_TREE walks the 8-wide hierarchy depth first, nearest child first, from a per-thread stack of (child word, L~) entries,
// L~ a lower bound in f32 on dist_j of every sphere under that child (-inf when the point may lie inside the child's box). A
// child is pruned iff L~ > D~, the current best distance (or the bound) rounded up to f32; a popped entry is re-tested against
// the D~ of that moment before its node or leaf is loaded. Leaves get the exact f64 distance of every member. The always-list
// is evaluated exactly for every point; a point outside the f32 frame's range (or with a non-finite coordinate) scans every
// sphere in f64 instead. MODE_BRUTE and MODE_EXACT scan every sphere in f64: the flat records carry no radius to filter by.
//
// ANY (overlaps): D~ is r rounded up and never shrinks; the first sphere with dist_j < r answers the ball.
#include "rtb200_query.cuh"

namespace rtk {

namespace {

constexpr uint32_t kNone = 0xffffffffu;
constexpr double kInfD = __builtin_huge_val();
constexpr int kDistStack = 7 * rtbvh::kMaxDepth + 1;   // one pop and at most 8 pushes per level below the root entry

// dist_j of the contract
RT_DEV double sphere_dist(const double4& g, double px, double py, double pz) {
    const double x = __dsub_rn(px, g.x), y = __dsub_rn(py, g.y), z = __dsub_rn(pz, g.z);
    const double s = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
    return __dsub_rn(s, fabs(g.w));
}

template <uint32_t MODE, bool ANY>
__global__ void __launch_bounds__(kQueryBlock) rt_nearest_kernel(const __grid_constant__ DistanceParams q) {
    const TraceParams& p = q.p;
    const int lane = threadIdx.x & 31;
    Stats st;
    const uint64_t stride = (uint64_t)gridDim.x * kQueryBlock;
    for (uint64_t i = (uint64_t)blockIdx.x * kQueryBlock + threadIdx.x; i < q.n; i += stride) {
        const double px = q.point[3 * i], py = q.point[3 * i + 1], pz = q.point[3 * i + 2];
        const double b = q.bound ? q.bound[i] : kInfD;
        ++st.rays;
        double best = b;   // the best distance, or the bound before any sphere qualifies
        uint32_t bj = kNone;
        // sphere j: the nearest kind keeps the least (dist_j, j) below the bound; the overlaps kind stops at dist_j < r
        auto eval = [&](uint32_t j) {
            const double d = sphere_dist(p.geo[j], px, py, pz);
            ++st.cand;
            if (ANY) { if (d < b) bj = j; }
            else if (d < best || (d == best && bj != kNone && j < bj)) { best = d; bj = j; }
        };
        if (b > -kInfD) {   // a NaN or -inf bound admits no sphere
            const float ofx = __double2float_rn(__dsub_rn(px, p.gx)), ofy = __double2float_rn(__dsub_rn(py, p.gy)),
                        ofz = __double2float_rn(__dsub_rn(pz, p.gz));
            const float oo = fmaf(ofx, ofx, fmaf(ofy, ofy, ofz * ofz));
            if (MODE != MODE_TREE || !(oo < 1e30f)) {   // the f32 frame's range of the rays (closest_hit)
                ++st.ovf;
                for (uint32_t j = 0; j < p.n; ++j) {
                    eval(j);
                    if (ANY && bj != kNone) break;
                }
            } else {
                for (uint32_t k = 0; k < p.n_always && !(ANY && bj != kNone); ++k) eval(p.always[k]);
                // slack of the recentred point: |pf - (p - g)| <= u|p - g| + 2^-53|p - g| <= 2u|pf| (+ 1e-30 below the normal range)
                const float nrm = __fsqrt_ru(__fadd_ru(__fadd_ru(__fmul_ru(ofx, ofx), __fmul_ru(ofy, ofy)), __fmul_ru(ofz, ofz)));
                const float slack = __fadd_ru(__fmul_ru(1.1920928955078125e-7f, nrm), 1e-30f);
                uint2 stack[kDistStack];
                int sp = 0;
                if (p.n_nodes != 0u && !(ANY && bj != kNone)) stack[sp++] = make_uint2(0u, __float_as_uint(-INFINITY));   // the root node
                while (sp > 0) {
                    const uint2 e = stack[--sp];
                    const float Dt = __double2float_ru(best);   // D~ (ANY: r rounded up, as best stays b)
                    if (__uint_as_float(e.y) > Dt) continue;
                    if (e.x & kLeafBit) {
                        const uint32_t* ids = p.leaf_id + (size_t)(e.x & ~kLeafBit) * kLeafK;
                        ++st.leaves;
#pragma unroll
                        for (int k = 0; k < kLeafK; ++k) {
                            const uint32_t j = ids[k];
                            if (j != rtbvh::kPadId && !(ANY && bj != kNone)) eval(j);
                        }
                        if (ANY && bj != kNone) break;
                        continue;
                    }
                    ++st.nodes;
                    const float* N = reinterpret_cast<const float*>(p.nodes + (size_t)e.x * kNodeVec);
                    const uint32_t* refs = reinterpret_cast<const uint32_t*>(N + rtbvh::kChildOff);
                    float L[8];
                    uint32_t keep = 0u;
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        // distance from pf to the stored box, every step rounded down, minus the slack; <= 0: no bound
                        const float ex = fmaxf(fmaxf(__fsub_rd(N[c], ofx), __fsub_rd(ofx, N[24 + c])), 0.f);
                        const float ey = fmaxf(fmaxf(__fsub_rd(N[8 + c], ofy), __fsub_rd(ofy, N[32 + c])), 0.f);
                        const float ez = fmaxf(fmaxf(__fsub_rd(N[16 + c], ofz), __fsub_rd(ofz, N[40 + c])), 0.f);
                        const float l = __fsub_rd(__fsqrt_rd(__fadd_rd(__fadd_rd(__fmul_rd(ex, ex), __fmul_rd(ey, ey)), __fmul_rd(ez, ez))), slack);
                        L[c] = l > 0.f ? l : -INFINITY;
                        keep |= (refs[c] != rtbvh::kEmptyChild && !(L[c] > Dt) ? 1u : 0u) << c;
                    }
                    const int cnt = __popc(keep);
                    if (sp + cnt > kDistStack) { atomicAdd(&p.err[1], 1ull); break; }   // cannot happen (depth <= kMaxDepth)
                    // nearest child on top: child c goes below the `rank` children that are nearer (ties by slot)
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        int rank = 0;
#pragma unroll
                        for (int k = 0; k < 8; ++k)
                            rank += ((keep >> k) & 1u) && (L[k] < L[c] || (L[k] == L[c] && k < c)) ? 1 : 0;
                        if ((keep >> c) & 1u) stack[sp + cnt - 1 - rank] = make_uint2(refs[c], __float_as_uint(L[c]));
                    }
                    sp += cnt;
                }
            }
        }
        if (ANY) {
            q.overlaps[i] = bj != kNone ? 1u : 0u;
        } else {
            if (q.distance) q.distance[i] = bj != kNone ? best : kInfD;
            if (q.sphere) q.sphere[i] = bj;
        }
    }
    if (p.stat) flush_stats(p, st, lane);
}

template <bool ANY, typename F>
static auto dispatch_nearest(uint32_t mode, F&& f) {
    if (mode == MODE_EXACT) return f(rt_nearest_kernel<MODE_EXACT, ANY>);
    if (mode == MODE_BRUTE) return f(rt_nearest_kernel<MODE_BRUTE, ANY>);
    return f(rt_nearest_kernel<MODE_TREE, ANY>);
}

}  // namespace

int distance_max_ctas_per_sm(uint32_t mode, bool any) {
    auto occ = [](auto kern) -> int { return query_ctas_per_sm(kern, 0); };
    return any ? dispatch_nearest<true>(mode, occ) : dispatch_nearest<false>(mode, occ);
}

cudaError_t launch_distance(const DistanceParams& q, uint32_t mode, bool any, int max_grid, cudaStream_t st) {
    auto go = [&](auto kern) { return query_launch(kern, 0, q, max_grid, st); };
    return any ? dispatch_nearest<true>(mode, go) : dispatch_nearest<false>(mode, go);
}

}  // namespace rtk
