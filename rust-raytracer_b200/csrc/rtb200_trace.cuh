// rtb200_trace.cuh — the three stages of the render path as device functions of the trace kernel (rtb200_wavefront.cu; a
// queue-driven kernel without CTA barriers was built on the same functions in round 2 and lost to instruction-cache misses -
// DESIGN.md §4.5, `git show 1f183f9:tools/experiments/rtb200_stream.cu.txt`):
//
//   closest_hit<MODE>   hit_world (raytracer.rs:44-59) for the 32 rays a warp holds: WARP-COOPERATIVE traversal of the
//                       8-wide BVH (node / leaf / exact steps over three per-warp work lists, one pair per lane), or the
//                       linear scans of the validation modes;
//   shade_slot<LIGHTS>  ray_color's body for one path vertex (raytracer.rs:71-165): Material::scatter of all five
//                       materials, the sky, the stochastic light test with its shadow-frame stack, and - when the path
//                       ends - the backwards unwinding of the albedo stack that reproduces the recursion's f32 products;
//   regenerate_slot     render_line's per-sample set-up (raytracer.rs:199-201) + Camera::get_ray (camera.rs:79-84) through
//                       primary_ray, or a caller-supplied primary ray (Q_RAYS).
//
// Ray state lives in shared memory, SoA over the slots of a CTA's pool (struct Pool).
#pragma once
#include "rtb200_kernels.cuh"

namespace rtk {

using namespace rtd;

#ifndef RT_SCATTER_TRIPS
// Rejection-loop trips (two trials each) of the unit-sphere sampler per shade stage; a scatter still unresolved after them
// carries over to the next iteration. On C2 on an H100, 2 trips beat 1 (16 % more iterations) and 3 (DESIGN.md §4.3).
#define RT_SCATTER_TRIPS 2
#endif
#ifndef RT_SMEM_STACK
// Albedo-stack levels kept in shared memory per slot; deeper levels live in global memory, and every bounce there costs a
// global store and, when the path is unwound, a dependent global load. On C2 on an H100 each step from 3 to 5, 8 and 12
// levels was faster (DESIGN.md §4.3), but 12 levels (67,152 B per CTA) need the 228 KiB shared-memory carveout for 3 CTAs
// per SM and leave 28 KiB of L1; 10 levels (65,104 B) fit the 196 KiB carveout and leave 60 KiB, which is faster (§4.5).
#define RT_SMEM_STACK 10
#endif

enum : uint32_t { CLS_MISS = 0, CLS_DIFFUSE = 1, CLS_METAL = 2, CLS_GLASS = 3, CLS_LIGHT = 4, CLS_DEAD = 5, N_CLS = 6 };
constexpr uint32_t kDeadLevel = 0xffffffffu;
// Pool.shd bit: the slot's scatter sample is still being drawn; its hit record (bt/bi) and path state are those of the
// vertex being shaded. The shadow depth in the low bits never exceeds max_shadow (<= 384), so the bit is free.
constexpr uint32_t kScatterPending = 0x80000000u;
using rtbvh::kLeafBit;
constexpr unsigned long long kNoHitBits = 0x7ff0000000000000ull;   // +inf as the "no root yet" key (roots are > t_min > 0)
constexpr uint32_t kNoSphere = 0xffffffffu;     // Pool.src: the ray does not start on a known sphere
// skip_pos / WarpCtx.skip: where the traversal leaves the certified source sphere out. kSkipNodeBit | node * 8 + child: the
// node step drops child `child` of `node` (a leaf holding only that sphere); else leaf * kLeafK + slot: the leaf step drops
// the slot. kNoSkip: nothing (kNoSkip / kLeafK and (kNoSkip & ~kSkipNodeBit) / 8 are no leaf's or node's index, < 2^27).
using rtbvh::kSkipNodeBit;
using rtbvh::kNoSkip;
constexpr uint32_t kSlotBytes = 7 * 8 + 10 * 4 + RT_SMEM_STACK * 4;   // shared memory per pool slot
constexpr uint32_t kFrameSlotBytes = 4;                               // + Pool.frm per slot in a multi-frame launch

// SoA ray pool of a CTA: n_slots slots.
struct Pool {
    double *ox, *oy, *oz, *dx, *dy, *dz, *bt;                    // ray origin / direction, best root (also updated as u64 bits)
    uint32_t *bi, *work, *pix, *smp, *blk, *clo, *chi, *lvl, *shd;   // hit index, work id, RNG (pixel, sample, block|has, cached draw), path level, shadow depth | kScatterPending
    uint32_t *src;                                               // the sphere the ray starts on (kNoSphere: a primary ray, or not known)
    uint32_t *stk;                                               // [RT_SMEM_STACK][n_slots] first levels of the albedo stack
    uint32_t *frm;                                               // multi-frame launches: the slot's frame (index into TraceParams::ftab), kFrameSlotBytes per slot
    uint32_t n_slots;
    uint32_t stack_col;                                          // this CTA's first column of the global per-slot arrays (stack / frames / lterm)
};
RT_DEV Pool pool_at(unsigned char* base, uint32_t n_slots, uint32_t stack_col) {
    Pool P;
    double* d = reinterpret_cast<double*>(base);
    P.ox = d; P.oy = d + n_slots; P.oz = d + 2 * n_slots; P.dx = d + 3 * n_slots; P.dy = d + 4 * n_slots; P.dz = d + 5 * n_slots; P.bt = d + 6 * n_slots;
    uint32_t* u = reinterpret_cast<uint32_t*>(d + 7 * n_slots);
    P.bi = u; P.work = u + n_slots; P.pix = u + 2 * n_slots; P.smp = u + 3 * n_slots; P.blk = u + 4 * n_slots; P.clo = u + 5 * n_slots;
    P.chi = u + 6 * n_slots; P.lvl = u + 7 * n_slots; P.shd = u + 8 * n_slots; P.src = u + 9 * n_slots; P.stk = u + 10 * n_slots;
    P.frm = u + (10 + RT_SMEM_STACK) * n_slots;   // only multi-frame launches reserve it (and touch it)
    P.n_slots = n_slots; P.stack_col = stack_col;
    return P;
}

// per-warp scratch of the closest-hit stage
struct WarpCtx {
    float4 *cA, *cB, *cC;          // [32] per-ray f32 constants: {o.xyz, slab margin}, {1/d^.xyz, thr}, {d^.xyz, -o.d^}
    uint32_t *skip;                // [32] per ray: skip_pos of the certified source sphere, or kNoSkip
    uint32_t *l_in, *l_lf, *l_cd;  // work lists: (ray, node), (ray, leaf), (ray, sphere); entries id << 5 | ray
};
// Rounded up to 16 B: the contexts of a CTA's warps lie back to back, and each one's float4 constants (then the pool's
// doubles after the last one) must stay aligned whatever the list capacities add up to.
constexpr uint32_t kWarpCtxBytes = (3 * 32 * 16 + 32 * 4 + (uint32_t)(kCapIn + kCapLf + kCapCd) * 4 + 15u) & ~15u;
RT_DEV WarpCtx warpctx_at(unsigned char* base) {
    WarpCtx W;
    W.cA = reinterpret_cast<float4*>(base); W.cB = W.cA + 32; W.cC = W.cB + 32;
    W.skip = reinterpret_cast<uint32_t*>(W.cC + 32);
    W.l_in = W.skip + 32; W.l_lf = W.l_in + kCapIn; W.l_cd = W.l_lf + kCapLf;
    return W;
}

struct SceneRefs {
    const float4* nodes; const float4* leaf_rec; const uint32_t* leaf_id; const float4* filt;
    const double4* geo; const DevMat* mat;
};

struct Stats {   // per thread and launch: far below 2^32
    uint32_t rays = 0, cand = 0, ovf = 0, samples = 0, leaves = 0, nodes = 0;
#if RT_PHASE_CLOCKS
    unsigned long long t_node = 0, t_leaf = 0, t_exact = 0;   // lane 0: clock64() cycles of the warp's node / leaf / exact steps
    uint32_t exact_steps = 0, exact_tests = 0, src_skips = 0;
#endif
};

RT_DEV void bulk_stage(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    const uint32_t CH = 32768u;
    for (uint32_t o = 0; o < bytes; o += CH) {
        uint32_t nb = bytes - o < CH ? bytes - o : CH;
        tma_bulk_g2s((char*)dst + o, (const char*)src + o, nb, bar);
    }
}

RT_DEV void albedo_of(uint32_t code, const DevMat* mat, float& r, float& g, float& b) {
    if (code == 0xffffffffu) { r = g = b = 1.0f; return; }   // Light: Srgb(1,1,1) (materials.rs:67)
    if (code & 0x80000000u) {   // packed texel (materials.rs:248-252: pixel as f32 / 255.0)
        r = __fdiv_rn((float)(code & 0xffu), 255.0f);
        g = __fdiv_rn((float)((code >> 8) & 0xffu), 255.0f);
        b = __fdiv_rn((float)((code >> 16) & 0xffu), 255.0f);
    } else {
        const DevMat& m = mat[code];
        r = m.r; g = m.g; b = m.b;
    }
}

// sm_90 has only two-operand min / max; like the three-operand form, a NaN operand is dropped
RT_DEV float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
RT_DEV float fmin3(float a, float b, float c) { return fminf(fminf(a, b), c); }

// inclusive warp prefix sum (of a packed pair of 16-bit counters)
RT_DEV uint32_t warp_scan_incl(uint32_t v, int lane) {
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, v, off);
        if (lane >= off) v += t;
    }
    return v;
}

// FMA on both lanes of a float2, each lane rounded once like fmaf. sm_90 has no packed FP32 FMA: this issues two FFMA.
RT_DEV float2 fma2_rn(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

// the 7-FMA conservative sphere test on NP pair-packed records: D = (c.d^ - o.d^)^2 + 2 c.o + nk   (candidate iff D >= thr)
#define RT_FILTER_PAIRS(REC, DV, NP)                                                                                                  \
    _Pragma("unroll") for (int q = 0; q < (NP); ++q) {                                                                              \
        float4 A_ = (REC)[2 * q], B_ = (REC)[2 * q + 1];                                                                             \
        float2 cx = make_float2(A_.x, A_.y), cy = make_float2(A_.z, A_.w), cz = make_float2(B_.x, B_.y), nk = make_float2(B_.z, B_.w); \
        float2 bb = fma2_rn(cz, dz2, nod2);                                                                                          \
        float2 tt = fma2_rn(cz, oz2, nk);                                                                                            \
        bb = fma2_rn(cy, dy2, bb);                                                                                                   \
        tt = fma2_rn(cy, oy2, tt);                                                                                                   \
        bb = fma2_rn(cx, dx2, bb);                                                                                                   \
        tt = fma2_rn(cx, ox2, tt);                                                                                                   \
        (DV)[q] = fma2_rn(bb, bb, tt);                                                                                               \
    }

RT_DEV uint32_t class_of(uint32_t kind) {
    return (kind == RT_METAL) ? CLS_METAL : (kind == RT_GLASS) ? CLS_GLASS : (kind == RT_LIGHT) ? CLS_LIGHT : CLS_DIFFUSE;
}

// =====================================================================================================================
// closest-hit. Every lane of the warp calls it; lane l owns the ray in pool slot `slot` when `alive`. On return
// P.bt[slot] / P.bi[slot] hold hit_world's result (bi = 0xffffffff: miss) and the lane's class is returned.
// hit_world (raytracer.rs:44-59) keeps the closest root and, on equal t, the first sphere in list order; because
// Sphere::hit(t_max) accepts exactly r < t_max with r the first root beyond t_min, that fold equals the lexicographic
// minimum of (r, index) over all spheres - so spheres may be tested in any order, by any lane.
//
// ANY (occlusion queries, DESIGN.md §4.11): the same traversal asks only whether some sphere accepts a root below the ray's
// bound t_hi (0.001 < t_hi <= f64::MAX). On return P.bi[slot] is one such sphere (which one depends on the order of the
// steps), or 0xffffffff; P.bt is not meaningful. The node step also drops children that lie wholly beyond the ray's f32
// bound tcap[lane] (written here), the first acceptance marks the ray done, entries of done rays are popped without work,
// and the warp leaves the traversal once every ray in it is done. The thread-private loops stop at their first acceptance.
// =====================================================================================================================
template <uint32_t MODE, bool ANY = false>
RT_DEV uint32_t closest_hit(const TraceParams& p, const SceneRefs& sc, const Pool& P, const WarpCtx& W, bool alive, uint32_t slot, int lane, Stats& st,
                            double t_hi = DBL_MAX, float* tcap = nullptr) {
    const unsigned FULL = 0xffffffffu;
    uint32_t cls = CLS_DEAD;
    if (__ballot_sync(FULL, alive) == 0u) return cls;   // a warp without rays skips the stage (frame tail)
    const uint32_t lt_mask = (1u << lane) - 1u;
    unsigned long long* btu = reinterpret_cast<unsigned long long*>(P.bt);
    const D3 o = mk(P.ox[slot], P.oy[slot], P.oz[slot]), d = mk(P.dx[slot], P.dy[slot], P.dz[slot]);
    const double a = length_squared(d);
    const double thi = ANY ? t_hi : DBL_MAX;   // the bound of every exact test
    bool ovf = false;
    uint32_t done = 0u;   // ANY: the rays (by owning lane) with a proven hit below their bound; warp-uniform
    // thread-private exact f64 confirmation (fallback paths: every sphere / the always-list / MODE_BRUTE candidates)
    double best_t = DBL_MAX;
    int best = -1;
    auto confirm = [&](int j) {
        if constexpr (ANY) { if (best >= 0) return; }   // one acceptance answers the ray
        double4 gq = sc.geo[j];
        double root;
        if (sphere_root(mk(gq.x, gq.y, gq.z), gq.w, o, d, a, 0.001, thi, root)) {
            if (best < 0 || root < best_t || (root == best_t && j < best)) { best_t = root; best = j; }
        }
        ++st.cand;
    };
    if (alive) { btu[slot] = kNoHitBits; P.bi[slot] = 0xffffffffu; }
    if (MODE != MODE_EXACT) {
        // per-ray constants in the recentred f32 frame (DESIGN.md "soundness of the conservative tests")
        const float ofx = __double2float_rn(__dsub_rn(o.x, p.gx)), ofy = __double2float_rn(__dsub_rn(o.y, p.gy)),
                    ofz = __double2float_rn(__dsub_rn(o.z, p.gz));
        const float dfx = __double2float_rn(d.x), dfy = __double2float_rn(d.y), dfz = __double2float_rn(d.z);
        const float s = fmaf(dfx, dfx, fmaf(dfy, dfy, dfz * dfz));
        const float oo = fmaf(ofx, ofx, fmaf(ofy, ofy, ofz * ofz));
        const bool ok = (s > 1e-30f) && (s < 1e30f) && (oo < 1e30f);
        const float inv = rsqrtf(s);
        const float dnx = dfx * inv, dny = dfy * inv, dnz = dfz * inv;
        const float nod = -fmaf(ofx, dnx, fmaf(ofy, dny, ofz * dnz));
        const float thr = __fmul_rd(oo, p.er_coef);
        if (alive && !ok) ovf = true;
        if (MODE == MODE_TREE) {
            // slab constants: 1/d^ with |d^| clamped away from zero (keeps every product finite), margin 32u|o| rounded up
            const float ax = fabsf(dnx) < 1e-20f ? copysignf(1e-20f, dnx) : dnx;
            const float ay = fabsf(dny) < 1e-20f ? copysignf(1e-20f, dny) : dny;
            const float az = fabsf(dnz) < 1e-20f ? copysignf(1e-20f, dnz) : dnz;
            const float mray = __fmul_ru(1.9073486328125e-6f, __fsqrt_ru(oo));
            W.cA[lane] = make_float4(ofx, ofy, ofz, mray);
            W.cB[lane] = make_float4(__frcp_rn(ax), __frcp_rn(ay), __frcp_rn(az), thr);
            W.cC[lane] = make_float4(dnx, dny, dnz, nod);
            // ANY: the bound on the distance along d^, T~ >= t_hi * |d| (DESIGN.md §4.11): the f64 product rounded up, a 2^-40
            // margin for the rounding of a = |d|^2, then rounded up to f32 (+inf when it exceeds the f32 range: no pruning)
            if constexpr (ANY) tcap[lane] = __double2float_ru(__dmul_ru(__dmul_ru(t_hi, __dsqrt_ru(a)), 1.0 + 0x1p-40));
            // The sphere the ray starts on is left out of its candidates when a cheap f64 certificate proves that the exact
            // test rejects it (a ray leaving the surface outwards; DESIGN.md §4.2). The certificate is evaluated on this ray's
            // own o and d, so even a wrong Pool.src could only cost a missed skip, never a wrong hit.
            uint32_t skp = kNoSkip;
            const uint32_t src = alive ? P.src[slot] : kNoSphere;
            if (src != kNoSphere) {
                const uint32_t pos = p.skip_pos[src];
                const double4 gs = sc.geo[src];
                if (pos != kNoSkip && leaves_sphere(mk(gs.x, gs.y, gs.z), gs.w, o, d, a)) skp = pos;
            }
            W.skip[lane] = skp;
            // LIFO reserve: single-entry descents grow the node stack by at most 7 per level, so multi-entry steps may fill it
            // only up to fat_in; above that the stack is popped one entry at a time and can never overflow (DESIGN.md §4.1).
            const uint32_t fat_in = (uint32_t)kCapIn - 7u * p.depth - 8u;
            // ---- warp-cooperative traversal ----
            const bool enter = alive && ok && p.n_nodes != 0u;
            const unsigned em = __ballot_sync(FULL, enter);
            uint32_t n_in = (uint32_t)__popc(em), n_lf = 0u, n_cd = 0u;
            if (enter) W.l_in[__popc(em & lt_mask)] = (uint32_t)lane;   // (root node 0) << 5 | ray
            __syncwarp();
            uint32_t guard = 0;
            for (;;) {
#if RT_PHASE_CLOCKS
                const unsigned long long t_step = clock64();
#endif
                if (n_in != 0u && n_lf <= (uint32_t)(kCapLf - 64)) {
                    // ---------------- node step: lane <-> one (ray, node) pair from the top of the stack ----------------
                    const uint32_t m = n_in < 32u ? n_in : 32u;
                    const bool act = (uint32_t)lane < m;
                    const uint32_t e = act ? W.l_in[n_in - 1u - (uint32_t)lane] : 0u;
                    const uint32_t ray = e & 31u, node = e >> 5;
                    uint32_t hit = 0u, leafbits = 0u;
                    const float4* N = sc.nodes + (size_t)node * kNodeVec;
                    bool test = act;   // ANY: a done ray's entry is popped without a test
                    if constexpr (ANY) test = act && !((done >> ray) & 1u);
                    if (test) {
                        const float4 A = W.cA[ray], B = W.cB[ray];
                        float tcr = 0.f;
                        if constexpr (ANY) tcr = tcap[ray];
                        auto far_ = [&](float f) { if constexpr (ANY) return fminf(f, tcr); else return f; };   // ANY: min(t_far, T~)
                        // near/far plane of each axis by the sign of d^; planes shifted outwards by the per-ray margin
                        const uint32_t sx = __float_as_uint(B.x) >> 31, sy = __float_as_uint(B.y) >> 31, sz = __float_as_uint(B.z) >> 31;
                        const float mx = copysignf(A.w, B.x), my = copysignf(A.w, B.y), mz = copysignf(A.w, B.z);
                        const float cnx = __fmul_rn(__fadd_rn(A.x, mx), -B.x), cfx = __fmul_rn(__fsub_rn(A.x, mx), -B.x);
                        const float cny = __fmul_rn(__fadd_rn(A.y, my), -B.y), cfy = __fmul_rn(__fsub_rn(A.y, my), -B.y);
                        const float cnz = __fmul_rn(__fadd_rn(A.z, mz), -B.z), cfz = __fmul_rn(__fsub_rn(A.z, mz), -B.z);
                        const float2 ix2 = make_float2(B.x, B.x), iy2 = make_float2(B.y, B.y), iz2 = make_float2(B.z, B.z);
                        const float2 cnx2 = make_float2(cnx, cnx), cny2 = make_float2(cny, cny), cnz2 = make_float2(cnz, cnz);
                        const float2 cfx2 = make_float2(cfx, cfx), cfy2 = make_float2(cfy, cfy), cfz2 = make_float2(cfz, cfz);
                        const float4* Nnx = N + (sx ? 6 : 0); const float4* Nfx = N + (sx ? 0 : 6);
                        const float4* Nny = N + (sy ? 8 : 2); const float4* Nfy = N + (sy ? 2 : 8);
                        const float4* Nnz = N + (sz ? 10 : 4); const float4* Nfz = N + (sz ? 4 : 10);
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const float4 NX = Nnx[h], NY = Nny[h], NZ = Nnz[h], FX = Nfx[h], FY = Nfy[h], FZ = Nfz[h];
                            const float2 tnx0 = fma2_rn(make_float2(NX.x, NX.y), ix2, cnx2), tnx1 = fma2_rn(make_float2(NX.z, NX.w), ix2, cnx2);
                            const float2 tny0 = fma2_rn(make_float2(NY.x, NY.y), iy2, cny2), tny1 = fma2_rn(make_float2(NY.z, NY.w), iy2, cny2);
                            const float2 tnz0 = fma2_rn(make_float2(NZ.x, NZ.y), iz2, cnz2), tnz1 = fma2_rn(make_float2(NZ.z, NZ.w), iz2, cnz2);
                            const float2 tfx0 = fma2_rn(make_float2(FX.x, FX.y), ix2, cfx2), tfx1 = fma2_rn(make_float2(FX.z, FX.w), ix2, cfx2);
                            const float2 tfy0 = fma2_rn(make_float2(FY.x, FY.y), iy2, cfy2), tfy1 = fma2_rn(make_float2(FY.z, FY.w), iy2, cfy2);
                            const float2 tfz0 = fma2_rn(make_float2(FZ.x, FZ.y), iz2, cfz2), tfz1 = fma2_rn(make_float2(FZ.z, FZ.w), iz2, cfz2);
                            // hit iff max(t_near, 0) <= t_far
                            hit |= (fmaxf(fmax3(tnx0.x, tny0.x, tnz0.x), 0.f) <= far_(fmin3(tfx0.x, tfy0.x, tfz0.x)) ? 1u : 0u) << (4 * h + 0);
                            hit |= (fmaxf(fmax3(tnx0.y, tny0.y, tnz0.y), 0.f) <= far_(fmin3(tfx0.y, tfy0.y, tfz0.y)) ? 1u : 0u) << (4 * h + 1);
                            hit |= (fmaxf(fmax3(tnx1.x, tny1.x, tnz1.x), 0.f) <= far_(fmin3(tfx1.x, tfy1.x, tfz1.x)) ? 1u : 0u) << (4 * h + 2);
                            hit |= (fmaxf(fmax3(tnx1.y, tny1.y, tnz1.y), 0.f) <= far_(fmin3(tfx1.y, tfy1.y, tfz1.y)) ? 1u : 0u) << (4 * h + 3);
                        }
                        const uint4 R0 = *reinterpret_cast<const uint4*>(N + kChildVec), R1 = *reinterpret_cast<const uint4*>(N + kChildVec + 1);
                        leafbits = (R0.x >> 31) | ((R0.y >> 31) << 1) | ((R0.z >> 31) << 2) | ((R0.w >> 31) << 3) |
                                   ((R1.x >> 31) << 4) | ((R1.y >> 31) << 5) | ((R1.z >> 31) << 6) | ((R1.w >> 31) << 7);
                    }
                    {   // a leaf that holds nothing but the certified source sphere is not visited at all
                        const uint32_t sk = W.skip[ray] ^ (kSkipNodeBit | node << 3);   // < 8: the child to drop
                        if (sk < 8u) {
#if RT_PHASE_CLOCKS
                            st.src_skips += (hit >> sk) & 1u;
#endif
                            hit &= ~(1u << sk);
                        }
                    }
                    const uint32_t packed = (uint32_t)__popc(hit & ~leafbits) | ((uint32_t)__popc(hit & leafbits) << 16);
                    const uint32_t inc = warp_scan_incl(packed, lane);
                    // commit the longest prefix of lanes (top of the stack first) whose pushes fit
                    const uint32_t new_in = n_in - ((uint32_t)lane + 1u) + (inc & 0xffffu);
                    const bool fits = new_in <= (lane == 0 ? (uint32_t)kCapIn : fat_in) && n_lf + (inc >> 16) <= (uint32_t)kCapLf;
                    const unsigned okm = __ballot_sync(FULL, fits || !act);
                    uint32_t k = okm == FULL ? 32u : (uint32_t)(__ffs(~okm) - 1);
                    k = k < m ? k : m;
                    if (k == 0u) { if (lane == 0) atomicAdd(&p.err[1], 1ull); break; }   // cannot happen (reserve argument); never spin
                    const uint32_t tot = __shfl_sync(FULL, inc, (int)k - 1);
                    __syncwarp();   // every lane has read its entry before the stack is overwritten
                    if (act && (uint32_t)lane < k) {
                        const uint32_t exc = inc - packed;
                        uint32_t pi = (n_in - k) + (exc & 0xffffu), pl = n_lf + (exc >> 16);
                        const uint32_t* refs = reinterpret_cast<const uint32_t*>(N + kChildVec);
                        uint32_t mm = hit;
                        while (mm) {
                            const int c = __ffs(mm) - 1;
                            mm &= mm - 1u;
                            const uint32_t ref = refs[c];
                            if (ref & kLeafBit) W.l_lf[pl++] = (ref << 5) | ray;   // the shift drops the leaf bit
                            else W.l_in[pi++] = (ref << 5) | ray;
                        }
                        if constexpr (ANY) st.nodes += test ? 1u : 0u; else ++st.nodes;
                    }
                    n_in = n_in - k + (tot & 0xffffu);
                    n_lf += tot >> 16;
                    __syncwarp();
#if RT_PHASE_CLOCKS
                    if (lane == 0) st.t_node += clock64() - t_step;
#endif
                } else if (n_lf != 0u && n_cd <= (uint32_t)(kCapCd - 32)) {
                    // ---------------- leaf step: lane <-> one (ray, leaf) pair: conservative sphere test on its spheres ----------------
                    const uint32_t m = n_lf < 32u ? n_lf : 32u;
                    const bool act = (uint32_t)lane < m;
                    const uint32_t e = act ? W.l_lf[n_lf - 1u - (uint32_t)lane] : 0u;
                    const uint32_t ray = e & 31u, leaf = e >> 5;
                    uint32_t hit = 0u;
                    bool test = act;   // ANY: a done ray's entry is popped without a test
                    if constexpr (ANY) test = act && !((done >> ray) & 1u);
                    if (test) {
                        const float4 A = W.cA[ray], C = W.cC[ray];
                        const float th = W.cB[ray].w;
                        const float2 dx2 = make_float2(C.x, C.x), dy2 = make_float2(C.y, C.y), dz2 = make_float2(C.z, C.z);
                        const float2 ox2 = make_float2(2.f * A.x, 2.f * A.x), oy2 = make_float2(2.f * A.y, 2.f * A.y), oz2 = make_float2(2.f * A.z, 2.f * A.z);
                        const float2 nod2 = make_float2(C.w, C.w);
                        float2 Dv[kLeafK / 2];
                        const float4* rec = sc.leaf_rec + (size_t)leaf * kLeafK;
                        RT_FILTER_PAIRS(rec, Dv, kLeafK / 2)
#pragma unroll
                        for (int q = 0; q < kLeafK / 2; ++q) hit |= (Dv[q].x >= th ? 1u : 0u) << (2 * q) | (Dv[q].y >= th ? 1u : 0u) << (2 * q + 1);
                        // the sphere the ray starts on, when its certificate proved that the exact test rejects it
                        const uint32_t sk = W.skip[ray];
                        if (sk / (uint32_t)kLeafK == leaf) {
#if RT_PHASE_CLOCKS
                            st.src_skips += (hit >> (sk % (uint32_t)kLeafK)) & 1u;
#endif
                            hit &= ~(1u << (sk % (uint32_t)kLeafK));
                        }
                    }
                    const uint32_t cntc = (uint32_t)__popc(hit);
                    const uint32_t inc = warp_scan_incl(cntc, lane);
                    const bool fits = n_cd + inc <= (uint32_t)kCapCd;
                    const unsigned okm = __ballot_sync(FULL, fits || !act);
                    uint32_t k = okm == FULL ? 32u : (uint32_t)(__ffs(~okm) - 1);
                    k = k < m ? k : m;
                    if (k == 0u) { if (lane == 0) atomicAdd(&p.err[1], 1ull); break; }
                    const uint32_t tot = __shfl_sync(FULL, inc, (int)k - 1);
                    if (act && (uint32_t)lane < k) {
                        uint32_t pc = n_cd + inc - cntc;
                        const uint32_t* ids = sc.leaf_id + (size_t)leaf * kLeafK;
                        uint32_t mm = hit;
                        while (mm) {
                            const int c = __ffs(mm) - 1;
                            mm &= mm - 1u;
                            W.l_cd[pc++] = (ids[c] << 5) | ray;
                        }
                        if constexpr (ANY) st.leaves += test ? 1u : 0u; else ++st.leaves;
                    }
                    n_lf -= k;
                    n_cd += tot;
                    __syncwarp();
#if RT_PHASE_CLOCKS
                    if (lane == 0) st.t_leaf += clock64() - t_step;
#endif
                } else if (n_cd != 0u) {
                    // ---------------- exact step: lane <-> one (ray, sphere) candidate, reference-exact f64 Sphere::hit ----------------
                    const uint32_t m = n_cd < 32u ? n_cd : 32u;
                    const bool act = (uint32_t)lane < m;
                    const uint32_t e = act ? W.l_cd[n_cd - 1u - (uint32_t)lane] : 0u;
                    const uint32_t rs = __shfl_sync(FULL, slot, (int)(e & 31u)), sph = e >> 5;   // pool slot of the candidate's ray
                    if constexpr (ANY) {
                        // Sphere::hit under the ray's own bound; one acceptance answers the ray, in whatever order it comes
                        const uint32_t ray = e & 31u;
                        const double tr = __shfl_sync(FULL, t_hi, (int)ray);
                        bool acc = false;
                        if (act && !((done >> ray) & 1u)) {
                            const D3 ro = mk(P.ox[rs], P.oy[rs], P.oz[rs]), rd = mk(P.dx[rs], P.dy[rs], P.dz[rs]);
                            const double4 gq = sc.geo[sph];
                            double root;
                            acc = sphere_root(mk(gq.x, gq.y, gq.z), gq.w, ro, rd, length_squared(rd), 0.001, tr, root);
                            ++st.cand;
#if RT_PHASE_CLOCKS
                            ++st.exact_tests;
#endif
                        }
                        if (acc) P.bi[rs] = sph;   // lanes of one ray may race here: any of their spheres will do
                        done |= __reduce_or_sync(FULL, acc ? 1u << ray : 0u);
                        n_cd -= m;
                        __syncwarp();
                        if ((em & ~done) == 0u) break;   // every ray of the warp is answered
                    } else {
                        unsigned long long key = ~0ull;
                        if (act) {
                            const D3 ro = mk(P.ox[rs], P.oy[rs], P.oz[rs]), rd = mk(P.dx[rs], P.dy[rs], P.dz[rs]);
                            const double4 gq = sc.geo[sph];
                            double root;
                            if (sphere_root(mk(gq.x, gq.y, gq.z), gq.w, ro, rd, length_squared(rd), 0.001, DBL_MAX, root)) key = (unsigned long long)__double_as_longlong(root);
                            ++st.cand;
#if RT_PHASE_CLOCKS
                            ++st.exact_tests;
#endif
                        }
                        // per-ray lexicographic minimum of (root, sphere index): roots are positive, so their bit patterns order like the values
                        const bool h = key != ~0ull;
                        const unsigned long long before = h ? btu[rs] : 0ull;
                        __syncwarp();
                        if (h && key < before) atomicMin(&btu[rs], key);
                        __syncwarp();
                        const bool mine = h && key == btu[rs];
                        if (mine && key < before) atomicMax(&P.bi[rs], 0xffffffffu);   // the root got smaller in this step: forget the old index
                        __syncwarp();
                        if (mine) atomicMin(&P.bi[rs], sph);
                        n_cd -= m;
                        __syncwarp();
                    }
#if RT_PHASE_CLOCKS
                    if (lane == 0) { st.t_exact += clock64() - t_step; ++st.exact_steps; }
#endif
                } else {
                    break;
                }
                if (++guard > (1u << 22)) { if (lane == 0) atomicAdd(&p.err[1], 1ull); break; }
            }
        } else {   // MODE_BRUTE: hit_world's linear scan with the conservative sphere test in front of the exact one
            if (alive && ok) {
                const float2 dx2 = make_float2(dnx, dnx), dy2 = make_float2(dny, dny), dz2 = make_float2(dnz, dnz);
                const float2 ox2 = make_float2(2.f * ofx, 2.f * ofx), oy2 = make_float2(2.f * ofy, 2.f * ofy), oz2 = make_float2(2.f * ofz, 2.f * ofz);
                const float2 nod2 = make_float2(nod, nod);
#pragma unroll 1
                for (uint32_t pp = 0; pp < p.n_pairs; pp += 4) {
                    float2 Dv[4];
                    const float4* rec = sc.filt + 2 * pp;
                    RT_FILTER_PAIRS(rec, Dv, 4)
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const uint32_t j = 2u * (pp + (uint32_t)q);
                        if (Dv[q].x >= thr && j < p.n) confirm((int)j);
                        if (Dv[q].y >= thr && j + 1u < p.n) confirm((int)j + 1);
                    }
                    if constexpr (ANY) { if (best >= 0) break; }
                }
            }
        }
    } else {
        ovf = alive;
    }
    if (alive) {
        if constexpr (ANY) { if ((done >> lane) & 1u) best = (int)P.bi[slot]; }   // answered by the traversal
        if (ovf) {   // MODE_EXACT, or a ray outside the f32 frame's safe range: every sphere in f64
            ++st.ovf;
            for (int k = 0; k < (int)p.n; ++k) {
                confirm(k);
                if constexpr (ANY) { if (best >= 0) break; }
            }
        } else if (MODE == MODE_TREE) {
            for (uint32_t k = 0; k < p.n_always; ++k) {
                if constexpr (ANY) { if (best >= 0) break; }
                confirm((int)p.always[k]);
            }
        }
        if constexpr (ANY) {
            if (best >= 0) P.bi[slot] = (uint32_t)best;
            ++st.rays;
            return CLS_MISS;   // the caller reads P.bi
        }
        // merge the thread-private result with the traversal's (this slot is only touched by its own thread now)
        const unsigned long long tb = btu[slot];
        const uint32_t ti = P.bi[slot];
        if (best >= 0) {
            const unsigned long long kb = (unsigned long long)__double_as_longlong(best_t);
            if (ti == 0xffffffffu || kb < tb || (kb == tb && (uint32_t)best < ti)) { P.bt[slot] = best_t; P.bi[slot] = (uint32_t)best; }
        }
        const uint32_t fin = P.bi[slot];
        cls = CLS_MISS;
        if (fin != 0xffffffffu) cls = class_of(sc.mat[fin].kind);
        ++st.rays;
    }
    return cls;
}

// =====================================================================================================================
// The render's primary ray of local pixel (x, y_local) of the launch's rows and sample s0 + s_local, under camera `cam` and the
// Philox key (k0, k1): the pixel's image row (row band y_local / band_rows is the shard's, raytracer.rs:254-262), the two
// jitter draws of raytracer.rs:199-200 from the stream of (pixel, sample), then Camera::get_ray (camera.rs:79-84), moved onto
// the lens `lens` when LENS and its radius is not 0 (lens_apply, whose draws are a domain of their own, DESIGN.md §4.17). `rng`
// is left after the two draws. The trace kernel (regenerate_slot) and the auxiliary buffers (rtb200_aov.cu) both make their
// camera rays here. The lens is a compile-time choice of the launch: a pinhole launch (LENS false) carries no lens code, so the
// kernels of pinhole renders are the ones they were before the lens existed.
// =====================================================================================================================
template <bool LENS = false>
RT_DEV void primary_ray(const TraceParams& p, const rt_camera& cam, const rt_lens& lens, uint32_t k0, uint32_t k1, uint32_t x,
                        uint32_t y_local, uint32_t s0, uint32_t s_local, Rng& rng, D3& o, D3& d) {
    const uint32_t band_rows = p.band_rows, width = p.width, height = p.height;
    uint32_t band = y_local / band_rows;
    uint32_t y = (band * (uint32_t)p.world + (uint32_t)p.rank) * band_rows + (y_local - band * band_rows);
    rng_init(rng, y * width + x, s0 + s_local);
    double xi1 = rng_f64(rng, k0, k1);
    double u = __ddiv_rn(__dadd_rn((double)x, xi1), __dsub_rn((double)width, 1.0));
    double xi2 = rng_f64(rng, k0, k1);
    double v = __ddiv_rn(__dsub_rn((double)height, __dadd_rn((double)y, xi2)), __dsub_rn((double)height, 1.0));
    get_ray(cam, u, v, o, d);
    if constexpr (LENS) {
        if (lens.radius != 0.0) lens_apply(lens, rng.pixel, rng.sample, k0, k1, o, d);
    }
}

// =====================================================================================================================
// Regenerate pool slot `s` from the global (pixel,sample) queue. Warp-synchronous: every lane of the warp calls it,
// `want` says whether this lane's slot needs a new path; `exhausted` is the warp's (uniform) knowledge that the queue is
// dry. Returns true when the slot received a new primary ray. raytracer.rs:199-201 + camera.rs:79-84.
// FRAMES: the queue spans several frames, frame outermost; the frame's camera and key come from p.ftab (read once per
// sample, off the bounce loop) and the frame is kept in Pool.frm for the shade stage's draws.
// Q_LIST: the queue spans samples [s0, s0 + s_count) of the n_list pixels p.list[0, n_list) (an adaptive round, DESIGN.md
// §4.9); n_list is read from p.list_n once per launch by the caller.
// Q_RAYS: the queue spans samples [s0, s0 + s_count) of the n = p.npix_local caller-supplied rays p.ray_o / p.ray_d (DESIGN.md
// §4.12); the slot gets the ray itself instead of a camera ray.
// LENS (FRAMES or Q_LIST only): the camera rays go through the lens, a frame's from p.ltab, an adaptive round's p.lens.
// =====================================================================================================================
template <bool LIGHTS, uint32_t QUEUE, bool LENS = false>
RT_DEV bool regenerate_slot(const TraceParams& p, const Pool& P, bool want, uint32_t s, int lane, bool& exhausted, Stats& st,
                            uint32_t n_list = 0u) {
    constexpr bool FRAMES = QUEUE == Q_FRAMES;
    const unsigned FULL = 0xffffffffu;
    want = want && !exhausted;
    unsigned need = __ballot_sync(FULL, want);
    if (!need) return false;
    int leader = __ffs(need) - 1;
    unsigned base = 0;
    if (lane == leader) base = atomicAdd(p.work_counter, (unsigned)__popc(need));
    base = __shfl_sync(FULL, base, leader);
    if (base + (unsigned)__popc(need) >= (QUEUE == Q_LIST ? n_list * p.s_count : p.total_work)) exhausted = true;
    if (!want) return false;
    unsigned my = base + __popc(need & ((1u << lane) - 1u));
    if (my >= (QUEUE == Q_LIST ? n_list * p.s_count : p.total_work)) return false;
    uint32_t f = 0u, k0 = p.key0, k1 = p.key1;
    uint32_t x, s_local, y_local, lp, k_list = 0u;
    Rng rng;
    D3 o, d;
    if constexpr (QUEUE == Q_RAYS) {
        // Ray index innermost: neighbouring lanes take neighbouring, usually coherent, rays, and every sample of the launch
        // re-reads its ray. Ray i's sample s0 + j draws from the stream of the render's (pixel stream0 + i, sample s0 + j)
        // past the two jitter draws of raytracer.rs:199-200, which are the two u64 of the stream's first Philox block.
        const uint32_t i = my % p.npix_local;
        rng_init(rng, p.stream0 + i, p.s0 + my / p.npix_local);
        rng.blk = 1u;
        const double* ro = p.ray_o + 3 * (size_t)i;
        const double* rd = p.ray_d + 3 * (size_t)i;
        o = mk(ro[0], ro[1], ro[2]);
        d = mk(rd[0], rd[1], rd[2]);
    } else {
        if constexpr (FRAMES) { f = my / p.frame_work; my -= f * p.frame_work; k0 = p.ftab[f].key0; k1 = p.ftab[f].key1; }
        // Order of the global queue: image rows from the BOTTOM up, all samples of a row before the next row, x innermost.
        // The long paths of these scenes start at the ground / the spheres; the rows handed out last are the top of the image -
        // sky, one ray per sample - so that the stragglers of the last expensive rows finish under the cover of cheap work
        // instead of holding nearly empty CTAs for ~50 iterations after the queue ran dry (DESIGN.md §5: 0.5 ms per launch).
        // The (pixel, sample) -> RNG stream and the samplebuf index do not depend on the order.
        // Q_LIST: the list is in increasing pixel order and is handed out from its end, so bottom rows go first here too; the
        // samples of one pixel are consecutive work ids.
        if constexpr (QUEUE == Q_LIST) {
            s_local = my % p.s_count;
            k_list = n_list - 1u - my / p.s_count;
            lp = p.list[k_list];
            y_local = lp / p.width;
            x = lp - y_local * p.width;
        } else {
            x = my % p.width;
            const uint32_t t_ = my / p.width;
            s_local = t_ % p.s_count;
            const uint32_t rr = t_ / p.s_count;
            y_local = p.rows_local - 1u - rr;
            lp = y_local * p.width + x;
        }
        if constexpr (FRAMES) primary_ray<LENS>(p, p.ftab[f].cam, LENS ? p.ltab[f] : p.lens, k0, k1, x, y_local, p.s0, s_local, rng, o, d);
        else primary_ray<LENS>(p, p.cam, p.lens, k0, k1, x, y_local, p.s0, s_local, rng, o, d);
    }
    P.ox[s] = o.x; P.oy[s] = o.y; P.oz[s] = o.z; P.dx[s] = d.x; P.dy[s] = d.y; P.dz[s] = d.z;
    // samplebuf index [sample][pixel], [frame][sample][pixel], [sample][list position] (Q_LIST) or [sample][ray] (Q_RAYS)
    if constexpr (FRAMES) { P.work[s] = (f * p.s_count + s_local) * p.npix_local + lp; P.frm[s] = f; }
    else if constexpr (QUEUE == Q_LIST) P.work[s] = s_local * n_list + k_list;
    else if constexpr (QUEUE == Q_RAYS) P.work[s] = my;
    else P.work[s] = s_local * p.npix_local + lp;
    P.pix[s] = rng.pixel; P.smp[s] = rng.sample;
    P.blk[s] = (rng.blk << 1) | rng.has; P.clo[s] = rng.c_lo; P.chi[s] = rng.c_hi;
    P.lvl[s] = 0u;
    P.shd[s] = 0u;
    P.src[s] = kNoSphere;
    if (LIGHTS) {
        for (int q = 0; q < 6; ++q) p.lterm[(size_t)q * p.stack_stride + P.stack_col + s] = 0.0f;
    }
    ++st.samples;
    return true;
}

// =====================================================================================================================
// One path vertex of slot `s` whose closest-hit result is in the pool; c = the ray's class. Writes the continuation ray
// (or a shadow ray) back to the pool, or - when the sample is finished - its radiance to samplebuf and marks the slot
// dead (returns true). A diffuse or metal vertex whose scatter sample is not accepted within RT_SCATTER_TRIPS trips of
// the rejection loop saves only its RNG position, is marked kScatterPending and is shaded again in the next iteration
// (returns false), so that a warp does not loop for its unluckiest lane while the other lanes idle.
// FRAMES: the key is the slot's frame's (Pool.frm, p.ftab).
// =====================================================================================================================
template <bool LIGHTS, bool FRAMES>
RT_DEV bool shade_slot(const TraceParams& p, const SceneRefs& sc, const Pool& P, uint32_t s, uint32_t c) {
    uint32_t k0 = p.key0, k1 = p.key1;
    if constexpr (FRAMES) { const FrameRec& fr = p.ftab[P.frm[s]]; k0 = fr.key0; k1 = fr.key1; }
    const DevMat* mat = sc.mat;
    const double4* geo = sc.geo;
    const size_t col = (size_t)P.stack_col + s;
    auto stack_push = [&](uint32_t lvl, uint32_t code) {
        if (lvl < (uint32_t)RT_SMEM_STACK) P.stk[lvl * P.n_slots + s] = code; else p.stack[(size_t)lvl * p.stack_stride + col] = code;
    };
    auto stack_get = [&](uint32_t lvl) -> uint32_t {
        return lvl < (uint32_t)RT_SMEM_STACK ? P.stk[lvl * P.n_slots + s] : p.stack[(size_t)lvl * p.stack_stride + col];
    };
    Rng rng; rng.pixel = P.pix[s]; rng.sample = P.smp[s];
    { uint32_t bh = P.blk[s]; rng.blk = bh >> 1; rng.has = bh & 1u; }
    rng.c_lo = P.clo[s]; rng.c_hi = P.chi[s];
    bool done = false;
    D3 o = mk(P.ox[s], P.oy[s], P.oz[s]), d = mk(P.dx[s], P.dy[s], P.dz[s]);
    uint32_t level = P.lvl[s];
    uint32_t shd = LIGHTS ? (P.shd[s] & ~kScatterPending) : 0u;   // > 0: this ray is a shadow ray of the light test (raytracer.rs:103-106)
    const uint32_t rays_sample = level + 1u;   // main-path hit_world calls so far, this one included
    float cr = 0.f, cg = 0.f, cb = 0.f;
    bool have_tc = false;                      // a shadow ray's ray_color(.., 2, 1) value is ready
    float tr = 0.f, tg = 0.f, tb = 0.f;
    bool state_dirty = false;                  // o/d/rng/level must be written back to the pool
    if (c == CLS_MISS) {                                                // raytracer.rs:134-163
        float x, y, z;
        sky_color(d, length(d), p.sky_mode, p.sky, x, y, z);
        if (shd == 0u) { cr = x; cg = y; cb = z; done = true; }
        else { tr = x; tg = y; tb = z; have_tc = true; }
    } else {
        const uint32_t best = P.bi[s];
        const double best_t = P.bt[s];
        double4 gq = geo[best];
        const D3 center = mk(gq.x, gq.y, gq.z);
        HitRec h = hit_record(center, gq.w, o, d, best_t);
        const DevMat m = mat[best];
        uint32_t code = best;
        D3 nd = d;
        bool absorbed = false;
        const bool is_light = (c == CLS_LIGHT);                         // materials.rs:65-69: Some((None, white))
        D3 rs = mk(0, 0, 0);
        if (c == CLS_DIFFUSE || c == CLS_METAL) {   // one rejection loop for a warp that straddles both classes
            const unsigned group = __activemask();
            const bool sampled = random_in_unit_sphere_ilp<RT_SCATTER_TRIPS>(rng, k0, k1, rs);
            // Reconverge here. The early return below would otherwise put the reconvergence point at the end of the function,
            // and lanes accepted after different numbers of trips would run the rest of the vertex one group after another.
            __syncwarp(group);
            // the scatter draws are the vertex's first draws: a vertex deferred here has changed nothing but its RNG position
            if (!sampled) {
                P.blk[s] = (rng.blk << 1) | rng.has; P.clo[s] = rng.c_lo; P.chi[s] = rng.c_hi;
                P.shd[s] |= kScatterPending;
                return false;
            }
        }
        if (c == CLS_DIFFUSE) {                                         // materials.rs:84-95, 256-267
            D3 sd = add(h.normal, rs);
            if (near_zero(sd)) sd = h.normal;
            D3 target = add(h.point, sd);
            nd = sub(target, h.point);
            if (m.kind == RT_TEXTURE) {
                double tu, tv;
                sphere_uv(sub(h.point, center), tu, tv);
                code = 0x80000000u | texture_texel(p.tex[m.tex], m.param, tu, tv);
            }
        } else if (c == CLS_METAL) {                                    // materials.rs:115-129
            D3 refl = reflect(d, h.normal);
            nd = add(refl, mul(rs, m.param));
            if (!(dot(nd, h.normal) > 0.0)) absorbed = true;            // None -> black, no light test (raytracer.rs:127-131)
        } else if (c == CLS_GLASS) {                                    // materials.rs:176-199
            double ratio = h.front_face ? __ddiv_rn(1.0, m.param) : m.param;
            D3 ud = unit_vector(d);
            double cos_theta = fmin(dot(neg(ud), h.normal), 1.0);
            double sin_theta = __dsqrt_rn(__dsub_rn(1.0, __dmul_rn(cos_theta, cos_theta)));
            bool refl = __dmul_rn(ratio, sin_theta) > 1.0;              // cannot_refract
            if (!refl) refl = reflectance(cos_theta, ratio) > rng_f64(rng, k0, k1);   // drawn only if refraction is possible
            nd = refl ? reflect(ud, h.normal) : refract(ud, h.normal, ratio);
        }
        state_dirty = true;
        if (absorbed) {
            if (shd == 0u) done = true;            // main path ends black
            else have_tc = true;                   // the shadow ray returns black
        } else {
            // ---- light test, raytracer.rs:89-101 (the uniform is drawn whenever the scene has lights) ----
            bool pass = false;
            if (LIGHTS) {
                const double prob = (c == CLS_GLASS) ? 0.05 : 0.1;
                const double xi = rng_f64(rng, k0, k1);
                const unsigned long long depth_now = (unsigned long long)p.max_depth - level;
                const bool depth_ok = (shd > 0u) ? true : (depth_now > (unsigned long long)p.max_depth - 2ull);   // usize wrap like a release build
                pass = (xi > __dsub_rn(1.0, __dmul_rn((double)p.n_lights, prob))) && depth_ok;
                if (pass && shd >= p.max_shadow) { pass = false; atomicAdd(&p.err[0], 1ull); }   // reported as an error by the host
            }
            if (pass) {
                float ar, ag, ab;
                albedo_of(is_light ? 0xffffffffu : code, mat, ar, ag, ab);
                ShadowFrame f;
                f.px = h.point.x; f.py = h.point.y; f.pz = h.point.z; f.ndx = nd.x; f.ndy = nd.y; f.ndz = nd.z;
                f.ar = ar; f.ag = ag; f.ab = ab; f.sr = 0.f; f.sg = 0.f; f.sb = 0.f; f.li = 0u; f.code = code; f.is_light = is_light ? 1u : 0u; f.pad = 0u;
                p.frames[(size_t)shd * p.stack_stride + col] = f;
                ++shd;
                double4 lq = geo[p.lights[0]];
                o = h.point; d = sub(mk(lq.x, lq.y, lq.z), h.point);   // Ray::new(point, light.center - point)
                P.src[s] = best;
            } else if (shd == 0u) {
                if (is_light) { cr = 1.f; cg = 1.f; cb = 1.f; done = true; }   // `None => albedo` (raytracer.rs:124)
                else {
                    stack_push(level, code);
                    ++level;
                    o = h.point; d = nd; P.src[s] = best;
                    if (level == p.max_depth) done = true;   // the next ray_color call returns black (raytracer.rs:80-82)
                }
            } else {
                // nested vertex without light contribution: clamp(0 + albedo * black), or white for a Light. That is 0 for a
                // finite albedo; only a scene with a non-finite one reads it.
                tr = tg = tb = is_light ? 1.f : 0.f;
                if (p.albedo_nonfinite && !is_light) {
                    float ar, ag, ab;
                    albedo_of(code, mat, ar, ag, ab);
                    tr = clampf(__fadd_rn(0.f, __fmul_rn(ar, 0.f))); tg = clampf(__fadd_rn(0.f, __fmul_rn(ag, 0.f))); tb = clampf(__fadd_rn(0.f, __fmul_rn(ab, 0.f)));
                }
                have_tc = true;
            }
        }
    }
    if (LIGHTS) {
        // return values travel up the shadow-frame stack without tracing (raytracer.rs:103-114)
        while (have_tc) {
            ShadowFrame f = p.frames[(size_t)(shd - 1u) * p.stack_stride + col];
            f.sr = __fadd_rn(f.sr, __fmul_rn(f.ar, tr)); f.sg = __fadd_rn(f.sg, __fmul_rn(f.ag, tg)); f.sb = __fadd_rn(f.sb, __fmul_rn(f.ab, tb));
            ++f.li;
            state_dirty = true;
            if (f.li < p.n_lights) {                                   // next light of the same vertex
                p.frames[(size_t)(shd - 1u) * p.stack_stride + col] = f;
                double4 lq = geo[p.lights[f.li]];
                o = mk(f.px, f.py, f.pz); d = sub(mk(lq.x, lq.y, lq.z), o);
                P.src[s] = kNoSphere;   // reading the frame's sphere here made the LIGHTS kernel spill 116 B instead of 76 B
                have_tc = false;
            } else {
                const float nl = (float)p.n_lights;
                const float Lr = __fdiv_rn(f.sr, nl), Lg = __fdiv_rn(f.sg, nl), Lb = __fdiv_rn(f.sb, nl);
                --shd;
                if (shd == 0u) {                                        // back on the main path
                    have_tc = false;
                    if (f.is_light) { cr = 1.f; cg = 1.f; cb = 1.f; done = true; }
                    else {
                        p.lterm[(size_t)(level * 3u + 0u) * p.stack_stride + col] = Lr;   // level is 0 or 1 here
                        p.lterm[(size_t)(level * 3u + 1u) * p.stack_stride + col] = Lg;
                        p.lterm[(size_t)(level * 3u + 2u) * p.stack_stride + col] = Lb;
                        stack_push(level, f.code);
                        ++level;
                        o = mk(f.px, f.py, f.pz); d = mk(f.ndx, f.ndy, f.ndz);
                        P.src[s] = kNoSphere;
                        if (level == p.max_depth) done = true;
                    }
                } else if (f.is_light) { tr = tg = tb = 1.f; }
                else {                                                  // clamp(light + albedo * ray_color(depth 0) = black)
                    tr = clampf(__fadd_rn(Lr, __fmul_rn(f.ar, 0.0f))); tg = clampf(__fadd_rn(Lg, __fmul_rn(f.ag, 0.0f))); tb = clampf(__fadd_rn(Lb, __fmul_rn(f.ab, 0.0f)));
                }
            }
        }
    }
    if (state_dirty && !done) {
        P.ox[s] = o.x; P.oy[s] = o.y; P.oz[s] = o.z; P.dx[s] = d.x; P.dy[s] = d.y; P.dz[s] = d.z;
        P.blk[s] = (rng.blk << 1) | rng.has; P.clo[s] = rng.c_lo; P.chi[s] = rng.c_hi;
        P.lvl[s] = level;
        P.shd[s] = shd;   // also clears kScatterPending
    }
    if (done) {
        // unwind the recursion: c = clamp(light + albedo * c) per level, innermost first (raytracer.rs:117-122). A black path
        // without light terms stays black unless an albedo is non-finite (albedo * 0 = NaN).
        if (LIGHTS || p.albedo_nonfinite || cr != 0.f || cg != 0.f || cb != 0.f) {
            for (int l = (int)level - 1; l >= 0; --l) {
                float ar, ag, ab;
                albedo_of(stack_get((uint32_t)l), mat, ar, ag, ab);
                float Lr = 0.f, Lg = 0.f, Lb = 0.f;
                if (LIGHTS && l < 2) {
                    Lr = p.lterm[(size_t)(l * 3 + 0) * p.stack_stride + col];
                    Lg = p.lterm[(size_t)(l * 3 + 1) * p.stack_stride + col];
                    Lb = p.lterm[(size_t)(l * 3 + 2) * p.stack_stride + col];
                }
                cr = clampf(__fadd_rn(Lr, __fmul_rn(ar, cr)));
                cg = clampf(__fadd_rn(Lg, __fmul_rn(ag, cg)));
                cb = clampf(__fadd_rn(Lb, __fmul_rn(ab, cb)));
            }
        }
        p.samplebuf[P.work[s]] = make_float4(cr, cg, cb, __uint_as_float(rays_sample));
        P.lvl[s] = kDeadLevel;
    }
    return done;
}

RT_DEV void flush_stats(const TraceParams& p, const Stats& st, int lane) {
    unsigned long long v[6] = {st.rays, st.cand, st.ovf, st.samples, st.leaves, st.nodes};
#pragma unroll
    for (int k = 0; k < 6; ++k) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], off);
    }
    if (lane == 0) {
        atomicAdd(&p.stat[0], v[0]);
        atomicAdd(&p.stat[1], v[1]);
        atomicAdd(&p.stat[2], v[2]);
        atomicAdd(&p.stat[3], v[3]);
        atomicAdd(&p.stat[4], v[4]);
        atomicAdd(&p.stat[6], v[5]);
    }
#if RT_PHASE_CLOCKS
    unsigned long long w[6] = {st.t_node, st.t_leaf, st.t_exact, st.exact_steps, st.exact_tests, st.src_skips};
#pragma unroll
    for (int k = 0; k < 6; ++k) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) w[k] += __shfl_down_sync(0xffffffffu, w[k], off);
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < 6; ++k) atomicAdd(&p.stat[kPhaseStat + PH_NODE + k], w[k]);
    }
#endif
}

}  // namespace rtk
