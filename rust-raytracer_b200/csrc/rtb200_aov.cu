// rtb200_aov.cu — the auxiliary buffers of a resident scene's camera samples (rtb200_scene_aov[_device], DESIGN.md §4.14):
// per pixel the mean first-hit albedo and normal, the samples that hit, and the sphere and hit point of the first sample.
//
// The kernel uses the query kernels' CTA (rtb200_query.cuh). A warp takes chunks of 32 consecutive local pixels, x innermost,
// in grid-stride order, so that neighbouring lanes trace neighbouring camera rays. For each sample in order every lane writes
// its pixel's primary ray into its slot - the render's own, made by primary_ray (rtb200_trace.cuh) - and the warp runs
// closest_hit<MODE> unchanged; each lane then adds the sample's albedo and normal to its f32 sums in registers. Nothing goes
// through a sample buffer and no random number is drawn beyond the render's two jitter draws (and, on a lens handle, the
// lens draws of primary_ray<true>, in a domain of their own: rt_aov_lens_kernel, DESIGN.md §4.17).
#include "rtb200_query.cuh"

namespace rtk {

namespace {

template <uint32_t MODE, bool LENS>
__device__ __forceinline__ void aov_body(const AovParams& q) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const uint32_t warp = threadIdx.x >> 5;
    unsigned char* base = smem_raw + warp * query_warp_bytes(MODE);
    const WarpCtx W = warpctx_at(base);   // read by MODE_TREE only
    const Pool P = query_pool_at(base + (MODE == MODE_TREE ? kWarpCtxBytes : 0u));
    const SceneRefs sc = scene_refs(q.p);
    const float scale = __fdiv_rn(1.0f, (float)q.samples);   // the resolve's 1.0f / spp
    Stats st;
    const uint64_t chunks = ((uint64_t)q.n + 31u) / 32u;
    for (uint64_t c = (uint64_t)blockIdx.x * kQueryWarps + warp; c < chunks; c += (uint64_t)gridDim.x * kQueryWarps) {
        const uint64_t i = c * 32u + (uint64_t)lane;
        const bool alive = i < q.n;   // the last chunk has dead lanes
        const uint32_t y_local = alive ? (uint32_t)i / q.p.width : 0u, x = alive ? (uint32_t)i - y_local * q.p.width : 0u;
        float ar = 0.f, ag = 0.f, ab = 0.f, nx = 0.f, ny = 0.f, nz = 0.f;
        uint32_t hits = 0u, sphere = kNoSphere;
        D3 point = mk(0, 0, 0);
        for (uint32_t k = 0; k < q.samples; ++k) {
            D3 o = mk(0, 0, 0), d = mk(0, 0, 0);
            if (alive) {
                Rng rng;
                primary_ray<LENS>(q.p, q.p.cam, q.p.lens, q.p.key0, q.p.key1, x, y_local, q.sample0, k, rng, o, d);
                P.ox[lane] = o.x; P.oy[lane] = o.y; P.oz[lane] = o.z; P.dx[lane] = d.x; P.dy[lane] = d.y; P.dz[lane] = d.z;
                P.src[lane] = kNoSphere;   // a camera ray starts on no sphere
                ++st.samples;
            }
            __syncwarp();   // the exact step reads the other lanes' rays
            closest_hit<MODE>(q.p, sc, P, W, alive, (uint32_t)lane, lane, st);
            if (alive) {
                const uint32_t j = P.bi[lane];
                float r, g, b;
                if (j != kNoSphere) {
                    const double4 gq = sc.geo[j];
                    const D3 center = mk(gq.x, gq.y, gq.z);
                    const HitRec h = hit_record(center, gq.w, o, d, P.bt[lane]);
                    // Material::scatter's attenuation without its draws: a texel, white for Glass and Light, else the albedo
                    const DevMat m = sc.mat[j];
                    uint32_t code = j;
                    if (m.kind == RT_TEXTURE) {
                        double tu, tv;
                        sphere_uv(sub(h.point, center), tu, tv);
                        code = 0x80000000u | texture_texel(q.p.tex[m.tex], m.param, tu, tv);
                    } else if (m.kind == RT_GLASS || m.kind == RT_LIGHT) {
                        code = 0xffffffffu;
                    }
                    albedo_of(code, sc.mat, r, g, b);
                    nx = __fadd_rn(nx, __double2float_rn(h.normal.x));
                    ny = __fadd_rn(ny, __double2float_rn(h.normal.y));
                    nz = __fadd_rn(nz, __double2float_rn(h.normal.z));
                    ++hits;
                    if (k == 0u) { sphere = j; point = h.point; }
                } else {
                    sky_color(d, length(d), q.p.sky_mode, q.p.sky, r, g, b);   // a miss: the sky; its normal is 0
                    nx = __fadd_rn(nx, 0.f); ny = __fadd_rn(ny, 0.f); nz = __fadd_rn(nz, 0.f);
                }
                ar = __fadd_rn(ar, r); ag = __fadd_rn(ag, g); ab = __fadd_rn(ab, b);
            }
            __syncwarp();   // every lane is done with the slots before the next sample overwrites them
        }
        if (alive) {
            if (q.albedo) { q.albedo[3 * i] = __fmul_rn(scale, ar); q.albedo[3 * i + 1] = __fmul_rn(scale, ag); q.albedo[3 * i + 2] = __fmul_rn(scale, ab); }
            if (q.normal) { q.normal[3 * i] = __fmul_rn(scale, nx); q.normal[3 * i + 1] = __fmul_rn(scale, ny); q.normal[3 * i + 2] = __fmul_rn(scale, nz); }
            if (q.hits) q.hits[i] = hits;
            if (q.sphere) q.sphere[i] = sphere;
            if (q.point) { q.point[3 * i] = point.x; q.point[3 * i + 1] = point.y; q.point[3 * i + 2] = point.z; }
        }
    }
    if (q.p.stat) flush_stats(q.p, st, lane);
}

template <uint32_t MODE>
__global__ void __launch_bounds__(kQueryBlock) rt_aov_kernel(const __grid_constant__ AovParams q) { aov_body<MODE, false>(q); }
// the camera rays through the handle's lens, q.p.lens (its radius is not 0)
template <uint32_t MODE>
__global__ void __launch_bounds__(kQueryBlock) rt_aov_lens_kernel(const __grid_constant__ AovParams q) { aov_body<MODE, true>(q); }

template <typename F>
static auto dispatch_aov(uint32_t mode, bool lens, F&& f) {
    if (lens) {
        if (mode == MODE_EXACT) return f(rt_aov_lens_kernel<MODE_EXACT>);
        if (mode == MODE_BRUTE) return f(rt_aov_lens_kernel<MODE_BRUTE>);
        return f(rt_aov_lens_kernel<MODE_TREE>);
    }
    if (mode == MODE_EXACT) return f(rt_aov_kernel<MODE_EXACT>);
    if (mode == MODE_BRUTE) return f(rt_aov_kernel<MODE_BRUTE>);
    return f(rt_aov_kernel<MODE_TREE>);
}

}  // namespace

int aov_max_ctas_per_sm(uint32_t mode, bool lens) {
    return dispatch_aov(mode, lens, [&](auto kern) { return query_ctas_per_sm(kern, query_smem_bytes(mode)); });
}

cudaError_t launch_aov(const AovParams& q, uint32_t mode, int max_grid, cudaStream_t st) {
    return dispatch_aov(mode, q.p.lens.radius != 0.0, [&](auto kern) { return query_launch(kern, query_smem_bytes(mode), q, max_grid, st); });
}

}  // namespace rtk
