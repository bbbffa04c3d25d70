// rtb200_temporal.cu — the temporal accumulation of rtb200_temporal[_device] (DESIGN.md §4.16): each pixel of a frame is
// reprojected into the previous frame through its first hit and blended with the history found there, as include/rtb200.h
// states it and tests/temporal_restatement.py restates it in numpy. Every f64 and f32 operation goes through the __d*_rn /
// __f*_rn intrinsics, so nothing is contracted or reordered.
//
// rt_temporal_kernel   one thread per pixel: the pixel's two projections in f64, then a 2x2 gather of the previous frame's
//                      history colour and length, sphere and point around the reprojected position, in the contract's tap
//                      order. Memory-bound: about 40 B of the pixel's own inputs, up to 4 x 44 B of neighbours (mostly the
//                      pixel's own neighbourhood, so L1/L2 hits) and 16 B of output.
// rt_temporal_clamped_kernel   the same with the history clamp of rtb200_temporal_clamped[_device] (DESIGN.md §4.20): where a
//                      pixel keeps a history, its colour is clamped to mean +- gamma * sd of the current frame's colours in the
//                      (2r + 1)^2 window around the pixel, read through the read-only path, before the blend.
// rt_temporal_var_kernel, rt_temporal_var_clamped_kernel   either of the above that also carries the variance of each pixel's
//                      mean through the accumulation (rtb200_temporal_var[_device], DESIGN.md §4.21): the history's variance is
//                      gathered over the same valid taps with the same weights, and blended with the frame's as b^2 Vh + a^2 v.
//                      Its three planes are a kernel parameter of their own (TemporalVar), so the kernels above keep theirs.
#include "rtb200_kernels.cuh"

using namespace rtd;

namespace rtk {

constexpr int kTemporalBlock = 256;

namespace {

// (y1 z2 - z1 y2, z1 x2 - x1 z2, x1 y2 - y1 x2)
RT_DEV D3 cross(D3 a, D3 b) {
    return mk(__dsub_rn(__dmul_rn(a.y, b.z), __dmul_rn(a.z, b.y)), __dsub_rn(__dmul_rn(a.z, b.x), __dmul_rn(a.x, b.z)),
              __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x)));
}

// The image coordinates (u, v) of direction d under camera c; false when d does not project (behind the camera, parallel to
// the image plane, or u or v not finite).
RT_DEV bool project(const rt_camera& c, D3 d, double& u, double& v) {
    const D3 a = sub(from(c.lower_left_corner), from(c.origin)), h = from(c.horizontal), vt = from(c.vertical);
    const D3 cn = cross(h, vt);
    const double den = dot(cn, d);
    const double front = __ddiv_rn(dot(cn, a), den);
    u = __ddiv_rn(dot(cross(vt, a), d), den);
    v = __ddiv_rn(dot(cross(a, h), d), den);
    return den != 0.0 && front > 0.0 && isfinite(u) && isfinite(v);
}

RT_DEV bool finite3(float a, float b, float c) { return isfinite(a) && isfinite(b) && isfinite(c); }

// The history h_k of pixel (x, y) clamped to [mean - gamma * sd, mean + gamma * sd] of the current colours in the window of
// radius r around the pixel, per channel; a window pixel counts when it is inside the image and its colour is finite.
RT_DEV void clamp_history(const TemporalArgs& a, uint32_t x, uint32_t y, float gamma, uint32_t r, float& h0, float& h1, float& h2) {
    const int64_t W = a.width, H = a.height, R = r;
    float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, q0 = 0.0f, q1 = 0.0f, q2 = 0.0f;
    uint32_t m = 0;
    for (int64_t dy = -R; dy <= R; ++dy) {
        const int64_t qy = (int64_t)y + dy;
        if (qy < 0 || qy >= H) continue;
        for (int64_t dx = -R; dx <= R; ++dx) {
            const int64_t qx = (int64_t)x + dx;
            if (qx < 0 || qx >= W) continue;
            const uint64_t q = (uint64_t)(qy * W + qx);
            const float c0 = __ldg(a.color + 3 * q), c1 = __ldg(a.color + 3 * q + 1), c2 = __ldg(a.color + 3 * q + 2);
            if (!finite3(c0, c1, c2)) continue;
            s0 = __fadd_rn(s0, c0); q0 = __fadd_rn(q0, __fmul_rn(c0, c0));
            s1 = __fadd_rn(s1, c1); q1 = __fadd_rn(q1, __fmul_rn(c1, c1));
            s2 = __fadd_rn(s2, c2); q2 = __fadd_rn(q2, __fmul_rn(c2, c2));
            ++m;
        }
    }
    const float fm = __uint2float_rn(m);
    auto clamp1 = [&](float s, float q, float& h) {
        const float mean = __fdiv_rn(s, fm);
        const float var = __fsub_rn(__fdiv_rn(q, fm), __fmul_rn(mean, mean));
        const float d = __fmul_rn(gamma, __fsqrt_rn(var < 0.0f ? 0.0f : var));
        const float lo = __fsub_rn(mean, d), hi = __fadd_rn(mean, d);
        h = h < lo ? lo : (h > hi ? hi : h);   // a NaN lo, hi or h leaves h as it is
    };
    clamp1(s0, q0, h0); clamp1(s1, q1, h1); clamp1(s2, q2, h2);
}

// One pixel of any of the kernels; CLAMP adds clamp_history between the gathered history and the blend, and VAR the variance
// planes of vr beside the colour (a tap's variance is read only when the tap is valid); neither changes anything else.
template <bool CLAMP, bool VAR>
__device__ __forceinline__ void temporal_pixel(const TemporalArgs& a, float gamma, uint32_t radius, const TemporalVar& vr) {
    const uint64_t W = a.width, H = a.height;
    const uint64_t p = (uint64_t)blockIdx.x * kTemporalBlock + threadIdx.x;
    if (p >= W * H) return;
    const uint32_t x = (uint32_t)(p % W), y = (uint32_t)(p / W);
    const float c0 = a.color[3 * p], c1 = a.color[3 * p + 1], c2 = a.color[3 * p + 2];
    float o0 = c0, o1 = c1, o2 = c2;
    float v0 = 0.0f, v1 = 0.0f, v2 = 0.0f;
    if constexpr (VAR) { v0 = vr.var[3 * p]; v1 = vr.var[3 * p + 1]; v2 = vr.var[3 * p + 2]; }
    float ov0 = v0, ov1 = v1, ov2 = v2;   // no history: the frame's variance as given
    uint32_t len = 1;
    if (a.h_color && finite3(c0, c1, c2)) {
        const uint32_t j = a.sphere[p];
        const bool hit = j != 0xffffffffu;
        D3 pp = mk(0.0, 0.0, 0.0), dc, dp;
        if (hit) {
            const D3 P = mk(a.point[3 * p], a.point[3 * p + 1], a.point[3 * p + 2]);
            pp = j < a.n_motion ? sub(P, mk(a.motion[3 * (uint64_t)j], a.motion[3 * (uint64_t)j + 1], a.motion[3 * (uint64_t)j + 2])) : P;
            dc = sub(P, from(a.cam.origin));
            dp = sub(pp, from(a.prev_cam.origin));
        } else {
            const double u = __ddiv_rn(__dadd_rn((double)x, 0.5), __dsub_rn((double)W, 1.0));
            const double v = __ddiv_rn(__dsub_rn((double)H, __dadd_rn((double)y, 0.5)), __dsub_rn((double)H, 1.0));
            D3 o;
            get_ray(a.cam, u, v, o, dc);
            dp = dc;
        }
        double uc, vc, up, vp;
        if (project(a.cam, dc, uc, vc) && project(a.prev_cam, dp, up, vp)) {
            const double fx = __dadd_rn((double)x, __dmul_rn(__dsub_rn(up, uc), __dsub_rn((double)W, 1.0)));
            const double fy = __dsub_rn((double)y, __dmul_rn(__dsub_rn(vp, vc), __dsub_rn((double)H, 1.0)));
            if (isfinite(fx) && isfinite(fy)) {
                const double x0 = floor(fx), y0 = floor(fy);
                const float ax = __double2float_rn(__dsub_rn(fx, x0)), ay = __double2float_rn(__dsub_rn(fy, y0));
                const float bx = __fsub_rn(1.0f, ax), by = __fsub_rn(1.0f, ay);
                const float w[4] = {__fmul_rn(bx, by), __fmul_rn(ax, by), __fmul_rn(bx, ay), __fmul_rn(ax, ay)};
                const double tol2 = __dmul_rn(a.depth_tol, a.depth_tol);
                const double lim = hit ? __dmul_rn(tol2, dot(dp, dp)) : 0.0;
                float s = 0.0f, n0 = 0.0f, n1 = 0.0f, n2 = 0.0f;
                float m0 = 0.0f, m1 = 0.0f, m2 = 0.0f;   // VAR: sum of w * prev_variance
                uint32_t L = 0xffffffffu;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const double tx = __dadd_rn(x0, (double)(k & 1)), ty = __dadd_rn(y0, (double)(k >> 1));
                    if (!(w[k] > 0.0f && tx >= 0.0 && tx < (double)W && ty >= 0.0 && ty < (double)H)) continue;
                    const uint64_t q = (uint64_t)ty * W + (uint64_t)tx;
                    const uint32_t lq = a.h_length[q];
                    if (lq < 1 || a.h_sphere[q] != j) continue;
                    const float h0 = a.h_color[3 * q], h1 = a.h_color[3 * q + 1], h2 = a.h_color[3 * q + 2];
                    if (!finite3(h0, h1, h2)) continue;
                    if (hit) {
                        const D3 e = sub(mk(a.h_point[3 * q], a.h_point[3 * q + 1], a.h_point[3 * q + 2]), pp);
                        if (!(dot(e, e) <= lim)) continue;
                    }
                    s = __fadd_rn(s, w[k]);
                    n0 = __fadd_rn(n0, __fmul_rn(w[k], h0));
                    n1 = __fadd_rn(n1, __fmul_rn(w[k], h1));
                    n2 = __fadd_rn(n2, __fmul_rn(w[k], h2));
                    if constexpr (VAR) {
                        m0 = __fadd_rn(m0, __fmul_rn(w[k], vr.h_var[3 * q]));
                        m1 = __fadd_rn(m1, __fmul_rn(w[k], vr.h_var[3 * q + 1]));
                        m2 = __fadd_rn(m2, __fmul_rn(w[k], vr.h_var[3 * q + 2]));
                    }
                    L = min(L, lq);
                }
                if (s != 0.0f) {
                    const uint32_t n = min(L, a.max_history - 1) + 1;
                    if (n >= 2) {
                        float g0 = __fdiv_rn(n0, s), g1 = __fdiv_rn(n1, s), g2 = __fdiv_rn(n2, s);
                        if constexpr (CLAMP) clamp_history(a, x, y, gamma, radius, g0, g1, g2);
                        const float alpha = __fdiv_rn(1.0f, __uint2float_rn(n));
                        o0 = __fadd_rn(g0, __fmul_rn(alpha, __fsub_rn(c0, g0)));
                        o1 = __fadd_rn(g1, __fmul_rn(alpha, __fsub_rn(c1, g1)));
                        o2 = __fadd_rn(g2, __fmul_rn(alpha, __fsub_rn(c2, g2)));
                        if constexpr (VAR) {   // b^2 Vh + a^2 v: the clamp moves the colour only
                            const float b = __fsub_rn(1.0f, alpha), bb = __fmul_rn(b, b), aa = __fmul_rn(alpha, alpha);
                            ov0 = __fadd_rn(__fmul_rn(bb, __fdiv_rn(m0, s)), __fmul_rn(aa, v0));
                            ov1 = __fadd_rn(__fmul_rn(bb, __fdiv_rn(m1, s)), __fmul_rn(aa, v1));
                            ov2 = __fadd_rn(__fmul_rn(bb, __fdiv_rn(m2, s)), __fmul_rn(aa, v2));
                        }
                        len = n;
                    }
                }
            }
        }
    }
    a.out_color[3 * p] = o0; a.out_color[3 * p + 1] = o1; a.out_color[3 * p + 2] = o2;
    a.out_length[p] = len;
    if constexpr (VAR) { vr.out_var[3 * p] = ov0; vr.out_var[3 * p + 1] = ov1; vr.out_var[3 * p + 2] = ov2; }
}

}  // namespace

__global__ void __launch_bounds__(kTemporalBlock) rt_temporal_kernel(const TemporalArgs a) { temporal_pixel<false, false>(a, 0.0f, 0, TemporalVar{}); }

__global__ void __launch_bounds__(kTemporalBlock) rt_temporal_clamped_kernel(const TemporalArgs a, const float gamma, const uint32_t radius) {
    temporal_pixel<true, false>(a, gamma, radius, TemporalVar{});
}

__global__ void __launch_bounds__(kTemporalBlock) rt_temporal_var_kernel(const TemporalArgs a, const TemporalVar v) {
    temporal_pixel<false, true>(a, 0.0f, 0, v);
}

__global__ void __launch_bounds__(kTemporalBlock) rt_temporal_var_clamped_kernel(const TemporalArgs a, const float gamma, const uint32_t radius,
                                                                                 const TemporalVar v) {
    temporal_pixel<true, true>(a, gamma, radius, v);
}

cudaError_t launch_temporal(const TemporalArgs& a, const TemporalClamp* clamp, const TemporalVar* var, cudaStream_t st) {
    const uint64_t npix = (uint64_t)a.width * a.height;
    const unsigned grid = (unsigned)((npix + kTemporalBlock - 1) / kTemporalBlock);
    if (var && clamp)
        rt_temporal_var_clamped_kernel<<<grid, kTemporalBlock, 0, st>>>(a, clamp->gamma, clamp->radius, *var);
    else if (var)
        rt_temporal_var_kernel<<<grid, kTemporalBlock, 0, st>>>(a, *var);
    else if (clamp)
        rt_temporal_clamped_kernel<<<grid, kTemporalBlock, 0, st>>>(a, clamp->gamma, clamp->radius);
    else
        rt_temporal_kernel<<<grid, kTemporalBlock, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace rtk
