// rtb200_adaptive.cu — the per-pixel kernels of adaptive rendering (rtb200_adaptive_*, DESIGN.md §4.9).
//
// A round traces samples [n, n + s_count) of every pixel still on the list (rt_wavefront_kernel<.., Q_LIST>), then:
//   rt_adaptive_accumulate_kernel  adds them to the pixel's f32 sums S_c and Q_c in sample order, advances n and applies the
//                                  stopping rule; keep[k] says whether list position k stays;
//   cub::DeviceSelect::Flagged     writes the kept pixels, in list order, into the other list buffer and their number into
//                                  device memory, where the next round's trace kernel reads it.
// rt_adaptive_resolve_kernel turns S and n into the outputs. Every f32 operation rounds to nearest and none is contracted, so
// mean_c = (1/n) * S_c is exactly the one-shot render's value at samples_per_pixel = n (rt_resolve_kernel).
#include <cub/cub.cuh>

#include "rtb200_kernels.cuh"

using namespace rtd;

namespace rtk {

__global__ void __launch_bounds__(256) rt_adaptive_accumulate_kernel(const AdaptiveParams q) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= q.npix_local) return;
    const uint32_t n_list = *q.list_n;
    const bool listed = k < n_list;
    if (q.black_samples) {   // max_depth 0: no trace kernel counted these samples
        const unsigned b = __ballot_sync(__activemask(), listed);
        if (b && (threadIdx.x & 31u) == (uint32_t)(__ffs(b) - 1)) atomicAdd(q.black_samples, (unsigned long long)__popc(b) * q.s_count);
    }
    if (!listed) { q.keep[k] = 0u; return; }
    const uint32_t lp = q.list[k];
    float S[3], Q[3];
    for (int c = 0; c < 3; ++c) { S[c] = q.sum[3 * (size_t)lp + c]; Q[c] = q.sq[3 * (size_t)lp + c]; }
    for (uint32_t s = 0; s < q.s_count; ++s) {
        const float4 x = q.samplebuf[(size_t)s * n_list + k];
        S[0] = __fadd_rn(S[0], x.x); S[1] = __fadd_rn(S[1], x.y); S[2] = __fadd_rn(S[2], x.z);
        Q[0] = __fadd_rn(Q[0], __fmul_rn(x.x, x.x)); Q[1] = __fadd_rn(Q[1], __fmul_rn(x.y, x.y)); Q[2] = __fadd_rn(Q[2], __fmul_rn(x.z, x.z));
    }
    for (int c = 0; c < 3; ++c) { q.sum[3 * (size_t)lp + c] = S[c]; q.sq[3 * (size_t)lp + c] = Q[c]; }
    const uint32_t n = q.n_after;
    q.count[lp] = n;
    // the stopping rule (include/rtb200.h, rt_adaptive_params)
    bool stop = n >= q.max_samples;
    if (!stop && n >= q.min_samples) {
        const float inv = __fdiv_rn(1.0f, (float)n);
        bool ok = true;
        for (int c = 0; c < 3; ++c) {
            const float mean = __fmul_rn(inv, S[c]);
            const float var = __fsub_rn(__fmul_rn(inv, Q[c]), __fmul_rn(mean, mean));
            const float err = __fsqrt_rn(__fmul_rn(var > 0.0f ? var : 0.0f, inv));
            const float tol = __fadd_rn(q.abs_tol, __fmul_rn(q.rel_tol, mean));
            ok = ok && isfinite(S[c]) && isfinite(Q[c]) && err <= tol;
        }
        stop = ok;
    }
    q.keep[k] = stop ? 0u : 1u;
}

__global__ void __launch_bounds__(256) rt_adaptive_resolve_kernel(const AdaptiveResolveParams q) {
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= q.npix_local) return;
    const uint32_t n = q.count[lp];
    if (q.out_count) q.out_count[lp] = n;
    float m[3] = {0.0f, 0.0f, 0.0f};
    if (n) {
        const float inv = __fdiv_rn(1.0f, (float)n);
        for (int c = 0; c < 3; ++c) m[c] = __fmul_rn(inv, q.sum[3 * (size_t)lp + c]);
    }
    for (int c = 0; c < 3; ++c) {
        if (q.out_linear) q.out_linear[3 * (size_t)lp + c] = m[c];
        if (q.out_rgb8) q.out_rgb8[3 * (size_t)lp + c] = quantise_u8(m[c]);
    }
}

// rt_adaptive_resolve_kernel plus the variance of each pixel's mean from S, Q and n (0 where n = 0), as rt_resolve_var_kernel
__global__ void __launch_bounds__(256) rt_adaptive_resolve_var_kernel(const AdaptiveResolveVarParams v) {
    const AdaptiveResolveParams& q = v.r;
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= q.npix_local) return;
    const uint32_t n = q.count[lp];
    if (q.out_count) q.out_count[lp] = n;
    float m[3] = {0.0f, 0.0f, 0.0f}, var[3] = {0.0f, 0.0f, 0.0f};
    if (n) {
        const float inv = __fdiv_rn(1.0f, (float)n);
        for (int c = 0; c < 3; ++c) {
            const float S = q.sum[3 * (size_t)lp + c], Q = v.sq[3 * (size_t)lp + c];
            m[c] = __fmul_rn(inv, S);
            const float d = __fsub_rn(__fmul_rn(inv, Q), __fmul_rn(m[c], m[c]));
            var[c] = __fmul_rn(d < 0.0f ? 0.0f : d, inv);
        }
    }
    for (int c = 0; c < 3; ++c) {
        if (q.out_linear) q.out_linear[3 * (size_t)lp + c] = m[c];
        if (q.out_rgb8) q.out_rgb8[3 * (size_t)lp + c] = quantise_u8(m[c]);
        v.out_variance[3 * (size_t)lp + c] = var[c];
    }
}

// begin: every pixel on the list, in increasing order
__global__ void __launch_bounds__(256) rt_adaptive_list_kernel(uint32_t* list, uint32_t* list_n, uint32_t npix_local) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < npix_local) list[k] = k;
    if (k == 0) *list_n = npix_local;
}

cudaError_t launch_adaptive_list(uint32_t* list, uint32_t* list_n, uint32_t npix_local, cudaStream_t st) {
    rt_adaptive_list_kernel<<<(npix_local + 255u) / 256u, 256, 0, st>>>(list, list_n, npix_local);
    return cudaGetLastError();
}

cudaError_t launch_adaptive_accumulate(const AdaptiveParams& q, cudaStream_t st) {
    rt_adaptive_accumulate_kernel<<<(q.npix_local + 255u) / 256u, 256, 0, st>>>(q);
    return cudaGetLastError();
}

size_t adaptive_compact_bytes(uint32_t npix_local) {
    size_t bytes = 0;
    cub::DeviceSelect::Flagged(nullptr, bytes, (const uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                               (int)npix_local);
    return bytes;
}

cudaError_t launch_adaptive_compact(void* temp, size_t temp_bytes, const uint32_t* list_in, const uint32_t* keep, uint32_t* list_out,
                                    uint32_t* list_n_out, uint32_t npix_local, cudaStream_t st) {
    return cub::DeviceSelect::Flagged(temp, temp_bytes, list_in, keep, list_out, list_n_out, (int)npix_local, st);
}

cudaError_t launch_adaptive_resolve(const AdaptiveResolveParams& q, cudaStream_t st) {
    rt_adaptive_resolve_kernel<<<(q.npix_local + 255u) / 256u, 256, 0, st>>>(q);
    return cudaGetLastError();
}

cudaError_t launch_adaptive_resolve_var(const AdaptiveResolveVarParams& v, cudaStream_t st) {
    rt_adaptive_resolve_var_kernel<<<(v.r.npix_local + 255u) / 256u, 256, 0, st>>>(v);
    return cudaGetLastError();
}

}  // namespace rtk
