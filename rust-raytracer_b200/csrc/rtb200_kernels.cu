// rtb200_kernels.cu — the resolve kernel and the device-routine probes.
//
// rt_resolve_kernel: adds each pixel's samples in sample order (raytracer.rs:203-205), then scale*sum, sqrt and the u8
// quantisation (raytracer.rs:207-216). Used after every trace launch of the production kernel (rtb200_wavefront.cu).
// (The lane-autonomous trace kernel of round 1, RT_VARIANT_LANES, was retired in round 2: git history, DESIGN.md §4.5.)
#include "rtb200_kernels.cuh"

using namespace rtd;

namespace rtk {

// Per pixel: add the batch's samples in sample order, f32, exactly like raytracer.rs:197-206; on the last batch
// produce mean = scale*sum (raytracer.rs:207), the linear output and the quantised RGB8 pixel (raytracer.rs:208-216).
__global__ void __launch_bounds__(256) rt_resolve_kernel(const ResolveParams q) {
    uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= q.npix_local) return;
    float r = 0.f, g = 0.f, b = 0.f;
    if (!q.first) { r = q.accum[3 * (size_t)lp]; g = q.accum[3 * (size_t)lp + 1]; b = q.accum[3 * (size_t)lp + 2]; }
    for (uint32_t s = 0; s < q.s_count; ++s) {
        float4 c = q.samplebuf[(size_t)s * q.npix_local + lp];
        r = __fadd_rn(r, c.x); g = __fadd_rn(g, c.y); b = __fadd_rn(b, c.z);
    }
    if (!q.last) {
        q.accum[3 * (size_t)lp] = r; q.accum[3 * (size_t)lp + 1] = g; q.accum[3 * (size_t)lp + 2] = b;
        return;
    }
    float scale = __fdiv_rn(1.0f, (float)q.spp);
    float mr = __fmul_rn(scale, r), mg = __fmul_rn(scale, g), mb = __fmul_rn(scale, b);
    if (q.out_linear) { q.out_linear[3 * (size_t)lp] = mr; q.out_linear[3 * (size_t)lp + 1] = mg; q.out_linear[3 * (size_t)lp + 2] = mb; }
    if (q.out_rgb8) {
        q.out_rgb8[3 * (size_t)lp] = quantise_u8(mr);
        q.out_rgb8[3 * (size_t)lp + 1] = quantise_u8(mg);
        q.out_rgb8[3 * (size_t)lp + 2] = quantise_u8(mb);
    }
}

// The variance of a pixel's mean from its sums S_c and Q_c over n samples: inv = 1/n, mean_c = inv * S_c,
// d_c = inv * Q_c - mean_c * mean_c, var_c = (d_c < 0 ? 0 : d_c) * inv (a NaN d_c stays NaN). n = 0 gives 0.
static RT_DEV float mean_variance(float S, float Q, float inv) {
    const float mean = __fmul_rn(inv, S);
    const float d = __fsub_rn(__fmul_rn(inv, Q), __fmul_rn(mean, mean));
    return __fmul_rn(d < 0.0f ? 0.0f : d, inv);
}

// rt_resolve_kernel with the running sums Q_c of x_c * x_c beside S_c and, on the last batch, the variance of the mean: the
// linear and RGB8 outputs are rt_resolve_kernel's, operation for operation. A separate kernel, so that a render without a
// variance output launches rt_resolve_kernel exactly as before.
__global__ void __launch_bounds__(256) rt_resolve_var_kernel(const ResolveVarParams v) {
    const ResolveParams& q = v.r;
    uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= q.npix_local) return;
    float S[3] = {0.f, 0.f, 0.f}, Q[3] = {0.f, 0.f, 0.f};
    if (!q.first)
        for (int c = 0; c < 3; ++c) { S[c] = q.accum[3 * (size_t)lp + c]; Q[c] = v.accum_sq[3 * (size_t)lp + c]; }
    for (uint32_t s = 0; s < q.s_count; ++s) {
        const float4 x = q.samplebuf[(size_t)s * q.npix_local + lp];
        S[0] = __fadd_rn(S[0], x.x); S[1] = __fadd_rn(S[1], x.y); S[2] = __fadd_rn(S[2], x.z);
        Q[0] = __fadd_rn(Q[0], __fmul_rn(x.x, x.x)); Q[1] = __fadd_rn(Q[1], __fmul_rn(x.y, x.y)); Q[2] = __fadd_rn(Q[2], __fmul_rn(x.z, x.z));
    }
    if (!q.last) {
        for (int c = 0; c < 3; ++c) { q.accum[3 * (size_t)lp + c] = S[c]; v.accum_sq[3 * (size_t)lp + c] = Q[c]; }
        return;
    }
    const float scale = __fdiv_rn(1.0f, (float)q.spp);
    for (int c = 0; c < 3; ++c) {
        const float m = __fmul_rn(scale, S[c]);
        if (q.out_linear) q.out_linear[3 * (size_t)lp + c] = m;
        if (q.out_rgb8) q.out_rgb8[3 * (size_t)lp + c] = quantise_u8(m);
        v.out_variance[3 * (size_t)lp + c] = mean_variance(S[c], Q[c], scale);
    }
}

cudaError_t trace_configure(int device, int* sm_count, size_t* max_smem_optin) {
    cudaDeviceProp prop;
    cudaError_t e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) return e;
    *sm_count = prop.multiProcessorCount;
    *max_smem_optin = prop.sharedMemPerBlockOptin;
    return cudaSuccess;
}

cudaError_t launch_resolve(const ResolveParams& q, cudaStream_t st) {
    int grid = (int)((q.npix_local + 255u) / 256u);
    rt_resolve_kernel<<<grid, 256, 0, st>>>(q);
    return cudaGetLastError();
}

cudaError_t launch_resolve_var(const ResolveVarParams& v, cudaStream_t st) {
    rt_resolve_var_kernel<<<(v.r.npix_local + 255u) / 256u, 256, 0, st>>>(v);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// probes: the same device routines on one thread (known-answer tests of the reference, see include/rtb200.h)
// ---------------------------------------------------------------------------------------------------
__global__ void k_probe_sphere_hit(const double* in, double* out) {
    D3 c = mk(in[0], in[1], in[2]); double r = in[3];
    D3 o = mk(in[4], in[5], in[6]), d = mk(in[7], in[8], in[9]);
    double root = 0.0;
    bool ok = sphere_root(c, r, o, d, length_squared(d), in[10], in[11], root);
    out[0] = ok ? 1.0 : 0.0;
    if (ok) {
        HitRec h = hit_record(c, r, o, d, root);
        out[1] = root; out[2] = h.point.x; out[3] = h.point.y; out[4] = h.point.z;
        out[5] = h.normal.x; out[6] = h.normal.y; out[7] = h.normal.z; out[8] = h.front_face ? 1.0 : 0.0;
    }
}
__global__ void k_probe_refract(const double* in, double* out) {
    D3 r = refract(mk(in[0], in[1], in[2]), mk(in[3], in[4], in[5]), in[6]);
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
__global__ void k_probe_reflectance(const double* in, double* out) { out[0] = reflectance(in[0], in[1]); }
__global__ void k_probe_sky(const double* in, uint32_t mode, float* out) {
    DevTex none; none.rgb8 = nullptr; none.width = 0; none.height = 0;
    D3 dd = mk(in[0], in[1], in[2]);
    sky_color(dd, length(dd), mode, none, out[0], out[1], out[2]);
}
__global__ void k_probe_get_ray(const rt_camera* cam, const double* in, double* out) {
    D3 o, d;
    get_ray(*cam, in[0], in[1], o, d);
    out[0] = o.x; out[1] = o.y; out[2] = o.z; out[3] = d.x; out[4] = d.y; out[5] = d.z;
}
// the pinhole ray moved onto the lens, as primary_ray makes it; out[6] = the lens trials drawn
__global__ void k_probe_lens_ray(const rt_camera* cam, const rt_lens* lens, const double* in, uint32_t k0, uint32_t k1, uint32_t pixel,
                                 uint32_t sample, double* out) {
    D3 o, d;
    get_ray(*cam, in[0], in[1], o, d);
    uint32_t trials = 0;
    if (lens->radius != 0.0) trials = lens_apply(*lens, pixel, sample, k0, k1, o, d);
    out[0] = o.x; out[1] = o.y; out[2] = o.z; out[3] = d.x; out[4] = d.y; out[5] = d.z; out[6] = (double)trials;
}
__global__ void k_probe_rng(uint32_t k0, uint32_t k1, uint32_t pixel, uint32_t sample, uint32_t kind, uint32_t n, double* out) {
    Rng g; rng_init(g, pixel, sample);
    for (uint32_t i = 0; i < n; ++i) out[i] = kind == 0 ? rng_f64(g, k0, k1) : rng_m1_1(g, k0, k1);
}
__global__ void k_probe_quantise(const float* in, uint32_t n, uint8_t* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = quantise_u8(in[i]);
}

__global__ void k_probe_sphere_uv(const double* in, uint32_t n, double* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) sphere_uv(mk(in[3 * i], in[3 * i + 1], in[3 * i + 2]), out[2 * i], out[2 * i + 1]);
}
cudaError_t probe_sphere_uv(const double* in, uint32_t n, double* out, cudaStream_t st) {
    k_probe_sphere_uv<<<(n + 255) / 256, 256, 0, st>>>(in, n, out);
    return cudaGetLastError();
}

cudaError_t probe_sphere_hit(const double* in, double* out, cudaStream_t st) { k_probe_sphere_hit<<<1, 1, 0, st>>>(in, out); return cudaGetLastError(); }
cudaError_t probe_refract(const double* in, double* out, cudaStream_t st) { k_probe_refract<<<1, 1, 0, st>>>(in, out); return cudaGetLastError(); }
cudaError_t probe_reflectance(const double* in, double* out, cudaStream_t st) { k_probe_reflectance<<<1, 1, 0, st>>>(in, out); return cudaGetLastError(); }
cudaError_t probe_sky(const double* in, uint32_t mode, float* out, cudaStream_t st) { k_probe_sky<<<1, 1, 0, st>>>(in, mode, out); return cudaGetLastError(); }
cudaError_t probe_get_ray(const rt_camera* cam, const double* in, double* out, cudaStream_t st) { k_probe_get_ray<<<1, 1, 0, st>>>(cam, in, out); return cudaGetLastError(); }
cudaError_t probe_lens_ray(const rt_camera* cam, const rt_lens* lens, const double* in, uint64_t seed, uint32_t pixel, uint32_t sample,
                           double* out, cudaStream_t st) {
    k_probe_lens_ray<<<1, 1, 0, st>>>(cam, lens, in, (uint32_t)seed, (uint32_t)(seed >> 32), pixel, sample, out);
    return cudaGetLastError();
}
cudaError_t probe_rng(uint64_t seed, uint32_t pixel, uint32_t sample, uint32_t kind, uint32_t n, double* out, cudaStream_t st) {
    k_probe_rng<<<1, 1, 0, st>>>((uint32_t)seed, (uint32_t)(seed >> 32), pixel, sample, kind, n, out);
    return cudaGetLastError();
}
cudaError_t probe_quantise(const float* in, uint32_t n, uint8_t* out, cudaStream_t st) {
    k_probe_quantise<<<(n + 255) / 256, 256, 0, st>>>(in, n, out);
    return cudaGetLastError();
}

}  // namespace rtk
