// rtb200_denoise_var.cu — the variance-guided à-trous filter of rtb200_denoise_var[_device] (DESIGN.md §4.18): §4.15's filter
// with each pixel's colour distance divided by its prefiltered variance, and the variance filtered beside the colour with the
// squared weights (SVGF). Every f32 operation is a correctly rounded __f*_rn (never contracted, denormals kept), as
// tests/denoise_var_restatement.py states it in float32 numpy.
//
// rt_denoise_var_pack_kernel       packs the colour into float4 {r, g, b, ok}, where ok = 1.0f when the colour, the variance
//                                  and every given guide of the pixel are finite and the variance is >= 0; the variance into
//                                  float4 {v0, v1, v2, (v0 + v1) + v2}; the guides into float4 {x, y, z, 0}.
// rt_denoise_var_prefilter_kernel  one thread per pixel: 1 / (eps + vbar_p), vbar_p the g x g weighted mean of the summed
//                                  variance over the ok pixels of p's 3 x 3 neighbourhood (step 1 in every iteration).
// rt_denoise_var_step_kernel       one iteration on shared-memory tiles of one residue class of the step, as
//                                  rt_denoise_step_kernel, staging the variance plane beside the colour; ping-pongs between
//                                  two colour and two variance buffers, and the last iteration writes the caller's outputs.
#include "rtb200_kernels.cuh"

using namespace rtd;

namespace rtk {

constexpr int kVarBX = 32, kVarBY = 8;

struct DenoiseVarLayout { float4* col[2]; float4* var[2]; float4* alb; float4* nrm; float* scale; };

// the scratch: two colour and two variance buffers and the albedo and normal guides, npix float4 each, then npix f32 of
// eps + vbar
static DenoiseVarLayout denoise_var_carve(void* base, uint64_t npix, uint64_t* bytes) {
    Carver c(base);
    DenoiseVarLayout l;
    for (auto& p : l.col) p = (float4*)c.take(npix * 16);
    for (auto& p : l.var) p = (float4*)c.take(npix * 16);
    l.alb = (float4*)c.take(npix * 16);
    l.nrm = (float4*)c.take(npix * 16);
    l.scale = (float*)c.take(npix * 4);
    if (bytes) *bytes = c.off;
    return l;
}

static RT_DEV bool finite3v(float a, float b, float c) { return isfinite(a) && isfinite(b) && isfinite(c); }

// ((q0 - p0)^2 + (q1 - p1)^2) + (q2 - p2)^2
static RT_DEV float dist2v(float4 q, float4 p) {
    const float e0 = __fsub_rn(q.x, p.x), e1 = __fsub_rn(q.y, p.y), e2 = __fsub_rn(q.z, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(e0, e0), __fmul_rn(e1, e1)), __fmul_rn(e2, e2));
}

__global__ void __launch_bounds__(256) rt_denoise_var_pack_kernel(const float* color, const float* variance, const float* albedo,
                                                                  const float* normal, uint64_t npix, DenoiseVarLayout l) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    const float r = color[3 * p], g = color[3 * p + 1], b = color[3 * p + 2];
    const float v0 = variance[3 * p], v1 = variance[3 * p + 1], v2 = variance[3 * p + 2];
    // -0 >= 0 holds; a NaN fails both tests
    bool ok = finite3v(r, g, b) && finite3v(v0, v1, v2) && v0 >= 0.0f && v1 >= 0.0f && v2 >= 0.0f;
    if (albedo) {
        const float x = albedo[3 * p], y = albedo[3 * p + 1], z = albedo[3 * p + 2];
        ok = ok && finite3v(x, y, z);
        l.alb[p] = make_float4(x, y, z, 0.0f);
    }
    if (normal) {
        const float x = normal[3 * p], y = normal[3 * p + 1], z = normal[3 * p + 2];
        ok = ok && finite3v(x, y, z);
        l.nrm[p] = make_float4(x, y, z, 0.0f);
    }
    l.col[0][p] = make_float4(r, g, b, ok ? 1.0f : 0.0f);
    l.var[0][p] = make_float4(v0, v1, v2, __fadd_rn(__fadd_rn(v0, v1), v2));
}

// scale_p = eps + (sum of g[dx] g[dy] v_q) / (sum of g[dx] g[dy]) over the ok q of the 3 x 3 around p, dy outer and dx inner.
// Written for ok pixels only (a pixel that is not ok reads no scale).
__global__ void __launch_bounds__(256) rt_denoise_var_prefilter_kernel(const float4* col, const float4* var, float* scale,
                                                                       uint32_t width, uint32_t height, float eps) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (uint64_t)width * height || col[p].w == 0.0f) return;
    const uint32_t x = (uint32_t)(p % width), y = (uint32_t)(p / width);
    const float g[3] = {0.25f, 0.5f, 0.25f};
    float sw = 0.0f, sv = 0.0f;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            const int64_t qx = (int64_t)x + dx, qy = (int64_t)y + dy;
            if (qx < 0 || qx >= width || qy < 0 || qy >= height) continue;
            const uint64_t q = (uint64_t)qy * width + (uint64_t)qx;
            if (col[q].w == 0.0f) continue;
            const float k = __fmul_rn(g[dx + 1], g[dy + 1]);
            sw = __fadd_rn(sw, k);
            sv = __fadd_rn(sv, __fmul_rn(k, var[q].w));
        }
    }
    scale[p] = __fadd_rn(eps, __fdiv_rn(sv, sw));
}

struct DenoiseVarStep {
    const float4* in; const float4* vin; float4* out; float4* vout;   // out, vout: null in the last iteration
    const float4* alb; const float4* nrm;                             // null when that guide is off
    const float* scale;
    float* out_linear; uint8_t* out_rgb8; float* out_variance;        // the last iteration's outputs (each may be null)
    uint32_t width, height, step;
    AtrousTiles tiles;               // the step's grid
    float lc, la, ln;
};

// One iteration on shared-memory tiles of step h's residue classes (see rt_denoise_step_kernel): a CTA stages a
// (kVarBX + 4) x (kVarBY + 4) block of the colour, the variance and each guide that is on, taps outside the image with ok = 0.
constexpr int kVHX = kVarBX + 4, kVHY = kVarBY + 4;
__global__ void __launch_bounds__(kVarBX * kVarBY) rt_denoise_var_step_kernel(const DenoiseVarStep s) {
    __shared__ float4 sc[kVHY][kVHX], sv[kVHY][kVHX], sa[kVHY][kVHX], sn[kVHY][kVHX];
    const uint32_t h = s.step;
    uint32_t tix, tiy, rx, ry;
    s.tiles.decode(blockIdx.x, tix, tiy, rx, ry);
    const int64_t gx0 = (int64_t)tix * kVarBX - 2, gy0 = (int64_t)tiy * kVarBY - 2;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = threadIdx.y * kVarBX + threadIdx.x; k < kVHX * kVHY; k += kVarBX * kVarBY) {
        const int ly = k / kVHX, lx = k % kVHX;
        const int64_t x = (int64_t)rx + (gx0 + lx) * h, y = (int64_t)ry + (gy0 + ly) * h;
        const bool in = x >= 0 && x < s.width && y >= 0 && y < s.height;
        const uint64_t q = in ? (uint64_t)y * s.width + (uint64_t)x : 0;
        sc[ly][lx] = in ? s.in[q] : z;
        sv[ly][lx] = in ? s.vin[q] : z;
        if (s.alb) sa[ly][lx] = in ? s.alb[q] : z;
        if (s.nrm) sn[ly][lx] = in ? s.nrm[q] : z;
    }
    __syncthreads();
    const int tx = threadIdx.x + 2, ty = threadIdx.y + 2;
    const int64_t x = (int64_t)rx + ((int64_t)tix * kVarBX + threadIdx.x) * h, y = (int64_t)ry + ((int64_t)tiy * kVarBY + threadIdx.y) * h;
    if (x >= s.width || y >= s.height) return;
    const uint64_t p = (uint64_t)y * s.width + (uint64_t)x;
    const float4 cp = sc[ty][tx];
    float4 o = cp, vo = sv[ty][tx];   // a pixel that is not ok keeps its colour and variance
    if (cp.w != 0.0f) {
        const float4 ap = s.alb ? sa[ty][tx] : z, np = s.nrm ? sn[ty][tx] : z;
        const float scale = s.scale[p];
        const float B[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
        float n0 = 0.0f, n1 = 0.0f, n2 = 0.0f, den = 0.0f, m0 = 0.0f, m1 = 0.0f, m2 = 0.0f;
#pragma unroll
        for (int dy = -2; dy <= 2; ++dy) {
#pragma unroll
            for (int dx = -2; dx <= 2; ++dx) {
                const float4 cq = sc[ty + dy][tx + dx];
                if (cq.w == 0.0f) continue;
                // the factors left to right; an off guide's is left out
                float f = 1.0f;
                if (s.lc != 0.0f) f = __fadd_rn(1.0f, __fmul_rn(s.lc, __fdiv_rn(dist2v(cq, cp), scale)));
                if (s.alb) f = __fmul_rn(f, __fadd_rn(1.0f, __fmul_rn(s.la, dist2v(sa[ty + dy][tx + dx], ap))));
                if (s.nrm) f = __fmul_rn(f, __fadd_rn(1.0f, __fmul_rn(s.ln, dist2v(sn[ty + dy][tx + dx], np))));
                const float w = __fdiv_rn(__fmul_rn(B[dx + 2], B[dy + 2]), f);
                n0 = __fadd_rn(n0, __fmul_rn(w, cq.x));
                n1 = __fadd_rn(n1, __fmul_rn(w, cq.y));
                n2 = __fadd_rn(n2, __fmul_rn(w, cq.z));
                den = __fadd_rn(den, w);
                const float4 vq = sv[ty + dy][tx + dx];
                const float ww = __fmul_rn(w, w);
                m0 = __fadd_rn(m0, __fmul_rn(ww, vq.x));
                m1 = __fadd_rn(m1, __fmul_rn(ww, vq.y));
                m2 = __fadd_rn(m2, __fmul_rn(ww, vq.z));
            }
        }
        const float d2 = __fmul_rn(den, den);
        o = make_float4(__fdiv_rn(n0, den), __fdiv_rn(n1, den), __fdiv_rn(n2, den), 0.0f);
        vo.x = __fdiv_rn(m0, d2); vo.y = __fdiv_rn(m1, d2); vo.z = __fdiv_rn(m2, d2);
        vo.w = __fadd_rn(__fadd_rn(vo.x, vo.y), vo.z);
        o.w = finite3v(o.x, o.y, o.z) && finite3v(vo.x, vo.y, vo.z) ? 1.0f : 0.0f;
    }
    if (s.out) { s.out[p] = o; s.vout[p] = vo; return; }
    if (s.out_linear) { s.out_linear[3 * p] = o.x; s.out_linear[3 * p + 1] = o.y; s.out_linear[3 * p + 2] = o.z; }
    if (s.out_rgb8) { s.out_rgb8[3 * p] = quantise_u8(o.x); s.out_rgb8[3 * p + 1] = quantise_u8(o.y); s.out_rgb8[3 * p + 2] = quantise_u8(o.z); }
    if (s.out_variance) { s.out_variance[3 * p] = vo.x; s.out_variance[3 * p + 1] = vo.y; s.out_variance[3 * p + 2] = vo.z; }
}

uint64_t denoise_var_scratch_bytes(uint64_t npix) {
    uint64_t bytes = 0;
    denoise_var_carve(nullptr, npix, &bytes);
    return bytes;
}

cudaError_t launch_denoise_var(const DenoiseVarArgs& a, cudaStream_t st) {
    const uint64_t npix = (uint64_t)a.width * a.height;
    const DenoiseVarLayout l = denoise_var_carve(a.scratch, npix, nullptr);
    const unsigned pgrid = (unsigned)((npix + 255) / 256);
    rt_denoise_var_pack_kernel<<<pgrid, 256, 0, st>>>(a.color, a.variance, a.albedo, a.normal, npix, l);
    cudaError_t e = cudaGetLastError();
    const dim3 block(kVarBX, kVarBY);
    for (uint32_t i = 0; e == cudaSuccess && i < a.iterations; ++i) {
        const bool last = i + 1 == a.iterations;
        const uint32_t cur = i & 1, nxt = (i + 1) & 1;
        rt_denoise_var_prefilter_kernel<<<pgrid, 256, 0, st>>>(l.col[cur], l.var[cur], l.scale, a.width, a.height, a.variance_floor);
        if ((e = cudaGetLastError()) != cudaSuccess) break;
        DenoiseVarStep s{};
        s.in = l.col[cur]; s.vin = l.var[cur];
        s.out = last ? nullptr : l.col[nxt]; s.vout = last ? nullptr : l.var[nxt];
        s.alb = a.albedo && a.albedo_weight != 0.0f ? l.alb : nullptr;
        s.nrm = a.normal && a.normal_weight != 0.0f ? l.nrm : nullptr;
        s.scale = l.scale;
        s.out_linear = last ? a.out_linear : nullptr;
        s.out_rgb8 = last ? a.out_rgb8 : nullptr;
        s.out_variance = last ? a.out_variance : nullptr;
        s.width = a.width; s.height = a.height; s.step = 1u << i;
        s.lc = a.color_weight; s.la = a.albedo_weight; s.ln = a.normal_weight;
        s.tiles = AtrousTiles(a.width, a.height, s.step, kVarBX, kVarBY);
        rt_denoise_var_step_kernel<<<(unsigned)s.tiles.ctas(), block, 0, st>>>(s);   // <= width * height CTAs
        e = cudaGetLastError();
    }
    return e;
}

}  // namespace rtk
