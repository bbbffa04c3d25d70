// rtb200_denoise.cu — the edge-avoiding à-trous wavelet filter (Dammertz et al. 2010) of rtb200_denoise[_device] (DESIGN.md
// §4.15), with rational edge-stopping weights so that every operation is a correctly rounded f32 + - * / (__f*_rn: never
// contracted, denormals kept), as tests/denoise_restatement.py states it in float32 numpy.
//
// rt_denoise_pack_kernel   packs the caller's colour into float4 {r, g, b, ok}, where ok = 1.0f when the colour and every given
//                          guide of the pixel are finite, and the guides into float4 {x, y, z, 0}: a tap is one 16-byte value
//                          for the colour and the finite test, and one for each guide that is on.
// rt_denoise_step_kernel   one iteration on shared-memory tiles of one residue class of the step (below), one thread per output
//                          pixel and its 25 taps in the contract's order: a fixed-order sum, so the result is deterministic
//                          without atomics or grid-wide synchronisation. It ping-pongs between the two colour buffers; the last
//                          iteration writes the caller's linear and/or RGB8 outputs instead. A pixel's ok stays ok && its new
//                          colour is finite: a pixel that was not ok keeps its colour. A kernel reading the taps through L1/L2
//                          instead was 16-20 % slower (DESIGN.md §4.15).
#include "rtb200_kernels.cuh"

using namespace rtd;

namespace rtk {

constexpr int kDenoiseBX = 32, kDenoiseBY = 8;

struct DenoiseLayout { float4* col[2]; float4* alb; float4* nrm; };

// the scratch: two colour buffers, then the albedo and normal guides, npix float4 each
static DenoiseLayout denoise_carve(void* base, uint64_t npix, uint64_t* bytes) {
    Carver c(base);
    DenoiseLayout l;
    for (auto& p : l.col) p = (float4*)c.take(npix * 16);
    l.alb = (float4*)c.take(npix * 16);
    l.nrm = (float4*)c.take(npix * 16);
    if (bytes) *bytes = c.off;
    return l;
}

RT_DEV bool finite3(float a, float b, float c) { return isfinite(a) && isfinite(b) && isfinite(c); }

// ((q0 - p0)^2 + (q1 - p1)^2) + (q2 - p2)^2
RT_DEV float dist2(float4 q, float4 p) {
    const float e0 = __fsub_rn(q.x, p.x), e1 = __fsub_rn(q.y, p.y), e2 = __fsub_rn(q.z, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(e0, e0), __fmul_rn(e1, e1)), __fmul_rn(e2, e2));
}

__global__ void __launch_bounds__(256) rt_denoise_pack_kernel(const float* color, const float* albedo, const float* normal,
                                                              uint64_t npix, DenoiseLayout l) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    const float r = color[3 * p], g = color[3 * p + 1], b = color[3 * p + 2];
    bool ok = finite3(r, g, b);
    if (albedo) {
        const float x = albedo[3 * p], y = albedo[3 * p + 1], z = albedo[3 * p + 2];
        ok = ok && finite3(x, y, z);
        l.alb[p] = make_float4(x, y, z, 0.0f);
    }
    if (normal) {
        const float x = normal[3 * p], y = normal[3 * p + 1], z = normal[3 * p + 2];
        ok = ok && finite3(x, y, z);
        l.nrm[p] = make_float4(x, y, z, 0.0f);
    }
    l.col[0][p] = make_float4(r, g, b, ok ? 1.0f : 0.0f);
}

struct DenoiseStep {
    const float4* in; float4* out;   // out: null in the last iteration
    const float4* alb; const float4* nrm;   // null when that guide is off
    float* out_linear; uint8_t* out_rgb8;   // the last iteration's outputs (each may be null)
    uint32_t width, height, step;
    AtrousTiles tiles;               // the step's grid
    float lc, la, ln;                // the weights of this iteration (lc = color_weight * 4^i)
};

// Pixel p's output from its colour cp and guides ap, np (of the guides that are on) and tap(dx, dy, cq, aq, nq), which gives tap
// (dx, dy)'s colour and guides and returns false for a tap outside the image (a tap with cq.w == 0 is skipped as well).
template <typename Tap>
RT_DEV float4 denoise_pixel(const DenoiseStep& s, float4 cp, float4 ap, float4 np, Tap tap) {
    if (cp.w == 0.0f) return cp;
    const float B[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    float n0 = 0.0f, n1 = 0.0f, n2 = 0.0f, den = 0.0f;
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy) {
#pragma unroll
        for (int dx = -2; dx <= 2; ++dx) {
            float4 cq, aq, nq;
            if (!tap(dx, dy, cq, aq, nq) || cq.w == 0.0f) continue;
            // the factors left to right; an off guide's is left out (1 * f is f, so starting from 1 changes nothing)
            float f = 1.0f;
            if (s.lc != 0.0f) f = __fmul_rn(f, __fadd_rn(1.0f, __fmul_rn(s.lc, dist2(cq, cp))));
            if (s.alb) f = __fmul_rn(f, __fadd_rn(1.0f, __fmul_rn(s.la, dist2(aq, ap))));
            if (s.nrm) f = __fmul_rn(f, __fadd_rn(1.0f, __fmul_rn(s.ln, dist2(nq, np))));
            const float w = __fdiv_rn(__fmul_rn(B[dx + 2], B[dy + 2]), f);
            n0 = __fadd_rn(n0, __fmul_rn(w, cq.x));
            n1 = __fadd_rn(n1, __fmul_rn(w, cq.y));
            n2 = __fadd_rn(n2, __fmul_rn(w, cq.z));
            den = __fadd_rn(den, w);
        }
    }
    float4 o;
    o.x = __fdiv_rn(n0, den); o.y = __fdiv_rn(n1, den); o.z = __fdiv_rn(n2, den);
    o.w = finite3(o.x, o.y, o.z) ? 1.0f : 0.0f;
    return o;
}

RT_DEV void denoise_store(const DenoiseStep& s, uint64_t p, float4 o) {
    if (s.out) { s.out[p] = o; return; }
    if (s.out_linear) { s.out_linear[3 * p] = o.x; s.out_linear[3 * p + 1] = o.y; s.out_linear[3 * p + 2] = o.z; }
    if (s.out_rgb8) { s.out_rgb8[3 * p] = quantise_u8(o.x); s.out_rgb8[3 * p + 1] = quantise_u8(o.y); s.out_rgb8[3 * p + 2] = quantise_u8(o.z); }
}

// One iteration on shared-memory tiles of step h's residue classes: the pixels (rx + h i, ry + h j) of residue (rx, ry) form a
// dense sub-grid on which every tap is a neighbour at distance <= 2, so a CTA stages a (kDenoiseBX + 4) x (kDenoiseBY + 4) block
// of it (a halo of 2; taps outside the image are staged with w = 0) and reads its 25 taps from shared memory. A 1-D grid of
// tiles (a grid's y extent is limited to 65535) over the residue classes that hold a pixel (AtrousTiles).
constexpr int kHX = kDenoiseBX + 4, kHY = kDenoiseBY + 4;
__global__ void __launch_bounds__(kDenoiseBX * kDenoiseBY) rt_denoise_step_kernel(const DenoiseStep s) {
    __shared__ float4 sc[kHY][kHX], sa[kHY][kHX], sn[kHY][kHX];
    const uint32_t h = s.step;
    uint32_t tix, tiy, rx, ry;
    s.tiles.decode(blockIdx.x, tix, tiy, rx, ry);
    const int64_t gx0 = (int64_t)tix * kDenoiseBX - 2, gy0 = (int64_t)tiy * kDenoiseBY - 2;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = threadIdx.y * kDenoiseBX + threadIdx.x; k < kHX * kHY; k += kDenoiseBX * kDenoiseBY) {
        const int ly = k / kHX, lx = k % kHX;
        const int64_t x = (int64_t)rx + (gx0 + lx) * h, y = (int64_t)ry + (gy0 + ly) * h;
        const bool in = x >= 0 && x < s.width && y >= 0 && y < s.height;
        const uint64_t q = in ? (uint64_t)y * s.width + (uint64_t)x : 0;
        sc[ly][lx] = in ? s.in[q] : z;
        if (s.alb) sa[ly][lx] = in ? s.alb[q] : z;
        if (s.nrm) sn[ly][lx] = in ? s.nrm[q] : z;
    }
    __syncthreads();
    const int tx = threadIdx.x + 2, ty = threadIdx.y + 2;
    const int64_t x = (int64_t)rx + ((int64_t)tix * kDenoiseBX + threadIdx.x) * h, y = (int64_t)ry + ((int64_t)tiy * kDenoiseBY + threadIdx.y) * h;
    if (x >= s.width || y >= s.height) return;
    const float4 o = denoise_pixel(s, sc[ty][tx], s.alb ? sa[ty][tx] : z, s.nrm ? sn[ty][tx] : z,
                                   [&](int dx, int dy, float4& cq, float4& aq, float4& nq) {
        cq = sc[ty + dy][tx + dx];   // a tap outside the image is staged with w = 0
        aq = s.alb ? sa[ty + dy][tx + dx] : z;
        nq = s.nrm ? sn[ty + dy][tx + dx] : z;
        return true;
    });
    denoise_store(s, (uint64_t)y * s.width + (uint64_t)x, o);
}

uint64_t denoise_scratch_bytes(uint64_t npix) {
    uint64_t bytes = 0;
    denoise_carve(nullptr, npix, &bytes);
    return bytes;
}

cudaError_t launch_denoise(const DenoiseArgs& a, cudaStream_t st) {
    const uint64_t npix = (uint64_t)a.width * a.height;
    const DenoiseLayout l = denoise_carve(a.scratch, npix, nullptr);
    rt_denoise_pack_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, st>>>(a.color, a.albedo, a.normal, npix, l);
    cudaError_t e = cudaGetLastError();
    const dim3 block(kDenoiseBX, kDenoiseBY);
    for (uint32_t i = 0; e == cudaSuccess && i < a.iterations; ++i) {
        const bool last = i + 1 == a.iterations;
        DenoiseStep s{};
        s.in = l.col[i & 1];
        s.out = last ? nullptr : l.col[(i + 1) & 1];
        s.alb = a.albedo && a.albedo_weight != 0.0f ? l.alb : nullptr;
        s.nrm = a.normal && a.normal_weight != 0.0f ? l.nrm : nullptr;
        s.out_linear = last ? a.out_linear : nullptr;
        s.out_rgb8 = last ? a.out_rgb8 : nullptr;
        s.width = a.width; s.height = a.height; s.step = 1u << i;
        s.lc = a.color_weight * (float)(1u << (2 * i));   // exact: the host refused a color_weight whose 4^(L-1) multiple overflows
        s.la = a.albedo_weight; s.ln = a.normal_weight;
        s.tiles = AtrousTiles(a.width, a.height, s.step, kDenoiseBX, kDenoiseBY);
        rt_denoise_step_kernel<<<(unsigned)s.tiles.ctas(), block, 0, st>>>(s);   // <= width * height CTAs
        e = cudaGetLastError();
    }
    return e;
}

}  // namespace rtk
