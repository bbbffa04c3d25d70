// rtb200_device.cuh — device-side building blocks of the H100 render path.
//
// Numerical contract: geometry is evaluated in IEEE f64 with the reference's operation order and NO
// fused multiply-add (rustc never contracts), colour in f32 likewise. Every reference-exact operation
// therefore goes through the __d*_rn / __f*_rn intrinsics, which nvcc never contracts into FMAs.
// Citations are file:line under /root/reference/raytracer/src/.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <float.h>

#include "../../include/rtb200.h"

#define RT_DEV __device__ __forceinline__

namespace rtd {

// ---- Point3D (point3d.rs:52-171), exact f64 -------------------------------------------------------
struct D3 { double x, y, z; };

RT_DEV D3 mk(double x, double y, double z) { D3 r; r.x = x; r.y = y; r.z = z; return r; }
RT_DEV D3 from(const rt_vec3& v) { return mk(v.x, v.y, v.z); }
RT_DEV D3 add(D3 a, D3 b) { return mk(__dadd_rn(a.x, b.x), __dadd_rn(a.y, b.y), __dadd_rn(a.z, b.z)); }      // :89-99
RT_DEV D3 sub(D3 a, D3 b) { return mk(__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y), __dsub_rn(a.z, b.z)); }      // :101-111
RT_DEV D3 neg(D3 a) { return mk(-a.x, -a.y, -a.z); }                                                          // :113-123
RT_DEV D3 mul(D3 a, double s) { return mk(__dmul_rn(a.x, s), __dmul_rn(a.y, s), __dmul_rn(a.z, s)); }        // :137-147
RT_DEV D3 divs(D3 a, double s) { return mk(__ddiv_rn(a.x, s), __ddiv_rn(a.y, s), __ddiv_rn(a.z, s)); }       // :161-171
RT_DEV double dot(D3 a, D3 b) {                                                                               // :72-74
    return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}
RT_DEV double length_squared(D3 a) { return dot(a, a); }                                                      // :59-61
RT_DEV double length(D3 a) { return __dsqrt_rn(length_squared(a)); }                                          // :63-65 (x-0.0 is exact)
RT_DEV D3 unit_vector(D3 a) { double l = length(a); return divs(a, l); }                                      // :67-70
RT_DEV bool near_zero(D3 a) {                                                                                 // :84-86
    const double e = 2.220446049250313e-16;
    return fabs(a.x) < e && fabs(a.y) < e && fabs(a.z) < e;
}

// ---- Philox4x32-10 per-(pixel,sample) stream (DESIGN.md "RNG contract") ----------------------------
struct Rng {
    uint32_t pixel, sample, blk;
    uint32_t c_lo, c_hi;   // cached second u64 of the current block
    uint32_t has;
};

RT_DEV void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t out[4]) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
        uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
        uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += W0; k1 += W1;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

RT_DEV void rng_init(Rng& g, uint32_t pixel, uint32_t sample) { g.pixel = pixel; g.sample = sample; g.blk = 0; g.has = 0; g.c_lo = 0; g.c_hi = 0; }

RT_DEV void rng_next(Rng& g, uint32_t k0, uint32_t k1, uint32_t& lo, uint32_t& hi) {
    if (g.has) { g.has = 0; lo = g.c_lo; hi = g.c_hi; return; }
    uint32_t w[4];
    philox4x32_10(g.blk, g.sample, g.pixel, 0u, k0, k1, w);
    g.blk += 1;
    g.c_lo = w[2]; g.c_hi = w[3]; g.has = 1;
    lo = w[0]; hi = w[1];
}
// rand 0.8 Standard f64: (u64 >> 11) * 2^-53
RT_DEV double rng_f64(Rng& g, uint32_t k0, uint32_t k1) {
    uint32_t lo, hi; rng_next(g, k0, k1, lo, hi);
    unsigned long long v = (((unsigned long long)hi << 32) | lo) >> 11;
    return __dmul_rn((double)v, 1.0 / 9007199254740992.0);
}
// rand 0.8 UniformFloat::sample_single(-1,1): ((u64>>12 as mantissa in [1,2)) - 1) * 2 + (-1)
RT_DEV double rng_m1_1(Rng& g, uint32_t k0, uint32_t k1) {
    uint32_t lo, hi; rng_next(g, k0, k1, lo, hi);
    unsigned long long bits = ((((unsigned long long)hi << 32) | lo) >> 12) | 0x3FF0000000000000ull;
    double v01 = __dsub_rn(__longlong_as_double((long long)bits), 1.0);
    return __dadd_rn(__dmul_rn(v01, 2.0), -1.0);
}
RT_DEV double u64_to_m1_1(uint32_t lo, uint32_t hi) {
    unsigned long long bits = ((((unsigned long long)hi << 32) | lo) >> 12) | 0x3FF0000000000000ull;
    double v01 = __dsub_rn(__longlong_as_double((long long)bits), 1.0);
    return __dadd_rn(__dmul_rn(v01, 2.0), -1.0);
}
// random_in_unit_sphere (point3d.rs:22-38) on the same stream with the same draws, but two rejection trials per loop trip
// and their three Philox blocks computed together (instruction-level parallelism: the shade stage is bound by the latency
// of this dependent chain, not by throughput). At most TRIPS trips: returns true with the accepted point in `out`, or
// false with the stream position (blk, has, cached half-block) exactly where the unbounded loop stands after the same
// trips, so that a later call continues the same rejection sequence and accepts the same point.
template <int TRIPS>
RT_DEV bool random_in_unit_sphere_ilp(Rng& g, uint32_t k0, uint32_t k1, D3& out) {
#pragma unroll 1
    for (int trip = 0; trip < TRIPS; ++trip) {
        uint32_t A[4], B[4], Cc[4];
        philox4x32_10(g.blk, g.sample, g.pixel, 0u, k0, k1, A);
        philox4x32_10(g.blk + 1u, g.sample, g.pixel, 0u, k0, k1, B);
        philox4x32_10(g.blk + 2u, g.sample, g.pixel, 0u, k0, k1, Cc);
        // u[i] = the next unread u64 draws of the stream: (cached,) A.lo, A.hi, B.lo, B.hi, C.lo, C.hi
        uint32_t lo[7], hi[7];
        if (g.has) { lo[0] = g.c_lo; hi[0] = g.c_hi; lo[1] = A[0]; hi[1] = A[1]; lo[2] = A[2]; hi[2] = A[3]; lo[3] = B[0]; hi[3] = B[1]; lo[4] = B[2]; hi[4] = B[3]; lo[5] = Cc[0]; hi[5] = Cc[1]; lo[6] = Cc[2]; hi[6] = Cc[3]; }
        else { lo[0] = A[0]; hi[0] = A[1]; lo[1] = A[2]; hi[1] = A[3]; lo[2] = B[0]; hi[2] = B[1]; lo[3] = B[2]; hi[3] = B[3]; lo[4] = Cc[0]; hi[4] = Cc[1]; lo[5] = Cc[2]; hi[5] = Cc[3]; lo[6] = 0; hi[6] = 0; }
        D3 p1 = mk(u64_to_m1_1(lo[0], hi[0]), u64_to_m1_1(lo[1], hi[1]), u64_to_m1_1(lo[2], hi[2]));
        D3 p2 = mk(u64_to_m1_1(lo[3], hi[3]), u64_to_m1_1(lo[4], hi[4]), u64_to_m1_1(lo[5], hi[5]));
        const bool a1 = length_squared(p1) < 1.0, a2 = length_squared(p2) < 1.0;
        const uint32_t used = a1 ? 3u : 6u;                       // draws consumed by this trip
        // stream position in u64 units before the trip: 2*blk - has; advance it and rebuild (blk, has, cached)
        const uint32_t pos = 2u * g.blk - g.has + used;
        g.blk = (pos + 1u) >> 1;
        g.has = pos & 1u;
        g.c_lo = a1 ? lo[3] : lo[6]; g.c_hi = a1 ? hi[3] : hi[6];   // the next unread draw; it is a block's second half exactly when pos is odd
        if (a1) { out = p1; return true; }
        if (a2) { out = p2; return true; }
    }
    return false;
}

// ---- the thin lens (DESIGN.md §4.17) --------------------------------------------------------------
// The lens disk of sample (pixel, sample): trial k reads Philox block (k, sample, pixel, 1) - counter word 1, a domain of its
// own, so the path's stream is untouched - x from its first u64, y from its second, both gen_range(-1.0..1.0); the first
// trial with x*x + y*y < 1 is accepted. Two trials per loop trip, their blocks computed together (as random_in_unit_sphere_ilp).
// Returns the trials drawn (k + 1 of the accepted one).
RT_DEV uint32_t lens_disk(uint32_t pixel, uint32_t sample, uint32_t k0, uint32_t k1, double& x, double& y) {
#pragma unroll 1
    for (uint32_t k = 0;; k += 2u) {
        uint32_t A[4], B[4];
        philox4x32_10(k, sample, pixel, 1u, k0, k1, A);
        philox4x32_10(k + 1u, sample, pixel, 1u, k0, k1, B);
        const double x1 = u64_to_m1_1(A[0], A[1]), y1 = u64_to_m1_1(A[2], A[3]);
        const double x2 = u64_to_m1_1(B[0], B[1]), y2 = u64_to_m1_1(B[2], B[3]);
        if (__dadd_rn(__dmul_rn(x1, x1), __dmul_rn(y1, y1)) < 1.0) { x = x1; y = y1; return k + 1u; }
        if (__dadd_rn(__dmul_rn(x2, x2), __dmul_rn(y2, y2)) < 1.0) { x = x2; y = y2; return k + 2u; }
    }
}
// The pinhole ray (o, d) of (pixel, sample) moved onto the lens `L` of radius > 0: o + offset, d - offset with
// offset = L.u * (r x) + L.v * (r y). Out of line: it runs only for a lens camera, and inlined into the trace kernel's
// regeneration it would hold its registers across every path of a pinhole render too. Returns the trials drawn.
RT_DEV uint32_t lens_apply(const rt_lens& L, uint32_t pixel, uint32_t sample, uint32_t k0, uint32_t k1, D3& o, D3& d) {
    double x, y;
    const uint32_t trials = lens_disk(pixel, sample, k0, k1, x, y);
    const double rdx = __dmul_rn(L.radius, x), rdy = __dmul_rn(L.radius, y);
    const D3 off = add(mul(from(L.u), rdx), mul(from(L.v), rdy));
    o = add(o, off);
    d = sub(d, off);
    return trials;
}

// ---- Camera::get_ray (camera.rs:79-84) -------------------------------------------------------------
RT_DEV void get_ray(const rt_camera& c, double u, double v, D3& origin, D3& dir) {
    origin = from(c.origin);
    dir = sub(add(add(from(c.lower_left_corner), mul(from(c.horizontal), u)), mul(from(c.vertical), v)), origin);
}

// ---- Sphere::hit (sphere.rs:46-78), root selection only ---------------------------------------------
// Returns the first root in (t_min, t_max), near root first, or a negative sentinel (-1) when none.
// `a` = direction.length_squared() is the same for every sphere, so the caller computes it once.
RT_DEV bool sphere_root(D3 center, double radius, D3 o, D3 d, double a, double t_min, double t_max, double& root) {
    D3 oc = sub(o, center);
    double half_b = dot(oc, d);
    double cc = __dsub_rn(length_squared(oc), __dmul_rn(radius, radius));
    double disc = __dsub_rn(__dmul_rn(half_b, half_b), __dmul_rn(a, cc));
    if (disc >= 0.0) {
        double sq = __dsqrt_rn(disc);
        double ra = __ddiv_rn(__dsub_rn(-half_b, sq), a);
        if (ra < t_max && ra > t_min) { root = ra; return true; }
        double rb = __ddiv_rn(__dadd_rn(-half_b, sq), a);
        if (rb < t_max && rb > t_min) { root = rb; return true; }
    }
    return false;
}

// Certificate for a ray that starts on the sphere (center, radius), a = length_squared(d): true only when sphere_root(center,
// radius, o, d, a, 0.001, t_max) provably finds no root, decided with sphere_root's own rounded oc, half_b, c and a but
// without its square root and divisions (proof in DESIGN.md §4.2). half_b >= 0 (the ray leaves the centre behind) and
// c >= 0 (the origin rounded onto or outside the sphere): disc <= fl(half_b^2), whose rounded square root is half_b, so
// both roots are <= 0. c < 0 (rounded just inside): the far root is below fl(a|c|) / (2 half_b a) + 3u half_b / a, and
// the test bounds it by 0.0009 < t_min with room for every rounding. Inward rays (half_b < 0) are never certified.
RT_DEV bool leaves_sphere(D3 center, double radius, D3 o, D3 d, double a) {
    const D3 oc = sub(o, center);
    const double half_b = dot(oc, d);
    const double cc = __dsub_rn(length_squared(oc), __dmul_rn(radius, radius));
    // every product below is a normal finite double; NaNs fail these comparisons
    if (!(half_b >= 0x1p-300 && half_b <= 0x1p300 && a >= 0x1p-300 && a <= 0x1p300)) return false;
    if (cc >= 0.0) return true;
    if (!(cc <= -0x1p-300 && cc >= -0x1p300)) return false;
    // fl(a |c|) + 2^-48 fl(half_b^2) <= fl(fl(0.0018 a) half_b)
    return __dadd_rn(__dmul_rn(a, -cc), __dmul_rn(0x1p-48, __dmul_rn(half_b, half_b))) <= __dmul_rn(__dmul_rn(0.0018, a), half_b);
}

// Two spheres at once: the same operations in the same order per sphere, with the two dependent f64 chains interleaved
// (the confirmation stage is latency-bound). Root selection as in sphere_root with t_max = +max.
RT_DEV void sphere_root2(D3 c0, double r0, D3 c1, double r1, D3 o, D3 d, double a, double t_min, bool& h0, double& root0, bool& h1, double& root1) {
    D3 oc0 = sub(o, c0), oc1 = sub(o, c1);
    double hb0 = dot(oc0, d), hb1 = dot(oc1, d);
    double cc0 = __dsub_rn(length_squared(oc0), __dmul_rn(r0, r0)), cc1 = __dsub_rn(length_squared(oc1), __dmul_rn(r1, r1));
    double disc0 = __dsub_rn(__dmul_rn(hb0, hb0), __dmul_rn(a, cc0)), disc1 = __dsub_rn(__dmul_rn(hb1, hb1), __dmul_rn(a, cc1));
    h0 = false; h1 = false;
    if (disc0 >= 0.0 || disc1 >= 0.0) {
        // sqrt/div of a negative discriminant give NaN, which fails every comparison below
        double sq0 = __dsqrt_rn(disc0), sq1 = __dsqrt_rn(disc1);
        double ra0 = __ddiv_rn(__dsub_rn(-hb0, sq0), a), ra1 = __ddiv_rn(__dsub_rn(-hb1, sq1), a);
        double rb0 = __ddiv_rn(__dadd_rn(-hb0, sq0), a), rb1 = __ddiv_rn(__dadd_rn(-hb1, sq1), a);
        if (disc0 >= 0.0) {
            if (ra0 < DBL_MAX && ra0 > t_min) { root0 = ra0; h0 = true; }
            else if (rb0 < DBL_MAX && rb0 > t_min) { root0 = rb0; h0 = true; }
        }
        if (disc1 >= 0.0) {
            if (ra1 < DBL_MAX && ra1 > t_min) { root1 = ra1; h1 = true; }
            else if (rb1 < DBL_MAX && rb1 > t_min) { root1 = rb1; h1 = true; }
        }
    }
}

struct HitRec { D3 point, normal; bool front_face; };
// The rest of sphere.rs:59-76 for the accepted root: p = ray.at(t), normal = (p - c)/r, front-face flip.
RT_DEV HitRec hit_record(D3 center, double radius, D3 o, D3 d, double t) {
    HitRec h;
    h.point = add(o, mul(d, t));                              // ray.rs:18-20
    D3 n = divs(sub(h.point, center), radius);
    h.front_face = dot(d, n) < 0.0;
    h.normal = h.front_face ? n : neg(n);
    return h;
}
// f64::atan2 (sphere.rs:38). Rust forwards to the platform libm, so the last bit of the reference is platform-defined;
// CUDA's atan2 is a third implementation. Texel addresses must not depend on that, so the kernel evaluates one explicit
// algorithm in plain IEEE f64 (every operation rounded to nearest, never contracted): the table-free atan with argument
// reduction at 7/16, 11/16, 19/16, 39/16 and an odd polynomial of degree 23 (< 1 ulp), plus the usual quadrant logic.
// The CPU oracle evaluates the same operations in the same order; tests compare the two bit for bit.
RT_DEV double rt_atan(double x) {
    const uint32_t hx = (uint32_t)__double2hiint(x), ix = hx & 0x7fffffffu;
    const bool negative = (hx >> 31) != 0u;
    if (ix >= 0x44100000u) {                       // |x| >= 2^66, inf or NaN
        if (x != x) return __dadd_rn(x, x);
        const double r = __dadd_rn(1.57079632679489655800e+00, 6.12323399573676603587e-17);
        return negative ? -r : r;
    }
    int id;
    double h = 0.0, l = 0.0;
    if (ix < 0x3fdc0000u) {                        // |x| < 7/16
        if (ix < 0x3e400000u) return x;            // |x| < 2^-27
        id = -1;
    } else {
        x = fabs(x);
        if (ix < 0x3ff30000u) {                    // |x| < 19/16
            if (ix < 0x3fe60000u) { id = 0; h = 4.63647609000806093515e-01; l = 2.26987774529616870924e-17; x = __ddiv_rn(__dsub_rn(__dmul_rn(2.0, x), 1.0), __dadd_rn(2.0, x)); }
            else { id = 1; h = 7.85398163397448278999e-01; l = 3.06161699786838301793e-17; x = __ddiv_rn(__dsub_rn(x, 1.0), __dadd_rn(x, 1.0)); }
        } else if (ix < 0x40038000u) { id = 2; h = 9.82793723247329054082e-01; l = 1.39033110312309984516e-17; x = __ddiv_rn(__dsub_rn(x, 1.5), __dadd_rn(1.0, __dmul_rn(1.5, x))); }   // |x| < 39/16
        else { id = 3; h = 1.57079632679489655800e+00; l = 6.12323399573676603587e-17; x = __ddiv_rn(-1.0, x); }
    }
    const double z = __dmul_rn(x, x), w = __dmul_rn(z, z);
    double s1 = __dmul_rn(w, 1.62858201153657823623e-02);
    s1 = __dmul_rn(w, __dadd_rn(4.97687799461593236017e-02, s1));
    s1 = __dmul_rn(w, __dadd_rn(6.66107313738753120669e-02, s1));
    s1 = __dmul_rn(w, __dadd_rn(9.09088713343650656196e-02, s1));
    s1 = __dmul_rn(w, __dadd_rn(1.42857142725034663711e-01, s1));
    s1 = __dmul_rn(z, __dadd_rn(3.33333333333329318027e-01, s1));
    double s2 = __dmul_rn(w, -3.65315727442169155270e-02);
    s2 = __dmul_rn(w, __dadd_rn(-5.83357013379057348645e-02, s2));
    s2 = __dmul_rn(w, __dadd_rn(-7.69187620504482999495e-02, s2));
    s2 = __dmul_rn(w, __dadd_rn(-1.11111104054623557880e-01, s2));
    s2 = __dmul_rn(w, __dadd_rn(-1.99999999998764832476e-01, s2));
    const double xs = __dmul_rn(x, __dadd_rn(s1, s2));
    if (id < 0) return __dsub_rn(x, xs);
    const double r = __dsub_rn(h, __dsub_rn(__dsub_rn(xs, l), x));
    return negative ? -r : r;
}
RT_DEV double rt_atan2(double y, double x) {
    const double PI_HI = 3.1415926535897931160e+00, PI_LO = 1.2246467991473531772e-16, TINY = 1.0e-300;
    if (x != x || y != y) return __dadd_rn(x, y);
    const uint32_t hx = (uint32_t)__double2hiint(x), hy = (uint32_t)__double2hiint(y), ix = hx & 0x7fffffffu, iy = hy & 0x7fffffffu;
    if (x == 1.0) return rt_atan(y);
    const int m = (int)((hy >> 31) & 1u) | (int)((hx >> 30) & 2u);   // 2*sign(x) + sign(y)
    if ((iy | (uint32_t)__double2loint(y)) == 0u) {                 // y = +-0
        if (m < 2) return y;
        return m == 2 ? __dadd_rn(PI_HI, TINY) : __dsub_rn(-PI_HI, TINY);
    }
    const double half_pi = __ddiv_rn(PI_HI, 2.0);
    if ((ix | (uint32_t)__double2loint(x)) == 0u) return (hy >> 31) ? __dsub_rn(-half_pi, TINY) : __dadd_rn(half_pi, TINY);
    if (ix == 0x7ff00000u) {                       // x = +-inf
        const double q = __ddiv_rn(PI_HI, 4.0);
        if (iy == 0x7ff00000u) {
            if (m == 0) return __dadd_rn(q, TINY);
            if (m == 1) return __dsub_rn(-q, TINY);
            if (m == 2) return __dadd_rn(__dmul_rn(3.0, q), TINY);
            return __dsub_rn(__dmul_rn(-3.0, q), TINY);
        }
        if (m == 0) return 0.0;
        if (m == 1) return -0.0;
        return m == 2 ? __dadd_rn(PI_HI, TINY) : __dsub_rn(-PI_HI, TINY);
    }
    if (iy == 0x7ff00000u) return (hy >> 31) ? __dsub_rn(-half_pi, TINY) : __dadd_rn(half_pi, TINY);
    const int k = ((int)iy - (int)ix) >> 20;       // exponent difference
    double z;
    int mm = m;
    if (k > 60) { z = __dadd_rn(half_pi, __dmul_rn(0.5, PI_LO)); mm &= 1; }
    else if ((hx >> 31) && k < -60) z = 0.0;
    else z = rt_atan(fabs(__ddiv_rn(y, x)));
    if (mm == 0) return z;
    if (mm == 1) return -z;
    if (mm == 2) return __dsub_rn(PI_HI, __dsub_rn(z, PI_LO));
    return __dsub_rn(__dsub_rn(z, PI_LO), PI_HI);
}
// sphere.rs:35-43 (evaluated lazily: only Texture materials read u,v)
RT_DEV void sphere_uv(D3 hp, double& u, double& v) {
    const double PI = 3.14159265358979323846264338327950288;
    D3 n = unit_vector(hp);
    u = __dadd_rn(__ddiv_rn(rt_atan2(n.x, n.z), __dmul_rn(2.0, PI)), 0.5);
    v = __dadd_rn(__dmul_rn(n.y, 0.5), 0.5);
}

// ---- materials.rs ------------------------------------------------------------------------------------
RT_DEV D3 reflect(D3 v, D3 n) { return sub(v, mul(n, __dmul_rn(2.0, dot(v, n)))); }                          // :111-113
RT_DEV D3 refract(D3 uv, D3 n, double eta) {                                                                  // :144-149
    double cos_theta = fmin(dot(neg(uv), n), 1.0);
    D3 perp = mul(add(uv, mul(n, cos_theta)), eta);
    D3 par = mul(n, __dmul_rn(-1.0, __dsqrt_rn(fabs(__dsub_rn(1.0, length_squared(perp))))));
    return add(perp, par);
}
RT_DEV double reflectance(double cosine, double ref_idx) {                                                    // :151-155
    double r0 = __ddiv_rn(__dsub_rn(1.0, ref_idx), __dadd_rn(1.0, ref_idx));
    r0 = __dmul_rn(r0, r0);
    double x = __dsub_rn(1.0, cosine);
    double x2 = __dmul_rn(x, x), x4 = __dmul_rn(x2, x2);
    double x5 = __dmul_rn(x, x4);                      // f64::powi(5)
    return __dadd_rn(r0, __dmul_rn(__dsub_rn(1.0, r0), x5));
}

RT_DEV float clampf(float v) { return v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v); }                              // raytracer.rs:61-69

struct DevTex { const uint8_t* rgb8; unsigned long long width, height; };

RT_DEV unsigned long long f64_as_u64_sat(double x) {   // Rust `as u64`
    if (!(x > 0.0)) return 0ull;
    if (x >= 18446744073709551616.0) return ~0ull;
    return (unsigned long long)x;
}
RT_DEV unsigned long long f32_as_u64_sat(float x) {    // Rust `as usize`
    if (!(x > 0.0f)) return 0ull;
    if (x >= 18446744073709551616.0f) return ~0ull;
    return (unsigned long long)x;
}

// Texture::get_albedo (materials.rs:236-253) -> packed 0x00BBGGRR texel
RT_DEV uint32_t texture_texel(const DevTex& t, double h_offset, double u, double v) {
    double rot = __dadd_rn(u, h_offset);
    if (rot > 1.0) rot = __dsub_rn(rot, 1.0);
    double uu = __dmul_rn(rot, (double)t.width);
    double vv = __dmul_rn(__dsub_rn(1.0, v), (double)(t.height - 1ull));
    unsigned long long base = 3ull * (f64_as_u64_sat(floor(vv)) * t.width + f64_as_u64_sat(floor(uu)));
    unsigned long long limit = t.width * t.height * 3ull;
    if (base + 2ull >= limit) base = limit - 3ull;     // the reference panics here; clamp like the oracle
    const uint8_t* px = t.rgb8 + base;
    return (uint32_t)px[0] | ((uint32_t)px[1] << 8) | ((uint32_t)px[2] << 16);
}

// Miss branch of ray_color (raytracer.rs:134-163)
// `l` = dir.length() (the caller shares it with Glass lanes)
RT_DEV void sky_color(D3 dir, double l, uint32_t sky_mode, const DevTex& sky, float& r, float& g, float& b) {
    if (sky_mode == RT_SKY_NONE) { r = 0.0f; g = 0.0f; b = 0.0f; return; }
    float t = clampf(__fmul_rn(0.5f, __fadd_rn(__double2float_rn(__ddiv_rn(dir.y, l)), 1.0f)));
    if (sky_mode == RT_SKY_GRADIENT) {
        float omt = __fmul_rn(__fsub_rn(1.0f, t), 1.0f);
        r = __fadd_rn(omt, __fmul_rn(t, 0.5f));
        g = __fadd_rn(omt, __fmul_rn(t, 0.7f));
        b = __fadd_rn(omt, __fmul_rn(t, 1.0f));
        return;
    }
    float u = clampf(__fmul_rn(0.5f, __fadd_rn(__double2float_rn(__ddiv_rn(dir.x, l)), 1.0f)));
    unsigned long long x = f32_as_u64_sat(__fmul_rn(u, (float)(sky.width - 1ull)));
    unsigned long long y = f32_as_u64_sat(__fmul_rn(__fsub_rn(1.0f, t), (float)(sky.height - 1ull)));
    const uint8_t* px = sky.rgb8 + (y * sky.width + x) * 3ull;
    r = __fdiv_rn(__fmul_rn(0.7f, (float)px[0]), 255.0f);
    g = __fdiv_rn(__fmul_rn(0.7f, (float)px[1]), 255.0f);
    b = __fdiv_rn(__fmul_rn(0.7f, (float)px[2]), 255.0f);
}

// raytracer.rs:207-213: sqrt(mean) -> palette 0.6 into_format::<u8>() (min(x*255,255) + 2^23 trick)
RT_DEV uint8_t quantise_u8(float mean_linear) {
    float c = __fsqrt_rn(mean_linear);
    float scaled = fminf(__fmul_rn(c, 255.0f), 255.0f);
    float f = __fadd_rn(scaled, 8388608.0f);
    uint32_t bits = __float_as_uint(f);
    const uint32_t C23 = 0x4B000000u;
    uint32_t d = bits >= C23 ? bits - C23 : 0u;
    return (uint8_t)d;
}

// ---- async-proxy helpers: 1-D TMA bulk copy global -> shared with mbarrier completion ---------------
RT_DEV uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
RT_DEV void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
RT_DEV void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
RT_DEV void tma_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
RT_DEV void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

}  // namespace rtd
