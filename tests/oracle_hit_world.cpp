// oracle_hit_world.cpp — the CPU oracle's hit_world (oracle/rt_oracle.hpp, raytracer.rs:44-59) on caller-supplied rays: the
// reference answer of rtb200_scene_intersect[_device] (include/rtb200.h). Test infrastructure, built beside the tests by
// tests/oracle_hit_world.py (and __graft_entry__.build()) with the oracle's own flags; the oracle's sources are only included.
#include <cfloat>

#include "../oracle/rt_oracle.hpp"

using namespace rto;

extern "C" {

// For ray i: hit_world(scene, Ray{origin[3i..], direction[3i..]}, 0.001, t_max_i) with t_max_i = t_max[i] (DBL_MAX when t_max
// is NULL; a bound above DBL_MAX counts as DBL_MAX, as the query contract says). A miss writes sphere 0xffffffff, t = +inf,
// zeros and front_face 0. Every output may be NULL. OpenMP over rays.
int oracle_hit_world(const rt_scene* s, const double* origin, const double* direction, const double* t_max, uint32_t n,
                     double* t, uint32_t* sphere, double* point, double* normal, double* uv, uint8_t* front_face) {
    if (!s || (n && (!origin || !direction))) return -1;
    const Scene sc(s);
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t k = 0; k < (int64_t)n; ++k) {
        const size_t i = (size_t)k;
        double tm = t_max ? t_max[i] : DBL_MAX;
        if (tm > DBL_MAX) tm = DBL_MAX;
        const Ray r{P3{origin[3 * i], origin[3 * i + 1], origin[3 * i + 2]}, P3{direction[3 * i], direction[3 * i + 1], direction[3 * i + 2]}};
        Stats st;
        Hit h{};
        const bool hit = hit_world(sc, r, 0.001, tm, &h, st);
        if (!hit) { h = Hit{}; h.t = INFINITY; h.sphere = -1; }
        if (t) t[i] = h.t;
        if (sphere) sphere[i] = hit ? (uint32_t)h.sphere : 0xffffffffu;
        if (point) { point[3 * i] = h.point.x; point[3 * i + 1] = h.point.y; point[3 * i + 2] = h.point.z; }
        if (normal) { normal[3 * i] = h.normal.x; normal[3 * i + 1] = h.normal.y; normal[3 * i + 2] = h.normal.z; }
        if (uv) { uv[2 * i] = h.u; uv[2 * i + 1] = h.v; }
        if (front_face) front_face[i] = hit && h.front_face ? 1u : 0u;
    }
    return 0;
}

}  // extern "C"
