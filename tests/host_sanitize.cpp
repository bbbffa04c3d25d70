// Host-side robustness harness, built with -fsanitize=address,undefined by tests/test_host_sanitizers.py (no GPU, no CUDA).
// Exercises the three pieces of host code that consume untrusted or awkward input on the way to the render call:
//   1. the hierarchy builder (csrc/rtb200_bvh.hpp) on degenerate scenes, checking every index it emits and its level order;
//   2. the baseline JPEG decoder (host/jpeg_decode.cpp) on mutated / truncated files;
//   3. the scene reader (host/scene_json.cpp + json.hpp) on mutated / truncated / deeply nested JSON.
// Exit code 0 and the line "host_sanitize: ok" = no sanitizer report, no escaped exception, no out-of-range index.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <limits>
#include <random>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../rust-raytracer_b200/csrc/rtb200_bvh.hpp"
#include "../rust-raytracer_b200/host/jpeg_decode.hpp"
#include "../rust-raytracer_b200/host/scene_json.hpp"

// scene_json.cpp calls two entry points of librtb200.so (camera set-up lives next to the render path); the harness links
// without CUDA, so they are stubbed: the camera values are irrelevant to what is being checked here.
extern "C" int rtb200_camera_from_params(const rt_camera_params*, rt_camera* out) { std::memset(out, 0, sizeof *out); return RT_OK; }
extern "C" const char* rtb200_last_error(void) { return ""; }

static int g_fail = 0;
#define REQUIRE(c, ...) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); std::fprintf(stderr, __VA_ARGS__); std::fprintf(stderr, "\n"); ++g_fail; } } while (0)

static std::string slurp(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error("cannot open " + path);
    std::stringstream ss; ss << f.rdbuf();
    return ss.str();
}

// ---- 1. hierarchy builder ---------------------------------------------------------------------------
static void check_records(const char* what, const std::vector<rt_sphere>& sph, bool want_tree) {
    rt_scene s{};
    s.width = 4; s.height = 4; s.samples_per_pixel = 1; s.max_depth = 2;
    s.spheres = sph.empty() ? nullptr : sph.data(); s.n_spheres = sph.size();
    rtbvh::Records R;
    rtbvh::build_records(&s, want_tree, R);
    const uint32_t n = (uint32_t)sph.size();
    REQUIRE(R.geo.size() >= (size_t)n * 4 || n == 0, "%s: geo too small", what);
    if (!want_tree) return;
    REQUIRE(R.nodes.size() == (size_t)R.n_nodes * rtbvh::kNodeFloats, "%s: node array size", what);
    REQUIRE(R.leaf_id.size() == (size_t)R.n_leaves * rtbvh::kLeafK, "%s: leaf id array size", what);
    REQUIRE(R.leaf_rec.size() == (size_t)R.n_leaves * rtbvh::kLeafK * 4, "%s: leaf record array size", what);
    REQUIRE(R.depth <= (uint32_t)rtbvh::kMaxDepth, "%s: depth %u", what, R.depth);
    std::vector<uint8_t> seen(n, 0), leaf_seen(R.n_leaves, 0), node_seen(R.n_nodes, 0);
    for (uint32_t a : R.always) { REQUIRE(a < n, "%s: always index", what); if (a < n) { REQUIRE(!seen[a], "%s: sphere twice", what); seen[a] = 1; } }
    // level order: every node once, in groups (deepest level first) that match the depth
    const size_t n_groups = R.level_off.empty() ? 0 : R.level_off.size() - 1;
    REQUIRE(n_groups == R.depth, "%s: %zu level groups for depth %u", what, n_groups, R.depth);
    REQUIRE(R.level_nodes.size() == R.n_nodes && (R.level_off.empty() ? R.n_nodes == 0 : R.level_off.front() == 0 && R.level_off.back() == R.n_nodes),
            "%s: level order size", what);
    std::vector<uint32_t> group(R.n_nodes, ~0u);
    for (size_t g = 0; g < n_groups; ++g) {
        REQUIRE(R.level_off[g] < R.level_off[g + 1], "%s: empty level group %zu", what, g);
        for (uint32_t t = R.level_off[g]; t < R.level_off[g + 1] && t < R.level_nodes.size(); ++t) {
            const uint32_t v = R.level_nodes[t];
            REQUIRE(v < R.n_nodes, "%s: level order node %u of %u", what, v, R.n_nodes);
            if (v < R.n_nodes) { REQUIRE(group[v] == ~0u, "%s: node %u twice in the level order", what, v); group[v] = (uint32_t)g; }
        }
    }
    if (R.n_nodes) node_seen[0] = 1;
    for (uint32_t k = 0; k < R.n_nodes; ++k) {
        for (int i = 0; i < rtbvh::kWide; ++i) {
            const uint32_t ref = rtbvh::child_of(&R.nodes[(size_t)k * rtbvh::kNodeFloats], i);
            if (ref == rtbvh::kEmptyChild) continue;
            if (ref & rtbvh::kLeafBit) {
                const uint32_t l = ref & ~rtbvh::kLeafBit;
                REQUIRE(l < R.n_leaves, "%s: leaf reference %u of %u", what, l, R.n_leaves);
                if (l < R.n_leaves) { REQUIRE(!leaf_seen[l], "%s: leaf referenced twice", what); leaf_seen[l] = 1; }
            } else {
                REQUIRE(ref < R.n_nodes && ref > k, "%s: node reference %u from %u of %u", what, ref, k, R.n_nodes);
                if (ref < R.n_nodes) {
                    REQUIRE(!node_seen[ref], "%s: node referenced twice", what); node_seen[ref] = 1;
                    REQUIRE(group[ref] < group[k], "%s: node %u is not in a deeper level than its parent %u", what, ref, k);
                }
            }
        }
    }
    for (uint32_t k = 0; k < R.n_nodes; ++k) REQUIRE(node_seen[k], "%s: node %u unreachable", what, k);
    for (uint32_t l = 0; l < R.n_leaves; ++l) {
        REQUIRE(leaf_seen[l], "%s: leaf %u unreachable", what, l);
        for (int j = 0; j < rtbvh::kLeafK; ++j) {
            const uint32_t id = R.leaf_id[(size_t)l * rtbvh::kLeafK + j];
            if (id >= n) continue;   // padding slot
            REQUIRE(!seen[id], "%s: sphere %u twice", what, id); seen[id] = 1;
        }
    }
    for (uint32_t i = 0; i < n; ++i) REQUIRE(seen[i], "%s: sphere %u lost", what, i);
}

static rt_sphere sphere_at(double x, double y, double z, double r) {
    rt_sphere sp{}; sp.center = rt_vec3{x, y, z}; sp.radius = r; sp.kind = RT_LAMBERTIAN; sp.albedo[0] = sp.albedo[1] = sp.albedo[2] = 0.5f; sp.texture = -1;
    return sp;
}

static void builder_cases() {
    std::mt19937_64 rng(7);
    std::uniform_real_distribution<double> U(-1.0, 1.0);
    const double inf = std::numeric_limits<double>::infinity(), nan = std::numeric_limits<double>::quiet_NaN();
    for (uint32_t n : {0u, 1u, 2u, 7u, 8u, 9u, 63u, 64u, 65u, 511u, 4097u, 30000u}) {
        std::vector<rt_sphere> v;
        for (uint32_t i = 0; i < n; ++i) v.push_back(sphere_at(50 * U(rng), U(rng), 50 * U(rng), 0.2 + 0.2 * U(rng)));   // radii of both signs and near 0
        check_records("random", v, true);
        check_records("random flat", v, false);
    }
    { std::vector<rt_sphere> v(3000, sphere_at(1, 2, 3, 0.5)); check_records("coincident", v, true); }
    { std::vector<rt_sphere> v; for (int i = 0; i < 5000; ++i) v.push_back(sphere_at(i * 1e-3, 0, 0, 0.0)); check_records("collinear zero radius", v, true); }
    { std::vector<rt_sphere> v; for (int i = 0; i < 2000; ++i) v.push_back(sphere_at(std::ldexp(1.0, i % 60), 0, -std::ldexp(1.0, (i * 7) % 60), 1.0)); check_records("geometric spread", v, true); }
    { std::vector<rt_sphere> v; for (int i = 0; i < 4000; ++i) v.push_back(sphere_at(i < 3999 ? 1e-9 * i : 1e9, 0, 0, 1e-3)); check_records("one outlier", v, true); }
    {
        std::vector<rt_sphere> v;
        for (int i = 0; i < 100; ++i) v.push_back(sphere_at(U(rng), U(rng), U(rng), 0.1));
        v.push_back(sphere_at(nan, 0, 0, 1)); v.push_back(sphere_at(0, inf, 0, 1)); v.push_back(sphere_at(0, 0, -inf, 1));
        v.push_back(sphere_at(0, 0, 0, nan)); v.push_back(sphere_at(0, 0, 0, inf)); v.push_back(sphere_at(3e15, 0, 0, 1));
        v.push_back(sphere_at(1e300, -1e300, 1e300, 1e300)); v.push_back(sphere_at(0, 0, 0, -inf));
        check_records("non-finite", v, true);
        check_records("non-finite flat", v, false);
    }
    { std::vector<rt_sphere> v; for (int i = 0; i < 9; ++i) v.push_back(sphere_at(nan, nan, nan, nan)); check_records("all non-finite", v, true); }
    { std::vector<rt_sphere> v; for (int i = 0; i < 1000; ++i) v.push_back(sphere_at(7e6 + U(rng), -7e6 + U(rng), 7e6 + U(rng), 1e-3)); check_records("far from origin", v, true); }
    { std::vector<rt_sphere> v; for (int i = 0; i < 600; ++i) v.push_back(sphere_at(0, 0, 0, 1.0 + i)); check_records("concentric", v, true); }
}

// ---- 2. JPEG decoder --------------------------------------------------------------------------------
// `small_dir` holds small JPEGs written by the calling test (baseline 4:4:4 / 4:2:2 / 4:2:0 / grey, restart intervals,
// a progressive one the decoder must refuse): every one is mutated 400 times and truncated at every length.
static void jpeg_cases(const std::string& repo, const std::vector<std::string>& small) {
    std::mt19937 rng(11);
    for (const char* name : {"moon.jpg", "earth.jpg", "beach.jpg"}) {   // the reference's textures, as they are
        const std::string file = slurp(repo + "/scenes/data/" + name);
        rthost::Image img; std::string err;
        const bool ok = rthost::decode_jpeg((const uint8_t*)file.data(), file.size(), &img, &err);
        REQUIRE(ok && img.width > 0 && img.height > 0 && img.rgb.size() == (size_t)img.width * img.height * 3, "%s does not decode: %s", name, err.c_str());
    }
    int decoded = 0, refused = 0;
    for (const std::string& path : small) {
        const std::string file = slurp(path);
        {
            rthost::Image o; std::string e;
            if (rthost::decode_jpeg((const uint8_t*)file.data(), file.size(), &o, &e)) REQUIRE(o.rgb.size() == (size_t)o.width * o.height * 3, "%s: size", path.c_str());
        }
        for (int it = 0; it < 400; ++it) {
            std::string m = file;
            const int flips = 1 + (int)(rng() % 4);
            // two thirds of the edits land in the header area (markers, tables, frame / scan headers), the rest in the entropy-coded data
            for (int f = 0; f < flips; ++f) { const size_t span = (rng() % 3) ? std::min<size_t>(m.size(), 700) : m.size(); m[rng() % span] = (char)(rng() & 0xff); }
            rthost::Image o; std::string e;
            const bool ok = rthost::decode_jpeg((const uint8_t*)m.data(), m.size(), &o, &e);   // may fail; must stay in bounds
            ok ? ++decoded : ++refused;
            if (ok) REQUIRE(o.width > 0 && o.height > 0 && o.rgb.size() == (size_t)o.width * o.height * 3, "inconsistent image after mutation");
        }
        for (size_t cut = 0; cut < file.size(); ++cut) {
            // a heap copy of exactly `cut` bytes: reading one byte past the end is an ASan report
            std::vector<uint8_t> part(file.begin(), file.begin() + (long)cut);
            rthost::Image o; std::string e;
            (void)rthost::decode_jpeg(part.data(), part.size(), &o, &e);
        }
    }
    std::printf("jpeg: %zu small files; %d mutated files decoded, %d refused\n", small.size(), decoded, refused);
    rthost::Image o; std::string e;
    REQUIRE(!rthost::decode_jpeg(nullptr, 0, &o, &e), "empty input must fail");
}

// ---- 3. scene reader --------------------------------------------------------------------------------
static void json_cases() {
    const std::string good =
        "{\"width\":8,\"height\":6,\"samples_per_pixel\":2,\"max_depth\":5,\"sky\":{\"texture\":\"\"},"
        "\"camera\":{\"look_from\":{\"x\":1,\"y\":2,\"z\":3},\"look_at\":{\"x\":0,\"y\":0,\"z\":0},\"vup\":{\"x\":0,\"y\":1,\"z\":0},\"vfov\":30.0,\"aspect\":1.5},"
        "\"objects\":[{\"center\":{\"x\":0,\"y\":0,\"z\":-1},\"radius\":0.5,\"material\":{\"Lambertian\":{\"albedo\":[0.1,0.2,0.3]}}},"
        "{\"center\":{\"x\":1,\"y\":0,\"z\":-1},\"radius\":-0.4,\"material\":{\"Glass\":{\"index_of_refraction\":1.5}}},"
        "{\"center\":{\"x\":-1,\"y\":0,\"z\":-1},\"radius\":0.5,\"material\":{\"Metal\":{\"albedo\":[0.8,0.6,0.2],\"fuzz\":0.1}}},"
        "{\"center\":{\"x\":0,\"y\":3,\"z\":0},\"radius\":0.5,\"material\":{\"Light\":{}}}]}";
    {
        rthost::SceneHolder h;
        try { rthost::load_scene_json(good, "", &h); } catch (const std::exception& e) { REQUIRE(false, "good scene rejected: %s", e.what()); }
        REQUIRE(h.scene.n_spheres == 4 && h.scene.width == 8 && h.scene.height == 6, "good scene misread");
    }
    std::mt19937 rng(13);
    const char alphabet[] = "{}[]\":,0123456789.-eE+ \\ntrufalsx";
    int accepted = 0;
    for (int it = 0; it < 4000; ++it) {
        std::string m = good;
        const int edits = 1 + (int)(rng() % 3);
        for (int k = 0; k < edits; ++k) {
            const size_t at = rng() % m.size();
            switch (rng() % 4) {
                case 0: m[at] = alphabet[rng() % (sizeof alphabet - 1)]; break;
                case 1: m.erase(at, 1 + rng() % 8); break;
                case 2: m.insert(at, 1, alphabet[rng() % (sizeof alphabet - 1)]); break;
                default: m.resize(at); break;
            }
            if (m.empty()) m = "{";
        }
        rthost::SceneHolder h;
        try {
            rthost::load_scene_json(m, "", &h);
            ++accepted;
            REQUIRE(h.scene.spheres == (h.spheres.empty() ? h.scene.spheres : h.spheres.data()) && h.scene.n_spheres == h.spheres.size(), "holder inconsistent");
        } catch (const std::exception&) { /* rejected with a message: fine */ }
    }
    std::printf("json: %d of 4000 mutated scenes still parse\n", accepted);
    for (const std::string& deep : {std::string(200000, '['), std::string(200000, '{'), "{\"objects\":" + std::string(100000, '[')}) {
        rthost::SceneHolder h;
        bool threw = false;
        try { rthost::load_scene_json(deep, "", &h); } catch (const std::exception&) { threw = true; }
        REQUIRE(threw, "deeply nested input must be rejected");
    }
    for (const char* bad : {"", " ", "null", "[]", "{}", "{\"width\":-1}", "{\"width\":1e999}", "{\"width\":\"8\"}", "\"", "{\"a\":\"\\u12\"}", "{\"a\":\"\\"}) {
        rthost::SceneHolder h;
        bool threw = false;
        try { rthost::load_scene_json(bad, "", &h); } catch (const std::exception&) { threw = true; }
        REQUIRE(threw, "`%s` must be rejected", bad);
    }
}

int main(int argc, char** argv) {
    const std::string repo = argc > 1 ? argv[1] : ".";
    std::vector<std::string> small;
    for (int i = 2; i < argc; ++i) small.push_back(argv[i]);
    try {
        auto t0 = std::chrono::steady_clock::now();
        auto lap = [&](const char* what) { auto t1 = std::chrono::steady_clock::now(); std::printf("%s: %.1f s\n", what, std::chrono::duration<double>(t1 - t0).count()); t0 = t1; };
        builder_cases(); lap("hierarchy builder");
        jpeg_cases(repo, small); lap("jpeg decoder");
        json_cases(); lap("scene reader");
    } catch (const std::exception& e) {
        std::fprintf(stderr, "FAIL: escaped exception: %s\n", e.what());
        return 2;
    }
    if (g_fail) { std::fprintf(stderr, "host_sanitize: %d failure(s)\n", g_fail); return 1; }
    std::printf("host_sanitize: ok\n");
    return 0;
}
