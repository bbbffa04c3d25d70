#include "scene_json.hpp"

#include <cfloat>
#include <cmath>
#include <fstream>
#include <stdexcept>

#include "json.hpp"

namespace rthost {
namespace {
rt_vec3 vec3(const Json& j) { return rt_vec3{j.at("x").number(), j.at("y").number(), j.at("z").number()}; }   // point3d.rs:10-15
// Rust `as f32`: round to nearest, +-inf from the halfway point 0x1.ffffffp127 above FLT_MAX on. A plain (float) cast of a
// value beyond FLT_MAX is undefined behaviour in C++.
float f64_as_f32(double x) {
    if (std::fabs(x) >= 0x1.ffffffp127) return x > 0.0 ? INFINITY : -INFINITY;
    if (std::fabs(x) > FLT_MAX) return x > 0.0 ? FLT_MAX : -FLT_MAX;
    return (float)x;
}
void albedo(const Json& j, float out[3]) {                                                                  // SrgbAsArray, materials.rs:18-25
    if (j.kind != Json::Arr || j.arr.size() != 3) throw std::runtime_error("albedo: array of 3 numbers expected");
    for (int i = 0; i < 3; ++i) out[i] = f64_as_f32(j.arr[i].number());
}
// serde parses width/height/max_depth as usize and samples_per_pixel as u32 (config.rs:68-71): negative, fractional or
// out-of-range numbers are parse errors there; casting them blindly would be undefined behaviour here.
uint64_t uint_field(const Json& j, const char* name, double max_value) {
    const double v = j.number();
    if (!(v >= 0.0) || v > max_value || v != (double)(uint64_t)v) throw std::runtime_error(std::string(name) + ": non-negative integer expected");
    return (uint64_t)v;
}
// |look_from - look_at| (camera.rs:68, the reference's unused focal_length): the focus distance when none is given
double focal_length(const rt_camera_params& p) {
    const double dx = p.look_from.x - p.look_at.x, dy = p.look_from.y - p.look_at.y, dz = p.look_from.z - p.look_at.z;
    return std::sqrt(dx * dx + dy * dy + dz * dz);
}
// The lens of a camera: aperture finite and >= 0 (0: none); with a lens, focus_dist (has_focus false: focal_length) finite, > 0
LensSpec lens_spec(const rt_camera_params& p, double aperture, bool has_focus, double focus_dist, const std::string& what) {
    if (!std::isfinite(aperture) || aperture < 0.0) throw std::runtime_error(what + ": aperture must be finite and >= 0");
    LensSpec l{p, aperture, has_focus ? focus_dist : focal_length(p)};
    if (aperture != 0.0 && !(std::isfinite(l.focus_dist) && l.focus_dist > 0.0))
        throw std::runtime_error(what + ": focus_dist must be finite and > 0");
    return l;
}
bool load_image(const std::string& path, const std::string& base_dir, Image* img) {
    std::string err;
    if (decode_jpeg_file(path, img, &err)) return true;
    if (!base_dir.empty() && decode_jpeg_file(base_dir + "/" + path, img, &err)) return true;
    throw std::runtime_error(path + ": " + err);   // the reference panics with the path (materials.rs:214)
}
}  // namespace

void load_scene_json(const std::string& text, const std::string& base_dir, SceneHolder* out) {
    Json root = JsonParser::parse(text);
    if (root.kind != Json::Obj) throw std::runtime_error("Unable to parse config json: object expected");
    rt_scene& s = out->scene;
    s.width = (uint32_t)uint_field(root.at("width"), "width", 4294967295.0); s.height = (uint32_t)uint_field(root.at("height"), "height", 4294967295.0);
    s.samples_per_pixel = (uint32_t)uint_field(root.at("samples_per_pixel"), "samples_per_pixel", 4294967295.0);
    s.max_depth = (uint32_t)uint_field(root.at("max_depth"), "max_depth", 4294967295.0);
    s.seed = 0x5EED;
    // camera: CameraParams -> Camera::new (camera.rs:29-42)
    const Json& cam = root.at("camera");
    rt_camera_params cp{vec3(cam.at("look_from")), vec3(cam.at("look_at")), vec3(cam.at("vup")), cam.at("vfov").number(), cam.at("aspect").number()};
    // the optional thin lens (DESIGN.md §4.17): "aperture" (absent or 0: Camera::new, no lens) and "focus_dist"
    if (rtb200_camera_from_params(&cp, &s.camera) != 0) throw std::runtime_error(rtb200_last_error());
    const Json* ap = cam.find("aperture");
    const Json* fd = cam.find("focus_dist");
    out->has_focus = fd != nullptr;
    out->lens_spec = lens_spec(cp, ap ? ap->number() : 0.0, fd != nullptr, fd ? fd->number() : 0.0, "camera");
    // sky: missing or null -> None (black); {"texture": ""} -> gradient; path -> texture (config.rs:49-64)
    s.sky.mode = RT_SKY_NONE;
    if (const Json* sky = root.find("sky")) {
        if (sky->kind == Json::Obj) {
            const std::string& t = sky->at("texture").string();
            if (t.empty()) s.sky.mode = RT_SKY_GRADIENT;
            else {
                load_image(t, base_dir, &out->sky_image);
                s.sky.mode = RT_SKY_TEXTURE;
                s.sky.tex = rt_image{out->sky_image.rgb.data(), (uint64_t)out->sky_image.width, (uint64_t)out->sky_image.height, (uint64_t)out->sky_image.rgb.size()};
            }
        } else if (sky->kind != Json::Null) throw std::runtime_error("sky: object or null expected");
    }
    const Json& objs = root.at("objects");
    if (objs.kind != Json::Arr) throw std::runtime_error("objects: array expected");
    out->spheres.resize(objs.arr.size());
    out->images.reserve(objs.arr.size());
    std::vector<std::pair<uint64_t, uint64_t>> dims;
    for (size_t i = 0; i < objs.arr.size(); ++i) {
        const Json& o = objs.arr[i];
        rt_sphere& sp = out->spheres[i];
        sp = rt_sphere{};
        sp.center = vec3(o.at("center")); sp.radius = o.at("radius").number(); sp.texture = -1;
        const Json& m = o.at("material");
        if (m.kind != Json::Obj || m.obj.size() != 1) throw std::runtime_error("material: externally tagged enum expected (materials.rs:35-42)");
        const std::string& tag = m.obj[0].first; const Json& b = m.obj[0].second;
        if (tag == "Lambertian") { sp.kind = RT_LAMBERTIAN; albedo(b.at("albedo"), sp.albedo); }
        else if (tag == "Metal") { sp.kind = RT_METAL; albedo(b.at("albedo"), sp.albedo); sp.param = b.at("fuzz").number(); }
        else if (tag == "Glass") { sp.kind = RT_GLASS; sp.param = b.at("index_of_refraction").number(); }
        else if (tag == "Light") { sp.kind = RT_LIGHT; }
        else if (tag == "Texture") {
            sp.kind = RT_TEXTURE; albedo(b.at("albedo"), sp.albedo); sp.param = b.at("h_offset").number();
            out->images.emplace_back();
            load_image(b.at("pixels").string(), base_dir, &out->images.back());
            const uint64_t w = uint_field(b.at("width"), "texture width", 9007199254740992.0), h = uint_field(b.at("height"), "texture height", 9007199254740992.0);   // JSON dims (materials.rs:208-209)
            const uint64_t texels = out->images.back().rgb.size() / 3;
            if (w == 0 || h == 0 || w > texels || h > texels / w) throw std::runtime_error("texture: JSON width/height exceed the decoded image");   // overflow-safe w*h*3 <= size
            dims.emplace_back(w, h);
            sp.texture = (int32_t)out->images.size() - 1;
        } else throw std::runtime_error("unknown variant `" + tag + "`, expected one of `Lambertian`, `Metal`, `Glass`, `Texture`, `Light`");
    }
    out->textures.resize(out->images.size());
    for (size_t t = 0; t < out->images.size(); ++t) out->textures[t] = rt_image{out->images[t].rgb.data(), dims[t].first, dims[t].second, (uint64_t)out->images[t].rgb.size()};
    s.spheres = out->spheres.data(); s.n_spheres = out->spheres.size();
    s.textures = out->textures.data(); s.n_textures = out->textures.size();
}

std::vector<rt_frame> load_frames_json(const std::string& text, const rt_scene& scene) {
    SceneHolder h;
    h.scene = scene;
    std::vector<LensSpec> lenses;
    return load_frames_json(text, h, &lenses);
}

std::vector<rt_frame> load_frames_json(const std::string& text, const SceneHolder& holder, std::vector<LensSpec>* lenses) {
    const rt_scene& scene = holder.scene;
    Json root = JsonParser::parse(text);
    if (root.kind != Json::Arr) throw std::runtime_error("frames: array expected");
    if (root.arr.empty()) throw std::runtime_error("frames: at least one frame expected");
    if (root.arr.size() > 0xffffffffull) throw std::runtime_error("frames: too many frames");
    std::vector<rt_frame> frames(root.arr.size());
    lenses->assign(root.arr.size(), LensSpec{});
    for (size_t i = 0; i < root.arr.size(); ++i) {
        const Json& f = root.arr[i];
        if (f.kind != Json::Obj) throw std::runtime_error("frame " + std::to_string(i) + ": object expected");
        rt_frame& fr = frames[i];
        fr = rt_frame{};
        const Json& cam = f.at("camera");   // the config's camera schema (camera.rs:29-36)
        rt_camera_params cp{vec3(cam.at("look_from")), vec3(cam.at("look_at")), vec3(cam.at("vup")), cam.at("vfov").number(), cam.at("aspect").number()};
        if (rtb200_camera_from_params(&cp, &fr.camera) != 0) throw std::runtime_error("frame " + std::to_string(i) + ": invalid camera");
        const Json* a = cam.find("aperture");
        const Json* fd = cam.find("focus_dist");
        (*lenses)[i] = lens_spec(cp, a ? a->number() : holder.lens_spec.aperture, fd || holder.has_focus,
                                 fd ? fd->number() : holder.lens_spec.focus_dist, "frame " + std::to_string(i) + ": invalid camera");
        const Json* seed = f.find("seed");
        fr.seed = seed ? uint_field(*seed, "seed", 9007199254740992.0) : scene.seed;
        const Json* depth = f.find("max_depth");
        fr.max_depth = depth ? (uint32_t)uint_field(*depth, "max_depth", 4294967295.0) : scene.max_depth;
    }
    return frames;
}
}  // namespace rthost
