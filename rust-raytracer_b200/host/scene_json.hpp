// Config (reference config.rs:66-75) parsed from JSON and flattened into an rt_scene that owns its storage.
#pragma once
#include <string>
#include <vector>
#include "../../include/rtb200.h"
#include "jpeg_decode.hpp"
namespace rthost {
// A camera's optional thin lens (DESIGN.md §4.17), checked but not yet built: aperture 0 (absent) is no lens; focus_dist is
// resolved (the given one, else |look_from - look_at|). Build it with rtb200_camera_from_params_lens(&params, ...).
struct LensSpec {
    rt_camera_params params{};
    double aperture = 0.0;
    double focus_dist = 0.0;
};
struct SceneHolder {
    rt_scene scene{};
    std::vector<rt_sphere> spheres;
    std::vector<rt_image> textures;
    std::vector<Image> images;      // decoded texture pixels (textures[i].rgb8 points into images[i])
    Image sky_image;
    LensSpec lens_spec;             // the camera's thin lens (DESIGN.md §4.17); scene.camera is Camera::new's
    bool has_focus = false;         // the config gave focus_dist (frames inherit it)
};
// serde_json::from_slice::<Config> (main.rs:14-15). Texture paths resolve against the process CWD like the reference
// (materials.rs:214), then against `base_dir` if given. Throws std::runtime_error with serde-like messages.
void load_scene_json(const std::string& json_text, const std::string& base_dir, SceneHolder* out);
// An animation over `scene`: a JSON array of {"camera": {<the config's camera schema>}, "seed"?: n, "max_depth"?: n}; omitted
// fields are the scene's. Throws std::runtime_error on malformed input.
std::vector<rt_frame> load_frames_json(const std::string& json_text, const rt_scene& scene);
// The same with each frame's lens: a frame's camera may carry "aperture" and "focus_dist"; an omitted one is the scene's, and
// an omitted focus_dist with none in the scene is the frame's own |look_from - look_at|. frames[i].camera is Camera::new's.
std::vector<rt_frame> load_frames_json(const std::string& json_text, const SceneHolder& scene, std::vector<LensSpec>* lenses);
}  // namespace rthost
