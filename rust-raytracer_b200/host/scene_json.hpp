// Config (reference config.rs:66-75) parsed from JSON and flattened into an rt_scene that owns its storage.
#pragma once
#include <string>
#include <vector>
#include "../../include/rtb200.h"
#include "jpeg_decode.hpp"
namespace rthost {
struct SceneHolder {
    rt_scene scene{};
    std::vector<rt_sphere> spheres;
    std::vector<rt_image> textures;
    std::vector<Image> images;      // decoded texture pixels (textures[i].rgb8 points into images[i])
    Image sky_image;
};
// serde_json::from_slice::<Config> (main.rs:14-15). Texture paths resolve against the process CWD like the reference
// (materials.rs:214), then against `base_dir` if given. Throws std::runtime_error with serde-like messages.
void load_scene_json(const std::string& json_text, const std::string& base_dir, SceneHolder* out);
// An animation over `scene`: a JSON array of {"camera": {<the config's camera schema>}, "seed"?: n, "max_depth"?: n}; omitted
// fields are the scene's. Throws std::runtime_error on malformed input.
std::vector<rt_frame> load_frames_json(const std::string& json_text, const rt_scene& scene);
}  // namespace rthost
