"""rtb200 — Python host binding of the H100 render path (ctypes over the C ABI in include/rtb200.h).

Mirrors the reference's host-side interface for the path it replaces:
  * ``Config`` / ``Sphere`` / ``Camera`` JSON schema   (reference raytracer/src/config.rs:66-75, sphere.rs:18-23,
    camera.rs:29-36, materials.rs:35-42)  ->  :func:`load_scene`, :class:`Scene`
  * ``render(filename, scene)``                          (reference raytracer/src/raytracer.rs:250-266) -> :func:`render`
The hot path itself lives in ``librtb200.so`` (hand-written sm_90a CUDA). There is no CPU fallback: if the
library or an H100 is missing every render call raises :class:`RtError`.
"""
from __future__ import annotations

import ctypes as C
import functools
import json
import math
import os
from typing import Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RTB200_LIB") or os.path.join(os.path.dirname(_HERE), "librtb200.so")   # RTB200_LIB: experimental builds

RT_LAMBERTIAN, RT_METAL, RT_GLASS, RT_TEXTURE, RT_LIGHT = 0, 1, 2, 3, 4
RT_SKY_NONE, RT_SKY_GRADIENT, RT_SKY_TEXTURE = 0, 1, 2
RT_VARIANT_AUTO, RT_VARIANT_FILTERED, RT_VARIANT_EXACT_F64, RT_VARIANT_RETIRED_LANES, RT_VARIANT_BRUTE_FORCE = 0, 1, 2, 3, 4

DEFAULT_SEED = 0x5EED
CUDA_STREAM_LEGACY = 0x1   # cudaStreamLegacy: torch's default stream has handle 0, which the C ABI reads as "use the library's own stream"


class RtError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"rtb200 error {code}: {msg}")
        self.code = code


# ---- ctypes mirrors of include/rtb200.h ---------------------------------------------------------------
class rt_vec3(C.Structure):
    _fields_ = [("x", C.c_double), ("y", C.c_double), ("z", C.c_double)]

    def tup(self):
        return (self.x, self.y, self.z)


class rt_camera(C.Structure):
    _fields_ = [("origin", rt_vec3), ("lower_left_corner", rt_vec3), ("horizontal", rt_vec3), ("vertical", rt_vec3)]


class rt_camera_params(C.Structure):
    _fields_ = [("look_from", rt_vec3), ("look_at", rt_vec3), ("vup", rt_vec3), ("vfov_deg", C.c_double), ("aspect", C.c_double)]


class rt_sphere(C.Structure):
    _fields_ = [("center", rt_vec3), ("radius", C.c_double), ("kind", C.c_uint32), ("albedo", C.c_float * 3),
                ("param", C.c_double), ("texture", C.c_int32), ("reserved", C.c_int32)]


class rt_image(C.Structure):
    _fields_ = [("rgb8", C.c_void_p), ("width", C.c_uint64), ("height", C.c_uint64), ("bytes", C.c_uint64)]


class rt_sky(C.Structure):
    _fields_ = [("mode", C.c_uint32), ("reserved", C.c_uint32), ("tex", rt_image)]


class rt_scene(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("samples_per_pixel", C.c_uint32), ("max_depth", C.c_uint32),
                ("camera", rt_camera), ("sky", rt_sky),
                ("spheres", C.POINTER(rt_sphere)), ("n_spheres", C.c_uint64),
                ("textures", C.POINTER(rt_image)), ("n_textures", C.c_uint64),
                ("seed", C.c_uint64)]


class rt_options(C.Structure):
    _fields_ = [("device", C.c_int32), ("rank", C.c_int32), ("world", C.c_int32), ("band_rows", C.c_uint32),
                ("variant", C.c_uint32), ("flags", C.c_uint32), ("sample_buffer_bytes", C.c_uint64)]


class rt_stats(C.Structure):
    _fields_ = [("rays", C.c_uint64), ("samples", C.c_uint64), ("candidates", C.c_uint64),
                ("device_ms", C.c_double), ("trace_ms", C.c_double), ("wall_ms", C.c_double),
                ("kernel_launches", C.c_uint32), ("batches", C.c_uint32),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("clusters", C.c_uint64), ("frames", C.c_uint64),
                ("nodes", C.c_uint64), ("gpus_used", C.c_int32), ("reserved", C.c_int32)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class rt_kernel_info(C.Structure):
    _fields_ = [("registers", C.c_int32), ("local_bytes", C.c_int32), ("smem_bytes", C.c_uint32), ("grid", C.c_uint32),
                ("block", C.c_uint32), ("ctas_per_sm", C.c_uint32), ("smem_mask", C.c_uint32), ("bvh_nodes", C.c_uint32),
                ("bvh_leaves", C.c_uint32), ("bvh_depth", C.c_uint32), ("pool_slots", C.c_uint32), ("name", C.c_char * 96)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["name"] = d["name"].decode()
        return d


class rt_frame(C.Structure):
    """One frame of an animation over one scene: the view, the RNG key and the depth that replace the scene's own."""
    _fields_ = [("camera", rt_camera), ("seed", C.c_uint64), ("max_depth", C.c_uint32), ("reserved", C.c_uint32)]


class rt_lens(C.Structure):
    """A thin lens (rtb200_camera_from_params_lens): the camera's unit right and up vectors and radius = aperture / 2 (0: pinhole)."""
    _fields_ = [("u", rt_vec3), ("v", rt_vec3), ("radius", C.c_double), ("reserved", C.c_uint64)]


class rt_adaptive_params(C.Structure):
    """Adaptive rendering (rtb200_adaptive_*): samples per round, the sample budget (0: the scene's samples_per_pixel), the
    samples before a pixel may stop, and the f32 tolerances of the stopping rule err_c <= abs_tol + rel_tol * mean_c."""
    _fields_ = [("samples_per_round", C.c_uint32), ("max_samples", C.c_uint32), ("min_samples", C.c_uint32), ("reserved", C.c_uint32),
                ("abs_tol", C.c_float), ("rel_tol", C.c_float)]


class rt_rays(C.Structure):
    """Rays of a closest-hit query (rtb200_scene_intersect[_device]): origin and direction n x 3 f64, t_max n f64 or NULL."""
    _fields_ = [("origin", C.c_void_p), ("direction", C.c_void_p), ("t_max", C.c_void_p)]


class rt_hits(C.Structure):
    """Outputs of a closest-hit query, each NULL or n (t, sphere, front_face), n x 3 (point, normal) or n x 2 (uv) elements."""
    _fields_ = [("t", C.c_void_p), ("sphere", C.c_void_p), ("point", C.c_void_p), ("normal", C.c_void_p), ("uv", C.c_void_p),
                ("front_face", C.c_void_p)]


class rt_points(C.Structure):
    """Points of a point query (rtb200_scene_nearest[_device], rtb200_scene_overlaps[_device]): point n x 3 f64, bound n f64 or
    NULL (nearest only: +inf); the balls' radii for overlaps."""
    _fields_ = [("point", C.c_void_p), ("bound", C.c_void_p)]


class rt_nearest(C.Structure):
    """Outputs of a nearest-sphere query, each NULL or n elements (not both NULL): distance f64, sphere u32."""
    _fields_ = [("distance", C.c_void_p), ("sphere", C.c_void_p)]


class rt_trace_params(C.Structure):
    """Radiance of caller-supplied rays (rtb200_scene_trace_rays[_device]): the Philox key, samples per ray, the first sample
    index, the RNG stream of ray 0 (ray i draws from pixel stream stream0 + i) and the depth of ray_color."""
    _fields_ = [("seed", C.c_uint64), ("samples", C.c_uint32), ("sample0", C.c_uint32), ("stream0", C.c_uint32),
                ("max_depth", C.c_uint32), ("reserved", C.c_uint32 * 2)]


class rt_aov_params(C.Structure):
    """Auxiliary buffers of a resident scene's camera samples (rtb200_scene_aov[_device]): the samples per pixel and the index
    of the first."""
    _fields_ = [("samples", C.c_uint32), ("sample0", C.c_uint32), ("reserved", C.c_uint32 * 2)]


class rt_aov_out(C.Structure):
    """Outputs of rtb200_scene_aov[_device], each NULL or rows * width (hits, sphere) or rows * width * 3 (albedo, normal, point)
    elements."""
    _fields_ = [("albedo", C.c_void_p), ("normal", C.c_void_p), ("hits", C.c_void_p), ("sphere", C.c_void_p), ("point", C.c_void_p)]


class rt_denoise_params(C.Structure):
    """The edge-avoiding à-trous filter of rtb200_denoise[_device]: image size, iterations L in [1, 10], and the finite,
    non-negative weights of the colour, albedo and normal guides (0 turns a guide off)."""
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("iterations", C.c_uint32), ("reserved", C.c_uint32),
                ("color_weight", C.c_float), ("albedo_weight", C.c_float), ("normal_weight", C.c_float), ("reserved2", C.c_float)]


class rt_denoise_var_params(C.Structure):
    """The variance-guided à-trous filter of rtb200_denoise_var[_device]: image size, iterations L in [1, 10], the finite,
    non-negative weights of the colour, albedo and normal guides (0 turns a guide off), and the finite, positive variance floor."""
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("iterations", C.c_uint32), ("reserved", C.c_uint32),
                ("color_weight", C.c_float), ("albedo_weight", C.c_float), ("normal_weight", C.c_float), ("variance_floor", C.c_float)]


class rt_temporal_params(C.Structure):
    """The temporal accumulation of rtb200_temporal[_device]: image size, max_history N >= 1, the rows of motion, this frame's
    and the previous frame's cameras, and the finite, non-negative relative depth tolerance."""
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("max_history", C.c_uint32), ("n_motion", C.c_uint32),
                ("camera", rt_camera), ("prev_camera", rt_camera), ("depth_tol", C.c_double), ("reserved", C.c_uint32 * 2)]


class rt_temporal_frame(C.Structure):
    _fields_ = [("color", C.c_void_p), ("sphere", C.c_void_p), ("point", C.c_void_p)]


class rt_temporal_history(C.Structure):
    _fields_ = [("color", C.c_void_p), ("length", C.c_void_p), ("sphere", C.c_void_p), ("point", C.c_void_p)]


class rt_temporal_out(C.Structure):
    _fields_ = [("color", C.c_void_p), ("length", C.c_void_p)]


class rt_temporal_clamp(C.Structure):
    """The history clamp of rtb200_temporal_clamped[_device]: the finite, non-negative width gamma in standard deviations and
    the window radius in [1, 3]."""
    _fields_ = [("gamma", C.c_float), ("radius", C.c_uint32), ("reserved", C.c_uint32 * 2)]


HIT_FIELDS = (("t", 1, np.float64), ("sphere", 1, np.int32), ("point", 3, np.float64), ("normal", 3, np.float64),
              ("uv", 2, np.float64), ("front_face", 1, np.uint8))   # rt_hits: name, values per ray, dtype (sphere -1 = 0xffffffff)

assert C.sizeof(rt_sphere) == 64 and C.sizeof(rt_frame) == 112 and C.sizeof(rt_adaptive_params) == 24
assert C.sizeof(rt_rays) == 24 and C.sizeof(rt_hits) == 48 and C.sizeof(rt_trace_params) == 32
assert C.sizeof(rt_aov_params) == 16 and C.sizeof(rt_aov_out) == 40 and C.sizeof(rt_denoise_params) == 32
assert C.sizeof(rt_temporal_params) == 224 and C.sizeof(rt_temporal_frame) == 24 and C.sizeof(rt_temporal_history) == 32
assert C.sizeof(rt_temporal_out) == 16 and C.sizeof(rt_lens) == 64 and C.sizeof(rt_denoise_var_params) == 32
assert C.sizeof(rt_points) == 16 and C.sizeof(rt_nearest) == 16 and C.sizeof(rt_temporal_clamp) == 16
AOV_FIELDS = (("albedo", 3, np.float32), ("normal", 3, np.float32), ("hits", 1, np.uint32), ("sphere", 1, np.int32),
              ("point", 3, np.float64))   # rt_aov_out: name, values per pixel, dtype (sphere -1 = 0xffffffff)

# every symbol include/rtb200.h declares (tests check that the library exports all of them)
ABI_SYMBOLS = [
    "rtb200_abi_version", "rtb200_last_error", "rtb200_camera_from_params", "rtb200_shard_rows",
    "rtb200_render_rgb8", "rtb200_render_linear_f32", "rtb200_scene_upload", "rtb200_render_device",
    "rtb200_scene_release", "rtb200_probe_sphere_hit", "rtb200_probe_refract", "rtb200_probe_reflectance",
    "rtb200_probe_sky", "rtb200_probe_get_ray", "rtb200_probe_rng", "rtb200_probe_quantise",
    "rtb200_decode_jpeg_file", "rtb200_free", "rtb200_render_device_async", "rtb200_render_device_wait",
    "rtb200_debug_bvh", "rtb200_probe_sphere_uv", "rtb200_device_count", "rtb200_render_rgb8_multi", "rtb200_scene_kernel_info",
    "rtb200_render_frames", "rtb200_render_frames_device",
    "rtb200_scene_update_spheres", "rtb200_scene_update_geometry_device", "rtb200_scene_debug_records",
    "rtb200_scene_rebuild", "rtb200_scene_debug_topology",
    "rtb200_adaptive_begin", "rtb200_adaptive_step", "rtb200_adaptive_resolve", "rtb200_render_adaptive",
    "rtb200_scene_intersect_device", "rtb200_scene_intersect",
    "rtb200_scene_occluded_device", "rtb200_scene_occluded",
    "rtb200_scene_trace_rays_device", "rtb200_scene_trace_rays",
    "rtb200_scene_edit_spheres",
    "rtb200_scene_aov_device", "rtb200_scene_aov",
    "rtb200_denoise_scratch_bytes", "rtb200_denoise_device", "rtb200_denoise",
    "rtb200_temporal_device", "rtb200_temporal",
    "rtb200_camera_from_params_lens", "rtb200_scene_set_lens", "rtb200_render_frames_lens", "rtb200_render_frames_lens_device",
    "rtb200_probe_lens_ray",
    "rtb200_denoise_var_scratch_bytes", "rtb200_denoise_var_device", "rtb200_denoise_var",
    "rtb200_render_frames_var_device", "rtb200_render_frames_var", "rtb200_adaptive_resolve_var", "rtb200_render_adaptive_var",
    "rtb200_scene_nearest_device", "rtb200_scene_nearest", "rtb200_scene_overlaps_device", "rtb200_scene_overlaps",
    "rtb200_temporal_clamped_device", "rtb200_temporal_clamped",
    "rtb200_temporal_var_device", "rtb200_temporal_var",
]

_lib = None


def lib() -> C.CDLL:
    """Load librtb200.so (built in-tree by `make -C rust-raytracer_b200` / __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RtError(-2, f"{LIB_PATH} is missing: build it with `make -C rust-raytracer_b200` (there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    L.rtb200_abi_version.restype = C.c_int
    L.rtb200_last_error.restype = C.c_char_p
    L.rtb200_camera_from_params.argtypes = [C.POINTER(rt_camera_params), C.POINTER(rt_camera)]
    L.rtb200_shard_rows.restype = C.c_uint32
    L.rtb200_shard_rows.argtypes = [C.c_uint32, C.c_int32, C.c_int32, C.c_uint32]
    L.rtb200_render_rgb8.argtypes = [C.POINTER(rt_scene), C.POINTER(rt_options), C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_render_linear_f32.argtypes = [C.POINTER(rt_scene), C.POINTER(rt_options), C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_scene_upload.argtypes = [C.POINTER(rt_scene), C.POINTER(rt_options), C.POINTER(C.c_void_p)]
    L.rtb200_render_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_scene_release.argtypes = [C.c_void_p]
    L.rtb200_render_device_async.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.rtb200_render_device_wait.argtypes = [C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_probe_sphere_hit.argtypes = [C.POINTER(rt_vec3), C.c_double, C.POINTER(rt_vec3), C.POINTER(rt_vec3), C.c_double,
                                          C.c_double, C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(rt_vec3),
                                          C.POINTER(rt_vec3), C.POINTER(C.c_int32)]
    L.rtb200_probe_refract.argtypes = [C.POINTER(rt_vec3), C.POINTER(rt_vec3), C.c_double, C.POINTER(rt_vec3)]
    L.rtb200_probe_reflectance.argtypes = [C.c_double, C.c_double, C.POINTER(C.c_double)]
    L.rtb200_probe_sky.argtypes = [C.POINTER(rt_vec3), C.c_uint32, C.POINTER(C.c_float)]
    L.rtb200_probe_get_ray.argtypes = [C.POINTER(rt_camera), C.c_double, C.c_double, C.POINTER(rt_vec3), C.POINTER(rt_vec3)]
    L.rtb200_probe_rng.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_double)]
    L.rtb200_probe_quantise.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    L.rtb200_decode_jpeg_file.argtypes = [C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.rtb200_free.argtypes = [C.c_void_p]
    L.rtb200_free.restype = None
    L.rtb200_debug_bvh.argtypes = [C.POINTER(rt_scene), C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.c_void_p, C.c_uint64,
                                   C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    L.rtb200_probe_sphere_uv.argtypes = [C.POINTER(C.c_double), C.c_uint32, C.POINTER(C.c_double)]
    L.rtb200_device_count.restype = C.c_int
    L.rtb200_render_rgb8_multi.argtypes = [C.POINTER(rt_scene), C.POINTER(rt_options), C.c_int32, C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_scene_kernel_info.argtypes = [C.c_void_p, C.POINTER(rt_kernel_info)]
    L.rtb200_render_frames.argtypes = [C.POINTER(rt_scene), C.POINTER(rt_options), C.POINTER(rt_frame), C.c_uint32, C.c_void_p, C.c_void_p,
                                       C.POINTER(rt_stats)]
    L.rtb200_render_frames_device.argtypes = [C.c_void_p, C.POINTER(rt_frame), C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.POINTER(rt_stats)]
    L.rtb200_scene_update_spheres.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    L.rtb200_scene_update_geometry_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.rtb200_scene_debug_records.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                             C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    L.rtb200_scene_rebuild.argtypes = [C.c_void_p, C.c_void_p]
    L.rtb200_scene_debug_topology.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_uint32)] + [C.c_void_p, C.c_uint64] * 5
    L.rtb200_adaptive_begin.argtypes = [C.c_void_p, C.POINTER(rt_adaptive_params), C.c_void_p]
    L.rtb200_adaptive_step.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(rt_stats)]
    L.rtb200_adaptive_resolve.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.rtb200_render_adaptive.argtypes = [C.POINTER(rt_scene), C.POINTER(rt_options), C.POINTER(rt_adaptive_params), C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_scene_intersect_device.argtypes = [C.c_void_p, C.POINTER(rt_rays), C.c_uint32, C.POINTER(rt_hits), C.c_void_p]
    L.rtb200_scene_intersect.argtypes = [C.c_void_p, C.POINTER(rt_rays), C.c_uint32, C.POINTER(rt_hits), C.POINTER(rt_stats)]
    L.rtb200_scene_occluded_device.argtypes = [C.c_void_p, C.POINTER(rt_rays), C.c_uint32, C.c_void_p, C.c_void_p]
    L.rtb200_scene_occluded.argtypes = [C.c_void_p, C.POINTER(rt_rays), C.c_uint32, C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_scene_nearest_device.argtypes = [C.c_void_p, C.POINTER(rt_points), C.c_uint32, C.POINTER(rt_nearest), C.c_void_p]
    L.rtb200_scene_nearest.argtypes = [C.c_void_p, C.POINTER(rt_points), C.c_uint32, C.POINTER(rt_nearest), C.POINTER(rt_stats)]
    L.rtb200_scene_overlaps_device.argtypes = [C.c_void_p, C.POINTER(rt_points), C.c_uint32, C.c_void_p, C.c_void_p]
    L.rtb200_scene_overlaps.argtypes = [C.c_void_p, C.POINTER(rt_points), C.c_uint32, C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_scene_trace_rays_device.argtypes = [C.c_void_p, C.POINTER(rt_rays), C.c_uint32, C.POINTER(rt_trace_params), C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_scene_trace_rays.argtypes = [C.c_void_p, C.POINTER(rt_rays), C.c_uint32, C.POINTER(rt_trace_params), C.c_void_p,
                                          C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_scene_edit_spheres.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    L.rtb200_scene_aov_device.argtypes = [C.c_void_p, C.POINTER(rt_aov_params), C.POINTER(rt_frame), C.POINTER(rt_aov_out), C.c_void_p]
    L.rtb200_scene_aov.argtypes = [C.c_void_p, C.POINTER(rt_aov_params), C.POINTER(rt_frame), C.POINTER(rt_aov_out), C.POINTER(rt_stats)]
    L.rtb200_denoise_scratch_bytes.restype = C.c_uint64
    L.rtb200_denoise_scratch_bytes.argtypes = [C.c_uint32, C.c_uint32]
    L.rtb200_denoise_device.argtypes = [C.c_int32, C.POINTER(rt_denoise_params), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p]
    L.rtb200_denoise.argtypes = [C.c_int32, C.POINTER(rt_denoise_params), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.POINTER(rt_stats)]
    L.rtb200_render_frames_var_device.argtypes = [C.c_void_p, C.POINTER(rt_frame), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_render_frames_var.argtypes = [C.POINTER(rt_scene), C.POINTER(rt_options), C.POINTER(rt_frame), C.c_void_p, C.c_uint32,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_adaptive_resolve_var.argtypes = [C.c_void_p] + [C.c_void_p] * 5
    L.rtb200_render_adaptive_var.argtypes = [C.POINTER(rt_scene), C.POINTER(rt_options), C.POINTER(rt_adaptive_params), C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_denoise_var_scratch_bytes.restype = C.c_uint64
    L.rtb200_denoise_var_scratch_bytes.argtypes = [C.c_uint32, C.c_uint32]
    L.rtb200_denoise_var_device.argtypes = [C.c_int32, C.POINTER(rt_denoise_var_params)] + [C.c_void_p] * 9
    L.rtb200_denoise_var.argtypes = [C.c_int32, C.POINTER(rt_denoise_var_params)] + [C.c_void_p] * 7 + [C.POINTER(rt_stats)]
    L.rtb200_temporal_device.argtypes = [C.c_int32, C.POINTER(rt_temporal_params), C.POINTER(rt_temporal_frame),
                                         C.POINTER(rt_temporal_history), C.c_void_p, C.POINTER(rt_temporal_out), C.c_void_p]
    L.rtb200_temporal.argtypes = [C.c_int32, C.POINTER(rt_temporal_params), C.POINTER(rt_temporal_frame), C.POINTER(rt_temporal_history),
                                  C.c_void_p, C.POINTER(rt_temporal_out), C.POINTER(rt_stats)]
    L.rtb200_temporal_clamped_device.argtypes = [C.c_int32, C.POINTER(rt_temporal_params), C.POINTER(rt_temporal_clamp),
                                                 C.POINTER(rt_temporal_frame), C.POINTER(rt_temporal_history), C.c_void_p,
                                                 C.POINTER(rt_temporal_out), C.c_void_p]
    L.rtb200_temporal_clamped.argtypes = [C.c_int32, C.POINTER(rt_temporal_params), C.POINTER(rt_temporal_clamp), C.POINTER(rt_temporal_frame),
                                          C.POINTER(rt_temporal_history), C.c_void_p, C.POINTER(rt_temporal_out), C.POINTER(rt_stats)]
    L.rtb200_temporal_var_device.argtypes = [C.c_int32, C.POINTER(rt_temporal_params), C.POINTER(rt_temporal_clamp),
                                             C.POINTER(rt_temporal_frame), C.c_void_p, C.POINTER(rt_temporal_history), C.c_void_p,
                                             C.c_void_p, C.POINTER(rt_temporal_out), C.c_void_p, C.c_void_p]
    L.rtb200_temporal_var.argtypes = [C.c_int32, C.POINTER(rt_temporal_params), C.POINTER(rt_temporal_clamp), C.POINTER(rt_temporal_frame),
                                      C.c_void_p, C.POINTER(rt_temporal_history), C.c_void_p, C.c_void_p, C.POINTER(rt_temporal_out),
                                      C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_camera_from_params_lens.argtypes = [C.POINTER(rt_camera_params), C.c_double, C.c_double, C.POINTER(rt_camera), C.POINTER(rt_lens)]
    L.rtb200_scene_set_lens.argtypes = [C.c_void_p, C.POINTER(rt_lens)]
    L.rtb200_render_frames_lens.argtypes = [C.POINTER(rt_scene), C.POINTER(rt_options), C.POINTER(rt_frame), C.POINTER(rt_lens), C.c_uint32,
                                            C.c_void_p, C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_render_frames_lens_device.argtypes = [C.c_void_p, C.POINTER(rt_frame), C.POINTER(rt_lens), C.c_uint32, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.POINTER(rt_stats)]
    L.rtb200_probe_lens_ray.argtypes = [C.POINTER(rt_camera), C.POINTER(rt_lens), C.c_uint64, C.c_uint32, C.c_uint32, C.c_double, C.c_double,
                                        C.POINTER(rt_vec3), C.POINTER(rt_vec3), C.POINTER(C.c_uint32)]
    _lib = L
    return L


def _check(rc: int):
    if rc != 0:
        raise RtError(rc, (lib().rtb200_last_error() or b"").decode("utf-8", "replace"))


def vec3(v) -> rt_vec3:
    if isinstance(v, dict):
        return rt_vec3(float(v["x"]), float(v["y"]), float(v["z"]))
    return rt_vec3(float(v[0]), float(v[1]), float(v[2]))


_camera_backend = None   # bench.py's CPU reference arm installs the oracle's Camera::new here so that it never maps librtb200.so


def set_camera_backend(fn):
    """fn(rt_camera_params*, rt_camera*) -> int replacing rtb200_camera_from_params (None restores the library)."""
    global _camera_backend
    _camera_backend = fn


def camera_from_params(look_from, look_at, vup, vfov: float, aspect: float) -> rt_camera:
    """Camera::new (reference camera.rs:45-77), evaluated by the library's host code."""
    p = rt_camera_params(vec3(look_from), vec3(look_at), vec3(vup), float(vfov), float(aspect))
    out = rt_camera()
    if _camera_backend is not None:
        rc = _camera_backend(C.byref(p), C.byref(out))
        if rc != 0:
            raise RtError(rc, "camera backend failed")
        return out
    _check(lib().rtb200_camera_from_params(C.byref(p), C.byref(out)))
    return out


_lens_backend = None   # the lens twin of _camera_backend: fn(rt_camera_params*, double, double, rt_camera*, rt_lens*) -> int


def set_lens_backend(fn):
    """fn(rt_camera_params*, aperture, focus_dist, rt_camera*, rt_lens*) -> int replacing rtb200_camera_from_params_lens (None
    restores the library), so that CPU-only callers can build lens cameras without mapping librtb200.so."""
    global _lens_backend
    _lens_backend = fn


def camera_from_params_lens(look_from, look_at, vup, vfov: float, aspect: float, aperture: float, focus_dist: float):
    """The thin-lens camera (include/rtb200.h, DESIGN.md §4.17): (rt_camera, rt_lens). At focus_dist 1.0 the camera is
    camera_from_params' bit for bit; aperture 0 gives a lens of radius 0 (a pinhole)."""
    p = rt_camera_params(vec3(look_from), vec3(look_at), vec3(vup), float(vfov), float(aspect))
    cam, lens = rt_camera(), rt_lens()
    fn = _lens_backend if _lens_backend is not None else lib().rtb200_camera_from_params_lens
    rc = fn(C.byref(p), float(aperture), float(focus_dist), C.byref(cam), C.byref(lens))
    if rc != 0:
        if _lens_backend is not None:
            raise RtError(rc, "camera_from_params_lens: aperture must be finite and >= 0, focus_dist finite and > 0")
        _check(rc)
    return cam, lens


def focal_length(look_from, look_at) -> float:
    """|look_from - look_at| (camera.rs:68): a lens camera's focus distance when none is given."""
    a, b = vec3(look_from), vec3(look_at)
    d = (a.x - b.x, a.y - b.y, a.z - b.z)
    return math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])


def lens_from_params(p: dict):
    """(rt_camera, rt_lens or None) of a camera dict with optional "aperture" and "focus_dist" (None: no lens, the camera is
    camera_from_params'). focus_dist defaults to focal_length(look_from, look_at)."""
    aperture = float(p.get("aperture") or 0.0)
    if aperture == 0.0:
        return camera_from_params(p["look_from"], p["look_at"], p["vup"], p["vfov"], p["aspect"]), None
    fd = p.get("focus_dist")
    fd = focal_length(p["look_from"], p["look_at"]) if fd is None else float(fd)
    cam, lens = camera_from_params_lens(p["look_from"], p["look_at"], p["vup"], p["vfov"], p["aspect"], aperture, fd)
    return cam, (lens if lens.radius != 0.0 else None)


def shard_rows(height: int, rank: int, world: int, band_rows: int = 1) -> int:
    return int(lib().rtb200_shard_rows(height, rank, world, band_rows))


def shard_row_indices(height: int, rank: int, world: int, band_rows: int = 1) -> np.ndarray:
    y = np.arange(height)
    return y[((y // max(band_rows, 1)) % max(world, 1)) == rank]


def _decode_jpeg(path: str) -> np.ndarray:
    """load_texture_image (reference materials.rs:213-219): the library's own baseline JPEG decoder, so the Python host
    and the C++ CLI stage identical texels."""
    buf = C.c_void_p(); w = C.c_uint64(); h = C.c_uint64()
    rc = lib().rtb200_decode_jpeg_file(os.fsencode(path), C.byref(buf), C.byref(w), C.byref(h))
    if rc != 0:
        raise RtError(rc, f"cannot decode JPEG {path}")
    try:
        arr = np.ctypeslib.as_array(C.cast(buf, C.POINTER(C.c_uint8)), shape=(h.value, w.value, 3)).copy()
    finally:
        lib().rtb200_free(buf)
    return arr


def _set_material(s: rt_sphere, material):
    """Give sphere record s a JSON material ({"Metal": {"albedo": [...], "fuzz": f}}, ...; a Texture names one of the scene's
    textures by index: {"Texture": {"albedo": [...], "h_offset": f, "texture": k}}) or the material of an rt_sphere."""
    if isinstance(material, rt_sphere):
        s.kind, s.param, s.texture = material.kind, material.param, material.texture
        s.albedo[:] = list(material.albedo)
        return
    (kind, body), = material.items()
    s.texture, s.param = -1, 0.0
    s.albedo[:] = [np.float32(a) for a in body.get("albedo", [0.0, 0.0, 0.0])]
    if kind == "Lambertian":
        s.kind = RT_LAMBERTIAN
    elif kind == "Metal":
        s.kind = RT_METAL; s.param = float(body["fuzz"])
    elif kind == "Glass":
        s.kind = RT_GLASS; s.param = float(body["index_of_refraction"])
    elif kind == "Texture":
        s.kind = RT_TEXTURE; s.param = float(body["h_offset"]); s.texture = int(body["texture"])
    elif kind == "Light":
        s.kind = RT_LIGHT
    else:
        raise ValueError(f"unknown material {kind}")


def make_sphere(center, radius: float, material) -> rt_sphere:
    """A sphere record (for ResidentScene.edit_spheres and Scene.edited) from a centre, a radius and a material in the forms
    Scene.set_sphere takes."""
    s = rt_sphere()
    s.center = vec3(center)
    s.radius = float(radius)
    _set_material(s, material)
    return s


class Scene:
    """Parsed scene = the reference's ``Config`` (config.rs:66-75), flattened into an ``rt_scene``.

    Keeps every buffer the C struct points into alive. Mutating ``width/height/samples_per_pixel/max_depth``
    mirrors how the reference's own tests override a parsed Config (raytracer.rs:272-273, 281-282); call
    :meth:`set_camera` when the aspect ratio changes (aspect is a camera field, camera.rs:26,54).
    """

    def __init__(self):
        self.c = rt_scene()
        self.c.seed = DEFAULT_SEED
        self._spheres = None
        self._tex_arrays: list[np.ndarray] = []
        self._tex_structs = None
        self._sky_array = None
        self.camera_params: Optional[dict] = None
        self.lens: Optional[rt_lens] = None   # the thin lens of the camera (None: pinhole, DESIGN.md §4.17)
        self.source = None

    # -- construction ---------------------------------------------------------------------------------
    @staticmethod
    def from_config(cfg: dict, base_dir: str = ".", textures: bool = True) -> "Scene":
        sc = Scene()
        sc.source = cfg
        sc.c.width = int(cfg["width"]); sc.c.height = int(cfg["height"])
        sc.c.samples_per_pixel = int(cfg["samples_per_pixel"]); sc.c.max_depth = int(cfg["max_depth"])
        cam = cfg["camera"]
        sc.camera_params = dict(look_from=cam["look_from"], look_at=cam["look_at"], vup=cam["vup"], vfov=cam["vfov"], aspect=cam["aspect"])
        if cam.get("aperture") is not None:
            sc.camera_params["aperture"] = float(cam["aperture"])
        if cam.get("focus_dist") is not None:
            sc.camera_params["focus_dist"] = float(cam["focus_dist"])
        sc.c.camera, sc.lens = lens_from_params(sc.camera_params)
        # sky: missing/null -> None (black); {"texture": ""} -> gradient; path -> equirect texture (config.rs:49-64, raytracer.rs:137-161)
        sky = cfg.get("sky", None)
        sc.c.sky.mode = RT_SKY_NONE
        if sky is not None:
            tex = sky.get("texture", "")
            if tex in ("", None):
                sc.c.sky.mode = RT_SKY_GRADIENT
            else:
                arr = _decode_jpeg(os.path.join(base_dir, tex))
                sc._sky_array = arr
                sc.c.sky.mode = RT_SKY_TEXTURE
                sc.c.sky.tex = rt_image(arr.ctypes.data, arr.shape[1], arr.shape[0], arr.size)
        objs = cfg.get("objects", [])
        arr_t = rt_sphere * max(len(objs), 1)
        sc._spheres = arr_t()
        tex_structs = []
        for i, o in enumerate(objs):
            s = sc._spheres[i]
            s.center = vec3(o["center"]); s.radius = float(o["radius"]); s.texture = -1
            (kind, body), = o["material"].items()   # externally tagged enum (materials.rs:35-42)
            if kind == "Lambertian":
                s.kind = RT_LAMBERTIAN; s.albedo[:] = [np.float32(a) for a in body["albedo"]]
            elif kind == "Metal":
                s.kind = RT_METAL; s.albedo[:] = [np.float32(a) for a in body["albedo"]]; s.param = float(body["fuzz"])
            elif kind == "Glass":
                s.kind = RT_GLASS; s.param = float(body["index_of_refraction"])
            elif kind == "Texture":
                s.kind = RT_TEXTURE; s.albedo[:] = [np.float32(a) for a in body["albedo"]]; s.param = float(body["h_offset"])
                if not textures:
                    raise ValueError("texture material but textures=False")
                arr = _decode_jpeg(os.path.join(base_dir, body["pixels"]))
                w, h = int(body["width"]), int(body["height"])   # JSON dims, not the file's (materials.rs:208-209)
                if w * h * 3 > arr.size:
                    raise ValueError(f"texture {body['pixels']}: JSON says {w}x{h} but the file holds {arr.shape[1]}x{arr.shape[0]}")
                sc._tex_arrays.append(arr)
                tex_structs.append(rt_image(arr.ctypes.data, w, h, arr.size))
                s.texture = len(tex_structs) - 1
            elif kind == "Light":
                s.kind = RT_LIGHT
            else:
                raise ValueError(f"unknown material {kind}")
        sc.c.spheres = C.cast(sc._spheres, C.POINTER(rt_sphere)); sc.c.n_spheres = len(objs)
        if tex_structs:
            sc._tex_structs = (rt_image * len(tex_structs))(*tex_structs)
            sc.c.textures = C.cast(sc._tex_structs, C.POINTER(rt_image))
        sc.c.n_textures = len(tex_structs)
        return sc

    def set_camera(self, **kw):
        """Change camera fields (look_from, look_at, vup, vfov, aspect, and the lens's aperture and focus_dist; None removes
        aperture or focus_dist)."""
        self.camera_params.update(kw)
        for k in ("aperture", "focus_dist"):
            if k in self.camera_params and self.camera_params[k] is None:
                del self.camera_params[k]
        self.c.camera, self.lens = lens_from_params(self.camera_params)

    def resize(self, width: int, height: int, spp: Optional[int] = None, max_depth: Optional[int] = None, fix_aspect: bool = False):
        self.c.width, self.c.height = int(width), int(height)
        if spp is not None:
            self.c.samples_per_pixel = int(spp)
        if max_depth is not None:
            self.c.max_depth = int(max_depth)
        if fix_aspect:
            self.set_camera(aspect=float(width) / float(height))
        return self

    def set_sphere(self, i: int, center=None, radius: Optional[float] = None, material=None) -> rt_sphere:
        """Edit sphere i of the host scene in place and return a copy of its record (for ResidentScene.update_spheres, so
        that a resident handle, a fresh upload and the oracle can render the same edit). `material` is a JSON material
        ({"Metal": {"albedo": [...], "fuzz": f}}, ...; a Texture names one of the scene's textures by index:
        {"Texture": {"albedo": [...], "h_offset": f, "texture": k}}) or an rt_sphere whose material is copied."""
        if not 0 <= i < self.n_spheres:
            raise IndexError(f"sphere {i} of {self.n_spheres}")
        s = self._spheres[i]
        if center is not None:
            s.center = vec3(center)
        if radius is not None:
            s.radius = float(radius)
        if material is not None:
            _set_material(s, material)
        return rt_sphere.from_buffer_copy(s)

    def edited(self, remove: Sequence[int] = (), insert: Sequence[rt_sphere] = (), at: Optional[Sequence[int]] = None) -> "Scene":
        """A new host scene with the edited sphere list of ResidentScene.edit_spheres: this list without the spheres `remove`,
        with insert[k] placed just before old sphere at[k] (None: every insert appended). It shares the textures, sky, camera,
        size, samples, depth and seed of this scene, so a fresh upload of it and the oracle render what an edited handle does."""
        n = self.n_spheres
        rem = [int(i) for i in remove]
        if any(not 0 <= i < n for i in rem) or len(set(rem)) != len(rem):
            raise ValueError(f"remove holds distinct indices below {n}, got {rem}")
        at = [n] * len(insert) if at is None else [int(j) for j in at]
        if len(at) != len(insert):
            raise ValueError(f"{len(at)} positions for {len(insert)} inserts")
        if any(not 0 <= j <= n for j in at) or any(a > b for a, b in zip(at, at[1:])):
            raise ValueError(f"at is non-decreasing with values in [0, {n}], got {at}")
        gone, before = set(rem), {}
        for k, j in enumerate(at):
            before.setdefault(j, []).append(insert[k])
        spheres = []
        for j in range(n + 1):
            spheres += [rt_sphere.from_buffer_copy(s) for s in before.get(j, [])]
            if j < n and j not in gone:
                spheres.append(rt_sphere.from_buffer_copy(self._spheres[j]))
        sc = Scene()
        C.memmove(C.byref(sc.c), C.byref(self.c), C.sizeof(rt_scene))
        sc._tex_arrays, sc._tex_structs, sc._sky_array = self._tex_arrays, self._tex_structs, self._sky_array
        sc.camera_params = dict(self.camera_params) if self.camera_params is not None else None
        sc.lens = rt_lens.from_buffer_copy(self.lens) if self.lens is not None else None
        sc._spheres = (rt_sphere * max(len(spheres), 1))(*spheres)
        sc.c.spheres = C.cast(sc._spheres, C.POINTER(rt_sphere)); sc.c.n_spheres = len(spheres)
        return sc

    @property
    def n_spheres(self):
        return int(self.c.n_spheres)

    @property
    def seed(self):
        return int(self.c.seed)

    @seed.setter
    def seed(self, v):
        self.c.seed = int(v)


def read_config(path: str) -> dict:
    """Parse a scene file (plain JSON, or the gzip-compressed copies under scenes/)."""
    if path.endswith(".gz"):
        import gzip

        with gzip.open(path, "rb") as f:
            return json.loads(f.read())
    with open(path, "rb") as f:
        return json.loads(f.read())


def load_scene(path: str, base_dir: Optional[str] = None) -> Scene:
    """serde_json::from_slice::<Config> (reference main.rs:14-15). Texture paths resolve against ``base_dir``
    (the reference resolves them against the process CWD, materials.rs:214)."""
    cfg = read_config(path)
    if base_dir is None:
        base_dir = os.path.dirname(os.path.abspath(path))   # scenes say "data/earth.jpg"
        if not os.path.isdir(os.path.join(base_dir, "data")):
            base_dir = os.path.dirname(base_dir)
    return Scene.from_config(cfg, base_dir)


def _record_views(info, nodes: np.ndarray, rec: np.ndarray, flat: np.ndarray) -> dict:
    """The float arrays of rtb200_debug_bvh / rtb200_scene_debug_records, sized by their info[8], in their logical shapes:
    a node is lo[3][8], hi[3][8], child[8]; a leaf holds k/2 pair-packed records; a flat pair is one record pair."""
    n_nodes, n_leaves, depth, k, _, fpn, n_pairs, _ = (int(x) for x in info)
    nd = nodes[: n_nodes * fpn].reshape(n_nodes, fpn)
    return {"n_nodes": n_nodes, "n_leaves": n_leaves, "depth": depth,
            "lo": nd[:, :24].reshape(n_nodes, 3, 8), "hi": nd[:, 24:48].reshape(n_nodes, 3, 8), "child": nd[:, 48:56].view(np.uint32),
            "leaf_rec": rec[: n_leaves * k * 4].reshape(n_leaves, k // 2, 2, 4), "flat": flat[: n_pairs * 8].reshape(n_pairs, 2, 4)}


def bvh_records(scene: "Scene") -> dict:
    """Host-side diagnostic: the hierarchy the closest-hit stage traverses (no GPU needed). See rtb200_debug_bvh."""
    n = scene.n_spheres
    g = (C.c_double * 3)(); info = (C.c_uint32 * 8)()
    _check(lib().rtb200_debug_bvh(C.byref(scene.c), g, info, None, 0, None, 0, None, 0, None, 0, None, 0))
    n_nodes, n_leaves, depth, k, n_always, fpn, n_pairs, _ = (int(x) for x in info)
    nodes = np.zeros(max(n_nodes * fpn, 1), np.float32); rec = np.zeros(max(n_leaves * k * 4, 1), np.float32)
    ids = np.zeros(max(n_leaves * k, 1), np.uint32); always = np.zeros(max(n_always, 1), np.uint32); flat = np.zeros(max(n_pairs * 8, 1), np.float32)
    _check(lib().rtb200_debug_bvh(C.byref(scene.c), g, info, nodes.ctypes.data, nodes.size, rec.ctypes.data, rec.size, ids.ctypes.data, ids.size,
                                  always.ctypes.data, always.size, flat.ctypes.data, flat.size))
    return {**_record_views(info, nodes, rec, flat), "leaf_size": k, "recentre": np.array(g[:]), "n": n,
            "leaf_id": ids[: n_leaves * k].reshape(n_leaves, k), "always": always[:n_always]}


def make_options(device: int = -1, rank: int = 0, world: int = 1, band_rows: int = 1, variant: int = RT_VARIANT_AUTO,
                 sample_buffer_bytes: int = 0) -> rt_options:
    return rt_options(device, rank, world, band_rows, variant, 0, sample_buffer_bytes)


def render_rgb8(scene: Scene, opts: Optional[rt_options] = None, out: Optional[np.ndarray] = None):
    """Host in, host out: the replacement of reference raytracer.rs:259-263. Returns (uint8 [rows,w,3], stats dict)."""
    rows = scene.c.height if (opts is None or opts.world <= 1) else shard_rows(scene.c.height, opts.rank, opts.world, opts.band_rows)
    if out is None:
        out = np.empty((rows, scene.c.width, 3), dtype=np.uint8)
    if scene.lens is not None:   # the one-shot render of a lens camera: one frame of rtb200_render_frames_lens
        return _render_lens_once(scene, opts, out, False)
    st = rt_stats()
    _check(lib().rtb200_render_rgb8(C.byref(scene.c), C.byref(opts) if opts is not None else None, out.ctypes.data, C.byref(st)))
    return out, st.as_dict()


def render_linear(scene: Scene, opts: Optional[rt_options] = None):
    """Per-pixel mean radiance before sqrt/quantisation (float32 [rows,w,3]) and stats."""
    rows = scene.c.height if (opts is None or opts.world <= 1) else shard_rows(scene.c.height, opts.rank, opts.world, opts.band_rows)
    out = np.empty((rows, scene.c.width, 3), dtype=np.float32)
    if scene.lens is not None:
        return _render_lens_once(scene, opts, out, True)
    st = rt_stats()
    _check(lib().rtb200_render_linear_f32(C.byref(scene.c), C.byref(opts) if opts is not None else None, out.ctypes.data, C.byref(st)))
    return out, st.as_dict()


def _render_lens_once(scene: Scene, opts: Optional[rt_options], out: np.ndarray, linear: bool):
    f = rt_frame(scene.c.camera, scene.seed, scene.c.max_depth, 0)
    st = rt_stats()
    _check(lib().rtb200_render_frames_lens(C.byref(scene.c), C.byref(opts) if opts is not None else None, C.byref(f), C.byref(scene.lens), 1,
                                           None if linear else out.ctypes.data, out.ctypes.data if linear else None, C.byref(st)))
    return out, st.as_dict()


def _refuse_lens(scene: Scene, what: str):
    if scene.lens is not None:
        raise RtError(-1, f"{what} takes no lens: render a lens scene with render_rgb8 / render_frames or a ResidentScene")


def device_count() -> int:
    return int(lib().rtb200_device_count())


def render_rgb8_multi(scene: Scene, n_gpus: int = 0, opts: Optional[rt_options] = None, out: Optional[np.ndarray] = None):
    """One process, n_gpus devices (0 = all): rtb200_render_rgb8_multi. Returns (uint8 [h,w,3], stats dict)."""
    _refuse_lens(scene, "render_rgb8_multi")
    if out is None:
        out = np.empty((scene.c.height, scene.c.width, 3), dtype=np.uint8)
    st = rt_stats()
    _check(lib().rtb200_render_rgb8_multi(C.byref(scene.c), C.byref(opts) if opts is not None else None, int(n_gpus), out.ctypes.data, C.byref(st)))
    return out, st.as_dict()


def make_frame(scene: Scene, look_from=None, look_at=None, vup=None, vfov: Optional[float] = None, aspect: Optional[float] = None,
               seed: Optional[int] = None, max_depth: Optional[int] = None) -> rt_frame:
    """One frame of an animation over `scene`: camera fields, seed and max_depth that are not given are the scene's own. On a
    lens scene the camera is the lens camera's, focused like the scene's (make_frame_lens also returns the frame's lens)."""
    p = dict(scene.camera_params)
    for k, v in (("look_from", look_from), ("look_at", look_at), ("vup", vup), ("vfov", vfov), ("aspect", aspect)):
        if v is not None:
            p[k] = v
    cam, _ = lens_from_params(p)
    return rt_frame(cam, scene.seed if seed is None else int(seed), scene.c.max_depth if max_depth is None else int(max_depth), 0)


def make_frame_lens(scene: Scene, look_from=None, look_at=None, vup=None, vfov: Optional[float] = None, aspect: Optional[float] = None,
                    seed: Optional[int] = None, max_depth: Optional[int] = None, aperture: Optional[float] = None,
                    focus_dist: Optional[float] = None):
    """make_frame with a lens: (rt_frame, rt_lens). Omitted aperture and focus_dist are the scene's; with no focus_dist
    anywhere it is the frame's own |look_from - look_at|. An aperture of 0 gives a lens of radius 0 (a pinhole frame)."""
    p = dict(scene.camera_params)
    for k, v in (("look_from", look_from), ("look_at", look_at), ("vup", vup), ("vfov", vfov), ("aspect", aspect),
                 ("aperture", aperture), ("focus_dist", focus_dist)):
        if v is not None:
            p[k] = v
    cam, lens = lens_from_params(p)
    f = rt_frame(cam, scene.seed if seed is None else int(seed), scene.c.max_depth if max_depth is None else int(max_depth), 0)
    return f, (lens if lens is not None else rt_lens())


def _lens_array(lenses: Optional[Sequence[rt_lens]], n: int):
    if lenses is None:
        return None
    if len(lenses) != n:
        raise ValueError(f"{len(lenses)} lenses for {n} frames")
    return (rt_lens * max(n, 1))(*[l if l is not None else rt_lens() for l in lenses])


def _frame_array(frames: Sequence[rt_frame]):
    arr = (rt_frame * max(len(frames), 1))(*frames)
    return arr, len(frames)


def render_frames(scene: Scene, frames: Sequence[rt_frame], opts: Optional[rt_options] = None, linear: bool = False,
                  lenses: Optional[Sequence[rt_lens]] = None, variance: bool = False):
    """Render len(frames) frames of one scene in as few trace launches as the sample buffer allows (rtb200_render_frames).
    Frame i equals render_rgb8 / render_linear of the scene with frames[i]'s camera, seed and max_depth. lenses: frame i's
    lens (None or radius 0: pinhole; rtb200_render_frames_lens); without it a lens scene renders every frame with its own lens.
    Returns (uint8 [n,rows,w,3], or float32 with linear=True, stats dict); with variance=True (rtb200_render_frames_var)
    (image, variance float32 [n,rows,w,3] of each pixel's mean, stats dict)."""
    rows = scene.c.height if (opts is None or opts.world <= 1) else shard_rows(scene.c.height, opts.rank, opts.world, opts.band_rows)
    arr, n = _frame_array(frames)
    if lenses is None and scene.lens is not None:
        lenses = [scene.lens] * n
    out = np.empty((n, rows, scene.c.width, 3), dtype=np.float32 if linear else np.uint8)
    st = rt_stats()
    o = C.byref(opts) if opts is not None else None
    o8, ol = (None, out.ctypes.data) if linear else (out.ctypes.data, None)
    if variance:
        var = np.empty((n, rows, scene.c.width, 3), dtype=np.float32)
        _check(lib().rtb200_render_frames_var(C.byref(scene.c), o, arr, _lens_array(lenses, n) if lenses is not None else None, n,
                                              o8, ol, var.ctypes.data, C.byref(st)))
        return out, var, st.as_dict()
    if lenses is None:
        _check(lib().rtb200_render_frames(C.byref(scene.c), o, arr, n, o8, ol, C.byref(st)))
    else:
        _check(lib().rtb200_render_frames_lens(C.byref(scene.c), o, arr, _lens_array(lenses, n), n, o8, ol, C.byref(st)))
    return out, st.as_dict()


def make_adaptive(rel_tol: float, abs_tol: float = 0.0, samples_per_round: int = 8, min_samples: int = 16,
                  max_samples: int = 0) -> rt_adaptive_params:
    return rt_adaptive_params(int(samples_per_round), int(max_samples), int(min_samples), 0, float(abs_tol), float(rel_tol))


def render_adaptive(scene: Scene, params: rt_adaptive_params, opts: Optional[rt_options] = None, variance: bool = False):
    """Render adaptively (rtb200_render_adaptive): rounds of params.samples_per_round samples of the pixels that have not
    converged, until none is left. A pixel that received n samples equals the one-shot render at samples_per_pixel = n.
    Returns (uint8 [rows,w,3], float32 linear [rows,w,3], uint32 counts [rows,w], stats dict); with variance=True
    (rtb200_render_adaptive_var) the variance of each pixel's mean, float32 [rows,w,3], comes before the stats. A lens scene is refused:
    render it adaptively through ResidentScene.adaptive_*."""
    _refuse_lens(scene, "render_adaptive")
    rows = scene.c.height if (opts is None or opts.world <= 1) else shard_rows(scene.c.height, opts.rank, opts.world, opts.band_rows)
    img = np.empty((rows, scene.c.width, 3), dtype=np.uint8)
    lin = np.empty((rows, scene.c.width, 3), dtype=np.float32)
    cnt = np.empty((rows, scene.c.width), dtype=np.uint32)
    st = rt_stats()
    o = C.byref(opts) if opts is not None else None
    if variance:
        var = np.empty((rows, scene.c.width, 3), dtype=np.float32)
        _check(lib().rtb200_render_adaptive_var(C.byref(scene.c), o, C.byref(params), img.ctypes.data, lin.ctypes.data,
                                                cnt.ctypes.data, var.ctypes.data, C.byref(st)))
        return img, lin, cnt, var, st.as_dict()
    _check(lib().rtb200_render_adaptive(C.byref(scene.c), o, C.byref(params), img.ctypes.data, lin.ctypes.data, cnt.ctypes.data,
                                        C.byref(st)))
    return img, lin, cnt, st.as_dict()


def _current_device() -> Optional[int]:
    """The caller's current CUDA device, which an upload without opts.device uses (None when torch is not installed)."""
    try:
        import torch
    except ImportError:
        return None
    return torch.cuda.current_device()


@functools.cache   # np.dtype(...).name costs microseconds, and every array of a call asks
def _torch_dtype(dtype):
    """The torch dtype of a numpy type (float64, float32, int32, uint32, uint8: torch names them alike)."""
    import torch
    return getattr(torch, np.dtype(dtype).name)


class _Arrays:
    """The arrays of one call of an entry point that has a host form (C-contiguous numpy arrays; the library stages them and
    waits) and a device form (contiguous CUDA tensors on one device, on a stream). Unless `host` fixes the form, the first
    array checked picks it; in the device form that array's device is the call's, unless `device` (an ordinal) fixes it."""

    def __init__(self, what: str, host: Optional[bool] = None, device: Optional[int] = None):
        self.what, self.host, self.device = what, host, device

    def ptr(self, a):
        """The address of a numpy array or a tensor of the call's form; None for None."""
        if a is None:
            return None
        return a.ctypes.data if self.host else a.data_ptr()

    def arg(self, name: str, a, dtypes, shape, optional: bool = False):
        """ptr(a) once `a` (None too when `optional`) is an array of the call's form and device with a dtype of `dtypes` (numpy
        types) and `shape`: a tuple, where "n" stands for a length no array has, or an int, a number of elements in any shape.
        Raises ValueError naming `name` otherwise."""
        if a is None and optional:
            return None
        if self.host is None:
            self.host = isinstance(a, np.ndarray)
        if self.host:
            ok = isinstance(a, np.ndarray) and a.dtype in dtypes and a.flags.c_contiguous
        else:
            import torch
            ok = isinstance(a, torch.Tensor) and a.is_cuda and a.dtype in [_torch_dtype(d) for d in dtypes] and a.is_contiguous()
            if ok and self.device is None:
                self.device = a.device.index
            ok = ok and a.device.index == self.device
        if not ok or (math.prod(a.shape) != shape if isinstance(shape, int) else tuple(a.shape) != shape):
            kind = "C-contiguous numpy array" if self.host else "contiguous CUDA tensor" + (f" on cuda:{self.device}" if self.device is not None else "")
            want = f"{shape} elements" if isinstance(shape, int) else "shape [" + ", ".join(map(str, shape)) + "]"
            raise ValueError(f"{self.what}: {name} must be a {kind} of {'/'.join(np.dtype(d).name for d in dtypes)} with {want}, got "
                             f"{type(a).__name__} {getattr(a, 'dtype', '')} {tuple(getattr(a, 'shape', ()))} {getattr(a, 'device', '')}")
        return self.ptr(a)

    def empty(self, outs, stream=None) -> dict:
        """{name: a new array} of the outputs `outs` (name, shape, numpy dtype): numpy arrays in the host form; in the device
        form tensors on the call's device, allocated on `stream` when it is a torch stream (the caching allocator then orders
        their reuse after the call), else on the device's current stream."""
        if self.host:
            return {k: np.empty(s, dtype=d) for k, s, d in outs}
        import torch
        device = torch.device("cuda", self.device)
        with torch.cuda.stream(stream) if isinstance(stream, torch.cuda.Stream) else torch.cuda.device(device):
            return {k: torch.empty(s, dtype=_torch_dtype(d), device=device) for k, s, d in outs}


def _rays(A: _Arrays, origin, direction, t_max):
    """rt_rays and n of a query's rays, checked by A: origin and direction float64 [n, 3], t_max float64 [n] or None."""
    n = origin.shape[0] if getattr(origin, "ndim", 0) == 2 else "n"
    f64 = (np.float64,)
    return rt_rays(A.arg("origin", origin, f64, (n, 3)), A.arg("direction", direction, f64, (n, 3)), A.arg("t_max", t_max, f64, (n,), True)), n


def _points(A: _Arrays, point, bound, optional: bool):
    """rt_points and n of a point query, checked by A: point float64 [n, 3], bound float64 [n] (None when `optional`)."""
    n = point.shape[0] if getattr(point, "ndim", 0) == 2 else "n"
    f64 = (np.float64,)
    return rt_points(A.arg("point", point, f64, (n, 3)), A.arg("bound", bound, f64, (n,), optional)), n


class ResidentScene:
    """Scene kept in HBM between frames (rtb200_scene_upload / rtb200_render_device)."""

    def __init__(self, scene: Scene, opts: Optional[rt_options] = None):
        self.scene = scene
        self.opts = opts
        self.h = C.c_void_p()
        _check(lib().rtb200_scene_upload(C.byref(scene.c), C.byref(opts) if opts is not None else None, C.byref(self.h)))
        self.rows = scene.c.height if (opts is None or opts.world <= 1) else shard_rows(scene.c.height, opts.rank, opts.world, opts.band_rows)
        self.n = scene.n_spheres
        self.device = opts.device if opts is not None and opts.device >= 0 else _current_device()   # None: unknown without torch
        self.lens = None
        if scene.lens is not None:
            self.set_lens(scene.lens)

    def set_lens(self, lens: Optional[rt_lens]):
        """The lens of every later camera ray of this handle (rtb200_scene_set_lens; None: pinhole). An adaptive render has
        to begin again after it."""
        _check(lib().rtb200_scene_set_lens(self.h, C.byref(lens) if lens is not None else None))
        self.lens = rt_lens.from_buffer_copy(lens) if lens is not None and lens.radius != 0.0 else None

    def render(self, dev_rgb8_ptr: int = 0, dev_linear_ptr: int = 0, stream: int = 0) -> dict:
        st = rt_stats()
        _check(lib().rtb200_render_device(self.h, C.c_void_p(dev_rgb8_ptr or None), C.c_void_p(dev_linear_ptr or None),
                                          C.c_void_p(stream or None), C.byref(st)))
        return st.as_dict()

    def render_async(self, dev_rgb8_ptr: int = 0, dev_linear_ptr: int = 0, stream: int = 0):
        """Enqueue a frame without waiting (frame loops); pair with :meth:`wait`."""
        _check(lib().rtb200_render_device_async(self.h, C.c_void_p(dev_rgb8_ptr or None), C.c_void_p(dev_linear_ptr or None), C.c_void_p(stream or None)))

    def wait(self) -> dict:
        st = rt_stats()
        _check(lib().rtb200_render_device_wait(self.h, C.byref(st)))
        return st.as_dict()

    def render_frames(self, frames: Sequence[rt_frame], dev_rgb8_ptr: int = 0, dev_linear_ptr: int = 0, stream: int = 0,
                      lenses: Optional[Sequence[rt_lens]] = None, variance: int = 0) -> dict:
        """Render len(frames) frames into device buffers of n * rows * w * 3 elements (blocking; the handle's own camera,
        seed and max_depth stay as uploaded). lenses: frame i's lens (rtb200_render_frames_lens_device); None: the handle's.
        variance: the address of a float32 device buffer of n * rows * w * 3 elements for the variance of each pixel's mean
        (rtb200_render_frames_var_device); 0: none."""
        arr, n = _frame_array(frames)
        st = rt_stats()
        if variance:
            _check(lib().rtb200_render_frames_var_device(self.h, arr, _lens_array(lenses, n), n, C.c_void_p(dev_rgb8_ptr or None),
                                                         C.c_void_p(dev_linear_ptr or None), C.c_void_p(int(variance)),
                                                         C.c_void_p(stream or None), C.byref(st)))
            return st.as_dict()
        _check(lib().rtb200_render_frames_lens_device(self.h, arr, _lens_array(lenses, n), n, C.c_void_p(dev_rgb8_ptr or None), C.c_void_p(dev_linear_ptr or None),
                                                 C.c_void_p(stream or None), C.byref(st)))
        return st.as_dict()

    def update_spheres(self, indices: Sequence[int], spheres: Sequence[rt_sphere], stream: int = 0):
        """Replace spheres indices[k] by spheres[k] (centre, radius, material) without rebuilding the hierarchy
        (rtb200_scene_update_spheres). Stream-ordered: frames enqueued before see the old scene, frames enqueued after the new."""
        if len(indices) != len(spheres):
            raise ValueError(f"{len(indices)} indices but {len(spheres)} spheres")
        idx = np.ascontiguousarray(indices, dtype=np.uint32)
        arr = (rt_sphere * max(len(spheres), 1))(*spheres)
        _check(lib().rtb200_scene_update_spheres(self.h, idx.ctypes.data if idx.size else None, arr, len(spheres), C.c_void_p(stream or None)))

    def update_geometry(self, t, stream=None):
        """Replace the centre and radius of every sphere from a contiguous float64 CUDA tensor [n_spheres, 4] of
        {cx, cy, cz, radius} on the handle's device (rtb200_scene_update_geometry_device); materials stay. Runs on `stream`
        (a torch.cuda.Stream, or a cudaStream_t handle where 0 is the library's own stream, as in :meth:`render`), by default
        torch's current stream, so `t` may be computed on it just before and released just after."""
        A = _Arrays("update_geometry", False, self.device)
        _check(lib().rtb200_scene_update_geometry_device(self.h, A.arg("t", t, (np.float64,), (self.n, 4)), self._stream(stream, A.device)))

    def _stream(self, stream, device):
        """The cudaStream_t argument of `stream` (see :meth:`update_geometry`; handle 0 is NULL, the library's own stream);
        None: torch's current stream on `device`."""
        if stream is None:
            import torch
            stream = torch.cuda.current_stream(device)
        return C.c_void_p(((stream.cuda_stream or CUDA_STREAM_LEGACY) if hasattr(stream, "cuda_stream") else int(stream)) or None)

    def rebuild(self, stream=None):
        """Rebuild the hierarchy from the current spheres on the GPU (rtb200_scene_rebuild): a new topology for spheres that
        moved, ordered like an update on `stream` (as in :meth:`update_geometry`, by default torch's current stream). Returns
        when the new tree exists; later frames trace it and later updates refit it. A no-op without a hierarchy."""
        _check(lib().rtb200_scene_rebuild(self.h, self._stream(stream, self.device)))

    def edit_spheres(self, remove: Sequence[int] = (), insert: Sequence[rt_sphere] = (), at: Optional[Sequence[int]] = None, stream=None):
        """Remove the spheres `remove` and place insert[k] just before old sphere at[k] (None: append every insert), on the GPU
        (rtb200_scene_edit_spheres): the list of :meth:`Scene.edited`, lights included. Ordered like :meth:`rebuild` on
        `stream`; returns when the new list and its hierarchy exist, and later calls see n spheres of the new list."""
        rem = np.ascontiguousarray(remove, dtype=np.uint32)
        pos = None if at is None else np.ascontiguousarray(at, dtype=np.uint32)
        if pos is not None and pos.size != len(insert):
            raise ValueError(f"{pos.size} positions for {len(insert)} inserts")
        arr = (rt_sphere * max(len(insert), 1))(*insert)
        _check(lib().rtb200_scene_edit_spheres(self.h, rem.ctypes.data if rem.size else None, rem.size,
                                               pos.ctypes.data if pos is not None and pos.size else None, arr, len(insert),
                                               self._stream(stream, self.device)))
        self.n += len(insert) - rem.size

    def adaptive_begin(self, params: rt_adaptive_params, stream=None):
        """(Re)start an adaptive render of the handle (rtb200_adaptive_begin): n = 0 everywhere, every pixel active. `stream`
        as in :meth:`update_geometry`."""
        _check(lib().rtb200_adaptive_begin(self.h, C.byref(params), self._stream(stream, self.device)))

    def adaptive_step(self, rounds: int = 1, stream=None):
        """Run up to `rounds` rounds and wait (rtb200_adaptive_step). Returns (pixels still active, stats summed over the
        rounds)."""
        active = C.c_uint32(); st = rt_stats()
        _check(lib().rtb200_adaptive_step(self.h, int(rounds), self._stream(stream, self.device), C.byref(active), C.byref(st)))
        return int(active.value), st.as_dict()

    def adaptive_resolve(self, rgb8=None, linear=None, counts=None, stream=None, variance=None):
        """Write the current adaptive image into CUDA tensors (rtb200_adaptive_resolve), each optional: uint8 rgb8 and float32
        linear of rows * w * 3 elements, int32 or uint32-sized counts of rows * w elements, on the handle's device. variance: a
        float32 tensor of rows * w * 3 elements for the variance of each pixel's mean (rtb200_adaptive_resolve_var)."""
        n = self.rows * self.scene.c.width
        A = _Arrays("adaptive_resolve", False, self.device)
        ptrs = [A.arg("rgb8", rgb8, (np.uint8,), 3 * n, True), A.arg("linear", linear, (np.float32,), 3 * n, True),
                A.arg("counts", counts, (np.int32,), n, True)]
        if variance is not None:
            pv = A.arg("variance", variance, (np.float32,), 3 * n)
            _check(lib().rtb200_adaptive_resolve_var(self.h, *ptrs, pv, self._stream(stream, self.device)))
            return
        _check(lib().rtb200_adaptive_resolve(self.h, *ptrs, self._stream(stream, self.device)))

    def intersect(self, origin, direction, t_max=None, stream=None, outputs=None) -> dict:
        """Closest hits of caller-supplied rays on the handle's current spheres: for ray i, hit_world(world, Ray{origin[i],
        direction[i]}, 0.001, t_max[i]) (f64::MAX without t_max) as include/rtb200.h states it, bit for bit, in every variant.

        CUDA tensors (contiguous float64 [n, 3], [n, 3] and [n], on the handle's device) use the device form
        (rtb200_scene_intersect_device) on `stream` (as in :meth:`update_geometry`, by default torch's current stream), without
        waiting: the query sees every update enqueued before it, and updates enqueued after it wait for it. numpy arrays use
        the blocking host form (rtb200_scene_intersect) and the result also holds "stats".

        Returns a dict of tensors or arrays, one per name of `outputs` (default: all): "t" [n] (+inf: miss), "sphere" int32 [n]
        (-1: miss, the bits of 0xffffffff), "point" and "normal" [n, 3], "uv" [n, 2], "front_face" uint8 [n]."""
        names = [f[0] for f in HIT_FIELDS] if outputs is None else list(outputs)
        unknown = [k for k in names if k not in dict((f[0], f) for f in HIT_FIELDS)]
        if unknown or not names:
            raise ValueError(f"intersect outputs are a non-empty subset of {[f[0] for f in HIT_FIELDS]}, got {names}")
        A = _Arrays("intersect", device=self.device)
        rays, n = _rays(A, origin, direction, t_max)
        out = A.empty([(k, (n, c) if c > 1 else (n,), ty) for k, c, ty in HIT_FIELDS if k in names], stream)
        hits = rt_hits(*(A.ptr(out.get(k)) for k, _, _ in HIT_FIELDS))
        if A.host:
            st = rt_stats()
            _check(lib().rtb200_scene_intersect(self.h, C.byref(rays), n, C.byref(hits), C.byref(st)))
            out["stats"] = st.as_dict()
        elif n:
            _check(lib().rtb200_scene_intersect_device(self.h, C.byref(rays), n, C.byref(hits), self._stream(stream, A.device)))
        return out

    def occluded(self, origin, direction, t_max=None, stream=None) -> dict:
        """Occlusion of caller-supplied rays on the handle's current spheres: for ray i, 1 if hit_world(world, Ray{origin[i],
        direction[i]}, 0.001, t_max[i]) (f64::MAX without t_max) is Some, else 0, as include/rtb200.h states it, in every
        variant. It equals intersect(...)["sphere"] != -1 under the same t_max, but the traversal skips boxes beyond t_max and
        stops at the first sphere that is hit below it. A segment from a to b is origin a, direction b - a, t_max 1.

        CUDA tensors use the device form (rtb200_scene_occluded_device) and numpy arrays the blocking host form
        (rtb200_scene_occluded), with the same arguments, checks and stream ordering as :meth:`intersect`. Returns
        {"occluded": uint8 [n]}, and with numpy arrays also "stats"."""
        A = _Arrays("occluded", device=self.device)
        rays, n = _rays(A, origin, direction, t_max)
        out = A.empty([("occluded", (n,), np.uint8)], stream)
        if A.host:
            st = rt_stats()
            _check(lib().rtb200_scene_occluded(self.h, C.byref(rays), n, A.ptr(out["occluded"]), C.byref(st)))
            out["stats"] = st.as_dict()
        elif n:
            _check(lib().rtb200_scene_occluded_device(self.h, C.byref(rays), n, A.ptr(out["occluded"]), self._stream(stream, A.device)))
        return out

    def nearest(self, points, bound=None, stream=None, outputs=None) -> dict:
        """The nearest of the handle's current spheres to each point, as include/rtb200.h states it, in every variant: the
        sphere j with dist_j = fl(|p - c_j|) - |R_j| below bound[i] (+inf without a bound) and the least dist_j, the lowest
        index among equal distances. Negative inside a sphere.

        CUDA tensors (contiguous float64 [n, 3] and [n], on the handle's device) use the device form
        (rtb200_scene_nearest_device) on `stream`, numpy arrays the blocking host form (rtb200_scene_nearest), with the
        arguments, checks and stream ordering of :meth:`intersect`. Returns a dict with one entry per name of `outputs`
        (default: both): "sphere" int32 [n] (-1: none) and "distance" float64 [n] (+inf: none); numpy arrays add "stats"."""
        fields = (("distance", np.float64), ("sphere", np.int32))
        names = [f[0] for f in fields] if outputs is None else list(outputs)
        if not names or any(k not in dict(fields) for k in names):
            raise ValueError(f"nearest outputs are a non-empty subset of {[f[0] for f in fields]}, got {names}")
        A = _Arrays("nearest", device=self.device)
        q, n = _points(A, points, bound, True)
        out = A.empty([(k, (n,), ty) for k, ty in fields if k in names], stream)
        res = rt_nearest(A.ptr(out.get("distance")), A.ptr(out.get("sphere")))
        if A.host:
            st = rt_stats()
            _check(lib().rtb200_scene_nearest(self.h, C.byref(q), n, C.byref(res), C.byref(st)))
            out["stats"] = st.as_dict()
        elif n:
            _check(lib().rtb200_scene_nearest_device(self.h, C.byref(q), n, C.byref(res), self._stream(stream, A.device)))
        return out

    def overlaps(self, centers, radii, stream=None) -> dict:
        """Whether each ball (centers[i], radii[i]) overlaps one of the handle's current spheres: 1 iff some dist_j < radii[i]
        (touching does not count), bit for bit nearest(centers, radii)["sphere"] != -1, but the traversal stops at the first
        such sphere. Forms, checks and stream ordering as :meth:`nearest`. Returns {"overlaps": uint8 [n]}, and with numpy
        arrays also "stats"."""
        A = _Arrays("overlaps", device=self.device)
        q, n = _points(A, centers, radii, False)
        out = A.empty([("overlaps", (n,), np.uint8)], stream)
        if A.host:
            st = rt_stats()
            _check(lib().rtb200_scene_overlaps(self.h, C.byref(q), n, A.ptr(out["overlaps"]), C.byref(st)))
            out["stats"] = st.as_dict()
        elif n:
            _check(lib().rtb200_scene_overlaps_device(self.h, C.byref(q), n, A.ptr(out["overlaps"]), self._stream(stream, A.device)))
        return out

    def trace_rays(self, origin, direction, samples: int = 1, *, sample0: int = 0, stream0: int = 0, seed: Optional[int] = None,
                   max_depth: Optional[int] = None, linear: bool = True, rgb8: bool = False, stream=None) -> dict:
        """Radiance of caller-supplied primary rays on the handle's current spheres, as include/rtb200.h states it: `samples`
        samples of ray_color(Ray{origin[i], direction[i]}, max_depth, max_depth) per ray, sample j drawing from the RNG stream
        of (pixel stream0 + i, sample sample0 + j) past the render's two jitter draws, resolved like a render with spp =
        samples. Bit for bit in every variant; seed and max_depth default to the scene's own.

        CUDA tensors (contiguous float64 [n, 3], on the handle's device) use the device form (rtb200_scene_trace_rays_device)
        on `stream` (as in :meth:`update_geometry`, by default torch's current stream); numpy arrays use the host form
        (rtb200_scene_trace_rays). Both block until the outputs are written. Returns {"linear": float32 [n, 3]} and/or
        {"rgb8": uint8 [n, 3]}, whichever is asked for, and "stats"."""
        if not (linear or rgb8):
            raise ValueError("trace_rays: ask for linear, rgb8 or both")
        p = rt_trace_params(self.scene.seed if seed is None else int(seed), int(samples), int(sample0), int(stream0),
                            self.scene.c.max_depth if max_depth is None else int(max_depth))
        st = rt_stats()
        A = _Arrays("trace_rays", device=self.device)
        rays, n = _rays(A, origin, direction, None)
        out = A.empty(([("linear", (n, 3), np.float32)] if linear else []) + ([("rgb8", (n, 3), np.uint8)] if rgb8 else []), stream)
        lin_p, rgb_p = A.ptr(out.get("linear")), A.ptr(out.get("rgb8"))
        if n == 0:   # nothing to trace (the library's no-op)
            pass
        elif A.host:
            _check(lib().rtb200_scene_trace_rays(self.h, C.byref(rays), n, C.byref(p), lin_p, rgb_p, C.byref(st)))
        else:
            _check(lib().rtb200_scene_trace_rays_device(self.h, C.byref(rays), n, C.byref(p), lin_p, rgb_p,
                                                        self._stream(stream, A.device), C.byref(st)))
        out["stats"] = st.as_dict()
        return out

    def aov(self, samples: int = 1, *, sample0: int = 0, view: Optional[rt_frame] = None, outputs=None, on_device: bool = False,
            stream=None) -> dict:
        """Auxiliary buffers of the render's camera samples [sample0, sample0 + samples) of every pixel of the handle's rows, as
        include/rtb200.h states them: for each sample the render's primary ray and its first hit on the current spheres, then
        per pixel the mean albedo at the hit (the sky on a miss) and the mean normal (0 on a miss; not renormalised), the
        samples that hit, and the sphere and hit point of sample sample0. `view` (an rt_frame) replaces the handle's camera
        and seed, like a frame of :meth:`render_frames`.

        With on_device=False the blocking host form (rtb200_scene_aov) returns numpy arrays and "stats"; with on_device=True
        the device form (rtb200_scene_aov_device) returns CUDA tensors on `stream` (as in :meth:`update_geometry`, by default
        torch's current stream) without waiting. Returns one entry per name of `outputs` (default: all): "albedo" and
        "normal" float32 [rows, w, 3], "hits" uint32 [rows, w], "sphere" int32 [rows, w] (-1: miss, the bits of 0xffffffff),
        "point" float64 [rows, w, 3]."""
        names = [f[0] for f in AOV_FIELDS] if outputs is None else list(outputs)
        if not names or any(k not in [f[0] for f in AOV_FIELDS] for k in names):
            raise ValueError(f"aov outputs are a non-empty subset of {[f[0] for f in AOV_FIELDS]}, got {names}")
        shape = (self.rows, int(self.scene.c.width))
        p = rt_aov_params(int(samples), int(sample0))
        vp = C.byref(view) if view is not None else None
        device = self.device
        if on_device and device is None:
            import torch
            device = torch.cuda.current_device()
        A = _Arrays("aov", not on_device, device)
        out = A.empty([(k, shape + ((c,) if c > 1 else ()), ty) for k, c, ty in AOV_FIELDS if k in names], stream)
        o = rt_aov_out(*(A.ptr(out.get(k)) for k, _, _ in AOV_FIELDS))
        if A.host:
            st = rt_stats()
            _check(lib().rtb200_scene_aov(self.h, C.byref(p), vp, C.byref(o), C.byref(st)))
            out["stats"] = st.as_dict()
        elif self.rows:   # a shard with no rows is the library's no-op
            _check(lib().rtb200_scene_aov_device(self.h, C.byref(p), vp, C.byref(o), self._stream(stream, device)))
        return out

    def topology(self) -> dict:
        """The handle's current topology (rtb200_scene_debug_topology): recentre, leaf_id [n_leaves, k], always, skip_pos,
        level_nodes (deepest level first) and level_off, the upload's or the last rebuild's."""
        g = (C.c_double * 3)(); info = (C.c_uint32 * 8)()
        _check(lib().rtb200_scene_debug_topology(self.h, g, info, None, 0, None, 0, None, 0, None, 0, None, 0))
        n_nodes, n_leaves, depth, k, n_always = (int(x) for x in info[:5])
        ids = np.zeros(max(n_leaves * k, 1), np.uint32); always = np.zeros(max(n_always, 1), np.uint32)
        skip = np.zeros(max(self.n, 1), np.uint32); ln = np.zeros(max(n_nodes, 1), np.uint32); lo = np.zeros(depth + 1, np.uint32)
        _check(lib().rtb200_scene_debug_topology(self.h, g, info, ids.ctypes.data, ids.size, always.ctypes.data, always.size,
                                                 skip.ctypes.data, skip.size, ln.ctypes.data, ln.size, lo.ctypes.data, lo.size))
        return {"n": self.n, "leaf_size": k, "n_nodes": n_nodes, "n_leaves": n_leaves, "depth": depth, "recentre": np.array(g[:]),
                "leaf_id": ids[: n_leaves * k].reshape(n_leaves, k), "always": always[:n_always], "skip_pos": skip,
                "level_nodes": ln[:n_nodes], "level_off": lo}

    def bvh_records(self) -> dict:
        """The handle's current arrays (rtb200_scene_debug_records) in the layout of :func:`bvh_records`, plus "geo"
        (float64 [n, 4]) and the topology of :meth:`topology` (leaf_id, always, recentre, skip_pos, level order)."""
        b = self.topology()
        info = (C.c_uint32 * 8)()
        _check(lib().rtb200_scene_debug_records(self.h, info, None, 0, None, 0, None, 0, None, 0))
        n_nodes, n_leaves, depth, k, n_always, fpn, n_pairs, _ = (int(x) for x in info)
        nodes = np.zeros(max(n_nodes * fpn, 1), np.float32); rec = np.zeros(max(n_leaves * k * 4, 1), np.float32)
        flat = np.zeros(max(n_pairs * 8, 1), np.float32); geo = np.zeros(max(self.n * 4, 1), np.float64)
        _check(lib().rtb200_scene_debug_records(self.h, info, nodes.ctypes.data, nodes.size, rec.ctypes.data, rec.size,
                                                flat.ctypes.data, flat.size, geo.ctypes.data, geo.size))
        b.update(_record_views(info, nodes, rec, flat))
        b["geo"] = geo[: self.n * 4].reshape(self.n, 4)
        return b

    def kernel_info(self) -> dict:
        ki = rt_kernel_info()
        _check(lib().rtb200_scene_kernel_info(self.h, C.byref(ki)))
        return ki.as_dict()

    def release(self):
        if self.h:
            lib().rtb200_scene_release(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def _call_stream(stream, device, what: str, buffers: str):
    """The torch stream and the cudaStream_t handle a device-form call on `device` runs on: `stream` (a torch.cuda.Stream, a
    nonzero handle, CUDA_STREAM_LEGACY for torch's default stream) or by default torch's current stream. The library's own
    stream (0) is refused: torch could not order the reuse of `buffers` it allocates for the call after the call."""
    import torch
    if stream is None:
        stream = torch.cuda.current_stream(device)
    elif not isinstance(stream, torch.cuda.Stream):
        if int(stream) == 0:
            raise ValueError(f"{what} on CUDA tensors takes a torch stream or a nonzero cudaStream_t: the library's own stream "
                             f"(0) cannot order the reuse of {buffers} torch allocates")
        stream = torch.cuda.default_stream(device) if int(stream) == CUDA_STREAM_LEGACY else torch.cuda.ExternalStream(int(stream), device=device)
    return stream, stream.cuda_stream or CUDA_STREAM_LEGACY


# the denoise's defaults, include/rtb200.h's RTB200_DENOISE_DEFAULT_* (DESIGN.md §4.15: chosen on the oracle's 2-spp cover render at
# 64x48 with its AOV guides)
DENOISE_ITERATIONS, DENOISE_COLOR_WEIGHT, DENOISE_ALBEDO_WEIGHT, DENOISE_NORMAL_WEIGHT = 3, 16.0, 4.0, 1.0


def denoise(color, albedo=None, normal=None, *, iterations: int = DENOISE_ITERATIONS, color_weight: float = DENOISE_COLOR_WEIGHT,
            albedo_weight: Optional[float] = None, normal_weight: Optional[float] = None, linear: bool = True, rgb8: bool = False,
            stream=None) -> dict:
    """Denoise a [h, w, 3] float32 image (normally a render's linear mean) with the edge-avoiding à-trous filter of
    include/rtb200.h, guided by the optional albedo and normal of :meth:`ResidentScene.aov`. A guide's weight defaults to
    DENOISE_ALBEDO_WEIGHT / DENOISE_NORMAL_WEIGHT when the guide is given and to 0 (off) when it is not.

    numpy arrays use the blocking host form (rtb200_denoise) and the result also holds "stats". CUDA tensors (contiguous, on one
    device) use the device form (rtb200_denoise_device) on `stream` without waiting: a torch.cuda.Stream, a nonzero
    cudaStream_t handle (CUDA_STREAM_LEGACY is torch's default stream), or by default torch's current stream. The scratch and
    the outputs are allocated by torch on that stream, so the caching allocator hands the scratch to no other stream's
    allocation before the call has run; the library's own stream (handle 0) is refused for that reason. Returns
    {"linear": float32 [h, w, 3]} and/or {"rgb8": uint8 [h, w, 3]}, whichever is asked for."""
    if not (linear or rgb8):
        raise ValueError("denoise: ask for linear, rgb8 or both")
    if albedo_weight is None:
        albedo_weight = DENOISE_ALBEDO_WEIGHT if albedo is not None else 0.0
    if normal_weight is None:
        normal_weight = DENOISE_NORMAL_WEIGHT if normal is not None else 0.0
    shape = tuple(color.shape)
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"denoise: color must have shape [h, w, 3], got {shape}")
    A = _Arrays("denoise")
    guides = [A.arg(name, g, (np.float32,), shape, name != "color") for name, g in (("color", color), ("albedo", albedo), ("normal", normal))]
    p = rt_denoise_params(shape[1], shape[0], int(iterations), 0, float(color_weight), float(albedo_weight), float(normal_weight), 0.0)
    outs = [(k, shape, ty) for k, ty, want in (("linear", np.float32, linear), ("rgb8", np.uint8, rgb8)) if want]
    if A.host:
        out = A.empty(outs)
        st = rt_stats()
        _check(lib().rtb200_denoise(-1, C.byref(p), *guides, A.ptr(out.get("linear")), A.ptr(out.get("rgb8")), C.byref(st)))
        out["stats"] = st.as_dict()
        return out
    stream, handle = _call_stream(stream, A.device, "denoise", "the scratch")
    # the scratch and the outputs belong to the call's stream: the caching allocator reuses the scratch, freed when this
    # function returns, only for later work on that stream, which runs after the call
    out = A.empty(outs + [("scratch", (int(lib().rtb200_denoise_scratch_bytes(shape[1], shape[0])),), np.uint8)], stream)
    scratch = out.pop("scratch")
    if color.numel() == 0:   # a 0-pixel image (the library's no-op)
        return out
    _check(lib().rtb200_denoise_device(A.device, C.byref(p), *guides, A.ptr(scratch), A.ptr(out.get("linear")), A.ptr(out.get("rgb8")),
                                       C.c_void_p(handle)))
    return out


# the variance-guided denoise's defaults, include/rtb200.h's RTB200_DENOISE_VAR_DEFAULT_* (DESIGN.md §4.18: chosen on the oracle's
# cover render at 64x48 from 2 to 32 spp with its AOV guides)
DENOISE_VAR_ITERATIONS, DENOISE_VAR_COLOR_WEIGHT, DENOISE_VAR_ALBEDO_WEIGHT, DENOISE_VAR_NORMAL_WEIGHT = 3, 1.0, 4.0, 1.0
DENOISE_VAR_VARIANCE_FLOOR = 1e-4


def denoise_var(color, variance, albedo=None, normal=None, *, iterations: int = DENOISE_VAR_ITERATIONS,
                color_weight: float = DENOISE_VAR_COLOR_WEIGHT, albedo_weight: Optional[float] = None,
                normal_weight: Optional[float] = None, variance_floor: float = DENOISE_VAR_VARIANCE_FLOOR, linear: bool = True,
                rgb8: bool = False, out_variance: bool = False, stream=None) -> dict:
    """Denoise a [h, w, 3] float32 image with its per-pixel variance (normally a render's linear mean and the variance of that
    mean) by the variance-guided à-trous filter of include/rtb200.h, guided by the optional albedo and normal of
    :meth:`ResidentScene.aov`. A guide's weight defaults to DENOISE_VAR_ALBEDO_WEIGHT / DENOISE_VAR_NORMAL_WEIGHT when the guide
    is given and to 0 (off) when it is not. numpy arrays use the blocking host form (rtb200_denoise_var) and the result also holds
    "stats"; CUDA tensors use the device form on `stream` with the stream rules of :func:`denoise`. Returns {"linear": float32
    [h, w, 3]}, {"rgb8": uint8 [h, w, 3]} and/or {"variance": float32 [h, w, 3]} (out_variance), whichever is asked for."""
    if not (linear or rgb8 or out_variance):
        raise ValueError("denoise_var: ask for linear, rgb8, out_variance or several")
    if albedo_weight is None:
        albedo_weight = DENOISE_VAR_ALBEDO_WEIGHT if albedo is not None else 0.0
    if normal_weight is None:
        normal_weight = DENOISE_VAR_NORMAL_WEIGHT if normal is not None else 0.0
    shape = tuple(color.shape)
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"denoise_var: color must have shape [h, w, 3], got {shape}")
    A = _Arrays("denoise_var")
    ins = [A.arg(name, g, (np.float32,), shape, name in ("albedo", "normal"))
           for name, g in (("color", color), ("variance", variance), ("albedo", albedo), ("normal", normal))]
    p = rt_denoise_var_params(shape[1], shape[0], int(iterations), 0, float(color_weight), float(albedo_weight), float(normal_weight),
                              float(variance_floor))
    outs = [(k, shape, ty) for k, ty, want in (("linear", np.float32, linear), ("rgb8", np.uint8, rgb8),
                                               ("variance", np.float32, out_variance)) if want]
    if A.host:
        out = A.empty(outs)
        st = rt_stats()
        _check(lib().rtb200_denoise_var(-1, C.byref(p), *ins, A.ptr(out.get("linear")), A.ptr(out.get("rgb8")),
                                        A.ptr(out.get("variance")), C.byref(st)))
        out["stats"] = st.as_dict()
        return out
    stream, handle = _call_stream(stream, A.device, "denoise_var", "the scratch")
    # the scratch and the outputs belong to the call's stream, as in denoise
    out = A.empty(outs + [("scratch", (int(lib().rtb200_denoise_var_scratch_bytes(shape[1], shape[0])),), np.uint8)], stream)
    scratch = out.pop("scratch")
    if color.numel() == 0:   # a 0-pixel image (the library's no-op)
        return out
    _check(lib().rtb200_denoise_var_device(A.device, C.byref(p), *ins, A.ptr(scratch), A.ptr(out.get("linear")),
                                           A.ptr(out.get("rgb8")), A.ptr(out.get("variance")), C.c_void_p(handle)))
    return out


# the temporal accumulation's defaults, include/rtb200.h's RTB200_TEMPORAL_DEFAULT_* (DESIGN.md §4.16: chosen on an orbit of the
# oracle's 2-spp cover render at 64x48)
TEMPORAL_MAX_HISTORY, TEMPORAL_DEPTH_TOL = 2, 0.03
# the history clamp's, RTB200_TEMPORAL_DEFAULT_CLAMP_* (DESIGN.md §4.20): `clamp=TEMPORAL_CLAMP_GAMMA` turns it on
TEMPORAL_CLAMP_GAMMA, TEMPORAL_CLAMP_RADIUS = 0.5, 1


def _camera_of(c) -> rt_camera:
    """An rt_camera, or the camera of an rt_frame."""
    c = c.camera if isinstance(c, rt_frame) else c
    if not isinstance(c, rt_camera):
        raise ValueError(f"a camera is an rt_camera or an rt_frame, got {type(c).__name__}")
    return c


def temporal(color, sphere, point, camera, prev: Optional[dict] = None, *, motion=None, max_history: int = TEMPORAL_MAX_HISTORY,
             depth_tol: float = TEMPORAL_DEPTH_TOL, clamp: Optional[float] = None, clamp_radius: int = TEMPORAL_CLAMP_RADIUS,
             variance=None, stream=None) -> dict:
    """Accumulate a frame over time (include/rtb200.h, rtb200_temporal[_device]): each pixel of `color` ([h, w, 3] float32,
    normally a render's linear mean) is reprojected into the previous frame through its first hit (`sphere` [h, w] int32 or
    uint32 with -1 / 0xffffffff for a miss, `point` [h, w, 3] float64: :meth:`ResidentScene.aov`'s, of the same camera) and
    blended with the history there where it shows the same surface. `camera` is this frame's rt_camera (or rt_frame).
    `prev` is None for the first frame, else a dict of the previous call's "color" and "length" and the previous frame's
    "sphere", "point" and "camera". `motion` ([n, 3] float64, may be None) is the displacement of sphere j since the previous
    frame; spheres j >= n did not move. `clamp` (None: off) is the history clamp's gamma: the history is clamped to the mean
    +- clamp standard deviations of this frame's colours in the window of radius `clamp_radius` around the pixel before the
    blend (rtb200_temporal_clamped[_device]); :data:`TEMPORAL_CLAMP_GAMMA` is the default width.

    numpy arrays use the blocking host form (rtb200_temporal) and the result also holds "stats". CUDA tensors (contiguous, on one
    device) use the device form (rtb200_temporal_device) on `stream` without waiting, with the stream rules of :func:`denoise`:
    the outputs are allocated by torch on the call's stream, and handle 0 is refused. Returns {"color": float32 [h, w, 3],
    "length": uint32 [h, w]}, the new history: pass it back as prev's "color" and "length" with the next frame.

    `variance` ([h, w, 3] float32, the variance of each pixel's mean, normally render_frames(variance=True)'s) carries the
    variance through the accumulation (rtb200_temporal_var[_device], DESIGN.md §4.21, clamped or not): prev must then hold the
    previous call's "variance" too, and the result adds "variance", the new history's. "color" and "length" are the same as
    without it."""
    return _temporal(color, sphere, point, camera, prev, motion, max_history, depth_tol, stream, None, _clamp(clamp, clamp_radius),
                     variance)


def _max_history(n) -> int:
    """max_history as the u32 of rt_temporal_params; a value outside [0, 2^32 - 1] would wrap, and is refused here (0 is the
    library's refusal)."""
    n = int(n)
    if not 0 <= n <= 0xFFFFFFFF:
        raise ValueError(f"max_history must be an integer in [1, 2^32 - 1], got {n}")
    return n


def _clamp(gamma, radius) -> Optional[rt_temporal_clamp]:
    """The rt_temporal_clamp of a gamma (None: no clamp) and a radius; a radius outside the u32 field is refused here, the rest by
    the library."""
    if gamma is None:
        return None
    radius = int(radius)
    if not 0 <= radius <= 0xFFFFFFFF:
        raise ValueError(f"clamp_radius must be an integer in [1, 3], got {radius}")
    return rt_temporal_clamp(float(gamma), radius)


def _temporal(color, sphere, point, camera, prev, motion, max_history, depth_tol, stream, out, clamp=None, variance=None):
    """temporal(), writing into `out` ({"color", "length"} CUDA tensors of the right shapes, and "variance" with `variance`) when
    it is given; clamp is an rt_temporal_clamp or None."""
    shape = tuple(color.shape)
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"temporal: color must have shape [h, w, 3], got {shape}")
    hw = shape[:2]
    prev = dict(prev) if prev is not None else None
    if prev is not None and not {"color", "length", "sphere", "point", "camera"} <= set(prev):
        raise ValueError("temporal: prev holds the previous frame's color, length, sphere, point and camera")
    if variance is not None and prev is not None and "variance" not in prev:
        raise ValueError("temporal: with variance, prev holds the previous call's variance too")
    A = _Arrays("temporal")
    f32, f64, u32, ids = (np.float32,), (np.float64,), (np.uint32,), (np.int32, np.uint32)
    cur = rt_temporal_frame(A.arg("color", color, f32, shape), A.arg("sphere", sphere, ids, hw), A.arg("point", point, f64, shape))
    hist = None
    if prev is not None:
        hist = rt_temporal_history(A.arg("prev color", prev["color"], f32, shape), A.arg("prev length", prev["length"], u32, hw),
                                   A.arg("prev sphere", prev["sphere"], ids, hw), A.arg("prev point", prev["point"], f64, shape))
    mp = A.arg("motion", motion, f64, (motion.shape[0] if motion is not None and len(motion.shape) == 2 else "n", 3), True)
    p = rt_temporal_params(hw[1], hw[0], _max_history(max_history), 0 if motion is None else int(motion.shape[0]), _camera_of(camera),
                           _camera_of(prev["camera"]) if prev is not None else rt_camera(), float(depth_tol))
    hp = C.byref(hist) if hist is not None else None
    outs = [("color", shape, np.float32), ("length", hw, np.uint32)]
    if variance is not None:
        vp = A.arg("variance", variance, f32, shape)
        pvp = A.arg("prev variance", prev["variance"], f32, shape) if prev is not None else None
        outs.append(("variance", shape, np.float32))
    cp = C.byref(clamp) if clamp is not None else None
    if A.host:
        out = A.empty(outs)
        st = rt_stats()
        o = C.byref(rt_temporal_out(A.ptr(out["color"]), A.ptr(out["length"])))
        if variance is not None:
            _check(lib().rtb200_temporal_var(-1, C.byref(p), cp, C.byref(cur), vp, hp, pvp, mp, o, A.ptr(out["variance"]), C.byref(st)))
        else:
            _check(lib().rtb200_temporal(-1, C.byref(p), C.byref(cur), hp, mp, o, C.byref(st)) if clamp is None else
                   lib().rtb200_temporal_clamped(-1, C.byref(p), C.byref(clamp), C.byref(cur), hp, mp, o, C.byref(st)))
        out["stats"] = st.as_dict()
        return out
    stream, handle = _call_stream(stream, A.device, "temporal", "the outputs")
    if out is None:
        out = A.empty(outs, stream)
    if color.numel() == 0:   # a 0-pixel image (the library's no-op)
        return out
    o = C.byref(rt_temporal_out(A.ptr(out["color"]), A.ptr(out["length"])))
    if variance is not None:
        _check(lib().rtb200_temporal_var_device(A.device, C.byref(p), cp, C.byref(cur), vp, hp, pvp, mp, o, A.ptr(out["variance"]),
                                                C.c_void_p(handle)))
    else:
        _check(lib().rtb200_temporal_device(A.device, C.byref(p), C.byref(cur), hp, mp, o, C.c_void_p(handle)) if clamp is None else
               lib().rtb200_temporal_clamped_device(A.device, C.byref(p), C.byref(clamp), C.byref(cur), hp, mp, o, C.c_void_p(handle)))
    return out


class TemporalDenoiser:
    """An animation's low-sample frames made stable and clean on the GPU: each :meth:`push` accumulates the frame over time
    (:func:`temporal`) and denoises the result (:func:`denoise`, guided by the frame's albedo and normal). It owns two history
    buffers, which its pushes ping-pong between, and copies of the previous frame's sphere and point, on the device;
    :meth:`reset` forgets the history (after an edit that renumbers spheres, or a cut). `clamp` and `clamp_radius` are
    :func:`temporal`'s history clamp (None: off).

    With `variance=True` each push also takes the variance of the frame's pixel means, carries it through the accumulation
    (:func:`temporal` with `variance`) and denoises by it (:func:`denoise_var`, with `variance_floor`). The denoise weights left
    unset are the chosen filter's defaults: DENOISE_* without the variance, DENOISE_VAR_* with it."""

    def __init__(self, *, max_history: int = TEMPORAL_MAX_HISTORY, depth_tol: float = TEMPORAL_DEPTH_TOL,
                 iterations: Optional[int] = None, color_weight: Optional[float] = None, albedo_weight: Optional[float] = None,
                 normal_weight: Optional[float] = None, clamp: Optional[float] = None, clamp_radius: int = TEMPORAL_CLAMP_RADIUS,
                 variance: bool = False, variance_floor: float = DENOISE_VAR_VARIANCE_FLOOR):
        self.max_history, self.depth_tol = _max_history(max_history), float(depth_tol)
        if self.max_history < 1:
            raise ValueError("max_history must be >= 1")
        self.clamp = _clamp(clamp, clamp_radius)
        if self.clamp is not None and not (math.isfinite(self.clamp.gamma) and self.clamp.gamma >= 0 and 1 <= self.clamp.radius <= 3):
            raise ValueError("clamp must be finite and >= 0 as a float32, and clamp_radius in [1, 3]")
        self.variance = bool(variance)
        defaults = ((DENOISE_VAR_ITERATIONS, DENOISE_VAR_COLOR_WEIGHT, DENOISE_VAR_ALBEDO_WEIGHT, DENOISE_VAR_NORMAL_WEIGHT) if self.variance
                    else (DENOISE_ITERATIONS, DENOISE_COLOR_WEIGHT, DENOISE_ALBEDO_WEIGHT, DENOISE_NORMAL_WEIGHT))
        given = (iterations, color_weight, albedo_weight, normal_weight)
        self.denoise_kw = {k: d if v is None else v for k, v, d in zip(("iterations", "color_weight", "albedo_weight", "normal_weight"), given, defaults)}
        if self.variance:
            self.denoise_kw["variance_floor"] = variance_floor
        self._hist = None      # two {"color", "length"[, "variance"]} buffers; push k writes _hist[k % 2] and reads the other as the history
        self._k = 0
        self._sphere = self._point = self._camera = self._stream = None
        self._has_prev = False

    def reset(self):
        self._has_prev = False

    def push(self, linear, aov: dict, camera, motion=None, stream=None, variance=None) -> dict:
        """One frame: `linear` [h, w, 3] float32 CUDA tensor, `aov` the frame's :meth:`ResidentScene.aov` on the device with
        albedo, normal, sphere and point, `camera` its rt_camera or rt_frame, `motion` the spheres' displacement since the
        previous push, and with variance=True `variance` the [h, w, 3] float32 variance of the frame's pixel means (required).
        Runs on `stream` (by default torch's current stream) after the previous push, on whichever stream it ran.
        Returns {"color": the accumulated image, "length": its history lengths, "denoised": the accumulated image denoised}, and
        with variance=True "variance": the accumulated image's variance.
        "color", "length" and "variance" are the denoiser's own history buffer: the next push reads it as its history and the push
        after that overwrites it, so do not write to them, and clone them to keep them."""
        import torch
        if self.variance != (variance is not None):
            raise ValueError("TemporalDenoiser.push: variance is required with variance=True and refused without it")
        stream, _ = _call_stream(stream, linear.device, "TemporalDenoiser.push", "the history")
        shape = tuple(linear.shape)
        hw = shape[:2]
        if self._stream is not None and self._stream != stream:
            stream.wait_stream(self._stream)   # the previous push's reads and writes of the buffers come first
        if self._hist is None or tuple(self._hist[0]["color"].shape) != shape or self._hist[0]["color"].device != linear.device:
            with torch.cuda.stream(stream):
                self._hist = [{"color": torch.empty(shape, dtype=torch.float32, device=linear.device),
                               "length": torch.empty(hw, dtype=torch.uint32, device=linear.device)} for _ in range(2)]
                if self.variance:
                    for hb in self._hist:
                        hb["variance"] = torch.empty(shape, dtype=torch.float32, device=linear.device)
                self._sphere = torch.empty(hw, dtype=torch.int32, device=linear.device)
                self._point = torch.empty(shape, dtype=torch.float64, device=linear.device)
            self._has_prev = False
        out = self._hist[self._k]
        prev = None
        if self._has_prev:
            h = self._hist[self._k ^ 1]
            prev = {"color": h["color"], "length": h["length"], "sphere": self._sphere, "point": self._point, "camera": self._camera}
            if self.variance:
                prev["variance"] = h["variance"]
        _temporal(linear, aov["sphere"], aov["point"], camera, prev, motion, self.max_history, self.depth_tol, stream, out, self.clamp,
                  variance)
        with torch.cuda.stream(stream):   # the next push's previous frame, after this push has read the current one
            self._sphere.view(aov["sphere"].dtype).copy_(aov["sphere"])
            self._point.copy_(aov["point"])
        self._camera = rt_camera.from_buffer_copy(_camera_of(camera))
        self._has_prev, self._k, self._stream = True, self._k ^ 1, stream
        if self.variance:
            den = denoise_var(out["color"], out["variance"], aov["albedo"], aov["normal"], stream=stream, **self.denoise_kw)
            return {"color": out["color"], "length": out["length"], "variance": out["variance"], "denoised": den["linear"]}
        den = denoise(out["color"], aov["albedo"], aov["normal"], stream=stream, **self.denoise_kw)
        return {"color": out["color"], "length": out["length"], "denoised": den["linear"]}


def write_png(path: str, rgb8: np.ndarray):
    """write_image (reference raytracer.rs:33-42): RGB8 PNG."""
    from PIL import Image

    Image.fromarray(np.ascontiguousarray(rgb8, dtype=np.uint8), "RGB").save(path, format="PNG")


def render(filename: str, scene: Scene, opts: Optional[rt_options] = None) -> dict:
    """`pub fn render(filename, scene)` (reference raytracer.rs:250-266): render, print the frame time, write the PNG."""
    img, st = render_rgb8(scene, opts)
    print(f"Frame time: {int(st['wall_ms'])}ms")
    write_png(filename, img)
    return st
