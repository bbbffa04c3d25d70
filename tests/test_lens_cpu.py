"""The thin-lens camera (DESIGN.md §4.17) without a GPU: the rt_lens layout, the camera's construction and refusals, the
focus plane, the lens draws' own RNG domain, the scene loader's defaults and the Python refusals of lens scenes."""
import ctypes as C
import math
import os
import re
import sys

import numpy as np
import pytest

import oracle_lens as OL
import oracle_trace_rays as OT
import rtb200 as R
from rtb200 import scenes
from test_aov_cpu import mixed_lit_scene, textured_sky_scene

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle"))
import oracle_py  # noqa: E402

INVALID = -1
COVER = dict(look_from=(13.0, 2.0, 3.0), look_at=(0.0, 0.0, 0.0), vup=(0.0, 1.0, 0.0), vfov=20.0, aspect=4.0 / 3.0)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def vec(v):
    return np.array([v.x, v.y, v.z])


def cam_arrays(c):
    return np.array([vec(c.origin), vec(c.lower_left_corner), vec(c.horizontal), vec(c.vertical)])


def with_lens(sc, aperture, focus_dist=None):
    sc.set_camera(aperture=aperture, focus_dist=focus_dist)
    return sc


def test_rt_lens_layout_matches_the_header():
    assert C.sizeof(R.rt_lens) == 64
    assert [getattr(R.rt_lens, n).offset for n, _ in R.rt_lens._fields_] == [0, 24, 48, 56]
    txt = open(os.path.join(REPO, "include", "rtb200.h")).read()
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct \{([^}]*)\} rt_lens;", txt).group(1), flags=re.S)
    assert [tuple(d.split()) for d in body.strip().rstrip(";").split(";")] == [("rt_vec3", "u,", "v"), ("double", "radius"), ("uint64_t", "reserved")]


@pytest.mark.parametrize("aperture", [0.0, 0.1, 2.5])
def test_focus_one_is_camera_new_bit_for_bit(aperture):
    cam0 = R.camera_from_params(**COVER)
    cam, lens = R.camera_from_params_lens(**COVER, aperture=aperture, focus_dist=1.0)
    assert bits(cam_arrays(cam)).tobytes() == bits(cam_arrays(cam0)).tobytes()
    assert lens.radius == aperture / 2.0 and lens.reserved == 0
    assert abs(np.linalg.norm(vec(lens.u)) - 1.0) < 1e-15 and abs(np.linalg.norm(vec(lens.v)) - 1.0) < 1e-15


@pytest.mark.parametrize("fd", [1.0, 10.0, 0.37, 1e5])
def test_library_camera_equals_the_oracle(fd):
    p = R.rt_camera_params(R.vec3(COVER["look_from"]), R.vec3(COVER["look_at"]), R.vec3(COVER["vup"]), COVER["vfov"], COVER["aspect"])
    cam_o, lens_o = R.rt_camera(), R.rt_lens()
    assert OL.lib().oracle_camera_lens(C.byref(p), 0.1, fd, C.byref(cam_o), C.byref(lens_o)) == 0
    cam, lens = R.camera_from_params_lens(**COVER, aperture=0.1, focus_dist=fd)
    assert bytes(cam) == bytes(cam_o) and bytes(lens) == bytes(lens_o)


@pytest.mark.parametrize("aperture,fd", [(-0.1, 10.0), (math.nan, 10.0), (math.inf, 10.0), (0.1, 0.0), (0.1, -1.0),
                                         (0.1, math.nan), (0.1, math.inf), (0.0, 0.0)])
def test_bad_aperture_or_focus_is_refused(aperture, fd):
    with pytest.raises(R.RtError) as e:
        R.camera_from_params_lens(**COVER, aperture=aperture, focus_dist=fd)
    assert e.value.code == INVALID


def test_focus_plane_is_sharp():
    """Every lens ray of one image position passes through its pinhole target llc + h*u + vt*v (a few ulps)."""
    cam, lens = R.camera_from_params_lens(**COVER, aperture=0.8, focus_dist=10.0)
    rng = np.random.default_rng(5)
    for _ in range(20):
        u, v = rng.random(2)
        target = vec(cam.lower_left_corner) + vec(cam.horizontal) * u + vec(cam.vertical) * v
        seen = set()
        for s in range(40):
            o, d, t = OL.lens_ray(cam, lens, 77, 123, s, u, v)
            assert t >= 1
            seen.add(tuple(o))
            assert np.max(np.abs((o + d) - target)) <= 8 * np.spacing(np.max(np.abs(target)))
            assert np.linalg.norm(o - vec(cam.origin)) < lens.radius
        assert len(seen) == 40   # the origins differ: the lens is sampled


def test_pinhole_lens_draws_nothing():
    cam = R.camera_from_params(**COVER)
    o, d, t = OL.lens_ray(cam, R.rt_lens(), 1, 2, 3, 0.25, 0.75)
    assert t == 0 and np.array_equal(o, vec(cam.origin))


@pytest.mark.parametrize("name", ["cover", "mixed_lit", "textured_sky"])
def test_lens_radiance_is_trace_rays_of_the_lens_rays(name):
    """The lens draws take nothing from the path's stream: the lens render is, sample by sample, ray_color of the sample's
    lens ray with the stream at its third draw (the trace_rays rule), summed in f32 in sample order times 1/spp."""
    sc = {"cover": lambda: scenes.cover_scene(20, 15, 3, depth=6), "mixed_lit": lambda: mixed_lit_scene(18, 12, 3),
          "textured_sky": lambda: textured_sky_scene(16, 12, 3)}[name]()
    p = sc.camera_params
    fd = 0.5 * R.focal_length(p["look_from"], p["look_at"])
    sc = with_lens(sc, 0.3, fd)
    assert sc.lens is not None
    want = OL.render(sc, sc.lens)
    spp = int(sc.c.samples_per_pixel)
    acc = np.zeros((int(sc.c.height) * int(sc.c.width), 3), np.float32)
    rays = 0
    for s in range(spp):
        o, d = OL.primary(sc, sc.lens, s)
        got = OT.trace_rays(sc, o, d, samples=1, sample0=s)
        acc = acc + got["linear"]
        rays += got["rays"]
    mean = np.float32(1.0) / np.float32(spp) * acc
    assert bits(mean.reshape(want["linear"].shape)).tobytes() == bits(want["linear"]).tobytes()
    assert rays == want["rays"]


def test_radius_zero_renders_the_pinhole_oracle():
    sc = mixed_lit_scene(16, 12, 2)
    lin, rgb, st = oracle_py.render(sc)
    got = OL.render(sc, R.rt_lens())
    assert bits(got["linear"]).tobytes() == bits(lin.reshape(got["linear"].shape)).tobytes()
    assert np.array_equal(got["rgb8"], rgb.reshape(got["rgb8"].shape))


def test_out_of_focus_blurs_more_than_in_focus():
    """One sphere on the focus plane, one far behind it: the lens changes the far sphere's pixels much more."""
    sc = scenes.cover_scene(48, 36, 8, depth=4)
    sc.c.n_spheres = 3
    s = sc._spheres
    s[0].center = R.vec3((0.0, -1000.0, 0.0)); s[0].radius = 1000.0
    s[1].center = R.vec3((3.0, 1.0, 1.5)); s[1].radius = 1.0   # distance ~10 from (13, 2, 3)
    s[2].center = R.vec3((-30.0, 4.0, -8.0)); s[2].radius = 4.0
    for k in (1, 2):
        s[k].kind = R.RT_LAMBERTIAN; s[k].albedo[:] = [0.9, 0.2, 0.1] if k == 1 else [0.1, 0.3, 0.9]
    sc.set_camera(look_at=(0.0, 1.0, 0.0))
    fd = float(np.linalg.norm(np.array([13.0, 2.0, 3.0]) - np.array([3.0, 1.0, 1.5])))
    pin = OL.render(sc, R.rt_lens())["linear"]
    first = OL.hits(sc, R.rt_lens(), samples=1)["sphere"]
    sc = with_lens(sc, 1.0, fd)
    lens = OL.render(sc, sc.lens)["linear"]
    diff = np.abs(lens - pin).sum(axis=2)
    near, far = diff[first == 1].mean(), diff[first == 2].mean()
    assert (first == 1).sum() > 20 and (first == 2).sum() > 20
    assert near < 0.35 * far, (near, far)


def test_loader_defaults(tmp_path):
    cfg = scenes.cover_config()
    cfg = dict(cfg, width=40, height=30, samples_per_pixel=2, max_depth=5)
    sc = R.Scene.from_config(cfg, scenes.SCENES_DIR)
    assert sc.lens is None and "aperture" not in sc.camera_params
    cam = dict(cfg["camera"], aperture=0.1)
    sc = R.Scene.from_config(dict(cfg, camera=cam), scenes.SCENES_DIR)
    lf, la = cam["look_from"], cam["look_at"]
    want_cam, want_lens = R.camera_from_params_lens(lf, la, cam["vup"], cam["vfov"], cam["aspect"], 0.1, R.focal_length(lf, la))
    assert bytes(sc.c.camera) == bytes(want_cam) and bytes(sc.lens) == bytes(want_lens)
    sc = R.Scene.from_config(dict(cfg, camera=dict(cam, focus_dist=10.0)), scenes.SCENES_DIR)
    assert bytes(sc.c.camera) == bytes(R.camera_from_params_lens(lf, la, cam["vup"], cam["vfov"], cam["aspect"], 0.1, 10.0)[0])
    sc = R.Scene.from_config(dict(cfg, camera=dict(cam, aperture=0.0, focus_dist=10.0)), scenes.SCENES_DIR)
    assert sc.lens is None and bytes(sc.c.camera) == bytes(R.camera_from_params(lf, la, cam["vup"], cam["vfov"], cam["aspect"]))
    # a frame: omitted fields are the scene's; no focus_dist anywhere is the frame's own |look_from - look_at|
    sc = R.Scene.from_config(dict(cfg, camera=cam), scenes.SCENES_DIR)
    f, L = R.make_frame_lens(sc, look_from=(6.0, 2.0, 1.0))
    want = R.camera_from_params_lens((6.0, 2.0, 1.0), la, cam["vup"], cam["vfov"], cam["aspect"], 0.1, R.focal_length((6.0, 2.0, 1.0), la))
    assert bytes(f.camera) == bytes(want[0]) and bytes(L) == bytes(want[1])
    f, L = R.make_frame_lens(sc, aperture=0.0)
    assert L.radius == 0.0


def test_hosts_without_a_lens_refuse_a_lens_scene():
    sc = with_lens(scenes.cover_scene(16, 12, 1), 0.1, 10.0)
    with pytest.raises(R.RtError):
        R.render_rgb8_multi(sc)
    with pytest.raises(R.RtError):
        R.render_adaptive(sc, R.make_adaptive(0.1))


def test_make_frame_of_a_lens_scene_is_focused_like_the_scene():
    sc = with_lens(scenes.cover_scene(32, 24, 1), 0.1, 10.0)
    f = R.make_frame(sc)
    assert bytes(f.camera) == bytes(sc.c.camera)
    f2, L = R.make_frame_lens(sc)
    assert bytes(f2.camera) == bytes(sc.c.camera) and bytes(L) == bytes(sc.lens)
    pin = scenes.cover_scene(32, 24, 1)
    assert bytes(R.make_frame(pin).camera) == bytes(pin.c.camera)


# ---- the CLI: the two camera fields and the refusals that need no device ----
CLI = os.path.join(REPO, "rust-raytracer_b200", "raytracer")


def _cli(tmp_path, camera_extra, env, frames=None):
    import json
    import subprocess
    cfg = scenes._variant(scenes.cover_config(), 16, 12, 1, 3)
    cfg["camera"].update(camera_extra)
    p = tmp_path / "scene.json"
    p.write_text(json.dumps(cfg))
    e = dict(os.environ, **env)
    if frames is not None:
        fp = tmp_path / "frames.json"
        fp.write_text(json.dumps(frames))
        e["RTB200_FRAMES"] = str(fp)
    return subprocess.run([CLI, str(p), str(tmp_path / "out.png")], capture_output=True, text=True, env=e, cwd=REPO, timeout=120)


@pytest.mark.parametrize("var", ["RTB200_GPUS", "RTB200_ADAPTIVE", "RTB200_AOV", "RTB200_DENOISE"])
def test_cli_refuses_a_lens_where_it_has_no_lens_path(tmp_path, var):
    r = _cli(tmp_path, {"aperture": 0.1, "focus_dist": 10.0}, {var: "1"})
    assert r.returncode == 101 and "lens camera" in r.stderr, r.stderr


def test_cli_refuses_temporal_with_a_lens_frame(tmp_path):
    cam = scenes._variant(scenes.cover_config(), 16, 12, 1, 3)["camera"]
    r = _cli(tmp_path, {}, {"RTB200_TEMPORAL": "2"}, frames=[{"camera": dict(cam, aperture=0.2)}])
    assert r.returncode == 101 and "lens camera" in r.stderr, r.stderr


@pytest.mark.parametrize("extra", [{"aperture": -0.1}, {"aperture": 0.1, "focus_dist": 0.0}, {"aperture": 0.1, "focus_dist": -2.0}])
def test_cli_refuses_a_bad_lens(tmp_path, extra):
    r = _cli(tmp_path, extra, {})
    assert r.returncode == 101 and "Unable to parse config json" in r.stderr, r.stderr
    cam = scenes._variant(scenes.cover_config(), 16, 12, 1, 3)["camera"]
    r = _cli(tmp_path, {}, {}, frames=[{"camera": dict(cam, **extra)}])
    assert r.returncode == 101 and "Unable to parse frames json" in r.stderr, r.stderr
