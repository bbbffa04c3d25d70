"""Two restatements of the thin-lens camera, written separately, must produce the same bits: the C++ lens oracle
(tests/oracle_lens.cpp, on oracle/rt_oracle.hpp) and the pure-Python one (tests/lens_restatement.py, on
tests/py_restatement.py). Linear f32 frames, RGB8 frames and ray counts of small, non-square lens frames of the cover scene,
mixed materials with lights and fuzzed metal under a gradient sky and under no sky, and the reference's test_scene (textures,
sky texture, a light, the hollow glass shell); the lens rays and trial counts of single samples. No GPU needed."""
import copy

import numpy as np
import pytest

import oracle_lens as OL
import rtb200 as R
from lens_restatement import LensCamera, LensWorld
from rtb200 import scenes
from synth import _v, mixed_config


def _with_lens(cfg, aperture, focus_dist):
    cfg = copy.deepcopy(cfg)
    cfg["camera"]["aperture"] = aperture
    if focus_dist is not None:
        cfg["camera"]["focus_dist"] = focus_dist
    return cfg


def _both(cfg, aperture, focus_dist):
    cfg = _with_lens(cfg, aperture, focus_dist)
    sc = R.Scene.from_config(cfg, scenes.SCENES_DIR)
    want = OL.render(sc, sc.lens)
    tex, k = {}, 0
    for i, o in enumerate(cfg["objects"]):
        if "Texture" in o["material"]:
            tex[i] = sc._tex_arrays[k]; k += 1
    fd = focus_dist if focus_dist is not None else R.focal_length(sc.camera_params["look_from"], sc.camera_params["look_at"])
    w = LensWorld(cfg, aperture, fd, textures=tex, sky_texture=sc._sky_array, seed=sc.seed)
    lin, img, rays = w.render()
    assert rays == want["rays"], ("ray counts", rays, want["rays"])
    assert np.array_equal(lin, want["linear"]), f"linear frames differ: max |d| = {np.abs(lin - want['linear']).max()}"
    assert np.array_equal(img, want["rgb8"])
    return sc


def test_cover_scene_at_the_books_lens():
    _both(scenes._variant(scenes.cover_config(), 14, 10, 2, 50), 0.1, 10.0)


@pytest.mark.parametrize("sky,aperture,fd", [("gradient", 0.5, None), ("none", 1.5, 3.0)])
def test_mixed_materials_with_lights(sky, aperture, fd):
    cfg = mixed_config(10, 7, 2, 5, seed=31, n=10, sky=sky)
    for k, pos in enumerate([(0.0, 6.0, 0.0), (-4.0, 3.0, 5.0)]):
        cfg["objects"].insert(2 + 3 * k, {"center": _v(*pos), "radius": 1.0 + 0.5 * k, "material": {"Light": {}}})
    assert any("Metal" in o["material"] and o["material"]["Metal"]["fuzz"] > 0 for o in cfg["objects"])
    _both(cfg, aperture, fd)


def test_reference_test_scene_with_textures_and_the_glass_shell():
    cfg = scenes._variant(scenes.test_scene_config(), 16, 12, 2, 8)
    assert any(o["radius"] < 0 for o in cfg["objects"])
    _both(cfg, 0.4, None)


def test_lens_rays_and_trials():
    cfg = _with_lens(scenes._variant(scenes.cover_config(), 30, 20, 1, 5), 2.0, 7.5)
    sc = R.Scene.from_config(cfg, scenes.SCENES_DIR)
    lc = LensCamera(cfg["camera"], 2.0, 7.5)
    rng = np.random.default_rng(3)
    trials = set()
    for _ in range(200):
        pixel, sample, seed = int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 16)), int(rng.integers(0, 1 << 64, dtype=np.uint64))
        u, v = (float(t) for t in rng.random(2))
        o, d, t = OL.lens_ray(sc.c.camera, sc.lens, seed, pixel, sample, u, v)
        po, pd, pt = lc.get_ray(u, v, seed, pixel, sample)
        assert np.array_equal(o, np.array(po)) and np.array_equal(d, np.array(pd)) and t == pt
        trials.add(t)
    assert max(trials) >= 3   # rejected trials are exercised


def test_the_oracle_reproduces_the_golden_fixture():
    import json
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_lens
    want = json.load(open(make_lens.OUT))
    got = {name: make_lens.pins(sc) for name, sc in make_lens.cases().items()}
    assert got == want


# The degenerate lenses of tests/lens_edges.py (E1, E3, E4, E7) under a 64-bit key: radius, u and v as the case sets them
# (None: the camera's own), and the camera's aperture, focus distance and field of view.
SEED64 = 0x9E3779B97F4A7C15
EDGES = {
    "tiny": dict(aperture=2.0 ** -1073, fd=9.0),
    "zero_uv": dict(u=(0.0, 0.0, 0.0), v=(0.0, 0.0, 0.0), radius=0.3),
    "u_zero": dict(u=(0.0, 0.0, 0.0), radius=0.3),
    "u_eq_v": dict(v="u", radius=0.3),
    "u_1e3": dict(u=1e3, radius=3e-4),
    "huge": dict(radius=1e300),
    "fd_tiny": dict(aperture=0.4, fd=1e-300),
    "fd_huge": dict(aperture=0.4, fd=1e308, vfov=120.0),
}


@pytest.mark.parametrize("name", list(EDGES))
def test_degenerate_lenses_under_a_64_bit_key(name):
    e = dict(dict(aperture=0.6, fd=9.0, vfov=20.0), **EDGES[name])
    cfg = mixed_config(6, 4, 2, 6, seed=31, n=10)
    cfg["objects"].insert(2, {"center": _v(0.0, 6.0, 0.0), "radius": 1.0, "material": {"Light": {}}})
    cfg["camera"]["vfov"] = e["vfov"]
    cfg = _with_lens(cfg, e["aperture"], e["fd"])
    sc = R.Scene.from_config(cfg, scenes.SCENES_DIR)
    sc.seed = SEED64
    w = LensWorld(cfg, e["aperture"], e["fd"], seed=SEED64)
    lc = w.lens_camera
    u, v = np.array(lc.u, float), np.array(lc.v, float)
    u = u * e["u"] if isinstance(e.get("u"), float) else np.array(e.get("u", u), float)
    v = u if e.get("v") == "u" else np.array(e.get("v", v), float)
    lc.u, lc.v, lc.radius = tuple(u.tolist()), tuple(v.tolist()), float(e.get("radius", lc.radius))
    lens = R.rt_lens(R.vec3(lc.u), R.vec3(lc.v), lc.radius, 0)
    want = OL.render(sc, lens)
    lin, img, rays = w.render()
    assert rays == want["rays"], (rays, want["rays"])
    assert np.array_equal(np.isnan(lin), np.isnan(want["linear"]))
    assert np.array_equal(np.nan_to_num(lin).view(np.uint32), np.nan_to_num(want["linear"]).view(np.uint32)), name
    assert np.array_equal(img, want["rgb8"]), name
