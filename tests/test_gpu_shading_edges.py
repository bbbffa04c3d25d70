"""Shading at the edges of the material and camera parameters, on the GPU against the CPU oracle (oracle/rt_oracle.hpp).

The reference, and so the oracle, is defined far outside the ranges the other tests draw from: albedos that are infinite,
NaN, negative or far above 1 (serde reads a JSON albedo as f64 and converts it with `as f32`, so 1e39 is +inf), Metal fuzz
up to 1e20, Glass indices from 0 to +inf, texture offsets that push the lookup past the image's end (the reference panics
there; the oracle and the kernel clamp the index and must still agree), sky textures of one or two texels, and cameras whose
rays are too long, or start too far out, for the f32 filter, so that every ray takes the all-spheres f64 path.

Every case compares linear f32, RGB8, rays and samples with the oracle (`assert_frames_match`: bit-equal outside NaN, equal
NaN masks; the NaN payload is not compared, x86 gives 0xFFC00000 for inf * 0 where the GPU gives 0x7FFFFFFF), and asserts on
the oracle's output that the case reaches the edge it is written for: NaN pixels, `texture_oob` > 0, or all-spheres
candidates. The scene builders are shared with tests/test_shading_edges_cpu.py, which pins the oracle at the same edges to
the pure-Python restatement."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
import rtb200 as R
from synth import base_config, _v

AUTO, EXACT, BRUTE = R.RT_VARIANT_AUTO, R.RT_VARIANT_EXACT_F64, R.RT_VARIANT_BRUTE_FORCE
SUBJECT, METAL = 1, 2          # sphere indices in edge_config: the sphere under test and the large-fuzz Metal sphere


# ---- the comparison rule ----------------------------------------------------------------------------------------------
def assert_frames_match(got, want, what=""):
    """(linear f32, rgb8) frames: the NaN masks are equal, every other linear value is bit-equal, RGB8 is equal."""
    lin, img = got
    lin_w, img_w = want
    assert lin.shape == lin_w.shape and lin.dtype == lin_w.dtype == np.float32
    nan, nan_w = np.isnan(lin), np.isnan(lin_w)
    assert np.array_equal(nan, nan_w), \
        f"{what}: NaN in {int(nan.any(-1).sum())} pixels here, {int(nan_w.any(-1).sum())} in the reference, {int((nan != nan_w).any(-1).sum())} pixels differ"
    bits, bits_w = lin.view(np.uint32), lin_w.view(np.uint32)
    diff = (bits != bits_w) & ~nan
    assert not diff.any(), f"{what}: linear differs in {int(diff.any(-1).sum())} pixels, first at {np.argwhere(diff)[0].tolist()}"
    assert np.array_equal(img, img_w), f"{what}: rgb8 differs in {int((img != img_w).any(-1).sum())} pixels"


def test_assert_frames_match_rule():
    rng = np.random.default_rng(5)
    a = rng.uniform(0, 1, (4, 6, 3)).astype(np.float32)
    a[1, 2, 0] = np.float32(np.inf) * np.float32(0)   # x86 NaN: 0xFFC00000
    img = rng.integers(0, 256, (4, 6, 3), dtype=np.uint8)
    b = a.copy()
    b.view(np.uint32)[1, 2, 0] = 0x7FFFFFFF           # another NaN payload: still a match
    assert_frames_match((b, img.copy()), (a, img))
    c = a.copy(); c[3, 5, 1] = np.nextafter(c[3, 5, 1], np.float32(2))      # one finite value one ulp off
    with pytest.raises(AssertionError, match="linear differs in 1 pixels"):
        assert_frames_match((c, img), (a, img))
    d = a.copy(); d[0, 0, 2] = np.nan                                        # NaN in only one of the two frames
    with pytest.raises(AssertionError, match="1 pixels differ"):
        assert_frames_match((d, img), (a, img))
    with pytest.raises(AssertionError, match="1 pixels differ"):
        assert_frames_match((a, img), (d, img))
    e, f = a.copy(), a.copy()
    e[2, 2, 2], f[2, 2, 2] = -0.0, 0.0                                         # signed zeros are different bits
    with pytest.raises(AssertionError, match="linear differs"):
        assert_frames_match((e, img), (f, img))
    i2 = img.copy(); i2[0, 1, 0] ^= 1
    with pytest.raises(AssertionError, match="rgb8 differs"):
        assert_frames_match((a, i2), (a, img))


# ---- scenes ------------------------------------------------------------------------------------------------------------
LIGHT_POS = [(-3.0, 4.0, 2.0), (3.0, 5.0, -2.0), (0.0, 6.0, 4.0)]


def edge_config(w, h, spp, depth, subject, n_lights=0, fuzz=0.9, sky="gradient", extra=()):
    """The radius-1000 ground, the sphere under test at (0, 1, 0), a Metal sphere of large fuzz at (2.5, 1, 0) whose paths
    often end absorbed, `extra` objects and n_lights lights, seen from close enough that both spheres fill the view."""
    objs = [{"center": _v(0, -1000, 0), "radius": 1000.0, "material": {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}},
            {"center": _v(0, 1, 0), "radius": 1.0, "material": subject},
            {"center": _v(2.5, 1, 0), "radius": 1.0, "material": {"Metal": {"albedo": [0.8, 0.8, 0.8], "fuzz": fuzz}}}]
    objs += list(extra)
    for k in range(n_lights):
        objs.append({"center": _v(*LIGHT_POS[k]), "radius": 0.7, "material": {"Light": {}}})
    return base_config(w, h, spp, depth, objs, sky=sky, look_from=(3.5, 2, 4), look_at=(1.2, 0.8, 0), vfov=45.0)


def synthetic_texture(w, h):
    """An h x w RGB8 image whose texels are all different, so that a wrong index changes the colour."""
    k = np.arange(w * h * 3, dtype=np.int64).reshape(h, w, 3)
    return ((k * 97 + 13) % 251).astype(np.uint8)


def scene_of(cfg, textures=None, sky=None):
    """R.Scene of `cfg`. A Texture material names its image in `textures` ({"Texture": {"albedo", "h_offset", "width",
    "height", "pixels": key}}) instead of a JPEG file; `sky` replaces the sky by a texture image."""
    textures = textures or {}
    plain = json.loads(json.dumps(cfg))
    tex_objs = []
    for i, o in enumerate(plain["objects"]):
        if "Texture" in o["material"]:
            tex_objs.append((i, o["material"]["Texture"]))
            o["material"] = {"Lambertian": {"albedo": [0.0, 0.0, 0.0]}}
    if sky is not None:
        plain["sky"] = {"texture": ""}
    sc = R.Scene.from_config(plain)
    sc.source = cfg
    if tex_objs:
        structs = []
        for k, (i, body) in enumerate(tex_objs):
            arr = np.ascontiguousarray(textures[body["pixels"]])
            assert arr.shape == (int(body["height"]), int(body["width"]), 3)
            sc._tex_arrays.append(arr)
            structs.append(R.rt_image(arr.ctypes.data, arr.shape[1], arr.shape[0], arr.size))
            s = sc._spheres[i]
            s.kind = R.RT_TEXTURE; s.param = float(body["h_offset"]); s.texture = k
            s.albedo[:] = [np.float32(a) for a in body["albedo"]]
        sc._tex_structs = (R.rt_image * len(structs))(*structs)
        sc.c.textures = C.cast(sc._tex_structs, C.POINTER(R.rt_image))
        sc.c.n_textures = len(structs)
    if sky is not None:
        arr = np.ascontiguousarray(sky)
        sc._sky_array = arr
        sc.c.sky.mode = R.RT_SKY_TEXTURE
        sc.c.sky.tex = R.rt_image(arr.ctypes.data, arr.shape[1], arr.shape[0], arr.size)
    return sc


def set_albedo(sc, i, albedo):
    """Set sphere i's albedo in the C record (values the JSON route cannot carry: -inf, NaN)."""
    sc._spheres[i].albedo[:] = [np.float32(a) for a in albedo]


def nan_pixels(lin):
    return int(np.isnan(lin).any(-1).sum())


# the non-finite albedo cases: (name, value, channels)
NONFINITE = [("inf", math.inf, 1), ("inf", math.inf, 3), ("-inf", -math.inf, 1), ("-inf", -math.inf, 3), ("nan", math.nan, 1), ("nan", math.nan, 3)]
# (lights, max_depth) pairs every non-finite case runs
LIGHTS_DEPTHS = [(0, 1), (0, 2), (0, 5), (0, 50), (1, 1), (1, 5), (2, 2), (3, 50)]


def nonfinite_albedo(value, channels):
    return [value] * channels + [0.5] * (3 - channels)


def nonfinite_scene(w, h, spp, depth, n_lights, material, value, channels):
    """edge_config with a non-finite albedo on the Lambertian subject or on the Metal sphere. +inf goes through the JSON
    route (1e39 -> as f32), the others are set in the rt_sphere record."""
    alb = nonfinite_albedo(1e39 if value == math.inf else 0.5, channels)
    if material == "Lambertian":
        cfg = edge_config(w, h, spp, depth, {"Lambertian": {"albedo": alb}}, n_lights)
        idx = SUBJECT
    else:
        cfg = edge_config(w, h, spp, depth, {"Lambertian": {"albedo": [0.4, 0.6, 0.3]}}, n_lights)
        cfg["objects"][METAL]["material"]["Metal"]["albedo"] = alb
        idx = METAL
    sc = R.Scene.from_config(cfg)
    if value != math.inf:
        set_albedo(sc, idx, nonfinite_albedo(value, channels))
    return sc


# ---- the comparison against the oracle ---------------------------------------------------------------------------------
def render_vs_oracle(sc, variants=(AUTO,), what=""):
    """Linear and RGB8 renders of every variant against the oracle; returns the oracle's (linear, rgb8, stats) and the stats
    of the first variant's linear render."""
    lin_o, img_o, st_o = O.render(sc)
    first = None
    for v in variants:
        opts = R.make_options(variant=v)
        lin, st = R.render_linear(sc, opts)
        img, st8 = R.render_rgb8(sc, opts)
        assert_frames_match((lin, img), (lin_o, img_o), f"{what} variant {v}")
        assert st["rays"] == st8["rays"] == st_o["rays"], (what, v, st["rays"], st8["rays"], st_o["rays"])
        assert st["samples"] == st_o["samples"]
        first = first or st
    return lin_o, img_o, st_o, first


@pytest.mark.gpu
@pytest.mark.parametrize("material", ["Lambertian", "Metal"])
@pytest.mark.parametrize("name,value,channels", NONFINITE, ids=[f"{n}x{c}" for n, _, c in NONFINITE])
def test_nonfinite_albedo(material, name, value, channels):
    for n_lights, depth in LIGHTS_DEPTHS:
        sc = nonfinite_scene(24, 16, 4, depth, n_lights, material, value, channels)
        cheap = n_lights == 0 or depth <= 5
        lin_o, _, st_o, _ = render_vs_oracle(sc, (AUTO, EXACT, BRUTE) if cheap and channels == 3 else (AUTO,),
                                             f"{material} {name}x{channels} lights={n_lights} depth={depth}")
        assert nan_pixels(lin_o) > 0, "the case must produce NaN pixels"
        if material == "Metal":
            assert st_o["term_absorbed"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("n_lights,depth", [(0, 5), (0, 50), (3, 50)])
def test_nonfinite_albedo_in_a_closed_room(n_lights, depth):
    """Paths that end by reaching max_depth: the room of test_gpu_work_sets, one of whose spheres has an infinite albedo."""
    from test_gpu_work_sets import _room_cfg
    cfg = _room_cfg(n_lights, depth, w=32, h=24, spp=2)
    k = next(i for i, o in enumerate(cfg["objects"]) if "Lambertian" in o["material"] and i > 0)
    cfg["objects"][k]["material"]["Lambertian"]["albedo"] = [1e39, 0.3, 0.3]
    lin_o, _, st_o, _ = render_vs_oracle(R.Scene.from_config(cfg), what=f"room lights={n_lights} depth={depth}")
    assert nan_pixels(lin_o) > 0 and st_o["term_depth"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("n_lights", [0, 2])
def test_nonfinite_albedo_in_grouped_frames(n_lights):
    """render_frames of three frames in one launch group: the multi-frame kernels."""
    sc = nonfinite_scene(24, 16, 3, 6, n_lights, "Lambertian", -math.inf, 3)
    frames = [R.make_frame(sc, look_from=_v(6, 3, 6), seed=11), R.make_frame(sc, look_from=_v(-5, 2, 6), seed=12),
              R.make_frame(sc, look_from=_v(4, 6, -5), seed=13)]
    img, st = R.render_frames(sc, frames)
    lin, st_l = R.render_frames(sc, frames, linear=True)
    rays = 0
    for i, f in enumerate(frames):
        v = R.Scene()
        v.c = R.rt_scene.from_buffer_copy(sc.c)
        v.c.camera = f.camera; v.c.seed = f.seed; v.c.max_depth = f.max_depth
        v._keep = sc
        lin_o, img_o, st_o = O.render(v)
        assert nan_pixels(lin_o) > 0
        assert_frames_match((lin[i], img[i]), (lin_o, img_o), f"frame {i}")
        rays += st_o["rays"]
    assert st["rays"] == st_l["rays"] == rays


@pytest.mark.gpu
@pytest.mark.parametrize("n_lights", [0, 1])
def test_resident_handle_takes_a_nonfinite_albedo_by_update(n_lights):
    """Uploaded with finite albedos, then given +inf by update_spheres: the handle's next frame must follow the edit."""
    from test_gpu_scene_update import _render
    sc = R.Scene.from_config(edge_config(24, 16, 4, 8, {"Lambertian": {"albedo": [0.7, 0.5, 0.5]}}, n_lights))
    rs = R.ResidentScene(sc)
    try:
        img, lin, rays = _render(rs)
        lin_o, img_o, st_o = O.render(sc)
        assert nan_pixels(lin_o) == 0
        assert_frames_match((lin, img), (lin_o, img_o), "before the update")
        assert rays == st_o["rays"]
        rec = sc.set_sphere(SUBJECT, material={"Lambertian": {"albedo": [np.float32(1e39), 0.5, 0.5]}})
        rs.update_spheres([SUBJECT], [rec])
        img, lin, rays = _render(rs)
        lin_o, img_o, st_o = O.render(sc)
        assert nan_pixels(lin_o) > 0
        assert_frames_match((lin, img), (lin_o, img_o), "after the update")
        assert rays == st_o["rays"]
    finally:
        rs.release()


FINITE_ALBEDOS = [0.0, -0.0, -0.5, 1.5, 4.0, 1e30]


@pytest.mark.gpu
@pytest.mark.parametrize("n_lights", [0, 2])
def test_finite_albedo_outside_the_unit_range(n_lights):
    for a in FINITE_ALBEDOS:
        for material in ("Lambertian", "Metal"):
            sub = {"Lambertian": {"albedo": [a, a, a]}} if material == "Lambertian" else {"Metal": {"albedo": [a, 0.5, a], "fuzz": 0.3}}
            sc = R.Scene.from_config(edge_config(24, 16, 4, 6, sub, n_lights))
            lin_o, _, _, _ = render_vs_oracle(sc, what=f"{material} albedo {a} lights={n_lights}")
            assert nan_pixels(lin_o) == 0


FUZZ = [0.0, 1.0, 2.0, 50.0, -0.7, 1e16, 1e20]


def fallback_bound(st_o, n):
    """Exact f64 tests that the all-spheres path must have run at least: every Metal scatter that was not absorbed is traced
    next (unless its path had just reached max_depth), with every sphere, when its direction is longer than 1e15."""
    return n * (st_o["hits"][R.RT_METAL] - st_o["term_absorbed"] - st_o["term_depth"])


@pytest.mark.gpu
@pytest.mark.parametrize("n_lights", [0, 1])
def test_metal_fuzz(n_lights):
    for fuzz in FUZZ:
        sub = {"Metal": {"albedo": [0.9, 0.6, 0.4], "fuzz": fuzz}}
        sc = R.Scene.from_config(edge_config(24, 16, 4, 8, sub, n_lights, fuzz=fuzz))
        _, _, st_o, st = render_vs_oracle(sc, (AUTO, EXACT, BRUTE), f"fuzz {fuzz} lights={n_lights}")
        if fuzz == 1e20 and n_lights == 0:
            bound = fallback_bound(st_o, sc.n_spheres)
            assert bound > 0 and st["candidates"] >= bound, (st["candidates"], bound)


INDICES = [1.0, 0.5, 1e-3, 100.0, -1.5, 0.0, math.inf]


def glass_config(w, h, spp, depth, ior, n_lights):
    """A glass sphere and, at (-2.5, 1, 0), the hollow-shell pattern (outer radius 1, inner radius -0.9) of the same index."""
    g = {"Glass": {"index_of_refraction": ior}}
    shell = [{"center": _v(-2.5, 1, 0), "radius": 1.0, "material": g}, {"center": _v(-2.5, 1, 0), "radius": -0.9, "material": g}]
    return edge_config(w, h, spp, depth, g, n_lights, extra=shell)


@pytest.mark.gpu
@pytest.mark.parametrize("n_lights", [0, 1])
def test_glass_index(n_lights):
    for ior in INDICES:
        sc = R.Scene.from_config(glass_config(32, 24, 4, 10, ior, n_lights))
        _, _, st_o, _ = render_vs_oracle(sc, (AUTO, EXACT), f"index {ior} lights={n_lights}")
        assert st_o["hits"][R.RT_GLASS] > 0


TEX_SIZES = [(1, 1), (1, 7), (7, 1), (3, 2)]      # (width, height)
H_OFFSETS = [0.0, 0.5, 0.999999, 1.0, 1.5, 2.5, -0.5, -3.0]
OOB_OFFSETS = (1.5, 2.5)                          # the offsets whose lookup can run past the image's end


def texture_config(w, h, spp, depth, tw, th, h_offset, n_lights=0):
    """A textured sphere of positive radius (the subject) and one of negative radius at (-2.5, 1, 0), both on one image."""
    t = {"Texture": {"albedo": [0.0, 0.0, 0.0], "h_offset": h_offset, "width": tw, "height": th, "pixels": "tex"}}
    return edge_config(w, h, spp, depth, t, n_lights, extra=[{"center": _v(-2.5, 1, 0), "radius": -1.0, "material": t}])


@pytest.mark.gpu
@pytest.mark.parametrize("tw,th", TEX_SIZES, ids=[f"{a}x{b}" for a, b in TEX_SIZES])
def test_texture_lookup(tw, th):
    img = synthetic_texture(tw, th)
    oob = []
    for h_offset in H_OFFSETS:
        sc = scene_of(texture_config(24, 16, 3, 4, tw, th, h_offset, n_lights=1 if h_offset < 0 else 0), {"tex": img})
        _, _, st_o, _ = render_vs_oracle(sc, (AUTO, BRUTE), f"texture {tw}x{th} h_offset {h_offset}")
        assert st_o["hits"][R.RT_TEXTURE] > 0
        if st_o["texture_oob"]:
            oob.append(h_offset)
    # the lookup reaches the clamp where the reference panics: past the last row only for rot - 1 >= 0.5 (1.5, 2.5)
    assert oob and set(oob) <= set(OOB_OFFSETS), oob


SKY_SIZES = [(1, 1), (2, 1), (1, 2), (5, 3)]      # (width, height)


def sky_frames(sc):
    """Straight up and straight down (vfov 1e-3: |ud.y| rounds to 1 in f32, so t is exactly 1 and 0) and a wide view."""
    return [R.make_frame(sc, look_from=_v(0, 0, 0), look_at=_v(0, 1, 0), vup=_v(1, 0, 0), vfov=1e-3),
            R.make_frame(sc, look_from=_v(0, 0, 0), look_at=_v(0, -1, 0), vup=_v(1, 0, 0), vfov=1e-3),
            R.make_frame(sc, look_from=_v(0, 0, 0), look_at=_v(1, 0.2, 0.3), vup=_v(0, 1, 0), vfov=150.0)]


def sky_config(w, h, spp):
    sub = {"Metal": {"albedo": [0.9, 0.9, 0.9], "fuzz": 0.0}}
    return base_config(w, h, spp, 4, [{"center": _v(3, 0.5, 1), "radius": 1.0, "material": sub}], look_from=(0, 0, 0), look_at=(1, 0.2, 0.3), vfov=150.0)


@pytest.mark.gpu
@pytest.mark.parametrize("tw,th", SKY_SIZES, ids=[f"{a}x{b}" for a, b in SKY_SIZES])
def test_sky_texture(tw, th):
    sky = synthetic_texture(tw, th)
    sc = scene_of(sky_config(24, 16, 2), sky=sky)
    for i, f in enumerate(sky_frames(sc)):
        v = R.Scene()
        v.c = R.rt_scene.from_buffer_copy(sc.c)
        v.c.camera = f.camera
        v._keep = sc
        lin_o, _, _, _ = render_vs_oracle(v, (AUTO, EXACT), f"sky {tw}x{th} frame {i}")
        if i < 2:   # every ray reads the top row (t = 1) or the bottom row (t = 0)
            row = sky[0 if i == 0 else th - 1].astype(np.float32)
            want = [np.float32(0.7) * row[x] / np.float32(255.0) for x in range(tw)]
            assert any(np.array_equal(lin_o[0, 0], c) for c in want), (lin_o[0, 0], want)


def fallback_scene(kind):
    objs = [{"center": _v(0, -1000, 0), "radius": 1000.0, "material": {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}},
            {"center": _v(0, 1, 0), "radius": 1.0, "material": {"Metal": {"albedo": [0.8, 0.6, 0.2], "fuzz": 0.2}}},
            {"center": _v(-3, 1.5, 1), "radius": 1.5, "material": {"Glass": {"index_of_refraction": 1.5}}},
            {"center": _v(3, 2, -1), "radius": 2.0, "material": {"Lambertian": {"albedo": [0.2, 0.7, 0.3]}}}]
    if kind == "vfov180":     # tan(pi/2) = 1.6e16: every primary direction is longer than 1e15
        return base_config(24, 16, 2, 4, objs, look_from=(6, 3, 6), look_at=(0, 1, 0), vfov=180.0)
    if kind == "far":         # the camera 1e16 from the scene: |origin| is beyond the f32 frame's range
        return base_config(24, 16, 2, 4, objs, look_from=(1.0000000000000002e16, 1.0, 0.0), look_at=(0, 1, 0), vfov=2e-13)
    if kind == "vfov1e-6":
        return base_config(24, 16, 2, 4, objs, look_from=(6, 3, 6), look_at=(0, 1, 0), vfov=1e-6)
    cfg = base_config(24, 16, 2, 4, objs, look_from=(0, 6, 0), look_at=(0, 1, 0), vfov=60.0)
    cfg["camera"]["vup"] = _v(0, 1, 0)   # parallel to the view direction: a NaN camera
    return cfg


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["vfov180", "far", "vfov1e-6", "vup_parallel"])
def test_camera_edges(kind):
    sc = R.Scene.from_config(fallback_scene(kind))
    lin_o, _, st_o, st = render_vs_oracle(sc, (AUTO, EXACT, BRUTE), kind)
    if kind in ("vfov180", "far"):
        # every primary ray tests every sphere in f64: the all-spheres path ran
        assert st["candidates"] >= sc.n_spheres * st_o["samples"], (st["candidates"], st_o["samples"])
    if kind == "far":
        assert sum(st_o["hits"]) > 0      # (at vfov 180 every root is closer than t_min: |d| ~ 1e16)
    if kind == "vup_parallel":
        assert np.isnan(lin_o).all()


CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rust-raytracer_b200", "raytracer")


@pytest.mark.gpu
@pytest.mark.parametrize("n_lights", [0, 1])
def test_cli_reads_an_albedo_beyond_f32_as_infinity(tmp_path, n_lights):
    """JSON 1e39 through the C++ scene reader (`as f32`: +inf) and the CLI: its PNG equals the oracle's RGB8."""
    from PIL import Image
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-C", os.path.dirname(CLI), "raytracer"])
    cfg = edge_config(24, 16, 4, 6, {"Lambertian": {"albedo": [1e39, 0.5, -1e39]}}, n_lights)
    p = tmp_path / "scene.json"
    p.write_text(json.dumps(cfg))
    assert "1e+39" in p.read_text()
    out = tmp_path / "out.png"
    r = subprocess.run([CLI, str(p), str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    lin_o, img_o, _ = O.render(R.Scene.from_config(cfg))
    assert nan_pixels(lin_o) > 0
    assert np.array_equal(np.asarray(Image.open(out)), img_o)
