"""The oracle at the edges of the material and camera parameters, against the pure-Python restatement (no GPU).

tests/test_gpu_shading_edges.py holds the GPU to the oracle (oracle/rt_oracle.hpp) at these edges; a misreading of the
reference shared by the oracle and the kernel would pass it. So here the oracle is pinned, on tiny frames of the same scenes,
to tests/py_restatement.py, which shares no code with it: where the reference is defined (non-finite and out-of-range
albedos, any fuzz and index, in-range texture and sky lookups, cameras whose rays take the all-spheres path) the two agree
bit for bit, NaN as NaN; where the reference panics (a texture lookup past the image's end) the restatement raises while the
oracle counts the clamp in `texture_oob`."""
import copy
import math

import numpy as np
import pytest

import oracle_py as O
import rtb200 as R
from py_restatement import World
from test_gpu_shading_edges import (FINITE_ALBEDOS, FUZZ, H_OFFSETS, INDICES, METAL, NONFINITE, SKY_SIZES, TEX_SIZES,
                                    assert_frames_match, edge_config, fallback_scene, glass_config,
                                    nan_pixels, nonfinite_albedo, scene_of, sky_config, synthetic_texture, texture_config)

W, H, SPP = 8, 6, 2


def oracle_and_restatement(cfg, textures=None, sky=None):
    """Oracle and restatement renders of cfg: ((linear, rgb8), rays, oracle stats) and ((linear, rgb8), rays)."""
    sc = scene_of(cfg, textures, sky)
    lin_o, img_o, st_o = O.render(sc)
    tex = {i: textures[o["material"]["Texture"]["pixels"]] for i, o in enumerate(cfg["objects"]) if "Texture" in o["material"]}
    pcfg = cfg
    if sky is not None:
        pcfg = copy.deepcopy(cfg)
        pcfg["sky"] = {"texture": "synthetic"}
    with np.errstate(all="ignore"):   # inf * 0 and friends are the point here
        lin_p, img_p, rays_p = World(pcfg, textures=tex, sky_texture=sky, seed=sc.seed).render()
    return ((lin_o, img_o), st_o["rays"], st_o), ((lin_p, img_p), rays_p)


def assert_agree(cfg, what, textures=None, sky=None):
    o, p = oracle_and_restatement(cfg, textures, sky)
    assert_frames_match(p[0], o[0], what)
    assert o[1] == p[1], (what, "rays", o[1], p[1])
    return o


@pytest.mark.parametrize("material", ["Lambertian", "Metal"])
@pytest.mark.parametrize("name,value,channels", NONFINITE, ids=[f"{n}x{c}" for n, _, c in NONFINITE])
def test_nonfinite_albedo(material, name, value, channels):
    for n_lights, depth in [(0, 1), (0, 2), (1, 1), (2, 2), (3, 50)]:
        alb = nonfinite_albedo(1e39 if value == math.inf else value, channels)   # JSON 1e39: +inf as f32
        if material == "Lambertian":
            cfg = edge_config(W, H, SPP, depth, {"Lambertian": {"albedo": alb}}, n_lights)
        else:
            cfg = edge_config(W, H, SPP, depth, {"Lambertian": {"albedo": [0.4, 0.6, 0.3]}}, n_lights)
            cfg["objects"][METAL]["material"]["Metal"]["albedo"] = alb
        lin_o = assert_agree(cfg, f"{material} {name}x{channels} lights={n_lights} depth={depth}")[0][0]
        assert nan_pixels(lin_o) > 0


@pytest.mark.parametrize("n_lights", [0, 2])
def test_finite_albedo_outside_the_unit_range(n_lights):
    for a in FINITE_ALBEDOS:
        assert_agree(edge_config(W, H, SPP, 6, {"Lambertian": {"albedo": [a, a, a]}}, n_lights), f"albedo {a}")
        assert_agree(edge_config(W, H, SPP, 6, {"Metal": {"albedo": [a, 0.5, a], "fuzz": 0.3}}, n_lights), f"metal albedo {a}")


def test_metal_fuzz():
    for fuzz in FUZZ:
        assert_agree(edge_config(W, H, SPP, 8, {"Metal": {"albedo": [0.9, 0.6, 0.4], "fuzz": fuzz}}, 1, fuzz=fuzz), f"fuzz {fuzz}")


def test_glass_index():
    for ior in INDICES:
        for n_lights in (0, 1):
            st_o = assert_agree(glass_config(W, H, SPP, 10, ior, n_lights), f"index {ior}")[2]
            assert st_o["hits"][R.RT_GLASS] > 0


@pytest.mark.parametrize("tw,th", TEX_SIZES, ids=[f"{a}x{b}" for a, b in TEX_SIZES])
def test_texture_lookup(tw, th):
    img = {"tex": synthetic_texture(tw, th)}
    oob = 0
    for h_offset in H_OFFSETS:
        cfg = texture_config(W * 2, H * 2, SPP, 4, tw, th, h_offset)
        st_o = O.render(scene_of(cfg, img))[2]
        assert st_o["hits"][R.RT_TEXTURE] > 0
        if st_o["texture_oob"]:   # the reference panics: the restatement raises, the oracle clamps and counts
            oob += 1
            with pytest.raises(IndexError):
                oracle_and_restatement(cfg, img)
        else:
            assert_agree(cfg, f"texture {tw}x{th} h_offset {h_offset}", img)
    assert oob > 0


@pytest.mark.parametrize("tw,th", SKY_SIZES, ids=[f"{a}x{b}" for a, b in SKY_SIZES])
def test_sky_texture(tw, th):
    sky = synthetic_texture(tw, th)
    for look_at, vup, vfov in [((0, 1, 0), (1, 0, 0), 1e-3), ((0, -1, 0), (1, 0, 0), 1e-3), ((1, 0.2, 0.3), (0, 1, 0), 150.0)]:
        cfg = sky_config(W, H, SPP)
        cfg["camera"].update(look_at={"x": look_at[0], "y": look_at[1], "z": look_at[2]}, vup={"x": vup[0], "y": vup[1], "z": vup[2]}, vfov=vfov)
        assert_agree(cfg, f"sky {tw}x{th} looking at {look_at}", sky=sky)


@pytest.mark.parametrize("kind", ["vfov180", "far", "vfov1e-6"])
def test_camera_edges(kind):
    cfg = fallback_scene(kind)
    cfg["width"], cfg["height"] = W, H
    st_o = assert_agree(cfg, kind)[2]
    assert sum(st_o["hits"]) > 0 or kind == "vfov180"   # at vfov 180 every root is closer than t_min: |d| ~ 1e16
