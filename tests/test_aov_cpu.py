"""Auxiliary buffers of a resident scene's camera samples without a GPU (rtb200_scene_aov[_device], DESIGN.md §4.14): the exported
entry points, the layout of rt_aov_params and rt_aov_out, the argument checks that run before any device work, and the oracle
the GPU tests hold the kernel to, pinned by two independent restatements: its hits are oracle_hit_world's on the render's
primary rays, and its albedo is a numpy restatement of the material table, the texture lookup and the sky from those hits."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import intersect_rays as IR
import oracle_aov as OA
import oracle_hit_world as OH
import oracle_trace_rays as OT
import rtb200 as R
from rtb200 import scenes
from synth import _v, mixed_config
from test_gpu_shading_edges import scene_of, synthetic_texture, texture_config
from test_trace_rays_cpu import primary_rays

F32 = np.float32


# ---- scenes the AOV tests share ----------------------------------------------------------------------------------------

def textured_sky_scene(w=24, h=16, spp=1):
    """Two textured spheres (positive and negative radius, h_offset 0.7 so that the lookup wraps), a Metal and a Lambertian
    ground under a sky texture, with sky in the top rows of the view."""
    return scene_of(texture_config(w, h, spp, 4, 7, 5, 0.7), {"tex": synthetic_texture(7, 5)}, sky=synthetic_texture(5, 3))


def mixed_lit_scene(w=32, h=24, spp=1):
    """The mixed synth scene (Lambertian, Metal, Glass, a hollow shell, a coincident pair) without the glass bubble around its
    camera, whose first hits would all be that bubble, with two lights and non-finite albedos (NaN and +inf on a Lambertian,
    -inf on a Metal) in view."""
    sc = R.Scene.from_config(mixed_config(w, h, spp, 12, seed=11))
    assert sc._spheres[sc.n_spheres - 1].kind == R.RT_GLASS and sc._spheres[sc.n_spheres - 1].radius == 2.0
    extra = [R.make_sphere((0.0, 1.0, 0.0), 0.9, {"Light": {}}), R.make_sphere((2.5, 0.6, -2.0), 0.6, {"Light": {}}),
             R.make_sphere((-1.0, 0.5, -1.5), 0.5, {"Lambertian": {"albedo": [math.nan, 0.5, math.inf]}}),
             R.make_sphere((1.0, 0.5, 2.5), 0.5, {"Metal": {"albedo": [0.3, -math.inf, 0.7], "fuzz": 0.2}})]
    return sc.edited(remove=[sc.n_spheres - 1], insert=extra)


def aov_scenes():
    return {"cover_40x30": lambda: scenes.cover_scene(40, 30, 1), "textured_sky_24x16": textured_sky_scene,
            "mixed_lit_32x24": mixed_lit_scene}


def assert_f32_equal(got, want, what=""):
    """Bit for bit, except that NaN payloads are free (the NaN masks must be equal)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan, nan_w = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan, nan_w), f"{what}: NaN in {int(nan.sum())} values here, {int(nan_w.sum())} in the reference"
    diff = (got.view(np.uint32) != want.view(np.uint32)) & ~nan
    assert not diff.any(), f"{what}: {int(diff.sum())} values differ, first at {np.argwhere(diff)[0].tolist()}"


# ---- the ABI -----------------------------------------------------------------------------------------------------------

def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_scene_aov_device", "rtb200_scene_aov"):
        assert name in R.ABI_SYMBOLS
        assert getattr(L, name) is not None


def test_aov_structs_match_the_header(repo, tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rtb200.h"\nint main(void) {\n'
                   '    printf("%zu %zu %zu %zu\\n", sizeof(rt_aov_params), offsetof(rt_aov_params, samples),\n'
                   '           offsetof(rt_aov_params, sample0), offsetof(rt_aov_params, reserved));\n'
                   '    printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(rt_aov_out), offsetof(rt_aov_out, albedo), offsetof(rt_aov_out, normal),\n'
                   '           offsetof(rt_aov_out, hits), offsetof(rt_aov_out, sphere), offsetof(rt_aov_out, point));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Werror", "-I", os.path.join(repo, "include"), str(src), "-o", str(exe)])
    lines = subprocess.check_output([str(exe)]).decode().splitlines()
    for line, st, want in zip(lines, (R.rt_aov_params, R.rt_aov_out), ([16, 0, 4, 8], [40, 0, 8, 16, 24, 32])):
        got = [int(x) for x in line.split()]
        mirror = [C.sizeof(st)] + [getattr(st, f).offset for f, _ in st._fields_]
        assert got == mirror == want, (st.__name__, got, mirror)


def test_bad_arguments_are_refused_before_any_device_work():
    """A NULL handle, params or out, every output NULL, samples == 0, sample0 + samples above 2^32 and a nonzero reserved word
    of params or view are refused with RT_ERR_INVALID. The checks come before the handle is used, so a stand-in handle that is
    never dereferenced shows the order."""
    L = R.lib()
    buf = np.full(64, 7.0, np.float32)
    out = R.rt_aov_out(buf.ctypes.data, None, None, None, None)
    good = R.rt_aov_params(1, 0)
    st = R.rt_stats()
    forms = ((L.rtb200_scene_aov, C.byref(st)), (L.rtb200_scene_aov_device, None))
    for fn, last in forms:
        assert fn(None, C.byref(good), None, C.byref(out), last) == -1
        assert b"handle" in L.rtb200_last_error()
    fake = C.c_void_p(C.addressof(C.create_string_buffer(64)))

    def params(samples=1, sample0=0, reserved=(0, 0)):
        p = R.rt_aov_params(samples, sample0)
        p.reserved[0], p.reserved[1] = reserved
        return p

    bad_view = R.rt_frame()
    bad_view.reserved = 1
    cases = [(None, None, out, b"params"),
             (good, None, None, b"out is null"),
             (good, None, R.rt_aov_out(), b"every output"),
             (params(samples=0), None, out, b"samples"),
             (params(sample0=(1 << 32) - 3, samples=4), None, out, b"2^32"),
             (params(sample0=2, samples=(1 << 32) - 1), None, out, b"2^32"),
             (params(reserved=(1, 0)), None, out, b"reserved"),
             (params(reserved=(0, 9)), None, out, b"reserved"),
             (good, bad_view, out, b"view->reserved")]
    for p, view, o, what in cases:
        args = (C.byref(p) if p is not None else None, C.byref(view) if view is not None else None, C.byref(o) if o is not None else None)
        for fn, last in forms:
            assert fn(fake, *args, last) == -1, what
            assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
    assert (buf == 7.0).all()
    # the last sample index 2^32 - 1 is allowed: refused only later, for the stand-in handle's (absent) device memory, never here
    assert L.rtb200_scene_aov(None, C.byref(params(sample0=(1 << 32) - 1)), None, C.byref(out), None) == -1
    assert b"handle" in L.rtb200_last_error()


# ---- the oracle, pinned by two restatements ----------------------------------------------------------------------------

def _sat(x):
    """Rust `as u64` of a float: 0 for NaN and below 0."""
    return int(x) if x > 0 else 0


def _clamp(v):
    return F32(0) if v < 0 else (F32(1) if v > 1 else v)


def sky_restated(sc, d):
    """The miss branch of ray_color (raytracer.rs:134-163) for direction d, in f32 as the reference computes it."""
    mode = sc.c.sky.mode
    if mode == R.RT_SKY_NONE:
        return np.zeros(3, F32)
    l = math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
    t = _clamp(F32(0.5) * (F32(d[1] / l) + F32(1)))
    if mode == R.RT_SKY_GRADIENT:
        return np.array([(F32(1) - t) * F32(1) + t * F32(c) for c in (0.5, 0.7, 1.0)], F32)
    u = _clamp(F32(0.5) * (F32(d[0] / l) + F32(1)))
    W, H = int(sc.c.sky.tex.width), int(sc.c.sky.tex.height)
    x, y = _sat(u * F32(W - 1)), _sat((F32(1) - t) * F32(H - 1))
    px = sc._sky_array.reshape(-1)[(y * W + x) * 3:(y * W + x) * 3 + 3]
    return np.array([F32(0.7) * F32(c) / F32(255) for c in px], F32)


def texel_restated(sc, k, h_offset, u, v):
    """texture_get_albedo (materials.rs:236-253) of texture k at (u, v), clamped where the reference would panic."""
    img = sc.c.textures[k]
    W, H = int(img.width), int(img.height)
    rot = u + h_offset
    if rot > 1.0:
        rot = rot - 1.0
    base = 3 * (_sat(math.floor((1.0 - v) * float(H - 1))) * W + _sat(math.floor(rot * float(W))))
    base = min(base, W * H * 3 - 3)
    px = sc._tex_arrays[k].reshape(-1)[base:base + 3]
    return np.array([F32(c) / F32(255) for c in px], F32)


def albedo_restated(sc, d, hw):
    """albedo_s of every ray from the oracle's hits: the material table, the texture lookup at the hit's uv, the sky."""
    out = np.empty((len(d), 3), F32)
    for i in range(len(d)):
        j = int(hw["sphere"][i])
        if j < 0:
            out[i] = sky_restated(sc, d[i])
            continue
        s = sc._spheres[j]
        if s.kind in (R.RT_LAMBERTIAN, R.RT_METAL):
            out[i] = np.array(list(s.albedo), F32)
        elif s.kind == R.RT_TEXTURE:
            out[i] = texel_restated(sc, s.texture, s.param, hw["uv"][i, 0], hw["uv"][i, 1])
        else:
            out[i] = 1.0
    return out


def mean_in_sample_order(per_sample):
    acc = np.zeros_like(per_sample[0], F32)
    for x in per_sample:
        acc = (acc + x).astype(F32)
    return (F32(1) / F32(len(per_sample))) * acc


@pytest.mark.parametrize("name", list(aov_scenes()))
def test_one_sample_is_hit_world_of_the_primary_ray(name):
    sc = aov_scenes()[name]()
    w, h = int(sc.c.width), int(sc.c.height)
    for s in (0, 3):
        got = OA.aov(sc, 1, s)
        o, d = primary_rays(sc, s)
        hw = OH.hit_world(sc, o, d)
        hit = hw["sphere"] >= 0
        assert hit.any() and (~hit).any(), name   # both branches are exercised
        assert np.array_equal(got["sphere"].reshape(-1), hw["sphere"]), (name, s)
        assert np.array_equal(got["hits"].reshape(-1), hit.astype(np.uint32)), (name, s)
        pt = np.where(hit[:, None], hw["point"], 0.0)
        assert np.array_equal(got["point"].reshape(-1, 3).view(np.uint64), pt.view(np.uint64)), (name, s)
        nrm = np.where(hit[:, None], hw["normal"], 0.0).astype(F32)
        assert_f32_equal(got["normal"].reshape(-1, 3), nrm, f"{name}/s={s} normal")
        assert got["albedo"].shape == (h, w, 3)


@pytest.mark.parametrize("name", list(aov_scenes()))
def test_albedo_and_normal_equal_a_restatement_in_sample_order(name):
    sc = aov_scenes()[name]()
    for samples, sample0 in ((1, 0), (3, 2)):
        alb, nrm = [], []
        for s in range(sample0, sample0 + samples):
            o, d = primary_rays(sc, s)
            hw = OH.hit_world(sc, o, d)
            alb.append(albedo_restated(sc, d, hw))
            nrm.append(np.where((hw["sphere"] >= 0)[:, None], hw["normal"], 0.0).astype(F32))
        got = OA.aov(sc, samples, sample0)
        assert_f32_equal(got["albedo"].reshape(-1, 3), mean_in_sample_order(alb), f"{name}/{samples}@{sample0} albedo")
        assert_f32_equal(got["normal"].reshape(-1, 3), mean_in_sample_order(nrm), f"{name}/{samples}@{sample0} normal")
    if name == "mixed_lit_32x24":
        assert np.isnan(got["albedo"]).any() and np.isinf(got["albedo"]).any()


def test_a_scene_without_spheres_sees_the_sky():
    """No sphere: every sample misses, and the albedo of one sample is ray_color at max_depth 1 of the primary ray, the sky."""
    sc, _ = IR.scene_of([], 24, 16)
    for s in (0, 5):
        got = OA.aov(sc, 1, s)
        o, d = primary_rays(sc, s)
        want = OT.trace_rays(sc, o, d, 1, sample0=s, max_depth=1)["linear"]
        assert_f32_equal(got["albedo"].reshape(-1, 3), want, f"sky s={s}")
        assert (got["hits"] == 0).all() and (got["sphere"] == -1).all() and (got["point"] == 0).all() and (got["normal"] == 0).all()
