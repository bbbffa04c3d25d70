"""Radiance of caller-supplied rays without a GPU (rtb200_scene_trace_rays[_device], DESIGN.md §4.12): the exported entry points,
the layout of rt_trace_params, the argument checks that run before any device work, and the oracle the GPU tests hold the
kernel to, pinned to the render: when ray p is the render's primary ray of (pixel p, sample s), oracle_trace_rays with
sample0 = s equals that sample of the render bit for bit, and the f32 sums over samples equal the rendered image."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle_py as O
import oracle_trace_rays as OT
import rtb200 as R
from rtb200 import scenes


def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_scene_trace_rays_device", "rtb200_scene_trace_rays"):
        assert name in R.ABI_SYMBOLS
        assert getattr(L, name) is not None


def test_trace_params_layout_matches_the_header(repo, tmp_path):
    assert C.sizeof(R.rt_trace_params) == 32
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rtb200.h"\nint main(void) {\n'
                   '    printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(rt_trace_params), offsetof(rt_trace_params, seed),\n'
                   '           offsetof(rt_trace_params, samples), offsetof(rt_trace_params, sample0), offsetof(rt_trace_params, stream0),\n'
                   '           offsetof(rt_trace_params, max_depth), offsetof(rt_trace_params, reserved));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Werror", "-I", os.path.join(repo, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [C.sizeof(R.rt_trace_params)] + [getattr(R.rt_trace_params, f).offset for f, _ in R.rt_trace_params._fields_]
    assert got == want == [32, 0, 8, 12, 16, 20, 24]


def test_bad_arguments_are_refused_before_any_device_work():
    """A NULL handle, NULL rays or params, a NULL origin or direction, a t_max, both outputs NULL, samples == 0, a nonzero
    reserved word and u32 overflows of the streams and sample indices are refused with RT_ERR_INVALID. The checks come before
    the handle is used, so a stand-in handle that is never dereferenced shows the order."""
    L = R.lib()
    o = np.zeros((4, 3)); d = np.ones((4, 3)); t = np.ones(4)
    lin = np.full((4, 3), 7.0, np.float32); rgb = np.full((4, 3), 7, np.uint8)
    rays = R.rt_rays(o.ctypes.data, d.ctypes.data, None)
    good = R.rt_trace_params(1, 1, 0, 0, 4)
    st = R.rt_stats()
    for fn, last in ((L.rtb200_scene_trace_rays, (C.byref(st),)), (L.rtb200_scene_trace_rays_device, (None, C.byref(st)))):
        assert fn(None, C.byref(rays), 4, C.byref(good), lin.ctypes.data, rgb.ctypes.data, *last) == -1
        assert b"handle" in L.rtb200_last_error()
    fake = C.c_void_p(C.addressof(C.create_string_buffer(64)))

    def params(**kw):
        p = R.rt_trace_params(1, 1, 0, 0, 4)
        for k, v in kw.items():
            if k == "reserved":
                p.reserved[v[0]] = v[1]
            else:
                setattr(p, k, v)
        return p

    cases = [(None, good, 4, True, True, b"rays"),
             (rays, None, 4, True, True, b"params"),
             (R.rt_rays(None, d.ctypes.data, None), good, 4, True, True, b"origin"),
             (R.rt_rays(o.ctypes.data, None, None), good, 4, True, True, b"direction"),
             (R.rt_rays(o.ctypes.data, d.ctypes.data, t.ctypes.data), good, 4, True, True, b"t_max"),
             (rays, good, 4, False, False, b"both null"),
             (rays, params(samples=0), 4, True, False, b"samples"),
             (rays, params(reserved=(0, 1)), 4, False, True, b"reserved"),
             (rays, params(reserved=(1, 5)), 4, True, True, b"reserved"),
             (rays, params(stream0=(1 << 32) - 3), 4, True, True, b"stream0"),
             (rays, params(sample0=(1 << 32) - 2, samples=3), 4, True, True, b"sample0"),
             (rays, params(sample0=2, samples=(1 << 32) - 1), 4, True, True, b"sample0")]
    for r, p, n, want_lin, want_rgb, what in cases:
        rp = C.byref(r) if r is not None else None
        pp = C.byref(p) if p is not None else None
        lp = lin.ctypes.data if want_lin else None
        gp = rgb.ctypes.data if want_rgb else None
        assert L.rtb200_scene_trace_rays(fake, rp, n, pp, lp, gp, C.byref(st)) == -1, what
        assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
        assert L.rtb200_scene_trace_rays_device(fake, rp, n, pp, lp, gp, None, C.byref(st)) == -1, what
        assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
    assert (lin == 7.0).all() and (rgb == 7).all()


# ---- the oracle, pinned to the render ---------------------------------------------------------------------------------

def primary_rays(sc, s):
    """The render's primary ray of (pixel p, sample s) for every pixel p of the frame, top row first: the pixel jitter of
    raytracer.rs:199-200 from the oracle's RNG stream and Camera::get_ray (camera.rs:79-84) from the oracle."""
    w, h = int(sc.c.width), int(sc.c.height)
    L = O.lib()
    xi = np.empty((w * h, 2))
    for p in range(w * h):
        L.oracle_rng(sc.seed, p, s, 0, 2, xi[p].ctypes.data_as(C.POINTER(C.c_double)))
    y, x = np.divmod(np.arange(w * h, dtype=np.float64), w)
    u = (x + xi[:, 0]) / (w - 1.0)
    v = (h - (y + xi[:, 1])) / (h - 1.0)
    cam = sc.c.camera
    org = np.array(cam.origin.tup())
    # camera.rs:79-84 in the oracle's order of f64 operations (numpy rounds each one, like the oracle)
    d = ((np.array(cam.lower_left_corner.tup()) + np.array(cam.horizontal.tup()) * u[:, None]) + np.array(cam.vertical.tup()) * v[:, None]) - org
    o = np.broadcast_to(org, d.shape).copy()
    ro, rd = R.rt_vec3(), R.rt_vec3()
    for p in range(0, w * h, 97):   # the same rays as the oracle's own Camera::get_ray
        L.oracle_get_ray(C.byref(cam), float(u[p]), float(v[p]), C.byref(ro), C.byref(rd))
        assert ro.tup() == tuple(o[p]) and rd.tup() == tuple(d[p]), p
    return o, np.ascontiguousarray(d)


def quantise(lin):
    """The render's RGB8 of a linear mean: quantise(sqrt(mean)), the oracle's own routine."""
    flat = np.ascontiguousarray(lin, np.float32).reshape(-1)
    out = np.empty(flat.size, np.uint8)
    O.lib().oracle_quantise(flat.ctypes.data, flat.size, out.ctypes.data)
    return out.reshape(np.shape(lin))


def sum_samples(per_sample, spp):
    """The render's resolve of per-sample radiances [spp][n, 3]: f32 sums in sample order, times 1.0f / spp."""
    acc = np.zeros_like(per_sample[0], np.float32)
    for x in per_sample:
        acc = (acc + x).astype(np.float32)
    return (np.float32(1.0) / np.float32(spp)) * acc


def pinned_scenes():
    cover = scenes.cover_scene(40, 30, 4)
    test = R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 40, 30, 4, 12), scenes.SCENES_DIR)
    return {"cover_40x30_s4": cover, "test_scene_40x30_s4": test}


@pytest.mark.parametrize("name", ["cover_40x30_s4", "test_scene_40x30_s4"])
def test_the_oracle_is_pinned_to_the_render(name):
    sc = pinned_scenes()[name]
    w, h, spp = int(sc.c.width), int(sc.c.height), int(sc.c.samples_per_pixel)
    if name.startswith("test_scene"):
        assert any(sc._spheres[i].kind == R.RT_LIGHT for i in range(sc.n_spheres)) and sc.c.n_textures > 0
    lin_o, img_o, st_o = O.render(sc)
    per_sample, rays = [], 0
    for s in range(spp):
        o, d = primary_rays(sc, s)
        got = OT.trace_rays(sc, o, d, samples=1, sample0=s)
        rays += got["rays"]
        want = np.empty((w * h, 3), np.float32)
        for p in range(w * h):
            want[p], _, _ = O.sample(sc, p % w, p // w, s)
        assert np.array_equal(got["linear"].view(np.uint32), want.view(np.uint32)), f"{name}: sample {s}"
        assert np.array_equal(got["rgb8"], quantise(want))
        per_sample.append(got["linear"])
    lin = sum_samples(per_sample, spp).reshape(h, w, 3)
    assert np.array_equal(lin.view(np.uint32), lin_o.view(np.uint32)), name
    assert np.array_equal(quantise(lin), img_o), name
    assert rays == st_o["rays"]


def test_the_oracle_resolves_many_samples_like_a_render():
    """samples = m in one call equals m single-sample calls summed in sample order, for a pixel-centre ray set; and with
    sample0 it continues the streams where a shorter call stopped."""
    sc = scenes.cover_scene(16, 12, 1)
    rng = np.random.default_rng(3)
    o = np.broadcast_to(np.array(sc.c.camera.origin.tup()), (64, 3)).copy()
    d = rng.normal(size=(64, 3))
    d[:, 2] = -np.abs(d[:, 2]) - 0.5
    for m, s0, k in ((5, 0, 9), (3, 7, 1), (1, 2, 100)):
        one = OT.trace_rays(sc, o, d, samples=m, sample0=s0, stream0=k)
        parts = [OT.trace_rays(sc, o, d, samples=1, sample0=s0 + j, stream0=k)["linear"] for j in range(m)]
        want = sum_samples(parts, m)
        assert np.array_equal(one["linear"].view(np.uint32), want.view(np.uint32)), (m, s0, k)
        assert np.array_equal(one["rgb8"], quantise(want))
    # max_depth 0: black, no ray
    z = OT.trace_rays(sc, o, d, samples=3, max_depth=0)
    assert (z["linear"] == 0).all() and (z["rgb8"] == 0).all() and z["rays"] == 0
