"""Lenses at the edges of what the ABI accepts (tests/lens_edges.py, DESIGN.md §3) on the GPU, bit for bit against the lens
oracle in linear f32, RGB8 and rays (NaN payloads free): through a one-shot frame table, through rtb200_scene_set_lens on a
resident handle, and through the device's lens routine. tests/test_lens_edges_cpu.py checks that every case reaches its edge."""
import numpy as np
import pytest

import lens_edges as LE
import oracle_lens as OL
import rtb200 as R
from test_gpu_intersect import BRUTE, EXACT, FILTERED, _torch
from test_gpu_lens import bits

pytestmark = pytest.mark.gpu
CASES = LE.cases()


def probe(cam, lens, seed, pixel, sample, u=0.5, v=0.5):
    o, d, t = R.rt_vec3(), R.rt_vec3(), R.C.c_uint32()
    R._check(R.lib().rtb200_probe_lens_ray(R.C.byref(cam), R.C.byref(lens), seed, pixel, sample, u, v, R.C.byref(o), R.C.byref(d), R.C.byref(t)))
    return np.array([o.x, o.y, o.z, d.x, d.y, d.z]), int(t.value)


def assert_probe(cam, lens, seed, pixel, sample, what):
    got, t = probe(cam, lens, seed, pixel, sample)
    wo, wd, wt = OL.lens_ray(cam, lens, seed, pixel, sample, 0.5, 0.5)
    assert bits(got) == bits(np.concatenate([wo, wd])), what
    assert t == wt, (what, t, wt)
    return t


def one_shot(sc, lens, variant=FILTERED):
    """linear, RGB8 and stats of the one-frame lens render (rtb200_render_frames_lens)."""
    f = R.rt_frame(sc.c.camera, sc.seed, sc.c.max_depth, 0)
    opts = R.make_options(device=0, variant=variant)
    lin, st = R.render_frames(sc, [f], opts, linear=True, lenses=[lens])
    rgb, _ = R.render_frames(sc, [f], opts, lenses=[lens])
    return lin[0], rgb[0], st


def resident(sc, lens, variant=FILTERED):
    """linear f32 of the handle's render after set_lens(lens)."""
    torch = _torch()
    rs = R.ResidentScene(sc, R.make_options(device=0, variant=variant))
    try:
        rs.set_lens(lens)
        buf = torch.empty((int(sc.c.height), int(sc.c.width), 3), dtype=torch.float32, device="cuda:0")
        rs.render(0, buf.data_ptr())
        return buf.cpu().numpy()
    finally:
        rs.release()


@pytest.mark.parametrize("name", list(CASES))
def test_edge_lens_renders_the_oracle(name):
    sc, lens = CASES[name]
    want = OL.render(sc, lens)
    variants = [FILTERED, EXACT, BRUTE] if name in ("far_lens", "tiny_lens", "huge") else [FILTERED]
    for variant in variants:
        lin, rgb, st = one_shot(sc, lens, variant)
        assert bits(lin) == bits(want["linear"]), (name, variant)
        assert np.array_equal(rgb, want["rgb8"]), (name, variant)
        assert st["rays"] == want["rays"], (name, variant, st["rays"], want["rays"])
        assert bits(resident(sc, lens, variant)) == bits(want["linear"]), (name, variant, "set_lens")
    if name in LE.PINHOLE:   # the lens renders the pinhole frame, and the pinhole kernels render it too
        pin, _ = R.render_linear(sc, R.make_options(device=0))
        assert bits(lin) == bits(pin) == bits(OL.render(sc, None)["linear"]), name


def test_tiny_radius_draws_trials_on_the_device():
    """At radius 2^-1074 the device draws the oracle's trials, and at look_from.x == 0 moves origins to +-2^-1074."""
    for name in ("tiny", "tiny_zero_x"):
        sc, lens = CASES[name]
        n = int(sc.c.width) * int(sc.c.height)
        o, _ = LE.rays(sc, lens)
        for p in range(0, n, 7):
            assert assert_probe(sc.c.camera, lens, sc.seed, p, 1, f"{name} pixel {p}") > 0
        if name == "tiny_zero_x":   # streams whose origin the oracle moved off 0
            moved = np.nonzero(o[0, :, 0] != 0.0)[0][:16]
            assert len(moved) > 0
            for p in moved:
                got, _ = probe(sc.c.camera, lens, sc.seed, int(p), 0)
                assert got[0] in (LE.TINY, -LE.TINY), (p, got[0])


def test_deep_disk_trials_on_the_device():
    """The probe on the streams the oracle accepts at each trial 1..8: the same ray and the same trial count."""
    sc, lens = CASES["deep_disk"]
    t = LE.stream_trials(sc, lens)
    for k in LE.DEEP_TRIALS:
        s, p = (int(a[0]) for a in np.nonzero(t == k))
        assert assert_probe(sc.c.camera, lens, sc.seed, p, s, f"trial {k}") == k


def test_negative_zero_radius_uploads_no_lens_table():
    """Frames whose lenses all have radius -0.0 (or 0) run the pinhole kernels: the frame table alone is uploaded."""
    torch = _torch()
    sc, lens = CASES["negzero"]
    rs = R.ResidentScene(sc, R.make_options(device=0))
    try:
        w, h = int(sc.c.width), int(sc.c.height)
        frames = [R.rt_frame(sc.c.camera, sc.seed + k, sc.c.max_depth, 0) for k in range(3)]
        out = torch.empty((3, h, w, 3), dtype=torch.float32, device="cuda:0")
        st = rs.render_frames(frames, dev_linear_ptr=out.data_ptr(), lenses=[lens, R.rt_lens(), lens])
        assert st["h2d_bytes"] == 3 * 104, st["h2d_bytes"]
        for k in range(3):
            one = R.Scene.edited(sc)
            one.seed = sc.seed + k
            assert bits(out[k].cpu().numpy()) == bits(OL.render(one, None)["linear"]), k
    finally:
        rs.release()
