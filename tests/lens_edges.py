"""Lenses at the edges of what the ABI accepts (include/rtb200.h, DESIGN.md §3 and §4.17), shared by
tests/test_lens_edges_cpu.py, which checks on the host that every case reaches its edge, and tests/test_gpu_lens_edges.py,
which renders them. Every case is a scene and a lens; its reach is computed from the oracle's own rays (oracle_lens).

  E1 tiny       radius 2^-1074 (aperture 2^-1073): trials are drawn, but r*x rounds to 0 or +-2^-1074, so with a camera
                whose coordinates are neither 0 nor tiny the rays are the pinhole rays; tiny_zero_x puts look_from.x at 0,
                where some origins become +-2^-1074
  E2 negzero    radius -0.0: a pinhole
  E3 zero_uv    u = v = 0: trials are drawn and the offset vanishes (a pinhole); u_zero, v_zero and u_eq_v are line lenses,
                u_1e3 a lens with |u| = 1e3
  E4 huge       radius 1e300: every camera direction is about 1e300 long, so the f32 s of closest_hit is inf
  E5 glass_cut  the lens disk cuts a glass sphere; shell_cut, the hollow glass shell: some samples start inside it, some
                outside
  E6 far_lens   a spread scene seen through a lens of radius 1.4e15: |o - g| and |d| straddle 1e15; tiny_lens, focus_dist
                8e-16 and radius 1e-15: |d|^2 straddles 1e-30. Both put rays on either side of the flag test of closest_hit
  E7 fd_tiny    focus_dist 1e-300: the lower-left corner rounds to the origin and the pinhole direction is 0; fd_huge,
                focus_dist 1e308 at vfov 120: `horizontal` overflows and directions are not finite
  E8 deep_disk  a seed under which a small render has lens streams accepted at every trial 1..8 (both slots of trips 1-4)
"""
import math

import numpy as np

import f32_frame_cases as FC
import intersect_rays as IR
import oracle_lens as OL
import rtb200 as R
from test_aov_cpu import mixed_lit_scene

SEED64 = 0x9E3779B97F4A7C15    # a 64-bit key whose high word is nonzero and differs from its low word
TINY = 2.0 ** -1074
DEEP_SEED = 0x9E3779CC7F4A7C28  # found once by deep_seed_search(): the first seed it finds
DEEP_TRIALS = range(1, 9)


def lens_of(u, v, radius):
    return R.rt_lens(R.vec3(u), R.vec3(v), float(radius), 0)


def vec(v):
    return np.array(v.tup(), np.float64)


def _scene(w=24, h=16, spp=2, seed=SEED64, **cam):
    sc = mixed_lit_scene(w, h, spp)
    sc.c.max_depth = 6
    sc.seed = seed
    if cam:
        sc.set_camera(**cam)
    return sc


def _lensed(sc, aperture, focus_dist):
    """The scene's camera refocused at focus_dist, and its lens of radius aperture / 2; the scene keeps no lens."""
    p = sc.camera_params
    cam, lens = R.camera_from_params_lens(p["look_from"], p["look_at"], p["vup"], p["vfov"], p["aspect"], aperture, focus_dist)
    sc.c.camera = cam
    return sc, lens


def _basis(sc):
    """The lens of radius 0.3 on the scene's own camera basis (u, v)."""
    _, L = _lensed(_scene(), 0.6, 1.0)
    return vec(L.u), vec(L.v)


def _glass_scene(w=32, h=8, spp=2):
    """A glass sphere, a hollow glass shell (radius 1 around -0.8), ground and a light, seen from the side."""
    objs = [IR.sphere((0.0, -1000.0, 0.0), 1000.0),
            IR.sphere((0.0, 1.0, 0.0), 1.0, {"Glass": {"index_of_refraction": 1.5}}),
            IR.sphere((4.0, 1.0, 0.0), 1.0, {"Glass": {"index_of_refraction": 1.5}}),
            IR.sphere((4.0, 1.0, 0.0), -0.8, {"Glass": {"index_of_refraction": 1.5}}),
            IR.sphere((2.0, 4.0, -3.0), 0.7, {"Light": {}}),
            IR.sphere((1.0, 0.5, -4.0), 0.5, {"Metal": {"albedo": [0.8, 0.7, 0.6], "fuzz": 0.1}})]
    sc, _ = IR.scene_of(objs, w, h)
    sc.c.samples_per_pixel = spp
    sc.c.max_depth = 8
    sc.seed = SEED64
    return sc


GLASS = {"glass_cut": ((0.0, 1.0, 0.0), 1.0), "shell_cut": ((4.0, 1.0, 0.0), 0.8)}   # the sphere whose surface the disk cuts


def cases():
    """name -> (scene without a lens, lens)."""
    out = {}
    out["tiny"] = _lensed(_scene(), 2.0 ** -1073, 9.0)
    out["tiny_zero_x"] = _lensed(_scene(look_from=(0.0, 2.0, 10.0), look_at=(0.0, 0.5, 0.0)), 2.0 ** -1073, 9.0)
    u, v = _basis(_scene())
    out["negzero"] = (_scene(), lens_of(u, v, -0.0))
    out["zero_uv"] = (_scene(), lens_of((0, 0, 0), (0, 0, 0), 0.3))
    out["u_zero"] = (_scene(), lens_of((0, 0, 0), v, 0.3))
    out["v_zero"] = (_scene(), lens_of(u, (0, 0, 0), 0.3))
    out["u_eq_v"] = (_scene(), lens_of(u, u, 0.3))
    out["u_1e3"] = (_scene(), lens_of(1e3 * u, v, 3e-4))
    out["huge"] = (_scene(), lens_of(u, v, 1e300))
    for name, (c, r) in GLASS.items():
        sc = _glass_scene()
        lf = (c[0] + r - 0.05 + (0.1 if name == "shell_cut" else 0.0), c[1], c[2])
        sc.set_camera(look_from=lf, look_at=(lf[0], lf[1], -5.0), vfov=60.0)
        out[name] = _lensed(sc, 0.4, 3.0)
    far = FC.spread_scene(1e12)
    far.seed = SEED64
    far.c.samples_per_pixel = 2
    out["far_lens"] = _lensed(far, 2.8e15, 10.0)
    near = FC.spread_scene(1e12)
    near.seed = SEED64
    near.c.samples_per_pixel = 2
    out["tiny_lens"] = _lensed(near, 2e-15, 8e-16)
    out["fd_tiny"] = _lensed(_scene(), 0.4, 1e-300)
    out["fd_huge"] = _lensed(_scene(vfov=120.0), 0.4, 1e308)
    out["deep_disk"] = _lensed(_scene(32, 24, 8, seed=DEEP_SEED), 0.5, 9.0)
    return out


PINHOLE = ("tiny", "negzero", "zero_uv")   # cases whose rays are the pinhole rays bit for bit


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def rays(sc, lens):
    """(origins, directions) [spp, h*w, 3] of every camera sample of sc through `lens` (None: the pinhole)."""
    o, d = zip(*(OL.primary(sc, lens, s) for s in range(int(sc.c.samples_per_pixel))))
    return np.stack(o), np.stack(d)


def stream_trials(sc, lens):
    """The oracle's lens trials of every stream (pixel, sample) of sc's render: uint32 [spp, h*w]."""
    n, spp = int(sc.c.width) * int(sc.c.height), int(sc.c.samples_per_pixel)
    return np.array([[OL.lens_ray(sc.c.camera, lens, sc.seed, p, s, 0.5, 0.5)[2] for p in range(n)] for s in range(spp)], np.uint32)


def deep_seed_search(start=SEED64, tries=4096):
    """The first seed start + k * 0x100000001 whose deep_disk render has streams accepted at every trial of DEEP_TRIALS."""
    for k in range(tries):
        seed = (start + k * 0x100000001) & 0xFFFFFFFFFFFFFFFF
        sc, lens = _lensed(_scene(32, 24, 8, seed=seed), 0.5, 9.0)
        if set(DEEP_TRIALS) <= set(np.unique(stream_trials(sc, lens)).tolist()):
            return seed
    return None


def _runs_with_both(flags, w=32):
    """True when some run of w consecutive entries of some row of `flags` [rows, n] holds both True and False."""
    f = np.asarray(flags)
    n = f.shape[-1] // w * w
    r = f[..., :n].reshape(f.shape[0], -1, w)
    return bool((r.any(-1) & ~r.all(-1)).any())


def reach(name, sc, lens):
    """The edge case `name` reaches, computed from the oracle; raises AssertionError when it does not."""
    o, d = rays(sc, lens)
    po, pd = rays(sc, None)
    if name in PINHOLE:
        assert _same(o, po) and _same(d, pd), f"{name}: the lens rays are not the pinhole rays"
    if name in ("tiny", "tiny_zero_x"):
        assert lens.radius == TINY, lens.radius
    if name in ("tiny", "tiny_zero_x", "zero_uv", "u_zero", "v_zero", "u_eq_v", "u_1e3", "deep_disk"):
        t = stream_trials(sc, lens)
        assert (t > 0).all(), f"{name}: a lens stream drew no trial"
    if name == "tiny_zero_x":
        assert sc.c.camera.origin.x == 0.0
        x = o[..., 0]
        assert (x == TINY).any() and (x == -TINY).any() and (x == 0.0).any(), f"{name}: no origin at +-2^-1074"
    if name == "negzero":
        assert lens.radius == 0.0 and math.copysign(1.0, lens.radius) < 0
    if name in ("u_zero", "v_zero", "u_eq_v", "u_1e3"):
        assert not _same(o, po), f"{name}: the lens moved no origin"
        off = o - po
        axis = {"u_zero": vec(lens.v), "v_zero": vec(lens.u), "u_eq_v": vec(lens.u)}.get(name)
        if axis is not None:   # a line lens: every offset lies on one line
            assert np.allclose(np.cross(off.reshape(-1, 3), axis), 0.0, atol=1e-12), f"{name}: not a line lens"
        else:
            assert np.abs(off).max() > 0.2, f"{name}: |u| = 1e3 did not scale the offsets"
    if name == "huge":
        assert (FC.f32_s(d.reshape(-1, 3)) >= FC.S_HI).all(), f"{name}: some f32 s is below 1e30"
    if name in GLASS:
        c, r = GLASS[name]
        inside = ((o - np.array(c)) ** 2).sum(-1) < r * r
        w = int(sc.c.width)
        assert _runs_with_both(inside.reshape(-1, w)), f"{name}: no 32-pixel run of a row starts both inside and outside"
    if name in ("far_lens", "tiny_lens"):
        g = R.bvh_records(sc)["recentre"]
        s = np.stack([FC.sides(o[k], d[k], g) for k in range(len(o))])   # work ids: [sample][pixel]
        both = (s == 1).reshape(-1, 32).any(-1) & (s == -1).reshape(-1, 32).any(-1)
        assert both.any(), f"{name}: no warp-sized run of work ids on both sides of the flag test"
    if name == "fd_tiny":
        assert (pd == 0.0).all(), f"{name}: a pinhole direction is not 0"
        assert not (d == 0.0).all(-1).any(), f"{name}: the lens left a direction at 0"
    if name == "fd_huge":
        assert not np.isfinite(vec(sc.c.camera.horizontal)).all(), f"{name}: horizontal is finite"
        assert not np.isfinite(d).all(), f"{name}: every direction is finite"
    if name == "deep_disk":
        assert set(DEEP_TRIALS) <= set(np.unique(stream_trials(sc, lens)).tolist()), f"{name}: some trial of 1..8 never accepts"
