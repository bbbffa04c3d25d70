"""Temporal accumulation without a GPU (rtb200_temporal[_device], DESIGN.md §4.16): the two numpy restatements of the contract
held equal bit for bit on edge inputs, every branch of the contract reached, a static camera reprojecting every pixel onto
itself, the exported entry points, the layouts and defaults of include/rtb200.h, the argument checks that run before any device
work, and the quality of the chosen defaults on an orbit of the oracle's cover render."""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import temporal_restatement as TR
import rtb200 as R

F32, F64 = np.float32, np.float64
MISS = 0xFFFFFFFF
BIG = 0xFFFFFFFF


def assert_history_equal(got, want, what=""):
    (gc, gn), (wc, wn) = got, want
    gc, wc = np.asarray(gc, F32), np.asarray(wc, F32)
    assert gc.shape == wc.shape, (what, gc.shape, wc.shape)
    nan, nan_w = np.isnan(gc), np.isnan(wc)
    assert np.array_equal(nan, nan_w), f"{what}: NaN in {int(nan.sum())} values here, {int(nan_w.sum())} in the reference"
    diff = (gc.view(np.uint32) != wc.view(np.uint32)) & ~nan
    assert not diff.any(), f"{what}: {int(diff.sum())} colour values differ, first at {np.argwhere(diff)[0].tolist()}"
    assert np.array_equal(np.asarray(gn, np.uint32), np.asarray(wn, np.uint32)), f"{what}: lengths differ"


# ---- cases -----------------------------------------------------------------------------------------------------------------

def dyadic_camera(w, h, shift_px=(0.0, 0.0), origin=(0.0, 0.0, 0.0)):
    """An axis-aligned camera whose values are dyadic for w - 1 and h - 1 powers of two, shifted by whole or half pixels: its
    motion vectors are exact, so taps land exactly on pixel centres, halves and borders."""
    o = np.array(origin, F64)
    hx, vy = F64(2.0), F64(1.5)
    sx = shift_px[0] * hx / max(w - 1, 1)
    sy = shift_px[1] * vy / max(h - 1, 1)
    return (o, o + np.array([-1.0 + sx, -0.75 + sy, -1.0]), np.array([hx, 0.0, 0.0]), np.array([0.0, vy, 0.0]))


def orbit_camera(w, h, angle_deg, dist=13.0):
    a = math.radians(angle_deg)
    cam = R.camera_from_params([dist * math.cos(a), 2.0, dist * math.sin(a)], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0], 20.0, w / h)
    return TR.camera_arrays(cam)


def synth_frame(w, h, cam, rng, n_spheres=4, miss=0.2):
    """Points on the camera's rays at random depths, with random sphere ids and misses."""
    o, llc, hh, vt = cam
    y, x = np.meshgrid(np.arange(h, dtype=F64), np.arange(w, dtype=F64), indexing="ij")
    u = (x + rng.uniform(0, 1, (h, w))) / max(w - 1, 1)
    v = (h - (y + rng.uniform(0, 1, (h, w)))) / max(h - 1, 1)
    d = llc + hh * u[..., None] + vt * v[..., None] - o
    t = rng.uniform(0.5, 4.0, (h, w))
    point = o + d * t[..., None]
    sphere = rng.integers(0, n_spheres, (h, w)).astype(np.uint32)
    m = rng.random((h, w)) < miss
    sphere[m] = MISS
    point[m] = 0.0
    color = rng.uniform(0, 1.5, (h, w, 3)).astype(F32)
    return color, sphere, point


def edge_case(w, h, seed, *, cam=None, pcam=None, special=0.15, max_len=20):
    """A frame and a previous frame of w x h pixels with NaN and +-inf colours, points and history, points behind the cameras
    and on the camera origin (den = 0), mismatched and miss ids, and lengths 0, 1, big and 2^32 - 1."""
    rng = np.random.default_rng(seed)
    cam = cam if cam is not None else dyadic_camera(w, h)
    pcam = pcam if pcam is not None else dyadic_camera(w, h, (0.5, -1.0))
    color, sphere, point = synth_frame(w, h, cam, rng)
    hcol, hsph, hpt = synth_frame(w, h, pcam, rng)
    hsph = np.where(rng.random((h, w)) < 0.7, sphere, hsph).astype(np.uint32)     # mostly the same surfaces
    hpt = np.where(rng.random((h, w, 1)) < 0.7, point + rng.normal(0, 0.01, (h, w, 3)), hpt)
    hlen = rng.integers(0, max_len, (h, w)).astype(np.uint32)
    hlen[rng.random((h, w)) < 0.1] = BIG
    specials = np.array([np.nan, np.inf, -np.inf], F32)
    for a in (color, hcol):
        m = rng.random(a.shape) < special
        a[m] = rng.choice(specials, int(m.sum()))
    m = rng.random((h, w)) < special
    point[m] = rng.choice([np.nan, np.inf, -np.inf, 0.0], (int(m.sum()), 3))   # 0 is the dyadic cameras' origin: den = 0
    m = rng.random((h, w)) < special
    point[m] = cam[0] - (point[m] - cam[0])                                        # behind the camera
    m = rng.random((h, w, 3)) < special / 3
    hpt[m] = np.nan
    motion = rng.normal(0, 0.02, (3, 3))
    motion[1] = [np.nan, 0.0, 0.0]
    motion[2] = [np.inf, 0.0, 0.0] if seed % 2 else [0.0, 0.0, 0.0]
    prev = {"color": hcol, "length": hlen, "sphere": hsph, "point": hpt, "camera": pcam}
    return color, sphere, point, cam, prev, motion


CAMERA_PAIRS = {
    "static": (0.0, 0.0), "half_right": (0.5, 0.0), "half_diag": (-0.5, 0.5), "one_up": (0.0, 1.0), "border": (4.0, -2.0),
    "off_image": (40.0, 0.0),
}


@pytest.mark.parametrize("w,h", [(1, 1), (1, 2), (2, 1), (2, 2), (5, 3), (9, 5), (17, 9)])
@pytest.mark.parametrize("pair", list(CAMERA_PAIRS))
def test_restatements_agree_on_edge_inputs(w, h, pair):
    shift = CAMERA_PAIRS[pair]
    for seed, (N, tol, mot) in enumerate([(8, 0.03, True), (1, 0.03, False), (2, 0.0, True), (BIG, 1e300, False), (5, 0.5, True)]):
        color, sphere, point, cam, prev, motion = edge_case(w, h, 100 * seed + w * h, pcam=dyadic_camera(w, h, shift))
        kw = dict(motion=motion if mot else None, max_history=N, depth_tol=tol)
        a = TR.temporal(color, sphere, point, cam, prev, **kw)
        b = TR.temporal_scalar(color, sphere, point, cam, prev, **kw)
        assert_history_equal(a, b, f"{w}x{h}/{pair}/N={N}/tol={tol}")


@pytest.mark.parametrize("w,h", [(1, 1), (2, 2), (7, 5), (16, 12)])
def test_restatements_agree_on_an_orbit_step(w, h):
    for seed, step in enumerate((0.0, 0.5, 3.0, 179.0)):
        cam, pcam = orbit_camera(w, h, 10.0 + step), orbit_camera(w, h, 10.0)
        color, sphere, point, _, prev, motion = edge_case(w, h, seed, cam=cam, pcam=pcam, special=0.05)
        for kw in (dict(max_history=8, depth_tol=0.03), dict(max_history=2, depth_tol=1e-3, motion=motion)):
            assert_history_equal(TR.temporal(color, sphere, point, cam, prev, **kw),
                                 TR.temporal_scalar(color, sphere, point, cam, prev, **kw), f"{w}x{h}/step {step}/{kw}")


def test_no_previous_frame_and_non_finite_colours_pass_through():
    color, sphere, point, cam, prev, _ = edge_case(5, 3, 1)
    for fn in (TR.temporal, TR.temporal_scalar):
        c, n = fn(color, sphere, point, cam, None, max_history=8, depth_tol=0.03)
        assert (n == 1).all() and np.array_equal(c.view(np.uint32), color.view(np.uint32))
        c, n = fn(color, sphere, point, cam, prev, max_history=8, depth_tol=0.03)
        bad = ~np.isfinite(color).all(axis=2)
        assert bad.any() and (n[bad] == 1).all()
        assert np.array_equal(c[bad].view(np.uint32), color[bad].view(np.uint32))


def _one_pixel_prev(w, h, cam, color, sphere, point, length=3):
    return {"color": np.array(color, F32, copy=True), "length": np.full((h, w), length, np.uint32), "sphere": np.array(sphere, np.uint32),
            "point": np.array(point, F64, copy=True), "camera": cam}


def test_the_edge_values_reach_every_branch():
    """Each rule of the contract decides at least one pixel of a 5 x 5 image under a static dyadic camera."""
    w = h = 5
    cam = dyadic_camera(w, h)
    rng = np.random.default_rng(3)
    color, sphere, point = synth_frame(w, h, cam, rng, miss=0.0)
    sphere[:] = 1
    sphere[4, :] = MISS
    point[4, :] = 0.0
    prev = _one_pixel_prev(w, h, cam, np.full((h, w, 3), 0.25, F32), sphere, point)

    def run(prev=prev, color=color, sphere=sphere, point=point, **kw):
        kw = {"max_history": 8, "depth_tol": 0.03, **kw}
        a = TR.temporal(color, sphere, point, cam, prev, **kw)
        assert_history_equal(a, TR.temporal_scalar(color, sphere, point, cam, prev, **kw))
        return a

    c, n = run()
    assert (n == 4).all()                                   # min(3, 7) + 1 everywhere: hits and misses keep their history
    assert np.array_equal(c, 0.25 + F32(0.25) * (color - F32(0.25)))
    # 1. a non-finite colour
    col = color.copy(); col[0, 0, 1] = np.nan
    assert run(color=col)[1][0, 0] == 1
    # 2./3. a point on the camera origin (den = 0) and one behind the camera
    pt = point.copy(); pt[0, 1] = cam[0]; pt[0, 2] = cam[0] - (point[0, 2] - cam[0])
    _, n = run(point=pt)
    assert n[0, 1] == 1 and n[0, 2] == 1
    # 4. a non-finite motion
    _, n = run(motion=np.array([[0, 0, 0], [np.nan, 0, 0]], F64))
    assert (n[:4] == 1).all() and (n[4] == 4).all()         # sphere 1's pixels lose their history, the misses keep theirs
    # 5. taps: length 0, non-finite history, another sphere, a point beyond the depth tolerance
    pv = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in prev.items()}
    pv["length"][1, 0] = 0
    pv["color"][1, 1, 2] = np.inf
    pv["sphere"][1, 2] = 2
    pv["point"][1, 3] += 0.5
    _, n = run(prev=pv)
    assert (n[1, :4] == 1).all() and n[1, 4] == 4
    _, n = run(prev=pv, depth_tol=1e300)
    assert n[1, 3] == 4
    _, n = run(prev=pv, depth_tol=0.0)
    assert n[1, 3] == 1 and (n[0] == 4).all()              # depth_tol 0: the same point only
    # 6. N = 1 keeps nothing; N = 2^32 - 1 with L = 2^32 - 1 counts to 2^32 - 1 without wrapping
    assert (run(max_history=1)[1] == 1).all()
    pv = dict(prev, length=np.full((h, w), BIG, np.uint32))
    c, n = run(prev=pv, max_history=BIG)
    assert (n == BIG).all()
    assert np.array_equal(c, 0.25 + (F32(1) / F32(BIG)) * (color - F32(0.25)))
    # a camera 1.5 pixels to the left of the previous one puts both taps of the first column outside the image
    cam2 = dyadic_camera(w, h, (-1.5, 0.0))
    c, n = TR.temporal(color, sphere, point, cam2, dict(prev, camera=cam), max_history=8, depth_tol=1e300)
    assert (n[:, 0] == 1).all() and (n[:, 1:] == 4).all()
    assert_history_equal((c, n), TR.temporal_scalar(color, sphere, point, cam2, dict(prev, camera=cam), max_history=8, depth_tol=1e300))


def test_a_static_camera_reprojects_every_pixel_onto_itself():
    """With the same camera and no motion, fx = x and fy = y exactly: the one tap of weight 1 is the pixel's own history."""
    for w, h, cam in ((16, 12, orbit_camera(16, 12, 33.0)), (9, 5, dyadic_camera(9, 5))):
        rng = np.random.default_rng(w)
        color, sphere, point = synth_frame(w, h, cam, rng)
        hist = rng.uniform(0, 1, (h, w, 3)).astype(F32)
        # the neighbours of each pixel differ in colour and length: any other tap would show. Pixel (2, 2) has a history of
        # 1 frame among neighbours of 6 that see the same surface (the sky: no depth test), so each of them has a valid tap
        # of weight 0 on it; those taps are skipped, so pixel (2, 2) does not cut their lengths
        sphere[1:4, 1:4] = MISS
        point[1:4, 1:4] = 0.0
        length = np.full((h, w), 6, np.uint32)
        length[2, 2] = 1
        length[0, 1::2] = rng.integers(1, 9, length[0, 1::2].shape)
        prev = {"color": hist, "length": length, "sphere": sphere, "point": point, "camera": cam}
        c, n = TR.temporal(color, sphere, point, cam, prev, max_history=4, depth_tol=0.0)
        assert np.array_equal(n, np.minimum(length, 3) + 1)
        assert n[2, 2] == 2 and n[1, 2] == n[2, 1] == n[2, 3] == n[3, 2] == n[3, 3] == 4
        alpha = (F32(1) / (np.minimum(length, 3) + 1).astype(F32))[..., None]
        assert np.array_equal(c, hist + alpha * (color - hist))
        assert_history_equal((c, n), TR.temporal_scalar(color, sphere, point, cam, prev, max_history=4, depth_tol=0.0))


def test_restatement_refusals():
    c, s, p, cam, prev, _ = edge_case(2, 2, 0)
    for kw in (dict(max_history=0, depth_tol=0.0), dict(max_history=1, depth_tol=-1e-300), dict(max_history=1, depth_tol=np.nan),
               dict(max_history=1, depth_tol=np.inf)):
        with pytest.raises(ValueError):
            TR.temporal(c, s, p, cam, prev, **kw)


# ---- the ABI -----------------------------------------------------------------------------------------------------------

def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_temporal_device", "rtb200_temporal"):
        assert name in R.ABI_SYMBOLS
        assert getattr(L, name) is not None


def _compile_and_run(repo, tmp_path, name, body):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / f"{name}.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rtb200.h"\nint main(void) {\n' + body + '    return 0;\n}\n')
    exe = tmp_path / name
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Werror", "-I", os.path.join(repo, "include"), str(src), "-o", str(exe)])
    return subprocess.check_output([str(exe)]).decode().split()


@pytest.mark.parametrize("struct,size", [("rt_temporal_params", 224), ("rt_temporal_frame", 24), ("rt_temporal_history", 32),
                                         ("rt_temporal_out", 16)])
def test_struct_layouts_match_the_header(repo, tmp_path, struct, size):
    cls = getattr(R, struct)
    fields = [f for f, _ in cls._fields_]
    got = [int(x) for x in _compile_and_run(repo, tmp_path, "layout", '    printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(' + struct + ')'
                                            + "".join(f", offsetof({struct}, {f})" for f in fields) + ');\n')]
    mirror = [C.sizeof(cls)] + [getattr(cls, f).offset for f in fields]
    assert got == mirror and got[0] == size


def test_the_python_defaults_are_the_headers(repo, tmp_path):
    n, tol = _compile_and_run(repo, tmp_path, "defaults", '    printf("%d %.17g\\n", (int)RTB200_TEMPORAL_DEFAULT_MAX_HISTORY, '
                              '(double)RTB200_TEMPORAL_DEFAULT_DEPTH_TOL);\n')
    assert (int(n), float(tol)) == (R.TEMPORAL_MAX_HISTORY, R.TEMPORAL_DEPTH_TOL)


def _params(w=4, h=3, N=4, n_motion=0, tol=0.03, reserved=(0, 0)):
    p = R.rt_temporal_params(w, h, N, n_motion, R.rt_camera(), R.rt_camera(), tol)
    p.reserved[0], p.reserved[1] = reserved
    return p


def test_bad_arguments_are_refused_before_any_device_work():
    """Every refusal that needs no device, in both forms: the checks come before a device is looked up, so they hold on a machine
    without one (host pointers stand in for device buffers, which are only checked after these)."""
    L = R.lib()
    n = 12
    buf = np.full(200 * n, 7.0, F64)    # one 8-byte aligned block the arrays below are cut from
    base = buf.ctypes.data
    col, sph, pt = base, base + 16 * n, base + 24 * n
    hcol, hlen, hsph, hpt = base + 64 * n, base + 80 * n, base + 88 * n, base + 96 * n
    mot, ocol, olen = base + 128 * n, base + 160 * n, base + 176 * n
    st = R.rt_stats()

    def both(p, cur=(col, sph, pt), prev=(hcol, hlen, hsph, hpt), motion=None, out=(ocol, olen), host=True, null_cur=False, null_out=False):
        pp = C.byref(p) if p is not None else None
        cp = None if null_cur else C.byref(R.rt_temporal_frame(*cur))
        hp = None if prev is None else C.byref(R.rt_temporal_history(*prev))
        op = None if null_out else C.byref(R.rt_temporal_out(*out))
        rd = L.rtb200_temporal_device(0, pp, cp, hp, motion, op, None)
        ed = L.rtb200_last_error()
        if not host:
            return rd, ed, None, None
        rh = L.rtb200_temporal(0, pp, cp, hp, motion, op, C.byref(st))
        return rd, ed, rh, L.rtb200_last_error()

    cases = [
        (dict(p=None), b"params is null"),
        (dict(p=_params(), null_cur=True), b"cur or one"),
        (dict(p=_params(), cur=(None, sph, pt)), b"cur or one"),
        (dict(p=_params(), cur=(col, None, pt)), b"cur or one"),
        (dict(p=_params(), cur=(col, sph, None)), b"cur or one"),
        (dict(p=_params(), null_out=True), b"out or one"),
        (dict(p=_params(), out=(None, olen)), b"out or one"),
        (dict(p=_params(), out=(ocol, None)), b"out or one"),
        (dict(p=_params(), prev=(hcol, None, hsph, hpt)), b"partial"),
        (dict(p=_params(), prev=(None, hlen, hsph, hpt)), b"partial"),
        (dict(p=_params(), prev=(hcol, hlen, hsph, None)), b"partial"),
        (dict(p=_params(reserved=(1, 0))), b"reserved"),
        (dict(p=_params(reserved=(0, 1))), b"reserved"),
        (dict(p=_params(N=0)), b"max_history"),
        (dict(p=_params(tol=float("nan"))), b"depth_tol"),
        (dict(p=_params(tol=-1e-300)), b"depth_tol"),
        (dict(p=_params(tol=float("inf"))), b"depth_tol"),
        (dict(p=_params(n_motion=1)), b"motion is null"),
        (dict(p=_params(w=1 << 16, h=1 << 15)), b"2^31"),
        (dict(p=_params(w=65535, h=65535)), b"2^31"),
        (dict(p=_params(), out=(col + 4, olen)), b"out.color overlaps cur.color"),
        (dict(p=_params(), out=(ocol, pt + 8)), b"out.length overlaps cur.point"),
        (dict(p=_params(), out=(hcol, olen)), b"out.color overlaps prev.color"),
        (dict(p=_params(), out=(ocol, hlen + 4 * n - 4)), b"out.length overlaps prev.length"),
        (dict(p=_params(), out=(hpt + 16, olen)), b"out.color overlaps prev.point"),
        (dict(p=_params(n_motion=2), motion=mot, out=(mot + 40, olen)), b"out.color overlaps motion"),
        (dict(p=_params(), out=(ocol, ocol + 44)), b"out.length overlaps out.color"),
    ]
    for kw, what in cases:
        rd, ed, rh, eh = both(**kw)
        assert rd == -1 and what in ed, (what, ed)
        assert rh == -1 and what in eh, (what, eh)
    for kw, what in [(dict(p=_params(), cur=(col + 2, sph, pt)), b"cur.color is not 4-byte aligned"),
                     (dict(p=_params(), cur=(col, sph, pt + 4)), b"cur.point is not 8-byte aligned"),
                     (dict(p=_params(), prev=(hcol, hlen + 1, hsph, hpt)), b"prev.length is not 4-byte aligned"),
                     (dict(p=_params(n_motion=1), motion=mot + 4), b"motion is not 8-byte aligned"),
                     (dict(p=_params(), out=(ocol, olen + 2)), b"out.length is not 4-byte aligned")]:
        rd, ed, _, _ = both(host=False, **kw)
        assert rd == -1 and what in ed, (what, ed)
    assert (buf == 7.0).all()
    # a motion that overlaps nothing with n_motion 0, and no previous frame, pass these checks: the device lookup is next
    for kw in (dict(p=_params(), prev=None), dict(p=_params(w=(1 << 31) - 1, h=1), prev=None)):
        rd, ed, _, _ = both(host=False, **kw)
        if rd == -1:
            assert b"device" in ed or b"overlaps" in ed, ed


def test_a_zero_pixel_image_is_a_no_op():
    L = R.lib()
    o = np.full(3, 7.0, F32)
    ln = np.full(3, 7, np.uint32)
    st = R.rt_stats()
    st.rays = 5
    cur = R.rt_temporal_frame(o.ctypes.data, ln.ctypes.data, o.ctypes.data)
    out = R.rt_temporal_out(o.ctypes.data + 4, ln.ctypes.data + 4)
    for w, h in ((0, 0), (0, 5), (5, 0)):
        p = _params(w=w, h=h)
        assert L.rtb200_temporal(-1, C.byref(p), C.byref(cur), None, None, C.byref(out), C.byref(st)) == 0
        assert st.rays == 0 and st.kernel_launches == 0
        assert L.rtb200_temporal_device(-1, C.byref(p), C.byref(cur), None, None, C.byref(out), None) == 0
    assert (o == 7.0).all() and (ln == 7).all()
    r = R.temporal(np.zeros((0, 4, 3), F32), np.zeros((0, 4), np.int32), np.zeros((0, 4, 3), F64), R.rt_camera())
    assert r["color"].shape == (0, 4, 3) and r["length"].shape == (0, 4)


def test_python_argument_checks():
    c, s, p = np.zeros((2, 3, 3), F32), np.zeros((2, 3), np.int32), np.zeros((2, 3, 3), F64)
    cam = R.rt_camera()
    prev = {"color": c, "length": np.ones((2, 3), np.uint32), "sphere": s, "point": p, "camera": cam}
    for args, kw in [((c.astype(F64), s, p, cam), {}), ((c, s.astype(np.int64), p, cam), {}), ((c, s, p.astype(F32), cam), {}),
                     ((c, s, p[:1], cam), {}), ((c[0], s, p, cam), {}), ((c, s, p, "camera"), {}),
                     ((c, s, p, cam, {k: v for k, v in prev.items() if k != "point"}), {}),
                     ((c, s, p, cam, dict(prev, length=np.ones((2, 3), np.int32))), {}),
                     ((c, s, p, cam), dict(motion=np.zeros((2, 2), F64)))]:
        with pytest.raises(ValueError):
            R.temporal(*args, **kw)
    for kw in (dict(max_history=0), dict(depth_tol=float("nan")), dict(depth_tol=-1.0)):
        with pytest.raises(R.RtError):
            R.temporal(c, s, p, cam, prev, **kw)
    for n in (-1, 1 << 32):   # would wrap in the u32 field
        with pytest.raises(ValueError):
            R.temporal(c, s, p, cam, prev, max_history=n)
    for n in (0, -1, 1 << 32):
        with pytest.raises(ValueError):
            R.TemporalDenoiser(max_history=n)


# ---- quality of the defaults, on the oracle --------------------------------------------------------------------------------

ORBIT_STEP_DEG = 1.0


def orbit_frames(sc, n, step_deg=ORBIT_STEP_DEG, seed0=1000):
    """n frames of a camera orbiting the cover scene's centre by step_deg per frame, each with its own seed."""
    a0 = math.degrees(math.atan2(3.0, 13.0))
    out = []
    for i in range(n):
        a = math.radians(a0 + step_deg * i)
        out.append(R.make_frame(sc, look_from=[13.4 * math.cos(a), 2.0, 13.4 * math.sin(a)], seed=seed0 + i))
    return out


def oracle_orbit(w, h, spp, ref_spp, n):
    """Per frame of the orbit: the oracle's linear render at spp and at ref_spp, and its AOVs at spp."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import oracle_aov as OA
    import oracle_py
    from rtb200 import scenes
    low, ref = scenes.cover_scene(w, h, spp), scenes.cover_scene(w, h, ref_spp)
    frames = orbit_frames(low, n)
    out = []
    for f in frames:
        for sc in (low, ref):
            sc.c.camera = f.camera
            sc.seed = f.seed
        out.append((oracle_py.render(low, rgb8=False)[0].reshape(h, w, 3), oracle_py.render(ref, rgb8=False)[0].reshape(h, w, 3),
                    OA.aov(low, spp, 0), f))
    return out


def sequence_errors(orbit, max_history, depth_tol, temporal=True):
    """(MSE of the last frame, flicker error) against the reference frames of spatial denoise alone (temporal=False) or of
    temporal accumulation followed by the denoise. The flicker error is the mean over k >= 1 of |(o_k - o_k-1) - (r_k - r_k-1)|^2."""
    import denoise_restatement as DR
    prev, outs = None, []
    for raw, _, aov, f in orbit:
        acc = raw
        if temporal:
            acc, length = TR.temporal(raw, aov["sphere"], aov["point"], f.camera, prev, max_history=max_history, depth_tol=depth_tol)
            prev = {"color": acc, "length": length, "sphere": aov["sphere"], "point": aov["point"], "camera": f.camera}
        outs.append(DR.denoise(acc, aov["albedo"], aov["normal"], iterations=R.DENOISE_ITERATIONS, color_weight=R.DENOISE_COLOR_WEIGHT,
                               albedo_weight=R.DENOISE_ALBEDO_WEIGHT, normal_weight=R.DENOISE_NORMAL_WEIGHT).astype(F64))
    refs = [r.astype(F64) for _, r, _, _ in orbit]
    mse = float(np.mean((outs[-1] - refs[-1]) ** 2))
    flicker = float(np.mean([np.mean(((outs[k] - outs[k - 1]) - (refs[k] - refs[k - 1])) ** 2) for k in range(1, len(outs))]))
    return mse, flicker


def test_the_defaults_lower_the_error_and_the_flicker_of_an_orbit():
    """An orbit of 8 frames of the cover scene at 64x48 and 2 spp with distinct seeds, against the oracle's 256-spp frames:
    temporal accumulation at the defaults followed by the denoise has a lower last-frame MSE and a lower flicker error than the
    denoise alone (DESIGN.md §4.16 records the numbers)."""
    orbit = oracle_orbit(64, 48, 2, 256, 8)
    spatial = sequence_errors(orbit, 0, 0.0, temporal=False)
    both = sequence_errors(orbit, R.TEMPORAL_MAX_HISTORY, R.TEMPORAL_DEPTH_TOL)
    print(f"last-frame MSE / flicker against 256 spp: spatial {spatial[0]:.6f} / {spatial[1]:.6f}, "
          f"temporal + spatial {both[0]:.6f} / {both[1]:.6f}")
    assert both[0] < spatial[0] and both[1] < spatial[1]
