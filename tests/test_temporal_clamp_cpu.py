"""The history clamp of the temporal accumulation without a GPU (rtb200_temporal_clamped[_device], DESIGN.md §4.20): the two
numpy restatements held equal bit for bit on edge inputs, the unclamped path left as it is, every branch of the clamp reached,
the layout and defaults of include/rtb200.h, the exported entry points, the argument checks that run before any device work,
and the quality of the default clamp on orbits of the oracle's cover render."""
import ctypes as C
import functools

import numpy as np
import pytest

import temporal_clamp_restatement as TC
import temporal_restatement as TR
import rtb200 as R
from test_temporal_cpu import (CAMERA_PAIRS, _compile_and_run, _one_pixel_prev, _params, assert_history_equal, dyadic_camera,
                               edge_case, oracle_orbit, orbit_camera, sequence_errors, synth_frame)

F32, F64 = np.float32, np.float64
MISS = 0xFFFFFFFF
GAMMAS = (0.0, 0.5, 1.0, 3.0, 1e30)


# ---- the restatements ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("w,h", [(1, 1), (1, 6), (6, 1), (17, 9)])
@pytest.mark.parametrize("pair", list(CAMERA_PAIRS))
@pytest.mark.parametrize("radius", [1, 2, 3])
def test_restatements_agree_on_edge_inputs(w, h, pair, radius):
    for seed, (N, tol, mot) in enumerate([(8, 0.03, True), (2, 0.5, False), (BIG_N, 1e300, True)]):
        color, sphere, point, cam, prev, motion = edge_case(w, h, 100 * seed + w * h + radius, pcam=dyadic_camera(w, h, CAMERA_PAIRS[pair]))
        for gamma in GAMMAS:
            kw = dict(motion=motion if mot else None, max_history=N, depth_tol=tol, clamp=gamma, clamp_radius=radius)
            assert_history_equal(TC.temporal(color, sphere, point, cam, prev, **kw), TC.temporal_scalar(color, sphere, point, cam, prev, **kw),
                                 f"{w}x{h}/{pair}/r={radius}/gamma={gamma}/N={N}")


BIG_N = 0xFFFFFFFF


@pytest.mark.parametrize("w,h", [(1, 1), (7, 5), (16, 12)])
def test_restatements_agree_on_an_orbit_step(w, h):
    for seed, step in enumerate((0.0, 0.5, 3.0)):
        cam, pcam = orbit_camera(w, h, 10.0 + step), orbit_camera(w, h, 10.0)
        color, sphere, point, _, prev, motion = edge_case(w, h, seed, cam=cam, pcam=pcam, special=0.05)
        for radius in (1, 2, 3):
            kw = dict(max_history=4, depth_tol=0.03, motion=motion, clamp=R.TEMPORAL_CLAMP_GAMMA, clamp_radius=radius)
            assert_history_equal(TC.temporal(color, sphere, point, cam, prev, **kw),
                                 TC.temporal_scalar(color, sphere, point, cam, prev, **kw), f"{w}x{h}/step {step}/r={radius}")


@pytest.mark.parametrize("pair", list(CAMERA_PAIRS))
def test_no_clamp_is_the_unclamped_accumulation(pair):
    """clamp=None is tests/temporal_restatement.py's accumulation, in both forms: steps 1-6 are restated here as they are there."""
    for w, h in ((1, 1), (1, 6), (6, 1), (9, 5), (17, 9)):
        for seed, (N, tol, mot) in enumerate([(8, 0.03, True), (1, 0.03, False), (2, 0.0, True), (BIG_N, 1e300, False)]):
            color, sphere, point, cam, prev, motion = edge_case(w, h, 100 * seed + w * h, pcam=dyadic_camera(w, h, CAMERA_PAIRS[pair]))
            kw = dict(motion=motion if mot else None, max_history=N, depth_tol=tol)
            for clamped, plain in ((TC.temporal, TR.temporal), (TC.temporal_scalar, TR.temporal_scalar)):
                assert_history_equal(clamped(color, sphere, point, cam, prev, clamp=None, clamp_radius=3, **kw),
                                     plain(color, sphere, point, cam, prev, **kw), f"{w}x{h}/{pair}/N={N}")
    color, sphere, point, cam, _, _ = edge_case(5, 3, 1)
    assert_history_equal(TC.temporal(color, sphere, point, cam, None, max_history=8, depth_tol=0.03, clamp=1.0),
                         TR.temporal(color, sphere, point, cam, None, max_history=8, depth_tol=0.03))


def test_the_clamp_keeps_the_length_and_every_no_history_case():
    """The clamp changes colours only where n >= 2, and no length anywhere."""
    color, sphere, point, cam, prev, motion = edge_case(17, 9, 4, pcam=dyadic_camera(17, 9, (0.5, 0.0)))
    kw = dict(motion=motion, max_history=8, depth_tol=0.03)
    c0, n0 = TR.temporal(color, sphere, point, cam, prev, **kw)
    c1, n1 = TC.temporal(color, sphere, point, cam, prev, clamp=0.0, **kw)
    assert np.array_equal(n0, n1) and (n0 == 1).any() and (n0 >= 2).any()
    assert np.array_equal(c0[n0 == 1].view(np.uint32), c1[n1 == 1].view(np.uint32))
    assert not np.array_equal(c0[n0 >= 2], c1[n1 >= 2])


# ---- every branch ----------------------------------------------------------------------------------------------------------

def _static(w, h, color, hist, length=3):
    """A static dyadic camera over one sphere: each pixel's history is its own, with n = min(length, 7) + 1 at N = 8."""
    cam = dyadic_camera(w, h)
    _, sphere, point = synth_frame(w, h, cam, np.random.default_rng(w * h), miss=0.0)
    sphere[:] = 1
    prev = _one_pixel_prev(w, h, cam, hist, sphere, point, length)
    return sphere, point, cam, prev


def _run(color, hist, gamma, radius=1, length=3):
    h, w, _ = color.shape
    sphere, point, cam, prev = _static(w, h, color, hist, length)
    kw = dict(max_history=8, depth_tol=0.03, clamp=gamma, clamp_radius=radius)
    with np.errstate(all="ignore"):
        a = TC.temporal(color, sphere, point, cam, prev, **kw)
        assert_history_equal(a, TC.temporal_scalar(color, sphere, point, cam, prev, **kw))
    return a


def _blend(h, c, n=4):
    return F32(h) + (F32(1) / F32(n)) * (F32(c) - F32(h))


def _moments(vals):
    """mean and var of step 7 over a window's finite colours, in window order, for one channel."""
    s = q = F32(0)
    with np.errstate(all="ignore"):
        for v in vals:
            s, q = s + F32(v), q + F32(v) * F32(v)
        m = F32(len(vals))
        mean = s / m
        return mean, q / m - mean * mean


def test_clamped_low_clamped_high_and_inside():
    """A constant window has sd = 0: a history below it is raised to the mean and one above it lowered. A window of two values
    lets a history within mean +- sd through and lowers one above it."""
    color = np.full((3, 3, 3), 0.5, F32)
    hist = np.full((3, 3, 3), 0.5, F32)
    hist[0, 0] = 0.25
    hist[2, 2] = 0.75
    c, n = _run(color, hist, 3.0)
    assert (n == 4).all()
    assert np.array_equal(c, np.full((3, 3, 3), 0.5, F32))                    # both clamped to lo = hi = 0.5, then blended
    c, _ = _run(color, hist, None)                                             # unclamped for comparison
    assert c[0, 0, 0] == _blend(0.25, 0.5) and c[2, 2, 0] == _blend(0.75, 0.5)
    # inside: window {0, 1}, the histories lie within mean +- sd
    color = np.zeros((1, 2, 3), F32)
    color[0, 1] = 1.0
    hist = np.full((1, 2, 3), 0.5, F32)
    c, _ = _run(color, hist, 1.0)
    assert np.array_equal(c, np.stack([np.full(3, _blend(0.5, 0.0)), np.full(3, _blend(0.5, 1.0))])[None])
    # clamped high with sd > 0: mean 0.5, sd 0.5, gamma 0.5: hi = 0.75
    hist[:] = 2.0
    c, _ = _run(color, hist, 0.5)
    assert np.array_equal(c[0, :, 0], [_blend(0.75, 0.0), _blend(0.75, 1.0)])


def test_a_negative_var_gives_sd_zero():
    """A constant window whose f32 moments round Q / m below mean * mean: sd is 0, not NaN, and the history is clamped to the
    mean."""
    for v in np.linspace(0.1, 0.9, 4001, dtype=F32):
        mean, var = _moments([v] * 9)
        if var < 0:
            break
    else:
        pytest.fail("no constant window with var < 0")
    color = np.full((3, 3, 3), v, F32)
    hist = np.full((3, 3, 3), 0.0, F32)
    c, _ = _run(color, hist, 1.0)
    assert c[1, 1, 0] == _blend(mean, v)


def test_overflowing_sums_leave_the_history_as_it_is():
    """A NaN var (S and Q overflow: inf - inf), and an infinite var, where gamma = 0 makes lo and hi NaN (0 * inf): the
    history passes through unclamped. With gamma > 0 an infinite var makes [lo, hi] the whole line."""
    big = F32(3e38)
    hist = np.full((1, 3, 3), 0.25, F32)
    color = np.full((1, 3, 3), big, F32)                                       # S overflows: mean = inf, var = NaN
    mean, var = _moments([big] * 3)
    assert np.isinf(mean) and np.isnan(var)
    c, _ = _run(color, hist, 1.0)
    assert np.array_equal(c, _blend(F32(0.25), color))
    hist = hist[:, :2]
    color = np.array([[[1e20] * 3, [-1e20] * 3]], F32)                         # Q overflows alone: mean = 0, var = inf
    mean, var = _moments([1e20, -1e20])
    assert np.isfinite(mean) and np.isposinf(var)
    for gamma in (0.0, 2.0):                                                   # lo, hi NaN (0 * inf) / -inf, +inf
        c, _ = _run(color, hist, gamma)
        assert np.array_equal(c, _blend(F32(0.25), color)), gamma


def test_the_border_cuts_the_window_and_non_finite_neighbours_are_skipped():
    """The corner pixel's window of radius 1 holds its 4 pixels inside the image; a NaN or infinite neighbour is left out of
    every window it falls in, while it keeps its own colour with length 1."""
    rng = np.random.default_rng(9)
    color = rng.uniform(0, 1, (5, 5, 3)).astype(F32)
    hist = np.full((5, 5, 3), -1.0, F32)                                       # below every window: each history is raised to lo
    gamma = F32(0.5)

    def lo(vals):
        mean, var = _moments(vals)
        return mean - gamma * np.sqrt(F32(0) if var < 0 else var)

    c, n = _run(color, hist, gamma)
    assert c[0, 0, 1] == _blend(lo([color[0, 0, 1], color[0, 1, 1], color[1, 0, 1], color[1, 1, 1]]), color[0, 0, 1])
    assert c[4, 2, 0] == _blend(lo([color[y, x, 0] for y in (3, 4) for x in (1, 2, 3)]), color[4, 2, 0])
    bad = color.copy()
    bad[1, 1, 2] = np.nan
    bad[1, 2, 0] = np.inf
    c, n = _run(bad, hist, gamma)
    assert n[1, 1] == 1 and n[1, 2] == 1 and n[2, 2] == 4
    keep = [(y, x) for y in (1, 2, 3) for x in (1, 2, 3) if (y, x) not in ((1, 1), (1, 2))]
    for k in range(3):
        assert c[2, 2, k] == _blend(lo([bad[y, x, k] for y, x in keep]), bad[2, 2, k]), k
    # radius 2 over a 1 x 6 strip: the window is the row, cut at both ends
    strip = rng.uniform(0, 1, (1, 6, 3)).astype(F32)
    c, _ = _run(strip, np.full((1, 6, 3), -1.0, F32), gamma, radius=2)
    assert c[0, 0, 0] == _blend(lo(list(strip[0, 0:3, 0])), strip[0, 0, 0])
    assert c[0, 3, 0] == _blend(lo(list(strip[0, 1:6, 0])), strip[0, 3, 0])


def test_restatement_refusals():
    c, s, p, cam, prev, _ = edge_case(2, 2, 0)
    for kw in (dict(clamp=-1e-30), dict(clamp=np.nan), dict(clamp=np.inf), dict(clamp=1e39), dict(clamp=1.0, clamp_radius=0),
               dict(clamp=1.0, clamp_radius=4)):
        for fn in (TC.temporal, TC.temporal_scalar):
            with pytest.raises(ValueError):
                fn(c, s, p, cam, prev, max_history=2, depth_tol=0.03, **kw)


# ---- the ABI -----------------------------------------------------------------------------------------------------------

def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_temporal_clamped_device", "rtb200_temporal_clamped"):
        assert name in R.ABI_SYMBOLS
        assert getattr(L, name) is not None


def test_struct_layout_matches_the_header(repo, tmp_path):
    fields = [f for f, _ in R.rt_temporal_clamp._fields_]
    got = [int(x) for x in _compile_and_run(repo, tmp_path, "layout", '    printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(rt_temporal_clamp)'
                                            + "".join(f", offsetof(rt_temporal_clamp, {f})" for f in fields) + ');\n')]
    assert got == [C.sizeof(R.rt_temporal_clamp)] + [getattr(R.rt_temporal_clamp, f).offset for f in fields] and got[0] == 16


def test_the_python_defaults_are_the_headers(repo, tmp_path):
    g, r = _compile_and_run(repo, tmp_path, "defaults", '    printf("%.9g %d\\n", (double)RTB200_TEMPORAL_DEFAULT_CLAMP_GAMMA, '
                            '(int)RTB200_TEMPORAL_DEFAULT_CLAMP_RADIUS);\n')
    assert (F32(float(g)), int(r)) == (F32(R.TEMPORAL_CLAMP_GAMMA), R.TEMPORAL_CLAMP_RADIUS)
    assert 1 <= R.TEMPORAL_CLAMP_RADIUS <= 3 and R.TEMPORAL_CLAMP_GAMMA >= 0


def _clamp(gamma=1.0, radius=1, reserved=(0, 0)):
    c = R.rt_temporal_clamp(gamma, radius)
    c.reserved[0], c.reserved[1] = reserved
    return c


def test_bad_arguments_are_refused_before_any_device_work():
    """Every refusal of the clamped forms that needs no device: the unclamped checks (one of each kind) and the clamp's own,
    all before a device is looked up (host pointers stand in for device buffers)."""
    L = R.lib()
    n = 12
    buf = np.full(200 * n, 7.0, F64)
    base = buf.ctypes.data
    col, sph, pt = base, base + 16 * n, base + 24 * n
    hcol, hlen, hsph, hpt = base + 64 * n, base + 80 * n, base + 88 * n, base + 96 * n
    ocol, olen = base + 160 * n, base + 176 * n
    st = R.rt_stats()

    def both(p, clamp, prev=(hcol, hlen, hsph, hpt), out=(ocol, olen)):
        pp = C.byref(p) if p is not None else None
        cp = C.byref(clamp) if clamp is not None else None
        cur = C.byref(R.rt_temporal_frame(col, sph, pt))
        hp = C.byref(R.rt_temporal_history(*prev))
        op = C.byref(R.rt_temporal_out(*out))
        rd = L.rtb200_temporal_clamped_device(0, pp, cp, cur, hp, None, op, None)
        ed = L.rtb200_last_error()
        st.rays = 5
        rh = L.rtb200_temporal_clamped(0, pp, cp, cur, hp, None, op, C.byref(st))
        assert st.rays == 0
        return rd, ed, rh, L.rtb200_last_error()

    cases = [
        (dict(p=None, clamp=_clamp()), b"params is null"),
        (dict(p=_params(reserved=(0, 1)), clamp=_clamp()), b"rt_temporal_params.reserved"),
        (dict(p=_params(N=0), clamp=_clamp()), b"max_history"),
        (dict(p=_params(), clamp=_clamp(), prev=(hcol, None, hsph, hpt)), b"partial"),
        (dict(p=_params(), clamp=_clamp(), out=(hcol, olen)), b"out.color overlaps prev.color"),
        (dict(p=_params(), clamp=None), b"clamp is null"),
        (dict(p=_params(), clamp=_clamp(gamma=float("nan"))), b"gamma"),
        (dict(p=_params(), clamp=_clamp(gamma=-1e-30)), b"gamma"),
        (dict(p=_params(), clamp=_clamp(gamma=float("inf"))), b"gamma"),
        (dict(p=_params(), clamp=_clamp(gamma=1e39)), b"gamma"),                   # finite in Python, inf as a float
        (dict(p=_params(), clamp=_clamp(radius=0)), b"radius"),
        (dict(p=_params(), clamp=_clamp(radius=4)), b"radius"),
        (dict(p=_params(), clamp=_clamp(radius=0xFFFFFFFF)), b"radius"),
        (dict(p=_params(), clamp=_clamp(reserved=(1, 0))), b"rt_temporal_clamp.reserved"),
        (dict(p=_params(), clamp=_clamp(reserved=(0, 1))), b"rt_temporal_clamp.reserved"),
    ]
    for kw, what in cases:
        rd, ed, rh, eh = both(**kw)
        assert rd == -1 and what in ed, (what, ed)
        assert rh == -1 and what in eh, (what, eh)
    assert (buf == 7.0).all()
    # a valid clamp passes every check: the device lookup is next (a machine without a GPU refuses there)
    for g, r in ((0.0, 1), (1e30, 3)):
        rd = L.rtb200_temporal_clamped_device(0, C.byref(_params()), C.byref(_clamp(g, r)), C.byref(R.rt_temporal_frame(col, sph, pt)),
                                              None, None, C.byref(R.rt_temporal_out(ocol, olen)), None)
        if rd == -1:
            assert b"device" in L.rtb200_last_error(), L.rtb200_last_error()


def test_a_zero_pixel_image_is_a_no_op():
    L = R.lib()
    o = np.full(3, 7.0, F32)
    ln = np.full(3, 7, np.uint32)
    st = R.rt_stats()
    cur = R.rt_temporal_frame(o.ctypes.data, ln.ctypes.data, o.ctypes.data)
    out = R.rt_temporal_out(o.ctypes.data + 4, ln.ctypes.data + 4)
    for w, h in ((0, 0), (0, 5), (5, 0)):
        p = _params(w=w, h=h)
        assert L.rtb200_temporal_clamped(-1, C.byref(p), C.byref(_clamp()), C.byref(cur), None, None, C.byref(out), C.byref(st)) == 0
        assert st.kernel_launches == 0
        assert L.rtb200_temporal_clamped_device(-1, C.byref(p), C.byref(_clamp()), C.byref(cur), None, None, C.byref(out), None) == 0
    assert (o == 7.0).all() and (ln == 7).all()
    r = R.temporal(np.zeros((0, 4, 3), F32), np.zeros((0, 4), np.int32), np.zeros((0, 4, 3), F64), R.rt_camera(), clamp=1.0)
    assert r["color"].shape == (0, 4, 3)


def test_python_argument_checks():
    c, s, p = np.zeros((2, 3, 3), F32), np.zeros((2, 3), np.int32), np.zeros((2, 3, 3), F64)
    cam = R.rt_camera()
    prev = {"color": c, "length": np.ones((2, 3), np.uint32), "sphere": s, "point": p, "camera": cam}
    for kw in (dict(clamp=float("nan")), dict(clamp=-1.0), dict(clamp=1.0, clamp_radius=0), dict(clamp=1.0, clamp_radius=4)):
        with pytest.raises(R.RtError):
            R.temporal(c, s, p, cam, prev, **kw)
    for kw in (dict(clamp=1.0, clamp_radius=-1), dict(clamp=1.0, clamp_radius=1 << 32)):   # would wrap in the u32 field
        with pytest.raises(ValueError):
            R.temporal(c, s, p, cam, prev, **kw)
    for kw in (dict(clamp=float("nan")), dict(clamp=-1.0), dict(clamp=1e39), dict(clamp=1.0, clamp_radius=0), dict(clamp=1.0, clamp_radius=4)):
        with pytest.raises(ValueError):
            R.TemporalDenoiser(**kw)
    assert R.TemporalDenoiser().clamp is None
    td = R.TemporalDenoiser(clamp=R.TEMPORAL_CLAMP_GAMMA)
    assert td.clamp.radius == R.TEMPORAL_CLAMP_RADIUS and td.clamp.gamma == F32(R.TEMPORAL_CLAMP_GAMMA)


# ---- quality of the default clamp, on the oracle ---------------------------------------------------------------------------

def test_the_default_clamp_still_beats_the_denoise_alone_on_the_oracle_orbit(monkeypatch):
    """test_temporal_cpu's orbit (8 frames of the cover scene at 64x48 and 2 spp, one degree per frame, against 256-spp
    frames): clamped accumulation at the defaults followed by the denoise has a lower last-frame MSE and flicker error than the
    denoise alone (DESIGN.md §4.20 records the numbers)."""
    orbit = oracle_orbit(64, 48, 2, 256, 8)
    spatial = sequence_errors(orbit, 0, 0.0, temporal=False)
    # sequence_errors accumulates through temporal_restatement.temporal: here, through the clamped restatement at the defaults
    monkeypatch.setattr(TR, "temporal", functools.partial(TC.temporal, clamp=R.TEMPORAL_CLAMP_GAMMA, clamp_radius=R.TEMPORAL_CLAMP_RADIUS))
    clamped = sequence_errors(orbit, R.TEMPORAL_MAX_HISTORY, R.TEMPORAL_DEPTH_TOL)
    print(f"last-frame MSE / flicker against 256 spp: spatial {spatial[0]:.6f} / {spatial[1]:.6f}, "
          f"clamped temporal + spatial {clamped[0]:.6f} / {clamped[1]:.6f}")
    assert clamped[0] < spatial[0] and clamped[1] < spatial[1]
