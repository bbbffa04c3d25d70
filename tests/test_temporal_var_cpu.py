"""The variance of each pixel's mean through the temporal accumulation without a GPU (rtb200_temporal_var[_device], DESIGN.md
§4.21): the two numpy restatements held equal bit for bit on edge inputs, their colour and length held to the clamped
accumulation's, the no-history copy, the static-camera recursion, the exported entry points, the argument checks that run before
any device work, the CLI's refusals, and the accumulated variance calibrated against the error of an oracle sequence."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import temporal_clamp_restatement as TC
import temporal_var_restatement as TV
import rtb200 as R
from test_temporal_cpu import BIG, CAMERA_PAIRS, _params, assert_history_equal, dyadic_camera, edge_case, orbit_camera

F32, F64 = np.float32, np.float64
MISS = 0xFFFFFFFF
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(REPO, "rust-raytracer_b200", "raytracer")
VAR_SPECIALS = np.array([np.nan, np.inf, -np.inf, -1.0, -0.0, 1e-45, 1e-39, 0.0], F32)


def assert_bits_equal(got, want, what=""):
    """float32 arrays equal bit for bit, every NaN matching a NaN."""
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan, nan_w = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan, nan_w), f"{what}: NaN in {int(nan.sum())} variances here, {int(nan_w.sum())} in the reference"
    diff = (got.view(np.uint32) != want.view(np.uint32)) & ~nan
    assert not diff.any(), f"{what}: {int(diff.sum())} variances differ, first at {np.argwhere(diff)[0].tolist()}"


def assert_var_history_equal(got, want, what=""):
    assert_history_equal(got[:2], want[:2], what)
    assert_bits_equal(got[2], want[2], what)


def edge_variances(w, h, seed, special=0.2):
    """This frame's and the history's variances: non-negative values with NaN, +-inf, negative, -0, subnormal and 0 mixed in."""
    rng = np.random.default_rng(seed + 7919)
    out = []
    for _ in range(2):
        v = rng.uniform(0, 0.1, (h, w, 3)).astype(F32)
        m = rng.random(v.shape) < special
        v[m] = rng.choice(VAR_SPECIALS, int(m.sum()))
        out.append(v)
    return out


def var_case(w, h, seed, **kw):
    color, sphere, point, cam, prev, motion = edge_case(w, h, seed, **kw)
    v, hv = edge_variances(w, h, seed)
    prev["variance"] = hv
    return color, v, sphere, point, cam, prev, motion


# ---- the restatements ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("w,h", [(1, 1), (1, 6), (6, 1), (17, 9)])
@pytest.mark.parametrize("pair", list(CAMERA_PAIRS))
@pytest.mark.parametrize("clamp", [None, 0.0, 0.5, 1e30])
def test_restatements_agree_on_edge_inputs(w, h, pair, clamp):
    for seed, (N, tol, mot) in enumerate([(8, 0.03, True), (2, 0.5, False), (1, 0.03, True), (BIG, 1e300, True)]):
        color, v, sphere, point, cam, prev, motion = var_case(w, h, 100 * seed + w * h, pcam=dyadic_camera(w, h, CAMERA_PAIRS[pair]))
        for radius in ((1,) if clamp is None else (1, 2, 3)):
            kw = dict(motion=motion if mot else None, max_history=N, depth_tol=tol, clamp=clamp, clamp_radius=radius)
            a = TV.temporal(color, v, sphere, point, cam, prev, **kw)
            b = TV.temporal_scalar(color, v, sphere, point, cam, prev, **kw)
            what = f"{w}x{h}/{pair}/clamp={clamp}/r={radius}/N={N}"
            assert_var_history_equal(a, b, what)
            # steps 1-7 never read a variance: colour and length are the clamped restatement's
            assert_history_equal(a[:2], TC.temporal(color, sphere, point, cam, prev, **kw), what)


@pytest.mark.parametrize("w,h", [(1, 1), (7, 5), (16, 12)])
def test_restatements_agree_on_an_orbit_step(w, h):
    for seed, step in enumerate((0.0, 0.5, 3.0, 179.0)):
        cam, pcam = orbit_camera(w, h, 10.0 + step), orbit_camera(w, h, 10.0)
        color, v, sphere, point, _, prev, motion = var_case(w, h, seed, cam=cam, pcam=pcam, special=0.05)
        for kw in (dict(max_history=8, depth_tol=0.03), dict(max_history=2, depth_tol=1e-3, motion=motion),
                   dict(max_history=4, depth_tol=0.03, motion=motion, clamp=R.TEMPORAL_CLAMP_GAMMA, clamp_radius=2)):
            a = TV.temporal(color, v, sphere, point, cam, prev, **kw)
            assert_var_history_equal(a, TV.temporal_scalar(color, v, sphere, point, cam, prev, **kw), f"{w}x{h}/step {step}/{kw}")
            assert_history_equal(a[:2], TC.temporal(color, sphere, point, cam, prev, **dict(dict(clamp=None), **kw)))


def test_no_history_copies_the_variance_bit_for_bit():
    """No previous frame, non-finite colours, and n = 1 (N = 1): out_variance is this frame's variance as given."""
    color, v, sphere, point, cam, prev, _ = var_case(17, 9, 4, pcam=dyadic_camera(17, 9, (0.5, 0.0)))
    for fn in (TV.temporal, TV.temporal_scalar):
        _, n, ov = fn(color, v, sphere, point, cam, None, max_history=8, depth_tol=0.03)
        assert (n == 1).all() and np.array_equal(ov.view(np.uint32), v.view(np.uint32))
        _, n, ov = fn(color, v, sphere, point, cam, prev, max_history=1, depth_tol=0.03)
        assert (n == 1).all() and np.array_equal(ov.view(np.uint32), v.view(np.uint32))
        _, n, ov = fn(color, v, sphere, point, cam, prev, max_history=8, depth_tol=0.03)
        keep = n == 1
        assert keep.any() and (n >= 2).any()
        assert np.array_equal(ov[keep].view(np.uint32), v[keep].view(np.uint32))
    # the specials themselves reach the copy: NaN (with its payload), -0, negative, subnormal
    for s in VAR_SPECIALS:
        vv = np.full((1, 1, 3), s, F32)
        _, _, ov = TV.temporal(np.ones((1, 1, 3), F32), vv, np.full((1, 1), MISS, np.uint32), np.zeros((1, 1, 3)), cam, None,
                               max_history=4, depth_tol=0.0)
        assert np.array_equal(ov.view(np.uint32), vv.view(np.uint32)), s


def test_a_non_finite_tap_variance_propagates():
    """A history whose variance is NaN or infinite stays a valid tap: the colour blends as without it, the variance carries it."""
    w, h = 4, 3
    cam = dyadic_camera(w, h)
    color = np.full((h, w, 3), 0.5, F32)
    sphere, point = np.full((h, w), MISS, np.uint32), np.zeros((h, w, 3))
    hv = np.full((h, w, 3), 0.25, F32)
    hv[0, 0], hv[1, 1, 2], hv[2, 3, 0] = np.nan, np.inf, -np.inf
    prev = {"color": np.full((h, w, 3), 0.25, F32), "length": np.full((h, w), 3, np.uint32), "sphere": sphere, "point": point,
            "camera": cam, "variance": hv}
    v = np.full((h, w, 3), 0.125, F32)
    for fn in (TV.temporal, TV.temporal_scalar):
        c, n, ov = fn(color, v, sphere, point, cam, prev, max_history=8, depth_tol=0.0)
        assert (n == 4).all()
        assert np.isnan(ov[0, 0]).all() and np.isposinf(ov[1, 1, 2]) and np.isneginf(ov[2, 3, 0])
        a = F32(1) / F32(4)
        b = F32(1) - a
        assert ov[1, 2, 1] == (b * b) * F32(0.25) + (a * a) * F32(0.125)


def _static_sequence(v, N, frames, w=5, h=3, clamp=None):
    """Accumulate `frames` frames of constant variance v under a static camera (every pixel its own history, weight 1)."""
    cam = dyadic_camera(w, h)
    rng = np.random.default_rng(1)
    sphere, point = np.full((h, w), MISS, np.uint32), np.zeros((h, w, 3))
    var = np.full((h, w, 3), v, F32)
    prev, out = None, []
    for _ in range(frames):
        color = rng.uniform(0, 1, (h, w, 3)).astype(F32)
        c, n, ov = TV.temporal(color, var, sphere, point, cam, prev, max_history=N, depth_tol=0.0, clamp=clamp)
        out.append((n, ov))
        prev = {"color": c, "length": n, "sphere": sphere, "point": point, "camera": cam, "variance": ov}
    return out


@pytest.mark.parametrize("clamp", [None, 0.5])
def test_a_static_camera_gives_v_over_k_then_the_exponential_steady_state(clamp):
    """The exact recursion gives v / k after k <= N frames (exactly at k = 2 for a dyadic v, within a few ulps after), and
    a v / (2 - a) with a = 1 / N once the history is full. The clamp changes neither."""
    for v in (F32(0.25), F32(3.0), F32(0.013)):
        N = 6
        seq = _static_sequence(v, N, 80, clamp=clamp)
        for k, (n, ov) in enumerate(seq, 1):
            assert (n == min(k, N)).all()
            if k == 1:
                assert (ov == v).all()
            elif k == 2 and v in (F32(0.25), F32(3.0)):
                assert (ov == v / F32(2)).all()
            elif k <= N:
                np.testing.assert_allclose(ov, np.float64(v) / k, rtol=4 * 2.0 ** -23)
        a = 1.0 / N
        np.testing.assert_allclose(seq[-1][1], np.float64(v) * a / (2 - a), rtol=8 * 2.0 ** -23)


def test_restatement_refusals():
    color, v, sphere, point, cam, prev, _ = var_case(2, 2, 0)
    for fn in (TV.temporal, TV.temporal_scalar):
        with pytest.raises(ValueError):
            fn(color, v, sphere, point, cam, {k: x for k, x in prev.items() if k != "variance"}, max_history=2, depth_tol=0.03)
        for kw in (dict(max_history=0, depth_tol=0.0), dict(max_history=2, depth_tol=np.nan), dict(max_history=2, depth_tol=0.0, clamp=-1.0),
                   dict(max_history=2, depth_tol=0.0, clamp=1.0, clamp_radius=4)):
            with pytest.raises(ValueError):
                fn(color, v, sphere, point, cam, prev, **kw)


# ---- the ABI -----------------------------------------------------------------------------------------------------------

def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_temporal_var_device", "rtb200_temporal_var"):
        assert name in R.ABI_SYMBOLS
        assert getattr(L, name) is not None


def test_bad_arguments_are_refused_before_any_device_work():
    """Every refusal of the variance forms that needs no device, in both forms (host pointers stand in for device buffers)."""
    L = R.lib()
    n = 12
    buf = np.full(300 * n, 7.0, F64)
    base = buf.ctypes.data
    col, sph, pt = base, base + 16 * n, base + 24 * n
    hcol, hlen, hsph, hpt = base + 64 * n, base + 80 * n, base + 88 * n, base + 96 * n
    mot, ocol, olen = base + 128 * n, base + 160 * n, base + 176 * n
    var, hvar, ovar = base + 192 * n, base + 208 * n, base + 224 * n
    st = R.rt_stats()

    def both(p, clamp=None, prev=(hcol, hlen, hsph, hpt), v=var, hv=hvar, ov=ovar, motion=None, out=(ocol, olen), host=True):
        pp = C.byref(p) if p is not None else None
        cp = C.byref(clamp) if clamp is not None else None
        cur = C.byref(R.rt_temporal_frame(col, sph, pt))
        hp = None if prev is None else C.byref(R.rt_temporal_history(*prev))
        op = C.byref(R.rt_temporal_out(*out))
        rd = L.rtb200_temporal_var_device(0, pp, cp, cur, v, hp, hv, motion, op, ov, None)
        ed = L.rtb200_last_error()
        if not host:
            return rd, ed, None, None
        st.rays = 5
        rh = L.rtb200_temporal_var(0, pp, cp, cur, v, hp, hv, motion, op, ov, C.byref(st))
        assert st.rays == 0
        return rd, ed, rh, L.rtb200_last_error()

    cases = [
        (dict(p=None), b"params is null"),
        (dict(p=_params(N=0)), b"max_history"),
        (dict(p=_params(), prev=(hcol, None, hsph, hpt)), b"partial"),
        (dict(p=_params(), out=(hcol, olen)), b"out.color overlaps prev.color"),
        (dict(p=_params(), clamp=R.rt_temporal_clamp(float("nan"), 1)), b"gamma"),
        (dict(p=_params(), clamp=R.rt_temporal_clamp(1.0, 4)), b"radius"),
        (dict(p=_params(), v=None), b"variance is null"),
        (dict(p=_params(), ov=None), b"out_variance is null"),
        (dict(p=_params(), hv=None), b"prev is given without prev_variance"),
        (dict(p=_params(), prev=None), b"prev_variance is given without prev"),
        (dict(p=_params(), ov=var + 4), b"out_variance overlaps variance"),
        (dict(p=_params(), ov=hvar + 12 * n - 4), b"out_variance overlaps prev_variance"),
        (dict(p=_params(), ov=col), b"out_variance overlaps cur.color"),
        (dict(p=_params(), ov=sph), b"out_variance overlaps cur.sphere"),
        (dict(p=_params(), ov=hpt + 8), b"out_variance overlaps prev.point"),
        (dict(p=_params(), ov=hlen), b"out_variance overlaps prev.length"),
        (dict(p=_params(n_motion=2), motion=mot, ov=mot + 40), b"out_variance overlaps motion"),
        (dict(p=_params(), ov=ocol + 8), b"out_variance overlaps out.color"),
        (dict(p=_params(), ov=olen), b"out_variance overlaps out.length"),
        (dict(p=_params(), out=(var, olen)), b"out.color overlaps variance"),
        (dict(p=_params(), out=(ocol, hvar + 8)), b"out.length overlaps prev_variance"),
    ]
    for kw, what in cases:
        rd, ed, rh, eh = both(**kw)
        assert rd == -1 and what in ed, (what, ed)
        assert rh == -1 and what in eh, (what, eh)
    for kw, what in [(dict(p=_params(), v=var + 2), b"variance is not 4-byte aligned"),
                     (dict(p=_params(), hv=hvar + 1), b"prev_variance is not 4-byte aligned"),
                     (dict(p=_params(), ov=ovar + 2), b"out_variance is not 4-byte aligned"),
                     (dict(p=_params(), out=(ocol + 2, olen)), b"out.color is not 4-byte aligned")]:
        rd, ed, _, _ = both(host=False, **kw)
        assert rd == -1 and what in ed, (what, ed)
    assert (buf == 7.0).all()
    # valid arguments, clamped or not, with or without a history, pass every check: the device lookup is next
    for kw in (dict(p=_params()), dict(p=_params(), clamp=R.rt_temporal_clamp(0.5, 3)), dict(p=_params(), prev=None, hv=None)):
        rd, ed, _, _ = both(host=False, **kw)
        if rd == -1:
            assert b"device" in ed, ed


def test_a_zero_pixel_image_is_a_no_op():
    L = R.lib()
    o = np.full(6, 7.0, F32)
    ln = np.full(3, 7, np.uint32)
    st = R.rt_stats()
    cur = R.rt_temporal_frame(o.ctypes.data, ln.ctypes.data, o.ctypes.data)
    out = R.rt_temporal_out(o.ctypes.data + 4, ln.ctypes.data + 4)
    for w, h in ((0, 0), (0, 5), (5, 0)):
        p = _params(w=w, h=h)
        for cl in (None, C.byref(R.rt_temporal_clamp(1.0, 1))):
            assert L.rtb200_temporal_var(-1, C.byref(p), cl, C.byref(cur), o.ctypes.data + 8, None, None, None, C.byref(out),
                                         o.ctypes.data + 12, C.byref(st)) == 0
            assert st.kernel_launches == 0
            assert L.rtb200_temporal_var_device(-1, C.byref(p), cl, C.byref(cur), o.ctypes.data + 8, None, None, None, C.byref(out),
                                                o.ctypes.data + 12, None) == 0
    assert (o == 7.0).all() and (ln == 7).all()
    r = R.temporal(np.zeros((0, 4, 3), F32), np.zeros((0, 4), np.int32), np.zeros((0, 4, 3), F64), R.rt_camera(),
                   variance=np.zeros((0, 4, 3), F32))
    assert r["color"].shape == (0, 4, 3) and r["variance"].shape == (0, 4, 3)


def test_python_argument_checks():
    c, s, p = np.zeros((2, 3, 3), F32), np.zeros((2, 3), np.int32), np.zeros((2, 3, 3), F64)
    cam = R.rt_camera()
    prev = {"color": c, "length": np.ones((2, 3), np.uint32), "sphere": s, "point": p, "camera": cam}
    for v, pv in ((c, prev), (c.astype(F64), dict(prev, variance=c)), (c[:1], None), (c, dict(prev, variance=c[:, :2])),
                  (c, dict(prev, variance=c.astype(F64)))):
        with pytest.raises(ValueError):
            R.temporal(c, s, p, cam, pv, variance=v)
    with pytest.raises(R.RtError):
        R.temporal(c, s, p, cam, dict(prev, variance=c), variance=c, clamp=-1.0)
    # the denoiser's weights: the chosen filter's defaults where unset
    td = R.TemporalDenoiser()
    assert not td.variance and td.denoise_kw == dict(iterations=R.DENOISE_ITERATIONS, color_weight=R.DENOISE_COLOR_WEIGHT,
                                                     albedo_weight=R.DENOISE_ALBEDO_WEIGHT, normal_weight=R.DENOISE_NORMAL_WEIGHT)
    td = R.TemporalDenoiser(variance=True)
    assert td.denoise_kw == dict(iterations=R.DENOISE_VAR_ITERATIONS, color_weight=R.DENOISE_VAR_COLOR_WEIGHT,
                                 albedo_weight=R.DENOISE_VAR_ALBEDO_WEIGHT, normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT,
                                 variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR)
    td = R.TemporalDenoiser(variance=True, iterations=2, albedo_weight=0.5, variance_floor=1e-3)
    assert td.denoise_kw == dict(iterations=2, color_weight=R.DENOISE_VAR_COLOR_WEIGHT, albedo_weight=0.5,
                                 normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT, variance_floor=1e-3)
    assert R.TemporalDenoiser(color_weight=2.0).denoise_kw["color_weight"] == 2.0
    pytest.importorskip("torch")
    for td, kw in ((R.TemporalDenoiser(variance=True), {}), (R.TemporalDenoiser(), dict(variance=c))):
        with pytest.raises(ValueError):
            td.push(c, {}, cam, **kw)


# ---- the CLI ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def cli_config(tmp_path_factory):
    from rtb200 import scenes
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-C", os.path.join(REPO, "rust-raytracer_b200"), "raytracer"])
    d = tmp_path_factory.mktemp("cli")
    cfg = scenes._variant(scenes.cover_config(), 16, 12, 2, 4)
    plain = d / "scene.json"; plain.write_text(json.dumps(cfg))
    cam = {k: cfg["camera"][k] for k in ("look_from", "look_at", "vup", "vfov", "aspect")}
    frames = d / "frames.json"; frames.write_text(json.dumps([{"camera": cam, "seed": 1}, {"camera": cam, "seed": 2}]))
    lens = d / "lens.json"; lens.write_text(json.dumps([{"camera": cam, "seed": 1}, {"camera": dict(cam, aperture=0.2, focus_dist=9.0), "seed": 2}]))
    return d, plain, frames, lens


def _run_cli(cfg, out, **env):
    from rtb200 import scenes
    e = {k: v for k, v in os.environ.items() if not k.startswith("RTB200_")}
    e.update(env)
    return subprocess.run([CLI, str(cfg), str(out)], capture_output=True, text=True, cwd=scenes.SCENES_DIR, env=e, timeout=60)


@pytest.mark.parametrize("spec", ["", "x", "0", "-1", "2.5", "4294967296", "2,", "2,,1", "2,11", "2,-1", "2,1.5", "2,3,-1", "2,3,nan",
                                  "2,3,1,inf", "2,3,1,4,1e39", "2,3,1,4,1,0", "2,3,1,4,1,-1e-4", "2,3,1,4,1,1e-46", "2,3,1,4,1,nan",
                                  "2,3,1,4,1,1e-4,-1", "2,3,1,4,1,1e-4,nan", "2,3,1,4,1,1e-4,inf", "2,3,1,4,1,1e-4,0.5,1",
                                  "2,3,1,4,1,1e-4,", "2 ,3", "2,3x"])
def test_a_malformed_spec_exits_101(cli_config, spec):
    d, plain, frames, _ = cli_config
    r = _run_cli(plain, d / "o", RTB200_TEMPORAL_VAR=spec, RTB200_FRAMES=str(frames))
    assert r.returncode == 101 and "RTB200_TEMPORAL_VAR" in r.stderr, (spec, r.returncode, r.stderr)
    assert not list(d.glob("o_*.png"))


@pytest.mark.parametrize("other", ["RTB200_TEMPORAL", "RTB200_DENOISE", "RTB200_DENOISE_VAR", "RTB200_GPUS", "RTB200_ADAPTIVE", "RTB200_AOV"])
def test_the_modes_it_cannot_be_combined_with_exit_101(cli_config, other):
    d, plain, frames, _ = cli_config
    r = _run_cli(plain, d / "o", RTB200_TEMPORAL_VAR="2", RTB200_FRAMES=str(frames), **{other: "1"})
    assert r.returncode == 101 and "RTB200_TEMPORAL_VAR" in r.stderr and other in r.stderr, (other, r.stderr)
    assert not list(d.glob("o_*.png"))


def test_no_frames_and_a_lens_frame_exit_101(cli_config):
    d, plain, _, lens = cli_config
    r = _run_cli(plain, d / "o.png", RTB200_TEMPORAL_VAR="2")
    assert r.returncode == 101 and "RTB200_TEMPORAL_VAR" in r.stderr and "RTB200_FRAMES" in r.stderr
    r = _run_cli(plain, d / "o", RTB200_TEMPORAL_VAR="2", RTB200_FRAMES=str(lens))
    assert r.returncode == 101 and "RTB200_TEMPORAL_VAR" in r.stderr and "lens camera" in r.stderr, r.stderr
    assert not list(d.glob("o*.png"))


# ---- calibration on the oracle ---------------------------------------------------------------------------------------------

CALIBRATION_BAND = (0.55, 0.85)


def still_sequence(w, h, spp, ref_spp, n, seed0=1000):
    """n frames of the oracle's cover render at spp under its own camera, seeds seed0 + i: each frame's linear mean and variance
    from its per-sample radiances (in sample order, as the render sums them), its AOVs, and one ref_spp render."""
    sys.path.insert(0, os.path.join(REPO, "oracle"))
    import adaptive_restatement as AR
    import denoise_var_restatement as DV
    import oracle_aov as OA
    import oracle_py
    from rtb200 import scenes
    low, ref = scenes.cover_scene(w, h, spp), scenes.cover_scene(w, h, ref_spp)
    ref.seed = seed0 - 1
    truth = oracle_py.render(ref, rgb8=False)[0].reshape(h, w, 3)
    out = []
    for i in range(n):
        low.seed = seed0 + i
        x, _ = AR.render_samples(low, 0, spp)
        S = np.zeros((h, w, 3), F32)
        for s in range(spp):
            S = S + x[s]
        mean = (F32(1) / F32(spp)) * S
        out.append((mean, DV.render_variance(x), OA.aov(low, spp, 0)))
    return out, truth, low


def test_the_accumulated_variance_tracks_the_accumulated_error():
    """A still camera over 8 frames of the 64x48 cover render at 4 spp, N = 8: the mean accumulated variance over the mean
    squared error of the accumulated colour against a 256-spp render lies in CALIBRATION_BAND (DESIGN.md §4.21 records the
    ratio). It is below 1: each frame's estimate divides by n, not n - 1 (0.75 at 4 spp), and the 256-spp render's own noise
    adds to the error."""
    seq, truth, sc = still_sequence(64, 48, 4, 256, 8)
    cam = sc.c.camera
    prev = None
    for mean, var, aov in seq:
        c, n, v = TV.temporal(mean, var, aov["sphere"], aov["point"], cam, prev, max_history=8, depth_tol=R.TEMPORAL_DEPTH_TOL)
        prev = {"color": c, "length": n, "sphere": aov["sphere"], "point": aov["point"], "camera": cam, "variance": v}
    ok = np.isfinite(c).all(axis=2) & np.isfinite(v).all(axis=2) & np.isfinite(truth).all(axis=2)
    mse = float(np.mean((c[ok].astype(F64) - truth[ok]) ** 2))
    mv = float(np.mean(v[ok].astype(F64)))
    full = ok & (n == 8)
    single, mv8 = float(np.mean(seq[-1][1][full].astype(F64))), float(np.mean(v[full].astype(F64)))
    ratio = mv / mse
    print(f"accumulated: mean variance {mv:.6g}, MSE {mse:.6g}, ratio {ratio:.3f}; over the {int(full.sum())} pixels of length 8: "
          f"{mv8:.6g} against one frame's {single:.6g}")
    assert full.mean() > 0.5 and mv8 < single / 6, "eight accumulated frames hold about an eighth of one frame's variance"
    assert CALIBRATION_BAND[0] <= ratio <= CALIBRATION_BAND[1], ratio
