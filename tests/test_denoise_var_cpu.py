"""The variance-guided denoise without a GPU (rtb200_denoise_var[_device], DESIGN.md §4.18): the two numpy restatements of the
contract held equal bit for bit on small images with every kind of edge value, the variance of a render's pixel means from the
oracle's samples, the exported entry points, the layout of rt_denoise_var_params and the defaults, the argument checks that run
before any device work, and the quality of the defaults on the oracle's cover render against raw and the existing denoise."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import denoise_restatement as DR
import denoise_var_restatement as V
import rtb200 as R
from test_denoise_cpu import assert_bits_equal, edge_image

F32 = np.float32
VAR_SPECIAL = np.array([np.nan, np.inf, -np.inf, 1e-40, -3e-42, -0.5, 3e38, 0.0, -0.0, 1.5e19], F32)


def edge_variance(h, w, rng, special=0.25):
    """Random variances in [0, 0.05) with a share `special` of NaN, +-inf, subnormals, negatives, huge values, and zeros of
    both signs."""
    v = (rng.random((h, w, 3)) ** 3 * 0.05).astype(F32)
    m = rng.random((h, w, 3)) < special
    v[m] = rng.choice(VAR_SPECIAL, int(m.sum()))
    return v


GUIDE_SETS = {
    "colour_only": dict(albedo=False, normal=False, color_weight=1.0, albedo_weight=0.0, normal_weight=0.0, variance_floor=1e-4),
    "all_guides": dict(albedo=True, normal=True, color_weight=0.5, albedo_weight=40.0, normal_weight=9.0, variance_floor=1e-3),
    "guides_off_by_weight": dict(albedo=True, normal=True, color_weight=2.0, albedo_weight=0.0, normal_weight=0.0, variance_floor=0.5),
    "colour_off": dict(albedo=True, normal=False, color_weight=0.0, albedo_weight=5.0, normal_weight=0.0, variance_floor=1e-4),
    "no_weights": dict(albedo=False, normal=True, color_weight=0.0, albedo_weight=0.0, normal_weight=0.0, variance_floor=1.0),
    "huge_weights": dict(albedo=True, normal=True, color_weight=3e38, albedo_weight=3e38, normal_weight=1e-45, variance_floor=1e-45),
    "huge_floor": dict(albedo=True, normal=True, color_weight=1.0, albedo_weight=4.0, normal_weight=1.0, variance_floor=3e38),
}
KW = ("color_weight", "albedo_weight", "normal_weight", "variance_floor")


def case(h, w, seed, g, special=0.25):
    rng = np.random.default_rng(seed)
    color = edge_image(h, w, rng, special)
    variance = edge_variance(h, w, rng, special)
    albedo = edge_image(h, w, rng, special / 4) if g["albedo"] else None
    normal = edge_image(h, w, rng, special / 4) if g["normal"] else None
    return color, variance, albedo, normal, {k: g[k] for k in KW}


def assert_both_equal(a, b, what):
    assert_bits_equal(a[0], b[0], what + " colour")
    assert_bits_equal(a[1], b[1], what + " variance")


# ---- the two restatements ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (7, 1), (3, 3)])
@pytest.mark.parametrize("guides", list(GUIDE_SETS))
def test_restatements_agree_at_ten_iterations_on_tiny_images(h, w, guides):
    color, var, albedo, normal, kw = case(h, w, 10 * h + w, GUIDE_SETS[guides])
    a = V.denoise_var(color, var, albedo, normal, iterations=10, **kw)
    b = V.denoise_var_scalar(color, var, albedo, normal, iterations=10, **kw)
    assert_both_equal(a, b, f"{h}x{w}/{guides}")


@pytest.mark.parametrize("h,w,iterations", [(5, 9, 1), (9, 5, 2), (6, 11, 3), (13, 7, 4), (5, 6, 5), (4, 3, 7)])
@pytest.mark.parametrize("guides", list(GUIDE_SETS))
def test_restatements_agree_on_odd_sizes_with_edge_values(h, w, iterations, guides):
    for seed, special in ((1, 0.25), (2, 0.0), (3, 0.6)):
        color, var, albedo, normal, kw = case(h, w, 1000 * seed + h * w, GUIDE_SETS[guides], special)
        a = V.denoise_var(color, var, albedo, normal, iterations=iterations, **kw)
        b = V.denoise_var_scalar(color, var, albedo, normal, iterations=iterations, **kw)
        assert_both_equal(a, b, f"{h}x{w}/L={iterations}/{guides}/{special}")


@pytest.mark.parametrize("iterations", range(1, 11))
def test_restatements_agree_with_zero_variance_everywhere(iterations):
    rng = np.random.default_rng(iterations)
    color = rng.uniform(0, 1, (6, 5, 3)).astype(F32)
    for var in (np.zeros_like(color), np.full_like(color, -0.0)):
        a = V.denoise_var(color, var, iterations=iterations, color_weight=1.0, variance_floor=1e-4)
        b = V.denoise_var_scalar(color, var, iterations=iterations, color_weight=1.0, variance_floor=1e-4)
        assert_both_equal(a, b, f"zero variance/L={iterations}")
        assert (a[1] == 0).all()


def test_the_edge_values_reach_every_branch():
    """Pixels that are not ok (non-finite colour, negative or non-finite variance) keep their colour and variance; -0 is ok; an
    overflowing colour distance gives weight 0; an infinite prefiltered variance turns the colour factor to 1; results that are
    not finite leave the pixel not ok; subnormals survive."""
    rng = np.random.default_rng(5)
    color = rng.uniform(0, 1, (8, 8, 3)).astype(F32)
    var = np.full((8, 8, 3), 0.01, F32)
    color[2, 2] = [np.nan, 0.5, 0.5]
    var[0, 0] = [-0.25, 0, 0]          # negative: not ok
    var[0, 7] = [np.inf, 0, 0]         # infinite: not ok
    var[7, 0] = [-0.0, -0.0, -0.0]     # -0: ok
    color[5, 5] = 3e38                 # (q - p)^2 overflows
    out, ov = V.denoise_var(color, var, iterations=2, color_weight=1.0, variance_floor=1e-4)
    assert np.isnan(out[2, 2, 0]) and ov[2, 2, 0] == F32(0.01)
    assert (out[0, 0] == color[0, 0]).all() and ov[0, 0, 0] == F32(-0.25)
    assert (out[0, 7] == color[0, 7]).all() and ov[0, 7, 0] == np.inf
    assert (out[7, 0] != color[7, 0]).any() and (ov[7, 0] >= 0).all()   # filtered
    assert out[5, 5, 0] == F32(3e38)   # every neighbour's weight 0: only its own tap
    assert np.isfinite(out[1, 1]).all() and np.isfinite(out[4, 4]).all()
    # huge variances: v_p overflows to inf, vbar is inf, every colour factor is 1 (d_c / inf = 0); the result is the plain
    # B-spline of the colour
    big = np.full((5, 5, 3), 3e38, F32)
    c1, v1 = V.denoise_var(color[:5, :5], big, iterations=1, color_weight=1.0, variance_floor=1e-4)
    plain = DR.denoise(color[:5, :5], iterations=1, color_weight=0.0)
    assert_bits_equal(c1, plain, "infinite vbar")
    c2, v2 = V.denoise_var(color[:5, :5], big, iterations=2, color_weight=1.0, variance_floor=1e-4)
    assert_both_equal((c2, v2), V.denoise_var_scalar(color[:5, :5], big, iterations=2, color_weight=1.0, variance_floor=1e-4), "huge")
    # subnormal colours and variances are not flushed
    tiny = np.full((6, 6, 3), 1e-41, F32)
    tiny[3, 3] = 0.0
    sc, sv = V.denoise_var(tiny, tiny, iterations=1, color_weight=0.0, variance_floor=1e-4)
    assert (sc > 0).all() and (sc < np.finfo(F32).tiny).all()
    assert_both_equal((sc, sv), V.denoise_var_scalar(tiny, tiny, iterations=1, color_weight=0.0, variance_floor=1e-4), "subnormal")


def test_restatement_refusals():
    c = np.zeros((2, 2, 3), F32)
    for kw in (dict(iterations=0), dict(iterations=11), dict(color_weight=-1.0), dict(color_weight=np.nan),
               dict(normal_weight=np.inf), dict(variance_floor=0.0), dict(variance_floor=-1e-4), dict(variance_floor=np.inf),
               dict(variance_floor=np.nan), dict(albedo_weight=1.0)):
        args = {**dict(iterations=1, color_weight=1.0, variance_floor=1e-4), **kw}
        with pytest.raises(ValueError):
            V.denoise_var(c, c, **args)


# ---- the variance of a render's pixel means ----------------------------------------------------------------------------

def test_render_variance_of_the_oracles_samples_is_the_adaptive_rules_error():
    """The variance of the oracle's per-sample radiances of the cover render equals the formula on their f32 sums, its square
    root equals the adaptive rule's err_c (DESIGN.md §4.9) wherever d_c is not NaN, and n = 0 gives 0."""
    import adaptive_restatement as AR
    from rtb200 import scenes
    sc = scenes.cover_scene(24, 16, 16)
    x, _ = AR.render_samples(sc, 0, 16)
    for n in (1, 2, 5, 16):
        var = V.render_variance(x[:n])
        S = np.zeros(x.shape[1:], F32); Q = np.zeros(x.shape[1:], F32)
        for s in range(n):
            S = S + x[s]
            Q = Q + x[s] * x[s]
        inv = F32(1) / F32(n)
        mean = inv * S
        d = inv * Q - mean * mean
        want = np.where(d < 0, F32(0), d) * inv
        assert_bits_equal(var, want, f"n={n}")
        err = np.sqrt(np.where(d > F32(0), d, F32(0)) * inv)   # adaptive_restatement.leaves' err_c
        assert np.array_equal(np.sqrt(var), err)
        assert (var >= 0).all() and (n > 1 or (var == 0).all())
    assert (V.render_variance(x[:0]) == 0).all()
    assert (V.variance_of_sums(np.ones((2, 3), F32), np.ones((2, 3), F32), np.array([0, 0], np.uint32)) == 0).all()
    nan = V.variance_of_sums(np.array([[np.inf, 0, 0]], F32), np.array([[np.inf, 0, 0]], F32), np.array([2], np.uint32))
    assert np.isnan(nan[0, 0]) and nan[0, 1] == 0   # inf - inf: a NaN d_c stays NaN


# ---- the ABI -----------------------------------------------------------------------------------------------------------

def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_denoise_var_scratch_bytes", "rtb200_denoise_var_device", "rtb200_denoise_var"):
        assert name in R.ABI_SYMBOLS
        assert getattr(L, name) is not None
    assert L.rtb200_denoise_var_scratch_bytes(0, 0) == 0
    # two colour and two variance buffers and two guides of float4, then one f32 plane, each at a 256-byte boundary
    assert L.rtb200_denoise_var_scratch_bytes(1920, 1080) == 6 * 1920 * 1080 * 16 + 1920 * 1080 * 4
    assert L.rtb200_denoise_var_scratch_bytes(3, 1) == 7 * 256


def _compile_and_run(repo, tmp_path, name, body):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / f"{name}.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rtb200.h"\nint main(void) {\n' + body + '    return 0;\n}\n')
    exe = tmp_path / name
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Werror", "-I", os.path.join(repo, "include"), str(src), "-o", str(exe)])
    return subprocess.check_output([str(exe)]).decode().split()


def test_denoise_var_params_match_the_header(repo, tmp_path):
    fields = [f for f, _ in R.rt_denoise_var_params._fields_]
    got = _compile_and_run(repo, tmp_path, "layout", '    printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(rt_denoise_var_params)'
                           + "".join(f", offsetof(rt_denoise_var_params, {f})" for f in fields) + ');\n')
    mirror = [C.sizeof(R.rt_denoise_var_params)] + [getattr(R.rt_denoise_var_params, f).offset for f in fields]
    assert [int(x) for x in got] == mirror == [32, 0, 4, 8, 12, 16, 20, 24, 28]


def test_the_python_defaults_are_the_headers(repo, tmp_path):
    got = _compile_and_run(repo, tmp_path, "defaults",
                           '    printf("%d %.9g %.9g %.9g %.9g\\n", RTB200_DENOISE_VAR_DEFAULT_ITERATIONS,\n'
                           '           (double)RTB200_DENOISE_VAR_DEFAULT_COLOR_WEIGHT, (double)RTB200_DENOISE_VAR_DEFAULT_ALBEDO_WEIGHT,\n'
                           '           (double)RTB200_DENOISE_VAR_DEFAULT_NORMAL_WEIGHT, (double)RTB200_DENOISE_VAR_DEFAULT_VARIANCE_FLOOR);\n')
    it, cw, aw, nw, eps = got
    assert (int(it), float(cw), float(aw), float(nw), F32(eps)) == (
        R.DENOISE_VAR_ITERATIONS, R.DENOISE_VAR_COLOR_WEIGHT, R.DENOISE_VAR_ALBEDO_WEIGHT, R.DENOISE_VAR_NORMAL_WEIGHT,
        F32(R.DENOISE_VAR_VARIANCE_FLOOR))


def _params(w=4, h=3, iterations=2, reserved=0, cw=1.0, aw=0.0, nw=0.0, eps=1e-4):
    return R.rt_denoise_var_params(w, h, iterations, reserved, cw, aw, nw, eps)


def test_bad_arguments_are_refused_before_any_device_work():
    """Every refusal that needs no device, in both forms: the checks come before a device is looked up, so they hold on a machine
    without one (host pointers stand in for device buffers, which are only checked after these)."""
    L = R.lib()
    n = 12
    buf = np.full(16 * n * 6 + 64 * 8, 7.0, F32)   # one block the ranges below are cut from
    base = buf.ctypes.data
    color, var, albedo, normal = base, base + 12 * n, base + 24 * n, base + 36 * n
    lin, rgb, ov, scratch = base + 48 * n, base + 60 * n, base + 64 * n, base + 80 * n   # 16-byte aligned scratch
    assert scratch + L.rtb200_denoise_var_scratch_bytes(4, 3) <= base + buf.nbytes
    st = R.rt_stats()

    def both(p, c=color, v=var, a=None, nm=None, lo=lin, ro=None, vo=None, sc=scratch, host=True):
        pp = C.byref(p) if p is not None else None
        rd = L.rtb200_denoise_var_device(0, pp, c, v, a, nm, sc, lo, ro, vo, None)
        ed = L.rtb200_last_error()
        if not host:
            return rd, ed, None, None
        rh = L.rtb200_denoise_var(0, pp, c, v, a, nm, lo, ro, vo, C.byref(st))
        return rd, ed, rh, L.rtb200_last_error()

    cases = [
        (dict(p=None), b"params is null"),
        (dict(p=_params(), c=None), b"color is null"),
        (dict(p=_params(), v=None), b"variance is null"),
        (dict(p=_params(), lo=None), b"all null"),
        (dict(p=_params(reserved=1)), b"reserved"),
        (dict(p=_params(iterations=0)), b"iterations"),
        (dict(p=_params(iterations=11)), b"iterations"),
        (dict(p=_params(cw=float("nan"))), b"color_weight"),
        (dict(p=_params(cw=-1e-30)), b"color_weight"),
        (dict(p=_params(cw=float("inf"))), b"color_weight"),
        (dict(p=_params(nw=float("-inf")), nm=normal), b"normal_weight"),
        (dict(p=_params(aw=float("nan")), a=albedo), b"albedo_weight"),
        (dict(p=_params(eps=0.0)), b"variance_floor"),
        (dict(p=_params(eps=-0.0)), b"variance_floor"),
        (dict(p=_params(eps=-1e-4)), b"variance_floor"),
        (dict(p=_params(eps=float("inf"))), b"variance_floor"),
        (dict(p=_params(eps=float("nan"))), b"variance_floor"),
        (dict(p=_params(aw=1.0)), b"albedo is null"),
        (dict(p=_params(nw=0.5), a=albedo), b"normal is null"),
        (dict(p=_params(w=1 << 16, h=1 << 15)), b"2^31"),
        (dict(p=_params(w=65535, h=65535)), b"2^31"),
        (dict(p=_params(), lo=color + 4), b"out_linear overlaps color"),
        (dict(p=_params(), lo=var + 8), b"out_linear overlaps variance"),
        (dict(p=_params(), a=albedo, lo=albedo + 12 * n - 4), b"out_linear overlaps albedo"),
        (dict(p=_params(), nm=normal, ro=normal + 6, lo=None), b"out_rgb8 overlaps normal"),
        (dict(p=_params(), ro=lin + 12 * n - 1), b"out_rgb8 overlaps out_linear"),
        (dict(p=_params(), vo=var), b"out_variance overlaps variance"),
        (dict(p=_params(), vo=lin + 4), b"out_variance overlaps out_linear"),
        (dict(p=_params(), ro=rgb, vo=rgb + 32), b"out_variance overlaps out_rgb8"),
    ]
    for kw, what in cases:
        rd, ed, rh, eh = both(**kw)
        assert rd == -1 and what in ed, (what, ed)
        assert rh == -1 and what in eh, (what, eh)
    for kw, what in [(dict(p=_params(), sc=None), b"scratch is null"),
                     (dict(p=_params(), sc=color + 16), b"scratch overlaps color"),
                     (dict(p=_params(), sc=scratch + 8), b"16-byte aligned"),
                     (dict(p=_params(), lo=lin + 2), b"4-byte aligned"),
                     (dict(p=_params(), v=var + 2), b"variance is not 4-byte aligned"),
                     (dict(p=_params(), lo=None, vo=ov + 1), b"out_variance is not 4-byte aligned"),
                     (dict(p=_params(), sc=lin), b"scratch overlaps out_linear"),
                     (dict(p=_params(), lo=None, vo=ov, sc=ov + 16), b"scratch overlaps out_variance")]:
        rd, ed, _, _ = both(host=False, **kw)
        assert rd == -1 and what in ed, (what, ed)
    assert (buf == 7.0).all()
    # the smallest positive floor, the largest weights and the largest image below 2^31 pixels pass these checks: the device
    # lookup is next (no device here, or device 0 is one), never a refusal of the arguments
    for p in (_params(iterations=10, cw=float(np.finfo(F32).max), eps=1e-45), _params(w=(1 << 31) - 1, h=1)):
        if L.rtb200_denoise_var(0, C.byref(p), color, var, None, None, lin, None, None, None) == -1:
            assert b"overlaps" in L.rtb200_last_error()   # the 2^31 - 1 pixel ranges overlap here, after the parameter checks


def test_a_zero_pixel_image_is_a_no_op():
    L = R.lib()
    c = np.zeros(3, F32)
    o = np.full(3, 7.0, F32)
    sc = np.zeros(64, F32)
    st = R.rt_stats()
    st.rays = 5
    for w, h in ((0, 0), (0, 5), (5, 0)):
        p = _params(w=w, h=h)
        assert L.rtb200_denoise_var(-1, C.byref(p), c.ctypes.data, c.ctypes.data, None, None, None, None, o.ctypes.data, C.byref(st)) == 0
        assert st.rays == 0 and st.kernel_launches == 0
        assert L.rtb200_denoise_var_device(-1, C.byref(p), c.ctypes.data, c.ctypes.data, None, None, sc.ctypes.data, o.ctypes.data,
                                           None, None, None) == 0
    assert (o == 7.0).all()
    z = np.zeros((0, 4, 3), F32)
    out = R.denoise_var(z, z, rgb8=True, out_variance=True)
    assert out["linear"].shape == out["rgb8"].shape == out["variance"].shape == (0, 4, 3)


def test_python_argument_checks():
    c = np.zeros((2, 3, 3), F32)
    with pytest.raises(ValueError):
        R.denoise_var(c, c, linear=False)
    with pytest.raises(ValueError):
        R.denoise_var(c, c.astype(np.float64))
    with pytest.raises(ValueError):
        R.denoise_var(c, np.zeros((3, 2, 3), F32))
    with pytest.raises(ValueError):
        R.denoise_var(c, None)
    with pytest.raises(ValueError):
        R.denoise_var(c, c, np.zeros((3, 2, 3), F32))
    with pytest.raises(R.RtError):
        R.denoise_var(c, c, albedo_weight=1.0)   # a weight for an absent guide
    with pytest.raises(R.RtError):
        R.denoise_var(c, c, variance_floor=0.0)


# ---- quality of the defaults, on the oracle ----------------------------------------------------------------------------

def _mse(a, b):
    return float(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))


def test_the_defaults_beat_raw_and_the_existing_denoise_from_4_spp():
    """The oracle's cover render at 64x48 from its per-sample radiances at 2 .. 32 spp, its variance and the oracle AOV of the
    same samples, against the oracle's 256-spp render: at the defaults the variance-guided denoise beats the raw image and the
    existing denoise at 4, 8 and 16 spp and comes within 10 % of raw at 32 spp (DESIGN.md §4.18 records the table)."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import adaptive_restatement as AR
    import oracle_aov as OA
    import oracle_py
    from rtb200 import scenes
    truth = oracle_py.render(scenes.cover_scene(64, 48, 256), rgb8=False)[0].reshape(48, 64, 3)
    sc = scenes.cover_scene(64, 48, 32)
    x, _ = AR.render_samples(sc, 0, 32)
    rows = {}
    for spp in (2, 4, 8, 16, 32):
        S = np.zeros(x.shape[1:], F32)
        for s in range(spp):
            S = S + x[s]
        mean = F32(1) / F32(spp) * S
        if spp == 2:   # the samples are the render's: the 2-spp mean is the oracle's 2-spp render bit for bit
            assert_bits_equal(mean, oracle_py.render(scenes.cover_scene(64, 48, 2), rgb8=False)[0].reshape(48, 64, 3), "2 spp")
        aov = OA.aov(sc, spp, 0)
        old = DR.denoise(mean, aov["albedo"], aov["normal"], iterations=R.DENOISE_ITERATIONS, color_weight=R.DENOISE_COLOR_WEIGHT,
                         albedo_weight=R.DENOISE_ALBEDO_WEIGHT, normal_weight=R.DENOISE_NORMAL_WEIGHT)
        new, _ = V.denoise_var(mean, V.render_variance(x[:spp]), aov["albedo"], aov["normal"], iterations=R.DENOISE_VAR_ITERATIONS,
                               color_weight=R.DENOISE_VAR_COLOR_WEIGHT, albedo_weight=R.DENOISE_VAR_ALBEDO_WEIGHT,
                               normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT, variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR)
        rows[spp] = (_mse(mean, truth), _mse(old, truth), _mse(new, truth))
    print("\nMSE against 256 spp, cover 64x48    raw       denoise   denoise_var")
    for spp, (raw, old, new) in rows.items():
        print(f"  {spp:3d} spp                        {raw:.6f}  {old:.6f}  {new:.6f}")
    for spp in (4, 8, 16):
        raw, old, new = rows[spp]
        assert new < raw and new < old, spp
    assert rows[32][2] < 1.1 * rows[32][0]
