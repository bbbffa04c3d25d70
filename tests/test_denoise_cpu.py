"""Denoising with the auxiliary buffers without a GPU (rtb200_denoise[_device], DESIGN.md §4.15): the two numpy restatements of
the contract held equal bit for bit on small images with every kind of edge value, the exported entry points, the layout of
rt_denoise_params, the argument checks that run before any device work, and the quality of the chosen defaults on the oracle's
cover render."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import denoise_restatement as DR
import rtb200 as R

F32 = np.float32
SPECIAL = np.array([np.nan, np.inf, -np.inf, 1e-40, -3e-42, -0.75, 3e38, -2e38, 0.0, -0.0, 1.5e19], F32)


def edge_image(h, w, rng, special=0.25):
    """Random values in [-0.2, 1.5) with a share `special` of NaN, +-inf, subnormals, negatives, huge values whose squares
    overflow, and zeros of both signs."""
    a = rng.uniform(-0.2, 1.5, (h, w, 3)).astype(F32)
    m = rng.random((h, w, 3)) < special
    a[m] = rng.choice(SPECIAL, int(m.sum()))
    return a


def assert_bits_equal(got, want, what=""):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan, nan_w = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan, nan_w), f"{what}: NaN in {int(nan.sum())} values here, {int(nan_w.sum())} in the reference"
    diff = (got.view(np.uint32) != want.view(np.uint32)) & ~nan
    assert not diff.any(), f"{what}: {int(diff.sum())} values differ, first at {np.argwhere(diff)[0].tolist()}"


# ---- the two restatements ----------------------------------------------------------------------------------------------

GUIDE_SETS = {
    "colour_only": dict(albedo=False, normal=False, color_weight=2.0, albedo_weight=0.0, normal_weight=0.0),
    "all_guides": dict(albedo=True, normal=True, color_weight=3.0, albedo_weight=40.0, normal_weight=9.0),
    "guides_off_by_weight": dict(albedo=True, normal=True, color_weight=1.0, albedo_weight=0.0, normal_weight=0.0),
    "colour_off": dict(albedo=True, normal=False, color_weight=0.0, albedo_weight=5.0, normal_weight=0.0),
    "no_weights": dict(albedo=False, normal=True, color_weight=0.0, albedo_weight=0.0, normal_weight=0.0),
    "huge_weights": dict(albedo=True, normal=True, color_weight=1e30, albedo_weight=3e38, normal_weight=1e-45),
}


def case(h, w, seed, g, special=0.25):
    rng = np.random.default_rng(seed)
    color = edge_image(h, w, rng, special)
    albedo = edge_image(h, w, rng, special / 4) if g["albedo"] else None
    normal = edge_image(h, w, rng, special / 4) if g["normal"] else None
    kw = {k: g[k] for k in ("color_weight", "albedo_weight", "normal_weight")}
    return color, albedo, normal, kw


@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (7, 1), (3, 3)])
@pytest.mark.parametrize("guides", list(GUIDE_SETS))
def test_restatements_agree_at_ten_iterations_on_tiny_images(h, w, guides):
    color, albedo, normal, kw = case(h, w, 10 * h + w, GUIDE_SETS[guides])
    kw["color_weight"] = min(kw["color_weight"], 1e30 / 4 ** 9)
    a = DR.denoise(color, albedo, normal, iterations=10, **kw)
    b = DR.denoise_scalar(color, albedo, normal, iterations=10, **kw)
    assert_bits_equal(a, b, f"{h}x{w}/{guides}")


@pytest.mark.parametrize("h,w,iterations", [(5, 9, 1), (9, 5, 2), (6, 11, 3), (13, 7, 4)])
@pytest.mark.parametrize("guides", list(GUIDE_SETS))
def test_restatements_agree_on_odd_sizes_with_edge_values(h, w, iterations, guides):
    for seed, special in ((1, 0.25), (2, 0.0), (3, 0.6)):
        color, albedo, normal, kw = case(h, w, 1000 * seed + h * w, GUIDE_SETS[guides], special)
        a = DR.denoise(color, albedo, normal, iterations=iterations, **kw)
        b = DR.denoise_scalar(color, albedo, normal, iterations=iterations, **kw)
        assert_bits_equal(a, b, f"{h}x{w}/L={iterations}/{guides}/{special}")


def test_the_edge_values_reach_every_branch():
    """Non-finite pixels pass through, an overflowing factor gives weight 0, and subnormals survive (nothing is flushed)."""
    rng = np.random.default_rng(5)
    color = rng.uniform(0, 1, (6, 6, 3)).astype(F32)
    color[2, 2] = [np.nan, 0.5, 0.5]
    color[0, 0] = [np.inf, 1, 1]
    color[5, 5] = 3e38                # (q - p)^2 overflows: its neighbours give it, and it gives them, weight 0 with colour on
    tiny = np.full((6, 6, 3), 1e-41, F32)
    tiny[3, 3] = 0.0
    out = DR.denoise(color, iterations=2, color_weight=1.0)
    assert np.isnan(out[2, 2, 0]) and out[0, 0, 0] == np.inf
    assert out[5, 5, 0] == F32(3e38)
    assert np.isfinite(out[1, 1]).all() and np.isfinite(out[4, 4]).all()
    sub = DR.denoise(tiny, iterations=1, color_weight=0.0)
    assert (sub > 0).all() and (sub < np.finfo(F32).tiny).all()   # subnormal results
    assert_bits_equal(sub, DR.denoise_scalar(tiny, iterations=1, color_weight=0.0), "subnormal image")


def test_restatement_refusals():
    c = np.zeros((2, 2, 3), F32)
    for kw in (dict(iterations=0, color_weight=1.0), dict(iterations=11, color_weight=1.0), dict(iterations=1, color_weight=-1.0),
               dict(iterations=1, color_weight=np.nan), dict(iterations=1, color_weight=np.inf),
               dict(iterations=10, color_weight=3e38 / 4 ** 8), dict(iterations=1, color_weight=1.0, albedo_weight=1.0)):
        with pytest.raises(ValueError):
            DR.denoise(c, **kw)


# ---- the ABI -----------------------------------------------------------------------------------------------------------

def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_denoise_scratch_bytes", "rtb200_denoise_device", "rtb200_denoise"):
        assert name in R.ABI_SYMBOLS
        assert getattr(L, name) is not None
    assert L.rtb200_denoise_scratch_bytes(0, 0) == 0
    # two colour buffers and two guides of float4, each at a 256-byte boundary
    assert L.rtb200_denoise_scratch_bytes(1920, 1080) == 4 * 1920 * 1080 * 16
    assert L.rtb200_denoise_scratch_bytes(3, 1) == 4 * 256


def test_denoise_params_match_the_header(repo, tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    fields = [f for f, _ in R.rt_denoise_params._fields_]
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rtb200.h"\nint main(void) {\n'
                   '    printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(rt_denoise_params)'
                   + "".join(f", offsetof(rt_denoise_params, {f})" for f in fields) + ');\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Werror", "-I", os.path.join(repo, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    mirror = [C.sizeof(R.rt_denoise_params)] + [getattr(R.rt_denoise_params, f).offset for f in fields]
    assert got == mirror == [32, 0, 4, 8, 12, 16, 20, 24, 28]


def test_the_python_defaults_are_the_headers(repo, tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "defaults.c"
    src.write_text('#include <stdio.h>\n#include "rtb200.h"\nint main(void) {\n    printf("%d %.9g %.9g %.9g\\n", RTB200_DENOISE_DEFAULT_ITERATIONS,\n'
                   '           (double)RTB200_DENOISE_DEFAULT_COLOR_WEIGHT, (double)RTB200_DENOISE_DEFAULT_ALBEDO_WEIGHT,\n'
                   '           (double)RTB200_DENOISE_DEFAULT_NORMAL_WEIGHT);\n    return 0;\n}\n')
    exe = tmp_path / "defaults"
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Werror", "-I", os.path.join(repo, "include"), str(src), "-o", str(exe)])
    it, cw, aw, nw = subprocess.check_output([str(exe)]).decode().split()
    assert (int(it), float(cw), float(aw), float(nw)) == (R.DENOISE_ITERATIONS, R.DENOISE_COLOR_WEIGHT, R.DENOISE_ALBEDO_WEIGHT,
                                                          R.DENOISE_NORMAL_WEIGHT)


def _params(w=4, h=3, iterations=2, reserved=0, cw=1.0, aw=0.0, nw=0.0, reserved2=0.0):
    return R.rt_denoise_params(w, h, iterations, reserved, cw, aw, nw, reserved2)


def test_bad_arguments_are_refused_before_any_device_work():
    """Every refusal that needs no device, in both forms: the checks come before a device is looked up, so they hold on a machine
    without one (host pointers stand in for device buffers, which are only checked after these)."""
    L = R.lib()
    n = 12
    buf = np.full(16 * n * 3 + 64, 7.0, F32)   # one block the ranges below are cut from
    base = buf.ctypes.data
    color, albedo, normal = base, base + 12 * n, base + 24 * n
    lin, rgb, scratch = base + 36 * n, base + 48 * n, base + 64 * n     # 16-byte aligned scratch; its 4 * 256 bytes fit the block
    assert L.rtb200_denoise_scratch_bytes(4, 3) <= buf.nbytes - 64 * n
    st = R.rt_stats()

    def both(p, c=color, a=None, nm=None, lo=lin, ro=None, sc=scratch, host=True):
        pp = C.byref(p) if p is not None else None
        rd = L.rtb200_denoise_device(0, pp, c, a, nm, sc, lo, ro, None)
        ed = L.rtb200_last_error()
        if not host:
            return rd, ed, None, None
        rh = L.rtb200_denoise(0, pp, c, a, nm, lo, ro, C.byref(st))
        return rd, ed, rh, L.rtb200_last_error()

    cases = [
        (dict(p=None), b"params is null"),
        (dict(p=_params(), c=None), b"color is null"),
        (dict(p=_params(), lo=None), b"both null"),
        (dict(p=_params(reserved=1)), b"reserved"),
        (dict(p=_params(reserved2=-0.0)), b"reserved"),
        (dict(p=_params(iterations=0)), b"iterations"),
        (dict(p=_params(iterations=11)), b"iterations"),
        (dict(p=_params(cw=float("nan"))), b"color_weight"),
        (dict(p=_params(cw=-1e-30)), b"color_weight"),
        (dict(p=_params(cw=float("inf"))), b"color_weight"),
        (dict(p=_params(nw=float("-inf")), nm=normal), b"normal_weight"),
        (dict(p=_params(aw=float("nan")), a=albedo), b"albedo_weight"),
        (dict(p=_params(iterations=10, cw=3e38 / 4 ** 8)), b"4^(iterations - 1)"),
        (dict(p=_params(aw=1.0)), b"albedo is null"),
        (dict(p=_params(nw=0.5), a=albedo), b"normal is null"),
        (dict(p=_params(w=1 << 16, h=1 << 15)), b"2^31"),
        (dict(p=_params(w=65535, h=65535)), b"2^31"),
        (dict(p=_params(), lo=color + 4), b"out_linear overlaps color"),
        (dict(p=_params(), a=albedo, lo=albedo + 12 * n - 4), b"out_linear overlaps albedo"),
        (dict(p=_params(), nm=normal, ro=normal + 6, lo=None), b"out_rgb8 overlaps normal"),
        (dict(p=_params(), ro=lin + 12 * n - 1), b"out_rgb8 overlaps out_linear"),
    ]
    for kw, what in cases:
        rd, ed, rh, eh = both(**kw)
        assert rd == -1 and what in ed, (what, ed)
        assert rh == -1 and what in eh, (what, eh)
    for kw, what in [(dict(p=_params(), sc=None), b"scratch is null"),
                     (dict(p=_params(), sc=color + 16), b"scratch overlaps color"),
                     (dict(p=_params(), sc=scratch + 8), b"16-byte aligned"),
                     (dict(p=_params(), lo=lin + 2), b"4-byte aligned"),
                     (dict(p=_params(), sc=lin), b"scratch overlaps out_linear"),
                     (dict(p=_params(w=1, h=1), sc=rgb - 16, lo=lin, ro=rgb), b"scratch overlaps out_rgb8")]:
        rd, ed, _, _ = both(host=False, **kw)
        assert rd == -1 and what in ed, (what, ed)
    assert (buf == 7.0).all()
    # the largest weight that does not overflow at L = 10, and the largest image below 2^31 pixels, pass these checks: the
    # device lookup is next (no device here, or device 0 is one), never a refusal of the arguments
    for p in (_params(iterations=10, cw=float(np.finfo(F32).max) / 4 ** 9), _params(w=(1 << 31) - 1, h=1)):
        if L.rtb200_denoise(0, C.byref(p), color, None, None, lin, None, None) == -1:
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
        assert L.rtb200_denoise(-1, C.byref(p), c.ctypes.data, None, None, o.ctypes.data, None, C.byref(st)) == 0
        assert st.rays == 0 and st.kernel_launches == 0
        assert L.rtb200_denoise_device(-1, C.byref(p), c.ctypes.data, None, None, sc.ctypes.data, o.ctypes.data, None, None) == 0
    assert (o == 7.0).all()
    out = R.denoise(np.zeros((0, 4, 3), F32), rgb8=True)
    assert out["linear"].shape == (0, 4, 3) and out["rgb8"].shape == (0, 4, 3)


def test_python_argument_checks():
    c = np.zeros((2, 3, 3), F32)
    with pytest.raises(ValueError):
        R.denoise(c, linear=False)
    with pytest.raises(ValueError):
        R.denoise(c.astype(np.float64))
    with pytest.raises(ValueError):
        R.denoise(c, np.zeros((3, 2, 3), F32))
    with pytest.raises(ValueError):
        R.denoise(np.zeros((2, 3), F32))
    with pytest.raises(R.RtError):
        R.denoise(c, albedo_weight=1.0)   # a weight for an absent guide


# ---- quality of the defaults, on the oracle ----------------------------------------------------------------------------

def _mse(a, b):
    return float(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))


def test_the_defaults_lower_the_error_of_a_two_sample_render():
    """The oracle's 2-spp cover render at 64x48 and the oracle's AOV of the same samples, denoised at the defaults, are closer
    to the oracle's 256-spp render of the same view than the raw 2-spp image (DESIGN.md §4.15 records both errors)."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import oracle_aov as OA
    import oracle_py
    from rtb200 import scenes
    low = scenes.cover_scene(64, 48, 2)
    ref = scenes.cover_scene(64, 48, 256)
    raw = oracle_py.render(low, rgb8=False)[0].reshape(48, 64, 3)
    truth = oracle_py.render(ref, rgb8=False)[0].reshape(48, 64, 3)
    aov = OA.aov(low, 2, 0)
    den = DR.denoise(raw, aov["albedo"], aov["normal"], iterations=R.DENOISE_ITERATIONS, color_weight=R.DENOISE_COLOR_WEIGHT,
                     albedo_weight=R.DENOISE_ALBEDO_WEIGHT, normal_weight=R.DENOISE_NORMAL_WEIGHT)
    raw_mse, den_mse = _mse(raw, truth), _mse(den, truth)
    print(f"MSE against 256 spp: raw 2 spp {raw_mse:.6f}, denoised {den_mse:.6f}")
    assert den_mse < raw_mse
