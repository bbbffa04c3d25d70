"""The variance-guided denoise on the GPU (rtb200.denoise_var, rtb200_denoise_var[_device], DESIGN.md §4.18), held bit for bit to
the numpy restatement in tests/denoise_var_restatement.py: edge values on tiny and odd images at L = 1 .. 10, random images
larger than one tile grid at every iteration count, 800x600 and 1920x1080 frames, an oracle render with its variance and AOV guides; RGB8
against rtb200_probe_quantise; both forms; the stats of the host form; overlapping calls on two streams; refusals that enqueue
nothing."""
import ctypes as C

import numpy as np
import pytest

import denoise_restatement as DR
import denoise_var_restatement as V
import rtb200 as R
from test_denoise_cpu import assert_bits_equal
from test_denoise_var_cpu import GUIDE_SETS, case
from test_gpu_denoise import probe_quantise
from test_gpu_intersect import _torch

pytestmark = pytest.mark.gpu

F32 = np.float32


def both_forms(color, var, albedo, normal, what, **kw):
    """The host and device forms, linear, RGB8 and variance, against the restatement."""
    torch = _torch()
    want, want_v = V.denoise_var(color, var, albedo, normal, **kw)
    want8 = DR.quantise(want)
    h = R.denoise_var(color, var, albedo, normal, linear=True, rgb8=True, out_variance=True, **kw)
    tg = [None if a is None else torch.from_numpy(a).cuda() for a in (color, var, albedo, normal)]
    d = R.denoise_var(*tg, linear=True, rgb8=True, out_variance=True, **kw)
    torch.cuda.synchronize()
    for form, out in (("host", h), ("device", {k: v.cpu().numpy() for k, v in d.items()})):
        assert_bits_equal(out["linear"], want, f"{what}/{form} linear")
        assert_bits_equal(out["variance"], want_v, f"{what}/{form} variance")
        assert np.array_equal(out["rgb8"], want8), f"{what}/{form} rgb8"
        assert np.array_equal(out["rgb8"], probe_quantise(out["linear"])), f"{what}/{form} rgb8 vs probe_quantise"
    return h


@pytest.mark.parametrize("guides", list(GUIDE_SETS))
def test_edge_values_on_tiny_and_odd_images(guides):
    for h, w, iterations in ((1, 1, 10), (1, 7, 10), (7, 1, 10), (3, 3, 10), (5, 9, 1), (9, 5, 2), (6, 11, 3), (13, 7, 4),
                             (5, 6, 5), (4, 3, 7), (33, 65, 6), (17, 40, 8), (9, 70, 9)):
        for seed, special in ((1, 0.25), (2, 0.0), (3, 0.6)):
            color, var, albedo, normal, kw = case(h, w, 1000 * seed + h * w, GUIDE_SETS[guides], special)
            both_forms(color, var, albedo, normal, f"{h}x{w}/L={iterations}/{guides}/{special}", iterations=iterations, **kw)


def test_zero_variance_and_subnormals():
    rng = np.random.default_rng(3)
    color = rng.uniform(0, 1, (20, 37, 3)).astype(F32)
    for var in (np.zeros_like(color), np.full_like(color, -0.0)):
        for L in (1, 4, 10):
            both_forms(color, var, None, None, f"zero variance/L={L}", iterations=L, color_weight=1.0, variance_floor=1e-4)
    tiny = np.full((6, 6, 3), 1e-41, F32)
    tiny[3, 3] = 0.0
    h = both_forms(tiny, tiny, None, None, "subnormal", iterations=2, color_weight=0.0, variance_floor=1e-4)
    assert (h["linear"] > 0).all() and (h["linear"] < np.finfo(F32).tiny).all()


def _random_case(h, w, seed):
    rng = np.random.default_rng(seed)
    color = (rng.random((h, w, 3), dtype=F32) ** 3 * 2).astype(F32)
    var = (rng.random((h, w, 3), dtype=F32) ** 4 * 0.1).astype(F32)
    albedo = rng.random((h, w, 3), dtype=F32)
    normal = (rng.random((h, w, 3), dtype=F32) * 2 - 1).astype(F32)
    return color, var, albedo, normal


@pytest.mark.parametrize("iterations", range(1, 11))
def test_random_images_at_every_iteration_count(iterations):
    color, var, albedo, normal = _random_case(300, 401, iterations)
    both_forms(color, var, albedo, normal, f"300x401/L={iterations}", iterations=iterations, color_weight=1.0, albedo_weight=4.0,
               normal_weight=2.0, variance_floor=1e-4)


@pytest.mark.parametrize("iterations", [1, 3, 10])
def test_800x600(iterations):
    color, var, albedo, normal = _random_case(600, 800, 100 + iterations)
    h = both_forms(color, var, albedo, normal, f"800x600/L={iterations}", iterations=iterations,
                   color_weight=R.DENOISE_VAR_COLOR_WEIGHT, albedo_weight=R.DENOISE_VAR_ALBEDO_WEIGHT,
                   normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT, variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR)
    st = h["stats"]
    assert st["kernel_launches"] == 2 * iterations + 1
    assert st["h2d_bytes"] == 4 * 800 * 600 * 12 and st["d2h_bytes"] == 800 * 600 * 27
    assert st["trace_ms"] > 0 and st["device_ms"] >= st["trace_ms"] and st["wall_ms"] > 0


@pytest.mark.parametrize("iterations", [1, 3, 10])
def test_full_hd(iterations):
    color, var, albedo, normal = _random_case(1080, 1920, 200 + iterations)
    h = both_forms(color, var, albedo, normal, f"1920x1080/L={iterations}", iterations=iterations,
                   color_weight=R.DENOISE_VAR_COLOR_WEIGHT, albedo_weight=R.DENOISE_VAR_ALBEDO_WEIGHT,
                   normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT, variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR)
    st = h["stats"]
    assert st["kernel_launches"] == 2 * iterations + 1
    assert st["h2d_bytes"] == 4 * 1920 * 1080 * 12 and st["d2h_bytes"] == 1920 * 1080 * 27


def test_the_oracle_cover_render_with_its_variance_and_guides():
    """The oracle's 8-spp cover render at 64x48, the variance of its means and its AOV guides, at the defaults."""
    import adaptive_restatement as AR
    import oracle_aov as OA
    from rtb200 import scenes
    sc = scenes.cover_scene(64, 48, 8)
    x, _ = AR.render_samples(sc, 0, 8)
    S = np.zeros(x.shape[1:], F32)
    for s in range(8):
        S = S + x[s]
    mean = F32(1 / 8) * S
    aov = OA.aov(sc, 8, 0)
    for L in range(1, 6):
        both_forms(mean, V.render_variance(x), aov["albedo"], aov["normal"], f"cover/L={L}", iterations=L,
                   color_weight=R.DENOISE_VAR_COLOR_WEIGHT, albedo_weight=R.DENOISE_VAR_ALBEDO_WEIGHT,
                   normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT, variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR)


def test_overlapping_calls_on_two_streams_give_the_same_bytes():
    torch = _torch()
    color, var, albedo, normal = _random_case(600, 800, 7)
    kw = dict(iterations=5, color_weight=1.0, albedo_weight=4.0, normal_weight=2.0, variance_floor=1e-3)
    want, want_v = V.denoise_var(color, var, albedo, normal, **kw)
    tg = [torch.from_numpy(a).cuda() for a in (color, var, albedo, normal)]
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [R.denoise_var(*tg, out_variance=True, stream=a if k % 2 == 0 else b, **kw) for k in range(6)]
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        assert_bits_equal(o["linear"].cpu().numpy(), want, f"call {k}")
        assert_bits_equal(o["variance"].cpu().numpy(), want_v, f"call {k} variance")
    with pytest.raises(ValueError):   # the library's own stream cannot order torch's reuse of the scratch
        R.denoise_var(*tg, stream=0, **kw)


def test_refusals_enqueue_nothing():
    torch = _torch()
    L = R.lib()
    h, w = 12, 16
    n = h * w
    p = R.rt_denoise_var_params(w, h, 2, 0, 1.0, 0.0, 0.0, 1e-4)
    color = torch.rand((h, w, 3), device="cuda")
    var = torch.rand((h, w, 3), device="cuda")
    sb = int(L.rtb200_denoise_var_scratch_bytes(w, h))
    block = torch.full((sb + n * 12,), 7, dtype=torch.uint8, device="cuda")   # scratch, then an output
    scratch, out = block.data_ptr(), block.data_ptr() + sb
    host_out = np.full((h, w, 3), 7.0, F32)
    host_var = var.cpu().numpy()
    cp, vp = color.data_ptr(), var.data_ptr()
    cases = [
        ((0, C.byref(p), cp, host_var.ctypes.data, None, None, scratch, out, None, None, None), b"variance is not device"),
        ((0, C.byref(p), cp, vp, None, None, scratch, None, None, host_out.ctypes.data, None), b"out_variance is not device"),
        ((0, C.byref(p), cp, vp, None, None, host_out.ctypes.data, out, None, None, None), b"scratch is not device"),
        ((0, C.byref(p), cp, vp, None, None, scratch, None, None, vp + 8, None), b"out_variance overlaps variance"),
    ]
    for args, what in cases:
        assert L.rtb200_denoise_var_device(*args) == -1, what
        assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
    torch.cuda.synchronize()
    assert (block.cpu().numpy() == 7).all() and (host_out == 7.0).all()
    with pytest.raises(R.RtError):
        R.denoise_var(color, var, iterations=11)
    with pytest.raises(R.RtError):
        R.denoise_var(color, var, variance_floor=-1.0)
    ok = R.denoise_var(color, var, iterations=2, color_weight=1.0, out_variance=True)
    torch.cuda.synchronize()
    want, want_v = V.denoise_var(color.cpu().numpy(), host_var, iterations=2, color_weight=1.0,
                                 variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR)
    assert_bits_equal(ok["linear"].cpu().numpy(), want, "after refusals")
    assert_bits_equal(ok["variance"].cpu().numpy(), want_v, "after refusals: variance")
