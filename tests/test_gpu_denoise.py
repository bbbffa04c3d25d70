"""Denoising on the GPU (rtb200.denoise, rtb200_denoise[_device], DESIGN.md §4.15), held bit for bit to the numpy restatement in
tests/denoise_restatement.py: edge values, random images up to 1920x1080 at every iteration count, the render -> AOV -> denoise
pipeline in every variant; RGB8 against rtb200_probe_quantise; overlapping calls on two streams; refusals that enqueue
nothing; the CLI's _denoised.png; and the error of a denoised 4-spp C2 frame against a 256-spp one."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import denoise_restatement as DR
import rtb200 as R
from rtb200 import scenes
from test_denoise_cpu import GUIDE_SETS, assert_bits_equal, case
from test_gpu_intersect import REPO, VARIANTS, _torch

pytestmark = pytest.mark.gpu

CLI = os.path.join(REPO, "rust-raytracer_b200", "raytracer")
F32 = np.float32


def probe_quantise(linear):
    x = np.ascontiguousarray(linear, F32).reshape(-1)
    out = np.empty(x.size, np.uint8)
    R._check(R.lib().rtb200_probe_quantise(x.ctypes.data, x.size, out.ctypes.data))
    return out.reshape(np.shape(linear))


def both_forms(color, albedo, normal, what, **kw):
    """The host and device forms, linear and RGB8, against the restatement."""
    torch = _torch()
    want = DR.denoise(color, albedo, normal, **kw)
    want8 = DR.quantise(want)
    h = R.denoise(color, albedo, normal, linear=True, rgb8=True, **kw)
    tg = [None if a is None else torch.from_numpy(a).cuda() for a in (color, albedo, normal)]
    d = R.denoise(*tg, linear=True, rgb8=True, **kw)
    torch.cuda.synchronize()
    for form, out in (("host", h), ("device", {k: v.cpu().numpy() for k, v in d.items()})):
        assert_bits_equal(out["linear"], want, f"{what}/{form} linear")
        assert np.array_equal(out["rgb8"], want8), f"{what}/{form} rgb8"
        assert np.array_equal(out["rgb8"], probe_quantise(out["linear"])), f"{what}/{form} rgb8 vs probe_quantise"
    return h


# ---- the restatement ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("guides", list(GUIDE_SETS))
def test_edge_values_on_tiny_and_odd_images(guides):
    for h, w, iterations in ((1, 1, 10), (1, 7, 10), (7, 1, 10), (3, 3, 10), (5, 9, 1), (9, 5, 2), (6, 11, 3), (13, 7, 4), (33, 65, 6)):
        for seed, special in ((1, 0.25), (2, 0.0), (3, 0.6)):
            color, albedo, normal, kw = case(h, w, 1000 * seed + h * w, GUIDE_SETS[guides], special)
            kw["color_weight"] = min(kw["color_weight"], 1e30 / 4 ** (iterations - 1))
            both_forms(color, albedo, normal, f"{h}x{w}/L={iterations}/{guides}/{special}", iterations=iterations, **kw)


def test_subnormals_are_not_flushed():
    tiny = np.full((6, 6, 3), 1e-41, F32)
    tiny[3, 3] = 0.0
    h = both_forms(tiny, None, None, "subnormal", iterations=2, color_weight=0.0)
    assert (h["linear"] > 0).all() and (h["linear"] < np.finfo(F32).tiny).all()


def _random_case(h, w, seed):
    rng = np.random.default_rng(seed)
    color = (rng.random((h, w, 3), dtype=F32) ** 3 * 2).astype(F32)
    albedo = rng.random((h, w, 3), dtype=F32)
    normal = (rng.random((h, w, 3), dtype=F32) * 2 - 1).astype(F32)
    return color, albedo, normal


@pytest.mark.parametrize("iterations", range(1, 11))
def test_random_images_at_every_iteration_count(iterations):
    color, albedo, normal = _random_case(300, 401, iterations)
    both_forms(color, albedo, normal, f"300x401/L={iterations}", iterations=iterations, color_weight=8.0, albedo_weight=4.0,
               normal_weight=2.0)


@pytest.mark.parametrize("iterations", [1, 10])
def test_full_hd(iterations):
    color, albedo, normal = _random_case(1080, 1920, 100 + iterations)
    h = both_forms(color, albedo, normal, f"1920x1080/L={iterations}", iterations=iterations, color_weight=16.0, albedo_weight=4.0,
                   normal_weight=1.0)
    st = h["stats"]
    assert st["kernel_launches"] == iterations + 1
    assert st["h2d_bytes"] == 3 * 1920 * 1080 * 12 and st["d2h_bytes"] == 1920 * 1080 * 15
    assert st["trace_ms"] > 0 and st["device_ms"] >= st["trace_ms"] and st["wall_ms"] > 0


# ---- the pipeline ------------------------------------------------------------------------------------------------------

def _pipeline(sc, variant, iterations=R.DENOISE_ITERATIONS):
    """render_device (linear) -> aov(samples = spp) -> denoise, all on the device."""
    torch = _torch()
    w, h = int(sc.c.width), int(sc.c.height)
    rs = R.ResidentScene(sc, R.make_options(variant=variant))
    try:
        lin = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        rs.render(0, lin.data_ptr(), stream=torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY)
        aov = rs.aov(int(sc.c.samples_per_pixel), on_device=True, outputs=("albedo", "normal"))
        out = R.denoise(lin, aov["albedo"], aov["normal"], iterations=iterations, rgb8=True)
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in out.items()}, lin.cpu().numpy(), {k: v.cpu().numpy() for k, v in aov.items()}
    finally:
        rs.release()


def test_c2_pipeline_is_the_same_in_every_variant():
    sc = scenes.scene("C2")
    sc.c.samples_per_pixel = 4
    ref = None
    for name, v in VARIANTS.items():
        out, lin, aov = _pipeline(sc, v)
        if ref is None:
            want = DR.denoise(lin, aov["albedo"], aov["normal"], iterations=R.DENOISE_ITERATIONS, color_weight=R.DENOISE_COLOR_WEIGHT,
                              albedo_weight=R.DENOISE_ALBEDO_WEIGHT, normal_weight=R.DENOISE_NORMAL_WEIGHT)
            assert_bits_equal(out["linear"], want, f"C2/{name} vs the restatement")
            assert np.array_equal(out["rgb8"], DR.quantise(want))
            ref = (out, lin, aov)
            continue
        assert_bits_equal(lin, ref[1], f"C2/{name} render")
        for k in ("albedo", "normal"):
            assert_bits_equal(aov[k], ref[2][k], f"C2/{name} {k}")
        assert_bits_equal(out["linear"], ref[0]["linear"], f"C2/{name} denoised")
        assert np.array_equal(out["rgb8"], ref[0]["rgb8"]), name


def _mse(a, b):
    return float(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))


def test_denoised_c2_at_4_spp_is_closer_to_256_spp_than_the_raw_frame():
    torch = _torch()
    sc = scenes.scene("C2")
    sc.c.samples_per_pixel = 4
    out, lin, _ = _pipeline(sc, R.RT_VARIANT_AUTO)
    sc.c.samples_per_pixel = 256
    ref = R.ResidentScene(sc)
    try:
        truth = torch.empty((600, 800, 3), dtype=torch.float32, device="cuda")
        ref.render(0, truth.data_ptr(), stream=torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY)
        torch.cuda.synchronize()
        truth = truth.cpu().numpy()
    finally:
        ref.release()
    raw, den = _mse(lin, truth), _mse(out["linear"], truth)
    print(f"C2 MSE against 256 spp: raw 4 spp {raw:.6f}, denoised 4 spp {den:.6f}")
    assert den < raw


# ---- streams and refusals ----------------------------------------------------------------------------------------------

def test_overlapping_calls_on_two_streams_give_the_same_bytes():
    torch = _torch()
    color, albedo, normal = _random_case(600, 800, 7)
    want = DR.denoise(color, albedo, normal, iterations=5, color_weight=8.0, albedo_weight=4.0, normal_weight=2.0)
    tg = [torch.from_numpy(a).cuda() for a in (color, albedo, normal)]
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    for k in range(6):
        s = a if k % 2 == 0 else b
        outs.append(R.denoise(*tg, iterations=5, color_weight=8.0, albedo_weight=4.0, normal_weight=2.0, rgb8=True, stream=s))
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        assert_bits_equal(o["linear"].cpu().numpy(), want, f"call {k}")
        assert np.array_equal(o["rgb8"].cpu().numpy(), outs[0]["rgb8"].cpu().numpy())
    o = R.denoise(*tg, iterations=5, color_weight=8.0, albedo_weight=4.0, normal_weight=2.0, stream=R.CUDA_STREAM_LEGACY)
    torch.cuda.synchronize()
    assert_bits_equal(o["linear"].cpu().numpy(), want, "cudaStreamLegacy")
    with pytest.raises(ValueError):   # the library's own stream cannot order torch's reuse of the scratch
        R.denoise(*tg, iterations=5, color_weight=8.0, stream=0)


@pytest.mark.parametrize("form", ["torch_stream", "raw_handle"])
def test_the_scratch_is_not_reused_before_the_call_has_run(form):
    """The device form returns before its kernels run and drops its scratch. Allocations on torch's current stream right after
    the call, of the scratch's size and written at once, must not land on the scratch while a busy side stream still has the
    denoise queued."""
    torch = _torch()
    color, albedo, normal = _random_case(600, 800, 11)
    want = DR.denoise(color, albedo, normal, iterations=4, color_weight=8.0, albedo_weight=4.0, normal_weight=2.0)
    tg = [torch.from_numpy(a).cuda() for a in (color, albedo, normal)]
    sb = int(R.lib().rtb200_denoise_scratch_bytes(800, 600))
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        big = torch.randn(4096, 4096, device="cuda")
        for _ in range(8):
            big = big @ big / 64.0   # keeps the side stream busy so that the denoise runs late
    o = R.denoise(*tg, iterations=4, color_weight=8.0, albedo_weight=4.0, normal_weight=2.0,
                  stream=side if form == "torch_stream" else side.cuda_stream)
    junk = [torch.full((sb,), 255, dtype=torch.uint8, device="cuda") for _ in range(4)]
    torch.cuda.synchronize()
    del junk, big
    assert_bits_equal(o["linear"].cpu().numpy(), want, form)


def test_refusals_enqueue_nothing():
    torch = _torch()
    L = R.lib()
    h, w = 12, 16
    n = h * w
    p = R.rt_denoise_params(w, h, 2, 0, 1.0, 0.0, 0.0, 0.0)
    color = torch.rand((h, w, 3), device="cuda")
    sb = int(L.rtb200_denoise_scratch_bytes(w, h))
    block = torch.full((sb + n * 12,), 7, dtype=torch.uint8, device="cuda")   # scratch, then an output
    scratch, out = block.data_ptr(), block.data_ptr() + sb
    host_out = np.full((h, w, 3), 7.0, F32)
    host_color = color.cpu().numpy()
    cases = [
        ((0, C.byref(p), host_color.ctypes.data, None, None, scratch, out, None, None), b"color is not device"),
        ((0, C.byref(p), color.data_ptr(), None, None, scratch, host_out.ctypes.data, None, None), b"out_linear is not device"),
        ((0, C.byref(p), color.data_ptr(), None, None, host_out.ctypes.data, out, None, None), b"scratch is not device"),
        ((0, C.byref(p), color.data_ptr(), None, None, scratch, color.data_ptr() + 8, None, None), b"overlaps color"),
        ((0, C.byref(p), color.data_ptr(), None, None, scratch + 256, out, None, None), b"scratch overlaps out_linear"),
    ]
    if torch.cuda.device_count() > 1:
        other = torch.empty(n * 3, dtype=torch.float32, device="cuda:1")
        cases.append(((0, C.byref(p), color.data_ptr(), None, None, scratch, other.data_ptr(), None, None), b"out_linear is not device"))
    for args, what in cases:
        assert L.rtb200_denoise_device(*args) == -1, what
        assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
    torch.cuda.synchronize()
    assert (block.cpu().numpy() == 7).all() and (host_out == 7.0).all()
    with pytest.raises(R.RtError):
        R.denoise(color, iterations=11)
    with pytest.raises(R.RtError):
        R.denoise(color, normal_weight=1.0)
    # after the refusals the same call works
    ok = R.denoise(color, iterations=2, color_weight=1.0)
    torch.cuda.synchronize()
    assert_bits_equal(ok["linear"].cpu().numpy(), DR.denoise(host_color, iterations=2, color_weight=1.0), "after refusals")


# ---- the CLI -----------------------------------------------------------------------------------------------------------

def test_cli_writes_the_denoised_png_and_leaves_out_png_unchanged(tmp_path):
    from PIL import Image
    cfg = scenes._variant(scenes.cover_config(), 40, 30, 4, 8)
    p = tmp_path / "scene.json"; p.write_text(json.dumps(cfg))
    sc = R.Scene.from_config(cfg)
    env = dict(os.environ, RTB200_SEED=str(sc.seed))
    env.pop("RTB200_DENOISE", None)
    plain = tmp_path / "plain.png"
    r = subprocess.run([CLI, str(p), str(plain)], capture_output=True, text=True, cwd=scenes.SCENES_DIR, env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    out = tmp_path / "frame.png"
    r = subprocess.run([CLI, str(p), str(out)], capture_output=True, text=True, cwd=scenes.SCENES_DIR,
                       env=dict(env, RTB200_DENOISE="4,8,2"), timeout=300)
    assert r.returncode == 0, r.stderr
    assert out.read_bytes() == plain.read_bytes()
    assert not (tmp_path / "plain_denoised.png").exists()
    rs = R.ResidentScene(sc)
    try:
        lin, _ = R.render_linear(sc)
        aov = rs.aov(4)
    finally:
        rs.release()
    lin = lin.reshape(30, 40, 3)
    want = DR.denoise(lin, aov["albedo"], aov["normal"], iterations=4, color_weight=8.0, albedo_weight=2.0,
                      normal_weight=R.DENOISE_NORMAL_WEIGHT)
    got = np.asarray(Image.open(tmp_path / "frame_denoised.png").convert("RGB"))
    assert np.array_equal(got, DR.quantise(want))
    for other in ("RTB200_GPUS", "RTB200_FRAMES", "RTB200_ADAPTIVE"):
        bad = subprocess.run([CLI, str(p), str(tmp_path / "x.png")], capture_output=True, text=True,
                             env=dict(env, RTB200_DENOISE="2", **{other: "1"}), timeout=60)
        assert bad.returncode == 101 and "RTB200_DENOISE" in bad.stderr, other
    bad = subprocess.run([CLI, str(p), str(tmp_path / "y.png")], capture_output=True, text=True, env=dict(env, RTB200_DENOISE="11"), timeout=60)
    assert bad.returncode == 101 and "iterations" in bad.stderr
