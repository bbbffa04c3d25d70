"""The variance of a render's pixel means on the GPU (rtb200_render_frames_var[_device], rtb200_adaptive_resolve_var,
rtb200_render_adaptive_var, DESIGN.md §4.18), bit for bit against the formula on the oracle's per-sample radiances
(denoise_var_restatement.render_variance): every variant, lights, textures, a lens, row-band shards, a sample-buffer cap that
forces several batches, a multi-frame group and max_depth 0; the rgb8 and linear outputs unchanged against render_frames; the
adaptive variance against the adaptive restatement's S, Q and n; and the CLI's RTB200_DENOISE_VAR against the Python pipeline."""
import json
import os
import subprocess

import numpy as np
import pytest

import adaptive_restatement as A
import denoise_restatement as DR
import denoise_var_restatement as V
import oracle_lens as OL
import rtb200 as R
from rtb200 import scenes
from test_denoise_cpu import assert_bits_equal
from test_gpu_adaptive import SCENES as ADAPTIVE_SCENES, _params
from test_gpu_intersect import REPO, VARIANTS, _torch
from test_gpu_lens import lensed

pytestmark = pytest.mark.gpu
F32 = np.float32
CLI = os.path.join(REPO, "rust-raytracer_b200", "raytracer")


def want_variance(sc, frames):
    """[n, h, w, 3]: the formula on the oracle's samples of each frame (the scene's camera and lens, the frame's seed)."""
    out = []
    keep = sc.seed
    try:
        for f in frames:
            sc.seed = int(f.seed)
            spp = int(sc.c.samples_per_pixel)
            x = OL.render_samples(sc, sc.lens, 0, spp)[0] if sc.lens is not None else A.render_samples(sc, 0, spp)[0]
            out.append(V.render_variance(x))
    finally:
        sc.seed = keep
    return np.stack(out)


def check(sc, frames, opts=None, rows=None, want=None):
    """render_frames with variance=True, linear and rgb8, against render_frames and the restatement; returns the variance."""
    lin, var, st = R.render_frames(sc, frames, opts, linear=True, variance=True)
    img, var8, _ = R.render_frames(sc, frames, opts, variance=True)
    lin0, _ = R.render_frames(sc, frames, opts, linear=True)
    img0, _ = R.render_frames(sc, frames, opts)
    assert_bits_equal(lin, lin0, "linear unchanged")
    assert np.array_equal(img, img0), "rgb8 unchanged"
    assert_bits_equal(var8, var, "variance of the rgb8 call")
    if want is None:
        want = want_variance(sc, frames)
    if rows is not None:
        want = want[:, rows]
    assert_bits_equal(var, want, "variance")
    return var, st


def frames_of(sc, seeds):
    return [R.make_frame(sc, seed=s) for s in seeds]


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_every_variant(variant):
    sc = scenes.cover_scene(40, 30, 5, depth=8)
    var, _ = check(sc, frames_of(sc, [sc.seed]), R.make_options(variant=VARIANTS[variant]))
    assert (var > 0).any()


@pytest.mark.parametrize("name", ["mixed_1_light", "mixed_2_lights", "textured", "black_sky", "nonfinite_albedo"])
def test_lights_textures_and_edges(name):
    sc = ADAPTIVE_SCENES[name]()
    sc.c.samples_per_pixel = 6
    check(sc, frames_of(sc, [sc.seed]))


def test_lens_frame():
    sc = lensed(scenes.cover_scene(40, 30, 4, depth=8), 0.1, fd=10.0)
    check(sc, frames_of(sc, [sc.seed, sc.seed + 1]))


def test_sample_buffer_cap_forces_several_batches_and_a_multi_frame_group():
    sc = scenes.cover_scene(40, 30, 6, depth=8)
    frames = frames_of(sc, [11, 12, 13])
    want = want_variance(sc, frames)
    frame_bytes = 6 * 40 * 30 * 16
    for cap, batches in ((3 * frame_bytes, 1), (frame_bytes // 3, 3 * 3)):
        _, st = check(sc, frames, R.make_options(sample_buffer_bytes=cap), want=want)
        assert st["batches"] == batches, (cap, st)


def test_row_band_shards():
    sc = scenes.cover_scene(40, 31, 4, depth=8)
    frames = frames_of(sc, [sc.seed, 9])
    want = want_variance(sc, frames)
    for rank in range(3):
        check(sc, frames, R.make_options(rank=rank, world=3, band_rows=2), rows=R.shard_row_indices(31, rank, 3, 2), want=want)


def test_max_depth_0_gives_zero():
    sc = scenes.cover_scene(24, 16, 4, depth=0)
    var, _ = check(sc, frames_of(sc, [sc.seed]))
    assert (var == 0).all()


def test_resident_form_equals_the_host_form():
    torch = _torch()
    sc = ADAPTIVE_SCENES["mixed_2_lights"]()
    sc.c.samples_per_pixel = 6
    frames = frames_of(sc, [3, 4])
    lin_h, var_h, _ = R.render_frames(sc, frames, linear=True, variance=True)
    rs = R.ResidentScene(sc)
    try:
        lin = torch.empty((2, sc.c.height, sc.c.width, 3), dtype=torch.float32, device="cuda")
        var = torch.empty_like(lin)
        rs.render_frames(frames, 0, lin.data_ptr(), variance=var.data_ptr())
        torch.cuda.synchronize()
    finally:
        rs.release()
    assert_bits_equal(lin.cpu().numpy(), lin_h, "resident linear")
    assert_bits_equal(var.cpu().numpy(), var_h, "resident variance")


def test_adaptive_variance_is_the_formula_on_the_restatements_sums():
    torch = _torch()
    sc = ADAPTIVE_SCENES["mixed_2_lights"]()
    x, rays = A.render_samples(sc, 0, sc.c.samples_per_pixel)
    p = _params()
    want = A.run(x, rays, p.samples_per_round, sc.c.samples_per_pixel, p.min_samples, p.abs_tol, p.rel_tol)
    want_var = V.variance_of_sums(want["S"], want["Q"], want["counts"])
    img, lin, cnt, var, _ = R.render_adaptive(sc, p, variance=True)
    img0, lin0, cnt0, _ = R.render_adaptive(sc, p)
    assert np.array_equal(img, img0) and np.array_equal(cnt, cnt0) and np.array_equal(cnt, want["counts"])
    assert_bits_equal(lin, lin0, "adaptive linear unchanged")
    assert_bits_equal(var, want_var, "adaptive variance")
    assert len(np.unique(cnt)) >= 2
    rs = R.ResidentScene(sc)
    try:
        rs.adaptive_begin(p)
        rs.adaptive_step(1000)
        v = torch.empty((sc.c.height, sc.c.width, 3), dtype=torch.float32, device="cuda")
        ln = torch.empty_like(v)
        rs.adaptive_resolve(linear=ln, variance=v)
        torch.cuda.synchronize()
    finally:
        rs.release()
    assert_bits_equal(v.cpu().numpy(), want_var, "resident adaptive variance")
    assert_bits_equal(ln.cpu().numpy(), lin0, "resident adaptive linear")


def test_cli_denoise_var_png_equals_the_python_pipeline(tmp_path):
    from PIL import Image
    cfg = scenes._variant(scenes.cover_config(), 40, 30, 8, 8)
    p = tmp_path / "scene.json"; p.write_text(json.dumps(cfg))
    sc = R.Scene.from_config(cfg)
    env = dict(os.environ, RTB200_SEED=str(sc.seed))
    for k in ("RTB200_DENOISE", "RTB200_DENOISE_VAR"):
        env.pop(k, None)
    plain = tmp_path / "plain.png"
    r = subprocess.run([CLI, str(p), str(plain)], capture_output=True, text=True, cwd=scenes.SCENES_DIR, env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    out = tmp_path / "frame.png"
    r = subprocess.run([CLI, str(p), str(out)], capture_output=True, text=True, cwd=scenes.SCENES_DIR,
                       env=dict(env, RTB200_DENOISE_VAR="2,0.5,3,,"), timeout=300)
    assert r.returncode == 101   # an empty field is malformed
    r = subprocess.run([CLI, str(p), str(out)], capture_output=True, text=True, cwd=scenes.SCENES_DIR,
                       env=dict(env, RTB200_DENOISE_VAR="2,0.5,3"), timeout=300)
    assert r.returncode == 0, r.stderr
    assert out.read_bytes() == plain.read_bytes()
    lin, var, _ = R.render_frames(sc, frames_of(sc, [sc.seed]), linear=True, variance=True)
    rs = R.ResidentScene(sc)
    try:
        aov = rs.aov(8)
    finally:
        rs.release()
    den = R.denoise_var(lin[0], var[0], aov["albedo"], aov["normal"], iterations=2, color_weight=0.5, albedo_weight=3.0,
                        normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT, variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR, rgb8=True)
    got = np.asarray(Image.open(tmp_path / "frame_denoised.png").convert("RGB"))
    assert np.array_equal(got, den["rgb8"])
    assert np.array_equal(got, DR.quantise(den["linear"]))
