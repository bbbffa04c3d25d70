"""Animations on the GPU: rtb200_render_frames / rtb200_render_frames_device against the CPU oracle and against one
single-frame render per view. Every comparison is bit-exact: linear f32, RGB8 and ray counts. The reference of frame i is the
scene with frame i's camera, seed and max_depth."""
import json
import math
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from synth import mixed_config, _v

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _orbit(sc, n, depths=None, seeds=None, radius=13.4, height=2.0):
    """n views on a circle around the origin (the cover scene's camera orbits its centre)."""
    frames = []
    for i in range(n):
        a = math.atan2(3.0, 13.0) + 2.0 * math.pi * i / n
        frames.append(R.make_frame(sc, look_from=[radius * math.cos(a), height + 0.25 * i, radius * math.sin(a)],
                                   seed=None if seeds is None else seeds[i], max_depth=None if depths is None else depths[i]))
    return frames


class _View:
    """The scene with a frame's camera, seed and max_depth (restored on exit)."""

    def __init__(self, sc, f):
        self.sc, self.f = sc, f

    def __enter__(self):
        c = self.sc.c
        self.saved = (bytes(c.camera), c.seed, c.max_depth)
        c.camera = self.f.camera; c.seed = self.f.seed; c.max_depth = self.f.max_depth
        return self.sc

    def __exit__(self, *a):
        c = self.sc.c
        c.camera = R.rt_camera.from_buffer_copy(self.saved[0]); c.seed = self.saved[1]; c.max_depth = self.saved[2]


def _frames_both(sc, frames, opts=None):
    img, st = R.render_frames(sc, frames, opts)
    lin, st2 = R.render_frames(sc, frames, opts, linear=True)
    assert st["rays"] == st2["rays"] and st["frames"] == len(frames)
    return img, lin, st


def _check_against_oracle(sc, frames, opts=None):
    img, lin, st = _frames_both(sc, frames, opts)
    rays = samples = 0
    for i, f in enumerate(frames):
        with _View(sc, f) as v:
            lin_o, img_o, st_o = O.render(v)
        assert np.array_equal(lin[i], lin_o), f"frame {i}: linear differs, max {np.abs(lin[i] - lin_o).max()}"
        assert np.array_equal(img[i], img_o), f"frame {i}: rgb8 differs"
        rays += st_o["rays"]; samples += st_o["samples"]
    assert st["rays"] == rays and st["samples"] == samples
    return img, lin, st


def _check_against_single_frames(sc, frames, img, lin, st, opts=None):
    rays = 0
    for i, f in enumerate(frames):
        with _View(sc, f) as v:
            a, sa = R.render_rgb8(v, opts)
            b, _ = R.render_linear(v, opts)
        assert np.array_equal(img[i], a) and np.array_equal(lin[i], b), f"frame {i} differs from its single-frame render"
        rays += sa["rays"]
    assert st["rays"] == rays


def test_cover_orbit_matches_the_oracle_frame_by_frame():
    sc = scenes.cover_scene(64, 48, 4)
    frames = _orbit(sc, 5, depths=[50, 50, 3, 0, 50], seeds=[0x5EED, 7, 8, 9, 2**40 + 3])
    img, lin, st = _check_against_oracle(sc, frames)
    assert not np.array_equal(img[0], img[1]) and not img[3].any()          # different views; max_depth 0 is black
    # groups: {0,1} one multi-frame launch, {2}, {3} (black, no launch), {4}
    assert st["batches"] == 4 and st["kernel_launches"] == (1 + 2) + 2 + 2 + 2


def test_frames_equal_single_frame_calls():
    sc = scenes.cover_scene(64, 48, 4)
    frames = _orbit(sc, 5, depths=[12, 12, 3, 0, 12], seeds=[1, 2, 3, 4, 5])
    img, lin, st = _frames_both(sc, frames)
    _check_against_single_frames(sc, frames, img, lin, st)


def test_variants_agree_on_a_mixed_material_sequence():
    sc = R.Scene.from_config(mixed_config(64, 48, 3, 12, seed=3))
    frames = _orbit(sc, 4, seeds=[11, 12, 13, 14])
    ref = None
    for variant in (R.RT_VARIANT_FILTERED, R.RT_VARIANT_EXACT_F64, R.RT_VARIANT_BRUTE_FORCE):
        img, lin, st = _frames_both(sc, frames, R.make_options(variant=variant))
        assert st["batches"] == 1
        if ref is None:
            ref = (img, lin, st["rays"])
            _check_against_oracle(sc, frames[:2], R.make_options(variant=variant))
        else:
            assert np.array_equal(img, ref[0]) and np.array_equal(lin, ref[1]) and st["rays"] == ref[2]


def _light_cfg(n_lights, seed, sky="gradient", depth=6):
    cfg = mixed_config(80, 60, 6, depth, seed=seed, n=30, sky=sky)
    pos = [(0.0, 6.0, 0.0), (-4.0, 3.0, 5.0), (5.0, 2.5, -3.0)]
    for k in range(n_lights):
        cfg["objects"].insert(3 + 5 * k, {"center": _v(*pos[k]), "radius": 1.0 + 0.5 * k, "material": {"Light": {}}})
    return cfg


@pytest.mark.parametrize("n_lights,seed", [(1, 31), (2, 32)])
def test_lights_with_per_frame_depth(n_lights, seed):
    """max_depth 1 and 2 take the light test's usize wrap (raytracer.rs:89-101); equal depths share a launch."""
    sc = R.Scene.from_config(_light_cfg(n_lights, seed))
    frames = _orbit(sc, 6, depths=[1, 1, 2, 2, 6, 6], seeds=[41, 42, 43, 44, 45, 46])
    img, lin, st = _check_against_oracle(sc, frames)
    assert st["batches"] == 3 and st["kernel_launches"] == 3 * (1 + 2)


def test_textures_and_sky_texture():
    sc = R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 100, 75, 4, 8), scenes.SCENES_DIR)
    frames = [R.make_frame(sc, seed=3), R.make_frame(sc, look_from=[-1.5, 0.8, 1.5], seed=4), R.make_frame(sc, look_at=[0.3, 0.0, -1.0], seed=5)]
    _check_against_oracle(sc, frames)


def test_grouping_follows_the_sample_buffer_cap():
    sc = scenes.cover_scene(64, 48, 4, depth=20)
    frames = _orbit(sc, 6, seeds=list(range(100, 106)))
    frame_bytes = 4 * 64 * 48 * 16
    out = []
    for cap, batches, launches in ((6 * frame_bytes, 1, 1 + 6),            # one launch for all six frames
                                   (2 * frame_bytes, 3, 3 * (1 + 2)),      # groups of two
                                   (frame_bytes // 2, 12, 6 * 2 * 2)):     # one frame per launch, two sample batches each
        img, lin, st = _frames_both(sc, frames, R.make_options(sample_buffer_bytes=cap))
        assert (st["batches"], st["kernel_launches"]) == (batches, launches), (cap, st)
        out.append((img, lin, st["rays"]))
    for img, lin, rays in out[1:]:
        assert np.array_equal(img, out[0][0]) and np.array_equal(lin, out[0][1]) and rays == out[0][2]
    _check_against_single_frames(sc, frames, out[0][0], out[0][1], {"rays": out[0][2]})


def test_row_band_shards_of_frames():
    sc = scenes.cover_scene(64, 50, 4)
    frames = _orbit(sc, 3, seeds=[5, 6, 7])
    full, lin_full, st = _frames_both(sc, frames)
    rays = 0
    for r in range(3):
        o = R.make_options(rank=r, world=3, band_rows=1)
        part, lpart, s = _frames_both(sc, frames, o)
        rows = R.shard_row_indices(50, r, 3, 1)
        assert part.shape == (3, len(rows), 64, 3)
        assert np.array_equal(part, full[:, rows]) and np.array_equal(lpart, lin_full[:, rows])
        rays += s["rays"]
    assert rays == st["rays"]


def test_resident_scene_frames_leave_the_handle_view_alone():
    import torch
    sc = scenes.cover_scene(96, 72, 4)
    ref, st0 = R.render_rgb8(sc)
    frames = _orbit(sc, 4, seeds=[21, 22, 23, 24])
    want, want_lin, _ = _frames_both(sc, frames)
    rs = R.ResidentScene(sc)
    n = 96 * 72 * 3
    async_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
    for _ in range(3):                                     # frames in flight when render_frames is called
        rs.render_async(async_out.data_ptr(), 0, 0)
    out = torch.zeros(4 * n, dtype=torch.uint8, device="cuda")
    lin = torch.zeros(4 * n, dtype=torch.float32, device="cuda")
    st = rs.render_frames(frames, out.data_ptr(), lin.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(async_out.cpu().numpy().reshape(72, 96, 3), ref)
    assert np.array_equal(out.cpu().numpy().reshape(4, 72, 96, 3), want) and np.array_equal(lin.cpu().numpy().reshape(4, 72, 96, 3), want_lin)
    assert st["frames"] == 4 and st["device_ms"] > 0 and st["trace_ms"] > 0
    one = torch.zeros(n, dtype=torch.uint8, device="cuda")
    s1 = rs.render(one.data_ptr(), 0)                       # the uploaded camera, seed and depth
    torch.cuda.synchronize()
    assert np.array_equal(one.cpu().numpy().reshape(72, 96, 3), ref) and s1["rays"] == st0["rays"]
    # on a stream of the caller's
    s = torch.cuda.Stream()
    out.zero_()
    torch.cuda.synchronize()
    rs.render_frames(frames, out.data_ptr(), 0, s.cuda_stream)
    assert np.array_equal(out.cpu().numpy().reshape(4, 72, 96, 3), want)
    rs.release()


def test_cli_writes_one_png_per_frame(tmp_path):
    from PIL import Image
    cfg = scenes._variant(scenes.cover_config(), 64, 48, 4, 10)
    p = tmp_path / "scene.json"; p.write_text(json.dumps(cfg))
    cam = cfg["camera"]
    spec = [{"camera": cam, "seed": 3},
            {"camera": dict(cam, look_from={"x": 10.0, "y": 3.0, "z": 8.0}), "max_depth": 4},
            {"camera": dict(cam, vfov=30.0)}]
    fp = tmp_path / "frames.json"; fp.write_text(json.dumps(spec))
    prefix = tmp_path / "anim" / "frame"
    prefix.parent.mkdir()
    env = dict(os.environ, RTB200_FRAMES=str(fp), RTB200_SEED="77")
    env.pop("RTB200_GPUS", None)
    r = subprocess.run([os.path.join(REPO, "rust-raytracer_b200", "raytracer"), str(p), str(prefix)], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    files = [f"{prefix}_{i:03}.png" for i in range(3)]
    lines = r.stdout.split("\n")
    assert lines[:6] == ["", f"Rendering {files[0]}", "", f"Rendering {files[1]}", "", f"Rendering {files[2]}"]
    assert lines[6].startswith("Frames time: ") and lines[6].endswith("ms for 3 frames")
    sc = R.Scene.from_config(cfg, scenes.SCENES_DIR)
    sc.seed = 77
    frames = [R.make_frame(sc, seed=3), R.make_frame(sc, look_from=[10.0, 3.0, 8.0], max_depth=4), R.make_frame(sc, vfov=30.0)]
    want, _ = R.render_frames(sc, frames)
    for i, f in enumerate(files):
        assert np.array_equal(np.asarray(Image.open(f)), want[i])
