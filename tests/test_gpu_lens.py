"""The thin-lens camera on the GPU (DESIGN.md §4.17), bit for bit against the oracle's lens (tests/oracle_lens.cpp) in linear
f32, RGB8 and rays: every variant, shard and staged handles, the device's lens routine, pinhole invariance, trace_rays of the
lens rays, lens frames, adaptive rounds, auxiliary buffers and a lens handle after updates, rebuilds and edits."""
import numpy as np
import pytest

import oracle_lens as OL
import rtb200 as R
from rtb200 import scenes
from test_aov_cpu import mixed_lit_scene, textured_sky_scene
from test_gpu_intersect import BRUTE, EXACT, FILTERED, _torch

pytestmark = pytest.mark.gpu
VARIANTS = [FILTERED, EXACT, BRUTE]


def bits(a):
    """The bytes of `a` with every NaN made the same NaN: bit for bit, except that NaN payloads are free (scenes with
    non-finite albedos give NaN radiance, whose payload the GPU and the oracle need not share)."""
    a = np.array(a, copy=True)
    if a.dtype.kind == "f":
        a[np.isnan(a)] = np.nan
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def lensed(sc, aperture=0.1, fd_scale=None, fd=None):
    p = sc.camera_params
    if fd is None:
        fd = (fd_scale or 1.0) * R.focal_length(p["look_from"], p["look_at"])
    sc.set_camera(aperture=aperture, focus_dist=fd)
    return sc


def scene_set():
    return {"cover": lensed(scenes.cover_scene(40, 30, 3, depth=8), 0.1, fd=10.0),
            "mixed_lit": lensed(mixed_lit_scene(24, 18, 2), 0.4, 0.6),
            "textured_sky": lensed(textured_sky_scene(20, 14, 2), 0.3, 1.3)}


def assert_render(sc, lin, rgb, st, what):
    want = OL.render(sc, sc.lens)
    assert bits(lin) == bits(want["linear"]), what
    assert np.array_equal(rgb, want["rgb8"]), what
    assert st["rays"] == want["rays"], what


@pytest.mark.parametrize("variant", VARIANTS)
def test_every_variant_matches_the_oracle(variant):
    for name, sc in scene_set().items():
        opts = R.make_options(device=0, variant=variant)
        lin, st = R.render_linear(sc, opts)
        rgb, _ = R.render_rgb8(sc, opts)
        assert_render(sc, lin, rgb, st, f"{name}/{variant}")


def test_shard_handles_and_a_staged_handle(monkeypatch):
    torch = _torch()
    sc = scene_set()["mixed_lit"]
    want = OL.render(sc, sc.lens)
    w, h = int(sc.c.width), int(sc.c.height)
    for rank in range(3):
        opts = R.make_options(device=0, rank=rank, world=3, band_rows=2)
        rs = R.ResidentScene(sc, opts)
        rows = R.shard_row_indices(h, rank, 3, 2)
        lin = torch.empty((len(rows), w, 3), dtype=torch.float32, device="cuda:0")
        rs.render(0, lin.data_ptr())
        assert bits(lin.cpu().numpy()) == bits(want["linear"][rows]), rank
        rs.release()
    monkeypatch.setenv("RTB200_WF_SMEM", "7")   # the scene arrays staged in shared memory
    rs = R.ResidentScene(sc, R.make_options(device=0))
    monkeypatch.delenv("RTB200_WF_SMEM")
    assert rs.kernel_info()["smem_mask"] == 7
    lin = torch.empty((h, w, 3), dtype=torch.float32, device="cuda:0")
    rs.render(0, lin.data_ptr())
    assert bits(lin.cpu().numpy()) == bits(want["linear"])
    rs.release()


def test_probe_equals_the_oracle_lens_ray():
    cam, lens = R.camera_from_params_lens((13, 2, 3), (0, 0, 0), (0, 1, 0), 20.0, 1.5, 0.7, 10.0)
    L = R.lib()
    rng = np.random.default_rng(11)
    for k in range(300):
        pixel, sample = int(rng.integers(0, 1 << 31)), int(rng.integers(0, 4096))
        u, v = rng.random(2)
        o, d, t = R.rt_vec3(), R.rt_vec3(), R.C.c_uint32()
        R._check(L.rtb200_probe_lens_ray(R.C.byref(cam), R.C.byref(lens), 42 + k, pixel, sample, u, v, R.C.byref(o), R.C.byref(d), R.C.byref(t)))
        wo, wd, wt = OL.lens_ray(cam, lens, 42 + k, pixel, sample, u, v)
        assert bits(np.array([o.x, o.y, o.z, d.x, d.y, d.z])) == bits(np.concatenate([wo, wd])) and t.value == wt


def test_pinhole_stays_pinhole():
    torch = _torch()
    sc = mixed_lit_scene(24, 18, 2)
    pin_lin, _ = R.render_linear(sc, R.make_options(device=0))
    z = lensed(mixed_lit_scene(24, 18, 2), 0.0, fd=3.0)
    assert z.lens is None
    lin, _ = R.render_linear(z, R.make_options(device=0))
    assert bits(lin) == bits(pin_lin)
    # a pinhole handle given a lens renders the lens, and set_lens(None) gives today's render back byte for byte
    lens = lensed(mixed_lit_scene(24, 18, 2), 0.4, 0.6).lens
    rs = R.ResidentScene(sc, R.make_options(device=0))
    buf = torch.empty((18, 24, 3), dtype=torch.float32, device="cuda:0")
    rs.set_lens(lens)
    rs.render(0, buf.data_ptr())
    want = OL.render(sc, lens)["linear"]
    assert bits(buf.cpu().numpy()) == bits(want)
    rs.set_lens(None)
    rs.render(0, buf.data_ptr())
    assert bits(buf.cpu().numpy()) == bits(pin_lin)
    # render_frames_device without a table renders every frame with the handle's lens
    rs.set_lens(lens)
    f = R.rt_frame(sc.c.camera, sc.seed, sc.c.max_depth, 0)
    out = torch.empty((2, 18, 24, 3), dtype=torch.float32, device="cuda:0")
    arr, n = R._frame_array([f, f])
    R._check(R.lib().rtb200_render_frames_device(rs.h, arr, n, None, R.C.c_void_p(out.data_ptr()), None, None))
    assert bits(out[0].cpu().numpy()) == bits(want) and bits(out[1].cpu().numpy()) == bits(want)
    rs.release()


def test_trace_rays_of_the_lens_rays_is_the_lens_render():
    sc = scene_set()["cover"]
    rs = R.ResidentScene(sc, R.make_options(device=0))
    spp = int(sc.c.samples_per_pixel)
    acc = np.zeros((int(sc.c.height) * int(sc.c.width), 3), np.float32)
    for s in range(spp):
        o, d = OL.primary(sc, sc.lens, s)
        acc = acc + rs.trace_rays(o, d, samples=1, sample0=s)["linear"]
    lin, _ = R.render_linear(sc, R.make_options(device=0))
    assert bits((np.float32(1.0) / np.float32(spp) * acc).reshape(lin.shape)) == bits(lin)
    rs.release()


def test_frames_focus_pulls_and_mixed_frames_in_one_launch():
    sc = scene_set()["cover"]
    frames, lenses = [], []
    for k, (ap, fd) in enumerate([(0.1, 6.0), (0.0, 10.0), (0.3, 10.0), (0.1, 14.0), (0.0, None)]):
        f, L = R.make_frame_lens(sc, aperture=ap, focus_dist=fd, seed=sc.seed + k)
        frames.append(f); lenses.append(L)
    lin, st = R.render_frames(sc, frames, R.make_options(device=0), linear=True, lenses=lenses)
    assert st["batches"] == 1   # one multi-frame launch
    for k, (f, L) in enumerate(zip(frames, lenses)):
        one = R.Scene.edited(sc)
        one.c.camera = f.camera; one.seed = f.seed
        assert bits(lin[k]) == bits(OL.render(one, L)["linear"]), k
    # without lenses a pinhole scene's frames report the bytes they did before: the frame table only
    pin = scenes.cover_scene(40, 30, 3, depth=8)
    fr = [R.make_frame(pin, seed=9 + k) for k in range(3)]
    _, st = R.render_frames(pin, fr, R.make_options(device=0))
    assert st["h2d_bytes"] - R.render_frames(pin, fr[:1], R.make_options(device=0))[1]["h2d_bytes"] == 3 * 104


def test_adaptive_on_a_lens_handle():
    torch = _torch()
    sc = scene_set()["mixed_lit"]
    rs = R.ResidentScene(sc, R.make_options(device=0))
    rs.adaptive_begin(R.make_adaptive(0.05, samples_per_round=1, min_samples=1, max_samples=4))
    rs.set_lens(sc.lens)
    with pytest.raises(R.RtError):
        rs.adaptive_step(1)
    rs.adaptive_begin(R.make_adaptive(0.05, samples_per_round=1, min_samples=1, max_samples=4))
    for _ in range(8):
        if rs.adaptive_step(1)[0] == 0:
            break
    n = 18 * 24
    lin = torch.empty(n * 3, dtype=torch.float32, device="cuda:0")
    cnt = torch.empty(n, dtype=torch.int32, device="cuda:0")
    rs.adaptive_resolve(linear=lin, counts=cnt)
    lin = lin.cpu().numpy().reshape(18, 24, 3); cnt = cnt.cpu().numpy().reshape(18, 24)
    for k in np.unique(cnt):
        one = R.Scene.edited(sc)
        one.c.samples_per_pixel = int(k)
        want = OL.render(one, sc.lens)["linear"]
        assert bits(lin[cnt == k]) == bits(want[cnt == k]), k
    rs.release()


def test_aov_of_a_lens_handle_with_and_without_a_view():
    sc = scene_set()["mixed_lit"]
    rs = R.ResidentScene(sc, R.make_options(device=0))
    got = rs.aov(2, sample0=1)
    want = OL.hits(sc, sc.lens, samples=2, sample0=1)
    guides = OL.aov(sc, sc.lens, samples=2, sample0=1)
    for k in ("albedo", "normal"):
        assert bits(np.asarray(got[k]).reshape(guides[k].shape)) == bits(guides[k]), k
    assert np.array_equal(np.asarray(got["hits"]).reshape(want["hits"].shape), want["hits"])
    assert np.array_equal(np.asarray(got["sphere"]).reshape(want["sphere"].shape), want["sphere"])
    assert bits(np.asarray(got["point"]).reshape(want["point"].shape)) == bits(want["point"])
    f, _ = R.make_frame_lens(sc, look_from=(0.5, 0.8, 2.0), seed=77)
    got = rs.aov(1, view=f, outputs=("sphere", "point"))
    one = R.Scene.edited(sc)
    one.c.camera = f.camera; one.seed = 77
    want = OL.hits(one, sc.lens)
    assert np.array_equal(np.asarray(got["sphere"]).reshape(want["sphere"].shape), want["sphere"])
    assert bits(np.asarray(got["point"]).reshape(want["point"].shape)) == bits(want["point"])
    rs.release()


@pytest.mark.parametrize("variant", [FILTERED, BRUTE])
def test_updates_rebuilds_and_edits_keep_the_lens(variant):
    torch = _torch()
    sc = scene_set()["mixed_lit"]
    opts = R.make_options(device=0, variant=variant)
    rs = R.ResidentScene(sc, opts)
    buf = torch.empty((18, 24, 3), dtype=torch.float32, device="cuda:0")
    moved = sc.set_sphere(1, center=(sc._spheres[1].center.x + 0.2, sc._spheres[1].center.y, sc._spheres[1].center.z))
    rs.update_spheres([1], [moved])
    rs.render(0, buf.data_ptr())
    assert bits(buf.cpu().numpy()) == bits(OL.render(sc, sc.lens)["linear"])
    if variant == FILTERED:
        rs.rebuild()
        rs.render(0, buf.data_ptr())
        assert bits(buf.cpu().numpy()) == bits(OL.render(sc, sc.lens)["linear"])
    ed = sc.edited(remove=[0])
    rs.edit_spheres(remove=[0])
    rs.render(0, buf.data_ptr())
    assert bits(buf.cpu().numpy()) == bits(OL.render(ed, sc.lens)["linear"])
    rs.release()


def test_the_golden_fixture():
    import json
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_lens
    want = json.load(open(make_lens.OUT))
    for name, sc in make_lens.cases().items():
        for variant in VARIANTS:
            opts = R.make_options(device=0, variant=variant)
            lin, st = R.render_linear(sc, opts)
            rgb, _ = R.render_rgb8(sc, opts)
            assert make_lens.sha(lin) == want[name]["linear_sha256"], (name, variant)
            assert make_lens.sha(rgb) == want[name]["rgb8_sha256"], (name, variant)
            assert st["rays"] == want[name]["rays"], (name, variant)


def test_render_frames_of_make_frame_equals_the_scene_render():
    sc = scene_set()["cover"]
    lin, _ = R.render_linear(sc, R.make_options(device=0))
    fr, _ = R.render_frames(sc, [R.make_frame(sc), R.make_frame(sc)], R.make_options(device=0), linear=True)
    assert bits(fr[0]) == bits(lin) and bits(fr[1]) == bits(lin)


def test_a_lens_frame_over_several_sample_batches():
    """A sample-buffer cap below one frame's samples: the lens frame runs its kernel over batches with s0 > 0."""
    sc = scene_set()["textured_sky"]
    sc.c.samples_per_pixel = 5
    npix = int(sc.c.width) * int(sc.c.height)
    opts = R.make_options(device=0, sample_buffer_bytes=2 * npix * 16)
    lin, st = R.render_linear(sc, opts)
    assert st["batches"] == 3
    assert bits(lin) == bits(OL.render(sc, sc.lens)["linear"])


def test_cli_lens_config_and_frames_give_the_python_path(tmp_path):
    import json
    import os
    import subprocess
    from rtb200 import scenes as S
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cli = os.path.join(repo, "rust-raytracer_b200", "raytracer")
    cfg = S._variant(S.cover_config(), 40, 30, 2, 6)
    cfg["camera"].update(aperture=0.2, focus_dist=9.0)
    p = tmp_path / "lens.json"
    p.write_text(json.dumps(cfg))
    r = subprocess.run([cli, str(p), str(tmp_path / "out.png")], capture_output=True, text=True, cwd=repo, timeout=300)
    assert r.returncode == 0, r.stderr
    from PIL import Image

    def pixels(path):
        return np.asarray(Image.open(path).convert("RGB"))

    sc = R.Scene.from_config(cfg, S.SCENES_DIR)
    want, _ = R.render_rgb8(sc)
    assert np.array_equal(pixels(tmp_path / "out.png"), want)
    # a frames file with a focus pull, a pinhole frame and a frame that inherits the scene's lens
    cam = cfg["camera"]
    frames = [{"camera": dict(cam, focus_dist=6.0), "seed": 5}, {"camera": dict(cam, aperture=0.0), "seed": 6}, {"camera": dict(cam), "seed": 7}]
    fp = tmp_path / "frames.json"
    fp.write_text(json.dumps(frames))
    r = subprocess.run([cli, str(p), str(tmp_path / "anim")], capture_output=True, text=True, cwd=repo, timeout=300,
                       env=dict(os.environ, RTB200_FRAMES=str(fp)))
    assert r.returncode == 0, r.stderr
    fl = [R.make_frame_lens(sc, focus_dist=6.0, seed=5), R.make_frame_lens(sc, aperture=0.0, seed=6), R.make_frame_lens(sc, seed=7)]
    imgs, _ = R.render_frames(sc, [f for f, _ in fl], lenses=[l for _, l in fl])
    for i in range(3):
        assert np.array_equal(pixels(tmp_path / f"anim_{i:03d}.png"), imgs[i]), i
