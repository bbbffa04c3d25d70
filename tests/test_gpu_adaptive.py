"""Adaptive rendering on the GPU (rtb200_adaptive_*, rtb200_render_adaptive, the CLI's RTB200_ADAPTIVE) against the numpy
restatement of the rule over the oracle's per-sample radiances (tests/adaptive_restatement.py) and against the one-shot
render. Every comparison is bit-exact: linear f32 (NaN masks equal, other values bit-equal), RGB8, counts and rays.

Contract (include/rtb200.h): a pixel that received n samples has exactly the linear value, RGB8 value and rays of the one-shot
render of the same scene at samples_per_pixel = n. Each case asserts that it reaches the edges of the rule: at least three
distinct counts, and pixels both at min_samples and at max_samples."""
import json
import math
import os
import subprocess

import numpy as np
import pytest

import adaptive_restatement as A
import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from synth import mixed_config, _v
from test_gpu_shading_edges import assert_frames_match, nonfinite_scene

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, N, M, MIN = 48, 36, 24, 4, 8
TOL = dict(rel_tol=0.1, abs_tol=0.005)


def _lit(n_lights, sky="gradient", spp=N):
    cfg = mixed_config(W, H, spp, 8, seed=7, n=30, sky=sky)
    pos = [(0.0, 3.0, 0.0), (-3.0, 2.0, 3.0)]
    for k in range(n_lights):
        cfg["objects"].insert(3 + 5 * k, {"center": _v(*pos[k]), "radius": 0.6, "material": {"Light": {}}})
    return R.Scene.from_config(cfg)


SCENES = {
    "cover": lambda: scenes.cover_scene(W, H, N, depth=8),
    "mixed_1_light": lambda: _lit(1),
    "mixed_2_lights": lambda: _lit(2),
    "textured": lambda: R.Scene.from_config(scenes._variant(scenes.test_scene_config(), W, H, N, 8), scenes.SCENES_DIR),
    "black_sky": lambda: _lit(1, sky="none"),
    "max_depth_0": lambda: scenes.cover_scene(W, H, N, depth=0),
    "nonfinite_albedo": lambda: nonfinite_scene(W, H, N, 6, 0, "Lambertian", math.nan, 1),
}
_SAMPLES = {}


def _samples(name, sc):
    if name not in _SAMPLES:
        _SAMPLES[name] = A.render_samples(sc, 0, sc.c.samples_per_pixel)
    return _SAMPLES[name]


def _params(m=M, min_samples=MIN, **kw):
    t = dict(TOL, **kw)
    return R.make_adaptive(t["rel_tol"], t["abs_tol"], samples_per_round=m, min_samples=min_samples)


def _assert_matches(img, lin, cnt, st, want, what, rows=None):
    sl = slice(None) if rows is None else rows
    assert np.array_equal(cnt, want["counts"][sl]), f"{what}: counts differ in {int((cnt != want['counts'][sl]).sum())} pixels"
    assert_frames_match((lin, img), (want["linear"][sl], want["rgb8"][sl]), what)
    if rows is None:
        assert st["rays"] == want["rays"] and st["samples"] == want["samples"], (what, st["rays"], want["rays"], st["samples"], want["samples"])


def _assert_edges(cnt, name):
    u = np.unique(cnt)
    if name == "max_depth_0":   # black samples: every pixel stops at min_samples
        assert u.tolist() == [MIN]
        return
    assert len(u) >= 3 and u[0] == MIN and u[-1] == N, u


@pytest.mark.parametrize("name", list(SCENES))
def test_adaptive_render_matches_the_restatement(name):
    sc = SCENES[name]()
    x, rays = _samples(name, sc)
    p = _params()
    want = A.run(x, rays, M, N, MIN, p.abs_tol, p.rel_tol)
    img, lin, cnt, st = R.render_adaptive(sc, p)
    _assert_matches(img, lin, cnt, st, want, name)
    _assert_edges(cnt, name)
    if name == "max_depth_0":
        assert st["rays"] == 0
    if name == "nonfinite_albedo":
        nan = np.isnan(lin).any(-1)
        assert nan.any() and (cnt[nan] == N).all()


@pytest.mark.parametrize("m", [4, 5], ids=["m_divides_N", "m_does_not_divide_N"])
def test_negative_tolerances_give_the_one_shot_render(m):
    sc = SCENES["cover"]()
    img, lin, cnt, st = R.render_adaptive(sc, _params(m=m, min_samples=1, rel_tol=-1.0, abs_tol=-1e-30))
    lin1, st1 = R.render_linear(sc)
    img1, _ = R.render_rgb8(sc)
    assert (cnt == N).all()
    assert_frames_match((lin, img), (lin1, img1), f"m = {m}")
    assert st["rays"] == st1["rays"] and st["samples"] == st1["samples"] and st["batches"] == -(-N // m)


@pytest.mark.parametrize("variant", [R.RT_VARIANT_FILTERED, R.RT_VARIANT_BRUTE_FORCE, R.RT_VARIANT_EXACT_F64],
                         ids=["tree", "brute_force", "exact_f64"])
def test_variants_match_the_restatement(variant):
    sc = SCENES["mixed_2_lights"]()
    x, rays = _samples("mixed_2_lights", sc)
    p = _params()
    want = A.run(x, rays, M, N, MIN, p.abs_tol, p.rel_tol)
    img, lin, cnt, st = R.render_adaptive(sc, p, R.make_options(variant=variant))
    _assert_matches(img, lin, cnt, st, want, f"variant {variant}")
    _assert_edges(cnt, "mixed_2_lights")


def test_shard_rows_equal_the_full_frame_rows():
    sc = SCENES["cover"]()
    p = _params()
    img, lin, cnt, _ = R.render_adaptive(sc, p)
    for rank in range(3):
        o = R.make_options(rank=rank, world=3, band_rows=7)
        rows = R.shard_row_indices(H, rank, 3, 7)
        si, sl, sc_, _ = R.render_adaptive(sc, p, o)
        assert si.shape[0] == len(rows)
        assert np.array_equal(sc_, cnt[rows]) and np.array_equal(si, img[rows])
        assert np.array_equal(sl.view(np.uint32), lin[rows].view(np.uint32))


def test_each_pixel_equals_the_one_shot_render_at_its_count():
    sc = SCENES["mixed_1_light"]()
    img, lin, cnt, _ = R.render_adaptive(sc, _params())
    for n in np.unique(cnt):
        sc.c.samples_per_pixel = int(n)
        lin1, _ = R.render_linear(sc)
        img1, _ = R.render_rgb8(sc)
        at = cnt == n
        assert np.array_equal(lin[at].view(np.uint32), lin1[at].view(np.uint32)), n
        assert np.array_equal(img[at], img1[at]), n


def _resolve(rs):
    import torch
    n = rs.rows * rs.scene.c.width
    o8 = torch.zeros(3 * n, dtype=torch.uint8, device="cuda")
    ol = torch.zeros(3 * n, dtype=torch.float32, device="cuda")
    oc = torch.zeros(n, dtype=torch.int32, device="cuda")
    rs.adaptive_resolve(o8, ol, oc)
    sh = (rs.rows, rs.scene.c.width)
    return (o8.cpu().numpy().reshape(*sh, 3), ol.cpu().numpy().reshape(*sh, 3), oc.cpu().numpy().view(np.uint32).reshape(sh))


def test_round_by_round_and_a_second_begin():
    sc = SCENES["cover"]()
    x, rays = _samples("cover", sc)
    p = _params(m=5)
    rs = R.ResidentScene(sc)
    try:
        for attempt in range(2):
            rs.adaptive_begin(p)
            img, lin, cnt = _resolve(rs)
            assert not cnt.any() and not lin.any() and not img.any()
            r, active, rays_sum = 0, W * H, 0
            while active:
                active, st = rs.adaptive_step(1)
                r += 1
                want = A.run(x, rays, 5, N, MIN, p.abs_tol, p.rel_tol, rounds=r)
                img, lin, cnt = _resolve(rs)
                assert np.array_equal(cnt, want["counts"]) and active == want["active"], (attempt, r)
                assert_frames_match((lin, img), (want["linear"], want["rgb8"]), f"begin {attempt}, round {r}")
                rays_sum += st["rays"]
                assert st["batches"] == 1 and st["kernel_launches"] == 3
            assert r == want["rounds"] and rays_sum == want["rays"]
            assert rs.adaptive_step(4) == (0, rs.adaptive_step(1)[1])   # finished: a no-op
    finally:
        rs.release()


def test_update_between_steps_fails_and_a_rebuild_does_not_change_the_run():
    sc = SCENES["mixed_1_light"]()
    p = _params()
    rs = R.ResidentScene(sc)
    try:
        rs.adaptive_begin(p)
        rs.adaptive_step(1)
        rs.rebuild()
        rs.adaptive_step(100)
        img, lin, cnt = _resolve(rs)
        want = R.render_adaptive(sc, p)
        assert np.array_equal(cnt, want[2]) and np.array_equal(img, want[0])
        assert np.array_equal(lin.view(np.uint32), want[1].view(np.uint32))
        rs.adaptive_begin(p)
        rs.adaptive_step(1)
        edited = sc.set_sphere(5, center=[0.5, 0.6, 0.5], radius=0.6)
        rs.update_spheres([5], [edited])
        with pytest.raises(R.RtError) as e:
            rs.adaptive_step(1)
        assert e.value.code == -1 and "updated" in str(e.value)
        rs.adaptive_begin(p)
        rs.adaptive_step(100)
        img, lin, cnt = _resolve(rs)
        fresh = R.render_adaptive(sc, p)   # sc now holds the edit
        assert np.array_equal(cnt, fresh[2]) and np.array_equal(img, fresh[0])
        assert np.array_equal(lin.view(np.uint32), fresh[1].view(np.uint32))
        assert not np.array_equal(cnt, want[2]) or not np.array_equal(img, want[0])
    finally:
        rs.release()


def test_steps_beside_async_frames_of_another_handle():
    import torch
    sa = SCENES["cover"]()
    x, rays = _samples("cover", sa)
    sb = _lit(2)
    sb.seed = 99
    lin_b, img_b, st_b = O.render(sb)
    p = _params()
    want = A.run(x, rays, M, N, MIN, p.abs_tol, p.rel_tol)
    a, b = R.ResidentScene(sa), R.ResidentScene(sb)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    try:
        outs = [(torch.zeros(W * H * 3, dtype=torch.uint8, device="cuda"), torch.zeros(W * H * 3, dtype=torch.float32, device="cuda"))
                for _ in range(2)]
        a.adaptive_begin(p, stream=s1)
        with torch.cuda.stream(s2):
            torch.cuda._sleep(50_000_000)
        for o in outs:   # B's frames take sets 0 and 1 on s2, held back; A's steps take set 0 on s1
            b.render_async(o[0].data_ptr(), o[1].data_ptr(), s2.cuda_stream)
        active, st = a.adaptive_step(2, stream=s1)
        active, st2 = a.adaptive_step(100, stream=s1)
        stb = b.wait()
        torch.cuda.synchronize()
        img, lin, cnt = _resolve(a)
        assert active == 0 and np.array_equal(cnt, want["counts"])
        assert_frames_match((lin, img), (want["linear"], want["rgb8"]), "A's adaptive render")
        assert st["rays"] + st2["rays"] == want["rays"]
        for o in outs:
            assert_frames_match((o[1].cpu().numpy().reshape(H, W, 3), o[0].cpu().numpy().reshape(H, W, 3)), (lin_b, img_b), "B's frame")
        assert stb["rays"] == st_b["rays"]
    finally:
        torch.cuda.synchronize()
        a.release(); b.release()


def test_cli_writes_the_adaptive_image(tmp_path):
    from PIL import Image
    cfg = scenes._variant(scenes.cover_config(), W, H, N, 8)
    path = tmp_path / "scene.json"
    path.write_text(json.dumps(cfg))
    env = dict(os.environ, RTB200_ADAPTIVE="0.1,0.005,4,8", RTB200_STATS="1")
    env.pop("RTB200_GPUS", None); env.pop("RTB200_FRAMES", None)
    cli = os.path.join(REPO, "rust-raytracer_b200", "raytracer")
    r = subprocess.run([cli, str(path), str(tmp_path / "o.png")], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stderr
    assert r.stdout.splitlines()[1].startswith("Rendering") and r.stdout.splitlines()[2].startswith("Frame time:")
    img, _, cnt, st = R.render_adaptive(R.Scene.from_config(cfg), _params())
    assert np.array_equal(np.asarray(Image.open(tmp_path / "o.png").convert("RGB")), img)
    assert f"adaptive: {int(cnt.astype(np.uint64).sum())} of {N * W * H} samples" in r.stderr
    bad = subprocess.run([cli, str(path), str(tmp_path / "p.png")], capture_output=True, text=True, timeout=300,
                         env=dict(env, RTB200_GPUS="1"))
    assert bad.returncode == 101 and "not supported" in bad.stderr
