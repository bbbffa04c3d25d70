"""Adaptive rounds, auxiliary buffers, pinhole and lens frames, their variance, and caller-supplied rays at sizes that fill
an H100 (DESIGN.md §3, "At frame sizes that fill the GPU"), bit for bit against the oracle: counts equal, linear f32 under
assert_frames_match, RGB8 equal, rays and samples equal, auxiliary buffers and variances bit-equal; and the launch groups of
frames at the group bound kGroupMaxFrameWork.

The smaller frames of test_gpu_adaptive.py, test_gpu_aov.py, test_gpu_frames.py, test_gpu_lens.py and test_gpu_trace_rays.py
fit in the trace kernel's first fill of its slots, or barely leave it, and in one chunk per query warp, so they run few or no
second claims from the queue, no compaction over many tiles and no grid-stride step of the auxiliary-buffer kernels. Every
case here asserts that
it reaches past them, against the bound B = sm_count x max_threads_per_multi_processor of the device it runs on
(tests/test_full_frames_cpu.py, whose LEDGER names the case of each of the 36 trace kernels)."""
import time

import numpy as np
import pytest

import oracle_aov as OA
import oracle_lens as OL
import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from test_full_frames_cpu import (COVER_N, FRAME_SPP, FRAME_WORK, GROUP_SPP, GROUP_W, LENS_FRAMES, MIN, N, RAYS_KW, RAYS_N, RAYS_SPP,
                                  ROUNDS, SPLIT_DEPTH, H, W, assert_list_reach, assert_pixel_reach, cover_scene, frame_groups,
                                  frame_want, full_frames, full_rays, full_scene, lit_config, lit_scene, params, rays_want,
                                  restated, view_of, with_depth)
from test_denoise_cpu import assert_bits_equal
from test_gpu_aov import assert_aov_equal
from test_gpu_intersect import BRUTE, EXACT, FILTERED, _torch
from test_gpu_lens import SEED64, lensed
from test_gpu_shading_edges import assert_frames_match, scene_of, synthetic_texture

pytestmark = pytest.mark.gpu
VARIANTS = {"tree": FILTERED, "brute_force": BRUTE, "exact_f64": EXACT}
SCENES = ("lit", "unlit")   # the LIGHTS = true and false kernels
AOV_W, AOV_H = 1920, 1080


@pytest.fixture(scope="module")
def bound():
    p = _torch().cuda.get_device_properties(0)
    return p.multi_processor_count * p.max_threads_per_multi_processor


def resolve(rs):
    """(rgb8, linear, counts) of the handle's adaptive render so far."""
    torch = _torch()
    n = rs.rows * int(rs.scene.c.width)
    o8 = torch.zeros(3 * n, dtype=torch.uint8, device="cuda")
    ol = torch.zeros(3 * n, dtype=torch.float32, device="cuda")
    oc = torch.zeros(n, dtype=torch.int32, device="cuda")
    rs.adaptive_resolve(o8, ol, oc)
    sh = (rs.rows, int(rs.scene.c.width))
    return o8.cpu().numpy().reshape(*sh, 3), ol.cpu().numpy().reshape(*sh, 3), oc.cpu().numpy().view(np.uint32).reshape(sh)


def assert_adaptive(img, lin, cnt, st, want, what, rows=None):
    """The frame (or its rows `rows` of the full frame) equals the restatement's; rays and samples too when `st` is given."""
    sl = slice(None) if rows is None else rows
    assert np.array_equal(cnt, want["counts"][sl]), f"{what}: counts differ in {int((cnt != want['counts'][sl]).sum())} pixels"
    assert_frames_match((lin, img), (want["linear"][sl], want["rgb8"][sl]), what)
    if st is not None:
        assert (st["rays"], st["samples"]) == (want["rays"], want["samples"]), (what, st["rays"], want["rays"], st["samples"], want["samples"])


# ---- adaptive rounds (Q_LIST, Q_LIST_LENS) ---------------------------------------------------------------------------------

@pytest.mark.parametrize("m", ROUNDS)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_adaptive_rounds_at_scale(variant, m, bound):
    sc = lit_scene()
    want = restated("lit", sc, m)
    assert_list_reach(want, W * H, m, N, bound, f"lit, m = {m}")
    img, lin, cnt, st = R.render_adaptive(sc, params(m), R.make_options(variant=VARIANTS[variant]))
    assert_adaptive(img, lin, cnt, st, want, f"{variant}, m = {m}")


@pytest.mark.parametrize("m", ROUNDS)
def test_adaptive_round_by_round_at_scale(m):
    """After every round the active count and the resolved counts, linear and RGB8 are the restatement's after that many
    rounds: each compaction keeps exactly the pixels the rule keeps, in list order."""
    sc = lit_scene()
    full = restated("lit", sc, m)
    rs = R.ResidentScene(sc)
    try:
        rs.adaptive_begin(params(m))
        r, active, rays = 0, W * H, 0
        while active:
            active, st = rs.adaptive_step(1)
            r += 1
            want = restated("lit", sc, m, rounds=r)
            assert active == want["active"], (m, r, active, want["active"])
            img, lin, cnt = resolve(rs)
            assert np.array_equal(cnt, want["counts"]), f"m = {m}, round {r}: counts differ in {int((cnt != want['counts']).sum())} pixels"
            assert_frames_match((lin, img), (want["linear"], want["rgb8"]), f"m = {m}, round {r}")
            assert st["batches"] == 1 and st["kernel_launches"] == 3, st
            rays += st["rays"]
        assert r == full["rounds"] == len(full["list_sizes"]) and rays == full["rays"], (r, full["rounds"])
    finally:
        rs.release()


def check_cover_scene(variant, bound):
    """Q_LIST without lights: the cover scene's adaptive rounds in `variant`."""
    sc = cover_scene()
    want = restated("cover", sc, 8)
    assert_list_reach(want, W * H, 8, COVER_N, bound, "cover")
    img, lin, cnt, st = R.render_adaptive(sc, params(8), R.make_options(variant=VARIANTS[variant]))
    assert_adaptive(img, lin, cnt, st, want, f"cover {variant}")


def test_adaptive_cover_scene_at_scale(bound):
    check_cover_scene("tree", bound)


@pytest.mark.parametrize("variant", ["brute_force", "exact_f64"])
def test_adaptive_cover_scene_validation_modes_at_scale(variant, bound):
    check_cover_scene(variant, bound)


def test_adaptive_max_depth_0_at_1080p(bound):
    """Black samples: a memset per round and no ray; the samples are counted by the accumulate kernel's warp ballots."""
    sc = scenes.cover_scene(AOV_W, AOV_H, N, depth=0)
    npix, m = AOV_W * AOV_H, 4
    assert npix * m >= 4 * bound
    img, lin, cnt, st = R.render_adaptive(sc, params(m))
    assert (cnt == MIN).all() and not img.any() and not lin.view(np.uint32).any()
    assert st["rays"] == 0 and st["samples"] == npix * MIN, st


def test_adaptive_sample_buffer_cap_at_scale():
    """A cap of exactly one round's samples renders the restatement's frame; one sample fewer is refused before any device
    work, and a refused begin on a handle leaves its adaptive render in progress as it was."""
    sc = lit_scene()
    m, npix = 8, W * H
    want = restated("lit", sc, m)
    exact = R.make_options(sample_buffer_bytes=m * npix * 16)
    img, lin, cnt, st = R.render_adaptive(sc, params(m), exact)
    assert_adaptive(img, lin, cnt, st, want, "cap of one round")
    with pytest.raises(R.RtError) as e:
        R.render_adaptive(sc, params(m), R.make_options(sample_buffer_bytes=m * npix * 16 - 16))
    assert e.value.code == -1 and "sample-buffer cap" in str(e.value)
    rs = R.ResidentScene(sc, exact)
    try:
        rs.adaptive_begin(params(m))
        rs.adaptive_step(1)
        before = resolve(rs)
        with pytest.raises(R.RtError) as e:
            rs.adaptive_begin(params(m + 1))
        assert "sample-buffer cap" in str(e.value)
        after = resolve(rs)
        assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(before, after))
        active, _ = rs.adaptive_step(100)
        img, lin, cnt = resolve(rs)
        assert active == 0
        assert_adaptive(img, lin, cnt, None, want, "after a refused begin")
    finally:
        rs.release()


def test_adaptive_shard_handles_at_scale():
    sc = lit_scene()
    m = 8
    want = restated("lit", sc, m)
    img, lin, cnt, _ = R.render_adaptive(sc, params(m))
    for rank in range(3):
        rows = R.shard_row_indices(H, rank, 3, 7)
        si, sl, scnt, _ = R.render_adaptive(sc, params(m), R.make_options(rank=rank, world=3, band_rows=7))
        assert si.shape[0] == len(rows) > 0
        assert np.array_equal(scnt, cnt[rows]) and np.array_equal(si, img[rows]), rank
        assert np.array_equal(sl.view(np.uint32), lin[rows].view(np.uint32)), rank
        assert_adaptive(si, sl, scnt, None, want, f"rank {rank}", rows)


def check_lens_rounds(variant, m, scene, bound):
    """Q_LIST_LENS: the `scene` through a lens, against the restatement on the oracle's lens samples."""
    sc = lensed(full_scene(scene), 0.4, 0.6)
    want = restated(f"{scene}_lens", sc, m, lens=sc.lens)
    assert_list_reach(want, W * H, m, N, bound, f"{scene} lens, m = {m}")
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        rs.adaptive_begin(params(m))
        active, st = rs.adaptive_step(100)
        img, lin, cnt = resolve(rs)
        assert active == 0
        assert_adaptive(img, lin, cnt, st, want, f"{scene} lens {variant}, m = {m}")
    finally:
        rs.release()


@pytest.mark.parametrize("m", ROUNDS)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_adaptive_lens_rounds_at_scale(variant, m, bound):
    """Case 1's scene through a lens."""
    check_lens_rounds(variant, m, "lit", bound)


@pytest.mark.parametrize("m", ROUNDS)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_adaptive_lens_rounds_unlit_at_scale(variant, m, bound):
    """Case 1's scene without its lights through a lens: the LIGHTS = false kernels of Q_LIST_LENS."""
    check_lens_rounds(variant, m, "unlit", bound)


# ---- auxiliary buffers (rt_aov_kernel, rt_aov_lens_kernel) ----------------------------------------------------------------

AOV_SAMPLES, AOV_SAMPLE0 = 3, 5
_AOV = {}


def aov_scene():
    """The lit mixed scene under a sky texture, at 1920 x 1080, without the glass bubble around its camera (whose first hits
    would all be that bubble)."""
    cfg = lit_config(AOV_W, AOV_H, 1)
    bubble = cfg["objects"].pop()
    assert bubble["radius"] == 2.0 and "Glass" in bubble["material"]
    return scene_of(cfg, sky=synthetic_texture(5, 3))


def oracle_aov(key, fn):
    """The oracle's auxiliary buffers fn() once per key (the module's cache); prints the oracle's time."""
    if key not in _AOV:
        t = time.perf_counter()
        _AOV[key] = fn()
        print(f"[oracle] aov {key}: {time.perf_counter() - t:.1f} s")
    return _AOV[key]


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_aov_at_1080p(variant, bound):
    sc = aov_scene()
    assert_pixel_reach(AOV_W * AOV_H, bound, "aov")
    want = oracle_aov("lit", lambda: OA.aov(sc, AOV_SAMPLES, AOV_SAMPLE0))
    assert (want["hits"] == 0).any() and (want["hits"] == AOV_SAMPLES).any() and (want["sphere"] >= 0).any()
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        got = rs.aov(AOV_SAMPLES, sample0=AOV_SAMPLE0)
        assert_aov_equal(got, want, f"{variant}: host form")
        assert got["stats"]["rays"] == got["stats"]["samples"] == AOV_W * AOV_H * AOV_SAMPLES
        dv = rs.aov(AOV_SAMPLES, sample0=AOV_SAMPLE0, on_device=True)
        _torch().cuda.synchronize()
        assert_aov_equal(dv, want, f"{variant}: device form")
    finally:
        rs.release()


def test_aov_cover_scene_at_1080p(bound):
    sc = scenes.cover_scene(AOV_W, AOV_H, 1)
    assert_pixel_reach(AOV_W * AOV_H, bound, "aov cover")
    want = oracle_aov("cover", lambda: OA.aov(sc, 1, 0))
    rs = R.ResidentScene(sc, R.make_options(variant=FILTERED))
    try:
        assert_aov_equal(rs.aov(1), want, "cover")
    finally:
        rs.release()


def test_aov_view_at_1080p(bound):
    sc = aov_scene()
    assert_pixel_reach(AOV_W * AOV_H, bound, "aov view")
    view = R.make_frame(sc, look_from={"x": 9.0, "y": 4.0, "z": -6.0}, look_at={"x": 0.5, "y": 0.5, "z": 0.0}, vfov=35.0,
                        seed=2_718_281_828)
    want = oracle_aov("view", lambda: OA.aov(sc, AOV_SAMPLES, AOV_SAMPLE0, camera=view.camera, seed=view.seed))
    rs = R.ResidentScene(sc)
    try:
        assert_aov_equal(rs.aov(AOV_SAMPLES, sample0=AOV_SAMPLE0, view=view), want, "view")
    finally:
        rs.release()


def test_aov_lens_at_1080p(bound):
    sc = lensed(aov_scene(), 0.4, 0.6)
    sc.seed = SEED64
    assert_pixel_reach(AOV_W * AOV_H, bound, "aov lens")
    want = oracle_aov("lens", lambda: OL.aov_all(sc, sc.lens, AOV_SAMPLES, AOV_SAMPLE0))
    rs = R.ResidentScene(sc)
    try:
        assert_aov_equal(rs.aov(AOV_SAMPLES, sample0=AOV_SAMPLE0), want, "lens")
    finally:
        rs.release()


def test_aov_shard_handles_at_1080p():
    sc = aov_scene()
    want = oracle_aov("lit", lambda: OA.aov(sc, AOV_SAMPLES, AOV_SAMPLE0))
    full = R.ResidentScene(sc)
    try:
        whole = full.aov(AOV_SAMPLES, sample0=AOV_SAMPLE0)
    finally:
        full.release()
    for rank in range(3):
        rows = R.shard_row_indices(AOV_H, rank, 3, 16)
        rs = R.ResidentScene(sc, R.make_options(rank=rank, world=3, band_rows=16))
        try:
            got = rs.aov(AOV_SAMPLES, sample0=AOV_SAMPLE0)
            assert got["albedo"].shape[0] == len(rows) > 0
            assert_aov_equal(got, whole, f"rank {rank} vs the whole frame", rows)
            assert_aov_equal(got, want, f"rank {rank} vs the oracle", rows)
        finally:
            rs.release()


# ---- lens frames (Q_FRAMES_LENS) -----------------------------------------------------------------------------------------

_LENS_FRAMES = {}


def lens_frames(sc):
    """Four lens frames of sc, each with its own camera, lens and 64-bit key."""
    specs = [((13.0, 2.0, 3.0), 0.4, None), ((10.0, 3.0, -6.0), 0.2, 8.0), ((-9.0, 2.5, 7.0), 0.6, 5.0), ((4.0, 6.0, 12.0), 0.3, 14.0)]
    frames, lenses = [], []
    for k, (lf, ap, fd) in enumerate(specs):
        f, L = R.make_frame_lens(sc, look_from=list(lf), aperture=ap, focus_dist=fd, seed=SEED64 + k * 0x0000000100000003)
        assert L.radius > 0
        frames.append(f); lenses.append(L)
    return frames, lenses


def lens_frames_want(scene, sc, frames, lenses):
    """The oracle's lens renders of the frames, once per scene: [(linear, rgb8, rays)]."""
    if scene not in _LENS_FRAMES:
        t = time.perf_counter()
        outs = []
        for f, L in zip(frames, lenses):
            w = OL.render(view_of(sc, f), L)
            outs.append((w["linear"], w["rgb8"], w["rays"]))
        _LENS_FRAMES[scene] = outs
        print(f"[oracle] lens frames {scene}: {len(frames) * int(sc.c.width) * int(sc.c.height) * int(sc.c.samples_per_pixel):,} "
              f"samples in {time.perf_counter() - t:.1f} s")
    return _LENS_FRAMES[scene]


def check_lens_frames(variant, scene, bound):
    """Four lens frames of 960 x 540 x 4, each with its own camera, lens and 64-bit key, in one launch group."""
    w, h, spp = LENS_FRAMES
    sc = full_scene(scene, w, h, spp)
    frames, lenses = lens_frames(sc)
    work = len(frames) * w * h * spp
    assert_pixel_reach(work, bound, "lens frames")
    opts = R.make_options(variant=VARIANTS[variant])
    lin, st = R.render_frames(sc, frames, opts, linear=True, lenses=lenses)
    img, st8 = R.render_frames(sc, frames, opts, lenses=lenses)
    # one group: one trace launch for the four frames and a resolve per frame
    assert st["batches"] == st8["batches"] == 1 and st["kernel_launches"] == st8["kernel_launches"] == 1 + len(frames), st
    want = lens_frames_want(scene, sc, frames, lenses)
    for k, (wl, wi, _) in enumerate(want):
        assert_frames_match((lin[k], img[k]), (wl, wi), f"{scene} {variant} frame {k}")
    rays = sum(r for _, _, r in want)
    assert st["rays"] == st8["rays"] == rays and st["samples"] == work, (st["rays"], rays)


def test_lens_frames_at_scale(bound):
    check_lens_frames("tree", "lit", bound)


# the other five (mode, scene) pairs of Q_FRAMES_LENS
@pytest.mark.parametrize("variant, scene", [(v, s) for v in VARIANTS for s in SCENES if (v, s) != ("tree", "lit")])
def test_lens_frames_every_mode_and_scene_at_scale(variant, scene, bound):
    check_lens_frames(variant, scene, bound)


# ---- pinhole frames (Q_SINGLE, Q_FRAMES) and their variance ----------------------------------------------------------------

def assert_frame(lin, img, want, what):
    assert_frames_match((lin, img), (want["linear"], want["rgb8"]), what)


def frames_opts(variant, **kw):
    return R.make_options(variant=VARIANTS[variant], **kw)


@pytest.mark.parametrize("scene", SCENES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_single_frame_at_scale(variant, scene, bound):
    """Q_SINGLE: frame 0 rendered alone, the oracle's samples summed in sample order."""
    assert_pixel_reach(FRAME_WORK, bound, "one frame")
    sc = full_scene(scene, spp=FRAME_SPP)
    view = view_of(sc, full_frames(sc)[0])
    want = frame_want(scene, 0)
    lin, st = R.render_linear(view, frames_opts(variant))
    img, st8 = R.render_rgb8(view, frames_opts(variant))
    assert_frame(lin, img, want, f"{scene} {variant}")
    assert st["batches"] == st8["batches"] == 1, st
    assert st["rays"] == st8["rays"] == want["rays"] and st["samples"] == FRAME_WORK, (st["rays"], want["rays"])


@pytest.mark.parametrize("scene", SCENES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_frame_group_at_scale(variant, scene, bound):
    """Q_FRAMES: two frames with their own cameras and keys in one launch; with another max_depth for frame 1, two
    single-frame launches."""
    assert_pixel_reach(2 * FRAME_WORK, bound, "frame group")
    sc = full_scene(scene, spp=FRAME_SPP)
    frames = full_frames(sc)
    wants = [frame_want(scene, k) for k in range(2)]
    lin, st = R.render_frames(sc, frames, frames_opts(variant), linear=True)
    img, st8 = R.render_frames(sc, frames, frames_opts(variant))
    assert st["batches"] == st8["batches"] == 1 and st["kernel_launches"] == st8["kernel_launches"] == 1 + 2, st
    for k in range(2):
        assert_frame(lin[k], img[k], wants[k], f"{scene} {variant} frame {k}")
    rays = sum(w["rays"] for w in wants)
    assert st["rays"] == st8["rays"] == rays and st["samples"] == 2 * FRAME_WORK, (st["rays"], rays)

    split = [frames[0], with_depth(frames[1], SPLIT_DEPTH)]
    assert frame_groups([f.max_depth for f in split], FRAME_WORK) == [1, 1]
    wants[1] = frame_want(scene, 1, SPLIT_DEPTH)
    lin, st = R.render_frames(sc, split, frames_opts(variant), linear=True)
    img, st8 = R.render_frames(sc, split, frames_opts(variant))
    assert st["batches"] == st8["batches"] == 2 and st["kernel_launches"] == st8["kernel_launches"] == 2 + 2, st
    for k in range(2):
        assert_frame(lin[k], img[k], wants[k], f"{scene} {variant} split frame {k}")
    assert st["rays"] == sum(w["rays"] for w in wants), st["rays"]


@pytest.mark.parametrize("scene", SCENES)
def test_frame_variance_and_batches_at_scale(scene, bound):
    """The variance of the pixel means of the group and of frame 0 alone, and of frame 0 over three sample batches (3, 3
    and 2 samples, accum and accum_sq carried over 230,400 pixels), bit for bit against the formula on the oracle's
    samples; the image is unchanged by the batches."""
    sc = full_scene(scene, spp=FRAME_SPP)
    frames = full_frames(sc)
    wants = [frame_want(scene, k) for k in range(2)]
    lin, var, st = R.render_frames(sc, frames, linear=True, variance=True)
    img, _, _ = R.render_frames(sc, frames, variance=True)
    assert st["batches"] == 1 and st["kernel_launches"] == 1 + 2, st
    for k in range(2):
        assert_frame(lin[k], img[k], wants[k], f"{scene} variance group frame {k}")
        assert_bits_equal(var[k], wants[k]["variance"], f"{scene} variance of group frame {k}")
    img, var8, _ = R.render_frames(sc, frames[:1], variance=True)
    lin, var, st = R.render_frames(sc, frames[:1], linear=True, variance=True)
    assert st["batches"] == 1, st
    assert_frame(lin[0], img[0], wants[0], f"{scene} variance frame 0")
    assert_bits_equal(var[0], wants[0]["variance"], f"{scene} variance of frame 0")
    assert_bits_equal(var8, var, f"{scene} variance of the rgb8 call")

    capped = R.make_options(sample_buffer_bytes=3 * W * H * 16)
    assert 3 * W * H >= 2 * bound, ("a batch of 3 samples reaches past the first fill", 3 * W * H, bound)
    img, var8, st8 = R.render_frames(sc, frames[:1], capped, variance=True)
    lin, var, st = R.render_frames(sc, frames[:1], capped, linear=True, variance=True)
    assert st["batches"] == st8["batches"] == 3 and st["kernel_launches"] == 3 + 3, st
    assert_frame(lin[0], img[0], wants[0], f"{scene} frame 0 in three batches")
    assert_bits_equal(var[0], wants[0]["variance"], f"{scene} variance in three batches")
    assert_bits_equal(var8, var, f"{scene} variance of the rgb8 call in three batches")
    assert st["rays"] == wants[0]["rays"] and st["samples"] == FRAME_WORK, st


def test_frame_group_shards_at_scale(bound):
    """Row-band shard handles (world 3, band_rows 7) of the lit frame group in the tree mode: each rank's rows of both
    frames, one launch group per rank."""
    sc = full_scene("lit", spp=FRAME_SPP)
    frames = full_frames(sc)
    wants = [frame_want("lit", k) for k in range(2)]
    full, _ = R.render_frames(sc, frames, frames_opts("tree"), linear=True)
    for rank in range(3):
        rows = R.shard_row_indices(H, rank, 3, 7)
        assert_pixel_reach(2 * len(rows) * W * FRAME_SPP, bound, f"rank {rank}")
        opts = frames_opts("tree", rank=rank, world=3, band_rows=7)
        lin, st = R.render_frames(sc, frames, opts, linear=True)
        img, _ = R.render_frames(sc, frames, opts)
        assert lin.shape[1] == len(rows) > 0 and st["batches"] == 1 and st["kernel_launches"] == 1 + 2, (rank, st)
        assert_bits_equal(lin, full[:, rows], f"rank {rank} vs the full frames")
        for k in range(2):
            assert_frames_match((lin[k], img[k]), (wants[k]["linear"][rows], wants[k]["rgb8"][rows]), f"rank {rank} frame {k}")


# ---- caller-supplied rays (Q_RAYS) -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("scene", SCENES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_trace_rays_at_scale(variant, scene, bound):
    """300,001 rays x 4 samples in one launch from sample 3 and stream 7, against oracle_trace_rays; then on a handle whose
    cap holds one sample of every ray, four launches, the same bytes."""
    assert_pixel_reach(RAYS_N * RAYS_SPP, bound, "trace_rays")
    sc = full_scene(scene)
    o, d = full_rays()
    want = rays_want(scene)
    rs = R.ResidentScene(sc, frames_opts(variant))
    small = R.ResidentScene(sc, frames_opts(variant, sample_buffer_bytes=RAYS_N * 16))
    try:
        got = rs.trace_rays(o, d, RAYS_SPP, rgb8=True, **RAYS_KW)
        assert_frames_match((got["linear"], got["rgb8"]), (want["linear"], want["rgb8"]), f"{scene} {variant}")
        st = got["stats"]
        assert st["batches"] == 1 and st["kernel_launches"] == 2, st
        assert st["rays"] == want["rays"] and st["samples"] == RAYS_N * RAYS_SPP, (st["rays"], want["rays"])
        b = small.trace_rays(o, d, RAYS_SPP, rgb8=True, **RAYS_KW)
        assert b["stats"]["batches"] == RAYS_SPP and b["stats"]["kernel_launches"] == 2 * RAYS_SPP, b["stats"]
        assert np.array_equal(b["linear"].view(np.uint32), got["linear"].view(np.uint32)) and np.array_equal(b["rgb8"], got["rgb8"])
        assert b["stats"]["rays"] == st["rays"]
    finally:
        rs.release(); small.release()


# ---- the frame-group bound, kGroupMaxFrameWork = 2^24 ----------------------------------------------------------------------

GROUP_VIEWS = [dict(), dict(look_from=[-9.0, 2.5, 7.0], look_at=[0.0, 0.5, 0.0]), dict(look_from=[10.0, 3.0, -6.0]),
               dict(look_from=[4.0, 6.0, 12.0]), dict(look_from=[-12.0, 1.5, -4.0], look_at=[0.0, 1.0, 0.0])]


@pytest.mark.parametrize("rows, n, groups", [(512, 2, [2]), (513, 2, [1, 1]), (512, 5, [4, 1])],
                         ids=["at_the_bound", "one_row_over", "five_at_the_default_cap"])
def test_frame_groups_at_the_frame_work_bound(rows, n, groups):
    """Frames of exactly 2^24 samples (1024 x 512 x 32) group, one row more runs each frame alone, and at the default 1 GiB
    cap five of them form groups of 4 and 1; every frame equals its own single-frame render bit for bit, and the oracle on
    its top, middle and bottom rows."""
    sc = full_scene("lit", GROUP_W, rows, GROUP_SPP)
    frames = [R.make_frame(sc, seed=SEED64 + 0x100000001 * k, **GROUP_VIEWS[k]) for k in range(n)]
    assert frame_groups([f.max_depth for f in frames], GROUP_W * rows * GROUP_SPP) == groups
    lin, st = R.render_frames(sc, frames, linear=True)
    img, st8 = R.render_frames(sc, frames)
    assert st["batches"] == st8["batches"] == len(groups) and st["kernel_launches"] == len(groups) + n, st
    rays, t = 0, 0.0
    for k, f in enumerate(frames):
        view = view_of(sc, f)
        one, st1 = R.render_linear(view)
        one8, _ = R.render_rgb8(view)
        assert st1["batches"] == 1
        assert_frames_match((lin[k], img[k]), (one, one8), f"frame {k} vs its own render")
        rays += st1["rays"]
        t0 = time.perf_counter()
        for y in (0, rows // 2, rows - 1):
            wl, wi, _ = O.render(view, y0=y, y1=y + 1)
            assert_frames_match((lin[k, y], img[k, y]), (wl[y], wi[y]), f"frame {k} row {y} vs the oracle")
        t += time.perf_counter() - t0
    print(f"[oracle] group bound, {n} frames of {GROUP_W} x {rows}: 3 rows each in {t:.1f} s")
    assert st["rays"] == st8["rays"] == rays and st["samples"] == n * GROUP_W * rows * GROUP_SPP, (st["rays"], rays)
