"""Adaptive rounds, auxiliary buffers and lens frames at frame sizes that fill an H100 (DESIGN.md §3, "At frame sizes that fill
the GPU"), bit for bit against the oracle: counts equal, linear f32 under assert_frames_match, RGB8 equal, rays and samples
equal, auxiliary buffers bit-equal.

The smaller frames of test_gpu_adaptive.py, test_gpu_aov.py and test_gpu_lens.py fit in the trace kernel's first fill of its
slots and in one chunk per query warp, so they never run a Q_LIST slot's second claim from the queue, a compaction over many
tiles, or the auxiliary-buffer kernels' grid-stride step. Every case here asserts that it reaches past them, against the bound
B = sm_count x max_threads_per_multi_processor of the device it runs on (tests/test_full_frames_cpu.py)."""
import time

import numpy as np
import pytest

import oracle_aov as OA
import oracle_lens as OL
import rtb200 as R
from rtb200 import scenes
from test_full_frames_cpu import (COVER_N, MIN, N, ROUNDS, H, W, assert_list_reach, assert_pixel_reach, cover_scene, lit_config,
                                  lit_scene, params, restated)
from test_gpu_aov import assert_aov_equal
from test_gpu_intersect import BRUTE, EXACT, FILTERED, _torch
from test_gpu_lens import SEED64, lensed
from test_gpu_shading_edges import assert_frames_match, scene_of, synthetic_texture

pytestmark = pytest.mark.gpu
VARIANTS = {"tree": FILTERED, "brute_force": BRUTE, "exact_f64": EXACT}
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


def test_adaptive_cover_scene_at_scale(bound):
    sc = cover_scene()
    want = restated("cover", sc, 8)
    assert_list_reach(want, W * H, 8, COVER_N, bound, "cover")
    img, lin, cnt, st = R.render_adaptive(sc, params(8), R.make_options(variant=FILTERED))
    assert_adaptive(img, lin, cnt, st, want, "cover")


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


def lit_lens_scene():
    return lensed(lit_scene(), 0.4, 0.6)


@pytest.mark.parametrize("m", ROUNDS)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_adaptive_lens_rounds_at_scale(variant, m, bound):
    """Q_LIST_LENS: case 1's scene through a lens, against the restatement on the oracle's lens samples."""
    sc = lit_lens_scene()
    want = restated("lit_lens", sc, m, lens=sc.lens)
    assert_list_reach(want, W * H, m, N, bound, f"lit lens, m = {m}")
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        rs.adaptive_begin(params(m))
        active, st = rs.adaptive_step(100)
        img, lin, cnt = resolve(rs)
        assert active == 0
        assert_adaptive(img, lin, cnt, st, want, f"lens {variant}, m = {m}")
    finally:
        rs.release()


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

def test_lens_frames_at_scale(bound):
    """Four lens frames of 960 x 540 x 4, each with its own camera, lens and 64-bit key, in one launch group."""
    sc = lit_scene(960, 540, 4)
    specs = [((13.0, 2.0, 3.0), 0.4, None), ((10.0, 3.0, -6.0), 0.2, 8.0), ((-9.0, 2.5, 7.0), 0.6, 5.0), ((4.0, 6.0, 12.0), 0.3, 14.0)]
    frames, lenses = [], []
    for k, (lf, ap, fd) in enumerate(specs):
        f, L = R.make_frame_lens(sc, look_from=list(lf), aperture=ap, focus_dist=fd, seed=SEED64 + k * 0x0000000100000003)
        assert L.radius > 0
        frames.append(f); lenses.append(L)
    work = len(frames) * 960 * 540 * 4
    assert_pixel_reach(work, bound, "lens frames")
    lin, st = R.render_frames(sc, frames, linear=True, lenses=lenses)
    img, st8 = R.render_frames(sc, frames, lenses=lenses)
    # one group: one trace launch for the four frames and a resolve per frame
    assert st["batches"] == st8["batches"] == 1 and st["kernel_launches"] == st8["kernel_launches"] == 1 + len(frames), st
    rays, t = 0, time.perf_counter()
    for k, (f, L) in enumerate(zip(frames, lenses)):
        one = R.Scene.edited(sc)
        one.c.camera = f.camera; one.seed = f.seed
        want = OL.render(one, L)
        assert_frames_match((lin[k], img[k]), (want["linear"], want["rgb8"]), f"frame {k}")
        rays += want["rays"]
    print(f"[oracle] lens frames: {work:,} samples in {time.perf_counter() - t:.1f} s")
    assert st["rays"] == st8["rays"] == rays and st["samples"] == work, (st["rays"], rays)
