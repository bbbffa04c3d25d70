"""The full-frame cases of tests/test_gpu_full_frames.py without a GPU (DESIGN.md §3, "At frame sizes that fill the GPU"): the
scenes, parameters and reach rules they share, the oracle's bulk per-sample route they compare with, held to the per-sample
routine of the adaptive restatement, and the reach of the adaptive rounds, asserted on the restatement alone against the
bound of a 132-SM H100 so that a change of parameters cannot quietly drop it.

Reach: a case is big enough to leave the trace kernel's first fill of its slots, or an auxiliary-buffer warp's first chunk.
The bound B = sm_count x max_threads_per_multi_processor caps both the resident trace slots (CTAs of 256 slots) and the
resident query threads, whatever the occupancy, so 4B work ids (or pixels) take at least four fills (or passes)."""
import time

import numpy as np
import pytest

import adaptive_restatement as A
import oracle_lens as OL
import rtb200 as R
from rtb200 import scenes
from synth import mixed_config, _v

W, H = 640, 360            # the adaptive frames: 230,400 pixels
N, MIN = 32, 8
TOL = dict(rel_tol=0.3, abs_tol=0.02)   # the list shrinks over every round and ends at N with a few thousand pixels
ROUNDS = (8, 5)            # samples per round: m divides N, and m does not (a last round of 2 samples)
COVER_N = 16
H100_BOUND = 132 * 2048    # B of a 132-SM H100 (2,048 resident threads per SM)
OLD = (48, 36)             # the largest adaptive frame compared with the oracle before these cases


def lit_config(w=W, h=H, spp=N, sky="gradient"):
    """test_gpu_adaptive's mixed_2_lights at any size: the 30-sphere mixed scene with two lights."""
    cfg = mixed_config(w, h, spp, 8, seed=7, n=30, sky=sky)
    for k, pos in enumerate([(0.0, 3.0, 0.0), (-3.0, 2.0, 3.0)]):
        cfg["objects"].insert(3 + 5 * k, {"center": _v(*pos), "radius": 0.6, "material": {"Light": {}}})
    return cfg


def lit_scene(w=W, h=H, spp=N):
    return R.Scene.from_config(lit_config(w, h, spp))


def cover_scene(w=W, h=H, spp=COVER_N):
    return scenes.cover_scene(w, h, spp, depth=8)


def params(m, min_samples=MIN):
    return R.make_adaptive(TOL["rel_tol"], TOL["abs_tol"], samples_per_round=m, min_samples=min_samples)


_SAMPLES = {}


def oracle_samples(key, sc, lens=None):
    """Samples [0, spp) of every pixel of `sc` through `lens` (None: the pinhole) by the oracle's bulk route, once per key:
    (float32 radiance [spp, h, w, 3], uint32 rays [spp, h, w]). Prints the oracle's time."""
    if key not in _SAMPLES:
        t = time.perf_counter()
        _SAMPLES[key] = OL.render_samples(sc, lens, 0, int(sc.c.samples_per_pixel))
        print(f"[oracle] {key}: {int(sc.c.samples_per_pixel) * int(sc.c.width) * int(sc.c.height):,} samples in "
              f"{time.perf_counter() - t:.1f} s")
    return _SAMPLES[key]


def restated(key, sc, m, lens=None, rounds=None):
    """adaptive_restatement.run of `sc` (its spp is N) at m samples per round on the oracle's samples."""
    x, rays = oracle_samples(key, sc, lens)
    p = params(m)
    return A.run(x, rays, m, int(sc.c.samples_per_pixel), p.min_samples, p.abs_tol, p.rel_tol, rounds)


def assert_list_reach(want, npix, m, N, bound, what):
    """The rounds of an adaptive run reach past the trace kernel's first fill and the compaction's first tiles: a first
    round of at least 4B work ids; a later round whose list is at least 1,000 separate runs of pixels; a list that is not a
    multiple of 32; and a last round below one warp's pixels, or one that ends at N and does not fill the GPU."""
    sizes, runs, taken = want["list_sizes"], want["list_runs"], want["list_samples"]
    assert sizes[0] == npix and npix * m >= 4 * bound, (what, npix * m, 4 * bound)
    assert any(r >= 1000 for r in runs[1:]), (what, runs)
    assert any(s % 32 for s in sizes), (what, sizes)
    assert sizes[-1] < 32 or (sum(taken) == N and sizes[-1] * taken[-1] < bound), (what, sizes, taken)
    assert want["active"] == 0, what


def assert_pixel_reach(npix, bound, what):
    """An auxiliary-buffer pass or a frame group of at least 4B pixels or work ids."""
    assert npix >= 4 * bound, (what, npix, 4 * bound)


def test_the_bulk_route_is_the_per_sample_routine():
    """oracle_lens_samples through a lens of radius 0 is oracle_sample, bit for bit: the route the full-frame cases take is
    the routine the adaptive restatement was pinned with."""
    sc = lit_scene(24, 18, 4)
    x, rays = OL.render_samples(sc, None, 0, 4)
    x1, rays1 = A.render_samples(sc, 0, 4)
    assert x.shape == x1.shape == (4, 18, 24, 3)
    assert np.array_equal(x.view(np.uint32), x1.view(np.uint32))
    assert np.array_equal(rays, rays1) and rays.sum() > 4 * 18 * 24
    # past sample 0 too: the route keys each sample by its own index
    x2, rays2 = OL.render_samples(sc, R.rt_lens(), 2, 4)
    assert np.array_equal(x2.view(np.uint32), x1[2:].view(np.uint32)) and np.array_equal(rays2, rays1[2:])


@pytest.mark.parametrize("m", ROUNDS)
def test_the_adaptive_rounds_reach_past_the_first_fill(m):
    want = restated("lit", lit_scene(), m)
    assert_list_reach(want, W * H, m, N, H100_BOUND, f"lit, m = {m}")
    assert len(want["list_sizes"]) >= 4 and np.unique(want["counts"]).tolist()[0] <= MIN + m
    print(f"lit, m = {m}: lists {want['list_sizes']}, runs {want['list_runs']}")


def test_the_cover_rounds_reach_past_the_first_fill():
    want = restated("cover", cover_scene(), 8)
    assert_list_reach(want, W * H, 8, COVER_N, H100_BOUND, "cover")


def test_the_reach_fails_at_the_old_sizes():
    """Shrunk to the frames the suite compared before, every reach assertion of the full-frame cases fails."""
    w, h = OLD
    sc = lit_scene(w, h)
    x, rays = OL.render_samples(sc, None, 0, N)
    for m in ROUNDS:
        p = params(m)
        want = A.run(x, rays, m, N, p.min_samples, p.abs_tol, p.rel_tol)
        with pytest.raises(AssertionError):
            assert_list_reach(want, w * h, m, N, H100_BOUND, "old size")
    for what, npix in (("aov", 64 * 48), ("lens frames", 40 * 30 * 3 * 3)):
        with pytest.raises(AssertionError):
            assert_pixel_reach(npix, H100_BOUND, what)
