"""The full-frame cases of tests/test_gpu_full_frames.py without a GPU (DESIGN.md §3, "At frame sizes that fill the GPU"): the
scenes, parameters and reach rules they share, the oracle's bulk per-sample route they compare with, held to the per-sample
routine of the adaptive restatement, and the reach of the adaptive rounds, asserted on the restatement alone against the
bound of a 132-SM H100 so that a change of parameters cannot quietly drop it.

Reach: a case is big enough to leave the trace kernel's first fill of its slots, or an auxiliary-buffer warp's first chunk.
The bound B = sm_count x max_threads_per_multi_processor caps both the resident trace slots (CTAs of 256 slots) and the
resident query threads, whatever the occupancy, so 4B work ids (or pixels) take at least four fills (or passes).

LEDGER names, for each of the 36 trace kernels rt_wavefront_kernel<MODE, LIGHTS, QUEUE>, the GPU case that holds it to the
oracle at 4B work ids or more in one launch."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import adaptive_restatement as A
import denoise_var_restatement as V
import intersect_rays as IR
import oracle_lens as OL
import oracle_trace_rays as OT
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
FRAME_SPP = 8              # the pinhole frames: 640 x 360 x 8, 1.84 M work ids a frame
SPLIT_DEPTH = 3            # frame 1's max_depth when it leaves its group
FRAME_WORK = W * H * FRAME_SPP
# 64-bit keys whose high word is nonzero and differs from the low word, one per frame
FRAME_SEEDS = (0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F)
RAYS_N, RAYS_SPP = 300_001, 4   # Q_RAYS: n is not a multiple of 32 and ray i % n wraps inside a warp
RAYS_KW = dict(sample0=3, stream0=7, seed=0xD6E8FEB86659FD93)
LENS_FRAMES = (960, 540, 4)    # four lens frames of this size in one launch group
GROUP_W, GROUP_SPP = 1024, 32  # frames at the group bound: 1024 x 512 x 32 = 2^24 work ids
GROUP_MAX_FRAME_WORK = 1 << 24  # kGroupMaxFrameWork of csrc/rtb200_api_render.cu
DEFAULT_CAP = 1 << 30           # the default sample-buffer cap, bytes


def lit_config(w=W, h=H, spp=N, sky="gradient"):
    """test_gpu_adaptive's mixed_2_lights at any size: the 30-sphere mixed scene with two lights."""
    cfg = mixed_config(w, h, spp, 8, seed=7, n=30, sky=sky)
    for k, pos in enumerate([(0.0, 3.0, 0.0), (-3.0, 2.0, 3.0)]):
        cfg["objects"].insert(3 + 5 * k, {"center": _v(*pos), "radius": 0.6, "material": {"Light": {}}})
    return cfg


def unlit_config(w=W, h=H, spp=N):
    """lit_config without its two lights: the same scene through the trace kernels of LIGHTS = false."""
    cfg = lit_config(w, h, spp)
    cfg["objects"] = [o for o in cfg["objects"] if "Light" not in o["material"]]
    return cfg


def lit_scene(w=W, h=H, spp=N):
    return R.Scene.from_config(lit_config(w, h, spp))


def full_scene(name, w=W, h=H, spp=N):
    """The "lit" or "unlit" scene."""
    return R.Scene.from_config((lit_config if name == "lit" else unlit_config)(w, h, spp))


def full_frames(sc):
    """Two frames of `sc` with their own cameras and 64-bit keys."""
    return [R.make_frame(sc, seed=FRAME_SEEDS[0]),
            R.make_frame(sc, look_from=[-9.0, 2.5, 7.0], look_at=[0.0, 0.5, 0.0], seed=FRAME_SEEDS[1])]


def with_depth(f, depth):
    return R.rt_frame(f.camera, f.seed, depth, 0)


def view_of(sc, f):
    """`sc` with frame f's camera, key and max_depth."""
    v = R.Scene.edited(sc)
    v.c.camera = f.camera; v.seed = f.seed; v.c.max_depth = f.max_depth
    return v


def sum_frame(x, rays):
    """The one-shot render of the per-sample radiances x [spp, h, w, 3] (f32 sums in sample order, times 1.0f / spp) and
    the variance of its means: {linear, rgb8, rays, variance}."""
    S = np.zeros(x.shape[1:], np.float32)
    for s in range(len(x)):
        S = S + x[s]
    lin, img = A.resolve(np.full(x.shape[1:3], len(x), np.uint32), S)
    return dict(linear=lin, rgb8=img, rays=int(rays.sum(dtype=np.uint64)), variance=V.render_variance(x))


def frame_want(name, k, depth=None):
    """Frame k of full_frames on the `name` scene at FRAME_SPP (at `depth`, when given), from the oracle's samples."""
    sc = full_scene(name, spp=FRAME_SPP)
    f = full_frames(sc)[k]
    if depth is not None:
        f = with_depth(f, depth)
    return sum_frame(*oracle_samples(f"frame_{name}_{k}_{f.max_depth}", view_of(sc, f)))


def full_rays():
    """RAYS_N rays of the lit scene's families: its camera, from sphere surfaces, from the box of its centres, grazing its
    spheres, and toward its lights (which the unlit scene has removed)."""
    sc = lit_scene()
    rng = np.random.default_rng(80)
    c, r = IR.spheres_of(sc)
    lights = np.array([i for i in range(sc.n_spheres) if sc._spheres[i].kind == R.RT_LIGHT])
    lo, _ = IR.box_rays(sc, rng, 60_001)
    j = lights[rng.integers(0, len(lights), size=len(lo))]
    toward = (lo, c[j] - lo + rng.normal(size=lo.shape) * 0.05 * r[j][:, None])
    sets = [IR.camera_rays(sc, 400, 225), IR.surface_rays(sc, rng, 60_000), IR.box_rays(sc, rng, 60_000),
            IR.grazing_rays(sc, rng, 30_000), toward]
    o, d = np.concatenate([s[0] for s in sets]), np.concatenate([s[1] for s in sets])
    assert len(o) == RAYS_N
    return o, d


_RAYS = {}


def rays_want(name):
    """oracle_trace_rays of full_rays on the `name` scene, RAYS_SPP samples under RAYS_KW, once per scene."""
    if name not in _RAYS:
        t = time.perf_counter()
        _RAYS[name] = OT.trace_rays(full_scene(name), *full_rays(), RAYS_SPP, **RAYS_KW)
        print(f"[oracle] rays {name}: {RAYS_N * RAYS_SPP:,} samples in {time.perf_counter() - t:.1f} s")
    return _RAYS[name]


def frame_groups(depths, frame_work, cap=DEFAULT_CAP):
    """The launch groups of frames of these max_depths (frame_groups of csrc/rtb200_api_render.cu): their sizes."""
    groups, i = [], 0
    while i < len(depths):
        F = 1
        if depths[i] != 0 and frame_work <= GROUP_MAX_FRAME_WORK:
            while (i + F < len(depths) and depths[i + F] == depths[i] and (F + 1) * frame_work < 1 << 31
                   and (F + 1) * frame_work * 16 <= cap):
                F += 1
        groups.append(F)
        i += F
    return groups


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
    for what, npix in (("aov", 64 * 48), ("lens frames", 40 * 30 * 3 * 3), ("pinhole frames", 64 * 48 * 4 * 8),
                       ("trace_rays", 100_000 * 2)):
        with pytest.raises(AssertionError):
            assert_pixel_reach(npix, H100_BOUND, what)


def test_the_lit_and_unlit_scenes_differ_only_by_their_lights():
    lit, unlit = full_scene("lit", 24, 18, 1), full_scene("unlit", 24, 18, 1)
    kinds = [lit._spheres[i].kind for i in range(lit.n_spheres)]
    assert kinds.count(R.RT_LIGHT) == 2 and unlit.n_spheres == lit.n_spheres - 2
    assert not any(unlit._spheres[i].kind == R.RT_LIGHT for i in range(unlit.n_spheres))
    assert not any(cover_scene(24, 18)._spheres[i].kind == R.RT_LIGHT for i in range(cover_scene(24, 18).n_spheres))
    for s in FRAME_SEEDS + (RAYS_KW["seed"],):
        assert s >> 32 and s >> 32 != s & 0xFFFFFFFF, hex(s)
    f0, f1 = full_frames(lit)
    assert f0.seed != f1.seed and f0.camera.origin.tup() != f1.camera.origin.tup()


def test_the_rays_are_the_families_they_name():
    o, d = full_rays()
    assert o.shape == d.shape == (RAYS_N, 3) and RAYS_N % 32 and RAYS_SPP >= 2
    assert np.isfinite(o).all() and np.isfinite(d).all() and (np.abs(d).sum(axis=1) > 0).all()
    assert RAYS_KW["sample0"] and RAYS_KW["stream0"]


def test_frame_groups_at_the_frame_work_bound():
    """The launch groups the GPU cases assert, restated from the library's rule: frames of exactly kGroupMaxFrameWork
    samples group, one row more does not, and at the default cap four such frames fill a group."""
    at, over = GROUP_W * 512 * GROUP_SPP, GROUP_W * 513 * GROUP_SPP
    assert at == GROUP_MAX_FRAME_WORK < over
    assert frame_groups([8, 8], at) == [2] and frame_groups([8, 8], over) == [1, 1]
    assert frame_groups([8] * 5, at) == [4, 1]
    assert frame_groups([8, 8], FRAME_WORK) == [2] and frame_groups([8, SPLIT_DEPTH], FRAME_WORK) == [1, 1]
    assert frame_groups([8, 0, 0, 8], FRAME_WORK) == [1, 1, 1, 1]
    assert frame_groups([8] * 3, at, cap=3 * at * 16 - 1) == [2, 1]


# ---- the ledger: every trace kernel, held to the oracle at 4B work ids or more in one launch ---------------------------------

GPU = "tests/test_gpu_full_frames.py::"
LENS_FRAME_WORK = 4 * LENS_FRAMES[0] * LENS_FRAMES[1] * LENS_FRAMES[2]
# (queue, mode, lights) -> (test node, work ids in one launch of that kernel)
LEDGER = {
    ("Q_SINGLE", "tree", False): (GPU + "test_single_frame_at_scale[tree-unlit]", FRAME_WORK),
    ("Q_SINGLE", "tree", True): (GPU + "test_single_frame_at_scale[tree-lit]", FRAME_WORK),
    ("Q_SINGLE", "exact_f64", False): (GPU + "test_single_frame_at_scale[exact_f64-unlit]", FRAME_WORK),
    ("Q_SINGLE", "exact_f64", True): (GPU + "test_single_frame_at_scale[exact_f64-lit]", FRAME_WORK),
    ("Q_SINGLE", "brute_force", False): (GPU + "test_single_frame_at_scale[brute_force-unlit]", FRAME_WORK),
    ("Q_SINGLE", "brute_force", True): (GPU + "test_single_frame_at_scale[brute_force-lit]", FRAME_WORK),
    ("Q_FRAMES", "tree", False): (GPU + "test_frame_group_at_scale[tree-unlit]", 2 * FRAME_WORK),
    ("Q_FRAMES", "tree", True): (GPU + "test_frame_group_at_scale[tree-lit]", 2 * FRAME_WORK),
    ("Q_FRAMES", "exact_f64", False): (GPU + "test_frame_group_at_scale[exact_f64-unlit]", 2 * FRAME_WORK),
    ("Q_FRAMES", "exact_f64", True): (GPU + "test_frame_group_at_scale[exact_f64-lit]", 2 * FRAME_WORK),
    ("Q_FRAMES", "brute_force", False): (GPU + "test_frame_group_at_scale[brute_force-unlit]", 2 * FRAME_WORK),
    ("Q_FRAMES", "brute_force", True): (GPU + "test_frame_group_at_scale[brute_force-lit]", 2 * FRAME_WORK),
    ("Q_RAYS", "tree", False): (GPU + "test_trace_rays_at_scale[tree-unlit]", RAYS_N * RAYS_SPP),
    ("Q_RAYS", "tree", True): (GPU + "test_trace_rays_at_scale[tree-lit]", RAYS_N * RAYS_SPP),
    ("Q_RAYS", "exact_f64", False): (GPU + "test_trace_rays_at_scale[exact_f64-unlit]", RAYS_N * RAYS_SPP),
    ("Q_RAYS", "exact_f64", True): (GPU + "test_trace_rays_at_scale[exact_f64-lit]", RAYS_N * RAYS_SPP),
    ("Q_RAYS", "brute_force", False): (GPU + "test_trace_rays_at_scale[brute_force-unlit]", RAYS_N * RAYS_SPP),
    ("Q_RAYS", "brute_force", True): (GPU + "test_trace_rays_at_scale[brute_force-lit]", RAYS_N * RAYS_SPP),
    ("Q_LIST", "tree", False): (GPU + "test_adaptive_cover_scene_at_scale", W * H * 8),
    ("Q_LIST", "tree", True): (GPU + "test_adaptive_rounds_at_scale[tree-8]", W * H * 8),
    ("Q_LIST", "exact_f64", False): (GPU + "test_adaptive_cover_scene_validation_modes_at_scale[exact_f64]", W * H * 8),
    ("Q_LIST", "exact_f64", True): (GPU + "test_adaptive_rounds_at_scale[exact_f64-8]", W * H * 8),
    ("Q_LIST", "brute_force", False): (GPU + "test_adaptive_cover_scene_validation_modes_at_scale[brute_force]", W * H * 8),
    ("Q_LIST", "brute_force", True): (GPU + "test_adaptive_rounds_at_scale[brute_force-8]", W * H * 8),
    ("Q_LIST_LENS", "tree", False): (GPU + "test_adaptive_lens_rounds_unlit_at_scale[tree-8]", W * H * 8),
    ("Q_LIST_LENS", "tree", True): (GPU + "test_adaptive_lens_rounds_at_scale[tree-8]", W * H * 8),
    ("Q_LIST_LENS", "exact_f64", False): (GPU + "test_adaptive_lens_rounds_unlit_at_scale[exact_f64-8]", W * H * 8),
    ("Q_LIST_LENS", "exact_f64", True): (GPU + "test_adaptive_lens_rounds_at_scale[exact_f64-8]", W * H * 8),
    ("Q_LIST_LENS", "brute_force", False): (GPU + "test_adaptive_lens_rounds_unlit_at_scale[brute_force-8]", W * H * 8),
    ("Q_LIST_LENS", "brute_force", True): (GPU + "test_adaptive_lens_rounds_at_scale[brute_force-8]", W * H * 8),
    ("Q_FRAMES_LENS", "tree", False): (GPU + "test_lens_frames_every_mode_and_scene_at_scale[tree-unlit]", LENS_FRAME_WORK),
    ("Q_FRAMES_LENS", "tree", True): (GPU + "test_lens_frames_at_scale", LENS_FRAME_WORK),
    ("Q_FRAMES_LENS", "exact_f64", False): (GPU + "test_lens_frames_every_mode_and_scene_at_scale[exact_f64-unlit]", LENS_FRAME_WORK),
    ("Q_FRAMES_LENS", "exact_f64", True): (GPU + "test_lens_frames_every_mode_and_scene_at_scale[exact_f64-lit]", LENS_FRAME_WORK),
    ("Q_FRAMES_LENS", "brute_force", False): (GPU + "test_lens_frames_every_mode_and_scene_at_scale[brute_force-unlit]", LENS_FRAME_WORK),
    ("Q_FRAMES_LENS", "brute_force", True): (GPU + "test_lens_frames_every_mode_and_scene_at_scale[brute_force-lit]", LENS_FRAME_WORK),
}
QUEUES = ("Q_SINGLE", "Q_FRAMES", "Q_RAYS", "Q_LIST", "Q_LIST_LENS", "Q_FRAMES_LENS")   # csrc/rtb200_wavefront.cu's dispatch
MODES = ("tree", "exact_f64", "brute_force")


def test_the_ledger_holds_every_trace_kernel_past_its_first_fill():
    assert set(LEDGER) == {(q, m, lights) for q in QUEUES for m in MODES for lights in (False, True)}
    assert len(LEDGER) == 36
    for cell, (node, work) in LEDGER.items():
        assert work >= 4 * H100_BOUND, (cell, node, work, 4 * H100_BOUND)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    files = sorted({node.split("::")[0] for node, _ in LEDGER.values()})
    r = subprocess.run([sys.executable, "-m", "pytest", "--collect-only", "-q", "-p", "no:cacheprovider", *files],
                       capture_output=True, text=True, cwd=root, timeout=600)
    collected = set(r.stdout.split())
    missing = [node for node, _ in LEDGER.values() if node not in collected]
    assert not missing, (missing, r.stdout[-2000:], r.stderr[-2000:])
