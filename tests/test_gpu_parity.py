"""GPU parity tests: the CUDA path through the C ABI against the CPU oracle on the same seeded inputs.

Bar (north_star): per-pixel linear RGB within 1e-3 under matched RNG. What these tests actually assert is
stronger — BIT-EXACT linear f32 and RGB8 images and identical ray counts — because the kernel evaluates the
reference's f64/f32 operation order without FMA contraction; TOL documents the contractual tolerance."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from synth import base_config, mixed_config, _v

pytestmark = pytest.mark.gpu
TOL = 1e-3   # north_star tolerance on linear RGB; the assertions below use exact equality
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
V = R.vec3


def _exact(sc, opts=None):
    lin_o, img_o, st_o = O.render(sc)
    lin_g, st_g = R.render_linear(sc, opts)
    img_g, st2 = R.render_rgb8(sc, opts)
    assert float(np.abs(lin_g - lin_o).max()) <= TOL
    assert np.array_equal(lin_g, lin_o), f"linear differs: max {np.abs(lin_g - lin_o).max()}"
    assert np.array_equal(img_g, img_o)
    assert st_g["rays"] == st_o["rays"] == st2["rays"] and st_g["samples"] == st_o["samples"]
    return st_g


# ---- the reference's known-answer tests against the DEVICE routines ----------------------------------
def test_device_kats(kat):
    L = R.lib()
    k = kat["sphere_hit"]
    hit = C.c_int32(); t = C.c_double(); p = R.rt_vec3(); n = R.rt_vec3(); ff = C.c_int32()
    assert L.rtb200_probe_sphere_hit(V(k["center"]), k["radius"], V(k["origin"]), V(k["dir"]), 0.0, math.inf, C.byref(hit), C.byref(t), C.byref(p), C.byref(n), C.byref(ff)) == 0
    assert hit.value == 1 and t.value == 4.0 and p.tup() == (0.0, 0.0, -1.0) and ff.value == 1     # sphere.rs:81-88
    k = kat["refract"]; out = R.rt_vec3()
    assert L.rtb200_probe_refract(V(k["uv"]), V(k["n"]), k["eta"], C.byref(out)) == 0
    assert out.tup() == (0.0, 1.0, 0.0)                                                               # materials.rs:157-165
    r = C.c_double()
    assert L.rtb200_probe_reflectance(0.0, 1.5, C.byref(r)) == 0 and r.value == 1.0                   # materials.rs:167-174
    rgb = (C.c_float * 3)()
    assert L.rtb200_probe_sky(V([1, 0, 0]), R.RT_SKY_GRADIENT, rgb) == 0
    assert list(rgb) == [np.float32(0.75), np.float32(0.85), np.float32(1.0)]                        # raytracer.rs:167-189
    k = kat["camera_get_ray"]
    cam = R.camera_from_params(k["look_from"], k["look_at"], k["vup"], k["vfov"], k["aspect"])
    o = R.rt_vec3(); d = R.rt_vec3()
    assert L.rtb200_probe_get_ray(C.byref(cam), 0.5, 0.5, C.byref(o), C.byref(d)) == 0
    assert o.tup() == (-4.0, 4.0, 1.0)                                                                # camera.rs:105-122
    np.testing.assert_allclose(d.tup(), k["dir"], atol=1e-6, rtol=0)
    o2 = R.rt_vec3(); d2 = R.rt_vec3()
    O.lib().oracle_get_ray(C.byref(cam), 0.5, 0.5, C.byref(o2), C.byref(d2))
    assert d.tup() == d2.tup()


def test_device_sphere_hit_matches_oracle_on_random_rays():
    rng = np.random.default_rng(5)
    L = R.lib(); Lo = O.lib()
    for i in range(200):
        c = rng.uniform(-3, 3, 3); r = float(rng.uniform(0.2, 2.0)) * (1 if i % 7 else -1)
        o = rng.uniform(-4, 4, 3); d = rng.uniform(-1, 1, 3) * float(rng.uniform(0.1, 3))
        tmax = math.inf if i % 3 else float(rng.uniform(0.5, 6))
        h1 = C.c_int32(); t1 = C.c_double(); p1 = R.rt_vec3(); n1 = R.rt_vec3(); f1 = C.c_int32()
        h2 = C.c_int32(); t2 = C.c_double(); p2 = R.rt_vec3(); n2 = R.rt_vec3(); f2 = C.c_int32(); u = C.c_double(); v = C.c_double()
        assert L.rtb200_probe_sphere_hit(V(c), r, V(o), V(d), 0.001, tmax, C.byref(h1), C.byref(t1), C.byref(p1), C.byref(n1), C.byref(f1)) == 0
        Lo.oracle_sphere_hit(V(c), r, V(o), V(d), 0.001, tmax, C.byref(h2), C.byref(t2), C.byref(p2), C.byref(n2), C.byref(f2), C.byref(u), C.byref(v))
        assert h1.value == h2.value
        if h1.value:
            assert t1.value == t2.value and p1.tup() == p2.tup() and n1.tup() == n2.tup() and f1.value == f2.value


def test_device_rng_stream_is_the_oracle_stream():
    n = 2000
    for kind in (0, 1):
        a = (C.c_double * n)(); b = (C.c_double * n)()
        assert R.lib().rtb200_probe_rng(0x5EED, 123457, 77, kind, n, a) == 0
        O.lib().oracle_rng(0x5EED, 123457, 77, kind, n, b)
        assert list(a) == list(b)


def test_device_quantisation_is_the_oracle_quantisation():
    rng = np.random.default_rng(3)
    xs = np.concatenate([rng.uniform(0, 1.2, 5000), ((np.arange(0, 256) + 0.5) / 255.0) ** 2, [0.0, 1.0, 7.0, 1e-30]]).astype(np.float32)
    a = np.zeros(len(xs), np.uint8); b = np.zeros(len(xs), np.uint8)
    assert R.lib().rtb200_probe_quantise(xs.ctypes.data, len(xs), a.ctypes.data) == 0
    O.lib().oracle_quantise(xs.ctypes.data, len(xs), b.ctypes.data)
    assert np.array_equal(a, b)


# ---- images -----------------------------------------------------------------------------------------
GOLDEN = [   # (tests/golden/<name>.npz, the scene it was rendered from)
    ("cover_40x30_s4", lambda: scenes.cover_scene(40, 30, 4)),
    ("cover_64x48_s2_d3", lambda: scenes.cover_scene(64, 48, 2, depth=3)),
    ("mixed_48x36_s3", lambda: R.Scene.from_config(mixed_config(48, 36, 3, 12, seed=11), scenes.SCENES_DIR)),
]


@pytest.mark.parametrize("name,mk", GOLDEN)
def test_gpu_matches_committed_golden(name, mk):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    sc = mk()
    lin, st = R.render_linear(sc)
    img, _ = R.render_rgb8(sc)
    assert np.array_equal(lin, g["linear"]) and np.array_equal(img, g["rgb8"]) and st["rays"] == int(g["rays"])


@pytest.mark.parametrize("variant", [R.RT_VARIANT_FILTERED, R.RT_VARIANT_EXACT_F64, R.RT_VARIANT_BRUTE_FORCE])
def test_cover_scene_bit_exact(variant):
    st = _exact(scenes.cover_scene(200, 150, 8), R.make_options(variant=variant))
    if variant != R.RT_VARIANT_EXACT_F64:
        assert st["candidates"] / st["rays"] < 8.0     # the conservative f32 tests prune >98 % of the 484 sphere tests
    else:
        assert st["candidates"] == st["rays"] * 484
    if variant == R.RT_VARIANT_FILTERED:
        assert 0 < st["nodes"] / st["rays"] < 12.0 and 0 < st["clusters"] / st["rays"] < 12.0   # BVH nodes / leaves visited per ray


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_mixed_materials_bit_exact(seed):
    _exact(R.Scene.from_config(mixed_config(96, 72, 4, 20, seed=seed)))
    _exact(R.Scene.from_config(mixed_config(96, 72, 4, 20, seed=seed)), R.make_options(variant=R.RT_VARIANT_BRUTE_FORCE))


@pytest.mark.parametrize("offset", [(1.0e3, 50.0, -2.0e3), (1.0e5, 0.0, 1.0e5), (-3.0e6, 1.0e3, 7.0e6)])
def test_filter_is_sound_far_from_the_origin(offset):
    """The f32 filter must never drop a sphere the f64 test accepts, however large the coordinates."""
    sc = R.Scene.from_config(mixed_config(64, 48, 3, 12, seed=4, offset=offset))
    _exact(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
    _exact(sc, R.make_options(variant=R.RT_VARIANT_BRUTE_FORCE))


def test_black_sky_and_depth_edges():
    for depth in (0, 1, 2):
        _exact(scenes.cover_scene(48, 36, 2, depth=depth))
    cfg = mixed_config(48, 36, 2, 6, seed=9, sky="none")
    st = _exact(R.Scene.from_config(cfg))
    assert st["rays"] > 0


@pytest.mark.parametrize("n", [0, 1, 2, 3, 5])
def test_tiny_sphere_counts(n):
    objs = [{"center": _v(0.7 * i - 1.0, 0.3, 0.2 * i), "radius": 0.45, "material": [{"Lambertian": {"albedo": [0.8, 0.3, 0.3]}}, {"Metal": {"albedo": [0.8, 0.8, 0.8], "fuzz": 0.1}}, {"Glass": {"index_of_refraction": 1.5}}][i % 3]} for i in range(n)]
    _exact(R.Scene.from_config(base_config(40, 30, 3, 6, objs, look_from=(0, 1, 4), look_at=(0, 0, 0), vfov=40.0)))


def test_minimum_image_and_single_sample():
    _exact(scenes.cover_scene(2, 2, 1))
    _exact(scenes.cover_scene(3, 2, 5))


def test_batched_sample_staging_is_invisible():
    sc = scenes.cover_scene(64, 48, 16)
    a, sa = R.render_linear(sc)
    b, sb = R.render_linear(sc, R.make_options(sample_buffer_bytes=64 * 48 * 16 * 3))   # 3 samples per batch
    assert sb["batches"] > 1 and sa["batches"] == 1
    assert np.array_equal(a, b) and sa["rays"] == sb["rays"]
    _exact(sc, R.make_options(sample_buffer_bytes=64 * 48 * 16 * 5))


@pytest.mark.parametrize("world,band", [(2, 1), (3, 1), (8, 1), (4, 16), (8, 7)])
def test_row_band_shards_reassemble_to_the_single_gpu_image(world, band):
    sc = scenes.cover_scene(64, 50, 4)
    full, st = R.render_rgb8(sc)
    lin_full, _ = R.render_linear(sc)
    out = np.zeros_like(full); lin = np.zeros_like(lin_full); rays = 0
    for r in range(world):
        o = R.make_options(rank=r, world=world, band_rows=band)
        part, s = R.render_rgb8(sc, o)
        lpart, _ = R.render_linear(sc, o)
        rows = R.shard_row_indices(50, r, world, band)
        assert part.shape[0] == len(rows)
        out[rows] = part; lin[rows] = lpart; rays += s["rays"]
    assert np.array_equal(out, full) and np.array_equal(lin, lin_full) and rays == st["rays"]


def test_determinism_and_seed_sensitivity():
    sc = scenes.cover_scene(96, 72, 8)
    a, sa = R.render_linear(sc); b, sb = R.render_linear(sc)
    assert np.array_equal(a, b) and sa["rays"] == sb["rays"]
    sc.seed = 99
    c, _ = R.render_linear(sc)
    assert not np.array_equal(a, c)
    # two independent seeds agree statistically: per-channel frame means within a few sigma
    assert np.all(np.abs(a.mean(axis=(0, 1)) - c.mean(axis=(0, 1))) < 0.01)


def test_full_size_c2_against_oracle_rows_and_invariants():
    """BASELINE config C2 (cover 800x600x128, depth 50) at full size: a stripe of rows is compared with the
    oracle bit for bit, the rest through size-independent properties."""
    sc = scenes.scene("C2")
    lin, st = R.render_linear(sc)
    img, st8 = R.render_rgb8(sc)
    assert st["samples"] == 800 * 600 * 128 and st["rays"] == st8["rays"]
    assert 2.6 < st["rays"] / st["samples"] < 2.75
    ys = (0, 299, 437, 599)
    for y in ys:
        lo, io, _ = O.render(sc, y0=y, y1=y + 1)
        assert np.array_equal(lin[y], lo[y]) and np.array_equal(img[y], io[y])
    assert np.isfinite(lin).all() and lin.min() >= 0.0 and lin.max() <= 1.0
    q = np.zeros(lin.size, np.uint8)
    O.lib().oracle_quantise(np.ascontiguousarray(lin).ctypes.data, lin.size, q.ctypes.data)
    assert np.array_equal(q.reshape(img.shape), img)       # RGB8 = quantise(sqrt(linear)) everywhere
    # sharded render of the full frame == the full render
    o = R.make_options(rank=1, world=4, band_rows=1)
    part, _ = R.render_rgb8(sc, o)
    assert np.array_equal(part, img[R.shard_row_indices(600, 1, 4, 1)])


def test_resident_scene_renders_into_device_buffers():
    import torch
    sc = scenes.cover_scene(120, 90, 4)
    ref, st0 = R.render_rgb8(sc)
    rs = R.ResidentScene(sc)
    out = torch.zeros(90 * 120 * 3, dtype=torch.uint8, device="cuda")
    lin = torch.zeros(90 * 120 * 3, dtype=torch.float32, device="cuda")
    st = rs.render(out.data_ptr(), lin.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().reshape(90, 120, 3), ref) and st["rays"] == st0["rays"]
    assert st["kernel_launches"] == 2 and st["device_ms"] > 0 and st["frames"] == 1
    out.zero_()
    for _ in range(4):                     # non-blocking frame loop
        rs.render_async(out.data_ptr(), 0, 0)
    st4 = rs.wait()
    assert st4["frames"] == 4 and st4["kernel_launches"] == 8 and st4["rays"] == st0["rays"] and st4["trace_ms"] > 0
    assert np.array_equal(out.cpu().numpy().reshape(90, 120, 3), ref)
    rs.release()


@pytest.mark.parametrize("variant", [R.RT_VARIANT_FILTERED, R.RT_VARIANT_EXACT_F64, R.RT_VARIANT_BRUTE_FORCE])
def test_resident_scene_launch_shape(variant):
    """Persistent grid = every SM x the resident CTAs of the variant's kernel; the BVH path runs 3 CTAs of 80 registers."""
    import torch
    rs = R.ResidentScene(scenes.cover_scene(32, 24, 1), R.make_options(variant=variant))
    ki = rs.kernel_info()
    rs.release()
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    assert ki["grid"] == sms * ki["ctas_per_sm"] and ki["smem_mask"] == 0
    if variant == R.RT_VARIANT_FILTERED:
        assert ki["ctas_per_sm"] == 3 and ki["registers"] == 80
    else:
        assert ki["ctas_per_sm"] >= 1


def test_retired_variant_reports_an_error_not_a_wrong_image():
    cfg = mixed_config(16, 12, 1, 4, seed=1)
    with pytest.raises(R.RtError) as e:
        R.render_rgb8(R.Scene.from_config(cfg), R.make_options(variant=R.RT_VARIANT_RETIRED_LANES))
    assert e.value.code == -4


# ---- N1/N2: lights (shadow-ray recursion), textures, sky texture ---------------------------------------
def _light_cfg(n_lights, seed, sky="gradient", depth=6):
    cfg = mixed_config(80, 60, 6, depth, seed=seed, n=30, sky=sky)
    pos = [(0.0, 6.0, 0.0), (-4.0, 3.0, 5.0), (5.0, 2.5, -3.0)]
    for k in range(n_lights):
        cfg["objects"].insert(3 + 5 * k, {"center": _v(*pos[k]), "radius": 1.0 + 0.5 * k, "material": {"Light": {}}})
    return cfg


@pytest.mark.parametrize("n_lights,seed,sky,depth", [(1, 21, "gradient", 6), (3, 22, "gradient", 6), (2, 23, "none", 6), (1, 24, "none", 1), (1, 25, "gradient", 2)])
def test_lights_bit_exact(n_lights, seed, sky, depth):
    """Stochastic light test + shadow sub-paths with (max_depth 2, depth 1) semantics incl. nested light tests
    (raytracer.rs:89-114); `depth > max_depth - 2` wraps for max_depth < 2 like a release build."""
    st = _exact(R.Scene.from_config(_light_cfg(n_lights, seed, sky, depth)))
    assert st["rays"] >= st["samples"] and (depth < 2 or st["rays"] > st["samples"])


def test_reference_test_scene_c1():
    """BASELINE config C1: data/test_scene.json (2 textured spheres, metal, light, hollow glass, sky texture) at
    400x300, 16 spp, depth 8. Texel addresses go through f64::atan2 (sphere.rs:35-43), which the kernel and the oracle
    evaluate with one explicit algorithm (rtd::rt_atan2 / rto::rt_atan2), so this frame is bit-exact like the others."""
    sc = scenes.scene("C1")
    lin_o, img_o, st_o = O.render(sc)
    lin_g, st_g = R.render_linear(sc)
    img_g, _ = R.render_rgb8(sc)
    assert st_o["texture_oob"] == 0
    assert np.array_equal(lin_g, lin_o) and np.array_equal(img_g, img_o) and st_g["rays"] == st_o["rays"]


def test_device_sphere_uv_is_the_oracle_sphere_uv():
    """u_v_from_sphere_hit_point (sphere.rs:35-43) on the device vs the oracle, bit for bit, incl. the axes and poles."""
    rng = np.random.default_rng(17)
    n = 1 << 16
    hp = rng.normal(size=(n, 3)) * rng.uniform(1e-3, 1e3, size=(n, 1))
    special = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [1, 0, 1], [-1, 0, 1], [1, 0, -1], [-1, 0, -1],
                        [1e-300, 1, 1e-300], [0.0, 1, -0.0], [-0.0, 1, -1e-200], [3, 4, 1e-17], [1e-17, 4, -3]], dtype=np.float64)
    hp[: len(special)] = special
    hp = np.ascontiguousarray(hp)
    a = np.zeros((n, 2)); b = np.zeros((n, 2))
    P = C.POINTER(C.c_double)
    assert R.lib().rtb200_probe_sphere_uv(hp.ctypes.data_as(P), n, a.ctypes.data_as(P)) == 0
    O.lib().oracle_sphere_uv(hp.ctypes.data_as(P), n, b.ctypes.data_as(P))
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def _sha(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("name", ["C1", "C2", "C3S", "C4S", "C5S"])
def test_golden_frames_of_the_baseline_configs(name):
    """The BASELINE configs against the ORACLE's committed frame hashes (tests/golden/frames.json, made by
    tests/golden/make_frames.py): full-size C2 (800x600x128), and C3 / C4 (all 10,000 spheres) / C5 at the same scene, 16:9
    aspect and depth with samples (C4: size) reduced to what the CPU oracle finishes. RGB8 and linear f32 frames and the ray
    count must be identical."""
    import json
    with open(os.path.join(GOLD, "frames.json")) as f:
        g = json.load(f)[name]
    sc = scenes.scene(name)
    assert (sc.c.width, sc.c.height, sc.c.samples_per_pixel, sc.c.max_depth, sc.n_spheres) == (g["width"], g["height"], g["samples_per_pixel"], g["max_depth"], g["n_spheres"])
    img, st = R.render_rgb8(sc)
    lin, st2 = R.render_linear(sc)
    assert st["rays"] == st2["rays"] == g["rays"] and st["samples"] == g["samples"]
    assert _sha(img) == g["sha256_rgb8"]
    assert _sha(lin) == g["sha256_linear_f32"]


def test_too_many_lights_is_refused():
    cfg = mixed_config(16, 12, 1, 4, seed=1)
    for k in range(10):
        cfg["objects"].append({"center": _v(k, 5, 0), "radius": 0.3, "material": {"Light": {}}})
    with pytest.raises(R.RtError) as e:
        R.render_rgb8(R.Scene.from_config(cfg))
    assert e.value.code == -4


# ---- N4: two-level culling on the large config ---------------------------------------------------------------
def test_rtiow_10k_spheres_bit_exact():
    """BASELINE config C4's scene (seeded restatement of config.rs:149-226 on a 100x100 grid, 10,000 spheres) at a
    size the oracle finishes in seconds. The hierarchy (~300 KB) does not fit shared memory next to the ray pool, so this
    also covers the path that reads nodes and leaves through L1/L2."""
    cfg = scenes._variant(scenes.rtiow_config(50), 128, 72, 3, 50)
    sc = R.Scene.from_config(cfg)
    st = _exact(sc)
    assert sc.n_spheres > 9900 and st["candidates"] / st["rays"] < 8.0 and 0 < st["clusters"] / st["rays"] < 16.0 and st["nodes"] / st["rays"] < 24.0
    _exact(sc, R.make_options(variant=R.RT_VARIANT_BRUTE_FORCE))


def test_two_level_equals_brute_force_on_awkward_cluster_shapes():
    """Clusters with 1..4 members, several radius classes, coincident spheres, zero and negative radii."""
    rng = np.random.default_rng(7)
    objs = []
    for i in range(75):
        r = float(rng.choice([0.05, 0.11, 0.3, 0.31, 0.9, 2.5])) * (-1.0 if i % 11 == 0 else 1.0)
        m = [{"Lambertian": {"albedo": [0.7, 0.6, 0.5]}}, {"Metal": {"albedo": [0.9, 0.9, 0.9], "fuzz": 0.05}}, {"Glass": {"index_of_refraction": 1.5}}][i % 3]
        objs.append({"center": _v(*rng.uniform(-5, 5, 3)), "radius": r, "material": m})
    objs.append({"center": _v(0, 0, 0), "radius": 0.0, "material": {"Lambertian": {"albedo": [1, 0, 0]}}})
    objs += [dict(objs[5]), dict(objs[5])]   # three coincident copies: the first index must win
    sc = R.Scene.from_config(base_config(72, 54, 3, 10, objs, look_from=(9, 3, 7), look_at=(0, 0, 0), vfov=50.0))
    a, sa = R.render_linear(sc)
    b, sb = R.render_linear(sc, R.make_options(variant=R.RT_VARIANT_BRUTE_FORCE))
    assert np.array_equal(a, b) and sa["rays"] == sb["rays"] and sa["clusters"] > 0 and sb["clusters"] == 0
    _exact(sc)


def test_100k_spheres_render_and_match_the_oracle():
    """Ten times the largest BASELINE scene: the hierarchy is sub-linear, nothing is refused (ABI 1 stopped at ~25 k spheres)."""
    cfg = scenes._variant(scenes.rtiow_config(158), 96, 54, 2, 12)
    sc = R.Scene.from_config(cfg)
    assert sc.n_spheres > 99000
    st = _exact(sc)
    assert st["nodes"] / st["rays"] < 40.0 and st["candidates"] / st["rays"] < 8.0


def test_spheres_outside_the_f32_frame_are_tested_for_every_ray():
    """Non-finite / astronomically distant spheres cannot live in the recentred f32 frame: they go to the always-list and are
    tested in f64 for every ray, like hit_world does."""
    cfg = mixed_config(48, 36, 2, 6, seed=5, n=12)
    cfg["objects"].insert(4, {"center": _v(-2e15 - 8.0, 0, 0), "radius": 2e15, "material": {"Lambertian": {"albedo": [0.3, 0.6, 0.9]}}})   # a wall at x = -8, behind the scene
    cfg["objects"].insert(7, {"center": _v(float("inf"), 0, 0), "radius": 1.0, "material": {"Metal": {"albedo": [0.9, 0.9, 0.9], "fuzz": 0.0}}})   # never hit, never in the tree
    sc = R.Scene.from_config(cfg)
    assert len(R.bvh_records(sc)["always"]) == 2
    lin_o, _, st_o = O.render(sc)
    assert np.isfinite(lin_o).all() and st_o["hits"][R.RT_LAMBERTIAN] > 0
    _exact(sc)


def test_one_process_multi_gpu_entry_point_matches_the_single_gpu_frame():
    """rtb200_render_rgb8_multi: with one visible device it degenerates to the single-GPU path; with G devices the row bands are
    dealt round-robin and the assembled frame is bit-identical (also for band sizes that leave a partial last band)."""
    sc = scenes.cover_scene(96, 70, 4)
    ref, st0 = R.render_rgb8(sc)
    n = R.device_count()
    for g in sorted({1, min(2, n), n}):
        for band in (1, 16):
            img, st = R.render_rgb8_multi(sc, g, R.make_options(band_rows=band))
            bands = (70 + band - 1) // band                     # a device needs at least one band
            assert np.array_equal(img, ref) and st["rays"] == st0["rays"] and st["gpus_used"] == min(g, n, bands)


def test_plain_c_host_drives_the_boundary_like_the_rust_shim(tmp_path, repo):
    """tests/abi_harness.c = the call sequence of integration/rust/render_replacement.rs in C11, built with gcc against
    librtb200.so (no Python, no torch in that process). Its frame must equal the Python host's byte for byte."""
    import shutil
    import struct
    import subprocess
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler on this box")
    libdir = os.path.join(repo, "rust-raytracer_b200")
    exe = tmp_path / "abi_harness"
    subprocess.check_call([cc, "-std=c11", "-O1", "-Wall", "-I", os.path.join(repo, "include"), os.path.join(repo, "tests", "abi_harness.c"),
                           "-L", libdir, "-lrtb200", f"-Wl,-rpath,{libdir}", "-o", str(exe)])
    sc = scenes.cover_scene(96, 72, 4, depth=12)
    blob = struct.pack("<4I", sc.c.width, sc.c.height, sc.c.samples_per_pixel, sc.c.max_depth) + bytes(sc.c.camera) + struct.pack("<2I", sc.c.sky.mode, sc.n_spheres)
    blob += bytes(C.string_at(C.addressof(sc._spheres), C.sizeof(R.rt_sphere) * sc.n_spheres))
    (tmp_path / "scene.bin").write_bytes(blob)
    ref, st0 = R.render_rgb8(sc)
    for n_gpus in (1, 0):
        r = subprocess.run([str(exe), str(tmp_path / "scene.bin"), str(tmp_path / "out.rgb"), str(n_gpus)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        assert r.stdout.startswith("Frame time: ") and f"rays={st0['rays']} " in r.stdout
        frame = np.frombuffer((tmp_path / "out.rgb").read_bytes(), np.uint8).reshape(72, 96, 3)
        assert np.array_equal(frame, ref)
