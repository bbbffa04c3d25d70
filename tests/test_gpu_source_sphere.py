"""The source-sphere certificate on the GPU: the BVH path leaves the sphere a ray starts on out of its exact tests when a
cheap f64 certificate proves that the test would reject it (DESIGN.md §4.2). The validation variants do not use the
certificate, so all three must still agree bit for bit, on scenes built to provoke self-intersection ("acne"): tiny and
huge radii far from the origin, cameras grazing a surface, hollow glass and lights."""
import numpy as np
import pytest

import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from synth import base_config, mixed_config, _v

pytestmark = pytest.mark.gpu

VARIANTS = [R.RT_VARIANT_FILTERED, R.RT_VARIANT_BRUTE_FORCE, R.RT_VARIANT_EXACT_F64]


def _lamb(x):
    return {"Lambertian": {"albedo": [x, x, x]}}


def _far_sizes_cfg(offset, seed):
    """A huge ground sphere, tiny and mid-size spheres on it, a hollow glass shell; everything translated by `offset`."""
    rng = np.random.default_rng(seed)
    ox, oy, oz = offset
    objs = [{"center": _v(ox, oy - 1.0e5, oz), "radius": 1.0e5, "material": _lamb(0.6)}]
    for _ in range(40):
        r = float(10.0 ** rng.uniform(-3.0, -0.3))
        c = _v(ox + rng.uniform(-3, 3), oy + r * rng.uniform(0.9, 1.1), oz + rng.uniform(-3, 3))
        k = rng.uniform()
        m = _lamb(float(np.float32(rng.uniform(0.2, 0.9)))) if k < 0.6 else (
            {"Metal": {"albedo": [0.8, 0.7, 0.6], "fuzz": float(rng.uniform(0, 0.3))}} if k < 0.85 else {"Glass": {"index_of_refraction": 1.5}})
        objs.append({"center": c, "radius": r, "material": m})
    objs.append({"center": _v(ox, oy + 1.0, oz), "radius": 1.0, "material": {"Glass": {"index_of_refraction": 1.5}}})
    objs.append({"center": _v(ox, oy + 1.0, oz), "radius": -0.95, "material": {"Glass": {"index_of_refraction": 1.5}}})
    return base_config(48, 36, 4, 24, objs, look_from=(ox + 6.0, oy + 1.5, oz + 4.0), look_at=(ox, oy + 0.3, oz))


def _grazing_cfg():
    """The camera sits just above a radius-1000 ground and looks along it: primary and secondary rays graze the surface."""
    objs = [{"center": _v(0.0, -1000.0, 0.0), "radius": 1000.0, "material": {"Metal": {"albedo": [0.9, 0.9, 0.9], "fuzz": 0.05}}},
            {"center": _v(0.0, 0.3, -6.0), "radius": 0.3, "material": _lamb(0.7)},
            {"center": _v(1.0, 1e-3, -3.0), "radius": 1e-3, "material": _lamb(0.4)},
            {"center": _v(-1.0, 0.5, -4.0), "radius": 0.5, "material": {"Glass": {"index_of_refraction": 1.33}}}]
    return base_config(48, 36, 4, 30, objs, look_from=(0.0, 1e-3, 0.0), look_at=(0.0, 1e-3, -10.0), vfov=30.0)


def _lights_cfg():
    cfg = mixed_config(48, 36, 4, 8, seed=31, n=30)
    cfg["objects"].insert(3, {"center": _v(0.0, 5.0, 0.0), "radius": 1.0, "material": {"Light": {}}})
    cfg["objects"].insert(9, {"center": _v(-3.0, 2.0, 4.0), "radius": 0.5, "material": {"Light": {}}})
    return cfg


CASES = {
    "far_1e6": lambda: _far_sizes_cfg((1.0e6, -2.0e5, 1.0e6), 5),
    "far_7e6": lambda: _far_sizes_cfg((-7.0e6, 3.0e3, 7.0e6), 6),
    "grazing": _grazing_cfg,
    "hollow_glass_and_lights": _lights_cfg,
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_tree_brute_and_exact_agree_on_acne_scenes(name):
    sc = R.Scene.from_config(CASES[name]())
    out = []
    for v in VARIANTS:
        opts = R.make_options(variant=v)
        lin, st = R.render_linear(sc, opts)
        img, st2 = R.render_rgb8(sc, opts)
        assert st["rays"] == st2["rays"]
        out.append((lin, img, st))
    for lin, img, st in out[1:]:
        assert np.array_equal(lin, out[0][0]) and np.array_equal(img, out[0][1]) and st["rays"] == out[0][2]["rays"]
    lin_o, img_o, st_o = O.render(sc)                                      # and all of them render the oracle's frame
    assert np.array_equal(out[0][0], lin_o) and np.array_equal(out[0][1], img_o) and out[0][2]["rays"] == st_o["rays"]
    assert out[0][2]["rays"] > out[0][2]["samples"]                        # secondary rays were traced


def test_reduced_c2_fewer_candidates_same_rays():
    """On the cover scene about a third of the exact tests were the sphere a ray leaves; with the certificate the BVH path
    runs about 1.2 exact tests per ray instead of 1.64, and renders the oracle's frame and ray count."""
    sc = scenes.cover_scene(160, 120, 8)
    lin_o, img_o, st_o = O.render(sc)
    lin, st = R.render_linear(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
    assert np.array_equal(lin, lin_o) and st["rays"] == st_o["rays"]
    assert st["candidates"] / st["rays"] < 1.3, st["candidates"] / st["rays"]
