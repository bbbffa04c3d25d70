"""Closest-hit queries without a GPU: the oracle's hit_world on caller-supplied rays (tests/oracle_hit_world.cpp), which the
GPU query is held to, against the independent Python restatement of Sphere::hit folded as hit_world folds it; the t_max
argument of DESIGN.md §4.10 on the oracle; the layout of rt_rays / rt_hits; and the checks reachable without a device."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import intersect_rays as IR
import oracle_py as O
import rtb200 as R
from py_restatement import World
from rtb200 import scenes

MAX = IR.MAX


def oracle_atan2(y, x):
    """The explicit atan2 the oracle and the kernel share (mode 1)."""
    yy, xx, out = C.c_double(float(y)), C.c_double(float(x)), C.c_double()
    O.lib().oracle_atan2(C.byref(yy), C.byref(xx), C.c_uint32(1), C.c_int(1), C.byref(out))
    return out.value


def restated(world, o, d, t_max=MAX):
    """hit_world (raytracer.rs:44-59) over World.sphere_hit, in numpy float64 scalars so that x / 0 is IEEE (inf or NaN)."""
    o = tuple(np.float64(v) for v in o)
    d = tuple(np.float64(v) for v in d)
    closest, rec = np.float64(t_max), None
    with np.errstate(all="ignore"):
        for i in range(len(world.spheres)):
            h = world.sphere_hit(i, o, d, 0.001, closest)
            if h is not None:
                closest, rec = h["t"], h
    return rec


def restated_all(world, o, d):
    n = len(o)
    out = {"t": np.full(n, np.inf), "sphere": np.full(n, -1, np.int32), "point": np.zeros((n, 3)), "normal": np.zeros((n, 3)),
           "uv": np.zeros((n, 2)), "front_face": np.zeros(n, np.uint8)}
    for i in range(n):
        h = restated(world, o[i], d[i])
        if h is None:
            continue
        out["t"][i] = h["t"]; out["sphere"][i] = h["idx"]; out["point"][i] = [float(v) for v in h["point"]]
        out["normal"][i] = [float(v) for v in h["normal"]]; out["uv"][i] = [float(h["u"]), float(h["v"])]
        out["front_face"][i] = 1 if h["front"] else 0
    return out


def check_against_restatement(sc, cfg, o, d, what):
    want = restated_all(World(cfg, atan2=oracle_atan2), o, d)
    got = IR.oracle(sc, o, d)
    IR.assert_hits_equal(got, want, what)
    return got


def _cover():
    cfg = scenes._variant(scenes.cover_config(), 32, 24, 1, 4)
    return R.Scene.from_config(cfg), cfg


def test_oracle_equals_the_restatement_on_the_cover_scene():
    sc, cfg = _cover()
    rng = np.random.default_rng(1)
    sets = {"camera": IR.camera_rays(sc, 12, 9), "surface": IR.surface_rays(sc, rng, 40), "box": IR.box_rays(sc, rng, 40),
            "grazing": IR.grazing_rays(sc, rng, 24), "axis": IR.axis_rays(sc, rng, 16)}
    hits = 0
    for name, (o, d) in sets.items():
        got = check_against_restatement(sc, cfg, o, d, f"cover/{name}")
        hits += int((got["sphere"] >= 0).sum())
    o, d = IR.secondary_rays(IR.oracle(sc, *sets["camera"]), rng)
    check_against_restatement(sc, cfg, o[:60], d[:60], "cover/secondary")
    assert hits > 100   # the sets reach the spheres


def test_oracle_equals_the_restatement_on_the_test_scene():
    cfg = scenes.test_scene_config()   # 7 spheres, among them a hollow glass shell (negative radius)
    sc = R.Scene.from_config(cfg, scenes.SCENES_DIR)
    rng = np.random.default_rng(2)
    o1, d1 = IR.camera_rays(sc, 16, 12)
    o2, d2 = IR.surface_rays(sc, rng, 60)
    o3, d3 = IR.secondary_rays(IR.oracle(sc, o1, d1), rng)
    for name, (o, d) in {"camera": (o1, d1), "surface": (o2, d2), "secondary": (o3, d3)}.items():
        check_against_restatement(sc, cfg, o, d, f"test_scene/{name}")


def _odd_scene():
    """Duplicate spheres (equal roots: the lowest index wins), a sphere inside another, negative and zero radii, and tiny and
    huge ones."""
    objs = [IR.sphere((0, 0, -3), 1.0), IR.sphere((0, 0, -3), 1.0), IR.sphere((0, 0, -3), 1.0),
            IR.sphere((2, 0, -3), -0.5), IR.sphere((2, 0, -3), 0.5), IR.sphere((-2, 0, -3), 0.0),
            IR.sphere((0, 0, -3), 0.25), IR.sphere((0, 2, -3), 1e-12), IR.sphere((0, -1e6, 0), 1e6 - 0.5),
            IR.sphere((0, 3, -3), -0.0), IR.sphere((2, 0, -3), -0.5)]
    return IR.scene_of(objs)


def test_duplicates_negative_and_zero_radii_match_the_restatement():
    sc, cfg = _odd_scene()
    rng = np.random.default_rng(3)
    o = np.zeros((60, 3)); d = np.zeros((60, 3))
    targets = np.array([[0, 0, -3], [2, 0, -3], [-2, 0, -3], [0, 2, -3], [0, 3, -3], [0, -0.5, -3]], np.float64)
    for i in range(60):
        t = targets[i % len(targets)] + rng.normal(size=3) * (0.0 if i < 12 else 0.3)
        d[i] = t - o[i]
    got = check_against_restatement(sc, cfg, o, d, "odd")
    # rays straight at the duplicates' centre hit sphere 0, never 1 or 2 (equal roots: hit_world keeps the first)
    assert (got["sphere"][0:60:6] == 0).all()
    o2, d2 = IR.surface_rays(sc, rng, 40)
    check_against_restatement(sc, cfg, o2, d2, "odd/surface")


@pytest.mark.parametrize("scale", [0.0, 1e-300, 1e-160, 1e-20, 1e20, 1e160, 1e300])
def test_zero_tiny_and_huge_directions_match_the_restatement(scale):
    sc, cfg = _odd_scene()
    rng = np.random.default_rng(4)
    o, d = IR.box_rays(sc, rng, 24, box=(np.array([-3.0, -1.0, -1.0]), np.array([3.0, 1.0, 0.0])))
    d = d / np.linalg.norm(d, axis=1, keepdims=True) * scale
    check_against_restatement(sc, cfg, o, d, f"|d| = {scale}")


def test_non_finite_rays_and_spheres_match_the_restatement():
    sc, cfg = _odd_scene()
    rng = np.random.default_rng(5)
    o, d = IR.degenerate_rays(sc, rng)
    check_against_restatement(sc, cfg, o, d, "degenerate rays")
    inf, nan = math.inf, math.nan
    objs = cfg["objects"] + [IR.sphere((nan, 0, -3), 1.0), IR.sphere((0, 0, -3), nan), IR.sphere((inf, 0, 0), 1.0),
                             IR.sphere((0, 0, -5), inf), IR.sphere((1e15, 0, 0), 1e15 - 10.0)]
    sc2, cfg2 = IR.scene_of(objs)
    o2, d2 = IR.box_rays(sc2, rng, 30, box=(np.array([-3.0, -1.0, -1.0]), np.array([3.0, 1.0, 0.0])))
    check_against_restatement(sc2, cfg2, np.concatenate([o, o2]), np.concatenate([d, d2]), "non-finite spheres")


# ---- t_max (DESIGN.md §4.10): hit_world under t_max = the unbounded closest hit, kept when its root is below t_max ----
def _tmax_cases(t):
    """Per ray, the edge bounds around its unbounded root t: at it, one ulp either side, at and just below 0.001, below it,
    +inf, NaN and f64::MAX."""
    f = np.where(np.isfinite(t), t, 1.0)
    return [f, np.nextafter(f, np.inf), np.nextafter(f, -np.inf), np.full_like(f, 0.001), np.full_like(f, np.nextafter(0.001, 0.0)),
            np.full_like(f, 0.0005), np.full_like(f, 0.0), np.full_like(f, -1.0), np.full_like(f, np.inf), np.full_like(f, np.nan),
            np.full_like(f, MAX), np.full_like(f, np.nextafter(0.001, 1.0))]


def test_t_max_equals_the_unbounded_hit_filtered_by_its_root():
    rng = np.random.default_rng(6)
    sets = []
    for sc, _ in (_cover(), _odd_scene()):
        o1, d1 = IR.camera_rays(sc, 24, 18)
        o2, d2 = IR.surface_rays(sc, rng, 300)   # roots near 0.001 and t_min edges
        sets.append((sc, np.concatenate([o1, o2]), np.concatenate([d1, d2])))
    for sc, o, d in sets:
        unbounded = IR.oracle(sc, o, d)
        assert (unbounded["sphere"] >= 0).sum() > 100
        IR.assert_hits_equal(IR.oracle(sc, o, d, np.full(len(o), MAX)), unbounded, "t_max = f64::MAX")
        for k, tm in enumerate(_tmax_cases(unbounded["t"])):
            IR.assert_hits_equal(IR.oracle(sc, o, d, tm), IR.filtered(unbounded, tm), f"t_max case {k}")


def test_t_max_at_a_root_is_exclusive_on_the_restatement():
    """Sphere::hit's bound is strict: under t_max = its root the hit is gone, one ulp above it is back; the restatement
    folded under t_max agrees with the oracle."""
    sc, cfg = _odd_scene()
    world = World(cfg, atan2=oracle_atan2)
    o, d = np.zeros((6, 3)), np.array([[0, 0, -1], [2, 0, -3], [0, 2, -3], [0.1, 0.1, -1], [-2, 0, -3], [0, -0.5, -3]], np.float64)
    un = IR.oracle(sc, o, d)
    for i in range(len(o)):
        t = un["t"][i]
        if not np.isfinite(t):
            continue
        for tm, hit in ((t, False), (np.nextafter(t, np.inf), True), (np.nextafter(t, -np.inf), False)):
            h = restated(world, o[i], d[i], tm)
            got = IR.oracle(sc, o[i:i + 1], d[i:i + 1], np.array([tm]))
            assert (h is not None) == hit == (got["sphere"][0] >= 0), (i, t, tm)
            if hit:
                assert h["idx"] == got["sphere"][0] and h["t"] == got["t"][0]


# ---- the C ABI ----
def test_rays_and_hits_layout_matches_the_header(repo, tmp_path):
    assert C.sizeof(R.rt_rays) == 24 and C.sizeof(R.rt_hits) == 48
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rtb200.h"\nint main(void) {\n'
                   '    printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(rt_rays), offsetof(rt_rays, origin),\n'
                   '           offsetof(rt_rays, direction), offsetof(rt_rays, t_max), sizeof(rt_hits), offsetof(rt_hits, t),\n'
                   '           offsetof(rt_hits, sphere), offsetof(rt_hits, point), offsetof(rt_hits, normal), offsetof(rt_hits, uv),\n'
                   '           offsetof(rt_hits, front_face));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Werror", "-I", os.path.join(repo, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [C.sizeof(R.rt_rays)] + [getattr(R.rt_rays, f).offset for f, _ in R.rt_rays._fields_] + \
           [C.sizeof(R.rt_hits)] + [getattr(R.rt_hits, f).offset for f, _ in R.rt_hits._fields_]
    assert got == want == [24, 0, 8, 16, 48, 0, 8, 16, 24, 32, 40]
    assert [f for f, _ in R.rt_hits._fields_] == IR.FIELDS


def test_null_handle_is_refused_without_a_device():
    L = R.lib()
    o = np.zeros((1, 3)); d = np.ones((1, 3)); t = np.zeros(1)
    rays = R.rt_rays(o.ctypes.data, d.ctypes.data, None)
    hits = R.rt_hits(t.ctypes.data, None, None, None, None, None)
    st = R.rt_stats()
    assert L.rtb200_scene_intersect(None, C.byref(rays), 1, C.byref(hits), C.byref(st)) == -1
    assert b"handle" in L.rtb200_last_error()
    assert L.rtb200_scene_intersect_device(None, C.byref(rays), 1, C.byref(hits), None) == -1
    assert L.rtb200_scene_intersect_device(None, None, 0, None, None) == -1
    assert t[0] == 0.0
