"""The GPU at the exact-equality edges of tests/exact_edges.py, bit for bit against the oracle: tangent rays (disc == 0, d·n
== 0) at every material, roots exactly at t_min, exact ties between different spheres (in different leaves, and with one
member on the always-list), the refraction limit fl(ratio·sin_theta) == 1 and the cos clamp. Each case's certificate and the
oracle's decisions are checked without a GPU in tests/test_exact_edges_cpu.py; here every variant, on the handle as uploaded
and after rebuild(), answers intersect and occluded like hit_world (unbounded, and bounded at each hit's root and the next
double), traces the rays like oracle_trace_rays at several sample counts and max_depth 1, 2 and 50, with 0 and 2 lights,
and the device's Sphere::hit probe answers like the oracle's. The stress builds run the same queries through
tests/exact_edges_worker.py. NaN follows the rule of tests/test_gpu_shading_edges.py."""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import exact_edges as E
import exact_edges_worker as EW
import intersect_rays as IR
import oracle_py as O
import oracle_trace_rays as OT
import rtb200 as R
from test_exact_edges_cpu import CASES, NAMES, leaf_of, scene
from test_gpu_intersect import BRUTE, EXACT, FILTERED, REPO, STRESS, query
from test_gpu_occlusion import assert_occluded_equal, occluded
from test_gpu_shading_edges import assert_frames_match
from test_gpu_trace_rays import check as check_trace

pytestmark = pytest.mark.gpu
VARIANTS = {"filtered": FILTERED, "brute_force": BRUTE, "exact_f64": EXACT}
STATES = ("uploaded", "rebuilt")
DEPTHS = (1, 2, 50)
SAMPLES = (1, 4)
E5_COPIES, E5_SAMPLES = 64, 16   # an unclamped cos_theta changes the reflect/refract draw of roughly 0.5 % of E5's samples


def handle(sc, variant, state):
    rs = R.ResidentScene(sc, R.make_options(variant=variant))
    if state == "rebuilt":
        rs.rebuild()
    return rs


def check_queries(rs, sc, case, un, what):
    """intersect and occluded: unbounded, and with t_max at each ray's root (its hit is rejected) and at the next double."""
    o, d = case.o, case.d
    IR.assert_hits_equal(query(rs, o, d), un, what + "/unbounded")
    assert_occluded_equal(occluded(rs, o, d), (un["sphere"] >= 0).astype(np.uint8), what + "/occluded")
    t = np.where(un["sphere"] >= 0, un["t"], 1.0)
    for tag, tm in (("t_max = root", t), ("t_max = next(root)", np.nextafter(t, np.inf))):
        want = IR.oracle(sc, o, d, tm)
        IR.assert_hits_equal(query(rs, o, d, tm), want, f"{what}/{tag}")
        assert_occluded_equal(occluded(rs, o, d, tm), (want["sphere"] >= 0).astype(np.uint8), f"{what}/{tag}/occluded")


def check_topology(rs, case, what):
    """The tied pairs' places in the hierarchy the FILTERED variant traverses."""
    top = rs.topology()
    always = set(int(v) for v in top["always"])
    if case.name.startswith("E3_leaves"):
        assert not always and leaf_of(top["leaf_id"], 0, rs.n) != leaf_of(top["leaf_id"], 1, rs.n), what
    elif case.name.startswith("E3_always"):
        a = E.always_member(case)
        assert always == {a}, (what, always)
        leaf_of(top["leaf_id"], 1 - a, rs.n)


@pytest.mark.parametrize("name", NAMES)
def test_every_variant_matches_the_oracle_on_the_exact_edges(name):
    case = CASES[name]
    o, d = case.o, case.d
    if name.startswith("E5"):     # many samples of each ray, each copy on a stream of its own
        o, d = np.repeat(o, E5_COPIES, axis=0), np.repeat(d, E5_COPIES, axis=0)
    for n_lights in (0, E.LIGHTS):
        sc = scene(case, n_lights)
        un = IR.oracle(sc, case.o, case.d)
        assert [int(s) for s in un["sphere"]] == [w["sphere"] for w in case.want], name   # the certified decisions
        for vname, v in VARIANTS.items():
            for state in STATES:
                what = f"{name}/lights={n_lights}/{vname}/{state}"
                rs = handle(sc, v, state)
                try:
                    check_queries(rs, sc, case, un, what)
                    if v == FILTERED:
                        check_topology(rs, case, what)
                    for depth in DEPTHS:
                        for samples in ((E5_SAMPLES,) if name.startswith("E5") else SAMPLES):
                            check_trace(rs, sc, o, d, f"{what}/depth={depth}/samples={samples}", samples=samples, max_depth=depth)
                finally:
                    rs.release()


@pytest.mark.parametrize("name", NAMES)
def test_the_device_sphere_hit_probe_matches_the_oracle(name):
    """rtb200_probe_sphere_hit (the device's Sphere::hit) against oracle_sphere_hit for every ray and its target sphere."""
    case = CASES[name]
    L, Lo, V = R.lib(), O.lib(), R.vec3
    for i, (o, d, k) in enumerate(zip(case.o, case.d, case.target)):
        c, r = case.sphere_of(k)
        h1 = C.c_int32(); t1 = C.c_double(); p1 = R.rt_vec3(); n1 = R.rt_vec3(); f1 = C.c_int32()
        h2 = C.c_int32(); t2 = C.c_double(); p2 = R.rt_vec3(); n2 = R.rt_vec3(); f2 = C.c_int32(); u = C.c_double(); v = C.c_double()
        assert L.rtb200_probe_sphere_hit(V(c), r, V(o), V(d), E.T_MIN, math.inf, C.byref(h1), C.byref(t1), C.byref(p1), C.byref(n1), C.byref(f1)) == 0
        Lo.oracle_sphere_hit(V(c), r, V(o), V(d), E.T_MIN, math.inf, C.byref(h2), C.byref(t2), C.byref(p2), C.byref(n2), C.byref(f2), C.byref(u), C.byref(v))
        what = (name, i)
        assert h1.value == h2.value, what
        if h1.value:
            assert np.array([t1.value, *p1.tup(), *n1.tup()]).view(np.uint64).tolist() == np.array([t2.value, *p2.tup(), *n2.tup()]).view(np.uint64).tolist(), what
            assert f1.value == f2.value, what
        h = E.sphere_hit(E.Chain(), c, r, tuple(o), tuple(d))
        assert bool(h1.value) == (h["which"] is not None), what
        if h1.value:
            assert t1.value == h["t"] and bool(f1.value) == h["front"], what


def test_stress_builds_answer_the_exact_edges(tmp_path):
    """Every stress build (leaves of 2, 6, 16 and 32, minimal work lists) as uploaded and after rebuild(): intersect, occluded
    and trace_rays like the oracle, the tied pair of E3_leaves in different leaves and E3_always's member on the always-list."""
    from test_gpu_build_invariance import constants
    manifest = json.load(open(os.path.join(STRESS, "manifest.json")))
    cases = E.cases()
    for build in manifest:
        out = tmp_path / f"{build}.npz"
        env = dict(os.environ, RTB200_LIB=os.path.join(STRESS, f"librtb200_{build}.so"))
        subprocess.run([sys.executable, os.path.join(REPO, "tests", "exact_edges_worker.py"), str(out)], env=env, check=True, timeout=900)
        z = np.load(out, allow_pickle=False)
        meta = json.loads(str(z["meta"]))
        assert meta["leaf_size"] == constants(manifest[build])["RT_LEAF_K"]
        for case in cases:
            sc = scene(case, E.LIGHTS)
            un = IR.oracle(sc, case.o, case.d)
            want = OT.trace_rays(sc, case.o, case.d, **EW.TRACE)
            for state in EW.STATES:
                key = f"{case.name}/{state}"
                what = f"{build}/{key}"
                IR.assert_hits_equal({k: z[f"{key}.{k}"] for k in IR.FIELDS}, un, what)
                assert_occluded_equal(z[f"{key}.occluded"], (un["sphere"] >= 0).astype(np.uint8), what + "/occluded")
                assert_frames_match((z[f"{key}.linear"], z[f"{key}.rgb8"]), (want["linear"], want["rgb8"]), what)
                assert meta["rays"][key] == want["rays"], what
                if case.name.startswith("E3_leaves"):
                    lid = z[f"{key}.leaf_id"]
                    assert len(z[f"{key}.always"]) == 0 and leaf_of(lid, 0, sc.n_spheres) != leaf_of(lid, 1, sc.n_spheres), what
                elif case.name.startswith("E3_always"):
                    assert z[f"{key}.always"].tolist() == [E.always_member(case)], what
