"""The exact-equality edges of tests/exact_edges.py without a GPU: every certificate holds; a vectorised numpy evaluation of
Sphere::hit gives the certificate's values; the oracle's hit_world makes the decision the certificate predicts (hit or miss,
which root, front_face, the sphere that wins a tie); the oracle's ray_color equals the pure-Python restatement
(tests/py_restatement.py) bit for bit at depth 1, 2 and 50 with 0 and 2 lights, so three independent restatements agree on
every edge; the tied pairs lie in different leaves and on the always-list where their case says so; the generators are
deterministic. Also the guard against FMA contraction in device code: every CUDA source with kernels compiles to the same
SASS with nvcc's --fmad=true (its default) and --fmad=false."""
import concurrent.futures as cf
import os
import re
import subprocess

import numpy as np
import pytest

import exact_edges as E
import oracle_hit_world as OH
import oracle_trace_rays as OT
import rtb200 as R
from py_restatement import Stream, World
from test_gpu_shading_edges import assert_frames_match, scene_of, synthetic_texture
from test_trace_rays_cpu import quantise

CASES = E.by_name()
NAMES = list(CASES)
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def scene(case, n_lights=0):
    """R.Scene of the case, with its lights when n_lights = 2 (the texture of TEX is synthetic_texture(5, 3))."""
    return scene_of(case.config(n_lights), {"tex": synthetic_texture(*E.TEX_SIZE)})


def world(case, n_lights, seed):
    cfg = case.config(n_lights)
    tex = {i: synthetic_texture(*E.TEX_SIZE) for i, o in enumerate(cfg["objects"]) if "Texture" in o["material"]}
    return World(cfg, textures=tex, seed=seed)


def restatement_trace(w, o, d, samples, max_depth):
    """oracle_trace_rays' contract in the restatement: sample j of ray i on the stream (pixel i, sample j) past its first two
    draws, ray_color(max_depth, max_depth), summed in f32 in sample order and scaled by 1/samples."""
    lin = np.empty((len(o), 3), np.float32)
    for i in range(len(o)):
        acc = [np.float32(0.0)] * 3
        for j in range(samples):
            rng = Stream(w.seed, i, j)
            rng.gen_f64(); rng.gen_f64()
            c = w.ray_color(tuple(float(x) for x in o[i]), tuple(float(x) for x in d[i]), rng, max_depth, max_depth)
            acc = [np.float32(acc[k] + c[k]) for k in range(3)]
        lin[i] = [np.float32(1.0) / np.float32(samples) * acc[k] for k in range(3)]
    return lin


@pytest.mark.parametrize("name", NAMES)
def test_every_certificate_holds(name):
    case = CASES[name]
    assert case.claims
    bad = [what for what, ok in case.claims if not ok]
    assert not bad, bad


@pytest.mark.parametrize("name", NAMES)
def test_numpy_evaluation_agrees_with_the_certificate(name):
    """Sphere::hit of every ray against its target sphere, vectorised in numpy in the reference's order, gives the chain's
    disc and roots bit for bit."""
    case = CASES[name]
    for i, (o, d, k) in enumerate(zip(case.o, case.d, case.target)):
        c, r = case.sphere_of(k)
        disc, ra, rb = E.np_sphere_hit(np.array([c]), np.array([r]), o[None], d[None])
        h = E.sphere_hit(E.Chain(), c, r, tuple(o), tuple(d))
        assert disc[0] == h["disc"], (name, i)
        if h["disc"] >= 0.0:
            assert ra[0] == h["root_a"] and rb[0] == h["root_b"], (name, i)


@pytest.mark.parametrize("n_lights", [0, E.LIGHTS])
@pytest.mark.parametrize("name", NAMES)
def test_the_oracle_makes_the_certified_decision(name, n_lights):
    case = CASES[name]
    sc = scene(case, n_lights)
    got = OH.hit_world(sc, case.o, case.d)
    for i, w in enumerate(case.want):
        what = f"{name} lights={n_lights} ray {i}"
        assert got["sphere"][i] == w["sphere"], (what, got["sphere"][i], w)
        if w["sphere"] >= 0:
            assert got["t"][i] == w["t"] and bool(got["front_face"][i]) == w["front"], (what, got["t"][i], got["front_face"][i], w)
    if name.startswith("E3"):   # the first index wins every tie
        assert (got["sphere"] == 0).all()
    hits = [w["which"] for w in case.want if w["sphere"] in case.target]
    if name.startswith("E1"):
        assert hits.count(None) == 0 and len(hits) > 0
    if name.startswith("E2"):
        assert "b" in hits and "a" in hits and any(w["sphere"] not in case.target for w in case.want)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_trace_rays_equals_the_restatement(name):
    case = CASES[name]
    samples = 2
    for n_lights in (0, E.LIGHTS):
        sc = scene(case, n_lights)
        w = world(case, n_lights, sc.seed)
        for depth in (1, 2, 50):
            want = OT.trace_rays(sc, case.o, case.d, samples, max_depth=depth)
            with np.errstate(all="ignore"):
                lin = restatement_trace(w, case.o, case.d, samples, depth)
            assert_frames_match((lin, quantise(lin)), (want["linear"], want["rgb8"]), f"{name} lights={n_lights} depth={depth}")


def test_the_generators_are_deterministic():
    a, b = E.cases(), E.cases()
    assert [c.name for c in a] == [c.name for c in b] and len(set(c.name for c in a)) == len(a)
    for x, y in zip(a, b):
        assert x.objects == y.objects and x.lights == y.lights and x.target == y.target and x.want == y.want
        assert np.array_equal(x.o.view(np.uint64), y.o.view(np.uint64)) and np.array_equal(x.d.view(np.uint64), y.d.view(np.uint64))
        assert [m for m, _ in x.claims] == [m for m, _ in y.claims]


def leaf_of(leaf_id, k, n):
    """The leaf that holds sphere k (leaf_id rows are padded with ids >= n)."""
    rows = [j for j, row in enumerate(leaf_id) if k in set(int(v) for v in row if v < n)]
    assert len(rows) == 1, (k, rows)
    return rows[0]


@pytest.mark.parametrize("name", [n for n in NAMES if n.startswith(("E3_leaves", "E3_always"))])
def test_the_host_hierarchy_splits_the_tied_pair(name):
    """E3_leaves: the pair in different leaves of the host build; E3_always: one member on the always-list, the other in a
    leaf. tests/test_gpu_exact_edges.py checks the same on the GPU's topology, after rebuild() and in every stress build."""
    case = CASES[name]
    for n_lights in (0, E.LIGHTS):
        sc = scene(case, n_lights)
        b = R.bvh_records(sc)
        always = set(int(v) for v in b["always"])
        if name.startswith("E3_leaves"):
            assert not always and leaf_of(b["leaf_id"], 0, sc.n_spheres) != leaf_of(b["leaf_id"], 1, sc.n_spheres)
        else:
            a = E.always_member(case)
            assert always == {a}, always
            leaf_of(b["leaf_id"], 1 - a, sc.n_spheres)


# ---- the FMA-contraction guard ----------------------------------------------------------------------------------------------
CSRC = os.path.join(REPO, "rust-raytracer_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")


def device_sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu") and "__global__" in open(os.path.join(CSRC, f)).read())


def _sass(src, fmad, out_dir):
    cubin = os.path.join(out_dir, f"{os.path.basename(src)}.{fmad}.cubin")
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++", f"--fmad={fmad}",
                    "-cubin", "-o", cubin, src], check=True, capture_output=True, cwd=CSRC)
    return subprocess.run([CUOBJDUMP, "-sass", cubin], check=True, capture_output=True, text=True).stdout


def test_device_code_is_not_contracted(tmp_path):
    """Device exactness rests on every f64/f32 operation being an explicit __d*_rn / __f*_rn intrinsic, which nvcc never
    fuses; a plain `a*b + c` in device code would be contracted to an FMA under nvcc's default --fmad=true and change the
    result. So each source with kernels must compile to identical SASS with and without contraction."""
    srcs = device_sources()
    assert len(srcs) >= 10, srcs
    jobs = [(s, f) for s in srcs for f in ("true", "false")]
    with cf.ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1)) as ex:
        out = dict(zip(jobs, ex.map(lambda j: _sass(os.path.join(CSRC, j[0]), j[1], str(tmp_path)), jobs)))
    differ = []
    for s in srcs:
        a, b = out[(s, "true")], out[(s, "false")]
        assert re.search(r"Function : \w+", a), f"{s}: no kernel in its SASS"
        if a != b:
            differ.append(f"{s} ({sum(1 for la, lb in zip(a.splitlines(), b.splitlines()) if la != lb)} SASS lines differ)")
    assert not differ, "device code contracted by --fmad=true: " + ", ".join(differ)
