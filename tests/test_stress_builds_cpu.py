"""The stress builds of the library (rust-raytracer_b200/stress, `make stress`; rendered against the oracle by
tests/test_gpu_build_invariance.py) are the builds their DEFS describe, checked without a GPU: each one loads in a process of
its own (rtb200 reads RTB200_LIB at import), exports every symbol of the C ABI, and builds hierarchies with its own leaf size
(rtb200_debug_bvh runs on the host); the host builder's hierarchies pass test_bvh_cpu's structure and soundness checks at
that leaf size; and the scenes the build-invariance test stages still have an odd number of leaves at leaves of 2 and 6,
where the staged leaf-id block is not a whole number of 16 B blocks."""
import json
import os
import subprocess
import sys

import pytest

from test_gpu_build_invariance import BUILDS, STRESS, constants

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r"""
import json, sys
sys.path[:0] = sys.argv[1:]
import rtb200 as R
from rtb200 import scenes
import build_worker as BW
L = R.lib()
missing = [s for s in R.ABI_SYMBOLS if not hasattr(L, s)]
t = R.bvh_records(scenes.cover_scene(32, 24, 1))
staged = {name: int(R.bvh_records(BW.CASES[name][1]())["n_leaves"]) for name in BW.STAGE_SCENES}
print(json.dumps({"lib": R.LIB_PATH, "missing": missing, "leaf_size": t["leaf_size"], "n_leaves": t["n_leaves"], "depth": t["depth"],
                  "staged_leaves": staged}))
"""
# test_bvh_cpu's checks of the host builder (structure; the float32 traversal never drops an exact hit) with the library
BVH_CHILD = r"""
import sys
sys.path[:0] = sys.argv[1:]
import test_bvh_cpu as T
for mk in T.SCENES:
    T.test_bvh_structure(mk)
for mk in T.SCENES[:4]:
    T.test_emulated_traversal_never_drops_a_sphere_the_exact_test_accepts(mk)
print('"ok"')
"""
PATHS = [os.path.join(REPO, "rust-raytracer_b200"), os.path.join(REPO, "oracle"), os.path.join(REPO, "tests")]


def _manifest():
    path = os.path.join(STRESS, "manifest.json")
    assert os.path.exists(path), f"{path} is missing: build() runs make -C rust-raytracer_b200 stress"
    with open(path) as f:
        return json.load(f)


def test_the_manifest_names_every_build_the_gpu_test_runs():
    assert sorted(_manifest()) == sorted(BUILDS)


def _probe(lib, child=CHILD, timeout=120):
    env = dict(os.environ, RTB200_LIB=lib)
    r = subprocess.run([sys.executable, "-c", child, *PATHS], capture_output=True, text=True, env=env, timeout=timeout)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("build", BUILDS)
def test_stress_build_loads_and_has_its_leaf_size(build):
    defs = _manifest()[build]
    lib = os.path.join(STRESS, f"librtb200_{build}.so")
    assert os.path.exists(lib), lib
    got = _probe(lib)
    assert os.path.samefile(got["lib"], lib)
    assert got["missing"] == []
    k = constants(defs)["RT_LEAF_K"]
    assert got["leaf_size"] == k, (got, defs)
    if k * 4 % 16:   # the staged leaf-id block of an odd leaf count is 8 B short of a 16 B multiple: a staged scene has one
        assert any(n % 2 for n in got["staged_leaves"].values()), got["staged_leaves"]


@pytest.mark.parametrize("build", BUILDS)
def test_the_host_builder_is_sound_at_the_builds_leaf_size(build):
    assert _probe(os.path.join(STRESS, f"librtb200_{build}.so"), BVH_CHILD, timeout=600) == "ok"


def test_the_default_library_has_leaves_of_8():
    got = _probe(os.path.join(REPO, "rust-raytracer_b200", "librtb200.so"))
    assert got["missing"] == [] and got["leaf_size"] == 8 and (got["n_leaves"], got["depth"]) == (68, 3), got
