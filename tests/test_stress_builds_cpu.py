"""The stress builds of the library (rust-raytracer_b200/stress, `make stress`; rendered against the oracle by
tests/test_gpu_build_invariance.py) are the builds their DEFS describe, checked without a GPU: each one loads in a process of
its own (rtb200 reads RTB200_LIB at import), exports every symbol of the C ABI, and builds hierarchies with its own leaf size
(rtb200_debug_bvh runs on the host)."""
import json
import os
import subprocess
import sys

import pytest

from test_gpu_build_invariance import BUILDS, STRESS, constants

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import rtb200 as R
from rtb200 import scenes
L = R.lib()
missing = [s for s in R.ABI_SYMBOLS if not hasattr(L, s)]
t = R.bvh_records(scenes.cover_scene(32, 24, 1))
print(json.dumps({"lib": R.LIB_PATH, "missing": missing, "leaf_size": t["leaf_size"], "n_leaves": t["n_leaves"], "depth": t["depth"]}))
"""


def _manifest():
    path = os.path.join(STRESS, "manifest.json")
    assert os.path.exists(path), f"{path} is missing: build() runs make -C rust-raytracer_b200 stress"
    with open(path) as f:
        return json.load(f)


def test_the_manifest_names_the_builds_the_gpu_test_runs():
    assert sorted(_manifest()) == sorted(BUILDS)


def _probe(lib):
    env = dict(os.environ, RTB200_LIB=lib)
    r = subprocess.run([sys.executable, "-c", CHILD, os.path.join(REPO, "rust-raytracer_b200")], capture_output=True, text=True,
                       env=env, timeout=120)
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
    assert got["leaf_size"] == constants(defs)["RT_LEAF_K"], (got, defs)


def test_the_default_library_has_leaves_of_8():
    got = _probe(os.path.join(REPO, "rust-raytracer_b200", "librtb200.so"))
    assert got["missing"] == [] and got["leaf_size"] == 8 and (got["n_leaves"], got["depth"]) == (68, 3), got
