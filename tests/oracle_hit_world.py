"""ctypes binding of the oracle's hit_world on caller-supplied rays (tests/oracle_hit_world.cpp -> tests/liboracle_hit_world.so).

TEST INFRASTRUCTURE ONLY: the reference answer of ResidentScene.intersect / rtb200_scene_intersect[_device].

    python tests/oracle_hit_world.py build     # (re)build the library; __graft_entry__.build() runs this
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_REPO = os.path.dirname(_HERE)
SRC = os.path.join(_HERE, "oracle_hit_world.cpp")
LIB_PATH = os.path.join(_HERE, "liboracle_hit_world.so")
# the oracle's compiler and flags (oracle/Makefile): no FMA contraction, as rustc
CXX = "/usr/bin/g++"
CXXFLAGS = ["-O3", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra"]

_lib = None


def build(force: bool = False):
    """Build liboracle_hit_world.so when it is missing or older than its sources."""
    deps = [SRC, os.path.join(_REPO, "oracle", "rt_oracle.hpp"), os.path.join(_REPO, "include", "rtb200.h")]
    stale = not os.path.exists(LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(LIB_PATH) for d in deps)
    if force or stale:
        subprocess.check_call([CXX, *CXXFLAGS, "-shared", "-o", LIB_PATH, SRC])


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        L.oracle_hit_world.argtypes = [C.c_void_p] + [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 6
        _lib = L
    return _lib


def hit_world(scene, origin, direction, t_max=None) -> dict:
    """hit_world(scene, Ray{origin[i], direction[i]}, 0.001, t_max[i]) for every ray (t_max None: f64::MAX). Returns numpy
    arrays: t [n], sphere int32 [n] (-1: miss), point [n, 3], normal [n, 3], uv [n, 2], front_face uint8 [n]."""
    o = np.ascontiguousarray(origin, dtype=np.float64).reshape(-1, 3)
    d = np.ascontiguousarray(direction, dtype=np.float64).reshape(-1, 3)
    n = o.shape[0]
    assert d.shape[0] == n
    tm = None if t_max is None else np.ascontiguousarray(t_max, dtype=np.float64).reshape(n)
    out = {"t": np.empty(n), "sphere": np.empty(n, np.int32), "point": np.empty((n, 3)), "normal": np.empty((n, 3)),
           "uv": np.empty((n, 2)), "front_face": np.empty(n, np.uint8)}
    rc = lib().oracle_hit_world(C.addressof(scene.c), o.ctypes.data, d.ctypes.data, None if tm is None else tm.ctypes.data, n,
                                *(out[k].ctypes.data for k in ("t", "sphere", "point", "normal", "uv", "front_face")))
    if rc != 0:
        raise RuntimeError(f"oracle_hit_world failed: {rc}")
    return out


if __name__ == "__main__":
    if sys.argv[1:] == ["build"]:
        build()
    else:
        sys.exit(__doc__)
