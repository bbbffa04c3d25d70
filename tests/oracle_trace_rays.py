"""ctypes binding of the oracle's ray_color on caller-supplied rays (tests/oracle_trace_rays.cpp -> tests/liboracle_trace_rays.so).

TEST INFRASTRUCTURE ONLY: the reference answer of ResidentScene.trace_rays / rtb200_scene_trace_rays[_device].

    python tests/oracle_trace_rays.py build     # (re)build the library; __graft_entry__.build() runs this
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_REPO = os.path.dirname(_HERE)
SRC = os.path.join(_HERE, "oracle_trace_rays.cpp")
LIB_PATH = os.path.join(_HERE, "liboracle_trace_rays.so")
# the oracle's compiler and flags (oracle/Makefile): no FMA contraction, as rustc
CXX = "/usr/bin/g++"
CXXFLAGS = ["-O3", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra"]

_lib = None


def build(force: bool = False):
    """Build liboracle_trace_rays.so when it is missing or older than its sources."""
    deps = [SRC, os.path.join(_REPO, "oracle", "rt_oracle.hpp"), os.path.join(_REPO, "include", "rtb200.h")]
    stale = not os.path.exists(LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(LIB_PATH) for d in deps)
    if force or stale:
        subprocess.check_call([CXX, *CXXFLAGS, "-shared", "-o", LIB_PATH, SRC])


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        L.oracle_trace_rays.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                        C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


def trace_rays(scene, origin, direction, samples: int = 1, sample0: int = 0, stream0: int = 0, seed=None, max_depth=None) -> dict:
    """`samples` samples of ray_color(Ray{origin[i], direction[i]}, max_depth, max_depth) per ray, sample j on the stream of
    (pixel stream0 + i, sample sample0 + j) past its first two draws, resolved like a render with spp = samples. seed and
    max_depth default to the scene's own. Returns {"linear": float32 [n, 3], "rgb8": uint8 [n, 3], "rays": hit_world calls}."""
    o = np.ascontiguousarray(origin, dtype=np.float64).reshape(-1, 3)
    d = np.ascontiguousarray(direction, dtype=np.float64).reshape(-1, 3)
    n = o.shape[0]
    assert d.shape[0] == n
    lin = np.empty((n, 3), np.float32)
    rgb = np.empty((n, 3), np.uint8)
    rays = C.c_uint64()
    keep = (scene.c.seed, scene.c.max_depth)
    try:
        if seed is not None:
            scene.c.seed = int(seed)
        if max_depth is not None:
            scene.c.max_depth = int(max_depth)
        rc = lib().oracle_trace_rays(C.addressof(scene.c), o.ctypes.data, d.ctypes.data, n, int(samples), int(sample0), int(stream0),
                                     lin.ctypes.data, rgb.ctypes.data, C.byref(rays))
    finally:
        scene.c.seed, scene.c.max_depth = keep
    if rc != 0:
        raise RuntimeError(f"oracle_trace_rays failed: {rc}")
    return {"linear": lin, "rgb8": rgb, "rays": int(rays.value)}


if __name__ == "__main__":
    if sys.argv[1:] == ["build"]:
        build()
    else:
        sys.exit(__doc__)
