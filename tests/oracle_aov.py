"""ctypes binding of the oracle's auxiliary buffers of a render's camera samples (tests/oracle_aov.cpp -> tests/liboracle_aov.so).

TEST INFRASTRUCTURE ONLY: the reference answer of ResidentScene.aov / rtb200_scene_aov[_device].

    python tests/oracle_aov.py build     # (re)build the library; __graft_entry__.build() runs this
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_REPO = os.path.dirname(_HERE)
SRC = os.path.join(_HERE, "oracle_aov.cpp")
LIB_PATH = os.path.join(_HERE, "liboracle_aov.so")
# the oracle's compiler and flags (oracle/Makefile): no FMA contraction, as rustc
CXX = "/usr/bin/g++"
CXXFLAGS = ["-O3", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra"]

_lib = None


def build(force: bool = False):
    """Build liboracle_aov.so when it is missing or older than its sources."""
    deps = [SRC, os.path.join(_REPO, "oracle", "rt_oracle.hpp"), os.path.join(_REPO, "include", "rtb200.h")]
    stale = not os.path.exists(LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(LIB_PATH) for d in deps)
    if force or stale:
        subprocess.check_call([CXX, *CXXFLAGS, "-shared", "-o", LIB_PATH, SRC])


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        L.oracle_aov.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 5
        _lib = L
    return _lib


def aov(scene, samples: int = 1, sample0: int = 0, camera=None, seed=None) -> dict:
    """The auxiliary buffers of samples [sample0, sample0 + samples) of every pixel of the whole frame, top row first, under
    the scene's camera and seed (or `camera`, an rt_camera, and `seed`). Returns numpy arrays: albedo and normal float32
    [h, w, 3], hits uint32 [h, w], sphere int32 [h, w] (-1: miss), point float64 [h, w, 3]."""
    w, h = int(scene.c.width), int(scene.c.height)
    out = {"albedo": np.empty((h, w, 3), np.float32), "normal": np.empty((h, w, 3), np.float32), "hits": np.empty((h, w), np.uint32),
           "sphere": np.empty((h, w), np.int32), "point": np.empty((h, w, 3))}
    keep = (scene.c.seed, type(scene.c.camera).from_buffer_copy(scene.c.camera))   # a field read is a view, not a copy
    try:
        if camera is not None:
            scene.c.camera = camera
        if seed is not None:
            scene.c.seed = int(seed)
        rc = lib().oracle_aov(C.addressof(scene.c), int(samples), int(sample0),
                              *(out[k].ctypes.data for k in ("albedo", "normal", "hits", "sphere", "point")))
    finally:
        scene.c.seed, scene.c.camera = keep
    if rc != 0:
        raise RuntimeError(f"oracle_aov failed: {rc}")
    return out


if __name__ == "__main__":
    if sys.argv[1:] == ["build"]:
        build()
    else:
        sys.exit(__doc__)
