"""ctypes binding of the oracle's thin-lens camera (tests/oracle_lens.cpp -> tests/liboracle_lens.so).

TEST INFRASTRUCTURE ONLY: the reference answer of rtb200_camera_from_params_lens, rtb200_probe_lens_ray and lens renders.

    python tests/oracle_lens.py build     # (re)build the library; __graft_entry__.build() runs this
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_REPO = os.path.dirname(_HERE)
sys.path.insert(0, os.path.join(_REPO, "rust-raytracer_b200"))
import rtb200 as R  # noqa: E402  (structures only: nothing here maps librtb200.so)

SRC = os.path.join(_HERE, "oracle_lens.cpp")
LIB_PATH = os.path.join(_HERE, "liboracle_lens.so")
# the oracle's compiler and flags (oracle/Makefile): no FMA contraction, as rustc
CXX = "/usr/bin/g++"
CXXFLAGS = ["-O3", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra"]

_lib = None


def build(force: bool = False):
    """Build liboracle_lens.so when it is missing or older than its sources."""
    deps = [SRC, os.path.join(_REPO, "oracle", "rt_oracle.hpp"), os.path.join(_REPO, "include", "rtb200.h")]
    stale = not os.path.exists(LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(LIB_PATH) for d in deps)
    if force or stale:
        subprocess.check_call([CXX, *CXXFLAGS, "-shared", "-o", LIB_PATH, SRC])


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        L.oracle_camera_lens.argtypes = [C.POINTER(R.rt_camera_params), C.c_double, C.c_double, C.POINTER(R.rt_camera), C.POINTER(R.rt_lens)]
        L.oracle_lens_ray.argtypes = [C.POINTER(R.rt_camera), C.POINTER(R.rt_lens), C.c_uint64, C.c_uint32, C.c_uint32, C.c_double,
                                      C.c_double, C.c_void_p, C.POINTER(C.c_uint32)]
        L.oracle_lens_primary.argtypes = [C.c_void_p, C.POINTER(R.rt_lens), C.c_uint32, C.c_void_p, C.c_void_p]
        L.oracle_lens_render.argtypes = [C.c_void_p, C.POINTER(R.rt_lens), C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        L.oracle_lens_hits.argtypes = [C.c_void_p, C.POINTER(R.rt_lens), C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_lens_aov.argtypes = [C.c_void_p, C.POINTER(R.rt_lens), C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def use_as_backend():
    """Install the oracle's lens camera as rtb200's camera_from_params_lens (rtb200.set_lens_backend)."""
    R.set_lens_backend(lambda p, a, f, cam, lens: lib().oracle_camera_lens(p, a, f, cam, lens))


def _lens(lens):
    return lens if lens is not None else R.rt_lens()


def lens_ray(cam, lens, seed: int, pixel: int, sample: int, u: float, v: float):
    """(origin[3], direction[3], trials) of the lens ray (numpy f64)."""
    out = np.empty(6)
    t = C.c_uint32()
    lib().oracle_lens_ray(C.byref(cam), C.byref(_lens(lens)), int(seed), int(pixel), int(sample), float(u), float(v), out.ctypes.data, C.byref(t))
    return out[:3], out[3:], int(t.value)


def primary(scene, lens, sample: int):
    """(origin, direction) [h*w, 3] of sample `sample` of every pixel of `scene` through `lens`."""
    n = int(scene.c.width) * int(scene.c.height)
    o, d = np.empty((n, 3)), np.empty((n, 3))
    lib().oracle_lens_primary(C.addressof(scene.c), C.byref(_lens(lens)), int(sample), o.ctypes.data, d.ctypes.data)
    return o, d


def render(scene, lens) -> dict:
    """The lens render of `scene`: {"linear": float32 [h, w, 3], "rgb8": uint8 [h, w, 3], "rays": hit_world calls}."""
    w, h = int(scene.c.width), int(scene.c.height)
    lin, rgb = np.empty((h, w, 3), np.float32), np.empty((h, w, 3), np.uint8)
    rays = C.c_uint64()
    rc = lib().oracle_lens_render(C.addressof(scene.c), C.byref(_lens(lens)), lin.ctypes.data, rgb.ctypes.data, C.byref(rays))
    if rc != 0:
        raise RuntimeError(f"oracle_lens_render failed: {rc}")
    return {"linear": lin, "rgb8": rgb, "rays": int(rays.value)}


def hits(scene, lens, samples: int = 1, sample0: int = 0) -> dict:
    """sphere (int32, -1 on a miss) and point of sample sample0's lens ray, and the samples that hit, per pixel [h, w]."""
    w, h = int(scene.c.width), int(scene.c.height)
    sph, pt, nh = np.empty((h, w), np.int32), np.empty((h, w, 3)), np.empty((h, w), np.uint32)
    lib().oracle_lens_hits(C.addressof(scene.c), C.byref(_lens(lens)), int(samples), int(sample0), sph.ctypes.data, pt.ctypes.data, nh.ctypes.data)
    return {"sphere": sph, "point": pt, "hits": nh}


def aov(scene, lens, samples: int = 1, sample0: int = 0) -> dict:
    """albedo and normal (float32 [h, w, 3]) of the lens rays of samples [sample0, sample0 + samples): oracle_aov's with the lens."""
    w, h = int(scene.c.width), int(scene.c.height)
    al, nm = np.empty((h, w, 3), np.float32), np.empty((h, w, 3), np.float32)
    lib().oracle_lens_aov(C.addressof(scene.c), C.byref(_lens(lens)), int(samples), int(sample0), al.ctypes.data, nm.ctypes.data)
    return {"albedo": al, "normal": nm}


if __name__ == "__main__":
    if sys.argv[1:] == ["build"]:
        build()
    else:
        sys.exit(__doc__)
