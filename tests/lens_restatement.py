"""The thin-lens camera (include/rtb200.h, DESIGN.md §4.17) restated a second time, in pure Python (TEST INFRASTRUCTURE).

tests/oracle_lens.cpp is the lens checker the GPU tests compare with. This module states the same contract again on top of
tests/py_restatement.py (its own Philox, vector arithmetic, camera basis and recursive ray_color), sharing no code with the
C++ oracle, so that tests/test_lens_restatement_cpu.py can demand bit-identical lens frames from the two. Small cases only.
"""
import math

import numpy as np

from py_restatement import Stream, World, add, cross, f32, mul, philox4x32_10, sub, unit_vector, vec


def m1_1(u64):
    """gen_range(-1.0..1.0) of one u64 (rand 0.8 UniformFloat::sample_single)."""
    value1_2 = np.array([(u64 >> 12) | 0x3FF0000000000000], dtype=np.uint64).view(np.float64)[0].item()
    return (value1_2 - 1.0) * 2.0 + -1.0


def lens_disk(seed, pixel, sample):
    """The accepted (x, y) and the trials drawn: trial k is Philox block (k, sample, pixel, 1) under the key `seed`."""
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    k = 0
    while True:
        w = philox4x32_10((k, sample, pixel, 1), key)
        x, y = m1_1(w[0] | (w[1] << 32)), m1_1(w[2] | (w[3] << 32))
        k += 1
        if x * x + y * y < 1.0:
            return x, y, k


class LensCamera:
    """Camera::new's basis with the image plane at focus_dist, and the lens {u, v, aperture / 2}."""

    def __init__(self, c, aperture, focus_dist):
        look_from, look_at, vup = vec(c["look_from"]), vec(c["look_at"]), vec(c["vup"])
        theta = float(c["vfov"]) * (math.pi / 180.0)
        half_height = math.tan(theta / 2.0)
        half_width = float(c["aspect"]) * half_height
        w = unit_vector(sub(look_from, look_at))
        self.u = unit_vector(cross(vup, w))
        self.v = cross(w, self.u)
        fd = float(focus_dist)
        self.origin = look_from
        self.lower_left_corner = sub(sub(sub(self.origin, mul(self.u, half_width * fd)), mul(self.v, half_height * fd)), mul(w, fd))
        self.horizontal = mul(mul(mul(self.u, 2.0), half_width), fd)
        self.vertical = mul(mul(mul(self.v, 2.0), half_height), fd)
        self.radius = float(aperture) / 2.0

    def get_ray(self, u, v, seed, pixel, sample):
        o = self.origin
        d = sub(add(add(self.lower_left_corner, mul(self.horizontal, u)), mul(self.vertical, v)), o)
        if self.radius == 0.0:
            return o, d, 0
        x, y, trials = lens_disk(seed, pixel, sample)
        rdx, rdy = self.radius * x, self.radius * y
        off = add(mul(self.u, rdx), mul(self.v, rdy))
        return add(o, off), sub(d, off), trials


class LensWorld(World):
    """py_restatement's World rendered through a lens camera."""

    def __init__(self, cfg, aperture, focus_dist, **kw):
        super().__init__(cfg, **kw)
        self.lens_camera = LensCamera(cfg["camera"], aperture, focus_dist)

    def render(self):
        w, h = self.width, self.height
        lin = np.zeros((h, w, 3), np.float32); img = np.zeros((h, w, 3), np.uint8)
        self.rays = 0
        for y in range(h):
            for x in range(w):
                acc = [f32(0.0), f32(0.0), f32(0.0)]
                for s in range(self.spp):
                    rng = Stream(self.seed, y * w + x, s)
                    u = (float(x) + rng.gen_f64()) / (float(w) - 1.0)
                    v = (float(h) - (float(y) + rng.gen_f64())) / (float(h) - 1.0)
                    o, d, _ = self.lens_camera.get_ray(u, v, self.seed, y * w + x, s)
                    c = self.ray_color(o, d, rng, self.max_depth, self.max_depth)
                    for k in range(3):
                        acc[k] = acc[k] + c[k]
                scale = f32(1.0) / f32(self.spp)
                for k in range(3):
                    m = scale * acc[k]
                    lin[y, x, k] = m
                    scaled = np.fmin(np.sqrt(m) * f32(255.0), f32(255.0))
                    bits = int(np.array([scaled + f32(8388608.0)], np.float32).view(np.uint32)[0])
                    img[y, x, k] = max(bits - 0x4B000000, 0) & 0xFF if bits >= 0x4B000000 else 0
        return lin, img, self.rays
