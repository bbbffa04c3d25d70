#!/usr/bin/env python3
"""A 360-degree equirectangular panorama of a scene, traced on the GPU through caller-supplied rays
(ResidentScene.trace_rays, DESIGN.md §4.12): a camera the renderer's pinhole Camera::get_ray cannot express.

    python tools/panorama.py scene.json out.png [--width 1024] [--samples 64] [--at x,y,z]

The image is width x width/2. Pixel (x, y) looks along longitude 2*pi*(x + 0.5)/width - pi and latitude
pi/2 - pi*(y + 0.5)/height: y is up, longitude 0 looks down -z, and the top row looks straight up. The rays start at `at`
(default: the scene's look_from), are built in float64 on the GPU, traced with `samples` samples each in one call, and the
RGB8 result is written as a PNG. Sample j of pixel p draws from the RNG stream of (pixel p, sample j) under the scene's seed,
with the scene's max_depth."""
import argparse
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rust-raytracer_b200"))

import rtb200 as R  # noqa: E402


def equirect_rays(width: int, height: int, at, device="cuda"):
    """(origin, direction), contiguous float64 tensors [height * width, 3], top row first."""
    import torch
    y, x = torch.meshgrid(torch.arange(height, dtype=torch.float64, device=device),
                          torch.arange(width, dtype=torch.float64, device=device), indexing="ij")
    lon = (x + 0.5) * (2.0 * math.pi / width) - math.pi
    lat = 0.5 * math.pi - (y + 0.5) * (math.pi / height)
    d = torch.stack([torch.cos(lat) * torch.sin(lon), torch.sin(lat), -torch.cos(lat) * torch.cos(lon)], dim=-1).reshape(-1, 3)
    o = torch.tensor([float(a) for a in at], dtype=torch.float64, device=device).expand_as(d)
    return o.contiguous(), d.contiguous()


def render_panorama(scene: "R.Scene", width: int, samples: int, at=None):
    """The panorama as uint8 [width // 2, width, 3] (numpy) and the call's stats."""
    height = width // 2
    if at is None:
        at = R.vec3(scene.camera_params["look_from"]).tup()
    o, d = equirect_rays(width, height, at)
    rs = R.ResidentScene(scene)
    try:
        out = rs.trace_rays(o, d, samples, linear=False, rgb8=True)
    finally:
        rs.release()
    return out["rgb8"].cpu().numpy().reshape(height, width, 3), out["stats"]


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("scene")
    ap.add_argument("out")
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--at", default=None, help="x,y,z (default: the scene's look_from)")
    a = ap.parse_args(argv)
    if a.width < 2 or a.width % 2:
        ap.error("--width must be an even number >= 2")
    at = None if a.at is None else [float(v) for v in a.at.split(",")]
    if at is not None and len(at) != 3:
        ap.error("--at takes x,y,z")
    img, st = render_panorama(R.load_scene(a.scene), a.width, a.samples, at)
    R.write_png(a.out, img)
    print(f"{a.out}: {a.width}x{a.width // 2}, {a.samples} samples, {st['rays']} rays, device {st['device_ms']:.1f} ms")
    return 0


if __name__ == "__main__":
    sys.exit(main())
