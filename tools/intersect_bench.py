#!/usr/bin/env python3
"""Closest-hit query throughput (ResidentScene.intersect, DESIGN.md §4.10) on the GPU.

    python tools/intersect_bench.py [--reps 20] [--out intersect_bench.jsonl]

For each (scene, variant) and ray set it prints one JSON line: device-time Mrays/s of the device form (CUDA events around the
query on its own stream, median of `reps` warm runs after two warm-up runs) and, from one run of the host form, f64 sphere
tests (candidates), leaf visits (clusters) and node visits per ray. Ray sets: the 800x600 camera rays through the pixel
centres, one diffuse secondary per camera hit (from its hit point, normal + a random unit vector), and uniform random rays
with origins in the box of the sphere centres. Scenes: the cover scene (FILTERED and BRUTE_FORCE), C4's 10k-sphere scene and a
100k-sphere one of the same generator (FILTERED). The first line names the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rust-raytracer_b200"))

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def camera_rays(sc, w, h):
    cam = sc.c.camera
    o = np.array(cam.origin.tup()); llc = np.array(cam.lower_left_corner.tup())
    hor = np.array(cam.horizontal.tup()); ver = np.array(cam.vertical.tup())
    y, x = np.mgrid[0:h, 0:w]
    u = ((x + 0.5) / (w - 1.0)).reshape(-1, 1)
    v = ((h - (y + 0.5)) / (h - 1.0)).reshape(-1, 1)
    d = ((llc + hor * u) + ver * v) - o
    return np.broadcast_to(o, d.shape).copy(), np.ascontiguousarray(d)


def ray_sets(sc, rs, rng):
    o, d = camera_rays(sc, 800, 600)
    h = rs.intersect(o, d, outputs=("sphere", "point", "normal"))
    m = h["sphere"] >= 0
    g = rng.normal(size=(int(m.sum()), 3))
    so, sd = h["point"][m], h["normal"][m] + g / np.linalg.norm(g, axis=1, keepdims=True)
    n = sc.n_spheres
    c = np.array([sc._spheres[i].center.tup() for i in range(n)])
    c = c[(np.abs(c) < 1e6).all(axis=1)]
    lo, hi = c.min(axis=0), c.max(axis=0)
    ro = lo + rng.random((480_000, 3)) * (hi - lo)
    return {"camera_800x600": (o, d), "diffuse_secondary": (np.ascontiguousarray(so), np.ascontiguousarray(sd)),
            "random_in_box": (ro, rng.normal(size=(480_000, 3)))}


def measure(rs, o, d, reps):
    import torch
    do, dd = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    s = torch.cuda.Stream()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    with torch.cuda.stream(s):
        for _ in range(2):
            rs.intersect(do, dd, stream=s)
        for a, b in ev:
            a.record(s)
            rs.intersect(do, dd, stream=s)
            b.record(s)
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2], ms[0], ms[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    rng = np.random.default_rng(7)
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)
    cases = [("cover", lambda: scenes.cover_scene(800, 600, 1), R.RT_VARIANT_FILTERED),
             ("cover", lambda: scenes.cover_scene(800, 600, 1), R.RT_VARIANT_BRUTE_FORCE),
             ("c4_10k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), 800, 600, 1, 50)), R.RT_VARIANT_FILTERED),
             ("rtiow_100k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(158), 800, 600, 1, 50)), R.RT_VARIANT_FILTERED)]
    for name, mk, variant in cases:
        sc = mk()
        rs = R.ResidentScene(sc, R.make_options(variant=variant))
        try:
            for set_name, (o, d) in ray_sets(sc, rs, rng).items():
                st = rs.intersect(o, d, outputs=("sphere",))["stats"]
                med, lo, hi = measure(rs, o, d, args.reps)
                n = len(o)
                rec = {"scene": name, "spheres": sc.n_spheres, "variant": {1: "FILTERED", 4: "BRUTE_FORCE"}[variant], "rays": set_name,
                       "n": n, "median_ms": round(med, 4), "min_ms": round(lo, 4), "max_ms": round(hi, 4),
                       "mrays_per_s": round(n / med / 1e3, 1), "candidates_per_ray": round(st["candidates"] / n, 3),
                       "leaves_per_ray": round(st["clusters"] / n, 3), "nodes_per_ray": round(st["nodes"] / n, 3)}
                lines.append(rec)
                print(json.dumps(rec), flush=True)
        finally:
            rs.release()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
