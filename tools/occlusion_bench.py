#!/usr/bin/env python3
"""Occlusion query throughput (ResidentScene.occluded, DESIGN.md §4.11) against the closest-hit query on the same rays.

    python tools/occlusion_bench.py [--reps 20] [--out occlusion_bench.jsonl]

For each scene and ray set it prints one JSON line with the device-time Mrays/s of both device forms, occluded(...) and
intersect(..., outputs=("sphere",)) under the same t_max (CUDA events around each query on its own stream, median of `reps`
warm runs after two warm-up runs), and, from one run of each host form, f64 sphere tests (candidates), leaf visits (clusters)
and node visits per ray. Ray sets: shadow segments from every hit of the 800x600 camera rays to a random point on another
sphere (t_max 1); 480,000 short segments (length <= 0.5) from random sphere surfaces (t_max 1); 480,000 unbounded rays with
origins uniform in the box of the sphere centres; the 800x600 camera rays (unbounded). Scenes: the cover scene (484 spheres),
C4's 10k-sphere scene and a 100k-sphere one of the same generator, all FILTERED. The first line names the card and its power
limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rust-raytracer_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import rtb200 as R  # noqa: E402
from intersect_bench import camera_rays, card  # noqa: E402
from rtb200 import scenes  # noqa: E402


def _spheres(sc):
    n = sc.n_spheres
    c = np.array([sc._spheres[i].center.tup() for i in range(n)]).reshape(n, 3)
    r = np.array([sc._spheres[i].radius for i in range(n)])
    return c, r


def ray_sets(sc, rs, rng, k=480_000):
    """name -> (origin, direction, t_max or None)."""
    c, r = _spheres(sc)
    ok = np.flatnonzero((np.abs(c) < 1e6).all(axis=1) & (np.abs(r) < 100))
    o, d = camera_rays(sc, 800, 600)
    h = rs.intersect(o, d, outputs=("sphere", "point"))
    m = h["sphere"] >= 0
    p, j = h["point"][m], h["sphere"][m]
    t = ok[rng.integers(0, len(ok), size=len(p))]
    t = np.where(t == j, ok[(np.searchsorted(ok, t) + 1) % len(ok)], t)
    g = rng.normal(size=(len(p), 3)); g /= np.linalg.norm(g, axis=1, keepdims=True)
    shadow = (np.ascontiguousarray(p), np.ascontiguousarray(c[t] + g * np.abs(r[t])[:, None] - p), np.ones(len(p)))
    s = ok[rng.integers(0, len(ok), size=k)]
    g = rng.normal(size=(k, 3)); g /= np.linalg.norm(g, axis=1, keepdims=True)
    v = g + rng.normal(size=(k, 3)); v /= np.linalg.norm(v, axis=1, keepdims=True)
    short = (c[s] + g * np.abs(r[s])[:, None], v * rng.uniform(0.01, 0.5, size=(k, 1)), np.ones(k))
    cc = c[ok]
    lo, hi = cc.min(axis=0), cc.max(axis=0)
    box = (lo + rng.random((k, 3)) * (hi - lo), rng.normal(size=(k, 3)), None)
    return {"shadow_segments": shadow, "short_segments": short, "random_in_box": box, "camera_800x600": (o, d, None)}


def measure(query, o, d, t, reps):
    import torch
    do, dd = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    dt = torch.from_numpy(t).cuda() if t is not None else None
    s = torch.cuda.Stream()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    with torch.cuda.stream(s):
        for _ in range(2):
            query(do, dd, dt, s)
        for a, b in ev:
            a.record(s)
            query(do, dd, dt, s)
            b.record(s)
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    rng = np.random.default_rng(7)
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)
    cases = [("cover", lambda: scenes.cover_scene(800, 600, 1)),
             ("c4_10k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), 800, 600, 1, 50))),
             ("rtiow_100k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(158), 800, 600, 1, 50)))]
    occ = lambda rs: lambda o, d, t, s: rs.occluded(o, d, t, stream=s)                               # noqa: E731
    clo = lambda rs: lambda o, d, t, s: rs.intersect(o, d, t, stream=s, outputs=("sphere",))         # noqa: E731
    for name, mk in cases:
        sc = mk()
        rs = R.ResidentScene(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
        try:
            for set_name, (o, d, t) in ray_sets(sc, rs, rng).items():
                n = len(o)
                ho = rs.occluded(o, d, t)
                hc = rs.intersect(o, d, t, outputs=("sphere",))
                assert np.array_equal(ho["occluded"], (hc["sphere"] != -1).astype(np.uint8)), (name, set_name)
                rec = {"scene": name, "spheres": sc.n_spheres, "rays": set_name, "n": n,
                       "occluded_fraction": round(float(ho["occluded"].mean()), 4)}
                for kind, q, st in (("occluded", occ(rs), ho["stats"]), ("intersect", clo(rs), hc["stats"])):
                    med = measure(q, o, d, t, args.reps)
                    rec[kind] = {"median_ms": round(med, 4), "mrays_per_s": round(n / med / 1e3, 1),
                                 "candidates_per_ray": round(st["candidates"] / n, 3), "leaves_per_ray": round(st["clusters"] / n, 3),
                                 "nodes_per_ray": round(st["nodes"] / n, 3)}
                rec["speedup"] = round(rec["occluded"]["mrays_per_s"] / rec["intersect"]["mrays_per_s"], 3)
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
