#!/usr/bin/env python3
"""Point query throughput (ResidentScene.nearest / .overlaps, DESIGN.md §4.19), FILTERED against BRUTE_FORCE, with the
closest-hit query on the same scene as a yardstick.

    python tools/distance_bench.py [--reps 20] [--out distance_bench.jsonl]

For each scene and point set it prints one JSON line with, for nearest and overlaps in FILTERED and BRUTE_FORCE, the
device-time queries/s of the device form (CUDA events around each query on its own stream, median of `reps` warm runs after
two warm-up runs; a quarter of them, at least 3, for BRUTE_FORCE) and, from one run of the host form, exact distance evaluations (candidates), leaf visits (clusters) and node
visits per point. Point sets of 480,000 points: uniform in the box of the sphere centres, near surfaces (within 1e-3 of a
random sphere's surface: the contact case), and the first-hit points of the 800x600 camera rays. The balls of overlaps have
radius 0.05. Every answer is checked against the other variant. Per scene a line gives the closest-hit query's Mrays/s on
the 800x600 camera rays. Scenes: the cover scene (484 spheres), C4's 10k-sphere scene and a 100k-sphere one of the same
generator. The first line names the card and its power limit."""
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
from occlusion_bench import _spheres, measure  # noqa: E402
from rtb200 import scenes  # noqa: E402


def point_sets(sc, rs, rng, k=480_000):
    c, r = _spheres(sc)
    ok = np.flatnonzero((np.abs(c) < 1e6).all(axis=1) & (np.abs(r) < 100))
    cc, rr = c[ok], np.abs(r[ok])
    lo, hi = cc.min(axis=0), cc.max(axis=0)
    u = rng.normal(size=(k, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    j = rng.integers(0, len(ok), size=k)
    o, d = camera_rays(sc, 800, 600)
    h = rs.intersect(o, d, outputs=("sphere", "point"))
    return {"uniform_in_box": lo + rng.random((k, 3)) * (hi - lo),
            "near_surfaces": cc[j] + u * (rr[j] + rng.uniform(-1e-3, 1e-3, size=k))[:, None],
            "camera_first_hits": np.ascontiguousarray(h["point"][h["sphere"] >= 0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    rng = np.random.default_rng(9)
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)
    cases = [("cover", lambda: scenes.cover_scene(800, 600, 1)),
             ("c4_10k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), 800, 600, 1, 50))),
             ("rtiow_100k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(158), 800, 600, 1, 50)))]
    near = lambda rs: lambda p, b, t, s: rs.nearest(p, stream=s)          # noqa: E731
    over = lambda rs: lambda p, b, t, s: rs.overlaps(p, b, stream=s)      # noqa: E731
    clo = lambda rs: lambda o, d, t, s: rs.intersect(o, d, stream=s, outputs=("sphere",))   # noqa: E731
    for name, mk in cases:
        sc = mk()
        hs = {v: R.ResidentScene(sc, R.make_options(variant=vv)) for v, vv in (("filtered", R.RT_VARIANT_FILTERED),
                                                                                 ("brute_force", R.RT_VARIANT_BRUTE_FORCE))}
        try:
            o, d = camera_rays(sc, 800, 600)
            med = measure(clo(hs["filtered"]), o, d, None, args.reps)
            rec = {"scene": name, "spheres": sc.n_spheres, "yardstick": "intersect camera_800x600", "n": len(o),
                   "median_ms": round(med, 4), "mrays_per_s": round(len(o) / med / 1e3, 1)}
            lines.append(rec)
            print(json.dumps(rec), flush=True)
            for set_name, p in point_sets(sc, hs["filtered"], rng).items():
                n = len(p)
                rad = np.full(n, 0.05)
                rec = {"scene": name, "spheres": sc.n_spheres, "points": set_name, "n": n}
                ans = {}
                for v, rs in hs.items():
                    hn, ho = rs.nearest(p), rs.overlaps(p, rad)
                    ans[v] = (hn["sphere"], hn["distance"].view(np.uint64), ho["overlaps"])
                    for kind, q, st in (("nearest", near(rs), hn["stats"]), ("overlaps", over(rs), ho["stats"])):
                        med = measure(q, p, rad, None, args.reps if v == "filtered" else max(3, args.reps // 4))
                        rec[f"{kind}_{v}"] = {"median_ms": round(med, 4), "mqueries_per_s": round(n / med / 1e3, 2),
                                              "exact_per_point": round(st["candidates"] / n, 2),
                                              "leaves_per_point": round(st["clusters"] / n, 3), "nodes_per_point": round(st["nodes"] / n, 3)}
                assert all(np.array_equal(a, b) for a, b in zip(ans["filtered"], ans["brute_force"])), (name, set_name)
                rec["overlap_fraction"] = round(float(ans["filtered"][2].mean()), 4)
                for kind in ("nearest", "overlaps"):
                    rec[f"{kind}_speedup"] = round(rec[f"{kind}_filtered"]["mqueries_per_s"] / rec[f"{kind}_brute_force"]["mqueries_per_s"], 2)
                lines.append(rec)
                print(json.dumps(rec), flush=True)
        finally:
            for rs in hs.values():
                rs.release()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
