#!/usr/bin/env python3
"""Adaptive rendering on the cover scene (DESIGN.md §4.9): for a few rel_tol values, the samples traced as a share of
N * pixels, device and wall time against the one-shot N-spp render on the same resident handle, and the linear RMSE against a
reference render of the same seed at `--ref-spp` and against a fixed-spp render that traces about as many samples.

    python tools/adaptive_bench.py [--w 800 --h 600 --spp 128 --m 8 --min 16 --rel 0.02,0.05,0.1,0.2] [--out result.json]

Prints one JSON object; the card and its power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rust-raytracer_b200"))
import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the numbers still stand; say what is missing
        q = f"nvidia-smi unavailable: {e}"
    return q


def rmse(a, b):
    ok = np.isfinite(a).all(-1) & np.isfinite(b).all(-1)
    d = a[ok].astype(np.float64) - b[ok].astype(np.float64)
    return float(np.sqrt((d * d).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--w", type=int, default=800); ap.add_argument("--h", type=int, default=600)
    ap.add_argument("--spp", type=int, default=128); ap.add_argument("--m", type=int, default=8)
    ap.add_argument("--min", type=int, default=16); ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--rel", default="0.02,0.05,0.1,0.2"); ap.add_argument("--abs", type=float, default=0.0)
    ap.add_argument("--reps", type=int, default=3); ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    npix = a.w * a.h
    sc = scenes.cover_scene(a.w, a.h, a.spp)
    rs = R.ResidentScene(sc)
    o8 = torch.zeros(npix * 3, dtype=torch.uint8, device="cuda")
    ol = torch.zeros(npix * 3, dtype=torch.float32, device="cuda")

    def one_shot():
        t = time.perf_counter()
        st = rs.render(o8.data_ptr(), ol.data_ptr())
        return st["device_ms"], (time.perf_counter() - t) * 1e3

    def adaptive(p):
        t = time.perf_counter()
        rs.adaptive_begin(p, stream=0)
        active, st = rs.adaptive_step(1 << 20, stream=0)
        rs.adaptive_resolve(o8, ol, stream=0)
        return st, (time.perf_counter() - t) * 1e3

    one_shot()   # warm-up: work buffers, occupancy queries
    base = [one_shot() for _ in range(a.reps)]
    base_dev = statistics.median(b[0] for b in base); base_wall = statistics.median(b[1] for b in base)
    ref_sc = scenes.cover_scene(a.w, a.h, a.ref_spp)
    ref, _ = R.render_linear(ref_sc)
    full, _ = R.render_linear(sc)
    res = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "scene": f"cover {a.w}x{a.h}", "N": a.spp, "m": a.m,
           "min_samples": a.min, "abs_tol": a.abs, "ref_spp": a.ref_spp,
           "one_shot": {"device_ms": base_dev, "wall_ms": base_wall, "rmse_vs_ref": rmse(full, ref)}, "runs": []}
    for rel in [float(x) for x in a.rel.split(",")]:
        p = R.make_adaptive(rel, a.abs, samples_per_round=a.m, min_samples=a.min)
        adaptive(p)   # warm-up (allocates the state at the first begin)
        runs = [adaptive(p) for _ in range(a.reps)]
        st = runs[-1][0]
        dev = statistics.median(r[0]["device_ms"] for r in runs); wall = statistics.median(r[1] for r in runs)
        lin = ol.cpu().numpy().reshape(a.h, a.w, 3)
        share = st["samples"] / (a.spp * npix)
        eq = max(1, round(st["samples"] / npix))
        eq_sc = scenes.cover_scene(a.w, a.h, eq)
        eq_lin, _ = R.render_linear(eq_sc)
        res["runs"].append({"rel_tol": rel, "samples_share": share, "rounds": st["batches"], "kernel_launches": st["kernel_launches"],
                            "device_ms": dev, "wall_ms": wall, "device_vs_one_shot": dev / base_dev, "wall_vs_one_shot": wall / base_wall,
                            "rmse_vs_ref": rmse(lin, ref), "fixed_spp_same_samples": eq, "fixed_rmse_vs_ref": rmse(eq_lin, ref)})
    rs.release()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt)


if __name__ == "__main__":
    main()
