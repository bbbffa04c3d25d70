#!/usr/bin/env python3
"""Throughput of caller-supplied primary rays (ResidentScene.trace_rays, DESIGN.md §4.12) against the resident render on the
BASELINE C2 scene and view (cover scene, 800x600, depth 50).

    python tools/trace_rays_bench.py [--reps 5] [--samples 128] [--jitter-samples 8] [--out trace_rays_bench.jsonl]

(a) the 800x600 pixel-centre camera rays with `samples` samples in ONE call, against rtb200_render_device at the same spp;
(b) the render's own jittered primary rays (built with the oracle's RNG and Camera::get_ray), one samples = 1 call per
    sample, against the render at spp = jitter-samples; the summed, scaled calls are checked bit for bit against the render.
Mrays/s = rays (hit_world calls) / device ms, median of `reps` runs after one warm-up. The first line names the card and
its power limit. (b) needs oracle/liboracle.so (built by __graft_entry__.build())."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rust-raytracer_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import rtb200 as R  # noqa: E402
from intersect_bench import camera_rays, card  # noqa: E402
from rtb200 import scenes  # noqa: E402


def _render(rs, torch, spp):
    n = rs.rows * rs.scene.c.width * 3
    dl = torch.empty(n, dtype=torch.float32, device="cuda")
    st = rs.render(0, dl.data_ptr())
    return dl, st


def _med(xs):
    return float(np.median(xs))


def main(argv=None):
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--jitter-samples", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)

    # (a) pixel-centre rays, one call of `samples` samples, against the render at spp = samples
    sc = scenes.scene("C2")
    sc.resize(800, 600, spp=a.samples)
    rs = R.ResidentScene(sc)
    o, d = camera_rays(sc, 800, 600)
    do, dd = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    try:
        rays_t, ms_t, rays_r, ms_r = [], [], [], []
        for k in range(a.reps + 1):
            st = rs.trace_rays(do, dd, a.samples)["stats"]
            _, sr = _render(rs, torch, a.samples)
            if k:
                rays_t.append(st["rays"]); ms_t.append(st["device_ms"]); rays_r.append(sr["rays"]); ms_r.append(sr["device_ms"])
        line = {"case": "a_pixel_centres_one_call", "n": len(o), "samples": a.samples, "batches": st["batches"],
                "trace_rays_mrays_s": _med(np.array(rays_t) / np.array(ms_t) / 1e3), "trace_rays_ms": _med(ms_t),
                "render_mrays_s": _med(np.array(rays_r) / np.array(ms_r) / 1e3), "render_ms": _med(ms_r)}
        line["ratio"] = line["trace_rays_mrays_s"] / line["render_mrays_s"]
        lines.append(line)
        print(json.dumps(line), flush=True)
    finally:
        rs.release()

    # (b) the render's own jittered rays, one samples = 1 call per sample, against the render at spp = jitter-samples
    from test_trace_rays_cpu import primary_rays, sum_samples
    S = a.jitter_samples
    sc = scenes.scene("C2")
    sc.resize(800, 600, spp=S)
    rays = [tuple(torch.from_numpy(x).cuda() for x in primary_rays(sc, s)) for s in range(S)]
    rs = R.ResidentScene(sc)
    try:
        per_ms, per_rays, ren_ms, ren_rays = [], [], [], []
        for k in range(a.reps + 1):
            outs, ms, nr = [], 0.0, 0
            for s in range(S):
                h = rs.trace_rays(*rays[s], 1, sample0=s)
                outs.append(h["linear"]); ms += h["stats"]["device_ms"]; nr += h["stats"]["rays"]
            dl, sr = _render(rs, torch, S)
            if k == 0:
                lin = sum_samples([x.cpu().numpy() for x in outs], S)
                assert np.array_equal(lin.reshape(-1).view(np.uint32), dl.cpu().numpy().view(np.uint32)), "per-sample calls differ from the render"
                assert nr == sr["rays"]
            else:
                per_ms.append(ms); per_rays.append(nr); ren_ms.append(sr["device_ms"]); ren_rays.append(sr["rays"])
        line = {"case": "b_render_rays_one_call_per_sample", "n": 800 * 600, "samples": S, "bit_identical_to_render": True,
                "trace_rays_mrays_s": _med(np.array(per_rays) / np.array(per_ms) / 1e3), "trace_rays_ms": _med(per_ms),
                "render_mrays_s": _med(np.array(ren_rays) / np.array(ren_ms) / 1e3), "render_ms": _med(ren_ms)}
        line["ratio"] = line["trace_rays_mrays_s"] / line["render_mrays_s"]
        lines.append(line)
        print(json.dumps(line), flush=True)
    finally:
        rs.release()
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
