"""Depth of field on an H100 (DESIGN.md §4.17): Mrays/s and rays per sample of the cover scene's C2 view at the book's lens
(aperture 0.1, focus 10) against the pinhole, the same view at 1920x1080x64, and the cost of the lens draw itself (the trace time of a
1-sample lens frame at max_depth 1 against the pinhole's). Prints one JSON object with the card's name and power limit.

    python tools/lens_bench.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "rust-raytracer_b200"))
import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402

CONFIGS = {"C2": (800, 600, 128), "cover_1080p": (1920, 1080, 64)}   # the cover scene's view at two sizes


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(0), "?")
    return {"gpu": name, "power_limit": power}


def timed(rs, buf, reps: int) -> dict:
    rs.render(0, buf.data_ptr())   # warm-up
    best = None
    for _ in range(reps):
        st = rs.render(0, buf.data_ptr())
        if best is None or st["trace_ms"] < best["trace_ms"]:
            best = st
    return {"trace_ms": best["trace_ms"], "rays": best["rays"], "samples": best["samples"],
            "mrays_s": best["rays"] / best["trace_ms"] / 1e3, "rays_per_sample": best["rays"] / max(best["samples"], 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    out = {**card()}
    for name, (w, h, spp) in CONFIGS.items():
        for depth, label in ((50, ""), (1, "_draw")):
            s = 1 if label else spp
            sc = scenes.cover_scene(w, h, s, depth=depth)
            buf = torch.empty((h, w, 3), dtype=torch.float32, device="cuda:0")
            rs = R.ResidentScene(sc, R.make_options(device=0))
            pin = timed(rs, buf, a.reps)
            cam, lens = R.camera_from_params_lens(**{k: sc.camera_params[k] for k in ("look_from", "look_at", "vup")},
                                                  vfov=sc.camera_params["vfov"], aspect=sc.camera_params["aspect"], aperture=0.1, focus_dist=10.0)
            rs.release()
            sc.c.camera = cam
            rs = R.ResidentScene(sc, R.make_options(device=0))
            rs.set_lens(lens)
            lz = timed(rs, buf, a.reps)
            rs.release()
            out[name + label] = {"pinhole": pin, "lens": lz, "lens_over_pinhole_time": lz["trace_ms"] / pin["trace_ms"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
