"""Animations: one N-frame rtb200_render_frames_device call against N one-frame calls on the same resident scene.

Renders an orbit of the cover scene around its centre and alternates the two arms run by run on one handle, so that both
see the same card state. Prints the card (name, power limit, SM clock) and, per size and arm, Mrays/s from the CUDA-event
time of the calls (device_ms) and from their wall time, and checks that both arms computed identical frames.

    python tools/frames_bench.py [--runs 5] [--json out.json]

Sizes: 160x120x16 N=64, 400x300x16 N=32, 800x600x128 N=4 at the default sample-buffer cap (1 GiB: every 800x600x128 frame is
its own launch) and at a 4 GiB cap (the four frames would fit one launch, but frames of more than 2^24 samples are traced one
launch each). RTB200_PRINT_TAIL is reported for one launch of each arm at the smallest size.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "rust-raytracer_b200"))

import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402

SIZES = [(160, 120, 16, 64, 0), (400, 300, 16, 32, 0), (800, 600, 128, 4, 0), (800, 600, 128, 4, 4 << 30)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return out


def orbit(sc, n):
    frames = []
    for i in range(n):
        a = math.atan2(3.0, 13.0) + 2.0 * math.pi * i / n
        frames.append(R.make_frame(sc, look_from=[13.4 * math.cos(a), 2.0, 13.4 * math.sin(a)], seed=1000 + i))
    return frames


def arm_batched(rs, frames, out):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = rs.render_frames(frames, out.data_ptr())
    return st["device_ms"], (time.perf_counter() - t0) * 1e3, st["rays"], st["kernel_launches"], st["trace_ms"]


def arm_loop(rs, frames, out, frame_elems):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dev = trace = 0.0; rays = launches = 0
    for i, f in enumerate(frames):
        st = rs.render_frames([f], out.data_ptr() + i * frame_elems)
        dev += st["device_ms"]; trace += st["trace_ms"]; rays += st["rays"]; launches += st["kernel_launches"]
    return dev, (time.perf_counter() - t0) * 1e3, rays, launches, trace


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    info = {"card": card(), "sizes": []}
    print(f"card (name, power limit, SM clock): {info['card']}", flush=True)
    for w, h, spp, n, cap in SIZES:
        sc = scenes.cover_scene(w, h, spp)
        frames = orbit(sc, n)
        rs = R.ResidentScene(sc, R.make_options(sample_buffer_bytes=cap))
        frame_elems = w * h * 3
        outs = {a: torch.zeros(n * frame_elems, dtype=torch.uint8, device="cuda") for a in ("batched", "loop")}
        run = {"batched": lambda: arm_batched(rs, frames, outs["batched"]), "loop": lambda: arm_loop(rs, frames, outs["loop"], frame_elems)}
        for a in ("batched", "loop"):   # warm-up: modules, buffers, occupancy queries
            run[a]()
        if (w, h) == SIZES[0][:2]:   # frame tail of one launch of each arm (printed by the library to stderr)
            def tail(what, call):
                print(f"[{w}x{h}x{spp} N={n}] {what}:", flush=True)
                os.environ["RTB200_PRINT_TAIL"] = "1"
                call()
                os.environ.pop("RTB200_PRINT_TAIL")
                sys.stderr.flush()
            tail("batched, the one launch of all frames", lambda: rs.render_frames(frames, outs["batched"].data_ptr()))
            tail("loop, a one-frame launch", lambda: rs.render_frames(frames[-1:], outs["loop"].data_ptr() + (n - 1) * frame_elems))
        res = {"batched": [], "loop": []}
        for _ in range(args.runs):
            for a in ("batched", "loop"):
                res[a].append(run[a]())
        torch.cuda.synchronize()
        same = bool(torch.equal(outs["batched"], outs["loop"]))
        entry = {"size": f"{w}x{h}x{spp}", "frames": n, "cap_bytes": cap or (1 << 30), "identical": same}
        for a in ("batched", "loop"):
            rays = res[a][0][2]
            assert all(r[2] == rays for r in res[a]), "ray counts differ between runs"
            dev = [rays / r[0] / 1e3 for r in res[a]]
            wall = [rays / r[1] / 1e3 for r in res[a]]
            entry[a] = {"rays": rays, "launches": res[a][0][3], "mrays_device": dev, "mrays_wall": wall,
                        "median_device_ms": statistics.median(r[0] for r in res[a]), "median_wall_ms": statistics.median(r[1] for r in res[a]),
                        "median_trace_ms": statistics.median(r[4] for r in res[a])}
        assert entry["batched"]["rays"] == entry["loop"]["rays"]
        info["sizes"].append(entry)
        rs.release()
        fmt = lambda v: f"{min(v):.0f}-{max(v):.0f}"
        print(f"{entry['size']} N={n} cap={entry['cap_bytes'] >> 20} MiB identical={same}: "
              f"batched ({entry['batched']['launches']} launches) device {fmt(entry['batched']['mrays_device'])} wall {fmt(entry['batched']['mrays_wall'])} Mrays/s | "
              f"loop ({entry['loop']['launches']} launches) device {fmt(entry['loop']['mrays_device'])} wall {fmt(entry['loop']['mrays_wall'])} Mrays/s | "
              f"median trace ms batched {entry['batched']['median_trace_ms']:.2f} loop {entry['loop']['median_trace_ms']:.2f}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(info, f, indent=1)
    if not all(e["identical"] for e in info["sizes"]):
        sys.exit("the two arms computed different frames")


if __name__ == "__main__":
    main()
