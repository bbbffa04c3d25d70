#!/usr/bin/env python3
"""Does L1 capacity limit the trace kernel? Renders a BASELINE config resident (like tools/render_once.py) with several
library builds, alternated round by round in fresh processes, and prints the card, its power limit and the SM clock
beside every rate.

usage: l1_probe.py [--config C2] [--rounds 3] [--reps 6] LABEL=LIB[@CARVEOUT_PCT] ...

Each build is a librtb200.so loaded with RTB200_LIB. @CARVEOUT_PCT pins the trace kernel's shared-memory carveout with
RTB200_WF_CARVEOUT (percent of the SM's shared memory, rounded up by the hardware to its next step; 100 = 228 KiB on an
H100, leaving 28 KiB of L1). Running one build with and without a pinned carveout isolates L1 capacity from any code
change: the kernel is the same binary and only the L1 left beside its shared memory differs (DESIGN.md §4.5)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CHILD = r"""
import json, sys, os
sys.path.insert(0, os.path.join(sys.argv[1], 'rust-raytracer_b200'))
import rtb200 as R
from rtb200 import scenes
import torch
name, reps = sys.argv[2], int(sys.argv[3])
sc = scenes.scene(name)
rs = R.ResidentScene(sc, R.make_options(variant=0, rank=0, world=1))
ki = rs.kernel_info()
out = torch.empty(sc.c.height * sc.c.width * 3, dtype=torch.uint8, device='cuda')
for _ in range(2):
    rs.render(out.data_ptr())
rates = []
for _ in range(reps):
    st = rs.render(out.data_ptr())
    rates.append(st['rays'] / st['device_ms'] / 1e3)
print(json.dumps({"rates": rates, "rays": st['rays'], "registers": ki['registers'], "local_bytes": ki['local_bytes'],
                  "smem_bytes": ki['smem_bytes'], "ctas_per_sm": ki['ctas_per_sm']}))
"""


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "nvidia-smi unavailable"


def run(lib, pct, config, reps):
    env = dict(os.environ, RTB200_LIB=os.path.abspath(lib))
    env.pop("RTB200_WF_CARVEOUT", None)
    if pct is not None:
        env["RTB200_WF_CARVEOUT"] = str(pct)
    r = subprocess.run([sys.executable, "-c", _CHILD, REPO, config, str(reps)], env=env, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(f"{lib}: exit {r.returncode}\n{r.stderr[-2000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("builds", nargs="+", help="LABEL=LIB[@CARVEOUT_PCT]")
    a = ap.parse_args()
    builds = []
    for b in a.builds:
        label, spec = b.split("=", 1)
        lib, _, pct = spec.partition("@")
        builds.append((label, lib, int(pct) if pct else None))
    print(f"card, power limit, SM clock, max SM clock: {gpu_state()}", flush=True)
    per = {label: [] for label, _, _ in builds}
    for rnd in range(a.rounds):
        for label, lib, pct in builds:
            res = run(lib, pct, a.config, a.reps)
            m = statistics.mean(res["rates"])
            per[label].append(m)
            print(f"round {rnd} {label:>12}: {m:8.1f} Mrays/s (reps {min(res['rates']):.1f}-{max(res['rates']):.1f}) rays={res['rays']} "
                  f"regs={res['registers']} local={res['local_bytes']} smem={res['smem_bytes']} ctas/SM={res['ctas_per_sm']} "
                  f"carveout={'auto' if pct is None else str(pct) + '%'} | {gpu_state()}", flush=True)
    print(f"{a.config} summary over {a.rounds} alternated rounds (mean Mrays/s of {a.reps} renders per round):")
    for label, _, pct in builds:
        v = per[label]
        print(f"  {label:>12}: {min(v):8.1f} - {max(v):8.1f}  spread {max(v) - min(v):6.1f}  carveout={'auto' if pct is None else str(pct) + '%'}")


if __name__ == "__main__":
    main()
