"""Time of the denoise (rtb200.denoise on CUDA tensors, DESIGN.md §4.15) against the traffic floor, the render and AOV pass it
follows, and the error it removes, on one GPU.

    python tools/denoise_bench.py [--runs 3] [--iters 20] [--iterations 1,2,3,4,5] [--scenes C2,C4] [--no-quality]

Per scene (C2: the cover scene at 800x600; C4: 10,000 spheres at 1920x1080), with the frame's own 4-spp linear image and AOV
guides as input:
  * "denoise": rtb200_denoise_device at each iteration count L with its scratch and output allocated once, `--iters` calls
    per timed window, the counts alternating within a run and the runs repeating the set; CUDA events around each window.
    "host_ms" is the host's time per call to enqueue the window: while it stays below "ms" the GPU never waits for the host,
    so "ms" is the kernels' time and not the launch rate. The traffic floor is 48 B per pixel per iteration (12 B of colour
    in, 24 B of guides, 12 B out), and GB/s is that floor over the measured time;
  * "frame": the render (linear) and the AOV pass (albedo and normal) of the same view at 4 and 16 spp, alternated the same way;
  * "quality" (unless --no-quality): the MSE against the 1024-spp render of the view of the denoised 4-spp frame (at the
    defaults) and of the raw 4, 16 and 64-spp frames.
Prints the device and its power limit, then one JSON line per scene and part."""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "rust-raytracer_b200"))

import ctypes as C  # noqa: E402

import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402

FLOOR_BYTES = 48   # per pixel per iteration


def timed(fn, iters, host=None):
    """GPU ms per call of fn over `iters` calls (CUDA events); with a list `host`, also appends the host's ms per enqueue."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    if host is not None:
        host.append(round((time.perf_counter() - t0) * 1e3 / iters, 4))
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def stream_handle():
    return torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY


def linear_of(sc, spp):
    sc.c.samples_per_pixel = spp
    rs = R.ResidentScene(sc)
    try:
        lin = torch.empty((int(sc.c.height), int(sc.c.width), 3), dtype=torch.float32, device="cuda")
        rs.render(0, lin.data_ptr(), stream=stream_handle())
        aov = rs.aov(spp, on_device=True, outputs=("albedo", "normal"))
        torch.cuda.synchronize()
        return lin, aov
    finally:
        rs.release()


def mse(a, b):
    return float(torch.mean((a.double() - b.double()) ** 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--iterations", default="1,2,3,4,5")
    ap.add_argument("--scenes", default="C2,C4")
    ap.add_argument("--no-quality", action="store_true")
    args = ap.parse_args()
    levels = [int(x) for x in args.iterations.split(",")]
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[:1]}), flush=True)
    for name in args.scenes.split(","):
        sc = scenes.scene(name)
        w, h = int(sc.c.width), int(sc.c.height)
        npix = w * h
        lin, aov = linear_of(sc, 4)
        # tests/test_gpu_denoise.py holds rtb200.denoise to the restatement; these calls must equal it bit for bit
        scratch = torch.empty(int(R.lib().rtb200_denoise_scratch_bytes(w, h)), dtype=torch.uint8, device="cuda")
        dst = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        arms = {}
        for L in levels:
            p = R.rt_denoise_params(w, h, L, 0, R.DENOISE_COLOR_WEIGHT, R.DENOISE_ALBEDO_WEIGHT, R.DENOISE_NORMAL_WEIGHT, 0.0)

            def arm(p=p):
                R._check(R.lib().rtb200_denoise_device(0, C.byref(p), lin.data_ptr(), aov["albedo"].data_ptr(), aov["normal"].data_ptr(),
                                                       scratch.data_ptr(), dst.data_ptr(), None, stream_handle()))
            arm()
            want = R.denoise(lin, aov["albedo"], aov["normal"], iterations=L)["linear"]
            assert torch.equal(dst.view(torch.int32), want.view(torch.int32)), (name, L)
            arms[L] = arm
        out = {"scene": name, "width": w, "height": h, "part": "denoise", "ms": {L: [] for L in levels}, "host_ms": {L: [] for L in levels}}
        for L in levels:   # warm-up
            timed(arms[L], 2)
        for _ in range(args.runs):
            for L in levels:
                out["ms"][L].append(round(timed(arms[L], args.iters, out["host_ms"][L]), 4))
        out["floor_gbs"] = {L: [round(FLOOR_BYTES * npix * L / (ms * 1e-3) / 1e9, 1) for ms in out["ms"][L]] for L in levels}
        print(json.dumps(out), flush=True)

        frame = {"scene": name, "part": "frame", "render_ms": {}, "aov_ms": {}}
        residents = {}
        for spp in (4, 16):
            sc.c.samples_per_pixel = spp
            residents[spp] = R.ResidentScene(sc)
        buf = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        parts = {}
        for spp, rs in residents.items():
            parts[("render_ms", spp)] = lambda rs=rs: rs.render(0, buf.data_ptr(), stream=stream_handle())
            parts[("aov_ms", spp)] = lambda rs=rs, spp=spp: rs.aov(spp, on_device=True, outputs=("albedo", "normal"))
        for fn in parts.values():
            timed(fn, 1)
        for _ in range(args.runs):
            for (key, spp), fn in parts.items():
                frame[key].setdefault(spp, []).append(round(timed(fn, 3), 3))
        for rs in residents.values():
            rs.release()
        print(json.dumps(frame), flush=True)

        if args.no_quality:
            continue
        truth, _ = linear_of(sc, 1024)
        q = {"scene": name, "part": "quality", "reference_spp": 1024,
             "mse_denoised_4spp": mse(R.denoise(lin, aov["albedo"], aov["normal"])["linear"], truth)}
        for spp in (4, 16, 64):
            q[f"mse_raw_{spp}spp"] = mse(linear_of(sc, spp)[0], truth)
        print(json.dumps(q), flush=True)


if __name__ == "__main__":
    main()
