"""Time and error of the variance-guided denoise (rtb200.denoise_var on CUDA tensors, DESIGN.md §4.18) against the existing denoise
(§4.15) on one GPU.

    python tools/denoise_var_bench.py [--runs 3] [--iters 20] [--iterations 1,2,3,4,5] [--scenes C2,C4] [--no-quality]

Per scene (C2: the cover scene at 800x600; C4: 10,000 spheres at 1920x1080). A frame of n spp is the render of the view at
n spp with the variance of its pixel means (rtb200_render_frames_var_device) and the AOV albedo and normal of its own samples
as guides.
  * "resolve": the same 4-spp frame through rtb200_render_frames_device and rtb200_render_frames_var_device, alternating,
    ms per call (CUDA events): the difference is the variance resolve's cost;
  * "time": rtb200_denoise_var_device and rtb200_denoise_device at each iteration count L on the 4-spp frame at the defaults,
    scratch and outputs allocated once, `--iters` calls per timed window, the arms alternating within a run and the runs
    repeating the set; CUDA events around each window; "host_ms" is the host's time per call to enqueue the window;
  * "quality" (unless --no-quality): MSE against the 1024-spp render of the view at 4, 8, 16 and 32 spp of the raw mean, the
    existing denoise and the variance-guided one, at the defaults;
  * "adaptive" (unless --no-quality): an adaptive render (rel_tol 0.05, rounds of 8 samples, 8 to 64 per pixel) with its
    variance (rtb200_adaptive_resolve_var), raw and denoised both ways, against the 1024-spp render.
Prints the device and its power limit, then one JSON line per scene and part."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "rust-raytracer_b200"))

import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402


def timed(fn, iters, host=None):
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


def frame_of(sc, spp):
    """(mean, variance, albedo, normal) of the render of the view at spp, CUDA tensors [h, w, 3]."""
    w, h = int(sc.c.width), int(sc.c.height)
    sc.c.samples_per_pixel = spp
    rs = R.ResidentScene(sc)
    try:
        mean = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        var = torch.empty_like(mean)
        rs.render_frames([R.make_frame(sc)], 0, mean.data_ptr(), stream=stream_handle(), variance=var.data_ptr())
        aov = rs.aov(spp, on_device=True, outputs=("albedo", "normal"))
        torch.cuda.synchronize()
        return mean, var, aov["albedo"], aov["normal"]
    finally:
        rs.release()


def truth_of(sc, spp):
    sc.c.samples_per_pixel = spp
    rs = R.ResidentScene(sc)
    try:
        lin = torch.empty((int(sc.c.height), int(sc.c.width), 3), dtype=torch.float32, device="cuda")
        rs.render(0, lin.data_ptr(), stream=stream_handle())
        torch.cuda.synchronize()
        return lin
    finally:
        rs.release()


def mse(a, b):
    return float(torch.mean((a.double() - b.double()) ** 2))


def old_denoise(mean, alb, nrm, L=R.DENOISE_ITERATIONS):
    return R.denoise(mean, alb, nrm, iterations=L)["linear"]


def new_denoise(mean, var, alb, nrm, L=R.DENOISE_VAR_ITERATIONS):
    return R.denoise_var(mean, var, alb, nrm, iterations=L)["linear"]


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
    L_ = R.lib()
    for name in args.scenes.split(","):
        sc = scenes.scene(name)
        w, h = int(sc.c.width), int(sc.c.height)
        mean, var, alb, nrm = frame_of(sc, 4)
        s_old = torch.empty(int(L_.rtb200_denoise_scratch_bytes(w, h)), dtype=torch.uint8, device="cuda")
        s_new = torch.empty(int(L_.rtb200_denoise_var_scratch_bytes(w, h)), dtype=torch.uint8, device="cuda")
        dst = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        arms = {}
        for L in levels:
            po = R.rt_denoise_params(w, h, L, 0, R.DENOISE_COLOR_WEIGHT, R.DENOISE_ALBEDO_WEIGHT, R.DENOISE_NORMAL_WEIGHT, 0.0)
            pn = R.rt_denoise_var_params(w, h, L, 0, R.DENOISE_VAR_COLOR_WEIGHT, R.DENOISE_VAR_ALBEDO_WEIGHT,
                                         R.DENOISE_VAR_NORMAL_WEIGHT, R.DENOISE_VAR_VARIANCE_FLOOR)

            def old(p=po):
                R._check(L_.rtb200_denoise_device(0, C.byref(p), mean.data_ptr(), alb.data_ptr(), nrm.data_ptr(), s_old.data_ptr(),
                                                  dst.data_ptr(), None, stream_handle()))

            def new(p=pn):
                R._check(L_.rtb200_denoise_var_device(0, C.byref(p), mean.data_ptr(), var.data_ptr(), alb.data_ptr(), nrm.data_ptr(),
                                                      s_new.data_ptr(), dst.data_ptr(), None, None, stream_handle()))
            new()
            want = R.denoise_var(mean, var, alb, nrm, iterations=L)["linear"]
            torch.cuda.synchronize()
            assert torch.equal(dst.view(torch.int32), want.view(torch.int32)), (name, L)
            arms[("denoise", L)], arms[("denoise_var", L)] = old, new
        out = {"scene": name, "width": w, "height": h, "part": "time", "ms": {}, "host_ms": {}}
        for fn in arms.values():   # warm-up
            timed(fn, 2)
        for _ in range(args.runs):
            for (kind, L), fn in arms.items():
                host = out["host_ms"].setdefault(f"{kind} L={L}", [])
                out["ms"].setdefault(f"{kind} L={L}", []).append(round(timed(fn, args.iters, host), 4))
        print(json.dumps(out), flush=True)

        sc.c.samples_per_pixel = 4
        rs = R.ResidentScene(sc)
        f = [R.make_frame(sc)]
        res = {"scene": name, "part": "resolve", "ms": {"render": [], "render_var": []}}
        arms_r = {"render": lambda: rs.render_frames(f, 0, dst.data_ptr(), stream=stream_handle()),
                  "render_var": lambda: rs.render_frames(f, 0, dst.data_ptr(), stream=stream_handle(), variance=var.data_ptr())}
        for fn in arms_r.values():
            timed(fn, 2)
        for _ in range(args.runs):
            for k, fn in arms_r.items():
                res["ms"][k].append(round(timed(fn, 5), 4))
        rs.release()
        print(json.dumps(res), flush=True)
        if args.no_quality:
            continue
        truth = truth_of(sc, 1024)
        q = {"scene": name, "part": "quality", "reference_spp": 1024, "mse": {}}
        for spp in (4, 8, 16, 32):
            m, v, a, n = frame_of(sc, spp)
            q["mse"][spp] = {"raw": mse(m, truth), "denoise": mse(old_denoise(m, a, n), truth),
                             "denoise_var": mse(new_denoise(m, v, a, n), truth)}
            del m, v, a, n
        print(json.dumps(q), flush=True)

        sc.c.samples_per_pixel = 64
        rs = R.ResidentScene(sc)
        try:
            p = R.make_adaptive(0.05, 0.0, samples_per_round=8, min_samples=8)
            rs.adaptive_begin(p)
            _, st = rs.adaptive_step(1000)
            m = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
            v = torch.empty_like(m)
            cnt = torch.empty((h, w), dtype=torch.int32, device="cuda")
            rs.adaptive_resolve(linear=m, counts=cnt, variance=v)
            aov = rs.aov(8, on_device=True, outputs=("albedo", "normal"))
            torch.cuda.synchronize()
        finally:
            rs.release()
        ad = {"scene": name, "part": "adaptive", "mean_spp": float(cnt.double().mean()), "mse": {
            "raw": mse(m, truth), "denoise": mse(old_denoise(m, aov["albedo"], aov["normal"]), truth),
            "denoise_var": mse(new_denoise(m, v, aov["albedo"], aov["normal"]), truth)}}
        print(json.dumps(ad), flush=True)


if __name__ == "__main__":
    main()
