"""Time and quality of the temporal accumulation (rtb200.temporal on CUDA tensors, DESIGN.md §4.16) on one GPU.

    python tools/temporal_bench.py [--runs 3] [--iters 50] [--frames 16] [--ref-spp 1024] [--no-quality]

  * "kernel": rtb200_temporal_device at 800x600 and 1920x1080 with every buffer allocated once (a random frame reprojected
    through a 1-degree orbit step, so that most pixels gather four taps), `--iters` calls per timed window, the two sizes
    alternating within a run and the runs repeating the pair; CUDA events around each window. "host_ms" is the host's time per
    call to enqueue the window: while it stays below "ms" the GPU never waits for the host. The traffic floor is 56 B per pixel
    (40 B of the pixel's own inputs and 16 B out; neighbours that hit in cache are not counted), and GB/s is that floor over
    the measured time;
  * "quality" (unless --no-quality): an orbit of C2 of `--frames` frames at 4 spp with distinct seeds, 1 degree per frame,
    against a `--ref-spp` render of each frame: the per-frame MSE and the flicker error mean |(o_k - o_k-1) - (r_k - r_k-1)|^2 of
    the raw frames, of the denoise alone and of temporal accumulation followed by the denoise (both at the defaults).
Prints the device, its power limit and SM clock read in the same run, then one JSON line per part."""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "rust-raytracer_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402

FLOOR_BYTES = 56


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


def orbit_camera(sc, deg):
    a = math.atan2(3.0, 13.0) + math.radians(deg)
    return R.make_frame(sc, look_from=[13.4 * math.cos(a), 2.0, 13.4 * math.sin(a)], seed=1000 + int(round(deg)))


def kernel_arm(w, h):
    """One preallocated call at w x h: random colours, points on the current camera's rays, and a previous frame one degree away."""
    sc = scenes.cover_scene(w, h, 1)
    cam, pcam = orbit_camera(sc, 1.0).camera, orbit_camera(sc, 0.0).camera
    g = torch.Generator(device="cuda").manual_seed(w)
    o = torch.tensor([cam.origin.x, cam.origin.y, cam.origin.z], dtype=torch.float64, device="cuda")
    llc = torch.tensor([cam.lower_left_corner.x, cam.lower_left_corner.y, cam.lower_left_corner.z], dtype=torch.float64, device="cuda")
    hh = torch.tensor([cam.horizontal.x, cam.horizontal.y, cam.horizontal.z], dtype=torch.float64, device="cuda")
    vt = torch.tensor([cam.vertical.x, cam.vertical.y, cam.vertical.z], dtype=torch.float64, device="cuda")
    ys, xs = torch.meshgrid(torch.arange(h, device="cuda", dtype=torch.float64), torch.arange(w, device="cuda", dtype=torch.float64), indexing="ij")
    u, v = (xs + 0.5) / (w - 1), (h - ys - 0.5) / (h - 1)
    d = llc + hh * u[..., None] + vt * v[..., None] - o
    t = 10.0 + torch.rand((h, w, 1), generator=g, device="cuda", dtype=torch.float64)
    point = (o + d * t).contiguous()
    sphere = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    color = torch.rand((h, w, 3), generator=g, device="cuda")
    prev = {"color": torch.rand((h, w, 3), generator=g, device="cuda"), "length": torch.full((h, w), 3, dtype=torch.uint32, device="cuda"),
            "sphere": sphere.clone(), "point": point.clone(), "camera": pcam}
    want = R.temporal(color, sphere, point, cam, prev, depth_tol=1e6)
    out_c, out_n = torch.empty_like(want["color"]), torch.empty_like(want["length"])
    p = R.rt_temporal_params(w, h, R.TEMPORAL_MAX_HISTORY, 0, cam, pcam, 1e6)
    cur = R.rt_temporal_frame(color.data_ptr(), sphere.data_ptr(), point.data_ptr())
    hist = R.rt_temporal_history(prev["color"].data_ptr(), prev["length"].data_ptr(), prev["sphere"].data_ptr(), prev["point"].data_ptr())
    out = R.rt_temporal_out(out_c.data_ptr(), out_n.data_ptr())

    def arm():
        R._check(R.lib().rtb200_temporal_device(0, C.byref(p), C.byref(cur), C.byref(hist), None, C.byref(out), stream_handle()))
    arm()
    torch.cuda.synchronize()
    assert torch.equal(out_c.view(torch.int32), want["color"].view(torch.int32)) and torch.equal(out_n, want["length"])
    kept = float((out_n.to(torch.int64) > 1).double().mean())
    return arm, kept, (color, sphere, point, prev, out_c, out_n)


def linear_and_aov(rs, frames, spp):
    w, h = int(rs.scene.c.width), int(rs.scene.c.height)
    lin = torch.empty((len(frames), h, w, 3), dtype=torch.float32, device="cuda")
    rs.render_frames(frames, 0, lin.data_ptr(), stream=stream_handle())
    aovs = [rs.aov(spp, view=f, on_device=True, outputs=("albedo", "normal", "sphere", "point")) for f in frames]
    torch.cuda.synchronize()
    return lin, aovs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--no-quality", action="store_true")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[:1]}), flush=True)

    sizes = [(800, 600), (1920, 1080)]
    arms, keep = {}, []
    out = {"part": "kernel", "ms": {}, "host_ms": {}, "taps_kept": {}}
    for w, h in sizes:
        arm, kept, bufs = kernel_arm(w, h)
        arms[(w, h)] = arm
        keep.append(bufs)
        out["taps_kept"][f"{w}x{h}"] = round(kept, 4)
        timed(arm, 5)
    for _ in range(args.runs):
        for w, h in sizes:
            key = f"{w}x{h}"
            out["ms"].setdefault(key, []).append(round(timed(arms[(w, h)], args.iters, out["host_ms"].setdefault(key, [])), 5))
    out["floor_gbs"] = {f"{w}x{h}": [round(FLOOR_BYTES * w * h / (ms * 1e-3) / 1e9, 1) for ms in out["ms"][f"{w}x{h}"]] for w, h in sizes}
    print(json.dumps(out), flush=True)
    if args.no_quality:
        return

    sc = scenes.scene("C2")
    frames = [orbit_camera(sc, float(i)) for i in range(args.frames)]
    sc.c.samples_per_pixel = 4
    rs = R.ResidentScene(sc)
    lin, aovs = linear_and_aov(rs, frames, 4)
    rs.release()
    sc.c.samples_per_pixel = args.ref_spp
    ref_rs = R.ResidentScene(sc)
    ref, _ = linear_and_aov(ref_rs, frames, 1)
    ref_rs.release()
    seqs = {"raw": [], "spatial": [], "temporal_spatial": []}
    td = R.TemporalDenoiser()
    for i, f in enumerate(frames):
        a = aovs[i]
        seqs["raw"].append(lin[i])
        seqs["spatial"].append(R.denoise(lin[i], a["albedo"], a["normal"])["linear"])
        seqs["temporal_spatial"].append(td.push(lin[i], a, f)["denoised"])
    torch.cuda.synchronize()
    q = {"part": "quality", "scene": "C2", "frames": args.frames, "spp": 4, "reference_spp": args.ref_spp, "orbit_deg_per_frame": 1.0}
    for k, s in seqs.items():
        mse = [float(torch.mean((s[i].double() - ref[i].double()) ** 2)) for i in range(len(frames))]
        fl = [float(torch.mean(((s[i] - s[i - 1]).double() - (ref[i] - ref[i - 1]).double()) ** 2)) for i in range(1, len(frames))]
        q[k] = {"mse_per_frame": [round(m, 7) for m in mse], "mse_last": round(mse[-1], 7), "mse_mean_after_first_4": round(float(np.mean(mse[4:])), 7),
                "flicker": round(float(np.mean(fl)), 7)}
    print(json.dumps(q), flush=True)


if __name__ == "__main__":
    main()
