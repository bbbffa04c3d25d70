"""Time and quality of the temporal accumulation's history clamp (rtb200.temporal(clamp=...), DESIGN.md §4.20) on one GPU.

    python tools/temporal_clamp_bench.py [--runs 3] [--iters 50] [--frames 16] [--ref-spp 1024] [--no-quality]

  * "kernel": rtb200_temporal_device and rtb200_temporal_clamped_device at radius 1, 2 and 3 (gamma 1) on the same buffers as
    tools/temporal_bench.py (a random frame reprojected through a one-degree orbit step), `--iters` calls per timed window, the
    four calls alternating within each size and the runs repeating them; CUDA events around each window;
  * "quality" (unless --no-quality): the four rows of DESIGN.md §4.16's ablation, C2 and C2 with every metal and glass sphere
    Lambertian (metal keeps its albedo, glass gets 0.8), each under the one-degree orbit and under a static camera: `--frames`
    frames at 4 spp with distinct seeds against a `--ref-spp` render of each frame. Columns: the denoise alone, the unclamped
    accumulation at N = 2 and 4, and the clamped accumulation at N in {2, 4}, gamma in {0.5, 1, 1.5, 2, 3}, r in {1, 2}, each
    followed by the denoise at its defaults. "mse" is the mean over frames 4 .. F-1; "flicker" the mean over k >= 1 of
    |(o_k - o_k-1) - (r_k - r_k-1)|^2 (§4.16's measure) and "flicker_4" the same over k >= 4.
Prints the device, its power limit and SM clock read in the same run, then one JSON line per part."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "rust-raytracer_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))

import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402
from temporal_bench import kernel_arm, linear_and_aov, orbit_camera, stream_handle, timed  # noqa: E402

RADII = (1, 2, 3)


def clamped_arm(w, h, bufs, radius):
    """rtb200_temporal_clamped_device on kernel_arm's buffers, checked against the unclamped call's lengths."""
    color, sphere, point, prev, _, _ = bufs
    sc = scenes.cover_scene(w, h, 1)
    cam, pcam = orbit_camera(sc, 1.0).camera, orbit_camera(sc, 0.0).camera
    want = R.temporal(color, sphere, point, cam, prev, depth_tol=1e6, clamp=1.0, clamp_radius=radius)
    out_c, out_n = torch.empty_like(want["color"]), torch.empty_like(want["length"])
    p = R.rt_temporal_params(w, h, R.TEMPORAL_MAX_HISTORY, 0, cam, pcam, 1e6)
    cl = R.rt_temporal_clamp(1.0, radius)
    cur = R.rt_temporal_frame(color.data_ptr(), sphere.data_ptr(), point.data_ptr())
    hist = R.rt_temporal_history(prev["color"].data_ptr(), prev["length"].data_ptr(), prev["sphere"].data_ptr(), prev["point"].data_ptr())
    out = R.rt_temporal_out(out_c.data_ptr(), out_n.data_ptr())

    def arm():
        R._check(R.lib().rtb200_temporal_clamped_device(0, C.byref(p), C.byref(cl), C.byref(cur), C.byref(hist), None, C.byref(out),
                                                        stream_handle()))
    arm()
    torch.cuda.synchronize()
    assert torch.equal(out_c.view(torch.int32), want["color"].view(torch.int32)) and torch.equal(out_n, want["length"])
    return arm, (want, out_c, out_n)


def kernel_part(args):
    out = {"part": "kernel", "ms": {}}
    arms, keep = {}, []
    for w, h in ((800, 600), (1920, 1080)):
        arm, _, bufs = kernel_arm(w, h)
        keep.append(bufs)
        arms[(w, h, "unclamped")] = arm
        for r in RADII:
            a, k = clamped_arm(w, h, bufs, r)
            keep.append(k)
            arms[(w, h, f"clamped_r{r}")] = a
    for a in arms.values():
        timed(a, 5)
    for _ in range(args.runs):
        for (w, h, name), a in arms.items():
            out["ms"].setdefault(f"{w}x{h}/{name}", []).append(round(timed(a, args.iters), 5))
    print(json.dumps(out), flush=True)


def make_diffuse(sc):
    for i in range(sc.n_spheres):
        s = sc._spheres[i]
        if s.kind == R.RT_METAL:
            s.kind, s.param = R.RT_LAMBERTIAN, 0.0
        elif s.kind == R.RT_GLASS:
            s.kind, s.param = R.RT_LAMBERTIAN, 0.0
            s.albedo[:] = [0.8, 0.8, 0.8]


def row_inputs(diffuse, orbit, n, ref_spp):
    sc = scenes.scene("C2")
    if diffuse:
        make_diffuse(sc)
    frames = [orbit_camera(sc, float(i) if orbit else 0.0) for i in range(n)]
    for i, f in enumerate(frames):
        f.seed = 1000 + i
    sc.c.samples_per_pixel = 4
    rs = R.ResidentScene(sc)
    lin, aovs = linear_and_aov(rs, frames, 4)
    rs.release()
    sc.c.samples_per_pixel = ref_spp
    ref_rs = R.ResidentScene(sc)
    ref, _ = linear_and_aov(ref_rs, frames, 1)
    ref_rs.release()
    return frames, lin, aovs, ref


def score(frames, lin, aovs, ref, N=None, clamp=None, radius=1):
    td = R.TemporalDenoiser(max_history=N, clamp=clamp, clamp_radius=radius) if N else None
    mse, fl, prev = [], [], None
    for i, f in enumerate(frames):
        a = aovs[i]
        o = td.push(lin[i], a, f)["denoised"] if td else R.denoise(lin[i], a["albedo"], a["normal"])["linear"]
        mse.append(float(torch.mean((o.double() - ref[i].double()) ** 2)))
        if prev is not None:
            fl.append(float(torch.mean(((o - prev).double() - (ref[i] - ref[i - 1]).double()) ** 2)))
        prev = o
    return {"mse": round(sum(mse[4:]) / len(mse[4:]), 7), "flicker": round(sum(fl) / len(fl), 7), "flicker_4": round(sum(fl[3:]) / len(fl[3:]), 7)}


def quality_part(args):
    cols = [("denoise", {}), ("N2", dict(N=2)), ("N4", dict(N=4))]
    cols += [(f"N{N} g{g} r{r}", dict(N=N, clamp=g, radius=r)) for N in (2, 4) for r in (1, 2) for g in (0.5, 1.0, 1.5, 2.0, 3.0)]
    for diffuse in (False, True):
        for orbit in (True, False):
            inputs = row_inputs(diffuse, orbit, args.frames, args.ref_spp)
            row = {"part": "quality", "scene": "C2 all diffuse" if diffuse else "C2", "camera": "orbit 1 deg/frame" if orbit else "static",
                   "frames": args.frames, "spp": 4, "reference_spp": args.ref_spp}
            for name, kw in cols:
                row[name] = score(*inputs, **kw)
            torch.cuda.synchronize()
            print(json.dumps(row), flush=True)
            del inputs


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
    kernel_part(args)
    if not args.no_quality:
        quality_part(args)


if __name__ == "__main__":
    main()
