"""Time and quality of the variance through the temporal accumulation (rtb200.temporal(variance=...), TemporalDenoiser(variance=True),
DESIGN.md §4.21) on one GPU.

    python tools/temporal_var_bench.py [--runs 3] [--iters 50] [--frames 16] [--ref-spp 1024] [--no-quality]

  * "kernel": rtb200_temporal_device, rtb200_temporal_var_device unclamped and rtb200_temporal_var_device clamped at r = 1
    (gamma 1) on tools/temporal_bench.py's buffers at 800x600 and 1920x1080 (a random frame reprojected through a one-degree
    orbit step) plus random variance planes; `--iters` calls per timed window, the three calls alternating within each size and
    the runs repeating them; CUDA events around each window. The traffic floor is 56 B per pixel for the call without variance
    and 80 B with it (12 B of the pixel's variance in, 12 B out); GB/s is that floor over the measured time;
  * "quality" (unless --no-quality): DESIGN.md §4.20's protocol. C2, and C2 with every metal and glass sphere Lambertian, each
    under the one-degree orbit and under a still camera, at 4 and 8 spp: `--frames` frames with seeds 1000, 1001, ... against a
    `--ref-spp` render of each frame. Rows: the denoise alone, denoise_var alone, §4.20's clamped accumulation (N = 2, the default
    clamp) followed by the denoise, and the accumulation with the variance, clamped at the default and unclamped, at N in
    {2, 4, 8}, followed by denoise_var (every filter at its defaults). "mse" is the mean over frames 4 .. F-1, "flicker" the mean
    over k >= 1 of |(o_k - o_k-1) - (r_k - r_k-1)|^2 (§4.16's measure).
Prints the device, its power limit and SM clocks read in the same run, then one JSON line per part."""
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
from temporal_bench import FLOOR_BYTES, kernel_arm, orbit_camera, stream_handle, timed  # noqa: E402
from temporal_clamp_bench import make_diffuse  # noqa: E402

VAR_FLOOR_BYTES = FLOOR_BYTES + 24


def var_arm(w, h, bufs, clamp):
    """rtb200_temporal_var_device on kernel_arm's buffers with random variances, checked against the Python call's outputs."""
    color, sphere, point, prev, _, _ = bufs
    sc = scenes.cover_scene(w, h, 1)
    cam, pcam = orbit_camera(sc, 1.0).camera, orbit_camera(sc, 0.0).camera
    g = torch.Generator(device="cuda").manual_seed(w + 1)
    var = torch.rand((h, w, 3), generator=g, device="cuda") * 0.01
    vprev = dict(prev, variance=torch.rand((h, w, 3), generator=g, device="cuda") * 0.01)
    kw = dict(clamp=1.0, clamp_radius=1) if clamp else {}
    want = R.temporal(color, sphere, point, cam, vprev, depth_tol=1e6, variance=var, **kw)
    out_c, out_n, out_v = torch.empty_like(want["color"]), torch.empty_like(want["length"]), torch.empty_like(want["variance"])
    p = R.rt_temporal_params(w, h, R.TEMPORAL_MAX_HISTORY, 0, cam, pcam, 1e6)
    cl = C.byref(R.rt_temporal_clamp(1.0, 1)) if clamp else None
    cur = R.rt_temporal_frame(color.data_ptr(), sphere.data_ptr(), point.data_ptr())
    hist = R.rt_temporal_history(prev["color"].data_ptr(), prev["length"].data_ptr(), prev["sphere"].data_ptr(), prev["point"].data_ptr())
    out = R.rt_temporal_out(out_c.data_ptr(), out_n.data_ptr())

    def arm():
        R._check(R.lib().rtb200_temporal_var_device(0, C.byref(p), cl, C.byref(cur), var.data_ptr(), C.byref(hist),
                                                    vprev["variance"].data_ptr(), None, C.byref(out), out_v.data_ptr(), stream_handle()))
    arm()
    torch.cuda.synchronize()
    for a, b in ((out_c, want["color"]), (out_v, want["variance"])):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert torch.equal(out_n, want["length"])
    return arm, (var, vprev, want, out_c, out_n, out_v)


def kernel_part(args):
    out = {"part": "kernel", "ms": {}}
    arms, keep, sizes = {}, [], ((800, 600), (1920, 1080))
    for w, h in sizes:
        arm, _, bufs = kernel_arm(w, h)
        keep.append(bufs)
        arms[(w, h, "temporal")] = arm
        for name, clamp in (("temporal_var", False), ("temporal_var_clamped_r1", True)):
            a, k = var_arm(w, h, bufs, clamp)
            keep.append(k)
            arms[(w, h, name)] = a
    for a in arms.values():
        timed(a, 5)
    for _ in range(args.runs):
        for (w, h, name), a in arms.items():
            out["ms"].setdefault(f"{w}x{h}/{name}", []).append(round(timed(a, args.iters), 5))
    out["floor_gbs"] = {}
    for (w, h, name) in arms:
        key = f"{w}x{h}/{name}"
        fb = FLOOR_BYTES if name == "temporal" else VAR_FLOOR_BYTES
        out["floor_gbs"][key] = [round(fb * w * h / (ms * 1e-3) / 1e9, 1) for ms in out["ms"][key]]
    print(json.dumps(out), flush=True)


def render(sc, frames, spp):
    """Linear frames and the variance of their pixel means [n, h, w, 3], and each frame's AOVs at spp, on the device."""
    sc.c.samples_per_pixel = spp
    rs = R.ResidentScene(sc)
    try:
        w, h = int(sc.c.width), int(sc.c.height)
        lin = torch.empty((len(frames), h, w, 3), dtype=torch.float32, device="cuda")
        var = torch.empty_like(lin)
        rs.render_frames(frames, 0, lin.data_ptr(), stream=stream_handle(), variance=var.data_ptr())
        aovs = [rs.aov(spp, view=f, on_device=True, outputs=("albedo", "normal", "sphere", "point")) for f in frames]
        torch.cuda.synchronize()
    finally:
        rs.release()
    return lin, var, aovs


def score(frames, lin, var, aovs, ref, mode, N=None, clamp=None):
    """mse and flicker of one row: mode "denoise" / "denoise_var" alone, "clamped" (TemporalDenoiser at N with the clamp, then the
    denoise) or "var" (TemporalDenoiser(variance=True) at N, clamp or not, then denoise_var)."""
    td = None
    if mode == "clamped":
        td = R.TemporalDenoiser(max_history=N, clamp=clamp)
    elif mode == "var":
        td = R.TemporalDenoiser(max_history=N, clamp=clamp, variance=True)
    mse, fl, prev = [], [], None
    for i, f in enumerate(frames):
        a = aovs[i]
        if mode == "denoise":
            o = R.denoise(lin[i], a["albedo"], a["normal"])["linear"]
        elif mode == "denoise_var":
            o = R.denoise_var(lin[i], var[i], a["albedo"], a["normal"])["linear"]
        elif mode == "clamped":
            o = td.push(lin[i], a, f)["denoised"]
        else:
            o = td.push(lin[i], a, f, variance=var[i])["denoised"]
        mse.append(float(torch.mean((o.double() - ref[i].double()) ** 2)))
        if prev is not None:
            fl.append(float(torch.mean(((o - prev).double() - (ref[i] - ref[i - 1]).double()) ** 2)))
        prev = o
    return {"mse": round(sum(mse[4:]) / len(mse[4:]), 7), "flicker": round(sum(fl) / len(fl), 7)}


def quality_part(args):
    g = R.TEMPORAL_CLAMP_GAMMA
    rows = [("denoise", dict(mode="denoise")), ("denoise_var", dict(mode="denoise_var")),
            ("clamped N2 + denoise", dict(mode="clamped", N=R.TEMPORAL_MAX_HISTORY, clamp=g))]
    rows += [(f"var{' clamped' if c is not None else ''} N{N} + denoise_var", dict(mode="var", N=N, clamp=c)) for c in (g, None) for N in (2, 4, 8)]
    for diffuse in (False, True):
        for orbit in (True, False):
            sc = scenes.scene("C2")
            if diffuse:
                make_diffuse(sc)
            frames = [orbit_camera(sc, float(i) if orbit else 0.0) for i in range(args.frames)]
            for i, f in enumerate(frames):
                f.seed = 1000 + i
            ref, _, _ = render(sc, frames, args.ref_spp)
            for spp in (4, 8):
                lin, var, aovs = render(sc, frames, spp)
                out = {"part": "quality", "scene": "C2 all diffuse" if diffuse else "C2", "camera": "orbit 1 deg/frame" if orbit else "still",
                       "frames": args.frames, "spp": spp, "reference_spp": args.ref_spp}
                for name, kw in rows:
                    out[name] = score(frames, lin, var, aovs, ref, **kw)
                torch.cuda.synchronize()
                print(json.dumps(out), flush=True)
                del lin, var, aovs
            del ref


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
