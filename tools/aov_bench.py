"""Throughput of the auxiliary-buffer pass (ResidentScene.aov, DESIGN.md §4.14) against the closest-hit query of the same primary
rays and the beauty render of the same view, alternated in one process on one GPU.

    python tools/aov_bench.py [--runs 3] [--iters 3] [--samples 16,128] [--scenes C2,C4]

Per scene (C2: the cover scene at 800x600; C4: 10,000 spheres at 1920x1080) and sample count: the AOV pass of every sample in
one device call; `intersect` of the same primary rays, one sample at a time (C4's 128-sample rays would take 12.7 GB at once),
with the rays of every sample made on the host and copied to the GPU before the timed region (24 B of direction per ray:
6.4 GB for C4 at 128 samples); and the beauty render of the view at that sample count. Every arm
is timed with CUDA events after a warm-up call; the arms alternate within a run and the runs repeat the set. Prints one JSON
line per (scene, samples) with the primary rays/s (millions) of each arm in each run."""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "rust-raytracer_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def jitter(seed, pixel, sample):
    """The first two f64 draws of the Philox4x32-10 stream of (pixel, sample) under `seed`: the render's pixel jitter
    (DESIGN.md "RNG contract"), vectorised over pixels."""
    mask = np.uint64(0xFFFFFFFF)
    c0 = np.zeros_like(pixel, np.uint64); c1 = np.full_like(c0, sample); c2 = pixel.astype(np.uint64); c3 = np.zeros_like(c0)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    for _ in range(10):
        p0, p1 = np.uint64(M0) * c0, np.uint64(M1) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & mask, (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & mask
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    first, second = (c1 << np.uint64(32)) | c0, (c3 << np.uint64(32)) | c2
    return [(u >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0) for u in (first, second)]


def primary_rays(sc, s):
    """The render's primary rays of sample s of every pixel, top row first (raytracer.rs:199-201, camera.rs:79-84)."""
    w, h = int(sc.c.width), int(sc.c.height)
    pix = np.arange(w * h, dtype=np.uint64)
    xi1, xi2 = jitter(sc.seed, pix, s)
    y, x = np.divmod(np.arange(w * h, dtype=np.float64), w)
    u = (x + xi1) / (w - 1.0)
    v = (h - (y + xi2)) / (h - 1.0)
    cam = sc.c.camera
    org = np.array(cam.origin.tup())
    d = ((np.array(cam.lower_left_corner.tup()) + np.array(cam.horizontal.tup()) * u[:, None]) + np.array(cam.vertical.tup()) * v[:, None]) - org
    return np.broadcast_to(org, d.shape).copy(), np.ascontiguousarray(d)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--samples", default="16,128")
    ap.add_argument("--scenes", default="C2,C4")
    args = ap.parse_args()
    sample_counts = [int(x) for x in args.samples.split(",")]
    print(json.dumps({"device": torch.cuda.get_device_name(0)}), flush=True)
    for name in args.scenes.split(","):
        sc = scenes.scene(name)
        w, h = int(sc.c.width), int(sc.c.height)
        npix = w * h
        rs = R.ResidentScene(sc)
        o0, d0 = primary_rays(sc, 0)
        # the bench's primary rays are the render's: sample 0's query equals the pass's sphere and point bit for bit
        chk = rs.aov(1, outputs=("sphere", "point"))
        q = rs.intersect(o0, d0, outputs=("sphere", "point"))
        assert np.array_equal(chk["sphere"].reshape(-1), q["sphere"]) and np.array_equal(chk["point"].reshape(-1, 3), q["point"]), name
        dev_o = torch.from_numpy(o0).cuda()
        dev_d = [torch.from_numpy(primary_rays(sc, s)[1]).cuda() for s in range(max(sample_counts))]   # 48 MB per sample on C4
        for n in sample_counts:
            out = {"scene": name, "width": w, "height": h, "samples": n, "aov_mrays": [], "intersect_mrays": [], "render_mrays": []}
            sc.c.samples_per_pixel = n
            beauty = R.ResidentScene(sc)
            d8 = torch.empty(npix * 3, dtype=torch.uint8, device="cuda")

            def aov_arm():
                for _ in range(args.iters):
                    rs.aov(n, on_device=True, outputs=("albedo", "normal", "hits", "sphere", "point"))

            def intersect_arm():
                for _ in range(args.iters):
                    for s in range(n):
                        rs.intersect(dev_o, dev_d[s], outputs=("sphere", "point", "normal"))

            stream = torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY   # the arms share torch's stream

            def render_arm():
                for _ in range(args.iters):
                    beauty.render(d8.data_ptr(), stream=stream)

            for arm in (aov_arm, intersect_arm, render_arm):   # warm-up
                arm()
            torch.cuda.synchronize()
            for _ in range(args.runs):
                for key, arm in (("aov_mrays", aov_arm), ("intersect_mrays", intersect_arm), ("render_mrays", render_arm)):
                    ms = timed(arm)
                    out[key].append(round(npix * n * args.iters / ms / 1e3, 1))
            beauty.release()
            print(json.dumps(out), flush=True)
        rs.release()


if __name__ == "__main__":
    main()
