"""Moving spheres: refit a resident scene on the GPU (ResidentScene.update_geometry) against releasing and uploading it again.

Every sphere moves every frame: it drifts in x/z and bounces in y, with positions computed by torch on the GPU. Two loops
render the same animation, frame by frame, into device buffers:
  update    update_geometry(positions) and render, on one resident handle;
  reupload  copy the positions to the host, release the handle, upload the edited scene (host SAH build + arena copy), render.
Per scene it prints the update's device time (CUDA events around back-to-back updates on their stream) and its host
wall time, the wall time per frame and the Mrays/s of
both loops, whether the two loops computed identical frames and ray counts, and the tree decay: Mrays/s (device time) of a
render after k frames of motion on the refitted handle against a fresh upload at the same positions. The card's name, power
limit and SM clock are read in the same run.

    python tools/update_bench.py [--size 960x540x16] [--frames 10] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "rust-raytracer_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402

SLEEP_CYCLES = 60_000_000   # ~30 ms at 1980 MHz: longer than the host needs to enqueue one batch of updates


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return out


class Motion:
    """Positions at frame t of every sphere: x/z drift and a bounce in y (the ground sphere moves a hundredth as much)."""

    def __init__(self, sc, seed=1):
        arr = np.frombuffer(sc._spheres, dtype=np.float64).reshape(-1, 8)[: sc.n_spheres, :4]   # rt_sphere: cx cy cz r first
        self.g0 = torch.tensor(arr, dtype=torch.float64, device="cuda")
        g = torch.Generator(device="cuda").manual_seed(seed)
        n = sc.n_spheres
        big = (self.g0[:, 3].abs() > 100.0).to(torch.float64)
        scale = 1.0 - 0.99 * big
        self.vel = (torch.rand(n, 2, generator=g, device="cuda", dtype=torch.float64) - 0.5) * 0.04 * scale[:, None]
        self.amp = 0.5 * scale
        self.phase = torch.rand(n, generator=g, device="cuda", dtype=torch.float64) * 6.283185307179586

    def at(self, t):
        p = self.g0.clone()
        p[:, 0] += self.vel[:, 0] * t
        p[:, 2] += self.vel[:, 1] * t
        p[:, 1] += self.amp * torch.sin(0.3 * t + self.phase).abs()
        return p


def set_host(sc, pos):
    np.frombuffer(sc._spheres, dtype=np.float64).reshape(-1, 8)[: sc.n_spheres, :4] = pos.cpu().numpy()


def upload(sc):
    h = C.c_void_p()
    R._check(R.lib().rtb200_scene_upload(C.byref(sc.c), None, C.byref(h)))
    return h


def render_raw(h, out):
    st = R.rt_stats()
    R._check(R.lib().rtb200_render_device(h, C.c_void_p(out.data_ptr()), None, None, C.byref(st)))
    return st


def bench_scene(name, sc, frames, updates):
    w, hgt = sc.c.width, sc.c.height
    n_px = w * hgt * 3
    mo = Motion(sc)
    res = {"scene": name, "spheres": sc.n_spheres, "size": f"{w}x{hgt}x{sc.c.samples_per_pixel}"}
    set_host(sc, mo.at(0))
    rs = R.ResidentScene(sc)
    res["bvh_nodes"] = rs.kernel_info()["bvh_nodes"]
    # The update's device time: CUDA events around batches of updates on the stream they run on (torch's current stream,
    # update_geometry's default; inputs precomputed). A sleep kernel ahead of each batch keeps that stream busy while the host
    # enqueues the batch, so the events bracket back-to-back device work instead of the host's enqueue rate; the result says
    # whether every batch was enqueued before its sleep ended.
    inputs = [mo.at(t) for t in range(1, 5)]
    rs.update_geometry(inputs[0])                    # the first update builds the refit's scratch
    torch.cuda.synchronize()
    es, e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    per, dev_ms, busy = 50, 0.0, True
    for b in range((updates + per - 1) // per):
        es.record()
        torch.cuda._sleep(SLEEP_CYCLES)
        e0.record()
        t0 = time.perf_counter()
        for i in range(per):
            rs.update_geometry(inputs[i % 4])
        enqueue_ms = (time.perf_counter() - t0) * 1e3
        e1.record()
        torch.cuda.synchronize()
        busy = busy and enqueue_ms < es.elapsed_time(e0)
        dev_ms += e0.elapsed_time(e1)
    res["update_device_us"] = dev_ms * 1e3 / (per * ((updates + per - 1) // per))
    res["update_stream_kept_busy"] = busy
    t0 = time.perf_counter()
    for i in range(updates):
        rs.update_geometry(inputs[i % 4])
    torch.cuda.synchronize()
    res["update_wall_us"] = (time.perf_counter() - t0) * 1e6 / updates

    # the two loops, the same frames; one warm-up frame each
    outs = {a: torch.zeros((frames, n_px), dtype=torch.uint8, device="cuda") for a in ("update", "reupload")}
    rays = {"update": [], "reupload": []}
    wall = {"update": [], "reupload": []}
    rs.update_geometry(mo.at(0)); rs.render(outs["update"][0].data_ptr())
    for t in range(frames + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rs.update_geometry(mo.at(t))
        st = rs.render(outs["update"][max(t - 1, 0)].data_ptr())
        if t:
            wall["update"].append(time.perf_counter() - t0); rays["update"].append(st["rays"])
    rs.release()
    h = upload(sc)
    for t in range(frames + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pos = mo.at(t)
        set_host(sc, pos)
        R.lib().rtb200_scene_release(h)
        h = upload(sc)
        st = render_raw(h, outs["reupload"][max(t - 1, 0)])
        if t:
            wall["reupload"].append(time.perf_counter() - t0); rays["reupload"].append(st.rays)
    R.lib().rtb200_scene_release(h)
    torch.cuda.synchronize()
    res["identical"] = bool(torch.equal(outs["update"], outs["reupload"])) and rays["update"] == rays["reupload"]
    for a in ("update", "reupload"):
        ms = statistics.median(wall[a]) * 1e3
        res[a] = {"median_wall_ms_per_frame": ms, "mrays_wall": sum(rays[a]) / sum(wall[a]) / 1e6}

    # tree decay: the refitted tree after k frames of motion against a fresh build at the same positions
    set_host(sc, mo.at(0))
    rs = R.ResidentScene(sc)
    out_a = torch.zeros(n_px, dtype=torch.uint8, device="cuda"); out_b = torch.zeros_like(out_a)
    res["decay"] = []
    for k in (1, 10, 100):
        pos = mo.at(k)
        rs.update_geometry(pos)
        set_host(sc, pos)
        fresh = R.ResidentScene(sc)
        rs.render(out_a.data_ptr()); fresh.render(out_b.data_ptr())   # warm-up
        ra = [rs.render(out_a.data_ptr()) for _ in range(3)]
        rb = [fresh.render(out_b.data_ptr()) for _ in range(3)]
        torch.cuda.synchronize()
        same = bool(torch.equal(out_a, out_b)) and ra[0]["rays"] == rb[0]["rays"]
        fresh.release()
        res["decay"].append({"k": k, "identical": same,
                             "refit_mrays_device": max(s["rays"] / s["device_ms"] / 1e3 for s in ra),
                             "fresh_mrays_device": max(s["rays"] / s["device_ms"] / 1e3 for s in rb),
                             "refit_nodes_per_ray": ra[0]["nodes"] / ra[0]["rays"], "fresh_nodes_per_ray": rb[0]["nodes"] / rb[0]["rays"]})
    rs.release()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--size", default="960x540x16")
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--updates", type=int, default=200)
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    w, h, spp = (int(x) for x in args.size.split("x"))
    info = {"card": card(), "scenes": []}
    print(f"card (name, power limit, SM clock): {info['card']}", flush=True)
    todo = [("cover", lambda: scenes.cover_scene(w, h, spp)),
            ("C4 10k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), w, h, spp, 50))),
            ("100k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(158), w, h, spp, 50)))]
    for name, mk in todo:
        r = bench_scene(name, mk(), args.frames, args.updates)
        info["scenes"].append(r)
        u, f = r["update"], r["reupload"]
        print(f"{name}: {r['spheres']} spheres, {r['bvh_nodes']} nodes, {r['size']}: update {r['update_device_us']:.1f} us device "
              f"({r['update_wall_us']:.1f} us host wall per update, stream kept busy: {r['update_stream_kept_busy']}) | per frame: update+render {u['median_wall_ms_per_frame']:.2f} ms "
              f"({u['mrays_wall']:.0f} Mrays/s), reupload+render {f['median_wall_ms_per_frame']:.2f} ms ({f['mrays_wall']:.0f} Mrays/s) | "
              f"identical={r['identical']}", flush=True)
        for d in r["decay"]:
            print(f"    after {d['k']:3d} frames of motion: refit {d['refit_mrays_device']:.0f} Mrays/s ({d['refit_nodes_per_ray']:.1f} nodes/ray), "
                  f"fresh upload {d['fresh_mrays_device']:.0f} Mrays/s ({d['fresh_nodes_per_ray']:.1f} nodes/ray), identical={d['identical']}", flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(info, fh, indent=1)
    if not all(r["identical"] and all(d["identical"] for d in r["decay"]) for r in info["scenes"]):
        sys.exit("a refitted handle and a fresh upload rendered different frames")


if __name__ == "__main__":
    main()
