"""Rebuilding the hierarchy of a resident scene on the GPU (ResidentScene.rebuild) against refitting it and against a fresh upload.

The scenes and the motion are those of tools/update_bench.py. After k = 1, 10 and 100 frames of motion it renders the same
frame on three handles at the same positions and reports their Mrays/s (device time, best of three after a warm-up) and
nodes visited per ray, and whether all three rendered identical frames and ray counts:
  refit     uploaded at frame 0 and moved with update_geometry (the upload's topology);
  rebuilt   the same, then rebuild() (a topology built on the GPU from the current spheres);
  fresh     the host scene at the same positions, uploaded (host SAH build).
At k = 100 it also rebuilds with RTB200_REBUILD_OVERSIZE=0, which leaves oversized spheres (the cover scene's ground) in the
Morton order instead of giving them their own subtree.
It also reports the rebuild's cost: device time (CUDA events around it on its stream; the call reads one header back in the
middle, so that host round trip is included), host wall time per call, and the host path it replaces (positions copied to
the host, handle released, scene uploaded again). The card's name, power limit and SM clock are read in the same run.

    python tools/rebuild_bench.py [--size 960x540x16] [--rebuilds 20] [--json out.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from update_bench import Motion, card, set_host  # noqa: E402  (also puts the package on sys.path)

import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402


def best(rs, out):
    rs.render(out.data_ptr())   # warm-up
    st = [rs.render(out.data_ptr()) for _ in range(3)]
    return st, max(s["rays"] / s["device_ms"] / 1e3 for s in st)


def bench_scene(name, sc, rebuilds):
    w, hgt = sc.c.width, sc.c.height
    n_px = w * hgt * 3
    mo = Motion(sc)
    res = {"scene": name, "spheres": sc.n_spheres, "size": f"{w}x{hgt}x{sc.c.samples_per_pixel}", "decay": []}
    set_host(sc, mo.at(0))
    refit, rebuilt = R.ResidentScene(sc), R.ResidentScene(sc)
    outs = [torch.zeros(n_px, dtype=torch.uint8, device="cuda") for _ in range(3)]
    for k in (1, 10, 100):
        pos = mo.at(k)
        refit.update_geometry(pos)
        rebuilt.update_geometry(pos)
        rebuilt.rebuild()
        set_host(sc, pos)
        fresh = R.ResidentScene(sc)
        row = {"k": k}
        stats = {}
        for key, rs, out in (("refit", refit, outs[0]), ("rebuilt", rebuilt, outs[1]), ("fresh", fresh, outs[2])):
            st, mr = best(rs, out)
            stats[key] = st[0]
            row[f"{key}_mrays_device"] = mr
            row[f"{key}_nodes_per_ray"] = st[0]["nodes"] / st[0]["rays"]
            row[f"{key}_bvh_nodes"] = rs.kernel_info()["bvh_nodes"]
        torch.cuda.synchronize()
        row["identical"] = bool(torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[2])) and \
            stats["refit"]["rays"] == stats["fresh"]["rays"] == stats["rebuilt"]["rays"]
        row["depth"] = rebuilt.kernel_info()["bvh_depth"]
        if k == 100:   # the same rebuild with oversized spheres (the cover scene's ground) left in the Morton order
            plain = R.ResidentScene(sc)
            os.environ["RTB200_REBUILD_OVERSIZE"] = "0"
            try:
                plain.rebuild()
            finally:
                del os.environ["RTB200_REBUILD_OVERSIZE"]
            st, mr = best(plain, outs[0])
            torch.cuda.synchronize()
            row["identical"] = row["identical"] and bool(torch.equal(outs[0], outs[2])) and st[0]["rays"] == stats["fresh"]["rays"]
            row["no_oversize_mrays_device"] = mr
            row["no_oversize_nodes_per_ray"] = st[0]["nodes"] / st[0]["rays"]
            plain.release()
        fresh.release()
        res["decay"].append(row)

    # cost of one rebuild at the k = 100 positions (the handle is warm: its rebuild memory exists)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev, wall = [], []
    for _ in range(rebuilds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        rebuilt.rebuild()
        e1.record()
        torch.cuda.synchronize()
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(e0.elapsed_time(e1))
    res["rebuild_device_ms"] = statistics.median(dev)
    res["rebuild_wall_ms"] = statistics.median(wall)
    # the host path a rebuild replaces: positions to the host, release, upload (host build + arena copy)
    pos = mo.at(100)
    up, h = [], None
    for _ in range(max(3, rebuilds // 4)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        set_host(sc, pos)
        if h is not None:
            h.release()
        h = R.ResidentScene(sc)
        torch.cuda.synchronize()
        up.append((time.perf_counter() - t0) * 1e3)
    h.release()
    res["reupload_wall_ms"] = statistics.median(up)
    refit.release(); rebuilt.release()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--size", default="960x540x16")
    ap.add_argument("--rebuilds", type=int, default=20)
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    w, h, spp = (int(x) for x in args.size.split("x"))
    info = {"card": card(), "scenes": []}
    print(f"card (name, power limit, SM clock): {info['card']}", flush=True)
    todo = [("cover", lambda: scenes.cover_scene(w, h, spp)),
            ("C4 10k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), w, h, spp, 50))),
            ("100k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(158), w, h, spp, 50)))]
    for name, mk in todo:
        r = bench_scene(name, mk(), args.rebuilds)
        info["scenes"].append(r)
        print(f"{name}: {r['spheres']} spheres, {r['size']}: rebuild {r['rebuild_device_ms']:.3f} ms device, {r['rebuild_wall_ms']:.3f} ms host "
              f"wall per call; host re-upload it replaces {r['reupload_wall_ms']:.2f} ms", flush=True)
        for d in r["decay"]:
            print(f"    after {d['k']:3d} frames: refit {d['refit_mrays_device']:.0f} Mrays/s ({d['refit_nodes_per_ray']:.1f} nodes/ray), "
                  f"rebuilt {d['rebuilt_mrays_device']:.0f} ({d['rebuilt_nodes_per_ray']:.1f}; {d['rebuilt_bvh_nodes']} nodes, depth {d['depth']}), "
                  f"fresh upload {d['fresh_mrays_device']:.0f} ({d['fresh_nodes_per_ray']:.1f}; {d['fresh_bvh_nodes']} nodes), "
                  f"identical={d['identical']}", flush=True)
            if "no_oversize_mrays_device" in d:
                print(f"        rebuilt with oversized spheres left in the Morton order: {d['no_oversize_mrays_device']:.0f} Mrays/s "
                      f"({d['no_oversize_nodes_per_ray']:.1f} nodes/ray)", flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(info, fh, indent=1)
    if not all(d["identical"] for r in info["scenes"] for d in r["decay"]):
        sys.exit("the refitted, rebuilt and freshly uploaded handles rendered different frames")


if __name__ == "__main__":
    main()
