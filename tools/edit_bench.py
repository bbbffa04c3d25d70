"""Inserting and removing spheres of a resident scene (ResidentScene.edit_spheres) against releasing the handle and uploading
the edited list again.

On the cover scene (484 spheres), C4 (10k) and a 100k-sphere scene it times five edits: append 1, append 1000, remove 1, remove
1 % and remove 1 % plus insert 1 % (at random positions). Each is timed over many warm calls, each call followed by the edit that
restores the list (not timed), and reported as the median device time (CUDA events around the call on its stream; the call
waits for its topology, so the host round trip is included) and host wall time per call (to a synchronise after the call). The
path it replaces is timed on the same edited lists: release the handle and upload the list (host SAH build and arena copy).
After a remove 1 % plus insert 1 % edit it renders one frame on the edited handle and on a fresh upload of the same list and
reports both in Mrays/s (device time, best of three after a warm-up) and whether they were identical. The card's name, power
limit and SM clock are read in the same run.

    python tools/edit_bench.py [--size 960x540x16] [--calls 30] [--json out.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from update_bench import card  # noqa: E402  (also puts the package on sys.path)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402


def new_spheres(rng, k):
    mats = [{"Lambertian": {"albedo": [0.7, 0.3, 0.2]}}, {"Metal": {"albedo": [0.8, 0.8, 0.9], "fuzz": 0.1}},
            {"Glass": {"index_of_refraction": 1.5}}]
    return [R.make_sphere([rng.uniform(-10, 10), 0.2, rng.uniform(-10, 10)], 0.2, mats[i % 3]) for i in range(k)]


def inverse(sc, remove, insert, at):
    """The edit that takes sc.edited(remove, insert, at) back to sc: the inserts out, and each removed sphere back before the
    first kept sphere above it."""
    n = sc.n_spheres
    rem = sorted(remove)
    at = [n] * len(insert) if at is None else list(at)
    gone = set(rem)
    kept_below = np.cumsum([0] + [0 if i in gone else 1 for i in range(n)])
    at_sorted = np.array(at, dtype=np.int64)
    newpos = lambda j: int(kept_below[j]) + int(np.searchsorted(at_sorted, j, side="right"))   # noqa: E731
    n_new = n - len(rem) + len(insert)
    back_out = [int(kept_below[a]) + k for k, a in enumerate(at)]
    back_in, back_at = [], []
    nxt = n   # the first kept sphere above each removed one, scanning down
    above = {}
    for i in range(n - 1, -1, -1):
        if i in gone:
            above[i] = nxt
        else:
            nxt = i
    for i in rem:
        back_in.append(R.rt_sphere.from_buffer_copy(sc._spheres[i]))
        back_at.append(n_new if above[i] == n else newpos(above[i]))
    return back_out, back_in, back_at


def edits(sc, rng):
    n = sc.n_spheres
    pct = max(1, n // 100)
    ins = new_spheres(rng, pct)
    return {"append 1": ([], new_spheres(rng, 1), None),
            "append 1000": ([], new_spheres(rng, 1000), None),
            "remove 1": ([int(rng.integers(1, n))], [], None),
            "remove 1%": (sorted(int(i) for i in rng.choice(np.arange(1, n), size=pct, replace=False)), [], None),
            "remove 1% + insert 1%": (sorted(int(i) for i in rng.choice(np.arange(1, n), size=pct, replace=False)), ins,
                                      sorted(int(j) for j in rng.integers(0, n + 1, size=pct)))}


def time_edit(rs, sc, e, calls):
    back = inverse(sc, *e)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev, wall = [], []
    for c in range(calls + 2):   # two warm-up calls
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev0.record()
        rs.edit_spheres(*e)
        ev1.record()
        torch.cuda.synchronize()
        if c >= 2:
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(ev0.elapsed_time(ev1))
        rs.edit_spheres(*back)
    torch.cuda.synchronize()
    return statistics.median(dev), statistics.median(wall)


def time_reupload(sc, calls):
    wall, h = [], None
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if h is not None:
            h.release()
        h = R.ResidentScene(sc)
        torch.cuda.synchronize()
        wall.append((time.perf_counter() - t0) * 1e3)
    h.release()
    return statistics.median(wall)


def best(rs, out):
    rs.render(out.data_ptr())   # warm-up
    st = [rs.render(out.data_ptr()) for _ in range(3)]
    return st[0], max(s["rays"] / s["device_ms"] / 1e3 for s in st)


def bench_scene(name, sc, calls):
    rng = np.random.default_rng(1)
    res = {"scene": name, "spheres": sc.n_spheres, "size": f"{sc.c.width}x{sc.c.height}x{sc.c.samples_per_pixel}", "edits": []}
    rs = R.ResidentScene(sc)
    for what, e in edits(sc, rng).items():
        d, w = time_edit(rs, sc, e, calls)
        up = time_reupload(sc.edited(*e), max(5, calls // 3))
        res["edits"].append({"edit": what, "device_ms": d, "wall_ms": w, "reupload_wall_ms": up})
    # throughput of the edited handle (the rebuild's Morton tree) against a fresh upload (host SAH tree) of the same list
    e = edits(sc, rng)["remove 1% + insert 1%"]
    rs.edit_spheres(*e)
    fresh = R.ResidentScene(sc.edited(*e))
    n_px = sc.c.width * sc.c.height * 3
    a, b = torch.zeros(n_px, dtype=torch.uint8, device="cuda"), torch.zeros(n_px, dtype=torch.uint8, device="cuda")
    st_e, mr_e = best(rs, a)
    st_f, mr_f = best(fresh, b)
    torch.cuda.synchronize()
    res.update(edited_mrays_device=mr_e, fresh_mrays_device=mr_f, identical=bool(torch.equal(a, b)) and st_e["rays"] == st_f["rays"])
    rs.release(); fresh.release()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--size", default="960x540x16")
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    w, h, spp = (int(x) for x in args.size.split("x"))
    info = {"card": card(), "scenes": []}
    print(f"card (name, power limit, SM clock): {info['card']}", flush=True)
    todo = [("cover", lambda: scenes.cover_scene(w, h, spp)),
            ("C4 10k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), w, h, spp, 50))),
            ("100k", lambda: R.Scene.from_config(scenes._variant(scenes.rtiow_config(158), w, h, spp, 50)))]
    for name, mk in todo:
        r = bench_scene(name, mk(), args.calls)
        info["scenes"].append(r)
        print(f"{name}: {r['spheres']} spheres, {r['size']}", flush=True)
        for d in r["edits"]:
            print(f"    {d['edit']:22s} edit {d['device_ms']:8.3f} ms device, {d['wall_ms']:8.3f} ms host wall; "
                  f"release + upload {d['reupload_wall_ms']:8.2f} ms", flush=True)
        print(f"    after remove 1% + insert 1%: edited handle {r['edited_mrays_device']:.0f} Mrays/s, fresh upload "
              f"{r['fresh_mrays_device']:.0f} Mrays/s, identical={r['identical']}", flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(info, fh, indent=1)
    if not all(r["identical"] for r in info["scenes"]):
        sys.exit("the edited and freshly uploaded handles rendered different frames")


if __name__ == "__main__":
    main()
