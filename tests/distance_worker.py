"""Runs the point queries of tests/test_gpu_distance.py with whichever library RTB200_LIB names (rtb200 reads it at import, so
each stress build runs in a process of its own) and writes the answers to an .npz:

    python tests/distance_worker.py <out.npz>

"<set>.<variant>.sphere", ".distance" and ".overlaps" for the points of cases(): FILTERED and BRUTE_FORCE on the 10k-sphere
scene, and FILTERED on the dense scenes of intersect_worker.SETS (as uploaded or after rebuild()). point_sets() is also the
point families of the GPU tests and tools/distance_bench.py."""
import os
import sys

TESTS = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(TESTS)
for _p in (REPO, os.path.join(REPO, "oracle"), os.path.join(REPO, "rust-raytracer_b200"), TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

import distance_restatement as DR  # noqa: E402
import rtb200 as R  # noqa: E402


def point_sets(sc, rng, k):
    """k points each: uniform in the box of the finite centres, near surfaces (within 1e-3 of one), inside spheres, and far
    away (10 to 1e6 times the box's extent)."""
    c, r = DR.sphere_arrays(sc)
    fin = np.isfinite(c).all(axis=1) & np.isfinite(r) & (np.abs(r) < 1e6)
    cc, rr = c[fin], np.abs(r[fin])
    lo, hi = cc.min(axis=0), cc.max(axis=0)
    ext = float(np.max(hi - lo)) + 1.0
    u = rng.normal(size=(k, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    j = rng.integers(0, len(rr), size=k)
    return {"box": lo + rng.uniform(size=(k, 3)) * (hi - lo),
            "near": cc[j] + u * (rr[j] + rng.uniform(-1e-3, 1e-3, size=k))[:, None],
            "inside": cc[j] + u * (rr[j] * rng.uniform(0, 0.999, size=k))[:, None],
            "far": (lo + hi) / 2 + u * ext * 10.0 ** rng.uniform(1, 6, size=k)[:, None]}


def cases():
    """(name, scene maker, rebuild, variants, seed) of the runs."""
    import intersect_worker as IW
    out = [("c4_10k", IW.c4_scene, False, (("filtered", R.RT_VARIANT_FILTERED), ("brute", R.RT_VARIANT_BRUTE_FORCE)), 81)]
    for name, (mk, _, rebuild) in IW.SETS.items():
        out.append((name, mk, rebuild, (("filtered", R.RT_VARIANT_FILTERED),), 82))
    return out


def points_of(sc, seed):
    p = np.concatenate(list(point_sets(sc, np.random.default_rng(seed), 1000).values()))
    rad = np.abs(np.random.default_rng(seed + 1).normal(size=len(p))) * 0.2
    return p, rad


def main(path):
    out = {}
    for name, mk, rebuild, variants, seed in cases():
        sc = mk()
        p, rad = points_of(sc, seed)
        for vname, v in variants:
            rs = R.ResidentScene(sc, R.make_options(variant=v))
            try:
                if rebuild:
                    rs.rebuild()
                h = rs.nearest(p)
                out[f"{name}.{vname}.sphere"] = h["sphere"]
                out[f"{name}.{vname}.distance"] = h["distance"]
                out[f"{name}.{vname}.overlaps"] = rs.overlaps(p, rad)["overlaps"]
            finally:
                rs.release()
    np.savez(path, **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
