"""Runs the occlusion queries of tests/test_gpu_occlusion.py with whichever library RTB200_LIB names (rtb200 reads it at import,
so each stress build runs in a process of its own) and writes the answers to an .npz:

    python tests/occlusion_worker.py <out.npz>

"<variant>.<bounds>" for FILTERED and BRUTE_FORCE on the 10k-sphere scene's rays (intersect_worker.c4_rays), and
"<set>.<bounds>" for every query set of intersect_worker.SETS (the dense scenes, as uploaded or after rebuild()), each under
no t_max ("none") and under the per-ray bounds of `bounds` ("t"); and "meta" (JSON: rays and candidates of the host form)."""
import json
import os
import sys

TESTS = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(TESTS)
for _p in (REPO, os.path.join(REPO, "oracle"), os.path.join(REPO, "rust-raytracer_b200"), TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

import intersect_worker as IW  # noqa: E402
import rtb200 as R  # noqa: E402


def bounds(n, seed):
    """Per-ray t_max: uniform in (0, 2) (segments, some shorter than 0.001), with 1 for every fourth ray."""
    t = np.random.default_rng(seed).uniform(0.0, 2.0, size=n)
    t[::4] = 1.0
    return t


def _run(rs, o, d, name, out, meta):
    for tag, t in (("none", None), ("t", bounds(len(o), 44))):
        h = rs.occluded(o, d, t)
        out[f"{name}.{tag}"] = h["occluded"]
        meta[f"{name}.{tag}"] = {k: int(h["stats"][k]) for k in ("rays", "candidates")}


def main(path):
    sc = IW.c4_scene()
    o, d = IW.c4_rays(sc)
    out, meta = {}, {}
    for name, variant in (("filtered", R.RT_VARIANT_FILTERED), ("brute", R.RT_VARIANT_BRUTE_FORCE)):
        rs = R.ResidentScene(sc, R.make_options(variant=variant))
        try:
            _run(rs, o, d, name, out, meta)
        finally:
            rs.release()
    for name, (mk, rays, rebuild) in IW.SETS.items():
        sc = mk()
        so, sd = rays(sc)
        rs = R.ResidentScene(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
        try:
            if rebuild:
                rs.rebuild()
            _run(rs, so, sd, name, out, meta)
        finally:
            rs.release()
    np.savez(path, meta=np.array(json.dumps(meta)), **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
