"""Runs the closest-hit query of tests/test_gpu_intersect.py with whichever library RTB200_LIB names (rtb200 reads it at import,
so each stress build runs in a process of its own) and writes the hits to an .npz:

    python tests/intersect_worker.py <out.npz>

"<variant>.<field>" for FILTERED and BRUTE_FORCE on the 10k-sphere scene's rays (C4_RAYS), "<set>.<field>" for every query
set of SETS (the dense scenes, as uploaded or after rebuild()), and "meta" (JSON: the leaf size of the build, rays and
candidates of the host form)."""
import json
import os
import sys

TESTS = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(TESTS)
for _p in (REPO, os.path.join(REPO, "oracle"), os.path.join(REPO, "rust-raytracer_b200"), TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

import intersect_rays as IR  # noqa: E402
import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402
from test_gpu_rebuild_restatement import _coincident, _deep_dense  # noqa: E402


def c4_scene():
    return R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), 96, 54, 1, 50))


def c4_rays(sc):
    rng = np.random.default_rng(41)
    sets = [IR.camera_rays(sc, 96, 54), IR.box_rays(sc, rng, 4000), IR.surface_rays(sc, rng, 2000), IR.grazing_rays(sc, rng, 1000)]
    return np.concatenate([s[0] for s in sets]), np.concatenate([s[1] for s in sets])


def _rays(sc, seed, sets):
    rng = np.random.default_rng(seed)
    made = [IR.camera_rays(sc, 48, 36) if kind == "camera" else getattr(IR, kind + "_rays")(sc, rng, k) for kind, k in sets]
    return np.concatenate([m[0] for m in made]), np.concatenate([m[1] for m in made])


# query set -> (scene maker, rays of the scene, rebuild() first). The 10,000 coincident spheres give a ray hundreds of
# candidates, many times the smallest candidate list; the deep construction is the deepest tree the rebuild makes.
SETS = {
    "coincident": (lambda: _coincident(0), lambda sc: _rays(sc, 42, [("box", 3000), ("surface", 2000)]), False),
    "coincident_rebuilt": (lambda: _coincident(0), lambda sc: _rays(sc, 42, [("box", 3000), ("surface", 2000)]), True),
    "deep_rebuilt": (lambda: _deep_dense(32_768, 0), lambda sc: _rays(sc, 43, [("camera", 0), ("box", 3000), ("surface", 2000)]), True),
}


def main(path):
    sc = c4_scene()
    o, d = c4_rays(sc)
    out, meta = {}, {"leaf_size": int(R.bvh_records(sc)["leaf_size"])}
    for name, variant in (("filtered", R.RT_VARIANT_FILTERED), ("brute", R.RT_VARIANT_BRUTE_FORCE)):
        rs = R.ResidentScene(sc, R.make_options(variant=variant))
        try:
            h = rs.intersect(o, d)
        finally:
            rs.release()
        meta[name] = {k: int(h["stats"][k]) for k in ("rays", "candidates")}
        for k in IR.FIELDS:
            out[f"{name}.{k}"] = h[k]
    for name, (mk, rays, rebuild) in SETS.items():
        sc = mk()
        o, d = rays(sc)
        rs = R.ResidentScene(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
        try:
            if rebuild:
                rs.rebuild()
            h = rs.intersect(o, d)
        finally:
            rs.release()
        meta[name] = {k: int(h["stats"][k]) for k in ("rays", "candidates")}
        for k in IR.FIELDS:
            out[f"{name}.{k}"] = h[k]
    np.savez(path, meta=np.array(json.dumps(meta)), **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
