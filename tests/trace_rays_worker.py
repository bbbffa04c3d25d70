"""Runs the trace_rays calls of tests/test_gpu_trace_rays.py with whichever library RTB200_LIB names (rtb200 reads it at import,
so each stress build runs in a process of its own) and writes the outputs to an .npz:

    python tests/trace_rays_worker.py <out.npz>

"<set>.linear", "<set>.rgb8" and "meta" (JSON: rays per set) for every set of SETS: the render's primary rays of the cover
scene (one call per sample), arbitrary rays of the lit, textured test scene with several samples, and the dense coincident
scene after rebuild()."""
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
from test_gpu_rebuild_restatement import _coincident  # noqa: E402
from test_trace_rays_cpu import primary_rays  # noqa: E402


def cover():
    return scenes.cover_scene(32, 24, 3)


def lit():
    return R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 32, 24, 1, 12), scenes.SCENES_DIR)


def mixed_rays(sc, seed, k=1500):
    rng = np.random.default_rng(seed)
    sets = [IR.camera_rays(sc, 32, 24), IR.box_rays(sc, rng, k), IR.surface_rays(sc, rng, k // 2), IR.degenerate_rays(sc, rng)]
    return np.concatenate([s[0] for s in sets]), np.concatenate([s[1] for s in sets])


# set -> (scene maker, [(origin, direction, trace_rays keywords)] of the scene, rebuild() first)
SETS = {
    "cover_render_rays": (cover, lambda sc: [(*primary_rays(sc, s), {"sample0": s}) for s in range(3)], False),
    "lit_mixed": (lit, lambda sc: [(*mixed_rays(sc, 61), {"samples": 5, "sample0": 2, "stream0": 7})], False),
    "coincident_rebuilt": (lambda: _coincident(0), lambda sc: [(*mixed_rays(sc, 62, 1000), {"samples": 2})], True),
}


def main(path):
    out, meta = {}, {}
    for name, (mk, calls, rebuild) in SETS.items():
        sc = mk()
        rs = R.ResidentScene(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
        try:
            if rebuild:
                rs.rebuild()
            for k, (o, d, kw) in enumerate(calls(sc)):
                h = rs.trace_rays(o, d, rgb8=True, **kw)
                out[f"{name}.{k}.linear"] = h["linear"]
                out[f"{name}.{k}.rgb8"] = h["rgb8"]
                meta[f"{name}.{k}"] = int(h["stats"]["rays"])
        finally:
            rs.release()
    np.savez(path, meta=np.array(json.dumps(meta)), **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
