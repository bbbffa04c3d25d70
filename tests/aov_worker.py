"""Runs the AOV passes of tests/test_gpu_aov.py with whichever library RTB200_LIB names (rtb200 reads it at import, so each stress
build runs in a process of its own) and writes the outputs to an .npz:

    python tests/aov_worker.py <out.npz>

"<set>.<output>" for every set of SETS and every output of rt_aov_out. A set whose scene has a lens renders through it
(rt_aov_lens_kernel)."""
import os
import sys

TESTS = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(TESTS)
for _p in (REPO, os.path.join(REPO, "oracle"), os.path.join(REPO, "rust-raytracer_b200"), TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402
from test_aov_cpu import mixed_lit_scene, textured_sky_scene  # noqa: E402
from test_gpu_rebuild_restatement import _coincident  # noqa: E402

def _lensed(mk, aperture, focus_dist=None):
    def make():
        sc = mk()
        sc.seed = 0x9E3779B97F4A7C15   # a 64-bit key whose high word is nonzero and differs from its low word
        sc.set_camera(aperture=aperture, focus_dist=focus_dist)
        return sc
    return make


# set -> (scene maker, samples, sample0, rebuild() first)
SETS = {
    "cover": (lambda: scenes.cover_scene(40, 30, 1), 4, 1, False),
    "textured_sky": (textured_sky_scene, 3, 0, False),
    "mixed_lit": (mixed_lit_scene, 2, 5, False),
    "coincident_rebuilt": (lambda: _coincident(0), 2, 0, True),
    "lens_mixed_lit": (_lensed(mixed_lit_scene, 0.4, 3.0), 3, 2, False),
    "lens_coincident_rebuilt": (_lensed(lambda: _coincident(0), 0.3), 2, 1, True),
}


def main(path):
    out = {}
    for name, (mk, samples, sample0, rebuild) in SETS.items():
        rs = R.ResidentScene(mk(), R.make_options(variant=R.RT_VARIANT_FILTERED))
        try:
            if rebuild:
                rs.rebuild()
            h = rs.aov(samples, sample0=sample0)
            for k, _, _ in R.AOV_FIELDS:
                out[f"{name}.{k}"] = h[k]
        finally:
            rs.release()
    np.savez(path, **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
