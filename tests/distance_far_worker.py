"""Runs the far point queries of tests/test_gpu_distance_far.py with whichever library RTB200_LIB names (rtb200 reads it at
import, so each stress build runs in a process of its own) and writes the answers to an .npz:

    python tests/distance_far_worker.py <out.npz>

"<case>/<state>.sphere", ".distance" and ".overlaps" for the points of cases() (FILTERED), as uploaded and after rebuild()."""
import os
import sys

TESTS = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(TESTS)
for _p in (REPO, os.path.join(REPO, "oracle"), os.path.join(REPO, "rust-raytracer_b200"), TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

import distance_far_cases as D  # noqa: E402
import f32_frame_cases as F  # noqa: E402
import intersect_rays as IR  # noqa: E402
import rtb200 as R  # noqa: E402
from rebuild_restatement import filled, rebuild  # noqa: E402


def cases():
    """(key, scene, points, overlaps radii): the families of spread_1e12 and threshold on the rebuild restatement with leaves
    of 8 (the same points under every library), and the tie points."""
    out = []
    for name in (F.spread_name(1e12), "threshold"):
        sc = F.SCENES[name]()
        c, r = IR.spheres_of(sc)
        p = D.concat(D.families(sc, filled(rebuild(c, r, leaf_size=8), c, r), 31))[0]
        out.append((name, sc, p, np.abs(np.random.default_rng(32).normal(size=len(p)))))
    sc, ties = D.ties_scene()
    p = D.tie_points(ties)["p"]
    out.append(("ties", sc, p, np.full(len(p), 8.0)))
    return out


def main(path):
    out = {}
    for key, sc, p, rad in cases():
        rs = R.ResidentScene(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
        try:
            for state in ("uploaded", "rebuilt"):
                if state == "rebuilt":
                    rs.rebuild()
                h = rs.nearest(p)
                out[f"{key}/{state}.sphere"], out[f"{key}/{state}.distance"] = h["sphere"], h["distance"]
                out[f"{key}/{state}.overlaps"] = rs.overlaps(p, rad)["overlaps"]
        finally:
            rs.release()
    np.savez(path, **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
