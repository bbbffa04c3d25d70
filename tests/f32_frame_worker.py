"""Runs the closest-hit queries of tests/test_gpu_f32_frame.py's stress-build test with whichever library RTB200_LIB names
(rtb200 reads it at import, so each stress build runs in a process of its own) and writes rays and hits to an .npz:

    python tests/f32_frame_worker.py <out.npz>

For every key of KEYS ("<scene>/<state>", state uploaded or rebuilt) the rays of f32_frame_cases.families on the handle's
hierarchy ("<key>.o", "<key>.d": the box-face rays depend on the build's leaf size) and the hits of the FILTERED variant
("<key>.<field>"); "meta" (JSON) holds the build's leaf size."""
import json
import os
import sys

TESTS = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(TESTS)
for _p in (REPO, os.path.join(REPO, "oracle"), os.path.join(REPO, "rust-raytracer_b200"), TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

import f32_frame_cases as F  # noqa: E402
import intersect_rays as IR  # noqa: E402
import rtb200 as R  # noqa: E402

KEYS = ["spread_1e12/uploaded", "spread_1e12/rebuilt", "threshold/uploaded", "threshold/rebuilt"]


def main(path):
    out, meta = {}, {}
    for key in KEYS:
        name, state = key.split("/")
        sc = F.SCENES[name]()
        rs = R.ResidentScene(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
        try:
            if state == "rebuilt":
                rs.rebuild()
            recs = rs.bvh_records()
            meta["leaf_size"] = int(recs["leaf_size"])
            o, d, _ = F.concat(F.families(sc, recs, 61))
            h = rs.intersect(o, d)
        finally:
            rs.release()
        out[f"{key}.o"], out[f"{key}.d"] = o, d
        for k in IR.FIELDS:
            out[f"{key}.{k}"] = h[k]
    np.savez(path, meta=np.array(json.dumps(meta)), **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
