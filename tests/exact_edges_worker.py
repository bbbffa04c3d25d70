"""Runs the exact-edge queries of tests/test_gpu_exact_edges.py's stress-build test with whichever library RTB200_LIB names
(rtb200 reads it at import, so each stress build runs in a process of its own) and writes the answers to an .npz:

    python tests/exact_edges_worker.py <out.npz>

For every case of tests/exact_edges.py with its lights, as uploaded and after rebuild(), on the FILTERED variant:
"<case>/<state>.<field>" the hits of intersect, "<case>/<state>.occluded", "<case>/<state>.linear" / ".rgb8" of trace_rays
(TRACE keywords), and for the E3_leaves and E3_always cases "<case>/<state>.leaf_id" / ".always" from the handle's topology.
"meta" (JSON) holds the build's leaf size and the rays of every trace_rays call."""
import json
import os
import sys

TESTS = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(TESTS)
for _p in (REPO, os.path.join(REPO, "oracle"), os.path.join(REPO, "rust-raytracer_b200"), TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

import exact_edges as E  # noqa: E402
import intersect_rays as IR  # noqa: E402
import rtb200 as R  # noqa: E402
from test_exact_edges_cpu import scene  # noqa: E402

TRACE = {"samples": 3, "max_depth": 8}
STATES = ("uploaded", "rebuilt")


def main(path):
    out, meta = {}, {"rays": {}}
    for case in E.cases():
        sc = scene(case, E.LIGHTS)
        for state in STATES:
            key = f"{case.name}/{state}"
            rs = R.ResidentScene(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
            try:
                if state == "rebuilt":
                    rs.rebuild()
                h = rs.intersect(case.o, case.d)
                for k in IR.FIELDS:
                    out[f"{key}.{k}"] = h[k]
                out[f"{key}.occluded"] = rs.occluded(case.o, case.d)["occluded"]
                t = rs.trace_rays(case.o, case.d, rgb8=True, **TRACE)
                out[f"{key}.linear"], out[f"{key}.rgb8"] = t["linear"], t["rgb8"]
                meta["rays"][key] = int(t["stats"]["rays"])
                if case.name.startswith(("E3_leaves", "E3_always")):
                    top = rs.topology()
                    out[f"{key}.leaf_id"], out[f"{key}.always"] = top["leaf_id"], top["always"]
                    meta["leaf_size"] = int(top["leaf_size"])
            finally:
                rs.release()
    np.savez(path, meta=np.array(json.dumps(meta)), **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
