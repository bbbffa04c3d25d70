"""Runs the edits of tests/test_gpu_scene_edit.py with whichever library RTB200_LIB names (rtb200 reads it at import, so each
stress build runs in a process of its own) and writes what the edited handles give to an .npz:

    python tests/edit_worker.py <out.npz>

For every set of SETS: "<set>.linear", "<set>.rgb8" (a render after the edits), "<set>.<field>" (intersect's outputs on the
set's rays), "<set>.occluded", and "meta" (JSON: rays per render)."""
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


def _spheres(k, seed, light=False):
    rng = np.random.default_rng(seed)
    mats = [{"Lambertian": {"albedo": [0.7, 0.3, 0.2]}}, {"Metal": {"albedo": [0.8, 0.8, 0.9], "fuzz": 0.1}},
            {"Glass": {"index_of_refraction": 1.5}}]
    out = [R.make_sphere([rng.uniform(-4, 4), rng.uniform(0.2, 1.0), rng.uniform(-3, 3)], rng.uniform(0.2, 0.5), mats[i % 3]) for i in range(k)]
    if light:
        out.append(R.make_sphere([0.0, 5.0, 1.0], 1.0, {"Light": {}}))
    return out


def _edits(sc, seed):
    """Three edits of sc: removes, inserts in the middle with a light among them, and both in one call."""
    rng = np.random.default_rng(seed)
    n = sc.n_spheres
    rem1 = sorted(int(i) for i in rng.choice(np.arange(1, n), size=min(5, n - 1), replace=False))
    n1 = n - len(rem1)
    ins2 = _spheres(4, seed + 1, light=True)
    at2 = sorted(int(j) for j in rng.integers(0, n1 + 1, size=len(ins2)))
    n2 = n1 + len(ins2)
    rem3 = sorted(int(i) for i in rng.choice(np.arange(1, n2), size=min(3, n2 - 1), replace=False))
    ins3 = _spheres(3, seed + 2)
    return [(rem1, [], None), ([], ins2, at2), (rem3, ins3, [0, n2 // 2, n2])]


def cover():
    return scenes.cover_scene(32, 24, 2)


def lit():
    return R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 32, 24, 1, 8), scenes.SCENES_DIR)


def coincident():
    return _coincident(0)


SETS = {"cover": (cover, 71), "lit": (lit, 72), "coincident": (coincident, 73)}


def edited(name):
    """The host scene of set `name` after its edits, and the edits."""
    mk, seed = SETS[name]
    sc = mk()
    edits = _edits(sc, seed)
    for rem, ins, at in edits:
        sc = sc.edited(rem, ins, at)
    return mk(), edits, sc


def rays(sc, seed):
    rng = np.random.default_rng(seed)
    sets = [IR.camera_rays(sc, 32, 24), IR.box_rays(sc, rng, 1500), IR.surface_rays(sc, rng, 700), IR.degenerate_rays(sc, rng)]
    return np.concatenate([s[0] for s in sets]), np.concatenate([s[1] for s in sets])


def main(path):
    import torch
    out, meta = {}, {}
    for name in SETS:
        sc0, edits, sc = edited(name)
        rs = R.ResidentScene(sc0, R.make_options(variant=R.RT_VARIANT_FILTERED))
        try:
            for rem, ins, at in edits:
                rs.edit_spheres(rem, ins, at)
            n = rs.rows * sc.c.width * 3
            d8 = torch.zeros(n, dtype=torch.uint8, device="cuda")
            dl = torch.zeros(n, dtype=torch.float32, device="cuda")
            st = rs.render(d8.data_ptr(), dl.data_ptr())
            out[f"{name}.rgb8"] = d8.cpu().numpy().reshape(rs.rows, sc.c.width, 3)
            out[f"{name}.linear"] = dl.cpu().numpy().reshape(rs.rows, sc.c.width, 3)
            meta[name] = int(st["rays"])
            o, d = rays(sc, 80)
            for k, v in rs.intersect(o, d).items():
                if k != "stats":
                    out[f"{name}.{k}"] = v
            out[f"{name}.occluded"] = rs.occluded(o, d)["occluded"]
        finally:
            rs.release()
    np.savez(path, meta=np.array(json.dumps(meta)), **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
