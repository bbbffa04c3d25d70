#!/usr/bin/env python3
"""Writes tests/golden/lens.json: SHA-256 of the lens ORACLE's (tests/oracle_lens.cpp) linear-f32 and RGB8 frames, its ray
count and the SHA-256 of sample 0's lens primary rays, for two lens scenes: the cover scene at the book's lens (aperture 0.1,
focus 10) at 200x150x8, and the reference's test_scene (textures, a sky texture, a light, the hollow glass shell) at
aperture 0.4 focused at |look_from - look_at|. Regression pins of the lens contract (DESIGN.md §4.17), asserted on the CPU by
tests/test_lens_restatement_cpu.py and on the GPU by tests/test_gpu_lens.py.
Usage: python tests/golden/make_lens.py
"""
import copy
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(REPO, "rust-raytracer_b200")); sys.path.insert(0, os.path.dirname(HERE))
import numpy as np          # noqa: E402
import oracle_lens as OL    # noqa: E402
import rtb200 as R          # noqa: E402
from rtb200 import scenes   # noqa: E402

OUT = os.path.join(HERE, "lens.json")


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def cases() -> dict:
    """name -> lens Scene, each built by the library's camera from a config whose camera carries the lens."""
    out = {}
    for name, cfg, aperture, fd in (("cover_200x150_s8", scenes._variant(scenes.cover_config(), 200, 150, 8, 50), 0.1, 10.0),
                                     ("test_scene_80x60_s4", scenes._variant(scenes.test_scene_config(), 80, 60, 4, 8), 0.4, None)):
        cfg = copy.deepcopy(cfg)
        cfg["camera"]["aperture"] = aperture
        if fd is not None:
            cfg["camera"]["focus_dist"] = fd
        out[name] = R.Scene.from_config(cfg, scenes.SCENES_DIR)
    return out


def pins(sc) -> dict:
    r = OL.render(sc, sc.lens)
    o, d = OL.primary(sc, sc.lens, 0)
    return {"linear_sha256": sha(r["linear"]), "rgb8_sha256": sha(r["rgb8"]), "rays": r["rays"],
            "primary_s0_sha256": sha(np.concatenate([o, d], axis=1))}


if __name__ == "__main__":
    res = {name: pins(sc) for name, sc in cases().items()}
    with open(OUT, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(res, indent=1))
