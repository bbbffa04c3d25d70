"""Renders the cases of tests/test_gpu_build_invariance.py with whichever library RTB200_LIB names (rtb200 reads it at import,
so each build runs in a process of its own) and writes what it rendered to an .npz:

    python tests/build_worker.py <out.npz>

For every case: "<case>.linear", "<case>.rgb8" (one frame, or [frames, ...]) and, for the adaptive case, "<case>.counts";
"meta" holds a JSON dict with each case's rays, samples and candidates, the kernel_info() and leaf size of the build, the
depth of the rebuilt tree, and every case that raised ("errors", with its traceback). The process exits 1 when a case raised.
The scene makers are the suite's own; CASES is shared with the parent test, which renders the references."""
import json
import os
import sys
import traceback

TESTS = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(TESTS)
for _p in (REPO, os.path.join(REPO, "oracle"), os.path.join(REPO, "rust-raytracer_b200"), TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402
from test_gpu_adaptive import SCENES as ADAPTIVE_SCENES, _params  # noqa: E402
from test_gpu_parity import GOLDEN  # noqa: E402
from test_gpu_rebuild_restatement import _coincident, _deep_dense, _render_stats  # noqa: E402
from test_gpu_scene_update import _jitter, _light_scene  # noqa: E402
from test_gpu_work_sets import _room_cfg, _room_frames, _textured_room  # noqa: E402

FILTERED, BRUTE, EXACT = R.RT_VARIANT_FILTERED, R.RT_VARIANT_BRUTE_FORCE, R.RT_VARIANT_EXACT_F64


def _rtiow_10k():
    return R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), 128, 72, 3, 50))


def moved_scene():
    """The resident-update case: a lit mixed scene and the edit that moves ten of its spheres (one of them the light).
    Returns (scene, indices, records); the scene holds the edit."""
    sc = _light_scene(1, 6, seed=46)
    idx, recs = _jitter(sc, np.random.default_rng(9), 10)
    return sc, idx, recs


def _unmoved_scene():
    return _light_scene(1, 6, seed=46)


# case -> (kind, scene maker, variant). Kinds: "one_shot" (render_linear and render_rgb8), "rebuilt" (a resident handle after
# rebuild()), "update" (a resident handle after update_spheres), "frames" (render_frames of _room_frames), "adaptive"
# (render_adaptive with test_gpu_adaptive's parameters).
CASES = {
    **{f"golden_{name}": ("one_shot", mk, FILTERED) for name, mk in GOLDEN},
    "room_3_lights_depth_50": ("one_shot", lambda: R.Scene.from_config(_room_cfg(3, 50)), FILTERED),
    "room_1_light_depth_10": ("one_shot", lambda: R.Scene.from_config(_room_cfg(1, 10)), FILTERED),
    "textured_room": ("one_shot", _textured_room, FILTERED),
    "coincident_10k_1_light": ("one_shot", lambda: _coincident(1), FILTERED),
    "deep_32768_rebuilt": ("rebuilt", lambda: _deep_dense(32_768, 0), FILTERED),
    "rtiow_10k_filtered": ("one_shot", _rtiow_10k, FILTERED),
    "rtiow_10k_brute_force": ("one_shot", _rtiow_10k, BRUTE),
    "resident_update": ("update", _unmoved_scene, FILTERED),
    "room_frames": ("frames", lambda: R.Scene.from_config(_room_cfg(3, 50)), FILTERED),
    "adaptive_mixed_2_lights": ("adaptive", ADAPTIVE_SCENES["mixed_2_lights"], FILTERED),
    "room_exact_f64": ("one_shot", lambda: R.Scene.from_config(_room_cfg(3, 50)), EXACT),
}


def _stats(st):
    return {k: int(st[k]) for k in ("rays", "samples", "candidates")}


def run_case(name, out, meta):
    kind, mk, variant = CASES[name]
    opts = R.make_options(variant=variant)
    sc = mk()
    if kind == "one_shot":
        lin, st = R.render_linear(sc, opts)
        img, st8 = R.render_rgb8(sc, opts)
        meta[name] = dict(_stats(st), rays_rgb8=int(st8["rays"]))
    elif kind in ("rebuilt", "update"):
        rs = R.ResidentScene(sc, opts)
        try:
            if kind == "rebuilt":
                rs.rebuild()
                meta["rebuilt_depth"] = int(rs.topology()["depth"])
            else:
                _, idx, recs = moved_scene()
                rs.update_spheres(idx, recs)
            (img, lin, _), st = _render_stats(rs)
            meta[name] = _stats(st)
        finally:
            rs.release()
    elif kind == "frames":
        frames = _room_frames(sc)
        img, st = R.render_frames(sc, frames, opts)
        lin, st2 = R.render_frames(sc, frames, opts, linear=True)
        meta[name] = dict(_stats(st), rays_linear=int(st2["rays"]), batches=int(st["batches"]))
    elif kind == "adaptive":
        img, lin, cnt, st = R.render_adaptive(sc, _params(), opts)
        out[name + ".counts"] = cnt
        meta[name] = _stats(st)
    else:
        raise ValueError(kind)
    out[name + ".linear"] = lin
    out[name + ".rgb8"] = img


def main(path):
    out, meta = {}, {"errors": {}}
    info = R.ResidentScene(scenes.cover_scene(32, 24, 1), R.make_options(variant=FILTERED))
    meta["kernel_info"] = info.kernel_info()
    info.release()
    meta["leaf_size"] = int(R.bvh_records(scenes.cover_scene(32, 24, 1))["leaf_size"])
    for name in CASES:
        try:
            run_case(name, out, meta)
        except Exception:
            meta["errors"][name] = traceback.format_exc()
            print(f"[build_worker] {name} raised:\n{meta['errors'][name]}", file=sys.stderr, flush=True)
    np.savez(path, meta=np.array(json.dumps(meta)), **out)
    return 1 if meta["errors"] else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
