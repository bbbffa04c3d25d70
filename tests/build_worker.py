"""Renders the cases of tests/test_gpu_build_invariance.py with whichever library RTB200_LIB names (rtb200 reads it at import,
so each build runs in a process of its own) and writes what it rendered to an .npz:

    python tests/build_worker.py <out.npz>

For every case: "<case>.linear", "<case>.rgb8" (one frame, or [frames, ...]) and, for the adaptive cases, "<case>.counts";
"meta" holds a JSON dict with each case's rays, samples and candidates (and the depth of a rebuilt tree; the shared memory
staging adds and the hierarchy the build stages, for a staged one-frame case), the kernel_info() and leaf size of the build,
and every case that raised ("errors", with its traceback). The "topology" cases render nothing: they rebuild a scene and hold
the device's topology to the numpy restatement at the build's leaf size, and raise when it differs. The process exits 1
when a case raised. The scene makers are the suite's own; CASES is shared with the parent test, which renders the
references."""
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
import test_full_frames_cpu as FF  # noqa: E402
from test_full_frames_cpu import lit_scene as full_frame_lit_scene, params as full_frame_params  # noqa: E402
from test_gpu_adaptive import SCENES as ADAPTIVE_SCENES, _params  # noqa: E402
from test_gpu_parity import GOLDEN  # noqa: E402
from test_gpu_rebuild_restatement import _coincident, _deep_dense, _drifted, _geometry, _render_stats, _scene, rebuilt  # noqa: E402
from test_gpu_scene_rebuild import _adversarial  # noqa: E402
from test_gpu_scene_update import _jitter, _light_scene  # noqa: E402
from test_gpu_work_sets import _room_cfg, _room_frames, _textured_room  # noqa: E402
from test_rebuild_restatement_cpu import deep_spheres  # noqa: E402

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


SEED64 = 0x9E3779B97F4A7C15   # a 64-bit key whose high word is nonzero and differs from its low word


def lens_room_frames(sc):
    """Frames and lenses of the room: two lens views, a pinhole view and a focus pull, each with its own 64-bit seed."""
    fl = [R.make_frame_lens(sc, aperture=0.3, focus_dist=8.0, seed=SEED64),
          R.make_frame_lens(sc, look_from=[-9.0, 3.0, 7.0], aperture=0.0, seed=SEED64 + 0x100000001),
          R.make_frame_lens(sc, look_from=[4.0, 8.0, -12.0], look_at=[0.0, 1.0, 0.0], aperture=0.6, seed=SEED64 ^ (5 << 40)),
          R.make_frame_lens(sc, aperture=0.3, focus_dist=20.0, seed=SEED64 + 7)]
    return [f for f, _ in fl], [L for _, L in fl]


def _with_lens(mk, aperture, focus_dist=None):
    def make():
        sc = mk()
        sc.seed = SEED64
        sc.set_camera(aperture=aperture, focus_dist=focus_dist)
        return sc
    return make


def lens_adaptive_params():
    return _params()


# the parameters of an "adaptive" case other than test_gpu_adaptive's
ADAPTIVE_PARAMS = {"adaptive_full_frame_lit": lambda: full_frame_params(8)}


# case -> (kind, scene maker, variant, RTB200_WF_SMEM mask). Kinds: "one_shot" (render_linear and render_rgb8), "rebuilt" (a
# resident handle after rebuild()), "update" (a resident handle after update_spheres), "frames" (render_frames of
# _room_frames), "adaptive" (render_adaptive with test_gpu_adaptive's parameters, or the case's ADAPTIVE_PARAMS), "topology"
# (see the module docstring), "full_frames" (render_frames of test_full_frames_cpu.full_frames), "full_rays" (trace_rays of
# test_full_frames_cpu.full_rays), and for a lens scene "lens_one_shot" (one_shot through its lens), "lens_frames" (render_frames of lens_room_frames, with their
# lenses) and "lens_adaptive" (the adaptive rounds of a resident handle with the scene's lens, run to the end).
CASES = {
    **{f"golden_{name}": ("one_shot", mk, FILTERED, 0) for name, mk in GOLDEN},
    "room_3_lights_depth_50": ("one_shot", lambda: R.Scene.from_config(_room_cfg(3, 50)), FILTERED, 0),
    "room_1_light_depth_10": ("one_shot", lambda: R.Scene.from_config(_room_cfg(1, 10)), FILTERED, 0),
    "textured_room": ("one_shot", _textured_room, FILTERED, 0),
    "coincident_10k_1_light": ("one_shot", lambda: _coincident(1), FILTERED, 0),
    # after the rebuild every leaf of the coincident spheres is full (the host builder fills at most 20 of 32 slots): at
    # leaves of 32 one ray's leaf step yields 32 candidates, RT_CAP_CD of the smallest lists
    "coincident_10k_rebuilt": ("rebuilt", lambda: _coincident(1), FILTERED, 0),
    "deep_32768_rebuilt": ("rebuilt", lambda: _deep_dense(32_768, 0), FILTERED, 0),
    "rtiow_10k_filtered": ("one_shot", _rtiow_10k, FILTERED, 0),
    "rtiow_10k_brute_force": ("one_shot", _rtiow_10k, BRUTE, 0),
    "resident_update": ("update", _unmoved_scene, FILTERED, 0),
    "room_frames": ("frames", lambda: R.Scene.from_config(_room_cfg(3, 50)), FILTERED, 0),
    "adaptive_mixed_2_lights": ("adaptive", ADAPTIVE_SCENES["mixed_2_lights"], FILTERED, 0),
    # the full-frame adaptive case (tests/test_gpu_full_frames.py): 640 x 360 at 8 samples a round, whose rounds refill the
    # trace kernel's slots many times over and compact lists of hundreds of thousands of pixels
    "adaptive_full_frame_lit": ("adaptive", full_frame_lit_scene, FILTERED, 0),
    "room_exact_f64": ("one_shot", lambda: R.Scene.from_config(_room_cfg(3, 50)), EXACT, 0),
    # the lens kernels (DESIGN.md §4.17): Q_FRAMES_LENS at deep albedo stacks, over the dense candidate lists of the
    # coincident spheres, and Q_LIST_LENS, under 64-bit keys
    "lens_room_frames": ("lens_frames", lambda: R.Scene.from_config(_room_cfg(3, 50, w=48, h=36, spp=4)), FILTERED, 0),
    "lens_coincident_10k": ("lens_one_shot", _with_lens(lambda: _coincident(1), 0.4), FILTERED, 0),
    "lens_adaptive_mixed_2_lights": ("lens_adaptive", _with_lens(ADAPTIVE_SCENES["mixed_2_lights"], 0.3, 12.0), FILTERED, 0),
    # the full-frame Q_FRAMES and Q_RAYS cases (tests/test_gpu_full_frames.py), whose slots are reclaimed many times over
    "full_frames_lit": ("full_frames", lambda: FF.full_scene("lit", spp=FF.FRAME_SPP), FILTERED, 0),
    "full_rays_lit": ("full_rays", lambda: FF.full_scene("lit"), FILTERED, 0),
}

# Scene staging (RTB200_WF_SMEM) on every build: every mask in both modes that stage bit 0, on scenes whose hierarchy has an
# odd number of leaves at leaves of 2 (the room) and of 6 (the cover scene), where the leaf-id block is not a whole number
# of 16 B blocks (tests/test_stress_builds_cpu.py holds that parity); and the multi-frame and list kernels with everything
# staged. Each renders the frames of the unstaged case it names in BASE.
STAGE_SCENES = ("golden_cover_40x30_s4", "room_1_light_depth_10")
BASE = {"rtiow_10k_brute_force": "rtiow_10k_filtered", "room_exact_f64": "room_3_lights_depth_50",
        "coincident_10k_rebuilt": "coincident_10k_1_light"}
for _base in STAGE_SCENES:
    for _mode, _variant in (("tree", FILTERED), ("brute_force", BRUTE)):
        for _mask in range(1, 8):
            _name = f"staged_{_base}_{_mode}_m{_mask}"
            CASES[_name] = ("one_shot", CASES[_base][1], _variant, _mask)
            BASE[_name] = _base
for _base in ("room_frames", "adaptive_mixed_2_lights", "lens_room_frames"):
    CASES[f"staged_{_base}_m7"] = CASES[_base][:3] + (7,)
    BASE[f"staged_{_base}_m7"] = _base


def _drifted_c4():
    sc = R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), 32, 18, 1, 4))
    return sc, lambda rs: _geometry(rs, sc, _drifted(sc, 7))


# The GPU rebuild at the build's leaf size k against its restatement (tests/test_gpu_rebuild_restatement.py): case ->
# (k -> the scene, and what to do to the handle before the rebuild, or None)
TOPOLOGY = {
    "topology_n_k": lambda k: (_adversarial(f"n{k}"), None),
    "topology_n_k_plus_1": lambda k: (_adversarial(f"n{k + 1}"), None),
    "topology_coincident": lambda k: (_adversarial("coincident"), None),
    "topology_deep_32768": lambda k: (_scene(*deep_spheres(32_768)), None),
    "topology_c4_drifted": lambda k: _drifted_c4(),
}
CASES.update({name: ("topology", mk, FILTERED, 0) for name, mk in TOPOLOGY.items()})


def _stats(st):
    return {k: int(st[k]) for k in ("rays", "samples", "candidates")}


def _kernel_info(sc, variant, mask):
    rs = R.ResidentScene(sc, R.make_options(variant=variant))
    try:
        return rs.kernel_info()
    finally:
        rs.release()


def run_case(name, out, meta, leaf_size):
    kind, mk, variant, mask = CASES[name]
    if kind == "topology":
        sc, prepare = mk(leaf_size)
        rs = R.ResidentScene(sc)
        try:
            if prepare:
                prepare(rs)
            meta[name] = {"depth": int(rebuilt(rs, sc, leaf_size=leaf_size)["depth"])}
        finally:
            rs.release()
        return
    opts = R.make_options(variant=variant)
    sc = mk()
    if mask:
        base = _kernel_info(sc, variant, 0)
        os.environ["RTB200_WF_SMEM"] = str(mask)   # read at every upload
    try:
        if mask:
            ki = _kernel_info(sc, variant, mask)
            t = R.bvh_records(sc)
            staged = dict(smem_mask=int(ki["smem_mask"]), smem_staged=int(ki["smem_bytes"] - base["smem_bytes"]),
                          records={k: int(t[k]) for k in ("n_nodes", "n_leaves", "leaf_size")})
        render_case(name, kind, sc, opts, out, meta)
    finally:
        os.environ.pop("RTB200_WF_SMEM", None)
    if mask:
        meta[name].update(staged)


def render_case(name, kind, sc, opts, out, meta):
    if kind == "one_shot":
        lin, st = R.render_linear(sc, opts)
        img, st8 = R.render_rgb8(sc, opts)
        meta[name] = dict(_stats(st), rays_rgb8=int(st8["rays"]))
    elif kind in ("rebuilt", "update"):
        rs = R.ResidentScene(sc, opts)
        try:
            extra = {}
            if kind == "rebuilt":
                rs.rebuild()
                extra["depth"] = int(rs.topology()["depth"])
            else:
                _, idx, recs = moved_scene()
                rs.update_spheres(idx, recs)
            (img, lin, _), st = _render_stats(rs)
            meta[name] = dict(_stats(st), **extra)
        finally:
            rs.release()
    elif kind == "frames":
        frames = _room_frames(sc)
        img, st = R.render_frames(sc, frames, opts)
        lin, st2 = R.render_frames(sc, frames, opts, linear=True)
        meta[name] = dict(_stats(st), rays_linear=int(st2["rays"]), batches=int(st["batches"]))
    elif kind == "adaptive":
        img, lin, cnt, st = R.render_adaptive(sc, ADAPTIVE_PARAMS.get(name, _params)(), opts)
        out[name + ".counts"] = cnt
        meta[name] = _stats(st)
    elif kind == "full_frames":
        frames = FF.full_frames(sc)
        img, st = R.render_frames(sc, frames, opts)
        lin, st2 = R.render_frames(sc, frames, opts, linear=True)
        meta[name] = dict(_stats(st), rays_linear=int(st2["rays"]), batches=int(st["batches"]))
    elif kind == "full_rays":
        rs = R.ResidentScene(sc, opts)
        try:
            got = rs.trace_rays(*FF.full_rays(), FF.RAYS_SPP, rgb8=True, **FF.RAYS_KW)
        finally:
            rs.release()
        lin, img = got["linear"], got["rgb8"]
        meta[name] = _stats(got["stats"])
    elif kind == "lens_one_shot":
        lin, st = R.render_linear(sc, opts)
        img, st8 = R.render_rgb8(sc, opts)
        meta[name] = dict(_stats(st), rays_rgb8=int(st8["rays"]))
    elif kind == "lens_frames":
        frames, lenses = lens_room_frames(sc)
        img, st = R.render_frames(sc, frames, opts, lenses=lenses)
        lin, st2 = R.render_frames(sc, frames, opts, linear=True, lenses=lenses)
        meta[name] = dict(_stats(st), rays_linear=int(st2["rays"]), batches=int(st["batches"]))
    elif kind == "lens_adaptive":
        import torch
        rs = R.ResidentScene(sc, opts)
        try:
            rs.adaptive_begin(lens_adaptive_params())
            active, st = rs.adaptive_step(1000)
            n = rs.rows * int(sc.c.width)
            o8 = torch.zeros(3 * n, dtype=torch.uint8, device="cuda")
            ol = torch.zeros(3 * n, dtype=torch.float32, device="cuda")
            oc = torch.zeros(n, dtype=torch.int32, device="cuda")
            rs.adaptive_resolve(o8, ol, oc)
            sh = (rs.rows, int(sc.c.width))
            img, lin = o8.cpu().numpy().reshape(*sh, 3), ol.cpu().numpy().reshape(*sh, 3)
            out[name + ".counts"] = oc.cpu().numpy().view(np.uint32).reshape(sh)
            meta[name] = dict(_stats(st), active=active)
        finally:
            rs.release()
    else:
        raise ValueError(kind)
    out[name + ".linear"] = lin
    out[name + ".rgb8"] = img


def main(path):
    out, meta = {}, {"errors": {}}
    os.environ.pop("RTB200_WF_SMEM", None)
    info = R.ResidentScene(scenes.cover_scene(32, 24, 1), R.make_options(variant=FILTERED))
    meta["kernel_info"] = info.kernel_info()
    info.release()
    meta["leaf_size"] = int(R.bvh_records(scenes.cover_scene(32, 24, 1))["leaf_size"])
    for name in CASES:
        try:
            run_case(name, out, meta, meta["leaf_size"])
        except Exception:
            meta["errors"][name] = traceback.format_exc()
            print(f"[build_worker] {name} raised:\n{meta['errors'][name]}", file=sys.stderr, flush=True)
    np.savez(path, meta=np.array(json.dumps(meta)), **out)
    return 1 if meta["errors"] else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
