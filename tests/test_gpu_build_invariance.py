"""The trace kernel's frames do not depend on its compile-time capacities (DESIGN.md §4.1): every stress build of the library
(rust-raytracer_b200/stress, made by `make stress`) renders the same linear f32, RGB8, rays and samples as the CPU oracle, on
the scenes that reach the hard paths of the closest-hit and shade stages - dense candidate lists, deep node stacks, deep albedo
stacks, deferred scatters - through every kernel (one frame, many frames, the adaptive list, the rebuild, the refit).

The library is chosen when rtb200 is imported (RTB200_LIB), so each build renders in a process of its own
(tests/build_worker.py); this process renders the references once per module. Each build also proves that it is the build
its DEFS describe: its block size, its shared-memory layout (wf_layout restated below, and the staged arrays of
test_gpu_scene_staging.staged_bytes), its leaf size, the depth the restatement gives its rebuilt deep tree, and, for the
builds with the smallest lists, that their edges were reached. Every build also stages the scene in shared memory (every
RTB200_WF_SMEM mask) and rebuilds topologies the numpy restatement checks at its leaf size (build_worker's "topology"
cases)."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import adaptive_restatement as A
import build_worker as BW
import oracle_lens as OL
import oracle_py as O
import test_full_frames_cpu as FF
from test_gpu_adaptive import M, MIN, N, _samples
from test_gpu_scene_staging import staged_bytes
from test_gpu_shading_edges import assert_frames_match
from test_gpu_work_sets import _deep, _room_frames, _view
from test_rebuild_restatement_cpu import DEEP_AT

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRESS = os.path.join(REPO, "rust-raytracer_b200", "stress")
GOLD = os.path.join(REPO, "tests", "golden")
BUILDS = ["lists_min", "leaf2", "block128_leaf16", "leaf6", "leaf32_lists_min"]
TIMEOUT = 900   # seconds per build; every case of a build takes well under a minute on an H100

# the constants as the sources define them when DEFS leave them alone
DEFAULTS = {"RT_CAP_IN": 192, "RT_CAP_LF": 160, "RT_CAP_CD": 96, "RT_SMEM_STACK": 10, "RT_SCATTER_TRIPS": 2, "RT_LEAF_K": 8,
            "RT_BLOCK": 256, "RT_PHASE_CLOCKS": 0}
PHASE_N = 14   # kPhaseN: the stage-clock counters per warp of an RT_PHASE_CLOCKS build


def constants(defs):
    c = dict(DEFAULTS)
    c.update({k: int(v) for k, v in re.findall(r"-D(\w+)=(\d+)", defs)})
    return c


def tree_smem_bytes(c):
    """wf_layout(..., MODE_TREE, mask 0, single frame).total: mbarrier, per-warp contexts, the pool, perm, counters, and the
    stage-clock table of an RT_PHASE_CLOCKS build."""
    warps = c["RT_BLOCK"] // 32
    warp_ctx = (1664 + 4 * (c["RT_CAP_IN"] + c["RT_CAP_LF"] + c["RT_CAP_CD"]) + 15) // 16 * 16   # kWarpCtxBytes
    slot = 96 + 4 * c["RT_SMEM_STACK"]                                        # kSlotBytes
    phase = warps * PHASE_N * 8 if c["RT_PHASE_CLOCKS"] else 0
    return 16 + warps * warp_ctx + slot * c["RT_BLOCK"] + 5 * c["RT_BLOCK"] * 2 + 2 * 8 * 4 + phase


def test_the_default_layout_is_the_one_design_md_gives():
    assert tree_smem_bytes(DEFAULTS) == 65_104


# ---- references, rendered once per module ----
_REF = {}


def reference(name):
    """{linear, rgb8, rays, samples[, counts]} that case `name` must render; frames carry a leading frame axis."""
    name = BW.BASE.get(name, name)
    if name in _REF:
        return _REF[name]
    kind, mk = BW.CASES[name][:2]
    if name.startswith("golden_"):
        g = np.load(os.path.join(GOLD, name[len("golden_"):] + ".npz"))
        sc = mk()
        ref = dict(linear=g["linear"], rgb8=g["rgb8"], rays=int(g["rays"]), samples=sc.c.width * sc.c.height * sc.c.samples_per_pixel)
    elif kind in ("one_shot", "rebuilt", "update"):
        sc = BW.moved_scene()[0] if kind == "update" else mk()
        lin, img, st = O.render(sc)
        ref = dict(linear=lin, rgb8=img, rays=st["rays"], samples=st["samples"], oracle_stats=st)
    elif kind == "frames":
        sc = mk()
        outs = [O.render(_view(sc, f)) for f in _room_frames(sc)]
        ref = dict(linear=np.stack([o[0] for o in outs]), rgb8=np.stack([o[1] for o in outs]),
                   rays=sum(o[2]["rays"] for o in outs), samples=sum(o[2]["samples"] for o in outs))
    elif kind == "adaptive" and name in BW.ADAPTIVE_PARAMS:   # a full-frame case: the oracle's bulk route
        sc = mk()
        x, rays = FF.oracle_samples(name, sc)
        p = BW.ADAPTIVE_PARAMS[name]()
        want = A.run(x, rays, p.samples_per_round, sc.c.samples_per_pixel, p.min_samples, p.abs_tol, p.rel_tol)
        ref = dict(linear=want["linear"], rgb8=want["rgb8"], counts=want["counts"], rays=want["rays"], samples=want["samples"])
    elif kind == "adaptive":
        sc = mk()
        x, rays = _samples("mixed_2_lights", sc)
        p = BW._params()
        want = A.run(x, rays, M, N, MIN, p.abs_tol, p.rel_tol)
        ref = dict(linear=want["linear"], rgb8=want["rgb8"], counts=want["counts"], rays=want["rays"], samples=want["samples"])
    elif kind == "lens_one_shot":
        sc = mk()
        want = OL.render(sc, sc.lens)
        ref = dict(linear=want["linear"], rgb8=want["rgb8"], rays=want["rays"], samples=sc.c.width * sc.c.height * sc.c.samples_per_pixel)
    elif kind == "lens_frames":
        sc = mk()
        frames, lenses = BW.lens_room_frames(sc)
        outs = [OL.render(_view(sc, f), L) for f, L in zip(frames, lenses)]
        ref = dict(linear=np.stack([o["linear"] for o in outs]), rgb8=np.stack([o["rgb8"] for o in outs]),
                   rays=sum(o["rays"] for o in outs), samples=len(frames) * sc.c.width * sc.c.height * sc.c.samples_per_pixel)
    elif kind == "lens_adaptive":
        sc = mk()
        want = OL.adaptive(sc, sc.lens, BW.lens_adaptive_params())
        ref = dict(linear=want["linear"], rgb8=want["rgb8"], counts=want["counts"], rays=want["rays"], samples=want["samples"])
    else:
        raise ValueError(kind)
    _REF[name] = ref
    return ref


def test_the_room_reaches_deep_albedo_levels():
    """The room's paths run past every shared-memory level of every build (RT_SMEM_STACK <= 10)."""
    st = reference("room_3_lights_depth_50")["oracle_stats"]
    assert _deep(st, 13) >= 10_000, st["path_len_hist"]


def compare(name, z, meta):
    ref = reference(name)
    lin, img = z[name + ".linear"], z[name + ".rgb8"]
    if BW.CASES[name][0] in ("frames", "lens_frames"):
        assert lin.shape == ref["linear"].shape, (name, lin.shape)
        for i in range(len(lin)):
            assert_frames_match((lin[i], img[i]), (ref["linear"][i], ref["rgb8"][i]), f"{name} frame {i}")
    else:
        assert_frames_match((lin, img), (ref["linear"], ref["rgb8"]), name)
    if "counts" in ref:
        cnt = z[name + ".counts"]
        assert np.array_equal(cnt, ref["counts"]), f"{name}: counts differ in {int((cnt != ref['counts']).sum())} pixels"
    m = meta[name]
    assert (m["rays"], m["samples"]) == (ref["rays"], ref["samples"]), (name, m, ref["rays"], ref["samples"])
    for k in ("rays_rgb8", "rays_linear"):
        assert m.get(k, m["rays"]) == m["rays"], (name, m)


def run_build(name, lib, tmp_path):
    out = str(tmp_path / f"{name}.npz")
    env = dict(os.environ, RTB200_LIB=lib, RTB200_PRINT_PHASES="1")
    r = subprocess.run([sys.executable, BW.__file__, out], capture_output=True, text=True, env=env, cwd=REPO, timeout=TIMEOUT)
    meta = None
    if os.path.exists(out):
        z = np.load(out)
        meta = json.loads(str(z["meta"]))
    if r.returncode != 0 or meta is None:
        errors = "\n".join(f"--- {k}:\n{v}" for k, v in (meta or {}).get("errors", {}).items())
        pytest.fail(f"{name}: the worker exited with {r.returncode}\n{errors or r.stderr[-4000:]}")
    return z, meta, r.stderr


@pytest.mark.parametrize("build", BUILDS)
def test_stress_build_renders_the_oracle_frames(build, tmp_path):
    with open(os.path.join(STRESS, "manifest.json")) as f:
        manifest = json.load(f)
    assert build in manifest, f"{build} is missing from the manifest: run make -C rust-raytracer_b200 stress"
    lib = os.path.join(STRESS, f"librtb200_{build}.so")
    assert os.path.exists(lib), lib
    c = constants(manifest[build])
    z, meta, stderr = run_build(build, lib, tmp_path)

    # the build is the one its DEFS describe
    ki = meta["kernel_info"]
    assert ki["block"] == c["RT_BLOCK"] and ki["pool_slots"] == c["RT_BLOCK"], ki
    assert ki["smem_mask"] == 0 and ki["smem_bytes"] == tree_smem_bytes(c), (ki, tree_smem_bytes(c))
    assert meta["leaf_size"] == c["RT_LEAF_K"], meta["leaf_size"]

    failures = []
    for name in BW.CASES:
        if BW.CASES[name][0] == "topology":   # checked in the worker: a difference raises there
            continue
        try:
            compare(name, z, meta)
        except AssertionError as e:
            failures.append(f"{name}: {e}")
    rendered = [name for name in BW.CASES if BW.CASES[name][0] != "topology"]
    per_ray = {name: round(meta[name]["candidates"] / max(meta[name]["rays"], 1), 1) for name in rendered}
    scatters = sum(int(x) for x in re.findall(r"scatters=(\d+)", stderr))
    deferred = sum(int(x) for x in re.findall(r"deferred=(\d+)", stderr))
    depths = {name: meta[name]["depth"] for name in BW.CASES if "depth" in meta[name]}
    print(f"{build}: {c}\n  candidates per ray {per_ray}\n  rebuilt depths {depths}; "
          f"scatters {scatters}, deferred {deferred} ({deferred / max(scatters, 1):.4f})")
    assert not failures, "\n".join(failures)

    k = c["RT_LEAF_K"]
    for name in BW.CASES:   # staging added exactly the arrays of the hierarchy this build makes, in whole 16 B blocks
        kind, mk, variant, mask = BW.CASES[name]
        if mask and kind == "one_shot":
            m = meta[name]
            assert m["records"]["leaf_size"] == k and m["smem_mask"] == mask, (name, m)
            assert m["smem_staged"] == staged_bytes(mk(), variant, mask, m["records"]), (name, m)
    if k * 4 % 16:   # the staged leaf-id block was 8 B short of a 16 B multiple in a staged scene
        assert any(meta[f"staged_{s}_tree_m1"]["records"]["n_leaves"] % 2 for s in BW.STAGE_SCENES)
    # the rebuilt deep tree is as deep as the restatement's at this leaf size
    assert depths["deep_32768_rebuilt"] == depths["topology_deep_32768"] == DEEP_AT[k][32_768], depths

    if c["RT_CAP_CD"] == 32:   # the smallest lists: a ray's candidates overflow the candidate list many times over
        for name in ("coincident_10k_1_light", "coincident_10k_rebuilt"):
            assert per_ray[name] >= 300 > c["RT_CAP_CD"], per_ray
    if build == "lists_min":   # the edges this build is made for were reached
        assert depths["deep_32768_rebuilt"] >= 14, depths   # fat_in = 187 - 7 * 14 - 8 = 81 node-stack entries
        # One trip is two rejection trials, both missing the unit sphere with probability (1 - pi/6)^2 = 0.2270. Over these
        # cases an H100 (at its default power limit) measured 3,211,706 deferred of 14,154,171 scatters: 0.2269.
        assert scatters > 0 and 0.20 <= deferred / scatters <= 0.25, (scatters, deferred, stderr[-2000:])
