"""Scene staging in shared memory (RTB200_WF_SMEM=<mask>, read at every upload): the trace kernel's prologue copies the
hierarchy or the flat records (bit 0), the f64 geometry (bit 1) and the materials (bit 2) into shared memory with TMA bulk
copies, and the closest-hit and shade stages read them there. Staging is a placement choice: for every mask, every kernel
(one frame, many frames, the adaptive list) renders the oracle's linear f32, RGB8, rays and samples, and the handle reports
the mask and exactly the shared memory the staged arrays add. A handle that stages its hierarchy refuses a rebuild and keeps
rendering; an update is staged at the next launch; a scene too large to stage is refused at upload."""
import numpy as np
import pytest

import adaptive_restatement as A
import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from test_gpu_adaptive import M, MIN, N, SCENES as ADAPTIVE_SCENES, _params, _samples
from test_gpu_scene_update import _jitter, _light_scene, _render
from test_gpu_shading_edges import assert_frames_match

pytestmark = pytest.mark.gpu
MASKS = list(range(1, 8))
FILTERED, BRUTE, EXACT = R.RT_VARIANT_FILTERED, R.RT_VARIANT_BRUTE_FORCE, R.RT_VARIANT_EXACT_F64
UNSUPPORTED = -4
SCENE_MAKERS = {"cover": lambda: scenes.cover_scene(48, 36, 4), "mixed_2_lights": lambda: _light_scene(2, 6, seed=47)}
_ORACLE = {}


def oracle(name):
    if name not in _ORACLE:
        _ORACLE[name] = O.render(SCENE_MAKERS[name]())
    return _ORACLE[name]


def _round16(b):
    return (b + 15) // 16 * 16


def staged_bytes(sc, variant, mask, t=None):
    """The arrays wf_layout adds for `mask`: 224 B per node, k * 16 B of records and k * 4 B of ids per leaf of k spheres
    (MODE_TREE) or 32 B per flat record pair (MODE_BRUTE) for bit 0, 32 B per sphere for bits 1 and 2. Each array is staged
    with one bulk copy, so it takes a multiple of 16 B: the leaf ids of an odd number of leaves of 2, 6, 10, ... spheres
    take 8 B more. t: the scene's hierarchy as the library that stages it builds it (default: R.bvh_records(sc))."""
    n = sc.n_spheres
    b = 0
    if mask & 1 and variant == FILTERED:
        t = R.bvh_records(sc) if t is None else t
        b += t["n_nodes"] * 224 + t["n_leaves"] * t["leaf_size"] * 16 + _round16(t["n_leaves"] * t["leaf_size"] * 4)
    if mask & 1 and variant == BRUTE:
        b += max(((n + 1) // 2 + 7) // 8 * 8, 8) * 32
    return b + (32 * n if mask & 2 else 0) + (32 * n if mask & 4 else 0)


def kernel_info(sc, variant, mask, monkeypatch):
    if mask:
        monkeypatch.setenv("RTB200_WF_SMEM", str(mask))
    else:
        monkeypatch.delenv("RTB200_WF_SMEM", raising=False)
    rs = R.ResidentScene(sc, R.make_options(variant=variant))
    try:
        return rs.kernel_info()
    finally:
        rs.release()


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("variant", [FILTERED, BRUTE], ids=["tree", "brute_force"])
@pytest.mark.parametrize("scene", list(SCENE_MAKERS))
def test_staged_one_frame_renders_match_the_oracle(scene, variant, mask, monkeypatch):
    sc = SCENE_MAKERS[scene]()
    base = kernel_info(sc, variant, 0, monkeypatch)
    ki = kernel_info(sc, variant, mask, monkeypatch)
    assert ki["smem_mask"] == mask and base["smem_mask"] == 0
    assert ki["smem_bytes"] - base["smem_bytes"] == staged_bytes(sc, variant, mask), (base["smem_bytes"], ki["smem_bytes"])
    opts = R.make_options(variant=variant)
    lin, st = R.render_linear(sc, opts)
    img, st8 = R.render_rgb8(sc, opts)
    lin_o, img_o, st_o = oracle(scene)
    assert_frames_match((lin, img), (lin_o, img_o), f"{scene} mask {mask}")
    assert st["rays"] == st8["rays"] == st_o["rays"] and st["samples"] == st_o["samples"]
    rs = R.ResidentScene(sc, opts)   # the staged resident handle against the one-shot render without staging's frame
    got = _render(rs)
    rs.release()
    assert np.array_equal(got[1], lin_o) and np.array_equal(got[0], img_o) and got[2] == st_o["rays"]


@pytest.mark.parametrize("mask", MASKS)
def test_staged_frames_and_adaptive_renders(mask, monkeypatch):
    """The multi-frame and the list kernels have layouts of their own."""
    sc = SCENE_MAKERS["mixed_2_lights"]()
    frames = [R.make_frame(sc, seed=3), R.make_frame(sc, look_from=[-6.0, 2.0, 9.0], seed=4)]
    want, st_want = R.render_frames(sc, frames)
    want_lin, _ = R.render_frames(sc, frames, linear=True)
    asc = ADAPTIVE_SCENES["mixed_2_lights"]()
    x, rays = _samples("mixed_2_lights", asc)
    p = _params()
    ad = A.run(x, rays, M, N, MIN, p.abs_tol, p.rel_tol)
    monkeypatch.setenv("RTB200_WF_SMEM", str(mask))
    img, st = R.render_frames(sc, frames)
    lin, _ = R.render_frames(sc, frames, linear=True)
    assert st["frames"] == 2 and st["batches"] == 1 and st["rays"] == st_want["rays"]
    for i in range(len(frames)):
        assert_frames_match((lin[i], img[i]), (want_lin[i], want[i]), f"mask {mask} frame {i}")
    sc.seed = 3   # frame 0 is the scene's own view at seed 3: the oracle checks it independently
    lin_o, img_o, _ = O.render(sc)
    assert_frames_match((lin[0], img[0]), (lin_o, img_o), f"mask {mask} frame 0 vs the oracle")
    img, lin, cnt, st = R.render_adaptive(asc, p)
    assert np.array_equal(cnt, ad["counts"]), f"mask {mask}: adaptive counts differ"
    assert_frames_match((lin, img), (ad["linear"], ad["rgb8"]), f"mask {mask} adaptive")
    assert st["rays"] == ad["rays"] and st["samples"] == ad["samples"]


@pytest.mark.parametrize("mask", [1, 7])
def test_exact_f64_ignores_bit_0(mask, monkeypatch):
    sc = SCENE_MAKERS["mixed_2_lights"]()
    base = kernel_info(sc, EXACT, 0, monkeypatch)
    ki = kernel_info(sc, EXACT, mask, monkeypatch)
    assert ki["smem_mask"] == mask and ki["smem_bytes"] - base["smem_bytes"] == staged_bytes(sc, EXACT, mask)
    lin, st = R.render_linear(sc, R.make_options(variant=EXACT))
    img, _ = R.render_rgb8(sc, R.make_options(variant=EXACT))
    lin_o, img_o, st_o = oracle("mixed_2_lights")
    assert_frames_match((lin, img), (lin_o, img_o), f"EXACT_F64 mask {mask}")
    assert st["rays"] == st_o["rays"]


def test_a_staged_hierarchy_refuses_a_rebuild_and_keeps_rendering(monkeypatch):
    monkeypatch.setenv("RTB200_WF_SMEM", "1")
    sc = SCENE_MAKERS["cover"]()
    rs = R.ResidentScene(sc)
    before = _render(rs)
    with pytest.raises(R.RtError) as e:
        rs.rebuild()
    assert e.value.code == UNSUPPORTED
    after = _render(rs)
    lin_o, img_o, st_o = oracle("cover")
    for got in (before, after):
        assert np.array_equal(got[1], lin_o) and np.array_equal(got[0], img_o) and got[2] == st_o["rays"]
    rs.release()


@pytest.mark.parametrize("mask", [1, 7])
def test_an_update_is_staged_at_the_next_launch(mask, monkeypatch):
    monkeypatch.setenv("RTB200_WF_SMEM", str(mask))
    sc = SCENE_MAKERS["mixed_2_lights"]()
    rs = R.ResidentScene(sc)
    _render(rs)
    idx, recs = _jitter(sc, np.random.default_rng(mask), 10)
    rs.update_spheres(idx, recs)
    got = _render(rs)
    rs.release()
    lin_o, img_o, st_o = O.render(sc)
    assert not np.array_equal(img_o, oracle("mixed_2_lights")[1])   # the edit shows in the frame
    assert np.array_equal(got[1], lin_o) and np.array_equal(got[0], img_o) and got[2] == st_o["rays"]


def test_a_scene_too_large_to_stage_is_refused_at_upload(monkeypatch):
    monkeypatch.setenv("RTB200_WF_SMEM", "7")
    sc = R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), 32, 18, 1, 4))
    assert sc.n_spheres > 9900
    with pytest.raises(R.RtError) as e:
        R.ResidentScene(sc)
    assert e.value.code == UNSUPPORTED and "no launch configuration fits shared memory" in str(e.value)
