"""Inserting and removing spheres of a resident scene on the GPU (ResidentScene.edit_spheres, rtb200_scene_edit_spheres,
DESIGN.md §4.13): after edits every call on the handle is bit-identical to the same call on a fresh upload of Scene.edited(...)
and, at small sizes, to the CPU oracle: renders in every variant on the cover, lit and textured, always-list and 10k scenes;
sequences of edits down to no spheres and from 1 sphere to 100k and back; the light list; the hierarchy, which is the GPU
rebuild's of the new list; queries, trace_rays, frames and adaptive renders; updates and rebuilds after an edit; ordering
against frames and queries on other streams; shard handles; refusals, which leave renders unchanged; the stress builds."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import edit_worker as EW
import intersect_rays as IR
import oracle_py as O
import oracle_trace_rays as OT
import rtb200 as R
from rebuild_restatement import rebuild as restate
from rtb200 import scenes
from synth import base_config, mixed_config
from test_gpu_intersect import AUTO, BRUTE, EXACT, FILTERED, REPO, STRESS, _always_scene, _rtiow
from test_gpu_rebuild_restatement import assert_same_topology
from test_gpu_scene_update import HOLD, _positions, _render

pytestmark = pytest.mark.gpu
INVALID, UNSUPPORTED = -1, -4
VARIANTS = {"filtered": FILTERED, "brute_force": BRUTE, "exact_f64": EXACT, "auto": AUTO}
MATS = [{"Lambertian": {"albedo": [0.7, 0.3, 0.2]}}, {"Metal": {"albedo": [0.8, 0.8, 0.9], "fuzz": 0.2}},
        {"Glass": {"index_of_refraction": 1.5}}, {"Metal": {"albedo": [0.9, 0.6, 0.3], "fuzz": 0.0}}]


def _same(got, want, what):
    """Linear f32 bit for bit (NaNs of any payload match), RGB8 and the ray count."""
    a, b = got[1], want[1]
    bits = (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    assert bits.all(), f"{what}: linear differs at {int((~bits).sum())} values"
    assert np.array_equal(got[0], want[0]), f"{what}: rgb8 differs"
    assert got[2] == want[2], f"{what}: rays {got[2]} != {want[2]}"


def _fresh(sc, opts):
    rs = R.ResidentScene(sc, opts)
    try:
        return _render(rs)
    finally:
        rs.release()


def check(rs, sc, what, oracle=True):
    """rs renders what a fresh upload of sc renders, and the oracle when `oracle`."""
    got = _render(rs)
    _same(got, _fresh(sc, rs.opts), what + " vs a fresh upload")
    if oracle:
        lin_o, img_o, st_o = O.render(sc)
        _same(got, (img_o, lin_o, st_o["rays"]), what + " vs the oracle")
    return got


def edit(rs, sc, remove=(), insert=(), at=None, **kw):
    """Edit the handle and return the host scene of the edited list."""
    rs.edit_spheres(remove, insert, at, **kw)
    assert rs.n == sc.n_spheres - len(remove) + len(insert)
    return sc.edited(remove, insert, at)


def spheres(rng, k, textured=False, box=4.0):
    out = []
    for i in range(k):
        m = MATS[i % len(MATS)]
        if textured and i % 3 == 2:
            m = {"Texture": {"albedo": [1.0, 1.0, 1.0], "h_offset": 0.25, "texture": 0}}
        out.append(R.make_sphere([rng.uniform(-box, box), rng.uniform(0.2, 1.2), rng.uniform(-box, box)], rng.uniform(0.2, 0.6), m))
    return out


def light(x=0.0, y=6.0, z=0.0, r=1.0):
    return R.make_sphere([x, y, z], r, {"Light": {}})


def _lit_textured():
    return R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 40, 30, 2, 6), scenes.SCENES_DIR)


SCENES = {"cover": lambda: scenes.cover_scene(40, 30, 2), "lit_textured": _lit_textured, "always_list": _always_scene,
          "c4_10k": lambda: _rtiow(50)}


def _sequence(rs, sc, rng, what, oracle, textured=False):
    """Appends, removes, inserts in the middle, and a remove plus insert in one call; each checked."""
    sc = edit(rs, sc, insert=spheres(rng, 3, textured))
    check(rs, sc, what + "/append", oracle)
    rem = sorted(int(i) for i in rng.choice(sc.n_spheres, size=5, replace=False))
    sc = edit(rs, sc, remove=rem)
    check(rs, sc, what + "/remove", oracle)
    at = sorted(int(j) for j in rng.integers(0, sc.n_spheres + 1, size=4))
    sc = edit(rs, sc, insert=spheres(rng, 4, textured), at=at)
    check(rs, sc, what + "/insert in the middle", oracle)
    rem = sorted(int(i) for i in rng.choice(sc.n_spheres, size=3, replace=False))
    at = [rem[0], rem[0], sc.n_spheres // 2, sc.n_spheres]
    sc = edit(rs, sc, remove=rem, insert=spheres(rng, 4, textured), at=sorted(at))
    check(rs, sc, what + "/remove and insert", oracle)
    return sc


@pytest.mark.parametrize("scene", list(SCENES))
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_edit_sequences_render_like_a_fresh_upload(scene, variant):
    sc = SCENES[scene]()
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        _sequence(rs, sc, np.random.default_rng(len(scene) + 7 * VARIANTS[variant]), f"{scene}/{variant}",
                  oracle=scene != "c4_10k", textured=sc.c.n_textures > 0)
    finally:
        rs.release()


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_remove_everything_then_insert_into_the_emptied_handle(variant):
    sc = scenes.cover_scene(32, 24, 2)
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        sc = edit(rs, sc, remove=list(range(sc.n_spheres)))
        assert sc.n_spheres == 0
        check(rs, sc, f"{variant}/emptied")
        t = rs.topology()
        assert (t["n_nodes"], t["n_leaves"], t["depth"], len(t["always"])) == (0, 0, 0, 0)
        if VARIANTS[variant] in (FILTERED, AUTO):                 # what an upload of no spheres holds
            assert t["skip_pos"].tolist() == [0xFFFFFFFF] and t["recentre"].tolist() == [0.0, 0.0, 0.0]
            assert t["level_off"].tolist() == [0]
        rs.rebuild()                                             # a no-op on no spheres
        sc = edit(rs, sc, insert=spheres(np.random.default_rng(2), 6) + [light()])
        check(rs, sc, f"{variant}/refilled")
    finally:
        rs.release()


def test_growth_from_one_sphere_to_100k_and_back():
    """The list grows by appends and inserts from 1 sphere to the 100k-sphere scene and shrinks back. At every step the tree is
    the restatement's of the list and the renders equal a fresh upload's (and the exact f64 variant's)."""
    full = R.Scene.from_config(scenes._variant(scenes.rtiow_config(158), 48, 27, 1, 8))
    objs = [R.rt_sphere.from_buffer_copy(full._spheres[i]) for i in range(full.n_spheres)]
    sc = full.edited(remove=range(1, full.n_spheres))          # the ground
    rs = R.ResidentScene(sc)
    exact = R.make_options(variant=EXACT)
    try:
        done = 1
        for size in (2, 10, 1000, 10_000, full.n_spheres):
            new = objs[done:size]
            at = [min(sc.n_spheres, k * sc.n_spheres // max(len(new), 1)) for k in range(len(new))] if size < 1000 else None
            sc = edit(rs, sc, insert=new, at=at)
            done = size
            assert_same_topology(rs.bvh_records(), restate(*_positions(sc)))
            got = check(rs, sc, f"grown to {size}", oracle=size <= 10)
            _same(got, _fresh(sc, exact), f"grown to {size} vs EXACT_F64")
        rng = np.random.default_rng(5)
        for size in (50_000, 10_000, 100, 1):
            rem = sorted(int(i) for i in rng.choice(sc.n_spheres, size=sc.n_spheres - size, replace=False))
            sc = edit(rs, sc, remove=rem)
            assert_same_topology(rs.bvh_records(), restate(*_positions(sc)))
            check(rs, sc, f"shrunk to {size}", oracle=size <= 100)
    finally:
        rs.release()


# ---- lights ------------------------------------------------------------------------------------------------------------

def _dark_scene():
    return R.Scene.from_config(mixed_config(40, 30, 3, 6, seed=31, n=25))


@pytest.mark.parametrize("variant", ["filtered", "brute_force", "exact_f64"])
def test_the_light_list_follows_the_edits(variant):
    sc = _dark_scene()
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        assert rs.kernel_info()["name"] == R.ResidentScene(sc, rs.opts).kernel_info()["name"]
        sc = edit(rs, sc, insert=[light(0.0, 5.0, 0.0)], at=[4])           # the first light: the lights kernel
        check(rs, sc, "first light")
        fresh = R.ResidentScene(sc, rs.opts)
        for key in ("name", "grid", "ctas_per_sm"):
            assert rs.kernel_info()[key] == fresh.kernel_info()[key], key
        fresh.release()
        first = [i for i in range(sc.n_spheres) if sc._spheres[i].kind == R.RT_LIGHT]
        assert first == [4]
        before = sc.edited(insert=[light(-4.0, 3.0, 5.0, 1.5)], at=[first[0]])   # a light before the existing one
        after = sc.edited(insert=[light(-4.0, 3.0, 5.0, 1.5)], at=[first[0] + 1])
        sc = edit(rs, sc, insert=[light(-4.0, 3.0, 5.0, 1.5)], at=[first[0]])
        got = check(rs, sc, "a light before the existing one")
        _same(got, _render_of(before, rs.opts), "the same list")
        assert not np.array_equal(got[1], _render_of(after, rs.opts)[1]), "light order did not matter"
        lights = [i for i in range(sc.n_spheres) if sc._spheres[i].kind == R.RT_LIGHT]
        sc = edit(rs, sc, remove=[lights[0]])
        check(rs, sc, "one light removed")
        lights = [i for i in range(sc.n_spheres) if sc._spheres[i].kind == R.RT_LIGHT]
        sc = edit(rs, sc, remove=lights, insert=spheres(np.random.default_rng(1), 2))   # the last light
        check(rs, sc, "no lights again")
        assert rs.kernel_info()["name"] == R.ResidentScene(sc, rs.opts).kernel_info()["name"]
    finally:
        rs.release()


def _render_of(sc, opts):
    return _fresh(sc, opts)


@pytest.mark.parametrize("variant", ["filtered", "brute_force"])
def test_nine_lights_and_the_tenth_refused(variant):
    """Nine lights, at max_depth 1: a light test spawns one ray per light, and every such ray that ends on a surface (a light
    included) runs a light test with probability 0.1 * n_lights, so past three lights the recursion is super-critical and a
    render at a depth that starts it does not finish, here or in the reference. At max_depth 1 no light test starts
    (raytracer.rs:99, `depth > max_depth - 2` wraps), and the handle renders with its nine-light list."""
    objs = [{"center": {"x": 0.0, "y": -1000.0, "z": 0.0}, "radius": 1000.0, "material": {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}}]
    objs += [{"center": {"x": -3.0 + 2.0 * k, "y": 0.5, "z": 0.0}, "radius": 0.5, "material": MATS[k % 3]} for k in range(4)]
    sc = R.Scene.from_config(base_config(24, 16, 2, 1, objs))
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        lamps = [light(-4.0 + k, 1.5, -1.0, 0.4) for k in range(9)]                 # in view
        sc = edit(rs, sc, insert=lamps[:2], at=[0, 3])
        sc = edit(rs, sc, insert=lamps[2:], at=[1, 1, 2, 4, 5, 6, sc.n_spheres])
        assert sum(sc._spheres[i].kind == R.RT_LIGHT for i in range(sc.n_spheres)) == 9
        before = check(rs, sc, "nine lights")
        with pytest.raises(R.RtError) as e:
            rs.edit_spheres([], [light(0.0, 3.0, 0.0, 0.5)])
        assert e.value.code == UNSUPPORTED and rs.n == sc.n_spheres
        _same(_render(rs), before, "after the refused tenth light")
    finally:
        rs.release()


# ---- the hierarchy and the arrays ----------------------------------------------------------------------------------------

def test_the_tree_is_the_rebuilds_of_the_new_list():
    """Topology word for word the restatement's; recentring offset, always-list and geo a fresh upload's."""
    sc = _always_scene()
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(8)
    try:
        for step in range(4):
            rem = sorted(int(i) for i in rng.choice(sc.n_spheres, size=3, replace=False))
            ins = spheres(rng, 5) + ([R.make_sphere([2e16, 0.0, 0.0], 1.0, MATS[0])] if step == 1 else [])
            sc = edit(rs, sc, remove=rem, insert=ins, at=sorted(int(j) for j in rng.integers(0, sc.n_spheres - 2, size=len(ins))))
            t = rs.bvh_records()
            assert_same_topology(t, restate(*_positions(sc)))
            host = R.bvh_records(sc)
            assert t["recentre"].view(np.uint64).tolist() == host["recentre"].view(np.uint64).tolist()
            assert np.array_equal(t["always"], host["always"])
            c, r = _positions(sc)
            want = np.concatenate([c, r[:, None]], 1)
            assert t["geo"].view(np.uint64).tolist() == want.view(np.uint64).tolist()
        check(rs, sc, "always-list edits")
    finally:
        rs.release()


@pytest.mark.parametrize("variant", ["brute_force", "exact_f64"])
def test_geo_and_the_flat_padding(variant):
    sc = R.Scene.from_config(mixed_config(24, 18, 1, 3, seed=4, n=40))
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    rng = np.random.default_rng(9)
    try:
        for rem, k in (([], 7), (list(range(0, 40, 3)), 0), ([1, 2, 3], 1), ("all", 0), ([], 3)):
            rem = list(range(rs.n)) if rem == "all" else rem
            sc = edit(rs, sc, remove=rem, insert=spheres(rng, k))
            t = rs.bvh_records()
            c, r = _positions(sc)
            want = np.concatenate([c.reshape(-1, 3), r.reshape(-1, 1)], 1)
            assert t["geo"].view(np.uint64).tolist() == want.view(np.uint64).tolist()
            if variant == "brute_force":
                n_pairs = max(((rs.n + 1) // 2 + 7) // 8 * 8, 8)
                flat = t["flat"].reshape(-1, 2, 4)
                assert len(flat) == n_pairs
                recs = np.array([[flat[s // 2, 0, s % 2], flat[s // 2, 0, 2 + s % 2], flat[s // 2, 1, s % 2], flat[s // 2, 1, 2 + s % 2]]
                                 for s in range(2 * n_pairs)], np.float32)
                pad = recs[rs.n:]
                assert (pad[:, :3] == 0).all() and np.isneginf(pad[:, 3]).all()
                assert np.isfinite(recs[: rs.n, :3]).all() and not np.isneginf(recs[: rs.n, 3]).any()
            check(rs, sc, f"{variant} after {len(rem)} removes, {k} inserts", oracle=False)
    finally:
        rs.release()


# ---- queries, trace_rays, frames, adaptive ------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", list(VARIANTS))
def test_queries_and_trace_rays_after_edits(variant):
    sc = _lit_textured()
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    fresh = None
    try:
        sc = _sequence(rs, sc, np.random.default_rng(11), variant, oracle=False, textured=True)
        fresh = R.ResidentScene(sc, rs.opts)
        rng = np.random.default_rng(12)
        sets = [IR.camera_rays(sc, 40, 30), IR.box_rays(sc, rng, 2000), IR.surface_rays(sc, rng, 1000), IR.degenerate_rays(sc, rng)]
        o = np.concatenate([s[0] for s in sets]); d = np.concatenate([s[1] for s in sets])
        got, want = rs.intersect(o, d), fresh.intersect(o, d)
        IR.assert_hits_equal(got, want, variant + " vs a fresh upload")
        IR.assert_hits_equal(got, IR.oracle(sc, o, d), variant + " vs hit_world")
        t_max = rng.uniform(0.0, 20.0, size=len(o))
        assert np.array_equal(rs.occluded(o, d, t_max)["occluded"], fresh.occluded(o, d, t_max)["occluded"])
        assert np.array_equal(rs.occluded(o, d, t_max)["occluded"], (IR.oracle(sc, o, d, t_max)["sphere"] >= 0).astype(np.uint8))
        tr, tw = rs.trace_rays(o[:1500], d[:1500], 3, rgb8=True), OT.trace_rays(sc, o[:1500], d[:1500], 3)
        bits = (tr["linear"].view(np.uint32) == tw["linear"].view(np.uint32)) | (np.isnan(tr["linear"]) & np.isnan(tw["linear"]))
        assert bits.all() and np.array_equal(tr["rgb8"], tw["rgb8"]) and tr["stats"]["rays"] == tw["rays"]
    finally:
        rs.release()
        if fresh is not None:
            fresh.release()


def test_frames_and_adaptive_renders_after_an_edit():
    import torch
    sc = scenes.cover_scene(40, 30, 2)
    rs = R.ResidentScene(sc)
    try:
        rng = np.random.default_rng(13)
        params = R.make_adaptive(0.05, samples_per_round=2, min_samples=2, max_samples=8)
        rs.adaptive_begin(params)
        sc = edit(rs, sc, remove=[5, 6, 7], insert=spheres(rng, 4) + [light()], at=[0, 10, 10, 20, 30])
        with pytest.raises(R.RtError) as e:                      # an adaptive step does not cross an edit
            rs.adaptive_step(1)
        assert e.value.code == INVALID
        frames = [R.make_frame(sc, seed=5), R.make_frame(sc, look_from=[11.0, 3.0, 6.0], seed=6), R.make_frame(sc, seed=7, max_depth=3)]
        want, _ = R.render_frames(sc, frames)
        want_lin, st_want = R.render_frames(sc, frames, linear=True)
        n = 3 * 40 * 30 * 3
        out = torch.zeros(n, dtype=torch.uint8, device="cuda"); lin = torch.zeros(n, dtype=torch.float32, device="cuda")
        st = rs.render_frames(frames, out.data_ptr(), lin.data_ptr())
        assert np.array_equal(out.cpu().numpy().reshape(want.shape), want)
        assert np.array_equal(lin.cpu().numpy().reshape(want_lin.shape), want_lin) and st["rays"] == st_want["rays"]
        img, lin_a, cnt, _ = R.render_adaptive(sc, params)
        rs.adaptive_begin(params)
        while rs.adaptive_step(4)[0]:
            pass
        d8 = torch.zeros(40 * 30 * 3, dtype=torch.uint8, device="cuda"); dl = torch.zeros(40 * 30 * 3, dtype=torch.float32, device="cuda")
        dc = torch.zeros(40 * 30, dtype=torch.int32, device="cuda")
        rs.adaptive_resolve(d8, dl, dc)
        torch.cuda.synchronize()
        assert np.array_equal(d8.cpu().numpy().reshape(img.shape), img)
        assert np.array_equal(dl.cpu().numpy().reshape(lin_a.shape), lin_a)
        assert np.array_equal(dc.cpu().numpy().reshape(cnt.shape).astype(np.uint32), cnt)
    finally:
        rs.release()


# ---- updates and rebuilds after an edit --------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", ["filtered", "brute_force", "exact_f64"])
def test_updates_and_rebuilds_after_an_edit(variant):
    import torch
    sc = _dark_scene()
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    rng = np.random.default_rng(14)
    try:
        sc = edit(rs, sc, remove=[3, 4], insert=spheres(rng, 6) + [light()], at=[0, 2, 9, 9, 15, 20, 27])
        idx = [1, 5, sc.n_spheres - 1]
        recs = [sc.set_sphere(i, center=[rng.uniform(-3, 3), rng.uniform(0.3, 1.0), rng.uniform(-3, 3)]) for i in idx]
        rs.update_spheres(idx, recs)
        check(rs, sc, "update after an edit")
        lamp = [i for i in range(sc.n_spheres) if sc._spheres[i].kind == R.RT_LIGHT][0]
        with pytest.raises(R.RtError) as e:                      # the light set still changes only by an edit
            rs.update_spheres([lamp], [R.make_sphere([0, 5, 0], 1.0, MATS[0])])
        assert e.value.code == UNSUPPORTED and b"the set of lights is fixed" in R.lib().rtb200_last_error()
        with pytest.raises(ValueError):
            rs.update_geometry(torch.zeros((sc.n_spheres + 2, 4), dtype=torch.float64, device="cuda"))
        c, r = _positions(sc)
        c = c + rng.normal(size=c.shape) * np.array([0.2, 0.0, 0.2]) * (np.abs(r) < 100)[:, None]
        rs.update_geometry(torch.tensor(np.concatenate([c, r[:, None]], 1), dtype=torch.float64, device="cuda"))
        for i in range(sc.n_spheres):
            s = sc._spheres[i]; s.center.x, s.center.y, s.center.z = c[i]
        check(rs, sc, "update_geometry after an edit")
        rs.rebuild()
        check(rs, sc, "rebuild after an edit")
        if variant == "filtered":
            assert_same_topology(rs.bvh_records(), restate(*_positions(sc)))
        sc = edit(rs, sc, remove=[0], insert=spheres(rng, 2))
        check(rs, sc, "edit after a rebuild")
    finally:
        rs.release()


# ---- ordering ----------------------------------------------------------------------------------------------------------

def test_frames_before_an_edit_render_the_old_list_and_frames_after_it_the_new():
    import torch
    sc = scenes.cover_scene(48, 36, 2)
    rs = R.ResidentScene(sc)
    n = 48 * 36 * 3
    s1, s2, s3 = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    bufs = [torch.zeros(n, dtype=torch.uint8, device="cuda") for _ in range(4)]
    rng = np.random.default_rng(15)
    try:
        for round_ in range(3):                                  # later rounds write the halves earlier rounds left
            old = _fresh(sc, None)
            torch.cuda.synchronize()
            for st in (s1, s2):
                with torch.cuda.stream(st):
                    torch.cuda._sleep(HOLD)
            rs.render_async(bufs[0].data_ptr(), 0, s1.cuda_stream)
            rs.render_async(bufs[1].data_ptr(), 0, s2.cuda_stream)
            rem = sorted(int(i) for i in rng.choice(sc.n_spheres, size=4, replace=False))
            sc = edit(rs, sc, remove=rem, insert=spheres(rng, 2 + 300 * (round_ == 1)), stream=s3)   # round 1 grows the block
            rs.render_async(bufs[2].data_ptr(), 0, s1.cuda_stream)
            rs.render_async(bufs[3].data_ptr(), 0, s2.cuda_stream)
            rs.wait()
            torch.cuda.synchronize()
            new = _fresh(sc, None)
            assert not np.array_equal(old[0], new[0])
            for k in range(4):
                assert np.array_equal(bufs[k].cpu().numpy().reshape(36, 48, 3), (old if k < 2 else new)[0]), (round_, k)
    finally:
        rs.release()


def test_queries_on_another_stream_before_an_edit_see_the_old_list():
    import torch
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    try:
        o, d = IR.camera_rays(sc, 64, 48)
        s = torch.cuda.Stream()
        od, dd = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(HOLD)
            h = rs.intersect(od, dd, stream=s)
        new = edit(rs, sc, remove=list(range(1, sc.n_spheres, 2)), insert=spheres(np.random.default_rng(16), 5), at=[0, 0, 1, 2, 3])
        h2 = rs.intersect(od, dd)
        torch.cuda.synchronize()
        IR.assert_hits_equal({k: v.cpu().numpy() for k, v in h.items()}, IR.oracle(sc, o, d), "query before the edit")
        IR.assert_hits_equal({k: v.cpu().numpy() for k, v in h2.items()}, IR.oracle(new, o, d), "query after the edit")
    finally:
        rs.release()


def test_two_handles_on_one_device_one_edited_while_the_other_renders():
    import torch
    a_sc, b_sc = scenes.cover_scene(48, 36, 2), R.Scene.from_config(mixed_config(48, 36, 2, 5, seed=17))
    a, b = R.ResidentScene(a_sc), R.ResidentScene(b_sc)
    try:
        want_b = _fresh(b_sc, None)
        s = torch.cuda.Stream()
        buf = torch.zeros(48 * 36 * 3, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(HOLD)
        b.render_async(buf.data_ptr(), 0, s.cuda_stream)
        a_sc = edit(a, a_sc, remove=[2, 3], insert=spheres(np.random.default_rng(18), 3))
        b.wait()
        torch.cuda.synchronize()
        assert np.array_equal(buf.cpu().numpy().reshape(36, 48, 3), want_b[0])
        check(a, a_sc, "edited beside another handle")
        _same(_render(b), want_b, "the other handle")
    finally:
        a.release(); b.release()


# ---- shards and staged handles -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("world", [2, 3])
def test_row_band_shards(world):
    sc = scenes.cover_scene(40, 30, 2)
    handles = [R.ResidentScene(sc, R.make_options(rank=r, world=world, band_rows=7)) for r in range(world)]
    try:
        rng = np.random.default_rng(world)
        rem = sorted(int(i) for i in rng.choice(sc.n_spheres, size=6, replace=False))
        ins = spheres(rng, 4) + [light()]
        for rs in handles:
            rs.edit_spheres(rem, ins, [0, 3, 3, 50, 100])
        new = sc.edited(rem, ins, [0, 3, 3, 50, 100])
        img_o = O.render(new)[1]
        for r, rs in enumerate(handles):
            got = _render(rs)
            _same(got, _fresh(new, rs.opts), f"shard {r}")
            assert np.array_equal(got[0], img_o[R.shard_row_indices(30, r, world, 7)])
    finally:
        for rs in handles:
            rs.release()


@pytest.mark.parametrize("mask", range(1, 8))
def test_handles_that_stage_the_scene_in_shared_memory_refuse(mask, monkeypatch):
    sc = scenes.cover_scene(32, 24, 1)
    monkeypatch.setenv("RTB200_WF_SMEM", str(mask))
    rs = R.ResidentScene(sc, R.make_options(variant=BRUTE if mask == 4 else FILTERED))
    monkeypatch.delenv("RTB200_WF_SMEM")
    try:
        before = _render(rs)
        with pytest.raises(R.RtError) as e:
            rs.edit_spheres([1], spheres(np.random.default_rng(1), 1))
        assert e.value.code == UNSUPPORTED and rs.n == sc.n_spheres
        _same(_render(rs), before, f"mask {mask} after the refusal")
    finally:
        rs.release()


# ---- refusals ----------------------------------------------------------------------------------------------------------

def test_refused_edits_leave_the_scene_unchanged():
    sc = R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 32, 24, 2, 5), scenes.SCENES_DIR)
    rs = R.ResidentScene(sc)
    L = R.lib()
    try:
        before = _render(rs)
        topo = rs.topology()
        rs.adaptive_begin(R.make_adaptive(0.1, samples_per_round=1, min_samples=1, max_samples=2))
        n = sc.n_spheres
        ok = spheres(np.random.default_rng(2), 2)
        bad_kind = R.make_sphere([0, 1, 0], 0.5, MATS[0]); bad_kind.kind = 9
        bad_tex = R.make_sphere([0, 1, 0], 0.5, {"Texture": {"albedo": [1, 1, 1], "h_offset": 0.0, "texture": 0}}); bad_tex.texture = 99
        cases = [([n], [], None, INVALID, b"not a sphere"), ([1, 1], [], None, INVALID, b"twice"),
                 ([], ok, [3, 2], INVALID, b"decreases"), ([], ok, [0, n + 1], INVALID, b"exceeds"),
                 ([], [bad_kind], None, INVALID, b"unknown material kind (insert[0])"),
                 ([], [ok[0], bad_tex], None, INVALID, b"texture index out of range"),
                 ([], [light(k, 9.0, 0.0, 0.2) for k in range(10 - sum(sc._spheres[i].kind == R.RT_LIGHT for i in range(n)))],
                  None, UNSUPPORTED, b"10 or more lights")]
        for rem, ins, at, code, msg in cases:
            r = np.ascontiguousarray(rem, dtype=np.uint32)
            a = None if at is None else np.ascontiguousarray(at, dtype=np.uint32)
            arr = (R.rt_sphere * max(len(ins), 1))(*ins)
            rc = L.rtb200_scene_edit_spheres(rs.h, r.ctypes.data if r.size else None, r.size, None if a is None else a.ctypes.data,
                                             arr, len(ins), None)
            assert rc == code and msg in L.rtb200_last_error(), (msg, rc, L.rtb200_last_error())
        assert L.rtb200_scene_edit_spheres(rs.h, None, 0, None, None, 0, None) == 0   # an edit of nothing
        rs.adaptive_step(1)                                      # no refused edit counted as an update
        _same(_render(rs), before, "after the refused edits")
        t = rs.topology()
        for key in ("leaf_id", "always", "skip_pos", "level_nodes"):
            assert np.array_equal(t[key], topo[key]), key
    finally:
        rs.release()


# ---- the stress builds -------------------------------------------------------------------------------------------------

def test_stress_builds_edit_exactly(tmp_path):
    """Every stress build's edited handles render what the oracle renders (the coincident scene: what a fresh RT_VARIANT_EXACT_F64
    upload of the default build renders) and answer queries as hit_world does."""
    manifest = json.load(open(os.path.join(STRESS, "manifest.json")))
    wants = {}
    for name in EW.SETS:
        _, _, sc = EW.edited(name)
        if name == "coincident":
            img, lin, rays = _fresh(sc, R.make_options(variant=EXACT))
        else:
            lin, img, st = O.render(sc)
            rays = st["rays"]
        o, d = EW.rays(sc, 80)
        hits = IR.oracle(sc, o, d)
        wants[name] = (img, lin, rays, hits, (hits["sphere"] >= 0).astype(np.uint8))
    for build in manifest:
        out = tmp_path / f"{build}.npz"
        env = dict(os.environ, RTB200_LIB=os.path.join(STRESS, f"librtb200_{build}.so"))
        subprocess.run([sys.executable, os.path.join(REPO, "tests", "edit_worker.py"), str(out)], env=env, check=True, timeout=900)
        z = np.load(out)
        meta = json.loads(str(z["meta"]))
        for name, (img, lin, rays, hits, occ) in wants.items():
            _same((z[f"{name}.rgb8"], z[f"{name}.linear"], meta[name]), (img, lin, rays), f"{build}/{name}")
            IR.assert_hits_equal({k: z[f"{name}.{k}"] for k in IR.FIELDS}, hits, f"{build}/{name}")
            assert np.array_equal(z[f"{name}.occluded"], occ), (build, name)
