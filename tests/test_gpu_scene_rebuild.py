"""Rebuilding the hierarchy of a resident scene on the GPU (rtb200_scene_rebuild): after moves and a rebuild every render of the
handle is bit-identical, in linear f32, RGB8 and ray count, to the CPU oracle and to a fresh upload of the current spheres;
the rebuilt topology keeps the invariants the traversal and the refit rely on, its recentring offset and always-list are a
fresh upload's, its values are the numpy refit of tests/test_scene_update_cpu.py on it, and it is deterministic."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from synth import base_config, mixed_config, _v
from rebuild_restatement import MAX_DEPTH, check_tree, skip_rule
from test_gpu_scene_update import HOLD, _assert_same, _check, _fresh, _jitter, _light_scene, _positions, _render
from test_scene_update_cpu import refit, same_bits

pytestmark = pytest.mark.gpu
EXACT = R.make_options(variant=R.RT_VARIANT_EXACT_F64)


def check_topology(rs, sc, rays=0):
    """Every invariant of a rebuilt hierarchy (rebuild_restatement.check_tree) for the host scene sc (the handle's current
    spheres), and the recentring offset (bit for bit) and always-list of a fresh upload of sc. Returns the records."""
    t = rs.bvh_records()
    c, r = _positions(sc)
    host = R.bvh_records(sc)
    assert np.array_equal(t["always"], host["always"]), "always-list differs from a fresh upload's"
    assert t["recentre"].view(np.uint64).tolist() == host["recentre"].view(np.uint64).tolist(), (t["recentre"], host["recentre"])
    cam = [sc.c.camera.origin.x, sc.c.camera.origin.y, sc.c.camera.origin.z]
    check_tree(t, c, r, rays=rays, cam=cam)
    return t


def _move_all(sc, rng, scale=0.5, ground=True):
    idx = list(range(sc.n_spheres)) if ground else list(range(1, sc.n_spheres))
    recs = []
    for i in idx:
        s = sc._spheres[i]
        recs.append(sc.set_sphere(i, center=[s.center.x + rng.normal() * scale, s.center.y + abs(rng.normal()) * scale * 0.3,
                                             s.center.z + rng.normal() * scale]))
    return idx, recs


def test_cover_scene_after_moves_and_a_rebuild():
    sc = scenes.cover_scene(64, 48, 4)
    rs = R.ResidentScene(sc)
    idx, recs = _move_all(sc, np.random.default_rng(1), scale=1.5)
    recs[0] = sc.set_sphere(0, center=[0.5, -1000.2, -0.3])          # the ground moves too
    rs.update_spheres(idx, recs)
    rs.rebuild()
    check_topology(rs, sc, rays=150)
    _check(rs, sc, what="cover after a rebuild")
    rs.release()


@pytest.mark.parametrize("n_lights,depth", [(1, 1), (2, 2), (1, 6), (2, 6)])
def test_mixed_scenes_with_lights(n_lights, depth):
    sc = _light_scene(n_lights, depth, seed=60 + depth)
    rs = R.ResidentScene(sc)
    lights = {i for i in range(sc.n_spheres) if sc._spheres[i].kind == R.RT_LIGHT}
    idx, recs = _jitter(sc, np.random.default_rng(depth), 20, scale=1.0)
    rs.update_spheres(idx, recs)
    rs.rebuild()
    assert lights
    check_topology(rs, sc)
    _check(rs, sc, what=f"{n_lights} lights, depth {depth}")
    rs.release()


def test_textured_test_scene():
    sc = R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 64, 48, 2, 6), scenes.SCENES_DIR)
    rs = R.ResidentScene(sc)
    idx, recs = _jitter(sc, np.random.default_rng(2), sc.n_spheres // 2, scale=0.8)
    rs.update_spheres(idx, recs)
    rs.rebuild()
    check_topology(rs, sc)
    _check(rs, sc, what="textured")
    rs.release()


@pytest.mark.parametrize("world", [2, 3])
def test_row_band_shards(world):
    sc = scenes.cover_scene(48, 40, 2)
    handles = [R.ResidentScene(sc, R.make_options(rank=r, world=world, band_rows=7)) for r in range(world)]
    idx, recs = _move_all(sc, np.random.default_rng(world))
    img_o, rays = O.render(sc)[1], 0
    for r, rs in enumerate(handles):
        rs.update_spheres(idx, recs)
        rs.rebuild()
        got = _check(rs, sc, oracle=False, what=f"shard {r}")
        assert np.array_equal(got[0], img_o[R.shard_row_indices(40, r, world, 7)])
        rays += got[2]
        rs.release()
    assert rays == _fresh(sc)[2]


def test_render_frames_after_a_rebuild():
    import torch
    sc = scenes.cover_scene(48, 36, 2)
    rs = R.ResidentScene(sc)
    idx, recs = _move_all(sc, np.random.default_rng(3))
    rs.update_spheres(idx, recs)
    rs.rebuild()
    frames = [R.make_frame(sc, seed=5), R.make_frame(sc, look_from=[11.0, 3.0, 6.0], seed=6), R.make_frame(sc, seed=7, max_depth=3)]
    want, _ = R.render_frames(sc, frames)
    want_lin, st_want = R.render_frames(sc, frames, linear=True)
    n = 3 * 48 * 36 * 3
    out = torch.zeros(n, dtype=torch.uint8, device="cuda"); lin = torch.zeros(n, dtype=torch.float32, device="cuda")
    st = rs.render_frames(frames, out.data_ptr(), lin.data_ptr())
    assert np.array_equal(out.cpu().numpy().reshape(want.shape), want)
    assert np.array_equal(lin.cpu().numpy().reshape(want_lin.shape), want_lin) and st["rays"] == st_want["rays"]
    rs.release()


def test_positions_from_a_tensor_on_a_torch_stream_right_before_the_rebuild():
    import torch
    sc = scenes.cover_scene(48, 36, 2)
    rs = R.ResidentScene(sc)
    c, r = _positions(sc)
    g = torch.tensor(np.concatenate([c, r[:, None]], axis=1), dtype=torch.float64, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(HOLD)                             # t is written only after the sleep
        t = g + torch.randn(g.shape, generator=torch.Generator(device="cuda").manual_seed(4), device="cuda", dtype=torch.float64) \
            * torch.tensor([0.8, 0.1, 0.8, 0.0], device="cuda", dtype=torch.float64)
        rs.update_geometry(t)
        rs.rebuild()                                        # on torch's current stream, s
    torch.cuda.synchronize()
    new = t.cpu().numpy()
    for i in range(sc.n_spheres):
        sc.set_sphere(i, center=new[i, :3].tolist(), radius=float(new[i, 3]))
    check_topology(rs, sc)
    _check(rs, sc, what="tensor positions")
    rs.release()


def test_frames_in_flight_keep_the_old_tree_and_later_frames_get_the_new_one():
    import torch
    sc = scenes.cover_scene(64, 48, 4)
    old = _fresh(sc)
    rs = R.ResidentScene(sc)
    n = 64 * 48 * 3
    s1, s2, s3 = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    bufs = [torch.zeros(n, dtype=torch.uint8, device="cuda") for _ in range(4)]
    for rebuilt_before in (False, True):                     # the second round overwrites the first rebuild's arrays
        torch.cuda.synchronize()
        for st in (s1, s2):
            with torch.cuda.stream(st):
                torch.cuda._sleep(HOLD)
        rs.render_async(bufs[0].data_ptr(), 0, s1.cuda_stream)
        rs.render_async(bufs[1].data_ptr(), 0, s2.cuda_stream)
        idx, recs = _move_all(sc, np.random.default_rng(5 + rebuilt_before))
        rs.update_spheres(idx, recs, s3.cuda_stream)
        rs.rebuild(s3)
        rs.render_async(bufs[2].data_ptr(), 0, s1.cuda_stream)
        rs.render_async(bufs[3].data_ptr(), 0, s2.cuda_stream)
        rs.wait()
        torch.cuda.synchronize()
        new = _fresh(sc)
        assert not np.array_equal(old[0], new[0])
        for k in range(4):
            assert np.array_equal(bufs[k].cpu().numpy().reshape(48, 64, 3), (old if k < 2 else new)[0]), (rebuilt_before, k)
        old = new
    rs.release()


def _arrays(rs):
    t = rs.bvh_records()
    return {k: t[k].copy() for k in ("lo", "hi", "child", "leaf_rec", "leaf_id", "always", "skip_pos", "level_nodes", "level_off", "recentre")}


def test_rebuilds_are_deterministic():
    sc = scenes.cover_scene(32, 24, 1)
    a = R.ResidentScene(sc)
    b = R.ResidentScene(sc)
    idx, recs = _move_all(sc, np.random.default_rng(9), scale=2.0)
    a.update_spheres(idx, recs); b.update_spheres(idx, recs)
    a.rebuild()
    first = _arrays(a)
    a.rebuild()
    b.rebuild()
    for other in (_arrays(a), _arrays(b)):
        for key, v in first.items():
            assert v.shape == other[key].shape and v.tobytes() == other[key].tobytes(), key
    a.release(); b.release()


def test_refit_after_a_rebuild():
    sc = scenes.cover_scene(48, 36, 2)
    rs = R.ResidentScene(sc)
    idx, recs = _move_all(sc, np.random.default_rng(12), scale=1.0)
    rs.update_spheres(idx, recs)
    rs.rebuild()
    topo = rs.bvh_records()
    idx, recs = _jitter(sc, np.random.default_rng(13), 80, scale=0.7)
    rs.update_spheres(idx, recs)
    got = rs.bvh_records()
    for key in ("child", "leaf_id", "skip_pos", "level_nodes", "always"):
        assert np.array_equal(got[key], topo[key]), key                  # an update keeps the rebuilt topology
    c, r = _positions(sc)
    b = dict(topo)
    b["flat"] = np.zeros((max((sc.n_spheres + 1) // 2, 1), 2, 4), np.float32)
    want = refit(b, c, r)
    for key in ("lo", "hi", "leaf_rec"):
        assert same_bits(got[key], want[key]), key
    _check(rs, sc, what="refit after a rebuild")
    rs.release()


def _objs(centres, radii):
    mats = [{"Lambertian": {"albedo": [0.7, 0.3, 0.2]}}, {"Metal": {"albedo": [0.8, 0.8, 0.9], "fuzz": 0.2}},
            {"Glass": {"index_of_refraction": 1.5}}]
    return [{"center": _v(*map(float, c)), "radius": float(r), "material": mats[i % 3]} for i, (c, r) in enumerate(zip(centres, radii))]


def _adversarial(kind):
    rng = np.random.default_rng(21)
    if kind[1:].isdigit():                            # n<m>: m spheres (n1, and n = leaf size and one more)
        m = int(kind[1:])
        c = rng.uniform(-2, 2, size=(m, 3)); c[:, 1] = np.abs(c[:, 1]); r = rng.uniform(0.2, 0.6, m)
    elif kind == "coincident":
        c = np.tile([[0.0, 0.5, 0.0]], (10_000, 1)); r = np.full(10_000, 0.5)
    elif kind == "exponential":
        m = 64
        c = np.stack([2.0 ** -np.arange(m), np.zeros(m), np.zeros(m)], 1); r = 2.0 ** -np.arange(m) * 0.4
    elif kind == "spread":
        m = 300
        c = rng.normal(size=(m, 3)) * np.logspace(0, 14, m)[:, None]; r = np.abs(c).max(axis=1) * 0.01 + 0.3
    elif kind == "nonfinite":
        m = 80
        c = rng.uniform(-4, 4, size=(m, 3)); r = rng.uniform(0.1, 0.5, m)
    return R.Scene.from_config(base_config(24, 18, 2, 4, _objs(c, r)))


@pytest.mark.parametrize("kind", ["n1", "n8", "n9", "coincident", "exponential", "spread", "nonfinite"])
def test_adversarial_inputs(kind):
    sc = _adversarial(kind)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(31)
    if kind == "nonfinite":
        recs = [sc.set_sphere(3, radius=np.nan), sc.set_sphere(4, radius=np.inf), sc.set_sphere(5, center=[np.inf, 0.0, 0.0]),
                sc.set_sphere(6, center=[1e16, 0.0, 0.0])]
        rs.update_spheres([3, 4, 5, 6], recs)
    else:
        idx, recs = _jitter(sc, rng, sc.n_spheres, scale=0.05 if kind != "coincident" else 0.0)
        rs.update_spheres(idx, recs)
    rs.rebuild()
    t = check_topology(rs, sc, rays=40 if kind not in ("coincident",) else 0)
    assert t["depth"] <= MAX_DEPTH
    got = _check(rs, sc, oracle=kind != "coincident", what=kind)   # a render that succeeds: the traversal guard never tripped
    if kind == "coincident":                                      # too many spheres per ray for the oracle: the exact variant
        _assert_same(got, _fresh(sc, EXACT), "coincident vs EXACT_F64")
    rs.release()


def test_spheres_leave_the_f32_frame_and_come_back():
    sc = R.Scene.from_config(mixed_config(32, 24, 2, 4, seed=14, n=100))
    rs = R.ResidentScene(sc)
    c0, r0 = _positions(sc)
    out = {2: [1e16, 0.0, 0.0], 5: [np.nan, 0.0, 0.0], 9: [0.0, 2e15, 0.0], 11: [-np.inf, 1.0, 1.0]}
    rs.update_spheres(list(out), [sc.set_sphere(i, center=v) for i, v in out.items()])
    rs.rebuild()
    t = check_topology(rs, sc)
    assert set(t["always"].tolist()) == set(out)
    _check(rs, sc, what="out of frame")
    rs.update_spheres(list(out), [sc.set_sphere(i, center=c0[i].tolist()) for i in out])
    rs.rebuild()
    t = check_topology(rs, sc, rays=60)
    assert len(t["always"]) == 0
    _check(rs, sc, what="back in the frame")
    rs.release()


def test_the_100k_sphere_scene():
    import torch
    sc = R.Scene.from_config(scenes._variant(scenes.rtiow_config(158), 48, 27, 2, 8))
    rs = R.ResidentScene(sc)
    c, r = _positions(sc)
    rng = np.random.default_rng(7)
    c = c + rng.normal(size=c.shape) * np.array([0.3, 0.0, 0.3]) * (np.abs(r) < 100)[:, None]
    rs.update_geometry(torch.tensor(np.concatenate([c, r[:, None]], 1), dtype=torch.float64, device="cuda"))
    for i in range(sc.n_spheres):
        s = sc._spheres[i]; s.center.x, s.center.y, s.center.z = c[i]
    rs.rebuild()
    t = check_topology(rs, sc)
    assert t["depth"] <= MAX_DEPTH and sc.n_spheres > 90_000
    got = _check(rs, sc, oracle=False, what="100k")
    _assert_same(got, _fresh(sc, EXACT), "100k vs EXACT_F64")
    rs.release()


@pytest.mark.parametrize("variant", [R.RT_VARIANT_EXACT_F64, R.RT_VARIANT_BRUTE_FORCE])
def test_rebuild_is_a_no_op_without_a_hierarchy(variant):
    sc = R.Scene.from_config(mixed_config(32, 24, 2, 4, seed=9))
    rs = R.ResidentScene(sc, R.make_options(variant=variant))
    idx, recs = _jitter(sc, np.random.default_rng(variant), 20, scale=1.0)
    rs.update_spheres(idx, recs)
    before = _render(rs)
    assert R.lib().rtb200_scene_rebuild(rs.h, None) == 0
    _assert_same(_render(rs), before, "after a no-op rebuild")
    _check(rs, sc, what=f"variant {variant}")
    rs.release()


def test_rebuild_of_an_empty_scene_is_a_no_op():
    sc = R.Scene.from_config(base_config(16, 12, 1, 2, []))
    rs = R.ResidentScene(sc)
    rs.rebuild()
    assert rs.topology()["n_nodes"] == 0
    _check(rs, sc, what="empty scene")
    rs.release()


def test_topology_of_a_handle_never_rebuilt_is_the_uploads():
    sc = R.Scene.from_config(mixed_config(32, 24, 1, 4, seed=12, n=120))
    rs = R.ResidentScene(sc)
    t, host = rs.bvh_records(), R.bvh_records(sc)
    for key in ("leaf_id", "always", "recentre", "child", "lo", "hi", "leaf_rec"):
        assert np.array_equal(t[key], host[key]), key
    assert np.array_equal(t["skip_pos"], skip_rule(host, sc.n_spheres))
    assert t["depth"] == host["depth"] and len(t["level_off"]) == host["depth"] + 1
    rs.release()
    info = (C.c_uint32 * 8)()
    assert R.lib().rtb200_scene_debug_topology(None, None, info, None, 0, None, 0, None, 0, None, 0, None, 0) == -1
