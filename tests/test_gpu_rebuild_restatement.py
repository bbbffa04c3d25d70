"""The GPU rebuild (rtb200_scene_rebuild) against its numpy restatement (tests/rebuild_restatement.py): after every rebuild
the device's topology equals the restatement field by field, the recentring offset bit for bit, and its values are the
numpy refit on it. On the deepest, densest rebuilt trees every render path (one frame, the multi-frame kernel, the lights
kernel) is bit-identical, in linear f32, RGB8 and ray count, to RT_VARIANT_EXACT_F64, which tests every sphere in f64 and
traverses nothing, and to the CPU oracle where it finishes."""
import os

import numpy as np
import pytest

import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from rebuild_restatement import K, check_tree, rebuild
from synth import base_config, mixed_config
from test_gpu_scene_rebuild import _adversarial, _move_all, _objs
from test_gpu_scene_update import _assert_same, _fresh, _positions
from test_rebuild_restatement_cpu import DEEP, deep_spheres, mixed_zero_centres, oversize_pair

pytestmark = pytest.mark.gpu
EXACT = R.make_options(variant=R.RT_VARIANT_EXACT_F64)


def assert_same_topology(dev, want):
    assert dev["recentre"].view(np.uint64).tolist() == want["recentre"].view(np.uint64).tolist(), \
        ("recentre", dev["recentre"], want["recentre"])
    for key in ("n_nodes", "n_leaves", "depth"):
        assert dev[key] == want[key], (key, dev[key], want[key])
    for key in ("always", "leaf_id", "child", "skip_pos", "level_nodes", "level_off"):
        a, b = np.asarray(dev[key]), np.asarray(want[key])
        assert a.shape == b.shape, (key, a.shape, b.shape)
        bad = np.nonzero(a.ravel() != b.astype(a.dtype).ravel())[0]
        assert not len(bad), (key, f"{len(bad)} words differ, first at {np.unravel_index(bad[0], a.shape)}")


def rebuilt(rs, sc, oversize=None, leaf_size=K):
    """Rebuild rs, whose spheres are sc's, and check the device's topology against the restatement and its values
    against the numpy refit, at the library's leaf size; returns the device's records."""
    if oversize is None:
        rs.rebuild()
        want = rebuild(*_positions(sc), leaf_size=leaf_size)
    else:
        old = os.environ.get("RTB200_REBUILD_OVERSIZE")
        os.environ["RTB200_REBUILD_OVERSIZE"] = str(oversize)
        try:
            rs.rebuild()
        finally:
            if old is None:
                del os.environ["RTB200_REBUILD_OVERSIZE"]
            else:
                os.environ["RTB200_REBUILD_OVERSIZE"] = old
        want = rebuild(*_positions(sc), oversize=oversize, leaf_size=leaf_size)
    dev = rs.bvh_records()
    assert_same_topology(dev, want)
    check_tree(dev, *_positions(sc), leaf_size=leaf_size)
    return dev


def _geometry(rs, sc, c):
    import torch
    _, r = _positions(sc)
    rs.update_geometry(torch.tensor(np.concatenate([c, r[:, None]], 1), dtype=torch.float64, device="cuda"))
    for i in range(sc.n_spheres):
        s = sc._spheres[i]; s.center.x, s.center.y, s.center.z = c[i]


def _drifted(sc, seed):
    c, r = _positions(sc)
    rng = np.random.default_rng(seed)
    return c + rng.normal(size=c.shape) * np.array([0.3, 0.0, 0.3]) * (np.abs(r) < 100)[:, None]


def _scene(c, r, w=24, h=18, spp=2, depth=4, **kw):
    return R.Scene.from_config(base_config(w, h, spp, depth, _objs(c, r), **kw))


def test_cover_scene_after_moves_with_the_ground():
    sc = scenes.cover_scene(64, 48, 2)
    rs = R.ResidentScene(sc)
    idx, recs = _move_all(sc, np.random.default_rng(1), scale=1.5)
    recs[0] = sc.set_sphere(0, center=[0.5, -1000.2, -0.3])
    rs.update_spheres(idx, recs)
    rebuilt(rs, sc)
    idx, recs = _move_all(sc, np.random.default_rng(2), scale=0.7)   # and a second rebuild on the first one's block
    rs.update_spheres(idx, recs)
    rebuilt(rs, sc)
    rs.release()


@pytest.mark.parametrize("what", ["c4_10k", "100k"])
def test_drifted_grid_scenes(what):
    sc = R.Scene.from_config(scenes._variant(scenes.rtiow_config(50 if what == "c4_10k" else 158), 32, 18, 1, 4))
    rs = R.ResidentScene(sc)
    _geometry(rs, sc, _drifted(sc, 7))
    t = rebuilt(rs, sc)
    assert t["depth"] >= 5
    rs.release()


@pytest.mark.parametrize("kind", ["n1", "n8", "n9", "coincident", "exponential", "spread", "nonfinite"])
def test_adversarial_inputs(kind):
    sc = _adversarial(kind)
    rs = R.ResidentScene(sc)
    if kind == "nonfinite":
        recs = [sc.set_sphere(3, radius=np.nan), sc.set_sphere(4, radius=np.inf), sc.set_sphere(5, center=[np.inf, 0.0, 0.0]),
                sc.set_sphere(6, center=[1e16, 0.0, 0.0])]
        rs.update_spheres([3, 4, 5, 6], recs)
    rebuilt(rs, sc)
    rs.release()


@pytest.mark.parametrize("n", [4_096, 32_768, 262_144])
def test_deep_constructions(n):
    c, r = deep_spheres(n)
    sc = _scene(c, r)
    rs = R.ResidentScene(sc)
    t = rebuilt(rs, sc)
    assert t["depth"] == DEEP[n]
    rs.release()


def test_the_oversize_edge_pair_and_the_rule_turned_off():
    c, r = oversize_pair()
    sc = _scene(c, r)
    rs = R.ResidentScene(sc)
    rebuilt(rs, sc)
    rs.release()
    sc = scenes.cover_scene(48, 36, 1)                     # the ground is the oversized sphere
    rs = R.ResidentScene(sc)
    idx, recs = _move_all(sc, np.random.default_rng(4), scale=1.0)
    rs.update_spheres(idx, recs)
    off = rebuilt(rs, sc, oversize=0)
    on = rebuilt(rs, sc)
    assert not np.array_equal(off["leaf_id"], on["leaf_id"])
    rs.release()


def test_nan_and_inf_centres():
    sc = R.Scene.from_config(mixed_config(32, 24, 1, 4, seed=14, n=100))
    rs = R.ResidentScene(sc)
    out = {2: [1e16, 0.0, 0.0], 5: [np.nan, 0.0, 0.0], 9: [0.0, 2e15, 0.0], 11: [-np.inf, 1.0, 1.0], 12: [1.0, np.nan, np.inf],
           13: [np.nan, np.nan, np.nan]}
    rs.update_spheres(list(out), [sc.set_sphere(i, center=v) for i, v in out.items()])
    t = rebuilt(rs, sc)
    assert set(t["always"].tolist()) == set(out)
    rs.release()


def test_a_median_that_is_a_zero_of_mixed_sign():
    c, r = mixed_zero_centres()
    for perm in (np.arange(len(r)), np.random.default_rng(5).permutation(len(r))):
        sc = _scene(c[perm], r[perm])
        rs = R.ResidentScene(sc)
        t = rebuilt(rs, sc)
        assert t["recentre"].view(np.uint64).tolist() == R.bvh_records(sc)["recentre"].view(np.uint64).tolist()   # a fresh upload's
        rs.release()


# ---- deep, dense trees traced against RT_VARIANT_EXACT_F64 ----

def _deep_dense(n, lights):
    """deep_spheres(n): the last cell holds thousands of spheres that overlap each other and the peeled ones near it. The
    camera looks into it from close by; `lights` light spheres sit in the far octant of the Morton box."""
    c, r = deep_spheres(n)
    objs = _objs(c, r)
    for k in range(lights):
        objs.append({"center": {"x": 100.0 + 6.0 * k, "y": 100.0, "z": 100.0}, "radius": 1.0, "material": {"Light": {}}})
    return R.Scene.from_config(base_config(48, 36, 2, 5, objs, look_from=(0.9, 0.35, 0.65), look_at=(0.06, 0.06, 0.06), vfov=30.0))


def _coincident(lights):
    """The 10,000 coincident spheres of test_gpu_scene_rebuild._adversarial, and `lights` light spheres beside them."""
    c = np.tile([[0.0, 0.5, 0.0]], (10_000, 1))
    objs = _objs(c, np.full(10_000, 0.5))
    objs += [{"center": {"x": 2.0 + 3.0 * k, "y": 3.0, "z": 0.0}, "radius": 0.7, "material": {"Light": {}}} for k in range(lights)]
    return R.Scene.from_config(base_config(24, 18, 2, 4, objs))


def _render_stats(rs):
    import torch
    n = rs.rows * rs.scene.c.width * 3
    d8 = torch.zeros(n, dtype=torch.uint8, device="cuda")
    dl = torch.zeros(n, dtype=torch.float32, device="cuda")
    st = rs.render(d8.data_ptr(), dl.data_ptr())            # a clean return: no traversal guard tripped
    shape = (rs.rows, rs.scene.c.width, 3)
    return (d8.cpu().numpy().reshape(shape), dl.cpu().numpy().reshape(shape), st["rays"]), st


def _frames_check(rs, sc, what):
    import torch
    frames = [R.make_frame(sc, seed=5), R.make_frame(sc, seed=6, max_depth=3)]
    w, h = sc.c.width, sc.c.height
    n = len(frames) * h * w * 3
    out = torch.zeros(n, dtype=torch.uint8, device="cuda")
    lin = torch.zeros(n, dtype=torch.float32, device="cuda")
    st = rs.render_frames(frames, out.data_ptr(), lin.data_ptr())
    want, st_want = R.render_frames(sc, frames, EXACT)
    want_lin, _ = R.render_frames(sc, frames, EXACT, linear=True)
    assert np.array_equal(lin.cpu().numpy().reshape(want_lin.shape), want_lin), f"{what}: frames linear differs"
    assert np.array_equal(out.cpu().numpy().reshape(want.shape), want), f"{what}: frames rgb8 differs"
    assert st["rays"] == st_want["rays"], (what, st["rays"], st_want["rays"])


# (construction, lights) -> at least this many f64-confirmed sphere tests per ray on the rebuilt handle (measured on an
# H100: about 2170 and 1860 for the deep construction, 397 for the coincident spheres)
DENSE = {("deep", 0): 1000, ("deep", 2): 1000, ("coincident", 0): 300, ("coincident", 1): 300}


@pytest.mark.parametrize("kind,lights", sorted(DENSE))
def test_deep_dense_trees_trace_like_the_exact_f64_variant(kind, lights):
    n = 32_768
    sc = _deep_dense(n, lights) if kind == "deep" else _coincident(lights)
    rs = R.ResidentScene(sc)
    t = rebuilt(rs, sc)
    assert t["depth"] >= (DEEP[n] if kind == "deep" else 4), t["depth"]
    got, st = _render_stats(rs)
    _assert_same(got, _fresh(sc, EXACT), f"{kind}, {lights} lights vs EXACT_F64")
    per_ray = st["candidates"] / st["rays"]
    print(f"{kind} lights={lights}: n={sc.n_spheres} depth={t['depth']} nodes={t['n_nodes']} rays={st['rays']} "
          f"candidates/ray={per_ray:.1f} nodes/ray={st['nodes'] / st['rays']:.1f}")
    assert per_ray >= DENSE[(kind, lights)], per_ray
    _frames_check(rs, sc, f"{kind}, {lights} lights")
    if kind == "coincident" or lights == 0:
        lin_o, img_o, st_o = O.render(sc)
        _assert_same(got, (img_o, lin_o, st_o["rays"]), f"{kind}, {lights} lights vs the oracle")
    rs.release()
