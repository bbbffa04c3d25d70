"""The topology of the GPU rebuild (rtb200_scene_rebuild, DESIGN.md §4.8) through its numpy restatement
(tests/rebuild_restatement.py), no GPU: on inputs at the leaf and fan-out edges, on degenerate inputs and on trees built to
be as deep as the key layout allows, the rebuilt tree keeps the depth bound the trace's node stack relies on and the sizes
rebuild_carve allocates, and the float32 traversal of the refitted tree never drops a sphere the exact f64 test accepts.
The host builder chooses the same recentring offset as the rebuild. The GPU tests compare the device's topology with this
restatement byte for byte. The edge cases and the deep constructions also run at every leaf size the stress builds use.
"""
import numpy as np
import pytest

import rtb200 as R
from rtb200 import scenes
from rebuild_restatement import K, MAX_DEPTH, OVERSIZE, check_tree, filled, rebuild, sort_keys, sound
from synth import base_config, _v
from test_bvh_cpu import _spheres

MORTON_LEVELS = 10                      # 30 Morton bits, 3 per wide level
PEEL = (1, 1, 8, 1, 8, 1, 8)            # spheres in octants 1..7 of a peeled level (see deep_spheres)


def deep_spheres(n, radius=0.75, scale=0.125):
    """(c, r) of n > 288 spheres whose rebuilt tree is about as deep as the key layout allows at that size. Every wide
    level cuts the deepest range at least 3 key bits further down, and the keys of n spheres differ in at most 30 Morton
    bits and log2(n) index bits, so the depth is about (30 + log2 n) / 3 at most. In cell units of the Morton grid (1024 cells on
    the box; world = cells * scale, so every coordinate is exact), level k of the first ten splits the cube [0, 2^(10-k))^3
    into its octants: octant 0 goes on, and octants 1..7 get PEEL spheres at their lower corner. Those sizes make the
    level's 7 splits cut the three Morton bits of level k breadth first (the ranges of octants {2,3}, {4,5}, {6,7} hold more
    than 8 spheres), so the deep range loses exactly 3 bits per level. The rest sit in the last cell, at sub-cell positions
    that keep Morton code 0, and are split by the bits of their index, the scene-list order, 3 per level: at the radix
    split points until level 13, by halving below. One peel sphere sits at (1024, 1024, 1024), on the upper face of the
    Morton box, where t = 1024 is clamped to 1023."""
    rng = np.random.default_rng(n)
    cells = []
    for k in range(MORTON_LEVELS):
        h = 2 ** (9 - k)
        for v, m in zip(range(1, 8), PEEL):
            cells += [[(v >> 2 & 1) * h, (v >> 1 & 1) * h, (v & 1) * h]] * m
    cells[sum(PEEL[:6])] = [1024, 1024, 1024]         # the first sphere of octant 7 on level 0
    rest = n - len(cells)
    assert rest > K
    last = rng.integers(0, 1024, size=(rest, 3)) / 1024.0
    last[0] = 0.0                                      # the box's lower corner
    c = np.concatenate([np.array(cells, np.float64), last]) * scale
    return c, np.full(n, radius * scale)


# depth of the rebuilt tree of deep_spheres(n): 10 Morton levels, then the index bits of the last cell, 3 per level
DEEP = {300: 11, 4_096: 13, 32_768: 14, 262_144: 15, 1_000_000: 16}


def _uniform(n, seed=1):
    rng = np.random.default_rng(seed)
    return rng.uniform(-50, 50, (n, 3)), rng.uniform(0.1, 0.6, n)


def _case(kind):
    rng = np.random.default_rng(3)
    if kind[1:].isdigit():
        return _uniform(int(kind[1:]))
    if kind == "coincident":
        return np.tile([[0.0, 0.5, 0.0]], (10_000, 1)), np.full(10_000, 0.5)
    if kind == "exponential":
        m = 1000
        return np.stack([2.0 ** -np.arange(m), np.zeros(m), np.zeros(m)], 1), 2.0 ** -np.arange(m) * 0.4
    if kind == "line":
        m = 5000
        return np.stack([np.arange(m) * 0.5, np.zeros(m), np.zeros(m)], 1), np.full(m, 0.3)
    if kind == "plane":
        m = 4096
        return np.stack([rng.uniform(-30, 30, m), np.zeros(m), rng.uniform(-30, 30, m)], 1), np.full(m, 0.2)
    if kind == "clusters":
        m = 3000
        c = rng.normal(size=(m, 3))
        c[m // 2:] += 1e12
        return c, np.full(m, 0.1)
    if kind == "all_oversized":                       # more than half the radii are 0: every other sphere is oversized
        c, r = _uniform(600)
        r[:301] = 0.0
        return c, r
    if kind == "median_radius_0":
        c, r = _uniform(500)
        r[::2] = 0.0
        r[1:12:2] = 0.0
        r[1::4] = -r[1::4]
        return c, r
    if kind == "one_in_frame":
        m = 50
        c = np.full((m, 3), np.inf)
        c[1::3] = (1e16, 0.0, 0.0)
        c[2::3, 0] = np.nan
        c[17] = (0.5, 0.5, 0.5)
        return c, np.full(m, 0.4)
    if kind == "none_in_frame":
        m = 40
        c = np.full((m, 3), np.inf)
        c[1::4] = -np.inf
        c[::4, 1] = np.nan
        c[2::4] = (1e16, 0.0, 0.0)
        return c, np.full(m, 0.4)
    if kind == "upper_face":                          # a grid with a quarter of its centres on the box's upper x face
        g = np.arange(16, dtype=np.float64)
        x, y, z = np.meshgrid(g, g, g, indexing="ij")
        c = np.stack([x.ravel(), y.ravel(), z.ravel()], 1)
        c[c[:, 0] >= 12, 0] = 15.0
        return c, np.full(len(c), 0.3)
    raise ValueError(kind)


def oversize_pair():
    """One sphere with |r| exactly OVERSIZE * median |r| (not oversized) and one just above it (oversized)."""
    c, r = _uniform(301, seed=8)
    r[:] = 0.5
    r[7] = OVERSIZE * 0.5
    r[8] = -np.nextafter(OVERSIZE * 0.5, np.inf)
    return c, r


SIZES = ["n1", "n8", "n9", "n64", "n65", "n72", "n73", "n512", "n513", "n4096", "n4097"]
KINDS = SIZES + ["coincident", "exponential", "line", "plane", "clusters", "all_oversized", "median_radius_0",
                 "one_in_frame", "none_in_frame", "upper_face"]


@pytest.mark.parametrize("kind", KINDS)
def test_the_rebuilt_tree_keeps_the_depth_bound_and_the_carved_sizes(kind):
    c, r = _case(kind)
    t = filled(rebuild(c, r), c, r)
    n = len(r)
    check_tree(t, c, r)
    assert max(t["level_count"], default=0) <= n // (K + 1) + 1 and t["depth"] <= MAX_DEPTH
    if kind == "one_in_frame":
        assert (t["n_nodes"], t["n_leaves"], t["depth"], t["leaf_id"][0, 0]) == (1, 1, 1, 17) and len(t["always"]) == n - 1
    if kind == "none_in_frame":
        assert t["n_nodes"] == 0 and t["n_leaves"] == 0 and t["depth"] == 0 and len(t["always"]) == n
    if kind in ("all_oversized", "median_radius_0"):
        g, r_big, _, keys = sort_keys(c, r)
        assert r_big == 0.0 and np.count_nonzero(keys >> np.uint64(63)) == np.count_nonzero(r)
    if kind == "upper_face":
        _, _, _, keys = sort_keys(c, r)
        x_bits = np.uint64(0o4444444444 << 26)
        assert np.count_nonzero((keys & x_bits) == x_bits) == 1024   # t = 1024 on the x face is clamped to cell 1023


def test_the_oversize_threshold_is_strict():
    c, r = oversize_pair()
    _, r_big, _, keys = sort_keys(c, r)
    big = {int(k & np.uint64((1 << 26) - 1)) for k in keys if k >> np.uint64(63)}
    assert r_big == OVERSIZE * 0.5 and big == {8}
    _, _, _, keys = sort_keys(c, r, oversize=0.0)                     # RTB200_REBUILD_OVERSIZE=0: nothing is oversized
    assert not np.any(keys >> np.uint64(63))
    check_tree(filled(rebuild(c, r), c, r), c, r)


@pytest.mark.parametrize("n", sorted(DEEP))
def test_deep_constructions_reach_their_depth(n):
    c, r = deep_spheres(n)
    t = rebuild(c, r)
    assert t["depth"] == DEEP[n], t["level_count"]
    assert t["level_count"][:MORTON_LEVELS] == [1] * MORTON_LEVELS                # one node per Morton level: the rest are leaves
    assert max(t["level_count"]) <= n // (K + 1) + 1 and t["n_leaves"] <= n and t["n_nodes"] <= n
    if n <= 32_768:
        check_tree(filled(t, c, r), c, r)


LEAF_SIZES = [2, 6, 8, 16, 32]   # RT_LEAF_K of the default build (8) and of the stress builds
# depth of the rebuilt tree of deep_spheres(n) at each leaf size: below leaves of 8 the peeled octants split further; from
# leaves of 16 up the 8 spheres of a peeled octant fit one leaf and the last cell needs fewer levels
DEEP_AT = {2: {4_096: 14, 32_768: 15, 262_144: 16}, 6: {4_096: 14, 32_768: 15, 262_144: 16},
           8: {4_096: 13, 32_768: 14, 262_144: 15}, 16: {4_096: 8, 32_768: 9, 262_144: 10},
           32: {4_096: 7, 32_768: 8, 262_144: 9}}


def _edge_case(kind, k):
    if kind == "n_k":
        return _uniform(k)
    if kind == "n_k_plus_1":
        return _uniform(k + 1)
    return _case(kind)


@pytest.mark.parametrize("kind", ["n_k", "n_k_plus_1", "coincident", "exponential", "line"])
@pytest.mark.parametrize("k", LEAF_SIZES)
def test_the_rebuilt_tree_at_every_leaf_size(k, kind):
    c, r = _edge_case(kind, k)
    t = filled(rebuild(c, r, leaf_size=k), c, r)
    n = len(r)
    check_tree(t, c, r, leaf_size=k)
    assert t["leaf_size"] == k and t["leaf_id"].shape == (t["n_leaves"], k)
    assert max(t["level_count"]) <= n // (k + 1) + 1 and t["depth"] <= MAX_DEPTH
    if kind == "n_k":          # one leaf under the root holds them all
        assert (t["n_nodes"], t["n_leaves"], t["depth"]) == (1, 1, 1)
    if kind == "n_k_plus_1":   # the root splits them
        assert t["n_nodes"] == 1 and t["n_leaves"] >= 2
    if kind != "coincident":
        assert sound(t, c, r, 40, [13.0, 2.0, 3.0] if kind[0] == "n" else [0.3, 2.0, 6.0]) > 0


def test_the_rebuild_fills_the_coincident_leaves_of_32():
    """10,000 coincident spheres rebuild into leaves of 32 that are all full but the remainder of 16 (and, in the
    build-invariance case coincident_10k_rebuilt, the light's own leaf): a ray through them makes one leaf step yield 32
    candidates, which fills RT_CAP_CD = 32 of the smallest lists exactly."""
    c = np.tile([[0.0, 0.5, 0.0]], (10_000, 1))
    r = np.full(10_000, 0.5)
    for light, leaves, fills in ((False, 313, [16] + [32] * 312), (True, 314, [1, 16] + [32] * 312)):
        if light:
            c, r = np.concatenate([c, [[2.0, 3.0, 0.0]]]), np.concatenate([r, [0.7]])
        t = rebuild(c, r, leaf_size=32)
        fill = (t["leaf_id"] != 0xFFFFFFFF).sum(axis=1)
        assert t["n_leaves"] == leaves and sorted(fill.tolist()) == fills, (t["n_leaves"], np.bincount(fill))


@pytest.mark.parametrize("n", [4_096, 32_768, 262_144])
@pytest.mark.parametrize("k", LEAF_SIZES)
def test_deep_constructions_at_every_leaf_size(k, n):
    c, r = deep_spheres(n)
    t = rebuild(c, r, leaf_size=k)
    assert t["depth"] == DEEP_AT[k][n], t["level_count"]
    assert max(t["level_count"]) <= n // (k + 1) + 1 and t["n_leaves"] <= n and t["n_nodes"] <= n
    if n == 4_096:
        check_tree(filled(t, c, r), c, r, leaf_size=k)


def _drift(c, r, rng, scale):
    moved = c + rng.normal(size=c.shape) * np.array([scale, 0.0, scale]) * (np.abs(r) < 100)[:, None]
    moved[:, 1] += np.abs(rng.normal(size=len(r))) * scale * 0.3 * (np.abs(r) < 100)
    return moved


@pytest.mark.parametrize("what", ["cover", "c4_10k", "deep_4096", "deep_32768"])
def test_traversal_of_the_rebuilt_tree_never_drops_a_sphere_the_exact_test_accepts(what):
    rng = np.random.default_rng(17)
    if what == "cover":
        sc = scenes.cover_scene(64, 48, 1)
        c, r = _spheres(sc)
        c = _drift(c, r, rng, 1.5)
        c[0] = (0.5, -1000.2, -0.3)                        # the ground moves too
        cam, rays = [13.0, 2.0, 3.0], 300
    elif what == "c4_10k":
        sc = R.Scene.from_config(scenes._variant(scenes.rtiow_config(50), 32, 24, 1, 4))
        c, r = _spheres(sc)
        c = _drift(c, r, rng, 0.6)
        cam, rays = [13.0, 2.0, 3.0], 150
    else:
        c, r = deep_spheres(int(what.split("_")[1]))
        cam, rays = [1.6, 0.4, 1.1], 60
    t = filled(rebuild(c, r), c, r)
    check_tree(t, c, r)
    assert sound(t, c, r, rays, cam) > rays


def _scene(c, r):
    objs = [{"center": _v(*map(float, p)), "radius": float(q), "material": {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}}
            for p, q in zip(c, r)]
    return R.Scene.from_config(base_config(8, 6, 1, 2, objs))


def mixed_zero_centres():
    """Centres whose median x (element n/2 in cub's order, where -0.0 and +0.0 rank equal and keep their order) is a zero
    of either sign, depending on the order of the zeros in the scene list."""
    rng = np.random.default_rng(4)
    m = 41
    c = rng.uniform(1, 3, (m, 3))
    c[:15, 0] = -c[:15, 0]
    c[15:27, 0] = np.where(np.arange(12) % 3 == 0, -0.0, 0.0)
    c[:, 2] = np.where(np.arange(m) % 2 == 0, 0.0, -0.0)             # the median z is a zero too
    return c, np.full(m, 0.3)


def test_the_host_builder_chooses_the_rebuilds_recentring_offset():
    """The host's recentring offset is the rebuild's bit for bit, also when the median of a column is a zero of mixed
    sign; the always-list is the rebuild's too."""
    c, r = mixed_zero_centres()
    for perm in (np.arange(len(r)), np.random.default_rng(5).permutation(len(r)), np.arange(len(r))[::-1]):
        g, _, always, _ = sort_keys(c[perm], r[perm])
        host = R.bvh_records(_scene(c[perm], r[perm]))
        assert host["recentre"].view(np.uint64).tolist() == g.view(np.uint64).tolist(), (host["recentre"], g)
        assert np.array_equal(host["always"], always)
