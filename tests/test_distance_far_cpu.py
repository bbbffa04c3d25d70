"""The point queries' pruning at the margins of the f32 frame (DESIGN.md §3, §4.19) without a GPU: the families of
tests/distance_far_cases.py are deterministic and reach their edges, the exact ties are certified and sit in different leaves
of every build, and the float32 emulation of tests/test_distance_cpu.py holds the soundness lemma (L~ <= dist_j for every
sphere under every child it bounds) and the restatement's answers on the scenes of tests/f32_frame_cases.py (out to 4e14),
on the host build and on the rebuild restatement. The deepest trees measure the traversal stack."""
import numpy as np
import pytest

import distance_far_cases as D
import distance_restatement as DR
import f32_frame_cases as F
import intersect_rays as IR
import rtb200 as R
from f32_frame_cases import _child_members
from rebuild_restatement import filled, rebuild
from test_distance_cpu import _subtrees, emulate
from test_rebuild_restatement_cpu import deep_spheres

INF = float("inf")
STACK = 7 * 21 + 1            # kDistStack
LEAF_SIZES = (2, 6, 8, 16, 32)
DEEPEST_STACK = 94            # the most entries the emulated traversal held on the deepest trees (below)


def _rebuilt(sc, k=8):
    c, r = IR.spheres_of(sc)
    return filled(rebuild(c, r, leaf_size=k), c, r)


def test_the_generators_are_deterministic():
    sc = F.SCENES[F.spread_name(1e12)]()
    recs = R.bvh_records(sc)
    a, b = D.families(sc, recs, 5), D.families(sc, recs, 5)
    for name in a:
        for key in a[name]:
            assert np.array_equal(a[name][key], b[name][key]), (name, key)
    s1, t1 = D.ties_scene()
    s2, t2 = D.ties_scene()
    assert np.array_equal(IR.spheres_of(s1)[1], IR.spheres_of(s2)[1]) and all(np.array_equal(x["p"], y["p"]) for x, y in zip(t1, t2))


def reach(sc, recs, fams):
    """Each family's reach on hierarchy `recs`; returns the counts it saw."""
    c, r = IR.spheres_of(sc)
    g = recs["recentre"]
    fb = fams["box_face"]
    apart, sign = D.face_offsets(fb, recs)
    on = fb["sub"] == 0
    assert np.array_equal(apart[on], fb["ulps"][on]), "box_face: pf is not the stored plane + ulps"
    assert (apart[~on] == 0).all() and np.array_equal(sign[~on], np.sign(fb["sub"][~on])), "box_face: f64 off the plane, f32 on it"
    ft = fams["near_tie"]
    d = DR.distances(ft["p"], c, r)
    gaps = 0
    for t, (i, j) in enumerate(ft["pair"]):
        node = ft["node"][t]
        kids = [k for k in range(8) if int(recs["child"][node][k]) != D.EMPTY]
        home = [k for k in kids if i in _child_members(recs, node, k) or j in _child_members(recs, node, k)]
        assert len(home) == 2, ("near_tie: members under one child", i, j, node)
        q = np.linalg.norm(ft["p"][t] - g)
        gap = abs(d[t, i] - d[t, j])
        assert gap <= D.NEAR_TIE_ULPS * np.spacing(max(abs(d[t, i]), abs(d[t, j]))) and gap < D.U32 * q
        assert np.linalg.norm(ft["p"][t] - (c[i] + c[j]) / 2) >= 10 * (np.linalg.norm(c[i] - c[j]) + abs(r[i]) + abs(r[j])) * 0.99
        assert np.sort(d[t])[1] == max(d[t, i], d[t, j]), "near_tie: the pair is not the two nearest"
        gaps += gap > 0
    fi = fams["inside"]
    if len(fi["p"]):
        d = DR.distances(fi["p"], c, r)
        ans = DR.nearest(fi["p"], c, r)[0]
        for t, (node, k1, k2) in enumerate(fi["where"]):
            assert D.inside_ok(recs, c, r, fi["p"][t], d[t], ans[t], node, k1, k2)
    fo = fams["oo_side"]
    ulps = D.oo_certified(fo, g)
    assert np.array_equal(np.where(ulps < 0, 1, -1), fo["side"]) and np.abs(ulps).max() <= 40
    return {"box_face": len(fb["p"]), "near_tie": len(ft["p"]), "near_tie_gaps": gaps, "inside": len(fi["p"]),
            "oo_below": int((fo["side"] == 1).sum()), "oo_above": int((fo["side"] == -1).sum()), "oo_at": int((ulps == 0).sum())}


@pytest.mark.parametrize("name", list(F.SCENES))
def test_each_family_reaches_its_edge(name):
    sc = F.SCENES[name]()
    for recs in (R.bvh_records(sc), _rebuilt(sc)):
        n = reach(sc, recs, D.families(sc, recs, 11))
        assert n["box_face"] >= 300 and n["oo_below"] >= 100 and n["oo_above"] >= 100, (name, n)
        if name.startswith("spread"):   # elsewhere a sphere of radius 1e14 or more is the nearest to every far point
            assert n["near_tie"] >= 40 and n["near_tie_gaps"] >= 5, (name, n)


def test_the_inside_family_reaches_its_edge():
    """The spheres of the f32-frame scenes that overlap under different children hold no point deeper in the later slot;
    the nested scene does, on both builds."""
    sc = D.nested_scene()
    for recs in (R.bvh_records(sc), _rebuilt(sc)):
        n = reach(sc, recs, D.families(sc, recs, 11))
        assert n["inside"] >= 30, n


def _visit_order(recs, c, r, x):
    """Whether the lower-index member of tie x is evaluated first by the emulated nearest query."""
    p = x["p"]
    _, _, evald, _ = emulate(recs, c, r, p, INF, False, d_all=DR.distances(p[None], c, r)[0])
    lo, hi = x["members"]
    assert lo in evald and hi in evald, (x, evald)
    return evald.index(lo) < evald.index(hi)


def test_ties_are_exact_across_leaves_in_both_orders():
    sc, ties = D.ties_scene()
    c, r = IR.spheres_of(sc)
    assert D.tie_certified(ties, c, r)
    host = R.bvh_records(sc)
    builds = {"host": host, **{f"rebuild_{k}": filled(rebuild(c, r, leaf_size=k), c, r) for k in LEAF_SIZES}}
    pts = D.tie_points(ties)
    for bname, recs in builds.items():
        always = set(recs["always"].tolist())
        orders = set()
        for x in ties:
            leaves = [D.leaf_of(recs, j) for j in x["members"]]
            if x["always"] >= 0:
                assert x["always"] in always and leaves.count(-1) == 1, (bname, x)
                orders.add(x["members"][0] == x["always"])          # the always-list is evaluated first
            else:
                assert -1 not in leaves and leaves[0] != leaves[1], (bname, x, leaves)
                orders.add(_visit_order(recs, c, r, x))
            s, dist = DR.nearest(x["p"][None], c, r)
            assert s[0] == x["members"][0] and dist[0] == x["dist"]
        assert orders == {True, False}, (bname, orders)
        for i, p in enumerate(pts["p"]):
            d_all = DR.distances(p[None], c, r)[0]
            got = emulate(recs, c, r, p, INF, False, d_all=d_all)
            want = DR.nearest(p[None], c, r)
            assert (got[0], got[1]) == (want[0][0], want[1][0]), (bname, p, got[:2], want)


def _bounds_of(d, rng):
    e = D.edge_bounds(d)
    names = list(e)
    pick = rng.integers(0, len(names), size=len(d))
    return [e["at"], e["above"], e["below"], np.array([e[names[q]][i] for i, q in enumerate(pick)])]


@pytest.mark.parametrize("name", list(F.SCENES))
def test_the_lemma_and_the_answers_hold_on_the_far_scenes(name):
    """The emulated traversal on every family, on the host build and the rebuild restatement: L~ <= dist_j under every child it
    bounds, the restatement's nearest unbounded and under the bounds of D.edge_bounds, and overlaps under the same radii."""
    sc = F.SCENES[name]()
    c, r = IR.spheres_of(sc)
    rng = np.random.default_rng(12)
    checked = 0
    for recs in (R.bvh_records(sc), _rebuilt(sc)):
        under = _subtrees(recs)
        p, names = D.concat(D.families(sc, recs, 13, small=True))
        sel = np.concatenate([rng.permutation(np.flatnonzero(names == n))[:12] for n in np.unique(names)])
        p = p[sel]
        d_pts = DR.distances(p, c, r)
        ws, wd = DR.nearest(p, c, r)
        for bi, b in enumerate(_bounds_of(wd, rng)):
            bs, bd = DR.nearest(p, c, r, b)
            ov = DR.overlaps(p, b, c, r)
            for i in range(len(p)):
                got = emulate(recs, c, r, p[i], float(b[i]), False, under=under if bi == 0 else None, d_all=d_pts[i])
                assert (got[0], got[1]) == (bs[i], bd[i]), (name, p[i], b[i], got[:2], bs[i], bd[i])
                assert (emulate(recs, c, r, p[i], float(b[i]), True, d_all=d_pts[i])[0] >= 0) == bool(ov[i])
        for i in range(len(p)):
            got = emulate(recs, c, r, p[i], INF, False, under=under, d_all=d_pts[i])
            assert (got[0], got[1]) == (ws[i], wd[i]), (name, p[i])
            checked += 1
    assert checked >= 40


def _far_points(c, k, seed):
    """k points 1e2 .. 1e6 times the centres' extent away from their box, in random directions."""
    rng = np.random.default_rng(seed)
    lo, hi = c.min(axis=0), c.max(axis=0)
    u = rng.normal(size=(k, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    return (lo + hi) / 2 + u * float(np.max(hi - lo) + 1.0) * 10.0 ** rng.uniform(2, 6, size=k)[:, None]


def _deepest(recs, c, r, pts):
    depth = 0
    for p in pts:
        info = {}
        got = emulate(recs, c, r, p, INF, False, d_all=DR.distances(p[None], c, r)[0], info=info)
        assert info["tree"] and got[0] == DR.nearest(p[None], c, r)[0][0]
        depth = max(depth, info["stack"])
    return depth


def test_the_traversal_stack_stays_within_its_reserve(monkeypatch):
    """Points far from everything: D~ = +inf down to the first leaf, so every child of the first descent is kept. The most
    entries the stack held, on deep_spheres(4096) rebuilt with leaves of 2 and 8 and host-built with the breadth-first collapse
    from the root (RTB200_BVH_AREA_LEVELS=1), stays within kDistStack = 148 and equals DEEPEST_STACK (DESIGN.md §4.19)."""
    c, r = deep_spheres(4096)
    seen = {}
    for k in (2, 8):
        recs = filled(rebuild(c, r, leaf_size=k), c, r)
        seen[f"rebuild_{k}"] = (_deepest(recs, c, r, _far_points(c, 24, 3)), recs["depth"])
    sc = IR.scene_of([IR.sphere(c[i], r[i]) for i in range(len(r))])[0]
    monkeypatch.setenv("RTB200_BVH_AREA_LEVELS", "1")
    recs = R.bvh_records(sc)
    monkeypatch.delenv("RTB200_BVH_AREA_LEVELS")
    seen["host_breadth_first"] = (_deepest(recs, c, r, _far_points(c, 24, 3)), recs["depth"])
    print("stack entries (most, tree depth):", seen)
    assert max(v[0] for v in seen.values()) <= STACK
    assert max(v[0] for v in seen.values()) == DEEPEST_STACK, seen
