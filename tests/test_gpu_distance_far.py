"""The point queries where their pruning is tight (DESIGN.md §3, §4.19), held bit for bit to the numpy restatement
(tests/distance_restatement.py): the scenes of tests/f32_frame_cases.py (spread to 4e14, a sphere of radius 1e14, the
always-list threshold) in every handle state (uploaded, rebuilt, staged, refit after a cluster moves to 2X and 3.2X) and
every variant, on the families of tests/distance_far_cases.py (box faces in the f32 frame, near-ties across subtrees at far
points, both sides of the oo test) under bounds at D~'s edges; exact ties across leaves in both index orders and with the
always-list; points inside overlapping spheres of two children; and the deepest trees. On each handle the float32
emulation checks the soundness lemma against the records the handle holds, and the host form's counters show each family's
reach."""
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import distance_far_cases as D
import distance_restatement as DR
import f32_frame_cases as F
import intersect_rays as IR
import rtb200 as R
from test_distance_cpu import _subtrees, emulate
from test_distance_far_cpu import _far_points
from test_gpu_distance import assert_nearest_equal, assert_overlaps_equal, check
from test_gpu_f32_frame import N_CLUSTER, VARIANTS, handle, states
from test_gpu_intersect import FILTERED, REPO, STRESS
from test_rebuild_restatement_cpu import deep_spheres

pytestmark = pytest.mark.gpu
INF = float("inf")


def check_points(rs, sc, p, what):
    """Both kinds, device form, unbounded and under every bound of D.edge_bounds (overlaps under |bound|)."""
    s, d = check(rs, sc, p, what + "/unbounded")
    for bname, b in D.edge_bounds(d).items():
        check(rs, sc, p, f"{what}/bound {bname}", b, radii=np.abs(b))
    return s, d


def host_form(rs, sc, p, what):
    """The host forms against the restatement; returns nearest's counters."""
    c, r = DR.sphere_arrays(sc)
    h = rs.nearest(p)
    assert_nearest_equal((h["sphere"], h["distance"]), DR.nearest(p, c, r), what + "/host form")
    rad = np.abs(np.random.default_rng(len(p)).normal(size=len(p)))
    assert_overlaps_equal(rs.overlaps(p, rad)["overlaps"], DR.overlaps(p, rad, c, r), what + "/host form overlaps")
    return h["stats"]


def lemma(recs, sc, p, what, k=24):
    """The emulation on k points against the handle's own records: L~ <= dist_j under every child it bounds, and the
    restatement's answer."""
    c, r = IR.spheres_of(sc)
    under = _subtrees(recs)
    pick = np.random.default_rng(k).choice(len(p), size=min(k, len(p)), replace=False)
    ws, wd = DR.nearest(p[pick], c, r)
    d = DR.distances(p[pick], c, r)
    for t, i in enumerate(pick):
        got = emulate(recs, c, r, p[i], INF, False, under=under, d_all=d[t])
        assert (got[0], got[1]) == (ws[t], wd[t]), (what, p[i])


@pytest.mark.parametrize("name", list(F.SCENES))
def test_point_queries_where_the_f32_margins_are_tight(name, monkeypatch):
    for state in states(name):
        fams = None
        for vname, v in VARIANTS.items():   # FILTERED first: its handle holds the hierarchy the families aim at
            sc, rs, recs = handle(name, state, v, monkeypatch)
            what = f"{name}/{state}/{vname}"
            try:
                if fams is None:
                    assert vname == "filtered"
                    if state != "uploaded":
                        recs = rs.bvh_records()
                    fams = D.families(sc, recs, zlib.crc32(f"{name}/{state}".encode()))
                    p, names = D.concat(fams)
                    if state.startswith("moved"):   # next to the moved cluster's spheres
                        c, r = IR.spheres_of(sc)
                        m = np.arange(N_CLUSTER, 2 * N_CLUSTER)
                        u = np.random.default_rng(3).normal(size=(len(m), 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
                        p = np.concatenate([p, c[m] + u * (np.abs(r[m]) * 1.01)[:, None], c[m] + u * (np.abs(r[m]) * 0.5)[:, None]])
                check_points(rs, sc, p, what)
                if vname == "filtered":
                    _reach(rs, sc, recs, fams, what)
                    if state != "uploaded":
                        lemma(recs, sc, p, what)
            finally:
                rs.release()


def _reach(rs, sc, recs, fams, what):
    """The host form on each side of the oo test: the tree side visits nodes, the scan side evaluates every sphere and visits
    none; the threshold scene's always-list; the infinite boxes of the refit past 1e15."""
    n = sc.n_spheres
    fo = fams["oo_side"]
    for s in (1, -1):
        p = np.ascontiguousarray(fo["p"][fo["side"] == s])
        assert len(p) >= 100, (what, s, len(p))
        st = host_form(rs, sc, p, f"{what}/oo side {s}")
        assert st["rays"] == len(p)
        if s == 1:   # so far out every sphere of a small scene may be evaluated: the nodes tell the tree
            assert st["nodes"] >= len(p), (what, st)
        else:
            assert st["nodes"] == 0 and st["candidates"] == n * len(p), (what, st)
    host_form(rs, sc, np.ascontiguousarray(D.concat(fams)[0]), what)
    if what.startswith("threshold"):
        ids, out = F.threshold_ids()
        always = set(recs["always"].tolist())
        assert [int(i) in always for i in ids] == out.tolist(), (what, sorted(always))
    if "moved_out" in what:
        assert (recs["lo"] == -np.inf).any() and (recs["hi"] == np.inf).any()


@pytest.mark.parametrize("state", ["uploaded", "rebuilt", "staged"])
def test_exact_ties_across_leaves(state, monkeypatch):
    """The lowest index among equal distances, with the members in different leaves, in both visit orders, and with one member
    on the always-list; and the tie points moved one ulp."""
    sc, ties = D.ties_scene()
    c, r = IR.spheres_of(sc)
    pts = D.tie_points(ties)
    for vname, v in VARIANTS.items():
        if state == "staged":
            monkeypatch.setenv("RTB200_WF_SMEM", "7")
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        monkeypatch.delenv("RTB200_WF_SMEM", raising=False)
        try:
            if state == "rebuilt":
                rs.rebuild()
            s, d = check_points(rs, sc, pts["p"], f"ties/{state}/{vname}")
            at = pts["tie"] >= 0
            assert np.array_equal(s[at], [ties[t]["members"][0] for t in pts["tie"][at]])
            if vname == "filtered":
                recs = rs.bvh_records()
                for x in ties:
                    leaves = [D.leaf_of(recs, j) for j in x["members"]]
                    assert leaves[0] != leaves[1] and leaves.count(-1) == (x["always"] >= 0), (state, x, leaves)
                host_form(rs, sc, pts["p"], f"ties/{state}")
                lemma(recs, sc, pts["p"], f"ties/{state}")
        finally:
            rs.release()


def test_inside_overlapping_spheres_of_two_children():
    sc = D.nested_scene()
    for state in ("uploaded", "rebuilt"):
        fam = None
        for vname, v in VARIANTS.items():   # FILTERED first: its handle holds the hierarchy the family aims at
            rs = R.ResidentScene(sc, R.make_options(variant=v))
            try:
                if state == "rebuilt":
                    rs.rebuild()
                if fam is None:
                    fam = D.inside(sc, rs.bvh_records(), np.random.default_rng(5), 60)
                    assert len(fam["p"]) >= 30, (state, len(fam["p"]))
                s, d = check_points(rs, sc, fam["p"], f"nested/{state}/{vname}")
                assert (d < 0).all()
            finally:
                rs.release()


@pytest.mark.parametrize("build", ["rebuild", "host_breadth_first"])
def test_the_deepest_trees(build, monkeypatch):
    """deep_spheres(4096) rebuilt on the GPU, and host-built with the breadth-first collapse from the root, from points far from
    everything: the restatement's answers, and the host form returns (the traversal guard never trips)."""
    c, r = deep_spheres(4096)
    sc = IR.scene_of([IR.sphere(c[i], r[i]) for i in range(len(r))])[0]
    p = np.concatenate([_far_points(c, 4096, 3), _far_points(c, 24, 3)])
    if build == "host_breadth_first":
        monkeypatch.setenv("RTB200_BVH_AREA_LEVELS", "1")
    rs = R.ResidentScene(sc, R.make_options(variant=FILTERED))
    monkeypatch.delenv("RTB200_BVH_AREA_LEVELS", raising=False)
    try:
        if build == "rebuild":
            rs.rebuild()
        check(rs, sc, p, f"deep/{build}")
        st = host_form(rs, sc, p, f"deep/{build}")
        assert st["nodes"] >= len(p) and rs.bvh_records()["depth"] >= (13 if build == "rebuild" else 6)
    finally:
        rs.release()


def test_stress_builds_answer_the_far_cases_exactly(tmp_path):
    """Every stress build (leaves of 2, 6, 16 and 32 move every leaf boundary) answers spread_1e12, threshold and the ties, as
    uploaded and after rebuild(), like the restatement."""
    import distance_far_worker as W
    manifest = json.load(open(os.path.join(STRESS, "manifest.json")))
    want = {}
    for key, sc, p, rad in W.cases():
        c, r = DR.sphere_arrays(sc)
        want[key] = (DR.nearest(p, c, r), DR.overlaps(p, rad, c, r))
    for build in manifest:
        out = tmp_path / f"{build}.npz"
        env = dict(os.environ, RTB200_LIB=os.path.join(STRESS, f"librtb200_{build}.so"))
        subprocess.run([sys.executable, "-B", os.path.join(REPO, "tests", "distance_far_worker.py"), str(out)], env=env, check=True, timeout=900)
        z = np.load(out)
        for key, (nw, ov) in want.items():
            for state in ("uploaded", "rebuilt"):
                assert_nearest_equal((z[f"{key}/{state}.sphere"], z[f"{key}/{state}.distance"]), nw, f"{build}/{key}/{state}")
                assert_overlaps_equal(z[f"{key}/{state}.overlaps"], ov, f"{build}/{key}/{state} overlaps")
