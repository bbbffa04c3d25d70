"""The closest-hit and occlusion queries where the margins of the f32 frame are tight (DESIGN.md §4.2, §4.11), held bit for bit
to the oracle's hit_world: scenes spread to 1e4 … 4e14 from the recentre, a sphere of radius 1e14, spheres one ulp either
side of the always-list threshold, and rays tangent to far spheres, in the planes of the boxes, with |d| scaled by 2^±49,
with s and oo a few f32 ulps either side of the flag test's thresholds, with direction components either side of the 1e-20
clamp, f32-subnormal or -0, and occlusion bounds at the roots ± 1 ulp (tests/f32_frame_cases.py). Every variant, on the
handle as uploaded, after rebuild(), after update_spheres moves an outer cluster from X to 2X (the GPU refit), and staged in
shared memory; one trace_rays check per spread scene; the stress builds. Each case asserts that it reaches its edge."""
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import f32_frame_cases as F
import intersect_rays as IR
import rtb200 as R
from test_gpu_intersect import AUTO, BRUTE, EXACT, FILTERED, REPO, STRESS, query
from test_gpu_occlusion import assert_occluded_equal, occluded
from test_gpu_trace_rays import check as check_trace

pytestmark = pytest.mark.gpu
VARIANTS = {"filtered": FILTERED, "brute_force": BRUTE, "exact_f64": EXACT, "auto": AUTO}
N_CLUSTER = 22                       # spheres per cluster of a spread scene (20 drawn, a coincident and a negative copy)
GRAZING_SHARE, BOX_FACE_SHARE = 0.5, 0.35   # least share of groups whose target is hit by some siblings and missed by others


def _outer(factor):
    """Move the +X cluster of a spread scene to factor * X: the indices and the records of update_spheres."""
    def move(sc):
        idx = list(range(N_CLUSTER, 2 * N_CLUSTER))
        recs = []
        for i in idx:
            s = sc._spheres[i]
            recs.append(sc.set_sphere(i, center=[s.center.x * factor, s.center.y * factor, s.center.z * factor]))
        return idx, recs
    return move


def states(name):
    out = ["uploaded", "rebuilt", "staged"]
    if name.startswith("spread_"):
        out.append("moved_2x")
        if name == "spread_4e14":
            out.append("moved_out")   # 3.2 X: the largest coordinate passes 1e15, the refit gives the cluster infinite boxes
    return out


def handle(name, state, variant, monkeypatch):
    """(Scene, ResidentScene, records of the handle) of scene `name` in `state` under `variant`."""
    sc = F.SCENES[name]()
    if state == "staged":
        monkeypatch.setenv("RTB200_WF_SMEM", "7")
    rs = R.ResidentScene(sc, R.make_options(variant=variant))
    monkeypatch.delenv("RTB200_WF_SMEM", raising=False)
    if state == "staged":
        assert rs.kernel_info()["smem_mask"] == 7
    elif state == "rebuilt":
        rs.rebuild()
    elif state.startswith("moved"):
        idx, recs = _outer(2.0 if state == "moved_2x" else 3.2)(sc)
        rs.update_spheres(idx, recs)
    recs = rs.bvh_records() if state in ("rebuilt", "moved_2x", "moved_out") else R.bvh_records(sc)
    return sc, rs, recs


def bounds_of(un, rng):
    """Per-ray bounds drawn from F.edge_bounds, and the two bounds every ray is also run under: its root and the next f64."""
    e = F.edge_bounds(un)
    mix = np.stack(e, axis=1)[np.arange(len(e[0])), rng.integers(0, len(e), size=len(e[0]))].copy()
    return mix, e[0], e[1]


def check_state(rs, sc, recs, what, seed):
    """Every family on the handle: intersect unbounded and under bounds, occluded under the same bounds (against the oracle
    and against intersect's sphere != -1), and shadow segments between the scene's spheres. Returns the oracle's answers."""
    fams = F.families(sc, recs, seed)
    o, d, names = F.concat(fams)
    un = IR.oracle(sc, o, d)
    IR.assert_hits_equal(query(rs, o, d), un, what + "/unbounded")
    rng = np.random.default_rng(seed)
    mix, at_root, above = bounds_of(un, rng)
    for tag, t in (("mixed bounds", mix), ("t_max = root", at_root), ("t_max = next(root)", above)):
        want = IR.oracle(sc, o, d, t) if tag == "mixed bounds" else IR.filtered(un, t)
        hits = query(rs, o, d, t)
        IR.assert_hits_equal(hits, want, f"{what}/{tag}")
        w = (want["sphere"] >= 0).astype(np.uint8)
        assert_occluded_equal(occluded(rs, o, d, t), w, f"{what}/{tag}/occluded")
        assert_occluded_equal((hits["sphere"] != -1).astype(np.uint8), w, f"{what}/{tag}/intersect under the bound")
    so, sd, st = F.segments(sc, rng)
    ws = (IR.oracle(sc, so, sd, st)["sphere"] >= 0).astype(np.uint8)
    assert_occluded_equal(occluded(rs, so, sd, st), ws, what + "/segments")
    assert 0 < ws.sum() < len(ws), (what, int(ws.sum()))
    # bounds reach: the root itself is rejected and the next double accepts it, on every ray that hits
    hit = un["sphere"] >= 0
    assert hit.mean() > 0.3 and ((IR.filtered(un, at_root)["sphere"] >= 0) != (IR.filtered(un, above)["sphere"] >= 0))[hit].all()
    return fams, un, names


@pytest.mark.parametrize("name", list(F.SCENES))
def test_queries_match_hit_world_where_the_f32_margins_are_tight(name, monkeypatch):
    for state in states(name):
        for vname, v in VARIANTS.items():
            sc, rs, recs = handle(name, state, v, monkeypatch)
            try:
                fams, un, names = check_state(rs, sc, recs, f"{name}/{state}/{vname}", seed=zlib.crc32(f"{name}/{state}".encode()))
                if vname == "filtered":
                    _reach(rs, sc, recs, fams, un, names, f"{name}/{state}")
            finally:
                rs.release()


def _reach(rs, sc, recs, fams, un, names, what):
    """Each family reaches its edge: grazing and box-face groups flip between hit and miss of their target, and the rays on
    either side of the flag test's thresholds take the tree (few candidates) or the f64 path (every sphere), counted by the
    host form."""
    n = sc.n_spheres
    for fam, share in (("grazing_far", GRAZING_SHARE), ("box_face", BOX_FACE_SHARE)):
        m = names == fam
        got, groups = F.flip_share(un["sphere"][m] == fams[fam]["target"], fams[fam]["group"])
        assert groups >= 20 and got >= share, (what, fam, got, groups)
    side = np.concatenate([f["side"] for f in fams.values()])
    o, d, _ = F.concat(fams)
    for s in (1, -1):
        sel = np.flatnonzero(side == s)
        assert len(sel) >= 90, (what, s, len(sel))
        st = rs.intersect(np.ascontiguousarray(o[sel]), np.ascontiguousarray(d[sel]))["stats"]
        assert st["rays"] == len(sel)
        if s == 1:
            assert st["candidates"] < 0.5 * n * len(sel), (what, st["candidates"], n, len(sel))
        else:
            assert st["candidates"] >= n * len(sel), (what, st["candidates"], n, len(sel))
    if what.startswith("threshold"):
        ids, out = F.threshold_ids()
        always = set(recs["always"].tolist())
        assert [int(i) in always for i in ids] == out.tolist(), (what, sorted(always))
    if what.endswith("moved_out"):   # the refit cannot move spheres to the always-list; their boxes become infinite instead
        assert (recs["lo"] == -np.inf).any() and (recs["hi"] == np.inf).any()


@pytest.mark.parametrize("x", F.SPREAD)
def test_trace_rays_on_spread_scenes(x):
    """trace_rays (3 samples, depth 8) from the grazing and box-face rays of a spread scene: secondary rays, lights and the
    source-sphere certificate at large |c|."""
    sc = F.spread_scene(x)
    fams = F.families(sc, R.bvh_records(sc), 5)
    o = np.concatenate([fams[k]["o"] for k in ("grazing_far", "box_face")])
    d = np.concatenate([fams[k]["d"] for k in ("grazing_far", "box_face")])
    for vname in ("filtered", "brute_force"):
        rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[vname]))
        try:
            want = check_trace(rs, sc, o, d, f"{F.spread_name(x)}/{vname}", samples=3, max_depth=8)
        finally:
            rs.release()
    assert want["rays"] > 1.5 * 3 * len(o), want["rays"]   # paths go on past their first hit


def test_stress_builds_answer_the_f32_frame_cases_exactly(tmp_path):
    """Every stress build answers spread_1e12, threshold and the box-face rays, as uploaded and after rebuild(), like the oracle:
    the leaf sizes 2, 6, 16 and 32 change every leaf box."""
    import f32_frame_worker as FW
    from test_gpu_build_invariance import constants
    manifest = json.load(open(os.path.join(STRESS, "manifest.json")))
    for build in manifest:
        out = tmp_path / f"{build}.npz"
        env = dict(os.environ, RTB200_LIB=os.path.join(STRESS, f"librtb200_{build}.so"))
        subprocess.run([sys.executable, os.path.join(REPO, "tests", "f32_frame_worker.py"), str(out)], env=env, check=True, timeout=900)
        z = np.load(out, allow_pickle=False)
        meta = json.loads(str(z["meta"]))
        assert meta["leaf_size"] == constants(manifest[build])["RT_LEAF_K"]
        for key in FW.KEYS:
            o, d = z[f"{key}.o"], z[f"{key}.d"]
            sc = F.SCENES[key.split("/")[0]]()
            want = IR.oracle(sc, o, d)
            IR.assert_hits_equal({k: z[f"{key}.{k}"] for k in IR.FIELDS}, want, f"{build}/{key}")
            assert (want["sphere"] >= 0).sum() > 500, (build, key)
