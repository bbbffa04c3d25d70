"""Host side of the f32-frame cases (tests/f32_frame_cases.py, no GPU): the generators are deterministic, every case reaches the
edge it is meant for (the oracle's answer flips inside each grazing and box-face group, the emulated s and oo fall on both
sides of the flag test's thresholds, the box-face rays lie in the planes of the hierarchy, the threshold spheres are on or
off the always-list as intended), and the float32 emulations of the traversal (test_bvh_cpu._traverse, test_occlusion_cpu.
_bounded) never drop a sphere the exact test accepts on these scenes and families. When tests/test_gpu_f32_frame.py fails,
these localise the failure: a case the emulation also drops is a margin, one it keeps is the kernel."""
import numpy as np
import pytest

import f32_frame_cases as F
import intersect_rays as IR
import rtb200 as R
from test_bvh_cpu import _exact_hits, _traverse
from test_occlusion_cpu import _bounded, _roots, tcap

f32 = np.float32


def _fams(name, seed=1):
    sc = F.SCENES[name]()
    recs = R.bvh_records(sc)
    return sc, recs, F.families(sc, recs, seed)


def test_generators_are_deterministic():
    for name in ("spread_1e12", "threshold"):
        sc1, _, a = _fams(name)
        sc2, _, b = _fams(name)
        assert [s.tup() for s in (x.center for x in sc1._spheres[: sc1.n_spheres])] == \
               [s.tup() for s in (x.center for x in sc2._spheres[: sc2.n_spheres])]
        assert a.keys() == b.keys()
        for k in a:
            for f in ("o", "d", "group", "target", "side"):
                assert np.array_equal(a[k][f].view(np.uint64) if a[k][f].dtype == np.float64 else a[k][f],
                                      b[k][f].view(np.uint64) if b[k][f].dtype == np.float64 else b[k][f]), (name, k, f)
        _, _, c = _fams(name, seed=2)
        assert not np.array_equal(a["grazing_far"]["o"], c["grazing_far"]["o"])


@pytest.mark.parametrize("name", list(F.SCENES))
def test_grazing_and_box_face_groups_flip_between_hit_and_miss(name):
    sc, _, fams = _fams(name)
    for fam, share in (("grazing_far", 0.5), ("box_face", 0.35)):
        f = fams[fam]
        un = IR.oracle(sc, f["o"], f["d"])
        got, groups = F.flip_share(un["sphere"] == f["target"], f["group"])
        assert groups >= 20 and got >= share, (name, fam, got, groups)


@pytest.mark.parametrize("name", list(F.SCENES))
def test_s_and_oo_fall_on_both_sides_of_the_flag_thresholds(name):
    sc, recs, fams = _fams(name)
    g = recs["recentre"]
    o = np.concatenate([fams[k]["o"] for k in ("d_sweep", "o_sweep")])
    d = np.concatenate([fams[k]["d"] for k in ("d_sweep", "o_sweep")])
    side = np.concatenate([fams[k]["side"] for k in ("d_sweep", "o_sweep")])
    s, oo = F.f32_s(d), F.f32_oo(o, g)
    with np.errstate(over="ignore"):
        for v, thr in ((s, F.S_LO), (s, F.S_HI), (oo, F.OO_HI)):
            apart = F._ulps_apart(v, thr)
            assert ((apart >= 2) & (apart <= 13)).sum() >= 40 and ((apart <= -2) & (apart >= -13)).sum() >= 40, (name, float(thr))
    ok = (s > F.S_LO) & (s < F.S_HI) & (oo < F.OO_HI)
    assert np.array_equal(ok[side != 0], side[side != 0] > 0)
    assert (side > 0).sum() > 1000 and (side < 0).sum() > 90
    # the 2^k scaled directions reach both ends of [2^-49, 2^49]
    n = np.linalg.norm(fams["d_sweep"]["d"], axis=1)
    assert n.min() < 2.0 ** -48 and n.max() > 2.0 ** 48
    # component_edges: every kind of small component is present in d^ = f32(d)
    df = fams["component_edges"]["d"].astype(f32)
    above, below, sub1, sub2 = np.array([1e-20 * (1 + 2.0 ** -20), 1e-20 * (1 - 2.0 ** -20), 1e-40, 1e-45]).astype(f32)
    assert below < f32(1e-20) < above and sub1 < np.finfo(f32).tiny and sub2 > 0
    for v in (above, below, sub1, sub2):
        assert (df == v).any() and (df == -v).any(), v
    assert (np.signbit(df) & (df == 0)).any() and ((fams["component_edges"]["d"] != 0) & (df == 0)).any()


@pytest.mark.parametrize("name", ["spread_1e4", "spread_4e14", "huge", "threshold"])
def test_box_face_rays_lie_in_the_planes_of_the_hierarchy(name):
    sc, recs, fams = _fams(name)
    g = recs["recentre"]
    f = fams["box_face"]
    c, r = IR.spheres_of(sc)
    in_plane = 0
    for ax in range(3):
        planes = np.concatenate([recs["lo"][:, ax, :].ravel(), recs["hi"][:, ax, :].ravel()]).astype(np.float64)
        flat = f["d"][:, ax] == 0
        in_plane += int((flat & np.isin(f["o"][:, ax] - g[ax], planes[np.isfinite(planes)])).sum())
    assert in_plane >= 60, in_plane
    # the unshifted ray of every group touches its target: its distance from the centre is |r| to rounding
    grp = f["group"]
    first = np.array([np.flatnonzero(grp == k)[0] for k in np.unique(grp[grp >= 0])])
    sel = first + int(np.flatnonzero(F.K == 0)[0])
    assert (grp[sel] == grp[first]).all()
    t = f["target"][sel]
    oc = c[t] - f["o"][sel]
    dist = np.linalg.norm(oc - f["d"][sel] * np.sum(oc * f["d"][sel], axis=1, keepdims=True), axis=1)
    tol = 1e-9 * np.abs(r[t]) + 4 * np.spacing(np.abs(c[t]).max(axis=1) + np.abs(r[t]))
    assert (np.abs(dist - np.abs(r[t])) <= tol).all(), np.max(np.abs(dist - np.abs(r[t])) / tol)


def test_threshold_spheres_are_on_the_always_list_as_intended():
    sc = F.threshold_scene()
    b = R.bvh_records(sc)
    ids, out = F.threshold_ids()
    always = set(b["always"].tolist())
    assert [int(i) in always for i in ids] == out.tolist()
    assert out.any() and not out.all()
    c, r = IR.spheres_of(sc)
    m = np.abs(c[ids] - b["recentre"]).max(axis=1) + np.abs(r[ids])
    assert np.array_equal(m, np.array([F.LIMIT + u * F.STEP for _, _, _, u in F.THRESHOLD]))


@pytest.mark.parametrize("name", list(F.SCENES))
def test_emulated_traversal_never_drops_an_accepted_sphere(name):
    sc, recs, fams = _fams(name)
    c, r = IR.spheres_of(sc)
    o, d, _ = F.concat(fams)
    g = recs["recentre"]
    s, oo = F.f32_s(d), F.f32_oo(o, g)
    rng = np.random.default_rng(4)
    idx = np.flatnonzero((s > F.S_LO) & (s < F.S_HI) & (oo < F.OO_HI))
    idx = np.sort(rng.choice(idx, size=min(600, len(idx)), replace=False))
    checked = 0
    for i in idx:
        exact = set(_exact_hits(c, r, o[i], d[i]).tolist())
        with np.errstate(over="ignore", under="ignore", invalid="ignore"):
            cand, _ = _traverse(recs, o[i], d[i])
        assert not exact - cand, (name, i, sorted(exact - cand))
        checked += len(exact)
    assert checked > 200


@pytest.mark.parametrize("name", ["spread_1e8", "spread_4e14", "huge"])
def test_emulated_bounded_traversal_never_prunes_an_accepted_sphere(name):
    sc, recs, fams = _fams(name)
    c, r = IR.spheres_of(sc)
    o, d, _ = F.concat(fams)
    g = recs["recentre"]
    s, oo = F.f32_s(d), F.f32_oo(o, g)
    rng = np.random.default_rng(5)
    idx = np.flatnonzero((s > F.S_LO) & (s < F.S_HI) & (oo < F.OO_HI))
    idx = np.sort(rng.choice(idx, size=min(200, len(idx)), replace=False))
    checked = 0
    for i in idx:
        with np.errstate(over="ignore", under="ignore", invalid="ignore"):
            root = _roots(c, r, o[i], d[i])
            acc = np.flatnonzero(~np.isnan(root))
            if not len(acc):
                continue
            r0 = float(root[acc].min())
            for t in (r0, float(np.nextafter(r0, np.inf)), float(np.nextafter(r0, -np.inf)), 1.0):
                want = set(acc[root[acc] < t].tolist())
                if not t > 0.001 or not want:
                    continue
                cand, _ = _bounded(recs, o[i], d[i], tcap(t, d[i]))
                assert not want - cand, (name, i, t, sorted(want - cand))
                checked += len(want)
    assert checked > 100
