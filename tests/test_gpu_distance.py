"""Point queries on a resident scene (ResidentScene.nearest / .overlaps, rtb200_scene_nearest[_device],
rtb200_scene_overlaps[_device], DESIGN.md §4.19), held bit for bit to the numpy restatement (tests/distance_restatement.py) in
both outputs: every variant on the cover scene, the always-list and no-sphere scenes, the 10k and 100k RTIOW grids and the
contract's edge cases; bounds at and around the answer; overlaps against nearest(bound = r); launch sizes; stream ordering
against updates, rebuilds, edits and frames; shard and shared-memory handles; the device form's refusals; the stress builds;
and the host form's counters as the evidence of pruning."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import distance_restatement as DR
import distance_worker as DW
import intersect_rays as IR
import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from test_gpu_intersect import BRUTE, EXACT, FILTERED, REPO, STRESS, VARIANTS, _always_scene, _rtiow, _torch, dev
from test_gpu_scene_update import _jitter, _render
from test_gpu_shading_edges import assert_frames_match

pytestmark = pytest.mark.gpu
INF, NAN = float("inf"), float("nan")
MAX = float(np.finfo(np.float64).max)


def nearest_dev(rs, p, b=None, stream=None):
    h = rs.nearest(dev(p), None if b is None else dev(b), stream=stream)
    _torch().cuda.synchronize()
    assert sorted(h) == ["distance", "sphere"]
    return h["sphere"].cpu().numpy(), h["distance"].cpu().numpy()


def overlaps_dev(rs, p, r, stream=None):
    h = rs.overlaps(dev(p), dev(r), stream=stream)
    _torch().cuda.synchronize()
    return h["overlaps"].cpu().numpy()


def assert_nearest_equal(got, want, what):
    (gs, gd), (ws, wd) = got, want
    assert gs.dtype == np.int32 and gd.dtype == np.float64 and gs.shape == ws.shape, what
    bad = (gs != ws) | (gd.view(np.uint64) != wd.view(np.uint64))
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {len(gs)} points differ, first {i}: got ({gs[i]}, {gd[i]!r}), "
                             f"want ({ws[i]}, {wd[i]!r})")


def assert_overlaps_equal(got, want, what):
    assert got.dtype == np.uint8 and got.shape == want.shape, what
    bad = got != want
    assert not bad.any(), f"{what}: {int(bad.sum())} of {len(got)} balls differ, first {int(np.flatnonzero(bad)[0])}"


def check(rs, sc, p, what, b=None, radii=None):
    """Both kinds, device form, against the restatement; overlaps also against nearest(bound = r)."""
    c, r = DR.sphere_arrays(sc)
    want = DR.nearest(p, c, r, b)
    assert_nearest_equal(nearest_dev(rs, p, b), want, what)
    rad = radii if radii is not None else np.abs(np.random.default_rng(len(p)).normal(size=len(p)))
    ov = overlaps_dev(rs, p, rad)
    assert_overlaps_equal(ov, DR.overlaps(p, rad, c, r), what + " overlaps")
    assert_overlaps_equal(ov, (nearest_dev(rs, p, rad)[0] != -1).astype(np.uint8), what + " overlaps = nearest(r) != -1")
    return want


def edge_bounds(d):
    """Per-point bounds at the unbounded answer d*, one ulp either side, 0, -0, negative, NaN, +-inf and f64::MAX."""
    f = np.where(np.isfinite(d), d, 1.0)
    return {"at": f, "above": np.nextafter(f, INF), "below": np.nextafter(f, -INF), "zero": np.zeros_like(f),
            "negzero": np.full_like(f, -0.0), "neg": -np.abs(f) - 0.5, "nan": np.full_like(f, NAN),
            "inf": np.full_like(f, INF), "neginf": np.full_like(f, -INF), "max": np.full_like(f, MAX)}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_every_variant_on_the_cover_scene_with_edge_bounds(variant):
    sc = scenes.cover_scene(64, 48, 1)
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        sets = DW.point_sets(sc, np.random.default_rng(70), 3000)
        p = np.concatenate(list(sets.values()))
        s, d = check(rs, sc, p, f"{variant}/unbounded")
        assert (s >= 0).sum() > 10000 and (d < 0).sum() > 1000
        for name, b in edge_bounds(d).items():
            check(rs, sc, p, f"{variant}/bound {name}", b, radii=np.abs(b))
    finally:
        rs.release()


def _edge_scene():
    """Ties (duplicate and mirrored spheres), zero, negative and radius-1000 spheres, and non-finite spheres."""
    objs = [IR.sphere((0, 0, 0), 1.0), IR.sphere((0, 0, 0), 1.0), IR.sphere((2, 0, 0), 0.5), IR.sphere((-2, 0, 0), 0.5),
            IR.sphere((0, 3, 0), -1.0), IR.sphere((5, 5, 5), 0.0), IR.sphere((1, 1, 1), -0.0), IR.sphere((0, -1000.5, 0), 1000.0),
            IR.sphere((7, 0, 0), NAN), IR.sphere((INF, 0, 0), 1.0), IR.sphere((0, NAN, 0), 1.0), IR.sphere((0, 0, -4), INF),
            IR.sphere((3, 3, 0), 2.0), IR.sphere((3, 3, 0), -2.0)]
    return IR.scene_of(objs)[0]


def _edge_points(sc, rng):
    c, r = DR.sphere_arrays(sc)
    pts = [(0, 0, 0), (2, 0, 0), (2.5, 0, 0), (0, 2, 0), (1, 0, 0), (0, 10, 0), (5, 5, 5), (1, 1, 1), (NAN, 0, 0), (INF, 0, 0),
           (-INF, 1, 1), (0, 0, INF), (1e300, 0, 0), (-1e300, -1e300, 1e300), (0, 0, 1e-300), (-0.0, -0.0, -0.0), (3, 3, 2),
           (1e16, 0, 0), (0, 0, -4)]
    for j in range(len(r)):
        if np.isfinite(c[j]).all():
            pts.append(tuple(c[j]))
            if np.isfinite(r[j]):
                for a in range(3):
                    q = c[j].copy(); q[a] += abs(r[j]); pts.append(tuple(q))
    return np.concatenate([np.array(pts, np.float64), rng.normal(size=(500, 3)) * 5])


@pytest.mark.parametrize("name", ["edges", "always_list", "no_spheres", "c4_10k", "c4_100k"])
def test_scenes_with_ties_always_lists_no_spheres_and_many_spheres(name):
    rng = np.random.default_rng(71)
    if name == "edges":
        sc = _edge_scene()
    elif name == "always_list":
        sc = _always_scene()
    elif name == "no_spheres":
        sc, _ = IR.scene_of([])
    else:
        sc = _rtiow(50 if name == "c4_10k" else 158)
    if name == "edges":
        p = _edge_points(sc, rng)
    elif name == "no_spheres":
        p = rng.normal(size=(1000, 3)) * 10
    else:
        sets = DW.point_sets(sc, rng, 2000 if name.startswith("c4") else 3000)
        p = np.concatenate(list(sets.values()) + ([_edge_points(sc, rng)] if name == "always_list" else []))
    for v in ((FILTERED, BRUTE, EXACT) if name != "c4_100k" else (FILTERED, BRUTE)):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            s, d = check(rs, sc, p, f"{name}/variant {v}")
            if name in ("edges", "always_list"):
                for bn, b in edge_bounds(d).items():
                    check(rs, sc, p, f"{name}/variant {v}/bound {bn}", b, radii=np.abs(b))
        finally:
            rs.release()
    if name == "no_spheres":
        assert (s == -1).all() and np.isinf(d).all()
    else:
        assert (s >= 0).sum() > len(p) // 2


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097, 1 << 20])
def test_launch_sizes(n):
    sc = scenes.cover_scene(32, 24, 1)
    rng = np.random.default_rng(72)
    c, r = DR.sphere_arrays(sc)
    p = DW.point_sets(sc, rng, max(n // 3, 1))["box"]
    p = np.concatenate([p, rng.normal(size=(n, 3)) * 3])[:n]
    rad = np.abs(rng.normal(size=n)) * 0.3
    rs = R.ResidentScene(sc)
    try:
        want = DR.nearest(p, c, r)
        assert_nearest_equal(nearest_dev(rs, p), want, f"n = {n}")
        assert_overlaps_equal(overlaps_dev(rs, p, rad), DR.overlaps(p, rad, c, r), f"n = {n} overlaps")
        if n < 5000:
            h = rs.nearest(p)
            assert_nearest_equal((h["sphere"], h["distance"]), want, "host form")
            assert h["stats"]["rays"] == n
            assert rs.nearest(p, outputs=["sphere"]).keys() == {"sphere", "stats"}
    finally:
        rs.release()


@pytest.mark.parametrize("handle", ["plain", "shard", "wf_smem"])
def test_queries_see_updates_rebuilds_and_edits(handle, monkeypatch):
    torch = _torch()
    sc = scenes.cover_scene(48, 36, 1)
    opts = R.make_options(rank=1, world=2) if handle == "shard" else None
    if handle == "wf_smem":
        monkeypatch.setenv("RTB200_WF_SMEM", "7")
    rs = R.ResidentScene(sc, opts)
    monkeypatch.delenv("RTB200_WF_SMEM", raising=False)
    rng = np.random.default_rng(73)
    p = np.concatenate(list(DW.point_sets(sc, rng, 2000).values()))
    try:
        check(rs, sc, p, f"{handle}/uploaded")
        idx, recs = _jitter(sc, rng, 60)
        rs.update_spheres(idx, recs)
        check(rs, sc, p, f"{handle}/update_spheres")
        c, r = IR.spheres_of(sc)
        c = c + rng.normal(size=c.shape) * 0.2
        c[0] = [0.0, -1000.0, 0.0]
        for i in range(sc.n_spheres):
            sc.set_sphere(i, center=c[i].tolist(), radius=float(r[i]))
        rs.update_geometry(torch.from_numpy(np.concatenate([c, r[:, None]], axis=1)).cuda())
        check(rs, sc, p, f"{handle}/update_geometry")
        if handle != "wf_smem":   # a staged hierarchy refuses a rebuild and an edit
            rs.rebuild()
            check(rs, sc, p, f"{handle}/rebuild")
            new = [R.make_sphere((0.5, 0.3, 0.2), 0.25, {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}),
                   R.make_sphere((-3.0, 0.5, 1.0), -0.4, {"Light": {}})]
            rs.edit_spheres(remove=[3, 17, 40], insert=new, at=[0, 20])
            sc = sc.edited(remove=[3, 17, 40], insert=new, at=[0, 20])
            check(rs, sc, p, f"{handle}/edit_spheres")
    finally:
        rs.release()


def test_query_after_an_update_on_another_stream_sees_the_update():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(74)
    p = np.concatenate(list(DW.point_sets(sc, rng, 20000).values()))
    try:
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        c, r = IR.spheres_of(sc)
        c = c + np.array([0.0, 0.35, 0.0])
        c[0] = [0.0, -1000.0, 0.0]
        for i in range(sc.n_spheres):
            sc.set_sphere(i, center=c[i].tolist())
        geo = torch.from_numpy(np.concatenate([c, r[:, None]], axis=1)).cuda()
        dp = dev(p)
        torch.cuda.synchronize()
        with torch.cuda.stream(a):
            big = torch.randn(4096, 4096, device="cuda")
            for _ in range(8):
                big = big @ big / 64.0   # keeps stream A busy so that the update runs late
            rs.update_geometry(geo, stream=a)
        h = rs.nearest(dp, stream=b)
        torch.cuda.synchronize()
        want = DR.nearest(p, *DR.sphere_arrays(sc))
        assert_nearest_equal((h["sphere"].cpu().numpy(), h["distance"].cpu().numpy()), want, "query on B after an update on A")
    finally:
        rs.release()


def test_large_query_then_update_sees_the_old_scene():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(75)
    p = DW.point_sets(sc, rng, 1 << 20)["box"]
    rad = np.abs(rng.normal(size=len(p))) * 0.2
    try:
        c, r = DR.sphere_arrays(sc)
        want, want_ov = DR.nearest(p, c, r), DR.overlaps(p, rad, c, r)
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        geo = torch.from_numpy(np.concatenate([c + 0.5, r[:, None]], axis=1)).cuda()
        dp, dr = dev(p), dev(rad)
        torch.cuda.synchronize()
        h = rs.nearest(dp, stream=b)
        ho = rs.overlaps(dp, dr, stream=b)
        rs.update_geometry(geo, stream=a)
        torch.cuda.synchronize()
        assert_nearest_equal((h["sphere"].cpu().numpy(), h["distance"].cpu().numpy()), want, "query on B, then an update on A")
        assert_overlaps_equal(ho["overlaps"].cpu().numpy(), want_ov, "overlaps on B, then an update on A")
    finally:
        rs.release()


def test_frames_and_queries_interleaved_on_two_streams():
    torch = _torch()
    sc = scenes.cover_scene(48, 36, 4)
    lin_o, img_o, st_o = O.render(sc)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(76)
    p = np.concatenate(list(DW.point_sets(sc, rng, 20000).values()))
    want = DR.nearest(p, *DR.sphere_arrays(sc))
    dp = dev(p)
    n = 48 * 36 * 3
    try:
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        outs, qs = [], []
        for _ in range(4):
            d8 = torch.zeros(n, dtype=torch.uint8, device="cuda"); dl = torch.zeros(n, dtype=torch.float32, device="cuda")
            rs.render_async(d8.data_ptr(), dl.data_ptr(), stream=a.cuda_stream)
            outs.append((d8, dl))
            qs.append(rs.nearest(dp, stream=b))
        st = rs.wait()
        torch.cuda.synchronize()
        for d8, dl in outs:
            assert_frames_match((dl.cpu().numpy().reshape(36, 48, 3), d8.cpu().numpy().reshape(36, 48, 3)), (lin_o, img_o), "async frame")
        assert st["rays"] == st_o["rays"]
        for h in qs:
            assert_nearest_equal((h["sphere"].cpu().numpy(), h["distance"].cpu().numpy()), want, "query beside frames")
    finally:
        rs.release()


def test_queries_leave_renders_alone():
    sc = scenes.cover_scene(48, 36, 4)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(77)
    try:
        img0, lin0, rays0 = _render(rs)
        for _ in range(3):
            p = DW.point_sets(sc, rng, 30000)["box"]
            nearest_dev(rs, p)
            overlaps_dev(rs, p, np.full(len(p), 0.1))
            rs.nearest(p[:3000])
        img1, lin1, rays1 = _render(rs)
        assert np.array_equal(img0, img1) and np.array_equal(lin0.view(np.uint32), lin1.view(np.uint32)) and rays0 == rays1
    finally:
        rs.release()


@pytest.mark.parametrize("name", ["c4_10k", "c4_100k"])
def test_host_form_counters_show_the_pruning(name):
    """Points uniform in the box of the centres: FILTERED makes fewer than n/20 exact evaluations per point (a sanity bound,
    not a measured figure), and overlaps makes no more than nearest on the same points."""
    sc = _rtiow(50 if name == "c4_10k" else 158)
    m = sc.n_spheres
    rng = np.random.default_rng(78)
    p = DW.point_sets(sc, rng, 4000)["box"]
    n = len(p)
    c, r = DR.sphere_arrays(sc)
    want = DR.nearest(p, c, r)
    rad = np.maximum(want[1], 0.0) * rng.uniform(0.5, 1.5, size=n)
    stats = {}
    for vname, v in (("tree", FILTERED), ("brute", BRUTE)):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            h = rs.nearest(p)
            ho = rs.overlaps(p, rad)
        finally:
            rs.release()
        assert_nearest_equal((h["sphere"], h["distance"]), want, vname)
        assert_overlaps_equal(ho["overlaps"], DR.overlaps(p, rad, c, r), vname + " overlaps")
        st = h["stats"]
        assert st["rays"] == n and st["kernel_launches"] == 1 and ho["stats"]["rays"] == n
        assert st["trace_ms"] > 0 and st["device_ms"] >= st["trace_ms"]
        assert st["h2d_bytes"] == n * 24 and st["d2h_bytes"] == n * 12 + 256
        assert ho["stats"]["h2d_bytes"] == n * 32 and ho["stats"]["d2h_bytes"] == n + 256
        stats[vname] = (st, ho["stats"])
    st, so = stats["tree"]
    print(f"{name}: {m} spheres, per point: nearest {st['candidates'] / n:.1f} exact, {st['clusters'] / n:.2f} leaves, "
          f"{st['nodes'] / n:.2f} nodes; overlaps {so['candidates'] / n:.1f} exact, {so['clusters'] / n:.2f} leaves, {so['nodes'] / n:.2f} nodes")
    assert st["candidates"] < n * m / 20, (st, m)
    assert so["candidates"] <= st["candidates"] and so["nodes"] <= st["nodes"], (so, st)
    assert stats["brute"][0]["candidates"] == n * m and stats["brute"][0]["nodes"] == 0


def test_device_form_refuses_host_pointers():
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    try:
        import ctypes as C
        p = np.zeros((4, 3)); b = np.ones(4); out_d = _torch().zeros(4, dtype=_torch().float64, device="cuda")
        q = R.rt_points(p.ctypes.data, None)
        res = R.rt_nearest(out_d.data_ptr(), None)
        assert R.lib().rtb200_scene_nearest_device(rs.h, C.byref(q), 4, C.byref(res), None) == -1
        assert b"q->point" in R.lib().rtb200_last_error()
        dp = dev(p)
        q = R.rt_points(dp.data_ptr(), b.ctypes.data)
        ov = _torch().zeros(4, dtype=_torch().uint8, device="cuda")
        assert R.lib().rtb200_scene_overlaps_device(rs.h, C.byref(q), 4, ov.data_ptr(), None) == -1
        assert b"q->bound" in R.lib().rtb200_last_error()
        host_out = np.zeros(4)
        q = R.rt_points(dp.data_ptr(), None)
        assert R.lib().rtb200_scene_nearest_device(rs.h, C.byref(q), 4, C.byref(R.rt_nearest(host_out.ctypes.data, None)), None) == -1
        assert b"out->distance" in R.lib().rtb200_last_error()
        with pytest.raises(ValueError):
            rs.nearest(dev(p), b)   # mixed forms
    finally:
        rs.release()


def test_stress_builds_answer_point_queries_exactly(tmp_path):
    """The shipped library and every stress build (other leaf sizes and capacities) give the restatement's answers on the
    10k-sphere scene and the dense, coincident and rebuilt scenes of intersect_worker."""
    manifest = json.load(open(os.path.join(STRESS, "manifest.json")))
    want = {}
    for name, mk, rebuild, variants, seed in DW.cases():
        sc = mk()
        p, rad = DW.points_of(sc, seed)
        c, r = DR.sphere_arrays(sc)
        s, d = DR.nearest(p, c, r)
        for vname, _ in variants:
            want[f"{name}.{vname}.sphere"], want[f"{name}.{vname}.distance"] = s, d
            want[f"{name}.{vname}.overlaps"] = DR.overlaps(p, rad, c, r)
    for build in [None] + list(manifest):
        out = tmp_path / f"{build or 'shipped'}.npz"
        env = dict(os.environ)
        if build:
            env["RTB200_LIB"] = os.path.join(STRESS, f"librtb200_{build}.so")
        subprocess.check_call([sys.executable, "-B", os.path.join(REPO, "tests", "distance_worker.py"), str(out)], env=env)
        got = np.load(out)
        assert sorted(got.files) == sorted(want), build
        for k, w in want.items():
            assert np.array_equal(got[k].view(np.uint8), w.view(np.uint8)), (build, k)
