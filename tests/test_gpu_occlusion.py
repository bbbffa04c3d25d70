"""Occlusion queries on a resident scene (ResidentScene.occluded, rtb200_scene_occluded[_device], DESIGN.md §4.11), held to the
oracle: for ray i the answer is whether hit_world(world, Ray{o, d}, 0.001, t_max_i) is Some, and it must equal the closest-hit
query's `sphere != -1` under the same bound. Every variant on the closest-hit tests' ray sets with per-ray bounds at and around
the roots, shadow segments, scenes with always-list spheres, no spheres and 10k / 100k spheres, launch sizes, edited scenes,
shard and shared-memory handles, stream ordering against updates and frames, the counters of the host form (the deterministic
evidence of pruning and early exit), the refusals of the device form, and the stress builds."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import intersect_rays as IR
import intersect_worker as IW
import occlusion_worker as OW
import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from test_gpu_intersect import BRUTE, EXACT, FILTERED, REPO, STRESS, VARIANTS, _always_scene, _rtiow, _torch, cover_sets, dev, query
from test_gpu_scene_update import _jitter, _render
from test_gpu_shading_edges import assert_frames_match

pytestmark = pytest.mark.gpu


def occluded(rs, o, d, t_max=None, stream=None):
    """The device form on CUDA tensors, as a numpy uint8 array."""
    h = rs.occluded(dev(o), dev(d), None if t_max is None else dev(t_max), stream=stream)
    _torch().cuda.synchronize()
    assert sorted(h) == ["occluded"] and h["occluded"].dtype == _torch().uint8
    return h["occluded"].cpu().numpy()


def want_of(sc, o, d, t_max=None):
    return (IR.oracle(sc, o, d, t_max)["sphere"] >= 0).astype(np.uint8)


def assert_occluded_equal(got, want, what):
    assert got.shape == want.shape and got.dtype == np.uint8, (what, got.shape, got.dtype)
    diff = got != want
    if diff.any():
        i = int(np.flatnonzero(diff)[0])
        raise AssertionError(f"{what}: {int(diff.sum())} of {len(got)} rays differ, first ray {i}: got {got[i]}, want {want[i]}")


def check(rs, sc, o, d, what, t_max=None):
    """The device form against the oracle and against the closest-hit query under the same bound."""
    got = occluded(rs, o, d, t_max)
    want = want_of(sc, o, d, t_max)
    assert_occluded_equal(got, want, what)
    assert_occluded_equal((query(rs, o, d, t_max)["sphere"] != -1).astype(np.uint8), want, what + " (intersect)")
    return want


def t_edges(un):
    """The bounds of test_gpu_intersect.test_per_ray_t_max_edges around the unbounded roots r*."""
    f = np.where(np.isfinite(un["t"]), un["t"], 1.0)
    return [f, np.nextafter(f, np.inf), np.nextafter(f, -np.inf), np.full_like(f, 0.001), np.full_like(f, np.nextafter(0.001, 0.0)),
            np.full_like(f, np.nextafter(0.001, 1.0)), np.full_like(f, 0.0), np.full_like(f, np.inf), np.full_like(f, np.nan),
            np.full_like(f, IR.MAX), np.full_like(f, -np.inf)]


def shadow_segments(sc, o, d, rng, targets=None):
    """From every hit of the rays (o, d) to a random point on a random other sphere (or on one of `targets`): t_max = 1."""
    first = IR.oracle(sc, o, d)
    m = first["sphere"] >= 0
    p, j = first["point"][m], first["sphere"][m]
    c, r = IR.spheres_of(sc)
    pool = np.flatnonzero(np.isfinite(c).all(axis=1) & np.isfinite(r) & (np.abs(r) < 100)) if targets is None else np.asarray(targets)
    k = pool[rng.integers(0, len(pool), size=len(p))]
    k = np.where(k == j, pool[(np.searchsorted(pool, k) + 1) % len(pool)], k) if len(pool) > 1 else k
    g = rng.normal(size=(len(p), 3))
    g /= np.linalg.norm(g, axis=1, keepdims=True)
    return p, (c[k] + g * np.abs(r[k])[:, None]) - p, np.ones(len(p))


def short_segments(sc, rng, k):
    """k segments of length <= 0.5 from random sphere surfaces, t_max = 1."""
    c, r = IR.spheres_of(sc)
    ok = np.flatnonzero(np.isfinite(c).all(axis=1) & np.isfinite(r) & (np.abs(r) < 1e6))
    j = ok[rng.integers(0, len(ok), size=k)]
    g = rng.normal(size=(k, 3)); g /= np.linalg.norm(g, axis=1, keepdims=True)
    v = g + rng.normal(size=(k, 3)); v /= np.linalg.norm(v, axis=1, keepdims=True)
    return c[j] + g * np.abs(r[j])[:, None], v * rng.uniform(0.01, 0.5, size=(k, 1)), np.ones(k)


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_every_variant_matches_the_oracle_on_the_cover_scene(variant):
    sc = scenes.cover_scene(64, 48, 1)
    rng = np.random.default_rng(50)
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        occ = 0
        for name, (o, d) in cover_sets(sc, rng).items():
            un = IR.oracle(sc, o, d)
            edges = t_edges(un)
            tm = np.stack(edges, axis=1)[np.arange(len(o)), rng.integers(0, len(edges), size=len(o))].copy()
            check(rs, sc, o, d, f"{variant}/{name}/edges", tm)
            f = np.where(np.isfinite(un["t"]), un["t"], 1.0)
            occ += int(check(rs, sc, o, d, f"{variant}/{name}/fractions", f * rng.uniform(0.0, 2.0, size=len(f))).sum())
            check(rs, sc, o, d, f"{variant}/{name}/unbounded")
        so, sd, st = shadow_segments(sc, *IR.camera_rays(sc, 64, 48), rng)
        occ += int(check(rs, sc, so, sd, f"{variant}/shadow segments", st).sum())
        assert occ > 10000
    finally:
        rs.release()


def test_every_edge_bound_alone():
    sc = scenes.cover_scene(64, 48, 1)
    rng = np.random.default_rng(51)
    o1, d1 = IR.camera_rays(sc, 64, 48)
    o2, d2 = IR.surface_rays(sc, rng, 3000)
    o = np.concatenate([o1, o2]); d = np.concatenate([d1, d2])
    un = IR.oracle(sc, o, d)
    for v in (FILTERED, BRUTE, EXACT):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            for k, e in enumerate(t_edges(un)):
                got = occluded(rs, o, d, e)
                assert_occluded_equal(got, (IR.filtered(un, e)["sphere"] >= 0).astype(np.uint8), f"edge {k}/variant {v}")
        finally:
            rs.release()


def test_shadow_segments_toward_the_lights_of_the_test_scene():
    cfg = scenes._variant(scenes.test_scene_config(), 64, 48, 1, 4)
    lights = [i for i, ob in enumerate(cfg["objects"]) if "Light" in ob["material"]]
    assert lights
    sc = R.Scene.from_config(cfg, scenes.SCENES_DIR)
    rng = np.random.default_rng(52)
    o, d = IR.camera_rays(sc, 64, 48)
    first = IR.oracle(sc, o, d)
    m = first["sphere"] >= 0
    p = first["point"][m]
    c, r = IR.spheres_of(sc)
    # Ray::new(point, light.center - point), as the light test casts it, up to just short of the light's near surface
    sd = c[lights[0]] - p
    sets = [(p, sd, 1.0 - 1.001 * abs(r[lights[0]]) / np.linalg.norm(sd, axis=1))]
    sets.append(shadow_segments(sc, o, d, rng, targets=lights))
    for v in (FILTERED, BRUTE, EXACT):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            for k, (so, sd, st) in enumerate(sets):
                w = check(rs, sc, so, sd, f"lights {k}/variant {v}", st)
                assert 0 < w.sum() < len(w)
        finally:
            rs.release()


@pytest.mark.parametrize("name", ["always_list", "no_spheres", "c4_10k", "c4_100k"])
def test_scenes_with_always_lists_no_spheres_and_many_spheres(name):
    rng = np.random.default_rng(53)
    if name == "always_list":
        sc = _always_scene()
    elif name == "no_spheres":
        sc, _ = IR.scene_of([])
    else:
        sc = _rtiow(50 if name == "c4_10k" else 158)
    o, d = IR.camera_rays(sc, 96, 54)
    sets = [(o, d), IR.degenerate_rays(sc, rng)]
    if sc.n_spheres:
        sets += [IR.box_rays(sc, rng, 3000), IR.surface_rays(sc, rng, 2000), IR.grazing_rays(sc, rng, 1000)]
    o = np.concatenate([s[0] for s in sets]); d = np.concatenate([s[1] for s in sets])
    t = rng.uniform(0.0, 3.0, size=len(o))
    segs = [short_segments(sc, rng, 3000), shadow_segments(sc, *IR.camera_rays(sc, 48, 27), rng)] if sc.n_spheres else []
    for v in ((FILTERED, BRUTE, EXACT) if name != "c4_100k" else (FILTERED, BRUTE)):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            w = check(rs, sc, o, d, f"{name}/variant {v}")
            check(rs, sc, o, d, f"{name}/variant {v}/random bounds", t)
            for k, (so, sd, st) in enumerate(segs):
                check(rs, sc, so, sd, f"{name}/variant {v}/segments {k}", st)
        finally:
            rs.release()
    if name == "no_spheres":
        assert (w == 0).all()
    else:
        assert w.sum() > 1000


@pytest.mark.parametrize("n", [1, 31, 33, 1 << 24])
def test_launch_sizes(n):
    if n < 1000:
        sc = scenes.cover_scene(32, 24, 1)
    else:
        sc, _ = IR.scene_of([IR.sphere((0, -1000, 0), 1000.0), IR.sphere((0, 1, 0), 1.0), IR.sphere((-4, 1, 0), 1.0),
                             IR.sphere((4, 1, 0), -1.0)])
    rng = np.random.default_rng(54)
    if n < 1000:
        c, _ = IR.spheres_of(sc)
        o = np.tile(np.array(sc.c.camera.origin.tup()), (n, 1))
        d = c[rng.integers(1, sc.n_spheres, size=n)] - o
    else:
        o, d = IR.box_rays(sc, rng, n, box=(np.array([-6.0, 0.1, -6.0]), np.array([6.0, 3.0, 6.0])))
    t = rng.uniform(0.0, 2.0, size=n)
    rs = R.ResidentScene(sc)
    try:
        want = want_of(sc, o, d, t)
        assert_occluded_equal(occluded(rs, o, d, t), want, f"n = {n}")
        if n < 1000:
            h = rs.occluded(o, d, t)
            assert_occluded_equal(h["occluded"], want, "host form")
            assert h["stats"]["rays"] == n
    finally:
        rs.release()
    assert want.any() and (n < 1000 or not want.all())


@pytest.mark.parametrize("handle", ["plain", "shard", "wf_smem"])
def test_queries_see_updates_and_rebuilds(handle, monkeypatch):
    torch = _torch()
    sc = scenes.cover_scene(48, 36, 1)
    opts = R.make_options(rank=1, world=2) if handle == "shard" else None
    if handle == "wf_smem":
        monkeypatch.setenv("RTB200_WF_SMEM", "7")
    rs = R.ResidentScene(sc, opts)
    monkeypatch.delenv("RTB200_WF_SMEM", raising=False)
    rng = np.random.default_rng(55)
    so, sd, st = shadow_segments(sc, *IR.camera_rays(sc, 96, 72), rng)
    o2, d2 = IR.box_rays(sc, rng, 4000)
    o = np.concatenate([so, o2]); d = np.concatenate([sd, d2]); t = np.concatenate([st, rng.uniform(0, 3, size=4000)])
    try:
        if handle == "wf_smem":
            assert rs.kernel_info()["smem_mask"] == 7
        check(rs, sc, o, d, f"{handle}/uploaded", t)
        idx, recs = _jitter(sc, rng, 60)
        rs.update_spheres(idx, recs)
        check(rs, sc, o, d, f"{handle}/update_spheres", t)
        c, r = IR.spheres_of(sc)
        c = c + rng.normal(size=c.shape) * 0.2
        c[0] = [0.0, -1000.0, 0.0]
        for i in range(sc.n_spheres):
            sc.set_sphere(i, center=c[i].tolist(), radius=float(r[i]))
        rs.update_geometry(torch.from_numpy(np.concatenate([c, r[:, None]], axis=1)).cuda())
        check(rs, sc, o, d, f"{handle}/update_geometry", t)
        if handle != "wf_smem":   # a staged hierarchy refuses a rebuild
            rs.rebuild()
            check(rs, sc, o, d, f"{handle}/rebuild", t)
    finally:
        rs.release()


def test_query_after_an_update_on_another_stream_sees_the_update():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(56)
    o, d = IR.camera_rays(sc, 128, 96)
    t = rng.uniform(0.5, 3.0, size=len(o))
    try:
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        c, r = IR.spheres_of(sc)
        c = c + np.array([0.0, 0.35, 0.0])
        c[0] = [0.0, -1000.0, 0.0]
        for i in range(sc.n_spheres):
            sc.set_sphere(i, center=c[i].tolist())
        geo = torch.from_numpy(np.concatenate([c, r[:, None]], axis=1)).cuda()
        do, dd, dt = dev(o), dev(d), dev(t)
        torch.cuda.synchronize()
        with torch.cuda.stream(a):
            big = torch.randn(4096, 4096, device="cuda")
            for _ in range(8):
                big = big @ big / 64.0   # keeps stream A busy so that the update runs late
            rs.update_geometry(geo, stream=a)
        h = rs.occluded(do, dd, dt, stream=b)
        torch.cuda.synchronize()
        assert_occluded_equal(h["occluded"].cpu().numpy(), want_of(sc, o, d, t), "query on B after an update on A")
    finally:
        rs.release()


def test_large_query_then_update_sees_the_old_scene():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(57)
    o, d = IR.box_rays(sc, rng, 1 << 20)
    t = rng.uniform(0.0, 4.0, size=len(o))
    try:
        want = want_of(sc, o, d, t)
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        c, r = IR.spheres_of(sc)
        geo = torch.from_numpy(np.concatenate([c + 0.5, r[:, None]], axis=1)).cuda()
        do, dd, dt = dev(o), dev(d), dev(t)
        torch.cuda.synchronize()
        h = rs.occluded(do, dd, dt, stream=b)
        rs.update_geometry(geo, stream=a)
        torch.cuda.synchronize()
        assert_occluded_equal(h["occluded"].cpu().numpy(), want, "query on B, then an update on A")
    finally:
        rs.release()


def test_frames_and_queries_interleaved_on_two_streams():
    torch = _torch()
    sc = scenes.cover_scene(48, 36, 4)
    lin_o, img_o, st_o = O.render(sc)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(58)
    o, d, t = shadow_segments(sc, *IR.camera_rays(sc, 160, 120), rng)
    want = want_of(sc, o, d, t)
    do, dd, dt = dev(o), dev(d), dev(t)
    n = 48 * 36 * 3
    try:
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        outs, occs = [], []
        for k in range(4):
            d8 = torch.zeros(n, dtype=torch.uint8, device="cuda"); dl = torch.zeros(n, dtype=torch.float32, device="cuda")
            rs.render_async(d8.data_ptr(), dl.data_ptr(), stream=a.cuda_stream)
            outs.append((d8, dl))
            occs.append(rs.occluded(do, dd, dt, stream=b))
        st = rs.wait()
        torch.cuda.synchronize()
        for d8, dl in outs:
            assert_frames_match((dl.cpu().numpy().reshape(36, 48, 3), d8.cpu().numpy().reshape(36, 48, 3)), (lin_o, img_o), "async frame")
        assert st["rays"] == st_o["rays"]
        for h in occs:
            assert_occluded_equal(h["occluded"].cpu().numpy(), want, "query beside frames")
    finally:
        rs.release()


def test_queries_leave_renders_alone():
    sc = scenes.cover_scene(48, 36, 4)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(59)
    try:
        img0, lin0, rays0 = _render(rs)
        for _ in range(3):
            o, d = IR.box_rays(sc, rng, 30000)
            occluded(rs, o, d, rng.uniform(0, 2, size=len(o)))
            rs.occluded(*IR.surface_rays(sc, rng, 3000))
        img1, lin1, rays1 = _render(rs)
        assert np.array_equal(img0, img1) and np.array_equal(lin0.view(np.uint32), lin1.view(np.uint32)) and rays0 == rays1
    finally:
        rs.release()


def test_host_form_counters_and_pruning():
    sc = _rtiow(50)
    rng = np.random.default_rng(60)
    o, d, t = short_segments(sc, rng, 3000)
    n, m = len(o), sc.n_spheres
    want = want_of(sc, o, d, t)
    assert 0 < want.sum() < n
    for name, v in (("tree", FILTERED), ("exact", EXACT), ("brute", BRUTE)):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            h = rs.occluded(o, d, t)
            h0 = rs.occluded(o, d)
            cl = rs.intersect(o, d, t)
        finally:
            rs.release()
        assert_occluded_equal(h["occluded"], want, name)
        assert_occluded_equal(h0["occluded"], want_of(sc, o, d), name + " unbounded")
        st = h["stats"]
        assert st["rays"] == n and st["kernel_launches"] == 1
        assert st["trace_ms"] > 0 and st["device_ms"] >= st["trace_ms"]
        assert st["h2d_bytes"] == n * 56 and st["d2h_bytes"] == n + 256
        assert h0["stats"]["h2d_bytes"] == n * 48 and h0["stats"]["d2h_bytes"] == n + 256
        if name == "tree":   # the pruning and the early exit: strictly fewer nodes and f64 tests than the closest-hit query
            assert st["nodes"] < cl["stats"]["nodes"] and st["candidates"] < cl["stats"]["candidates"], (st, cl["stats"])
            assert st["clusters"] <= cl["stats"]["clusters"]
        if name == "exact":   # every sphere up to the first acceptance, never more than the closest-hit query's n * m
            assert st["candidates"] < n * m
    # rays with t_max <= 0.001 are counted, answered 0, and tested against no sphere
    rs = R.ResidentScene(sc)
    try:
        h = rs.occluded(o, d, np.full(n, 0.001))
    finally:
        rs.release()
    assert (h["occluded"] == 0).all() and h["stats"]["rays"] == n and h["stats"]["candidates"] == 0 and h["stats"]["nodes"] == 0


def test_device_form_refuses_host_pointers_and_a_null_output():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    try:
        o = np.zeros((4, 3)); d = np.ones((4, 3)); t = np.full(4, 7.0); hout = np.full(4, 9, np.uint8)
        do, dd = dev(o), dev(d)
        dout = torch.full((4,), 9, dtype=torch.uint8, device="cuda")
        L = R.lib()
        for rays, out, what in ((R.rt_rays(o.ctypes.data, dd.data_ptr(), None), dout.data_ptr(), "rays->origin"),
                                (R.rt_rays(do.data_ptr(), d.ctypes.data, None), dout.data_ptr(), "rays->direction"),
                                (R.rt_rays(do.data_ptr(), dd.data_ptr(), t.ctypes.data), dout.data_ptr(), "rays->t_max"),
                                (R.rt_rays(do.data_ptr(), dd.data_ptr(), None), hout.ctypes.data, "occluded"),
                                (R.rt_rays(do.data_ptr(), dd.data_ptr(), None), None, "occluded")):
            assert L.rtb200_scene_occluded_device(rs.h, C.byref(rays), 4, out, None) == -1
            assert what.encode() in L.rtb200_last_error()
        torch.cuda.synchronize()
        assert (hout == 9).all() and (dout.cpu().numpy() == 9).all() and (t == 7.0).all()
        with pytest.raises(ValueError):
            rs.occluded(do, dd.float())
        with pytest.raises(ValueError):
            rs.occluded(o, d[:3])
        with pytest.raises(ValueError):
            rs.occluded(do, dd, torch.ones(3, dtype=torch.float64, device="cuda"))
        assert rs.occluded(o[:0], d[:0])["occluded"].shape == (0,)
        assert rs.occluded(do[:0], dd[:0])["occluded"].shape == (0,)
    finally:
        rs.release()


def test_stress_builds_answer_occlusion_queries_exactly(tmp_path):
    """Every stress build answers the 10k-sphere scene's queries and the dense scenes' (as uploaded and after rebuild()),
    unbounded and under per-ray bounds, like the oracle; the coincident spheres overflow the smallest candidate list."""
    manifest = json.load(open(os.path.join(STRESS, "manifest.json")))
    sc = IW.c4_scene()
    o, d = IW.c4_rays(sc)
    sets = {"filtered": (sc, o, d), "brute": (sc, o, d)}
    for name, (mk, rays, _) in IW.SETS.items():
        s = mk()
        sets[name] = (s, *rays(s))
    wants = {}
    for name, (s, so, sd) in sets.items():
        for tag, t in (("none", None), ("t", OW.bounds(len(so), 44))):
            wants[f"{name}.{tag}"] = want_of(s, so, sd, t)
            assert 100 < wants[f"{name}.{tag}"].sum() < len(so), (name, tag)
    for name in manifest:
        out = tmp_path / f"{name}.npz"
        env = dict(os.environ, RTB200_LIB=os.path.join(STRESS, f"librtb200_{name}.so"))
        subprocess.run([sys.executable, os.path.join(REPO, "tests", "occlusion_worker.py"), str(out)], env=env, check=True, timeout=900)
        z = np.load(out)
        meta = json.loads(str(z["meta"]))
        for key, w in wants.items():
            assert_occluded_equal(z[key], w, f"{name}/{key}")
            assert meta[key]["rays"] == len(w)
