"""Closest-hit queries on a resident scene (ResidentScene.intersect, rtb200_scene_intersect[_device], DESIGN.md §4.10), held bit
for bit to the oracle's hit_world on the same rays: every variant and the rays that reach the kernel's edge paths, scenes with
always-list spheres, no spheres and 10k / 100k spheres, per-ray t_max, launch sizes, edited scenes, shard and shared-memory
handles, stream ordering against updates and frames, the counters of the host form, the stress builds, and the refusal of host
pointers by the device form."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import intersect_rays as IR
import intersect_worker as IW
import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from test_gpu_scene_update import _jitter, _render
from test_gpu_shading_edges import assert_frames_match

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRESS = os.path.join(REPO, "rust-raytracer_b200", "stress")
FILTERED, BRUTE, EXACT, AUTO = R.RT_VARIANT_FILTERED, R.RT_VARIANT_BRUTE_FORCE, R.RT_VARIANT_EXACT_F64, R.RT_VARIANT_AUTO
VARIANTS = {"auto": AUTO, "filtered": FILTERED, "exact_f64": EXACT, "brute_force": BRUTE}


def _torch():
    import torch
    return torch


def dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def host(h):
    return {k: v.cpu().numpy() for k, v in h.items()}


def query(rs, o, d, t_max=None, stream=None):
    """The device form on CUDA tensors, returned as numpy arrays."""
    h = rs.intersect(dev(o), dev(d), None if t_max is None else dev(t_max), stream=stream)
    _torch().cuda.synchronize()
    return host(h)


def check(rs, sc, o, d, what, t_max=None):
    got = query(rs, o, d, t_max)
    want = IR.oracle(sc, o, d, t_max)
    IR.assert_hits_equal(got, want, what)
    return want


def cover_sets(sc, rng):
    o, d = IR.camera_rays(sc, 160, 120)
    first = IR.oracle(sc, o, d)
    so, sd = IR.secondary_rays(first, rng)
    return {"camera": (o, d), "secondary": (so, sd), "grazing": IR.grazing_rays(sc, rng, 4000), "axis": IR.axis_rays(sc, rng, 4000),
            "surface": IR.surface_rays(sc, rng, 4000), "d_1e-20": IR.scaled_rays(sc, rng, 2000, 1e-20),
            "d_1e20": IR.scaled_rays(sc, rng, 2000, 1e20), "degenerate": IR.degenerate_rays(sc, rng)}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_every_variant_matches_the_oracle_on_the_cover_scene(variant):
    sc = scenes.cover_scene(64, 48, 1)
    rng = np.random.default_rng(10)
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        hits = 0
        for name, (o, d) in cover_sets(sc, rng).items():
            want = check(rs, sc, o, d, f"{variant}/{name}")
            hits += int((want["sphere"] >= 0).sum())
        assert hits > 20000
    finally:
        rs.release()


def _always_scene():
    cfg = scenes._variant(scenes.cover_config(), 32, 24, 1, 4)
    inf, nan = float("inf"), float("nan")
    cfg["objects"] = cfg["objects"] + [IR.sphere((1e15, 0, 0), 1e15 - 5.0), IR.sphere((0, 2e15, 0), 2e15 - 3.0),
                                       IR.sphere((nan, 0, 0), 1.0), IR.sphere((0, 1, 0), nan), IR.sphere((0, 0, -50), inf),
                                       IR.sphere((-3e16, 1, 0), 1.0)]
    return R.Scene.from_config(cfg)


def _rtiow(half):
    return R.Scene.from_config(scenes._variant(scenes.rtiow_config(half), 96, 54, 1, 50))


@pytest.mark.parametrize("name", ["always_list", "no_spheres", "c4_10k", "c4_100k"])
def test_scenes_with_always_lists_no_spheres_and_many_spheres(name):
    rng = np.random.default_rng(11)
    if name == "always_list":
        sc = _always_scene()
    elif name == "no_spheres":
        sc, _ = IR.scene_of([])
    else:
        sc = _rtiow(50 if name == "c4_10k" else 158)
        assert sc.n_spheres > (9900 if name == "c4_10k" else 99000)
    o, d = IR.camera_rays(sc, 96, 54)
    sets = [(o, d), IR.degenerate_rays(sc, rng)]
    if sc.n_spheres:
        sets += [IR.box_rays(sc, rng, 3000), IR.surface_rays(sc, rng, 2000), IR.grazing_rays(sc, rng, 1000)]
        sets.append(IR.secondary_rays(IR.oracle(sc, o, d), rng))
    o = np.concatenate([s[0] for s in sets]); d = np.concatenate([s[1] for s in sets])
    for v in ((FILTERED, BRUTE, EXACT) if name != "c4_100k" else (FILTERED, BRUTE)):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            want = check(rs, sc, o, d, f"{name}/variant {v}")
        finally:
            rs.release()
    if name == "no_spheres":
        assert (want["sphere"] == -1).all() and np.isinf(want["t"]).all()
    else:
        assert (want["sphere"] >= 0).sum() > 1000


def test_per_ray_t_max_edges():
    sc = scenes.cover_scene(64, 48, 1)
    rng = np.random.default_rng(12)
    o1, d1 = IR.camera_rays(sc, 64, 48)
    o2, d2 = IR.surface_rays(sc, rng, 3000)
    o = np.concatenate([o1, o2]); d = np.concatenate([d1, d2])
    un = IR.oracle(sc, o, d)
    f = np.where(np.isfinite(un["t"]), un["t"], 1.0)
    edges = [f, np.nextafter(f, np.inf), np.nextafter(f, -np.inf), np.full_like(f, 0.001), np.full_like(f, np.nextafter(0.001, 0.0)),
             np.full_like(f, np.nextafter(0.001, 1.0)), np.full_like(f, 0.0), np.full_like(f, np.inf), np.full_like(f, np.nan),
             np.full_like(f, IR.MAX), np.full_like(f, -np.inf)]
    tm = np.stack(edges, axis=1)[np.arange(len(f)), rng.integers(0, len(edges), size=len(f))].copy()
    for v in (FILTERED, BRUTE, EXACT):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            check(rs, sc, o, d, f"t_max/variant {v}", tm)
            for k, e in enumerate(edges):
                got = query(rs, o, d, e)
                IR.assert_hits_equal(got, IR.filtered(un, e), f"t_max edge {k}/variant {v}")
        finally:
            rs.release()


@pytest.mark.parametrize("n", [1, 31, 33, 1 << 24])
def test_launch_sizes(n):
    if n < 1000:
        sc = scenes.cover_scene(32, 24, 1)
    else:   # many rays on a small scene, so that the oracle keeps up: the 64-bit indices of the last chunks
        sc, _ = IR.scene_of([IR.sphere((0, -1000, 0), 1000.0), IR.sphere((0, 1, 0), 1.0), IR.sphere((-4, 1, 0), 1.0),
                             IR.sphere((4, 1, 0), -1.0)])
    rng = np.random.default_rng(13)
    if n < 1000:   # from the camera towards random spheres' centres
        c, _ = IR.spheres_of(sc)
        o = np.tile(np.array(sc.c.camera.origin.tup()), (n, 1))
        d = c[rng.integers(1, sc.n_spheres, size=n)] - o
    else:
        o, d = IR.box_rays(sc, rng, n, box=(np.array([-6.0, 0.1, -6.0]), np.array([6.0, 3.0, 6.0])))
    rs = R.ResidentScene(sc)
    try:
        want = check(rs, sc, o, d, f"n = {n}")
        if n < 1000:
            got = rs.intersect(o, d)
            IR.assert_hits_equal(got, want, "host form")
            assert got["stats"]["rays"] == n
    finally:
        rs.release()
    assert (want["sphere"] >= 0).any()


def test_partial_outputs_leave_the_other_buffers_alone_and_forms_agree():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rng = np.random.default_rng(14)
    o, d = IR.box_rays(sc, rng, 5000)
    rs = R.ResidentScene(sc)
    try:
        want = IR.oracle(sc, o, d)
        do, dd = dev(o), dev(d)
        # one byte buffer per output, filled with 0x5A; only `sphere` is passed
        bufs = {k: torch.full((5000 * c * np.dtype(ty).itemsize,), 0x5A, dtype=torch.uint8, device="cuda") for k, c, ty in R.HIT_FIELDS}
        rays = R.rt_rays(do.data_ptr(), dd.data_ptr(), None)
        hits = R.rt_hits(*(bufs[k].data_ptr() if k == "sphere" else None for k in IR.FIELDS))
        assert R.lib().rtb200_scene_intersect_device(rs.h, C.byref(rays), 5000, C.byref(hits), None) == 0
        torch.cuda.synchronize()
        assert np.array_equal(bufs["sphere"].cpu().numpy().view(np.int32), want["sphere"])
        for k in IR.FIELDS:
            if k != "sphere":
                assert (bufs[k] == 0x5A).all().item(), k
        sub = rs.intersect(do, dd, outputs=("t", "uv"))
        assert sorted(sub) == ["t", "uv"]
        IR.assert_hits_equal(host(sub), want, "outputs t, uv", fields=["t", "uv"])
        IR.assert_hits_equal(rs.intersect(o, d), query(rs, o, d), "host form = device form")
    finally:
        rs.release()


@pytest.mark.parametrize("handle", ["plain", "shard", "wf_smem"])
def test_queries_see_updates_and_rebuilds(handle, monkeypatch):
    torch = _torch()
    sc = scenes.cover_scene(48, 36, 1)
    opts = R.make_options(rank=1, world=2) if handle == "shard" else None
    if handle == "wf_smem":
        monkeypatch.setenv("RTB200_WF_SMEM", "7")
    rs = R.ResidentScene(sc, opts)
    monkeypatch.delenv("RTB200_WF_SMEM", raising=False)
    rng = np.random.default_rng(15)
    o, d = IR.camera_rays(sc, 96, 72)
    o2, d2 = IR.box_rays(sc, rng, 4000)
    o = np.concatenate([o, o2]); d = np.concatenate([d, d2])
    try:
        if handle == "wf_smem":
            assert rs.kernel_info()["smem_mask"] == 7
        check(rs, sc, o, d, f"{handle}/uploaded")
        idx, recs = _jitter(sc, rng, 60)
        rs.update_spheres(idx, recs)
        check(rs, sc, o, d, f"{handle}/update_spheres")
        c, r = IR.spheres_of(sc)
        c = c + rng.normal(size=c.shape) * 0.2
        c[0] = [0.0, -1000.0, 0.0]
        for i in range(sc.n_spheres):
            sc.set_sphere(i, center=c[i].tolist(), radius=float(r[i]))
        rs.update_geometry(torch.from_numpy(np.concatenate([c, r[:, None]], axis=1)).cuda())
        check(rs, sc, o, d, f"{handle}/update_geometry")
        if handle != "wf_smem":   # a staged hierarchy refuses a rebuild (tests/test_gpu_scene_staging.py)
            rs.rebuild()
            check(rs, sc, o, d, f"{handle}/rebuild")
    finally:
        rs.release()


def test_query_after_an_update_on_another_stream_sees_the_update():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(16)
    o, d = IR.camera_rays(sc, 128, 96)
    try:
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        c, r = IR.spheres_of(sc)
        c = c + np.array([0.0, 0.35, 0.0])
        c[0] = [0.0, -1000.0, 0.0]
        for i in range(sc.n_spheres):
            sc.set_sphere(i, center=c[i].tolist())
        geo = torch.from_numpy(np.concatenate([c, r[:, None]], axis=1)).cuda()
        do, dd = dev(o), dev(d)
        torch.cuda.synchronize()
        with torch.cuda.stream(a):
            big = torch.randn(4096, 4096, device="cuda")
            for _ in range(8):
                big = big @ big / 64.0   # keeps stream A busy so that the update runs late
            rs.update_geometry(geo, stream=a)
        h = rs.intersect(do, dd, stream=b)
        torch.cuda.synchronize()
        IR.assert_hits_equal(host(h), IR.oracle(sc, o, d), "query on B after an update on A")
    finally:
        rs.release()


def test_large_query_then_update_sees_the_old_scene():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(17)
    o, d = IR.box_rays(sc, rng, 1 << 20)
    try:
        want = IR.oracle(sc, o, d)
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        c, r = IR.spheres_of(sc)
        geo = torch.from_numpy(np.concatenate([c + 0.5, r[:, None]], axis=1)).cuda()
        do, dd = dev(o), dev(d)
        torch.cuda.synchronize()
        h = rs.intersect(do, dd, stream=b)
        rs.update_geometry(geo, stream=a)
        torch.cuda.synchronize()
        IR.assert_hits_equal(host(h), want, "query on B, then an update on A")
    finally:
        rs.release()


def test_frames_and_queries_interleaved_on_two_streams():
    torch = _torch()
    sc = scenes.cover_scene(48, 36, 4)
    lin_o, img_o, st_o = O.render(sc)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(18)
    o, d = IR.box_rays(sc, rng, 20000)
    want = IR.oracle(sc, o, d)
    do, dd = dev(o), dev(d)
    n = 48 * 36 * 3
    try:
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        outs, hits = [], []
        for k in range(4):
            d8 = torch.zeros(n, dtype=torch.uint8, device="cuda"); dl = torch.zeros(n, dtype=torch.float32, device="cuda")
            rs.render_async(d8.data_ptr(), dl.data_ptr(), stream=a.cuda_stream)
            outs.append((d8, dl))
            hits.append(rs.intersect(do, dd, stream=b))
        st = rs.wait()
        torch.cuda.synchronize()
        for d8, dl in outs:
            assert_frames_match((dl.cpu().numpy().reshape(36, 48, 3), d8.cpu().numpy().reshape(36, 48, 3)), (lin_o, img_o), "async frame")
        assert st["rays"] == st_o["rays"]
        for h in hits:
            IR.assert_hits_equal(host(h), want, "query beside frames")
    finally:
        rs.release()


def test_queries_leave_renders_alone():
    sc = scenes.cover_scene(48, 36, 4)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(19)
    try:
        img0, lin0, rays0 = _render(rs)
        for _ in range(3):
            query(rs, *IR.box_rays(sc, rng, 30000))
            rs.intersect(*IR.surface_rays(sc, rng, 3000))
        img1, lin1, rays1 = _render(rs)
        assert np.array_equal(img0, img1) and np.array_equal(lin0.view(np.uint32), lin1.view(np.uint32)) and rays0 == rays1
    finally:
        rs.release()


def test_host_form_counters():
    sc = _rtiow(50)
    rng = np.random.default_rng(20)
    o, d = IR.box_rays(sc, rng, 3000)
    n, m = len(o), sc.n_spheres
    want = IR.oracle(sc, o, d)
    st = {}
    for name, v in (("tree", FILTERED), ("exact", EXACT), ("brute", BRUTE)):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            h = rs.intersect(o, d)
        finally:
            rs.release()
        IR.assert_hits_equal(h, want, name)
        st[name] = h["stats"]
        assert st[name]["rays"] == n and st[name]["kernel_launches"] == 1
        assert st[name]["trace_ms"] > 0 and st[name]["device_ms"] >= st[name]["trace_ms"]
        assert st[name]["h2d_bytes"] == n * 48 and st[name]["d2h_bytes"] == n * (8 + 4 + 24 + 24 + 16 + 1) + 256
    assert st["tree"]["candidates"] < 0.01 * n * m and st["tree"]["nodes"] > 0 and st["tree"]["clusters"] > 0
    assert st["exact"]["candidates"] == n * m


def test_device_form_refuses_host_pointers():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    try:
        o = np.zeros((4, 3)); d = np.ones((4, 3)); t = np.full(4, 7.0)
        do, dd, dt = dev(o), dev(d), torch.full((4,), 7.0, dtype=torch.float64, device="cuda")
        L = R.lib()
        for rays, hits, what in ((R.rt_rays(o.ctypes.data, dd.data_ptr(), None), R.rt_hits(dt.data_ptr(), None, None, None, None, None), "rays->origin"),
                                 (R.rt_rays(do.data_ptr(), d.ctypes.data, None), R.rt_hits(dt.data_ptr(), None, None, None, None, None), "rays->direction"),
                                 (R.rt_rays(do.data_ptr(), dd.data_ptr(), t.ctypes.data), R.rt_hits(dt.data_ptr(), None, None, None, None, None), "rays->t_max"),
                                 (R.rt_rays(do.data_ptr(), dd.data_ptr(), None), R.rt_hits(t.ctypes.data, None, None, None, None, None), "out->t")):
            assert L.rtb200_scene_intersect_device(rs.h, C.byref(rays), 4, C.byref(hits), None) == -1
            assert what.encode() in L.rtb200_last_error()
        torch.cuda.synchronize()
        assert (t == 7.0).all() and (dt.cpu().numpy() == 7.0).all()
        with pytest.raises(ValueError):
            rs.intersect(do, dd.float())
        with pytest.raises(ValueError):
            rs.intersect(o, d[:3])
        assert L.rtb200_scene_intersect_device(rs.h, C.byref(R.rt_rays(do.data_ptr(), dd.data_ptr(), None)), 4,
                                               C.byref(R.rt_hits()), None) == -1   # every output NULL
    finally:
        rs.release()


def test_stress_builds_answer_dense_and_rebuilt_queries_exactly(tmp_path):
    """Every stress build answers the 10k-sphere scene's queries, and the dense scenes' as uploaded and after rebuild(), bit
    for bit like the oracle; with the smallest lists the coincident spheres overflow the candidate list many times over."""
    from test_gpu_build_invariance import constants
    manifest = json.load(open(os.path.join(STRESS, "manifest.json")))
    sc = IW.c4_scene()
    o, d = IW.c4_rays(sc)
    want = IR.oracle(sc, o, d)
    wants = {}
    for name, (mk, rays, _) in IW.SETS.items():
        s = mk()
        so, sd = rays(s)
        wants[name] = IR.oracle(s, so, sd)
        assert (wants[name]["sphere"] >= 0).sum() > 1000, name
    for name in manifest:
        c = constants(manifest[name])
        out = tmp_path / f"{name}.npz"
        env = dict(os.environ, RTB200_LIB=os.path.join(STRESS, f"librtb200_{name}.so"))
        subprocess.run([sys.executable, os.path.join(REPO, "tests", "intersect_worker.py"), str(out)], env=env, check=True, timeout=900)
        z = np.load(out)
        meta = json.loads(str(z["meta"]))
        for v in ("filtered", "brute"):
            IR.assert_hits_equal({k: z[f"{v}.{k}"] for k in IR.FIELDS}, want, f"{name}/{v}")
            assert meta[v]["rays"] == len(o)
        for s, w in wants.items():
            IR.assert_hits_equal({k: z[f"{s}.{k}"] for k in IR.FIELDS}, w, f"{name}/{s}")
            assert meta[s]["rays"] == len(w["sphere"])
        assert meta["leaf_size"] == c["RT_LEAF_K"]
        if c["RT_CAP_CD"] == 32:
            for s in ("coincident", "coincident_rebuilt"):
                assert meta[s]["candidates"] / meta[s]["rays"] > c["RT_CAP_CD"], (name, s, meta[s])
