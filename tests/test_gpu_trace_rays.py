"""Radiance of caller-supplied rays on a resident scene (ResidentScene.trace_rays, rtb200_scene_trace_rays[_device], DESIGN.md
§4.12), held bit for bit to the render and to the oracle: the render's own primary rays, one call per sample, reproduce the
render in every variant; arbitrary rays (the closest-hit tests' families, origins inside and on spheres, rays toward lights,
zero, subnormal, huge and non-finite components) equal oracle_trace_rays under every sample count, depth and sky; splitting
by rays, by batches and by sample0 changes nothing; edited, shard and shared-memory handles; ordering against frames and
updates; refusals and the host form's counters; the panorama tool; and the stress builds."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import intersect_rays as IR
import oracle_trace_rays as OT
import rtb200 as R
import trace_rays_worker as TW
from rtb200 import scenes
from synth import mixed_config
from test_gpu_intersect import AUTO, BRUTE, EXACT, FILTERED, REPO, STRESS, VARIANTS, _always_scene, _rtiow, _torch, dev
from test_gpu_scene_update import _jitter, _render
from test_gpu_shading_edges import assert_frames_match, scene_of, sky_config, synthetic_texture
from test_trace_rays_cpu import primary_rays, quantise, sum_samples

pytestmark = pytest.mark.gpu


def trace(rs, o, d, samples=1, stream=None, **kw):
    """The device form on CUDA tensors (numpy arrays are copied to the device first): {"linear", "rgb8"} as numpy arrays, and
    "stats"."""
    if isinstance(o, np.ndarray):
        o, d = dev(o), dev(d)
        _torch().cuda.synchronize()   # the copies are done before a call on another stream reads them
    h = rs.trace_rays(o, d, samples, linear=True, rgb8=True, stream=stream, **kw)
    return {"linear": h["linear"].cpu().numpy(), "rgb8": h["rgb8"].cpu().numpy(), "stats": h["stats"]}


def assert_same(got, want, what):
    """Linear bit for bit (NaN masks equal, payloads free), RGB8 equal."""
    assert_frames_match((got["linear"], got["rgb8"]), (want["linear"], want["rgb8"]), what)


def check(rs, sc, o, d, what, samples=1, **kw):
    got = trace(rs, o, d, samples, **kw)
    want = OT.trace_rays(sc, o, d, samples, **kw)
    assert_same(got, want, what)
    assert got["stats"]["rays"] == want["rays"], (what, got["stats"]["rays"], want["rays"])
    assert got["stats"]["samples"] == len(o) * samples
    return want


# ---- the render's primary rays reproduce the render ------------------------------------------------------------------

def _identity_scenes():
    return {"cover_40x30_s4": lambda: scenes.cover_scene(40, 30, 4),
            "test_scene_40x30_s4": lambda: R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 40, 30, 4, 12), scenes.SCENES_DIR),
            "mixed_48x36_s3": lambda: R.Scene.from_config(mixed_config(48, 36, 3, 12, seed=11), scenes.SCENES_DIR)}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", list(_identity_scenes()))
def test_render_rays_reproduce_the_render(name, variant):
    sc = _identity_scenes()[name]()
    w, h, spp = int(sc.c.width), int(sc.c.height), int(sc.c.samples_per_pixel)
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        img, lin, rays = _render(rs)
        per, n_rays = [], 0
        for s in range(spp):
            o, d = primary_rays(sc, s)
            got = trace(rs, o, d, 1, sample0=s)
            per.append(got["linear"]); n_rays += got["stats"]["rays"]
            assert np.array_equal(got["rgb8"], quantise(got["linear"]))
        mine = sum_samples(per, spp).reshape(h, w, 3)
        assert_frames_match((mine, quantise(mine)), (lin, img), f"{name}/{variant}")
        assert n_rays == rays
    finally:
        rs.release()


# ---- arbitrary rays against the oracle ---------------------------------------------------------------------------------

def extreme_rays(sc, rng):
    """Camera-like rays whose directions are scaled to 1e-300, 1e300 or carry subnormal, zero and non-finite components."""
    o, d = IR.box_rays(sc, rng, 64)
    parts = [(o, d * 1e-300), (o, d * 1e300), (o, np.where(rng.random(d.shape) < 0.5, 5e-324, d)), IR.degenerate_rays(sc, rng)]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def toward_lights(sc, rng, k):
    """From random points near the spheres, straight at the lights' centres (and just off them)."""
    c, r = IR.spheres_of(sc)
    lights = [i for i in range(sc.n_spheres) if sc._spheres[i].kind == R.RT_LIGHT]
    o, _ = IR.box_rays(sc, rng, k)
    j = np.array(lights)[rng.integers(0, len(lights), size=k)]
    return o, c[j] - o + rng.normal(size=(k, 3)) * 0.05 * np.abs(r[j])[:, None]


def ray_set(sc, rng, k=600):
    o, d = IR.camera_rays(sc, 32, 24)
    sets = [(o, d), IR.surface_rays(sc, rng, k), IR.box_rays(sc, rng, k), IR.grazing_rays(sc, rng, k // 2), IR.axis_rays(sc, rng, k // 2),
            extreme_rays(sc, rng)]
    if any(sc._spheres[i].kind == R.RT_LIGHT for i in range(sc.n_spheres)):
        sets.append(toward_lights(sc, rng, k))
    return np.concatenate([s[0] for s in sets]), np.concatenate([s[1] for s in sets])


def _sky_scene(kind):
    if kind == "texture":
        return scene_of(sky_config(24, 18, 1), sky=synthetic_texture(5, 3))
    cfg = scenes._variant(scenes.cover_config(), 24, 18, 1, 50)
    if kind == "none":
        cfg["sky"] = None
    return R.Scene.from_config(cfg)


@pytest.mark.parametrize("sky", ["none", "gradient", "texture"])
def test_arbitrary_rays_match_the_oracle_under_every_depth_and_sample_count(sky):
    sc = _sky_scene(sky)
    rng = np.random.default_rng(70)
    o, d = ray_set(sc, rng)
    rs = R.ResidentScene(sc)
    try:
        for m, depth in ((1, 50), (3, 0), (3, 1), (3, 2), (3, 50)):
            check(rs, sc, o, d, f"{sky}/m={m}/depth={depth}", m, max_depth=depth, sample0=m, stream0=depth)
        check(rs, sc, o[:500], d[:500], f"{sky}/m=64", 64, seed=12345)
    finally:
        rs.release()


def test_lit_textured_scene_in_every_variant():
    sc = R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 32, 24, 1, 12), scenes.SCENES_DIR)
    rng = np.random.default_rng(71)
    o, d = ray_set(sc, rng)
    for v in VARIANTS.values():
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            for m, depth in ((1, 12), (3, 2), (3, 50)):
                check(rs, sc, o, d, f"variant {v}/m={m}/depth={depth}", m, max_depth=depth)
        finally:
            rs.release()


@pytest.mark.parametrize("name", ["always_list", "no_spheres", "c4_10k"])
def test_always_list_empty_and_many_spheres(name):
    rng = np.random.default_rng(72)
    if name == "always_list":
        sc = _always_scene()
    elif name == "no_spheres":
        sc, _ = IR.scene_of([])
    else:
        sc = _rtiow(50)
    o, d = IR.camera_rays(sc, 32, 24)
    parts = [(o, d), extreme_rays(sc, rng)] + ([IR.surface_rays(sc, rng, 400), IR.box_rays(sc, rng, 400)] if sc.n_spheres else [])
    o = np.concatenate([p[0] for p in parts]); d = np.concatenate([p[1] for p in parts])
    for v in (FILTERED, BRUTE, EXACT):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            check(rs, sc, o, d, f"{name}/variant {v}", 2)
        finally:
            rs.release()


@pytest.mark.parametrize("n", [1, 31, 33, 100_000])
def test_launch_sizes(n):
    sc = scenes.cover_scene(32, 24, 1)
    rng = np.random.default_rng(73)
    o, d = IR.box_rays(sc, rng, n)
    rs = R.ResidentScene(sc)
    try:
        check(rs, sc, o, d, f"n={n}", 2)
    finally:
        rs.release()


# ---- splitting is exact ------------------------------------------------------------------------------------------------

def test_splitting_by_rays_batches_and_sample0():
    sc = scenes.cover_scene(32, 24, 1)
    rng = np.random.default_rng(74)
    o, d = ray_set(sc, rng)
    n = len(o)
    rs = R.ResidentScene(sc)
    small = R.ResidentScene(sc, R.make_options(sample_buffer_bytes=n * 16 * 5))
    try:
        whole = trace(rs, o, d, 12, sample0=3, stream0=11)
        k = n // 3
        a = trace(rs, o[:k], d[:k], 12, sample0=3, stream0=11)
        b = trace(rs, o[k:], d[k:], 12, sample0=3, stream0=11 + k)
        assert_same({"linear": np.concatenate([a["linear"], b["linear"]]), "rgb8": np.concatenate([a["rgb8"], b["rgb8"]])}, whole, "stream0 split")
        assert a["stats"]["rays"] + b["stats"]["rays"] == whole["stats"]["rays"]
        batched = trace(small, o, d, 12, sample0=3, stream0=11)
        assert batched["stats"]["batches"] == 3 and whole["stats"]["batches"] == 1
        assert batched["stats"]["kernel_launches"] == 6
        assert_same(batched, whole, "batches of 5 samples")
        assert batched["stats"]["rays"] == whole["stats"]["rays"]
        parts = [trace(rs, o, d, 1, sample0=3 + j, stream0=11)["linear"] for j in range(12)]
        want = sum_samples(parts, 12)
        assert_same(whole, {"linear": want, "rgb8": quantise(want)}, "sample0 shifts")
        check(rs, sc, o, d, "sample0 = 3", 12, sample0=3, stream0=11)
        tiny = R.ResidentScene(sc, R.make_options(sample_buffer_bytes=n * 16 - 16))
        try:
            with pytest.raises(R.RtError, match="sample-buffer cap"):
                tiny.trace_rays(o, d)
            check(tiny, sc, o[:-1], d[:-1], "one sample of every ray fills the cap", 3)
        finally:
            tiny.release()
    finally:
        rs.release(); small.release()


# ---- edited scenes and other handles -----------------------------------------------------------------------------------

@pytest.mark.parametrize("handle", ["plain", "shard", "wf_smem"])
def test_edited_scenes_equal_a_fresh_upload(handle, monkeypatch):
    torch = _torch()
    sc = scenes.cover_scene(48, 36, 1)
    opts = R.make_options(rank=1, world=2) if handle == "shard" else None
    if handle == "wf_smem":
        monkeypatch.setenv("RTB200_WF_SMEM", "7")
    rs = R.ResidentScene(sc, opts)
    rng = np.random.default_rng(75)
    o, d = ray_set(sc, rng, 400)

    def same_as_fresh(what):
        got = trace(rs, o, d, 3)
        fresh = R.ResidentScene(sc, opts)
        try:
            want = trace(fresh, o, d, 3)
        finally:
            fresh.release()
        assert_same(got, want, what)
        assert got["stats"]["rays"] == want["stats"]["rays"]
        assert_same(got, OT.trace_rays(sc, o, d, 3), what + " vs the oracle")

    try:
        if handle == "wf_smem":
            assert rs.kernel_info()["smem_mask"] == 7
        same_as_fresh(f"{handle}/uploaded")
        idx, recs = _jitter(sc, rng, 60)
        rs.update_spheres(idx, recs)
        same_as_fresh(f"{handle}/update_spheres")
        c, r = IR.spheres_of(sc)
        c = c + rng.normal(size=c.shape) * 0.2
        c[0] = [0.0, -1000.0, 0.0]
        for i in range(sc.n_spheres):
            sc.set_sphere(i, center=c[i].tolist(), radius=float(r[i]))
        rs.update_geometry(torch.from_numpy(np.concatenate([c, r[:, None]], axis=1)).cuda())
        same_as_fresh(f"{handle}/update_geometry")
        if handle != "wf_smem":   # a staged hierarchy refuses a rebuild
            rs.rebuild()
            same_as_fresh(f"{handle}/rebuild")
    finally:
        monkeypatch.delenv("RTB200_WF_SMEM", raising=False)
        rs.release()


# ---- ordering ----------------------------------------------------------------------------------------------------------

def test_interleaved_with_async_frames_on_two_streams():
    torch = _torch()
    sc = scenes.cover_scene(48, 36, 4)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(76)
    o, d = ray_set(sc, rng, 400)
    want = OT.trace_rays(sc, o, d, 4)
    n = 48 * 36 * 3
    try:
        img0, lin0, rays0 = _render(rs)
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        outs, got = [], []
        for k in range(4):
            d8 = torch.zeros(n, dtype=torch.uint8, device="cuda"); dl = torch.zeros(n, dtype=torch.float32, device="cuda")
            rs.render_async(d8.data_ptr(), dl.data_ptr(), stream=(a if k % 2 else b).cuda_stream)
            outs.append((d8, dl))
            got.append(trace(rs, o, d, 4, stream=b if k % 2 else a))
        rs.wait()
        torch.cuda.synchronize()
        for d8, dl in outs:
            assert_frames_match((dl.cpu().numpy().reshape(36, 48, 3), d8.cpu().numpy().reshape(36, 48, 3)), (lin0, img0), "async frame")
        for g in got:
            assert_same(g, want, "trace_rays beside frames")
        img1, lin1, rays1 = _render(rs)
        assert np.array_equal(img0, img1) and np.array_equal(lin0.view(np.uint32), lin1.view(np.uint32)) and rays0 == rays1
    finally:
        rs.release()


def test_sees_an_update_enqueued_before_it_on_another_stream():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    o, d = IR.camera_rays(sc, 64, 48)
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
        got = trace(rs, do, dd, 2, stream=b)
        assert_same(got, OT.trace_rays(sc, o, d, 2), "trace_rays on B after an update on A")
    finally:
        rs.release()


# ---- refusals and the host form ----------------------------------------------------------------------------------------

def test_host_form_counters_and_bytes():
    sc = R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 32, 24, 1, 12), scenes.SCENES_DIR)
    rng = np.random.default_rng(77)
    o, d = ray_set(sc, rng)
    n = len(o)
    want = OT.trace_rays(sc, o, d, 3)
    rs = R.ResidentScene(sc)
    try:
        h = rs.trace_rays(o, d, 3, rgb8=True)
        assert_same(h, want, "host form")
        st = h["stats"]
        assert st["rays"] == want["rays"] and st["samples"] == 3 * n and st["frames"] == 1
        assert st["h2d_bytes"] == 48 * n and st["d2h_bytes"] == 15 * n
        assert st["kernel_launches"] == 2 and st["batches"] == 1 and st["trace_ms"] > 0 and st["device_ms"] >= st["trace_ms"]
        only8 = rs.trace_rays(o, d, 3, linear=False, rgb8=True)
        assert sorted(only8) == ["rgb8", "stats"] and np.array_equal(only8["rgb8"], want["rgb8"])
        assert only8["stats"]["d2h_bytes"] == 3 * n
        dv = trace(rs, o, d, 3)
        assert_same(dv, want, "device form")
        z = rs.trace_rays(o, d, 2, max_depth=0, rgb8=True)
        assert (z["linear"] == 0).all() and (z["rgb8"] == 0).all() and z["stats"]["rays"] == 0 and z["stats"]["samples"] == 2 * n
        e = rs.trace_rays(o[:0], d[:0])
        assert e["linear"].shape == (0, 3)
    finally:
        rs.release()


def test_refusals_of_both_forms():
    torch = _torch()
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    L = R.lib()
    try:
        o = np.zeros((4, 3)); d = np.ones((4, 3)); t = np.ones(4)
        do, dd = dev(o), dev(d)
        dl = torch.full((4, 3), 7.0, dtype=torch.float32, device="cuda")
        hl = np.full((4, 3), 7.0, np.float32)
        p = R.rt_trace_params(1, 1, 0, 0, 4)
        st = R.rt_stats()
        for rays, lin, what in ((R.rt_rays(o.ctypes.data, dd.data_ptr(), None), dl.data_ptr(), "rays->origin"),
                                (R.rt_rays(do.data_ptr(), d.ctypes.data, None), dl.data_ptr(), "rays->direction"),
                                (R.rt_rays(do.data_ptr(), dd.data_ptr(), None), hl.ctypes.data, "dev_linear_f32")):
            assert L.rtb200_scene_trace_rays_device(rs.h, C.byref(rays), 4, C.byref(p), lin, None, None, C.byref(st)) == -1
            assert what.encode() in L.rtb200_last_error()
        rays = R.rt_rays(do.data_ptr(), dd.data_ptr(), None)
        assert L.rtb200_scene_trace_rays_device(rs.h, C.byref(rays), 4, C.byref(p), None, hl.ctypes.data, None, C.byref(st)) == -1
        assert b"dev_rgb8" in L.rtb200_last_error()
        bad = R.rt_rays(do.data_ptr(), dd.data_ptr(), dev(t).data_ptr())
        assert L.rtb200_scene_trace_rays_device(rs.h, C.byref(bad), 4, C.byref(p), dl.data_ptr(), None, None, C.byref(st)) == -1
        assert b"t_max" in L.rtb200_last_error()
        q = R.rt_trace_params(1, 0, 0, 0, 4)
        assert L.rtb200_scene_trace_rays(rs.h, C.byref(R.rt_rays(o.ctypes.data, d.ctypes.data, None)), 4, C.byref(q), hl.ctypes.data, None, C.byref(st)) == -1
        assert b"samples" in L.rtb200_last_error()
        torch.cuda.synchronize()
        assert (hl == 7.0).all() and (dl.cpu().numpy() == 7.0).all()
        with pytest.raises(ValueError):
            rs.trace_rays(do, dd.float())
        with pytest.raises(ValueError):
            rs.trace_rays(o, d[:3])
        with pytest.raises(ValueError):
            rs.trace_rays(o, d, linear=False)
        # the handle still works
        check(rs, sc, *IR.camera_rays(sc, 16, 12), "after refusals", 2)
    finally:
        rs.release()


# ---- the panorama tool -------------------------------------------------------------------------------------------------

def test_panorama_tool_writes_the_oracle_image(tmp_path):
    from PIL import Image
    sys.path.insert(0, os.path.join(REPO, "tools"))
    import panorama
    path = os.path.join(REPO, "scenes", "cover_scene.json.gz")
    out = tmp_path / "pano.png"
    subprocess.run([sys.executable, os.path.join(REPO, "tools", "panorama.py"), path, str(out), "--width", "64", "--samples", "2",
                    "--at", "0,1.5,0"], check=True, timeout=300)
    png = np.asarray(Image.open(out).convert("RGB"))
    assert png.shape == (32, 64, 3)
    o, d = panorama.equirect_rays(64, 32, (0.0, 1.5, 0.0))
    sc = R.load_scene(path)
    want = OT.trace_rays(sc, o.cpu().numpy(), d.cpu().numpy(), 2)
    assert np.array_equal(png.reshape(-1, 3), want["rgb8"])
    assert len(np.unique(png.reshape(-1, 3), axis=0)) > 50   # sky, ground and spheres, not a flat image


# ---- the stress builds -------------------------------------------------------------------------------------------------

def test_stress_builds_trace_rays_exactly(tmp_path):
    """Every stress build gives the oracle's outputs and ray counts on the worker's sets."""
    manifest = json.load(open(os.path.join(STRESS, "manifest.json")))
    wants = {}
    for name, (mk, calls, _) in TW.SETS.items():
        sc = mk()
        for k, (o, d, kw) in enumerate(calls(sc)):
            wants[f"{name}.{k}"] = OT.trace_rays(sc, o, d, **kw)
    for build in manifest:
        out = tmp_path / f"{build}.npz"
        env = dict(os.environ, RTB200_LIB=os.path.join(STRESS, f"librtb200_{build}.so"))
        subprocess.run([sys.executable, os.path.join(REPO, "tests", "trace_rays_worker.py"), str(out)], env=env, check=True, timeout=900)
        z = np.load(out)
        meta = json.loads(str(z["meta"]))
        for key, w in wants.items():
            assert_same({"linear": z[f"{key}.linear"], "rgb8": z[f"{key}.rgb8"]}, w, f"{build}/{key}")
            assert meta[key] == w["rays"], (build, key)
