"""Auxiliary buffers of a resident scene's camera samples (ResidentScene.aov, rtb200_scene_aov[_device], DESIGN.md §4.14), held bit
for bit to oracle_aov: every variant under several sample counts and first samples; the sky modes, textures, lights and
non-finite albedos; shard and shared-memory handles; views; updates, rebuilds and edits against a fresh upload; the closest-hit
query of the same primary rays; ordering against updates on other streams; the host form's counters; refusals; the CLI's PNGs;
and the stress builds."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import intersect_rays as IR
import oracle_aov as OA
import rtb200 as R
from rtb200 import scenes
from test_aov_cpu import assert_f32_equal, mixed_lit_scene, textured_sky_scene
from test_gpu_intersect import AUTO, BRUTE, EXACT, FILTERED, REPO, STRESS, VARIANTS, _rtiow, _torch, dev
from test_gpu_scene_update import _jitter
from test_trace_rays_cpu import primary_rays

pytestmark = pytest.mark.gpu

CLI = os.path.join(REPO, "rust-raytracer_b200", "raytracer")


def assert_aov_equal(got, want, what, rows=None):
    """Every output `got` holds equals `want` (the oracle's whole frame, or its rows `rows`): albedo and normal bit for bit
    (NaN payloads free), hits and sphere equal, point bit for bit."""
    keys = [k for k, _, _ in R.AOV_FIELDS if k in got]
    assert keys, what
    for k in keys:
        g = np.asarray(got[k].cpu() if hasattr(got[k], "cpu") else got[k])
        w = want[k] if rows is None else want[k][rows]
        if k in ("albedo", "normal"):
            assert_f32_equal(g, w, f"{what}: {k}")
        elif k == "point":
            assert g.shape == w.shape and np.array_equal(g.view(np.uint64), w.view(np.uint64)), f"{what}: point"
        else:
            assert np.array_equal(g.view(np.int32), w.view(np.int32)), f"{what}: {k} differs in {int((g.view(np.int32) != w.view(np.int32)).sum())} pixels"


def scene_set():
    return {"cover": lambda: scenes.cover_scene(40, 30, 1), "textured_sky": textured_sky_scene, "mixed_lit": mixed_lit_scene}


# ---- the oracle, in every variant --------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", list(VARIANTS))
def test_every_variant_matches_the_oracle(variant):
    for name, mk in scene_set().items():
        sc = mk()
        rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
        try:
            for samples in (1, 4, 7):
                for sample0 in (0, 5):
                    got = rs.aov(samples, sample0=sample0)
                    assert_aov_equal(got, OA.aov(sc, samples, sample0), f"{name}/{variant}/{samples}@{sample0}")
                    assert got["stats"]["rays"] == got["stats"]["samples"] == sc.c.width * sc.c.height * samples
        finally:
            rs.release()


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_sphere_and_point_equal_the_query_of_the_primary_rays(variant):
    sc = mixed_lit_scene()
    rs = R.ResidentScene(sc, R.make_options(variant=VARIANTS[variant]))
    try:
        for s in (0, 5):
            got = rs.aov(3, sample0=s, outputs=("sphere", "point"))
            o, d = primary_rays(sc, s)
            q = rs.intersect(o, d, outputs=("sphere", "point"))
            assert np.array_equal(got["sphere"].reshape(-1), q["sphere"]), (variant, s)
            assert np.array_equal(got["point"].reshape(-1, 3).view(np.uint64), q["point"].view(np.uint64)), (variant, s)
            assert sorted(got) == ["point", "sphere", "stats"]
    finally:
        rs.release()


@pytest.mark.parametrize("sky", ["none", "gradient", "texture"])
def test_sky_modes_and_max_depth_zero(sky):
    if sky == "texture":
        sc = textured_sky_scene()
    else:
        cfg = scenes._variant(scenes.cover_config(), 32, 24, 1, 0)   # max_depth 0: the render is black, the AOVs are not
        if sky == "none":
            cfg["sky"] = None
        sc = R.Scene.from_config(cfg)
    rs = R.ResidentScene(sc)
    try:
        want = OA.aov(sc, 4, 2)
        assert_aov_equal(rs.aov(4, sample0=2), want, sky)
        assert (want["hits"] < 4).any()
        if sky == "none":
            assert (want["albedo"][want["hits"] == 0] == 0).all()
    finally:
        rs.release()


@pytest.mark.parametrize("name", ["always_list", "no_spheres", "c4_10k"])
def test_always_list_empty_and_many_spheres(name):
    if name == "always_list":
        from test_gpu_intersect import _always_scene
        sc = _always_scene()
    elif name == "no_spheres":
        sc, _ = IR.scene_of([])
    else:
        sc = _rtiow(50)
        sc.resize(64, 48, fix_aspect=True)
    want = OA.aov(sc, 2, 1)
    for v in (FILTERED, BRUTE, EXACT):
        rs = R.ResidentScene(sc, R.make_options(variant=v))
        try:
            assert_aov_equal(rs.aov(2, sample0=1), want, f"{name}/variant {v}")
        finally:
            rs.release()


# ---- shards, staged handles, views ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("rank,world,band_rows", [(0, 2, 1), (1, 2, 1), (2, 3, 4), (1, 4, 3), (5, 8, 8)])
def test_shard_rows_equal_the_full_handle(rank, world, band_rows):
    sc = textured_sky_scene(24, 30)
    rows = R.shard_row_indices(30, rank, world, band_rows)
    full = R.ResidentScene(sc)
    shard = R.ResidentScene(sc, R.make_options(rank=rank, world=world, band_rows=band_rows))
    try:
        want = full.aov(3, sample0=1)
        got = shard.aov(3, sample0=1)
        assert got["albedo"].shape[0] == len(rows)
        assert_aov_equal(got, want, f"shard {rank}/{world}/{band_rows}", rows)
        assert_aov_equal(got, OA.aov(sc, 3, 1), "shard vs the oracle", rows)
        dv = shard.aov(3, sample0=1, on_device=True)
        _torch().cuda.synchronize()
        assert_aov_equal(dv, want, "shard device form", rows)
    finally:
        full.release(); shard.release()


def test_shared_memory_staged_handle(monkeypatch):
    sc = mixed_lit_scene()
    monkeypatch.setenv("RTB200_WF_SMEM", "7")
    try:
        rs = R.ResidentScene(sc)
    finally:
        monkeypatch.delenv("RTB200_WF_SMEM")
    try:
        assert rs.kernel_info()["smem_mask"] == 7
        assert_aov_equal(rs.aov(4, sample0=5), OA.aov(sc, 4, 5), "staged")
    finally:
        rs.release()


def test_a_view_equals_a_fresh_upload_with_that_camera_and_seed():
    sc = textured_sky_scene(32, 24)
    view = R.make_frame(sc, look_from={"x": 4.0, "y": 2.5, "z": 2.0}, look_at={"x": 0.5, "y": 0.9, "z": 0.0}, vfov=60.0,
                        seed=987654321, max_depth=0)
    rs = R.ResidentScene(sc)
    try:
        got = rs.aov(3, sample0=2, view=view)
        moved = sc.edited()
        moved.c.camera = view.camera
        moved.seed = view.seed
        fresh = R.ResidentScene(moved)
        try:
            assert_aov_equal(got, fresh.aov(3, sample0=2), "view vs a fresh upload")
        finally:
            fresh.release()
        assert_aov_equal(got, OA.aov(sc, 3, 2, camera=view.camera, seed=view.seed), "view vs the oracle")
        assert_aov_equal(rs.aov(3, sample0=2), OA.aov(sc, 3, 2), "the handle's own view is unchanged")
    finally:
        rs.release()


# ---- updates, rebuilds and edits -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", ["filtered", "brute_force"])
def test_after_updates_rebuilds_and_edits_equal_a_fresh_upload(variant):
    torch = _torch()
    opts = R.make_options(variant=VARIANTS[variant])
    sc = scenes.cover_scene(40, 30, 1)
    rs = R.ResidentScene(sc, opts)
    rng = np.random.default_rng(90)

    def same_as_fresh(what):
        got = rs.aov(3, sample0=1)
        fresh = R.ResidentScene(sc, opts)
        try:
            want = fresh.aov(3, sample0=1)
        finally:
            fresh.release()
        assert_aov_equal(got, want, what)
        assert_aov_equal(got, OA.aov(sc, 3, 1), what + " vs the oracle")

    try:
        idx, recs = _jitter(sc, rng, 60)
        rs.update_spheres(idx, recs)
        same_as_fresh("update_spheres")
        c, r = IR.spheres_of(sc)
        c = c + rng.normal(size=c.shape) * 0.2
        c[0] = [0.0, -1000.0, 0.0]
        for i in range(sc.n_spheres):
            sc.set_sphere(i, center=c[i].tolist(), radius=float(r[i]))
        rs.update_geometry(torch.from_numpy(np.concatenate([c, r[:, None]], axis=1)).cuda())
        same_as_fresh("update_geometry")
        rs.rebuild()
        same_as_fresh("rebuild")
        ins = [R.make_sphere((0.0, 1.0, 0.0), 1.2, {"Light": {}}), R.make_sphere((-3.0, 0.8, 1.0), 0.8, {"Metal": {"albedo": [0.2, 0.4, 0.9], "fuzz": 0.1}})]
        rem = [3, 17, 40]
        rs.edit_spheres(remove=rem, insert=ins, at=[5, 100])
        sc = sc.edited(remove=rem, insert=ins, at=[5, 100])
        same_as_fresh("edit_spheres")
    finally:
        rs.release()


# ---- ordering, the device form -------------------------------------------------------------------------------------------

def test_device_form_sees_an_update_before_it_and_not_one_after_it():
    torch = _torch()
    sc = scenes.cover_scene(64, 48, 1)
    rs = R.ResidentScene(sc)
    try:
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        c0, r0 = IR.spheres_of(sc)
        c1 = c0 + np.array([0.0, 0.35, 0.0]); c1[0] = [0.0, -1000.0, 0.0]
        geo1 = torch.from_numpy(np.concatenate([c1, r0[:, None]], axis=1)).cuda()
        geo0 = torch.from_numpy(np.concatenate([c0, r0[:, None]], axis=1)).cuda()
        torch.cuda.synchronize()
        with torch.cuda.stream(a):
            big = torch.randn(4096, 4096, device="cuda")
            for _ in range(8):
                big = big @ big / 64.0   # keeps stream A busy so that the update runs late
            rs.update_geometry(geo1, stream=a)
        got = rs.aov(4, sample0=3, on_device=True, stream=b)
        rs.update_geometry(geo0, stream=a)   # enqueued after the pass: it must not change the pass's output
        torch.cuda.synchronize()
        for i in range(sc.n_spheres):
            sc.set_sphere(i, center=c1[i].tolist())
        assert_aov_equal(got, OA.aov(sc, 4, 3), "device form on B after an update on A")
        assert got["hits"].dtype == torch.uint32 and got["sphere"].dtype == torch.int32 and got["albedo"].shape == (48, 64, 3)
    finally:
        rs.release()


def test_host_form_counters_and_bytes():
    sc = mixed_lit_scene()
    npix = sc.c.width * sc.c.height
    rs = R.ResidentScene(sc)
    try:
        h = rs.aov(5, sample0=1)
        st = h["stats"]
        assert st["rays"] == st["samples"] == 5 * npix
        assert st["d2h_bytes"] == 256 + npix * (12 + 12 + 4 + 4 + 24) and st["h2d_bytes"] == 0
        assert st["kernel_launches"] == st["batches"] == st["frames"] == st["gpus_used"] == 1
        assert st["trace_ms"] > 0 and st["device_ms"] >= st["trace_ms"] and st["wall_ms"] > 0 and st["candidates"] > 0
        only = rs.aov(5, sample0=1, outputs=("hits", "normal"))
        assert sorted(only) == ["hits", "normal", "stats"]
        assert only["stats"]["d2h_bytes"] == 256 + npix * 16
        assert_aov_equal(only, OA.aov(sc, 5, 1), "two outputs")
    finally:
        rs.release()


def test_refusals_of_both_forms():
    torch = _torch()
    sc = scenes.cover_scene(16, 12, 1)
    rs = R.ResidentScene(sc)
    L = R.lib()
    try:
        host = np.full((12, 16, 3), 7.0, np.float32)
        dv = torch.full((12, 16, 3), 7.0, dtype=torch.float32, device="cuda")
        p = R.rt_aov_params(1, 0)
        assert L.rtb200_scene_aov_device(rs.h, C.byref(p), None, C.byref(R.rt_aov_out(host.ctypes.data)), None) == -1
        assert b"out->albedo" in L.rtb200_last_error()
        assert L.rtb200_scene_aov_device(rs.h, C.byref(p), None, C.byref(R.rt_aov_out(dv.data_ptr(), None, None, None, host.ctypes.data)), None) == -1
        assert b"out->point" in L.rtb200_last_error()
        torch.cuda.synchronize()
        assert (host == 7.0).all() and (dv.cpu().numpy() == 7.0).all()
        with pytest.raises(R.RtError):
            rs.aov(0)
        with pytest.raises(ValueError):
            rs.aov(1, outputs=("depth",))
        assert_aov_equal(rs.aov(2), OA.aov(sc, 2, 0), "after refusals")
    finally:
        rs.release()


# ---- the CLI -----------------------------------------------------------------------------------------------------------

def _to_u8(x):
    """The CLI's (and palette's) f32 -> u8: min(x * 255, 255) + 2^23, the low mantissa bits."""
    x = np.asarray(x, np.float32)
    with np.errstate(invalid="ignore"):
        scaled = np.fmin(x * np.float32(255), np.float32(255)).astype(np.float32)
    bits = (scaled + np.float32(8388608)).astype(np.float32).view(np.uint32)
    return np.where(bits >= 0x4B000000, bits - 0x4B000000, 0).astype(np.uint8)


def test_cli_writes_the_albedo_and_normal_pngs(tmp_path):
    from PIL import Image
    cfg = scenes._variant(scenes.cover_config(), 40, 30, 2, 8)
    p = tmp_path / "scene.json"; p.write_text(json.dumps(cfg))
    sc = R.Scene.from_config(cfg)
    out = tmp_path / "frame.png"
    env = dict(os.environ, RTB200_AOV="3,2", RTB200_SEED=str(sc.seed))
    r = subprocess.run([CLI, str(p), str(out)], capture_output=True, text=True, cwd=scenes.SCENES_DIR, env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    want = OA.aov(sc, 3, 2)
    albedo = np.asarray(Image.open(tmp_path / "frame_albedo.png").convert("RGB"))
    normal = np.asarray(Image.open(tmp_path / "frame_normal.png").convert("RGB"))
    assert np.array_equal(albedo, _to_u8(np.sqrt(want["albedo"])))
    assert np.array_equal(normal, _to_u8(np.float32(0.5) * want["normal"] + np.float32(0.5)))
    assert os.path.exists(out) and len(np.unique(normal.reshape(-1, 3), axis=0)) > 20
    for other in ("RTB200_GPUS", "RTB200_FRAMES", "RTB200_ADAPTIVE"):
        bad = subprocess.run([CLI, str(p), str(tmp_path / "x.png")], capture_output=True, text=True, env=dict(env, **{other: "1"}), timeout=60)
        assert bad.returncode == 101 and "RTB200_AOV" in bad.stderr, other


# ---- the stress builds ---------------------------------------------------------------------------------------------------

def test_stress_builds_match_the_oracle(tmp_path):
    """Every stress build gives the oracle's outputs on the worker's sets, and the lens oracle's on its lens sets."""
    import aov_worker as AW
    import oracle_lens as OL
    manifest = json.load(open(os.path.join(STRESS, "manifest.json")))

    def want(mk, samples, sample0):
        sc = mk()
        return OA.aov(sc, samples, sample0) if sc.lens is None else OL.aov_all(sc, sc.lens, samples, sample0)
    wants = {name: want(mk, samples, sample0) for name, (mk, samples, sample0, _) in AW.SETS.items()}
    assert sum(AW.SETS[name][0]().lens is not None for name in AW.SETS) == 2
    for build in manifest:
        out = tmp_path / f"{build}.npz"
        env = dict(os.environ, RTB200_LIB=os.path.join(STRESS, f"librtb200_{build}.so"))
        subprocess.run([sys.executable, os.path.join(REPO, "tests", "aov_worker.py"), str(out)], env=env, check=True, timeout=900)
        z = np.load(out)
        for name, w in wants.items():
            assert_aov_equal({k: z[f"{name}.{k}"] for k, _, _ in R.AOV_FIELDS}, w, f"{build}/{name}")
