"""The history clamp of the temporal accumulation on the GPU (rtb200_temporal_clamped[_device], rtb200.temporal(clamp=...),
TemporalDenoiser(clamp=...), DESIGN.md §4.20), held bit for bit to the numpy restatement in tests/temporal_clamp_restatement.py: edge
inputs for every camera pair and radius, random frames on an orbit step, C2's orbit pipeline through the device form, the host
form and the denoiser, overlapping calls on two streams, refusals that enqueue nothing, and the CLI's sixth field."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import denoise_restatement as DR
import temporal_clamp_restatement as TC
import temporal_restatement as TR
import rtb200 as R
from rtb200 import scenes
from test_gpu_intersect import _torch
from test_gpu_temporal import CLI, _cam
from test_temporal_cpu import BIG, CAMERA_PAIRS, assert_history_equal, dyadic_camera, edge_case, orbit_camera, orbit_frames

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
GAMMAS = (0.0, 0.5, 1.0, 3.0, 1e30)


def both_forms(color, sphere, point, cam, prev, what, motion=None, **kw):
    """The host and device forms of the clamped call against the clamped restatement."""
    torch = _torch()
    want = TC.temporal(color, sphere, point, cam, prev, motion=motion, **kw)
    rprev = None if prev is None else dict(prev, camera=_cam(prev["camera"]))
    h = R.temporal(color, sphere.view(np.int32), point, _cam(cam), rprev, motion=motion, **kw)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    dprev = None if prev is None else {"color": t(prev["color"]), "length": t(prev["length"]), "sphere": t(prev["sphere"].view(np.int32)),
                                       "point": t(prev["point"]), "camera": _cam(prev["camera"])}
    d = R.temporal(t(color), t(sphere.view(np.int32)), t(point), _cam(cam), dprev, motion=None if motion is None else t(motion), **kw)
    torch.cuda.synchronize()
    for form, out in (("host", h), ("device", {k: v.cpu().numpy() for k, v in d.items()})):
        assert_history_equal((out["color"], out["length"]), want, f"{what}/{form}")
    return h


@pytest.mark.parametrize("pair", list(CAMERA_PAIRS))
@pytest.mark.parametrize("radius", [1, 2, 3])
def test_edge_inputs(pair, radius):
    for w, h in ((1, 1), (1, 6), (6, 1), (2, 2), (9, 5), (17, 9), (65, 33)):
        for seed, (N, tol, mot) in enumerate([(8, 0.03, True), (2, 0.0, False), (BIG, 1e300, True)]):
            color, sphere, point, cam, prev, motion = edge_case(w, h, 100 * seed + w * h + radius, pcam=dyadic_camera(w, h, CAMERA_PAIRS[pair]))
            for gamma in GAMMAS:
                both_forms(color, sphere, point, cam, prev, f"{w}x{h}/{pair}/r={radius}/gamma={gamma}/N={N}", motion=motion if mot else None,
                           max_history=N, depth_tol=tol, clamp=gamma, clamp_radius=radius)


def test_overflowing_windows():
    """Colours near the f32 limit and of mixed sign: NaN and infinite window variances, on both forms."""
    w, h = 9, 5
    color, sphere, point, cam, prev, _ = edge_case(w, h, 7, pcam=dyadic_camera(w, h, (0.0, 0.0)), special=0.05)
    rng = np.random.default_rng(7)
    color[rng.random((h, w)) < 0.4] = F32(3e38)
    color[rng.random((h, w, 3)) < 0.3] *= F32(-1)
    prev["color"][rng.random((h, w)) < 0.3] = F32(2e38)
    for gamma in (0.0, 1.0):
        for radius in (1, 3):
            both_forms(color, sphere, point, cam, prev, f"overflow/gamma={gamma}/r={radius}", max_history=4, depth_tol=1e300, clamp=gamma,
                       clamp_radius=radius)


@pytest.mark.parametrize("w,h", [(801, 599), (1920, 1080)])
def test_random_frames_on_an_orbit_step(w, h):
    cam, pcam = orbit_camera(w, h, 11.0), orbit_camera(w, h, 10.0)
    color, sphere, point, _, prev, motion = edge_case(w, h, w, cam=cam, pcam=pcam, special=0.02)
    for radius in (1, 3):
        out = both_forms(color, sphere, point, cam, prev, f"{w}x{h}/r={radius}", motion=motion, max_history=R.TEMPORAL_MAX_HISTORY,
                         depth_tol=R.TEMPORAL_DEPTH_TOL, clamp=R.TEMPORAL_CLAMP_GAMMA, clamp_radius=radius)
        st = out["stats"]
        assert st["kernel_launches"] == 1 and st["trace_ms"] > 0
        assert st["h2d_bytes"] == w * h * 84 + 72 and st["d2h_bytes"] == w * h * 16


def test_c2_orbit_pipeline_is_the_same_through_every_form():
    """render_frames -> aov -> clamped accumulation -> denoise over an orbit of C2: the device form, the host form and
    TemporalDenoiser give the restatement's bytes."""
    torch = _torch()
    sc = scenes.scene("C2")
    sc.c.samples_per_pixel = 4
    frames = orbit_frames(sc, 6)
    w, h = int(sc.c.width), int(sc.c.height)
    kw = dict(max_history=R.TEMPORAL_MAX_HISTORY, depth_tol=R.TEMPORAL_DEPTH_TOL, clamp=R.TEMPORAL_CLAMP_GAMMA, clamp_radius=R.TEMPORAL_CLAMP_RADIUS)
    rs = R.ResidentScene(sc)
    try:
        lin = torch.empty((len(frames), h, w, 3), dtype=torch.float32, device="cuda")
        rs.render_frames(frames, 0, lin.data_ptr(), stream=torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY)
        aovs = [rs.aov(4, view=f, on_device=True, outputs=("albedo", "normal", "sphere", "point")) for f in frames]
        torch.cuda.synchronize()
    finally:
        rs.release()
    td = R.TemporalDenoiser(clamp=R.TEMPORAL_CLAMP_GAMMA, clamp_radius=R.TEMPORAL_CLAMP_RADIUS)
    prev = dprev = hprev = None
    lin_h = lin.cpu().numpy()
    changed = 0
    for i, f in enumerate(frames):
        a = aovs[i]
        ah = {k: v.cpu().numpy() for k, v in a.items()}
        want = TC.temporal(lin_h[i], ah["sphere"], ah["point"], f.camera, prev, **kw)
        plain = TR.temporal(lin_h[i], ah["sphere"], ah["point"], f.camera, prev, max_history=kw["max_history"], depth_tol=kw["depth_tol"])
        changed += int((want[0] != plain[0]).any(axis=2).sum())
        d = R.temporal(lin[i], a["sphere"], a["point"], f.camera, dprev, **kw)
        hh = R.temporal(lin_h[i], ah["sphere"], ah["point"], f.camera, hprev, **kw)
        o = td.push(lin[i], a, f)
        torch.cuda.synchronize()
        for form, got in (("device", (d["color"].cpu().numpy(), d["length"].cpu().numpy())), ("host", (hh["color"], hh["length"])),
                          ("denoiser", (o["color"].cpu().numpy(), o["length"].cpu().numpy()))):
            assert_history_equal(got, want, f"frame {i}/{form}")
        den = DR.denoise(want[0], ah["albedo"], ah["normal"], iterations=R.DENOISE_ITERATIONS, color_weight=R.DENOISE_COLOR_WEIGHT,
                         albedo_weight=R.DENOISE_ALBEDO_WEIGHT, normal_weight=R.DENOISE_NORMAL_WEIGHT)
        assert_history_equal((o["denoised"].cpu().numpy(), want[1]), (den, want[1]), f"frame {i}/denoised")
        prev = {"color": want[0], "length": want[1], "sphere": ah["sphere"], "point": ah["point"], "camera": f.camera}
        dprev = {"color": d["color"], "length": d["length"], "sphere": a["sphere"].clone(), "point": a["point"].clone(), "camera": f.camera}
        hprev = {"color": hh["color"], "length": hh["length"], "sphere": ah["sphere"], "point": ah["point"], "camera": f.camera}
    assert changed > 0, "the clamp changes some pixels of C2's orbit"


def test_overlapping_calls_on_two_streams_give_the_same_bytes():
    torch = _torch()
    w, h = 800, 600
    cam, pcam = orbit_camera(w, h, 11.0), orbit_camera(w, h, 10.0)
    color, sphere, point, _, prev, motion = edge_case(w, h, 5, cam=cam, pcam=pcam, special=0.02)
    kw = dict(max_history=6, depth_tol=0.02, clamp=0.75, clamp_radius=2)
    want = TC.temporal(color, sphere, point, cam, prev, motion=motion, **kw)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    args = (t(color), t(sphere.view(np.int32)), t(point), _cam(cam))
    dprev = {"color": t(prev["color"]), "length": t(prev["length"]), "sphere": t(prev["sphere"]), "point": t(prev["point"]), "camera": _cam(pcam)}
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [R.temporal(*args, dprev, motion=t(motion), stream=a if k % 2 == 0 else b, **kw) for k in range(6)]
    outs.append(R.temporal(*args, dprev, motion=t(motion), stream=R.CUDA_STREAM_LEGACY, **kw))
    torch.cuda.synchronize()
    for k, r in enumerate(outs):
        assert_history_equal((r["color"].cpu().numpy(), r["length"].cpu().numpy()), want, f"call {k}")


def test_refusals_enqueue_nothing():
    torch = _torch()
    L = R.lib()
    h, w = 12, 16
    n = h * w
    p = R.rt_temporal_params(w, h, 4, 0, R.rt_camera(), R.rt_camera(), 0.01)
    color = torch.rand((h, w, 3), device="cuda")
    sphere = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    point = torch.rand((h, w, 3), dtype=torch.float64, device="cuda")
    block = torch.full((n * 16,), 7, dtype=torch.uint8, device="cuda")
    oc, ol = block.data_ptr(), block.data_ptr() + n * 12
    host = np.full(n * 4, 7.0, F32)
    cur = R.rt_temporal_frame(color.data_ptr(), sphere.data_ptr(), point.data_ptr())
    out = R.rt_temporal_out(oc, ol)
    ok = R.rt_temporal_clamp(1.0, 1)
    cases = [
        ((ok, R.rt_temporal_frame(host.ctypes.data, sphere.data_ptr(), point.data_ptr()), out), b"cur.color is not device"),
        ((ok, cur, R.rt_temporal_out(host.ctypes.data, ol)), b"out.color is not device"),
        ((ok, cur, R.rt_temporal_out(color.data_ptr() + 8, ol)), b"overlaps cur.color"),
        ((None, cur, out), b"clamp is null"),
        ((R.rt_temporal_clamp(float("nan"), 1), cur, out), b"gamma"),
        ((R.rt_temporal_clamp(1.0, 4), cur, out), b"radius"),
    ]
    for (cl, c, o), what in cases:
        rc = L.rtb200_temporal_clamped_device(0, C.byref(p), C.byref(cl) if cl is not None else None, C.byref(c), None, None, C.byref(o), None)
        assert rc == -1 and what in L.rtb200_last_error(), (what, L.rtb200_last_error())
    torch.cuda.synchronize()
    assert (block.cpu().numpy() == 7).all() and (host == 7.0).all()
    with pytest.raises(R.RtError):
        R.temporal(color, sphere, point, R.rt_camera(), clamp=-1.0)
    with pytest.raises(R.RtError):
        R.temporal(color, sphere, point, R.rt_camera(), clamp=1.0, clamp_radius=0)


def test_cli_sixth_field_writes_the_clamped_denoised_frames(tmp_path):
    """RTB200_TEMPORAL with <clamp_gamma> writes the clamped accumulation's denoised frames and leaves the plain frames as they
    are; without it the denoised frames are the unclamped CLI's; a malformed gamma exits 101 before rendering."""
    from PIL import Image
    cfg = scenes._variant(scenes.cover_config(), 40, 30, 4, 8)
    p = tmp_path / "scene.json"; p.write_text(json.dumps(cfg))
    sc = R.Scene.from_config(cfg)
    frames = orbit_frames(sc, 5, step_deg=2.0)
    spec = [{"camera": {"look_from": {"x": f.camera.origin.x, "y": f.camera.origin.y, "z": f.camera.origin.z}, "look_at": cfg["camera"]["look_at"],
                        "vup": cfg["camera"]["vup"], "vfov": cfg["camera"]["vfov"], "aspect": cfg["camera"]["aspect"]}, "seed": int(f.seed)}
            for f in frames]
    fp = tmp_path / "frames.json"; fp.write_text(json.dumps(spec))
    env = dict(os.environ, RTB200_SEED=str(sc.seed), RTB200_FRAMES=str(fp))
    for k in ("RTB200_TEMPORAL", "RTB200_DENOISE", "RTB200_AOV", "RTB200_GPUS", "RTB200_ADAPTIVE"):
        env.pop(k, None)

    def run(prefix, spec_env):
        e = dict(env, RTB200_TEMPORAL=spec_env) if spec_env else env
        r = subprocess.run([CLI, str(p), str(tmp_path / prefix)], capture_output=True, text=True, cwd=scenes.SCENES_DIR, env=e, timeout=300)
        assert r.returncode == 0, r.stderr

    run("plain", None)
    run("unclamped", "3,2,8,2")
    rs = R.ResidentScene(sc)
    try:
        cams = [R.make_frame(sc, look_from=[f.camera.origin.x, f.camera.origin.y, f.camera.origin.z], seed=f.seed) for f in frames]
        lin, _ = R.render_frames(sc, cams, linear=True)
        aovs = [rs.aov(4, view=f) for f in cams]
    finally:
        rs.release()
    for spec_env, gamma in (("3,2,8,2,1,0.5", 0.5), ("3,2,8,2,1,0", 0.0)):
        run("clamped", spec_env)
        prev = None
        differs = False
        for i, f in enumerate(cams):
            assert (tmp_path / f"clamped_{i:03}.png").read_bytes() == (tmp_path / f"plain_{i:03}.png").read_bytes()
            a = aovs[i]
            c, n = TC.temporal(lin[i], a["sphere"], a["point"], f.camera, prev, max_history=3, depth_tol=R.TEMPORAL_DEPTH_TOL, clamp=gamma,
                               clamp_radius=R.TEMPORAL_CLAMP_RADIUS)
            prev = {"color": c, "length": n, "sphere": a["sphere"], "point": a["point"], "camera": f.camera}
            want = DR.denoise(c, a["albedo"], a["normal"], iterations=2, color_weight=8.0, albedo_weight=2.0, normal_weight=1.0)
            got = (tmp_path / f"clamped_{i:03}_denoised.png").read_bytes()
            assert np.array_equal(np.asarray(Image.open(tmp_path / f"clamped_{i:03}_denoised.png").convert("RGB")), DR.quantise(want)), (spec_env, i)
            differs = differs or got != (tmp_path / f"unclamped_{i:03}_denoised.png").read_bytes()
        assert differs, spec_env
    # the fields up to normal_weight alone are the unclamped accumulation, byte for byte
    run("five", "3,2,8,2,1")
    for i in range(len(cams)):
        assert (tmp_path / f"five_{i:03}_denoised.png").read_bytes() == (tmp_path / f"unclamped_{i:03}_denoised.png").read_bytes()
    for spec_env in ("3,2,8,2,1,-1", "3,2,8,2,1,nan", "3,2,8,2,1,inf", "3,2,8,2,1,1e39", "3,2,8,2,1,x", "3,2,8,2,1,0.5,1", "3,2,8,2,1,"):
        bad = subprocess.run([CLI, str(p), str(tmp_path / "bad")], capture_output=True, text=True, env=dict(env, RTB200_TEMPORAL=spec_env), timeout=60)
        assert bad.returncode == 101 and "RTB200_TEMPORAL" in bad.stderr, spec_env
        assert not list(tmp_path.glob("bad_*.png")), spec_env
