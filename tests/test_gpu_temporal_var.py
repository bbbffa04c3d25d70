"""The variance of each pixel's mean through the temporal accumulation on the GPU (rtb200_temporal_var[_device],
rtb200.temporal(variance=...), TemporalDenoiser(variance=True), DESIGN.md §4.21), held bit for bit to the numpy restatement in
tests/temporal_var_restatement.py: edge inputs for every camera pair and radius, clamped and not, random frames up to 1920x1080,
colour and length equal to the calls without the variance, a rendered orbit of C2 through every form and the denoiser, pushes on
two streams, refusals that enqueue nothing, and the CLI's RTB200_TEMPORAL_VAR."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import denoise_restatement as DR
import denoise_var_restatement as DV
import temporal_var_restatement as TV
import rtb200 as R
from rtb200 import scenes
from test_gpu_intersect import _torch
from test_gpu_temporal import CLI, _cam
from test_temporal_cpu import BIG, CAMERA_PAIRS, assert_history_equal, dyadic_camera, orbit_camera, orbit_frames
from test_temporal_var_cpu import assert_var_history_equal, var_case

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64


def both_forms(color, v, sphere, point, cam, prev, what, motion=None, **kw):
    """The host and device forms of the variance call against the restatement, and their colour and length against the call
    without the variance on the same inputs."""
    torch = _torch()
    want = TV.temporal(color, v, sphere, point, cam, prev, motion=motion, **kw)
    rprev = None if prev is None else dict(prev, camera=_cam(prev["camera"]))
    h = R.temporal(color, sphere.view(np.int32), point, _cam(cam), rprev, motion=motion, variance=v, **kw)
    plain = R.temporal(color, sphere.view(np.int32), point, _cam(cam), rprev, motion=motion, **kw)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    dprev = None if prev is None else {"color": t(prev["color"]), "length": t(prev["length"]), "sphere": t(prev["sphere"].view(np.int32)),
                                       "point": t(prev["point"]), "camera": _cam(prev["camera"]), "variance": t(prev["variance"])}
    d = R.temporal(t(color), t(sphere.view(np.int32)), t(point), _cam(cam), dprev, motion=None if motion is None else t(motion),
                   variance=t(v), **kw)
    torch.cuda.synchronize()
    for form, out in (("host", h), ("device", {k: x.cpu().numpy() for k, x in d.items()})):
        assert_var_history_equal((out["color"], out["length"], out["variance"]), want, f"{what}/{form}")
        assert_history_equal((out["color"], out["length"]), (plain["color"], plain["length"]), f"{what}/{form} without variance")
    return h


@pytest.mark.parametrize("pair", list(CAMERA_PAIRS))
@pytest.mark.parametrize("clamp,radius", [(None, 1), (0.0, 1), (0.5, 1), (1.0, 2), (1e30, 3)])
def test_edge_inputs(pair, clamp, radius):
    for w, h in ((1, 1), (1, 6), (6, 1), (2, 2), (9, 5), (17, 9), (65, 33)):
        for seed, (N, tol, mot) in enumerate([(8, 0.03, True), (2, 0.0, False), (1, 0.03, True), (BIG, 1e300, True)]):
            color, v, sphere, point, cam, prev, motion = var_case(w, h, 100 * seed + w * h + radius, pcam=dyadic_camera(w, h, CAMERA_PAIRS[pair]))
            both_forms(color, v, sphere, point, cam, prev, f"{w}x{h}/{pair}/clamp={clamp}/r={radius}/N={N}", motion=motion if mot else None,
                       max_history=N, depth_tol=tol, clamp=clamp, clamp_radius=radius)
    color, v, sphere, point, cam, prev, _ = var_case(9, 5, 1)
    both_forms(color, v, sphere, point, cam, None, f"no history/clamp={clamp}", max_history=4, depth_tol=0.03, clamp=clamp, clamp_radius=radius)


@pytest.mark.parametrize("w,h", [(801, 599), (1920, 1080)])
def test_random_frames_on_an_orbit_step(w, h):
    cam, pcam = orbit_camera(w, h, 11.0), orbit_camera(w, h, 10.0)
    color, v, sphere, point, _, prev, motion = var_case(w, h, w, cam=cam, pcam=pcam, special=0.02)
    for clamp, radius in ((None, 1), (R.TEMPORAL_CLAMP_GAMMA, 1), (R.TEMPORAL_CLAMP_GAMMA, 3)):
        out = both_forms(color, v, sphere, point, cam, prev, f"{w}x{h}/clamp={clamp}/r={radius}", motion=motion, max_history=4,
                         depth_tol=R.TEMPORAL_DEPTH_TOL, clamp=clamp, clamp_radius=radius)
        st = out["stats"]
        assert st["kernel_launches"] == 1 and st["trace_ms"] > 0
        assert st["h2d_bytes"] == w * h * 108 + 72 and st["d2h_bytes"] == w * h * 28


def _render_orbit(n, spp=4):
    torch = _torch()
    sc = scenes.scene("C2")
    sc.c.samples_per_pixel = spp
    frames = orbit_frames(sc, n)
    w, h = int(sc.c.width), int(sc.c.height)
    rs = R.ResidentScene(sc)
    try:
        lin = torch.empty((n, h, w, 3), dtype=torch.float32, device="cuda")
        var = torch.empty_like(lin)
        rs.render_frames(frames, 0, lin.data_ptr(), stream=torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY, variance=var.data_ptr())
        aovs = [rs.aov(spp, view=f, on_device=True, outputs=("albedo", "normal", "sphere", "point")) for f in frames]
        torch.cuda.synchronize()
    finally:
        rs.release()
    return frames, lin, var, aovs


@pytest.mark.parametrize("clamp", [None, R.TEMPORAL_CLAMP_GAMMA])
def test_c2_orbit_chain_is_the_restated_chain(clamp):
    """render_frames(variance) -> aov -> temporal with the variance over an orbit of C2: the device form, the host form and
    TemporalDenoiser(variance=True) give the restatement's bits, and the denoiser's denoised frame is denoise_var's of them."""
    torch = _torch()
    frames, lin, var, aovs = _render_orbit(5)
    kw = dict(max_history=4, depth_tol=R.TEMPORAL_DEPTH_TOL, clamp=clamp, clamp_radius=R.TEMPORAL_CLAMP_RADIUS)
    td = R.TemporalDenoiser(max_history=4, clamp=clamp, variance=True)
    prev = dprev = hprev = None
    lin_h, var_h = lin.cpu().numpy(), var.cpu().numpy()
    blended = 0
    for i, f in enumerate(frames):
        a = aovs[i]
        ah = {k: x.cpu().numpy() for k, x in a.items()}
        want = TV.temporal(lin_h[i], var_h[i], ah["sphere"], ah["point"], f.camera, prev, **kw)
        blended += int((want[1] >= 2).sum())
        d = R.temporal(lin[i], a["sphere"], a["point"], f.camera, dprev, variance=var[i], **kw)
        hh = R.temporal(lin_h[i], ah["sphere"], ah["point"], f.camera, hprev, variance=var_h[i], **kw)
        o = td.push(lin[i], a, f, variance=var[i])
        den = R.denoise_var(d["color"], d["variance"], a["albedo"], a["normal"])
        torch.cuda.synchronize()
        for form, got in (("device", (d["color"], d["length"], d["variance"])), ("host", (hh["color"], hh["length"], hh["variance"])),
                          ("denoiser", (o["color"], o["length"], o["variance"]))):
            got = tuple(x.cpu().numpy() if hasattr(x, "cpu") else x for x in got)
            assert_var_history_equal(got, want, f"frame {i}/{form}")
        assert torch.equal(o["denoised"].view(torch.int32), den["linear"].view(torch.int32)), f"frame {i}/denoised"
        prev = {"color": want[0], "length": want[1], "sphere": ah["sphere"], "point": ah["point"], "camera": f.camera, "variance": want[2]}
        dprev = {"color": d["color"], "length": d["length"], "sphere": a["sphere"].clone(), "point": a["point"].clone(), "camera": f.camera,
                 "variance": d["variance"]}
        hprev = {"color": hh["color"], "length": hh["length"], "sphere": ah["sphere"], "point": ah["point"], "camera": f.camera,
                 "variance": hh["variance"]}
    assert blended > 0
    # the last denoised frame against the filter's restatement
    ah = {k: x.cpu().numpy() for k, x in aovs[-1].items()}
    ref, _ = DV.denoise_var(want[0], want[2], ah["albedo"], ah["normal"], iterations=R.DENOISE_VAR_ITERATIONS,
                            color_weight=R.DENOISE_VAR_COLOR_WEIGHT, albedo_weight=R.DENOISE_VAR_ALBEDO_WEIGHT,
                            normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT, variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR)
    assert_history_equal((o["denoised"].cpu().numpy(), want[1]), (ref, want[1]), "last denoised frame")


def test_the_denoiser_on_two_streams_is_the_one_stream_chain():
    torch = _torch()
    frames, lin, var, aovs = _render_orbit(6)
    one, two = R.TemporalDenoiser(max_history=8, variance=True), R.TemporalDenoiser(max_history=8, variance=True)
    s = [torch.cuda.Stream(), torch.cuda.Stream()]
    for i, f in enumerate(frames):
        a = one.push(lin[i], aovs[i], f, variance=var[i])
        a = {k: x.clone() for k, x in a.items()}
        b = two.push(lin[i], aovs[i], f, variance=var[i], stream=s[i % 2])
        torch.cuda.synchronize()
        for k in ("color", "variance", "denoised"):
            assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), (i, k)
        assert torch.equal(a["length"], b["length"]), i


def test_refusals_enqueue_nothing():
    torch = _torch()
    L = R.lib()
    h, w = 12, 16
    n = h * w
    p = R.rt_temporal_params(w, h, 4, 0, R.rt_camera(), R.rt_camera(), 0.01)
    color = torch.rand((h, w, 3), device="cuda")
    var = torch.rand((h, w, 3), device="cuda")
    sphere = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    point = torch.rand((h, w, 3), dtype=torch.float64, device="cuda")
    block = torch.full((n * 28,), 7, dtype=torch.uint8, device="cuda")
    oc, ol, ov = block.data_ptr(), block.data_ptr() + n * 12, block.data_ptr() + n * 16
    host = np.full(n * 4, 7.0, F32)
    cur = R.rt_temporal_frame(color.data_ptr(), sphere.data_ptr(), point.data_ptr())
    out = R.rt_temporal_out(oc, ol)
    cases = [
        ((None, host.ctypes.data, ov), b"variance is not device"),
        ((None, var.data_ptr(), host.ctypes.data), b"out_variance is not device"),
        ((None, var.data_ptr(), var.data_ptr() + 8), b"out_variance overlaps variance"),
        ((None, var.data_ptr() + 2, ov), b"variance is not 4-byte aligned"),
        ((None, None, ov), b"variance is null"),
        ((R.rt_temporal_clamp(1.0, 4), var.data_ptr(), ov), b"radius"),
    ]
    for (cl, v, o), what in cases:
        rc = L.rtb200_temporal_var_device(0, C.byref(p), C.byref(cl) if cl is not None else None, C.byref(cur), v, None, None, None,
                                          C.byref(out), o, None)
        assert rc == -1 and what in L.rtb200_last_error(), (what, L.rtb200_last_error())
    torch.cuda.synchronize()
    assert (block.cpu().numpy() == 7).all() and (host == 7.0).all()


def test_cli_writes_the_variance_guided_accumulation(tmp_path):
    """RTB200_TEMPORAL_VAR writes each frame's accumulation with its variance, denoised by it, as the restated pipeline quantises
    it, clamped or not, and leaves the plain frames as the run without it writes them."""
    from PIL import Image
    cfg = scenes._variant(scenes.cover_config(), 40, 30, 4, 8)
    p = tmp_path / "scene.json"; p.write_text(json.dumps(cfg))
    sc = R.Scene.from_config(cfg)
    frames = orbit_frames(sc, 5, step_deg=2.0)
    spec = [{"camera": {"look_from": {"x": f.camera.origin.x, "y": f.camera.origin.y, "z": f.camera.origin.z}, "look_at": cfg["camera"]["look_at"],
                        "vup": cfg["camera"]["vup"], "vfov": cfg["camera"]["vfov"], "aspect": cfg["camera"]["aspect"]}, "seed": int(f.seed)}
            for f in frames]
    fp = tmp_path / "frames.json"; fp.write_text(json.dumps(spec))
    env = {k: v for k, v in os.environ.items() if not k.startswith("RTB200_")}
    env.update(RTB200_SEED=str(sc.seed), RTB200_FRAMES=str(fp))

    def run(prefix, spec_env):
        e = dict(env, RTB200_TEMPORAL_VAR=spec_env) if spec_env else env
        r = subprocess.run([CLI, str(p), str(tmp_path / prefix)], capture_output=True, text=True, cwd=scenes.SCENES_DIR, env=e, timeout=300)
        assert r.returncode == 0, r.stderr

    run("plain", None)
    rs = R.ResidentScene(sc)
    try:
        cams = [R.make_frame(sc, look_from=[f.camera.origin.x, f.camera.origin.y, f.camera.origin.z], seed=f.seed) for f in frames]
        lin, var, _ = R.render_frames(sc, cams, linear=True, variance=True)
        aovs = [rs.aov(4, view=f) for f in cams]
    finally:
        rs.release()
    for spec_env, N, dkw, clamp in (("3,2,2,3,0.5,1e-3", 3, dict(iterations=2, color_weight=2.0, albedo_weight=3.0, normal_weight=0.5,
                                                                    variance_floor=1e-3), None),
                                    ("4", 4, dict(iterations=R.DENOISE_VAR_ITERATIONS, color_weight=R.DENOISE_VAR_COLOR_WEIGHT,
                                                  albedo_weight=R.DENOISE_VAR_ALBEDO_WEIGHT, normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT,
                                                  variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR), None),
                                    ("4,2,1,4,1,1e-4,0.5", 4, dict(iterations=2, color_weight=1.0, albedo_weight=4.0, normal_weight=1.0,
                                                                   variance_floor=1e-4), 0.5),
                                    ("3,0", 3, None, None)):
        run("acc", spec_env)
        prev = None
        for i, f in enumerate(cams):
            assert (tmp_path / f"acc_{i:03}.png").read_bytes() == (tmp_path / f"plain_{i:03}.png").read_bytes()
            a = aovs[i]
            c, n, v = TV.temporal(lin[i], var[i], a["sphere"], a["point"], f.camera, prev, max_history=N, depth_tol=R.TEMPORAL_DEPTH_TOL,
                                  clamp=clamp, clamp_radius=R.TEMPORAL_CLAMP_RADIUS)
            prev = {"color": c, "length": n, "sphere": a["sphere"], "point": a["point"], "camera": f.camera, "variance": v}
            want = c if dkw is None else DV.denoise_var(c, v, a["albedo"], a["normal"], **dkw)[0]
            got = np.asarray(Image.open(tmp_path / f"acc_{i:03}_denoised.png").convert("RGB"))
            assert np.array_equal(got, DR.quantise(want)), (spec_env, i)
