"""Temporal accumulation on the GPU (rtb200.temporal, rtb200_temporal[_device], TemporalDenoiser, DESIGN.md §4.16), held bit for
bit to the numpy restatement in tests/temporal_restatement.py: edge inputs, random frames up to 1920x1080, the render_frames ->
aov -> temporal -> denoise pipeline over an orbit of C2 in every variant, moving spheres with and without their motion,
overlapping calls on two streams, refusals that enqueue nothing, and the CLI's _NNN_denoised.png files."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import denoise_restatement as DR
import temporal_restatement as TR
import rtb200 as R
from rtb200 import scenes
from test_gpu_intersect import REPO, VARIANTS, _torch
from test_temporal_cpu import BIG, CAMERA_PAIRS, assert_history_equal, dyadic_camera, edge_case, orbit_camera, orbit_frames

pytestmark = pytest.mark.gpu

CLI = os.path.join(REPO, "rust-raytracer_b200", "raytracer")
F32, F64 = np.float32, np.float64


def _cam(c):
    """An rt_camera of a restatement camera tuple."""
    if isinstance(c, R.rt_camera):
        return c
    return R.rt_camera(*(R.vec3(v.tolist()) for v in c))


def both_forms(color, sphere, point, cam, prev, what, motion=None, **kw):
    """The host and device forms against the restatement."""
    torch = _torch()
    want = TR.temporal(color, sphere, point, cam, prev, motion=motion, **kw)
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


# ---- the restatement ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("pair", list(CAMERA_PAIRS))
def test_edge_inputs(pair):
    for w, h in ((1, 1), (1, 2), (2, 1), (2, 2), (5, 3), (9, 5), (17, 9), (65, 33)):
        for seed, (N, tol, mot) in enumerate([(8, 0.03, True), (1, 0.03, False), (2, 0.0, True), (BIG, 1e300, False), (5, 0.5, True)]):
            color, sphere, point, cam, prev, motion = edge_case(w, h, 100 * seed + w * h, pcam=dyadic_camera(w, h, CAMERA_PAIRS[pair]))
            both_forms(color, sphere, point, cam, prev, f"{w}x{h}/{pair}/N={N}", motion=motion if mot else None, max_history=N, depth_tol=tol)
    color, sphere, point, cam, _, _ = edge_case(9, 5, 1)
    h = both_forms(color, sphere, point, cam, None, "no history", max_history=4, depth_tol=0.01)
    assert (h["length"] == 1).all()


@pytest.mark.parametrize("w,h", [(801, 599), (1920, 1080)])
def test_random_frames_on_an_orbit_step(w, h):
    cam, pcam = orbit_camera(w, h, 11.0), orbit_camera(w, h, 10.0)
    color, sphere, point, _, prev, motion = edge_case(w, h, w, cam=cam, pcam=pcam, special=0.02)
    out = both_forms(color, sphere, point, cam, prev, f"{w}x{h}", motion=motion, max_history=R.TEMPORAL_MAX_HISTORY,
                     depth_tol=R.TEMPORAL_DEPTH_TOL)
    st = out["stats"]
    assert st["kernel_launches"] == 1 and st["trace_ms"] > 0 and st["device_ms"] >= st["trace_ms"]
    assert st["h2d_bytes"] == w * h * 84 + 72 and st["d2h_bytes"] == w * h * 16


# ---- the pipeline ------------------------------------------------------------------------------------------------------

def _orbit_pipeline(sc, frames, variant):
    """render_frames (linear) -> aov(view = frame) -> TemporalDenoiser.push per frame, all on the device."""
    torch = _torch()
    w, h = int(sc.c.width), int(sc.c.height)
    rs = R.ResidentScene(sc, R.make_options(variant=variant))
    try:
        lin = torch.empty((len(frames), h, w, 3), dtype=torch.float32, device="cuda")
        rs.render_frames(frames, 0, lin.data_ptr(), stream=torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY)
        td = R.TemporalDenoiser()
        outs, aovs = [], []
        for i, f in enumerate(frames):
            aov = rs.aov(int(sc.c.samples_per_pixel), view=f, on_device=True, outputs=("albedo", "normal", "sphere", "point"))
            o = td.push(lin[i], aov, f)
            outs.append({k: v.cpu().numpy() for k, v in o.items()})
            aovs.append({k: v.cpu().numpy() for k, v in aov.items()})
        torch.cuda.synchronize()
        return outs, lin.cpu().numpy(), aovs
    finally:
        rs.release()


def _restated_pipeline(lin, aovs, frames, motions=None, max_history=R.TEMPORAL_MAX_HISTORY):
    prev, outs = None, []
    for i, f in enumerate(frames):
        a = aovs[i]
        c, n = TR.temporal(lin[i], a["sphere"], a["point"], f.camera, prev, motion=None if motions is None else motions[i],
                           max_history=max_history, depth_tol=R.TEMPORAL_DEPTH_TOL)
        prev = {"color": c, "length": n, "sphere": a["sphere"], "point": a["point"], "camera": f.camera}
        den = DR.denoise(c, a["albedo"], a["normal"], iterations=R.DENOISE_ITERATIONS, color_weight=R.DENOISE_COLOR_WEIGHT,
                         albedo_weight=R.DENOISE_ALBEDO_WEIGHT, normal_weight=R.DENOISE_NORMAL_WEIGHT)
        outs.append((c, n, den))
    return outs


def test_c2_orbit_pipeline_is_the_same_in_every_variant():
    sc = scenes.scene("C2")
    sc.c.samples_per_pixel = 4
    frames = orbit_frames(sc, 8)
    ref = None
    for name, v in VARIANTS.items():
        outs, lin, aovs = _orbit_pipeline(sc, frames, v)
        if ref is None:
            for i, (c, n, den) in enumerate(_restated_pipeline(lin, aovs, frames)):
                assert_history_equal((outs[i]["color"], outs[i]["length"]), (c, n), f"C2/{name}/frame {i}")
                assert_history_equal((outs[i]["denoised"], n), (den, n), f"C2/{name}/frame {i} denoised")
            assert (outs[-1]["length"] > 1).mean() > 0.25, "pixels keep a history on a slow orbit"
            ref = (outs, lin)
            continue
        assert np.array_equal(lin.view(np.uint32), ref[1].view(np.uint32)), name
        for i in range(len(frames)):
            for k in ("color", "length", "denoised"):
                assert np.array_equal(outs[i][k].view(np.uint32), ref[0][i][k].view(np.uint32)), (name, i, k)


def test_the_denoiser_ping_pongs_its_own_history_buffers_across_streams():
    """TemporalDenoiser owns two history buffers: pushes on alternating streams equal the restatement, a push's "color" and
    "length" are left as they were by the next push, and the push after that writes the same buffer again."""
    torch = _torch()
    sc = scenes.cover_scene(160, 120, 4)
    frames = orbit_frames(sc, 5)
    rs = R.ResidentScene(sc)
    try:
        lin = torch.empty((len(frames), 120, 160, 3), dtype=torch.float32, device="cuda")
        rs.render_frames(frames, 0, lin.data_ptr(), stream=torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY)
        aovs = [rs.aov(4, view=f, on_device=True, outputs=("albedo", "normal", "sphere", "point")) for f in frames]
        torch.cuda.synchronize()
    finally:
        rs.release()
    want = _restated_pipeline(lin.cpu().numpy(), [{k: v.cpu().numpy() for k, v in a.items()} for a in aovs], frames)
    streams = (torch.cuda.Stream(), torch.cuda.Stream())
    td = R.TemporalDenoiser()
    outs, snaps = [], []
    for i, f in enumerate(frames):
        outs.append(td.push(lin[i], aovs[i], f, stream=streams[i % 2]))
        streams[i % 2].synchronize()
        if snaps:   # this push read the previous push's output as its history and did not write it
            assert torch.equal(outs[-2]["color"].view(torch.int32), snaps[-1][0]) and torch.equal(outs[-2]["length"], snaps[-1][1]), i
        snaps.append((outs[-1]["color"].view(torch.int32).clone(), outs[-1]["length"].clone()))
        c, n, den = want[i]
        assert_history_equal((outs[-1]["color"].cpu().numpy(), outs[-1]["length"].cpu().numpy()), (c, n), f"push {i}")
        assert_history_equal((outs[-1]["denoised"].cpu().numpy(), n), (den, n), f"push {i} denoised")
    assert outs[2]["color"].data_ptr() == outs[0]["color"].data_ptr() != outs[1]["color"].data_ptr()
    td.reset()
    o = td.push(lin[0], aovs[0], frames[0])
    torch.cuda.synchronize()
    assert (o["length"].cpu().numpy() == 1).all()


def test_moving_spheres_keep_their_history_with_their_motion():
    """A sphere moved by update_geometry between frames: both with and without its motion the device equals the restatement, and
    more of the moving sphere's pixels keep their history with the motion than without."""
    torch = _torch()
    sc = scenes.cover_scene(160, 120, 4)
    frames = orbit_frames(sc, 6, step_deg=0.0)                          # a static camera: only the sphere moves
    centres = np.array([[s.center.x, s.center.y, s.center.z, s.radius] for s in sc._spheres[: sc.n_spheres]], F64)
    rs = R.ResidentScene(sc)
    try:
        first = rs.aov(4, view=frames[0], outputs=("sphere",))["sphere"]
        ids, counts = np.unique(first[first >= 0], return_counts=True)
        small = [(c, i) for i, c in zip(ids, counts) if centres[i, 3] < 10]
        j = max(small)[1]                                                # the smallest-radius sphere with the most pixels
        step = np.array([0.04, 0.0, 0.03], F64)
        lin, aovs, motions = [], [], []
        for i, f in enumerate(frames):
            geo = centres.copy()
            geo[j, :3] += step * i
            rs.update_geometry(torch.from_numpy(geo).cuda())
            out = torch.empty((120, 160, 3), dtype=torch.float32, device="cuda")
            rs.render_frames([f], 0, out.data_ptr(), stream=torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY)
            aov = rs.aov(4, view=f, on_device=True, outputs=("albedo", "normal", "sphere", "point"))
            torch.cuda.synchronize()
            lin.append(out.cpu().numpy())
            aovs.append({k: v.cpu().numpy() for k, v in aov.items()})
            m = np.zeros((sc.n_spheres, 3), F64)
            if i:
                m[j] = step
            motions.append(m)
    finally:
        rs.release()
    kept = {}
    for with_motion in (True, False):
        prev, dprev, n_kept = None, None, 0
        for i, f in enumerate(frames):
            a = aovs[i]
            mot = motions[i] if with_motion else None
            c, n = TR.temporal(lin[i], a["sphere"], a["point"], f.camera, prev, motion=mot, max_history=8, depth_tol=R.TEMPORAL_DEPTH_TOL)
            t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()  # noqa: E731
            d = R.temporal(t(lin[i]), t(a["sphere"]), t(a["point"]), f.camera, dprev, motion=None if mot is None else t(mot), max_history=8,
                           depth_tol=R.TEMPORAL_DEPTH_TOL)
            torch.cuda.synchronize()
            assert_history_equal((d["color"].cpu().numpy(), d["length"].cpu().numpy()), (c, n), f"motion={with_motion}/frame {i}")
            prev = {"color": c, "length": n, "sphere": a["sphere"], "point": a["point"], "camera": f.camera}
            dprev = {"color": d["color"], "length": d["length"], "sphere": t(a["sphere"]), "point": t(a["point"]), "camera": f.camera}
            if i:
                n_kept += int(((a["sphere"] == j) & (n > 1)).sum())
        kept[with_motion] = n_kept
    print(f"pixels of the moving sphere that kept their history: with motion {kept[True]}, without {kept[False]}")
    assert kept[True] > kept[False]


# ---- streams and refusals ----------------------------------------------------------------------------------------------

def test_overlapping_calls_on_two_streams_give_the_same_bytes():
    torch = _torch()
    w, h = 800, 600
    cam, pcam = orbit_camera(w, h, 11.0), orbit_camera(w, h, 10.0)
    color, sphere, point, _, prev, motion = edge_case(w, h, 5, cam=cam, pcam=pcam, special=0.02)
    want = TR.temporal(color, sphere, point, cam, prev, motion=motion, max_history=6, depth_tol=0.02)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    args = (t(color), t(sphere.view(np.int32)), t(point), _cam(cam))
    dprev = {"color": t(prev["color"]), "length": t(prev["length"]), "sphere": t(prev["sphere"]), "point": t(prev["point"]), "camera": _cam(pcam)}
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [R.temporal(*args, dprev, motion=t(motion), max_history=6, depth_tol=0.02, stream=a if k % 2 == 0 else b) for k in range(6)]
    o = R.temporal(*args, dprev, motion=t(motion), max_history=6, depth_tol=0.02, stream=R.CUDA_STREAM_LEGACY)
    torch.cuda.synchronize()
    for k, r in enumerate(outs + [o]):
        assert_history_equal((r["color"].cpu().numpy(), r["length"].cpu().numpy()), want, f"call {k}")
    with pytest.raises(ValueError):   # the library's own stream cannot order torch's reuse of the outputs
        R.temporal(*args, dprev, stream=0)


def test_refusals_enqueue_nothing():
    torch = _torch()
    L = R.lib()
    h, w = 12, 16
    n = h * w
    p = R.rt_temporal_params(w, h, 4, 0, R.rt_camera(), R.rt_camera(), 0.01)
    color = torch.rand((h, w, 3), device="cuda")
    sphere = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    point = torch.rand((h, w, 3), dtype=torch.float64, device="cuda")
    block = torch.full((n * 16,), 7, dtype=torch.uint8, device="cuda")   # the output colour, then the lengths
    oc, ol = block.data_ptr(), block.data_ptr() + n * 12
    host = np.full(n * 4, 7.0, F32)
    cur = R.rt_temporal_frame(color.data_ptr(), sphere.data_ptr(), point.data_ptr())
    cases = [
        ((R.rt_temporal_frame(host.ctypes.data, sphere.data_ptr(), point.data_ptr()), None, R.rt_temporal_out(oc, ol)), b"cur.color is not device"),
        ((cur, None, R.rt_temporal_out(host.ctypes.data, ol)), b"out.color is not device"),
        ((cur, R.rt_temporal_history(color.data_ptr(), host.ctypes.data, sphere.data_ptr(), point.data_ptr()), R.rt_temporal_out(oc, ol)),
         b"prev.length is not device"),
        ((cur, None, R.rt_temporal_out(color.data_ptr() + 8, ol)), b"overlaps cur.color"),
        ((cur, None, R.rt_temporal_out(oc, oc + 4)), b"out.length overlaps out.color"),
    ]
    for (c, hp, o), what in cases:
        assert L.rtb200_temporal_device(0, C.byref(p), C.byref(c), C.byref(hp) if hp is not None else None, None, C.byref(o), None) == -1, what
        assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
    torch.cuda.synchronize()
    assert (block.cpu().numpy() == 7).all() and (host == 7.0).all()
    with pytest.raises(R.RtError):
        R.temporal(color, sphere, point, R.rt_camera(), max_history=0)
    ok = R.temporal(color, sphere, point, R.rt_camera())
    torch.cuda.synchronize()
    assert_history_equal((ok["color"].cpu().numpy(), ok["length"].cpu().numpy()), (color.cpu().numpy(), np.ones((h, w), np.uint32)))


# ---- the CLI -----------------------------------------------------------------------------------------------------------

def test_cli_writes_the_denoised_frames_and_leaves_the_frames_unchanged(tmp_path):
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
    r = subprocess.run([CLI, str(p), str(tmp_path / "plain")], capture_output=True, text=True, cwd=scenes.SCENES_DIR, env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    for spec_env, iters in (("3,2,8,2", 2), ("6,0", 0)):
        r = subprocess.run([CLI, str(p), str(tmp_path / "anim")], capture_output=True, text=True, cwd=scenes.SCENES_DIR,
                           env=dict(env, RTB200_TEMPORAL=spec_env), timeout=300)
        assert r.returncode == 0, r.stderr
        assert not list(tmp_path.glob("plain_*_denoised.png"))
        rs = R.ResidentScene(sc)
        try:
            cams = [R.make_frame(sc, look_from=[f.camera.origin.x, f.camera.origin.y, f.camera.origin.z], seed=f.seed) for f in frames]
            lin, _ = R.render_frames(sc, cams, linear=True)
            prev = None
            for i, f in enumerate(cams):
                assert (tmp_path / f"anim_{i:03}.png").read_bytes() == (tmp_path / f"plain_{i:03}.png").read_bytes()
                a = rs.aov(4, view=f)
                c, n = TR.temporal(lin[i], a["sphere"], a["point"], f.camera, prev, max_history=int(spec_env.split(",")[0]),
                                   depth_tol=R.TEMPORAL_DEPTH_TOL)
                prev = {"color": c, "length": n, "sphere": a["sphere"], "point": a["point"], "camera": f.camera}
                want = DR.denoise(c, a["albedo"], a["normal"], iterations=iters, color_weight=8.0, albedo_weight=2.0,
                                  normal_weight=R.DENOISE_NORMAL_WEIGHT) if iters else c
                got = np.asarray(Image.open(tmp_path / f"anim_{i:03}_denoised.png").convert("RGB"))
                assert np.array_equal(got, DR.quantise(want)), (spec_env, i)
        finally:
            rs.release()
    for extra in ({"RTB200_FRAMES": None}, {"RTB200_GPUS": "1"}, {"RTB200_ADAPTIVE": "0.1"}, {"RTB200_AOV": "1"}, {"RTB200_DENOISE": "2"}):
        e = dict(env, RTB200_TEMPORAL="4")
        for k, v in extra.items():
            if v is None:
                e.pop(k)
            else:
                e[k] = v
        bad = subprocess.run([CLI, str(p), str(tmp_path / "x")], capture_output=True, text=True, env=e, timeout=60)
        assert bad.returncode == 101 and "RTB200_TEMPORAL" in bad.stderr, extra
    for spec_env, what in (("0", "max_history"), ("4,11", "iterations"), ("x", "expected")):
        bad = subprocess.run([CLI, str(p), str(tmp_path / "y")], capture_output=True, text=True, env=dict(env, RTB200_TEMPORAL=spec_env), timeout=60)
        assert bad.returncode == 101 and what in bad.stderr, spec_env
