"""Animations (rtb200_render_frames / rtb200_render_frames_device, the CLI's RTB200_FRAMES) on the host side: the rt_frame
layout, argument validation before any device is touched, the Python frame builder and the CLI's error exits. No GPU needed."""
import ctypes as C
import json
import os
import re
import subprocess

import pytest

import rtb200 as R
from rtb200 import scenes

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(REPO, "rust-raytracer_b200", "raytracer")
INVALID, NO_DEVICE = -1, -2


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_rt_frame_layout_matches_the_header():
    assert C.sizeof(R.rt_frame) == 112
    txt = open(os.path.join(REPO, "include", "rtb200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} rt_frame;", txt).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    decl = [tuple(d.split()) for d in body.strip().rstrip(";").split(";")]
    ctypes_of = {"rt_camera": R.rt_camera, "uint64_t": C.c_uint64, "uint32_t": C.c_uint32}
    assert [(ctypes_of[t], n) for t, n in decl] == [(t, n) for n, t in R.rt_frame._fields_]
    assert [getattr(R.rt_frame, n).offset for n, _ in R.rt_frame._fields_] == [0, 96, 104, 108]


def test_make_frame_defaults_to_the_scene():
    sc = scenes.cover_scene(32, 24, 2, depth=7)
    sc.seed = 1234
    f = R.make_frame(sc)
    assert bytes(f.camera) == bytes(sc.c.camera) and f.seed == 1234 and f.max_depth == 7 and f.reserved == 0
    g = R.make_frame(sc, look_from=[1, 2, 3], vfov=30.0, seed=5, max_depth=0)
    p = dict(sc.camera_params, look_from=[1, 2, 3], vfov=30.0)
    assert bytes(g.camera) == bytes(R.camera_from_params(p["look_from"], p["look_at"], p["vup"], p["vfov"], p["aspect"]))
    assert (g.seed, g.max_depth) == (5, 0)


def _frames(sc, n):
    return (R.rt_frame * max(n, 1))(*[R.make_frame(sc, seed=i) for i in range(n)])


def test_host_entry_point_validates_frames_before_touching_the_device():
    L = R.lib()
    sc = scenes.cover_scene(16, 12, 1)
    out = (C.c_uint8 * (16 * 12 * 3 * 4))()
    st = R.rt_stats()
    assert L.rtb200_render_frames(C.byref(sc.c), None, _frames(sc, 1), 0, out, None, C.byref(st)) == INVALID
    assert L.rtb200_render_frames(C.byref(sc.c), None, None, 2, out, None, C.byref(st)) == INVALID
    bad = _frames(sc, 3)
    bad[2].reserved = 1
    assert L.rtb200_render_frames(C.byref(sc.c), None, bad, 3, out, None, C.byref(st)) == INVALID
    assert b"reserved" in L.rtb200_last_error()
    assert L.rtb200_render_frames(C.byref(sc.c), None, _frames(sc, 2), 2, None, None, C.byref(st)) == INVALID
    # n_frames * rows * width * 3 beyond 64 bits (the frames array is never read that far)
    big = scenes.cover_scene(46341, 46340, 1)
    assert L.rtb200_render_frames(C.byref(big.c), None, _frames(sc, 1), 0xFFFFFFFF, out, None, C.byref(st)) == INVALID
    assert b"overflow" in L.rtb200_last_error()
    # an invalid scene or options are still refused as such
    sc.c.samples_per_pixel = 0
    assert L.rtb200_render_frames(C.byref(sc.c), None, _frames(sc, 1), 1, out, None, C.byref(st)) == INVALID


def test_device_entry_point_validates_its_arguments():
    L = R.lib()
    sc = scenes.cover_scene(16, 12, 1)
    st = R.rt_stats()
    for frames, n in ((_frames(sc, 1), 0), (None, 1), (_frames(sc, 1), 1)):
        assert L.rtb200_render_frames_device(None, frames, n, C.c_void_p(16), None, None, C.byref(st)) == INVALID


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_valid_frames_without_gpu_report_no_device():
    sc = scenes.cover_scene(16, 12, 1)
    with pytest.raises(R.RtError) as e:
        R.render_frames(sc, [R.make_frame(sc), R.make_frame(sc, seed=2)])
    assert e.value.code == NO_DEVICE


@pytest.fixture(scope="module")
def cli():
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-C", os.path.join(REPO, "rust-raytracer_b200"), "raytracer"])
    return CLI


def _scene_file(tmp_path):
    p = tmp_path / "scene.json"
    p.write_text(json.dumps(scenes._variant(scenes.cover_config(), 16, 12, 1, 4)))
    return p


def _run(cli, tmp_path, frames_text, **env):
    fp = tmp_path / "frames.json"
    fp.write_text(frames_text)
    e = {k: v for k, v in os.environ.items() if k != "RTB200_GPUS"}
    e.update(RTB200_FRAMES=str(fp), **env)
    return subprocess.run([cli, str(_scene_file(tmp_path)), str(tmp_path / "anim")], capture_output=True, text=True, timeout=300, env=e)


CAM = {"look_from": {"x": 13, "y": 2, "z": 3}, "look_at": {"x": 0, "y": 0, "z": 0}, "vup": {"x": 0, "y": 1, "z": 0}, "vfov": 20.0, "aspect": 4 / 3}


@pytest.mark.parametrize("text,message", [
    ('[{"camera": ', "Unable to parse frames json"),
    ('{"camera": {}}', "frames: array expected"),
    ("[]", "at least one frame"),
    ('[{"seed": 1}]', "missing field `camera`"),
    (json.dumps([{"camera": dict(CAM, vfov="wide")}]), "number expected"),
    (json.dumps([{"camera": CAM, "max_depth": -1}]), "max_depth: non-negative integer expected"),
    (json.dumps([{"camera": CAM, "seed": 0.5}]), "seed: non-negative integer expected"),
])
def test_cli_malformed_frames_file_exits_like_a_panic(cli, tmp_path, text, message):
    r = _run(cli, tmp_path, text)
    assert r.returncode == 101 and message in r.stderr, r.stderr
    assert "Unable to parse frames json" in r.stderr and not list(tmp_path.glob("anim_*.png"))


def test_cli_frames_with_several_gpus_is_refused(cli, tmp_path):
    r = _run(cli, tmp_path, json.dumps([{"camera": CAM}]), RTB200_GPUS="0")
    assert r.returncode == 101 and "not supported" in r.stderr


def test_cli_missing_frames_file(cli, tmp_path):
    e = dict(os.environ, RTB200_FRAMES=str(tmp_path / "nope.json"))
    r = subprocess.run([cli, str(_scene_file(tmp_path)), str(tmp_path / "anim")], capture_output=True, text=True, timeout=300, env=e)
    assert r.returncode == 101 and "Unable to read frames file" in r.stderr
