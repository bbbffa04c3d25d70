"""The CLI's RTB200_DENOISE_VAR mode without a GPU: malformed specs and the modes it cannot be combined with exit 101 with a
message before any rendering (the GPU test of the mode itself is in tests/test_gpu_render_variance.py)."""
import json
import os
import subprocess

import pytest

from rtb200 import scenes

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(REPO, "rust-raytracer_b200", "raytracer")


@pytest.fixture(scope="module")
def config(tmp_path_factory):
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-C", os.path.join(REPO, "rust-raytracer_b200"), "raytracer"])
    d = tmp_path_factory.mktemp("cli")
    cfg = scenes._variant(scenes.cover_config(), 16, 12, 2, 4)
    plain = d / "scene.json"; plain.write_text(json.dumps(cfg))
    cfg = json.loads(json.dumps(cfg))
    cfg["camera"].update(aperture=0.2, focus_dist=9.0)
    lens = d / "lens.json"; lens.write_text(json.dumps(cfg))
    return d, plain, lens


def _run(cfg, out, **env):
    e = {k: v for k, v in os.environ.items() if not k.startswith("RTB200_")}
    e.update(env)
    return subprocess.run([CLI, str(cfg), str(out)], capture_output=True, text=True, cwd=scenes.SCENES_DIR, env=e, timeout=60)


@pytest.mark.parametrize("spec", ["", "x", "0", "11", "2.5", "-1", "3,", "3,,1", "3,-1", "3,nan", "3,1e39", "3,1,inf",
                                  "3,1,4,-0.5", "3,1,4,1,0", "3,1,4,1,-1e-4", "3,1,4,1,nan", "3,1,4,1,1e-46",
                                  "3,1,4,1,1e-4,7", "3 ,1", "3,1x"])
def test_a_malformed_spec_exits_101(config, spec):
    d, plain, _ = config
    r = _run(plain, d / "o.png", RTB200_DENOISE_VAR=spec)
    assert r.returncode == 101 and "RTB200_DENOISE_VAR" in r.stderr, (spec, r.returncode, r.stderr)
    assert not (d / "o.png").exists() and not (d / "o_denoised.png").exists()


@pytest.mark.parametrize("other", ["RTB200_DENOISE", "RTB200_GPUS", "RTB200_FRAMES", "RTB200_ADAPTIVE"])
def test_the_modes_it_cannot_be_combined_with_exit_101(config, other):
    d, plain, _ = config
    r = _run(plain, d / "o.png", RTB200_DENOISE_VAR="2", **{other: "1"})
    assert r.returncode == 101 and "RTB200_DENOISE_VAR" in r.stderr and other in r.stderr, (other, r.stderr)


def test_temporal_and_a_lens_camera_exit_101(config):
    d, plain, lens = config
    r = _run(plain, d / "o.png", RTB200_DENOISE_VAR="2", RTB200_TEMPORAL="2", RTB200_FRAMES=str(d / "none.json"))
    assert r.returncode == 101 and "RTB200_DENOISE_VAR" in r.stderr
    r = _run(lens, d / "o.png", RTB200_DENOISE_VAR="2")
    assert r.returncode == 101 and "lens camera" in r.stderr and "RTB200_DENOISE_VAR" in r.stderr
