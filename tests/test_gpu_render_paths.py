"""One scheduler for one frame and for many: a one-frame call and a frames call of the same view launch the same work and
report the same statistics, and every render entry point reports a shard with no rows the same way."""
import numpy as np
import pytest

import rtb200 as R
from rtb200 import scenes

pytestmark = pytest.mark.gpu
W, H, SPP = 64, 48, 8
STATS = ("rays", "samples", "candidates", "batches", "kernel_launches", "frames", "h2d_bytes", "d2h_bytes")
CASES = ["default_cap", "sample_batches", "max_depth_0"]


def _case(case):
    sc = scenes.cover_scene(W, H, SPP)
    opts = None
    if case == "sample_batches":
        opts = R.make_options(sample_buffer_bytes=W * H * 16 * 3)   # 3 samples per batch: 3 batches
    if case == "max_depth_0":
        sc.c.max_depth = 0
    return sc, opts


def _stats(st):
    return {k: st[k] for k in STATS}


def _check_case(case, st):
    assert st["batches"] == (3 if case == "sample_batches" else 1) and st["frames"] == 1
    if case == "max_depth_0":
        assert st["rays"] == 0 and st["samples"] == W * H * SPP
    else:
        assert st["rays"] > 0


@pytest.mark.parametrize("case", CASES)
def test_host_one_frame_calls_equal_a_one_frame_frames_call(case):
    sc, opts = _case(case)
    frames = [R.make_frame(sc)]
    img, st8 = R.render_rgb8(sc, opts)
    lin, stl = R.render_linear(sc, opts)
    fimg, fst8 = R.render_frames(sc, frames, opts)
    flin, fstl = R.render_frames(sc, frames, opts, linear=True)
    assert np.array_equal(fimg[0], img) and np.array_equal(flin[0], lin)
    assert _stats(fst8) == _stats(st8) and _stats(fstl) == _stats(stl)
    _check_case(case, st8)
    if case == "max_depth_0":
        assert not img.any()


@pytest.mark.parametrize("case", CASES)
def test_resident_render_equals_a_one_frame_frames_call(case):
    import torch
    sc, opts = _case(case)
    rs = R.ResidentScene(sc, opts)
    n = W * H * 3
    a8, b8 = (torch.zeros(n, dtype=torch.uint8, device="cuda") for _ in range(2))
    al, bl = (torch.zeros(n, dtype=torch.float32, device="cuda") for _ in range(2))
    sa = rs.render(a8.data_ptr(), al.data_ptr())
    sb = rs.render_frames([R.make_frame(sc)], b8.data_ptr(), bl.data_ptr())
    torch.cuda.synchronize()
    rs.release()
    assert torch.equal(a8, b8) and torch.equal(al, bl)
    assert _stats(sb) == _stats(sa)
    _check_case(case, sa)


def test_a_shard_with_no_rows_reports_its_frames_on_every_entry_point():
    import torch
    sc = scenes.cover_scene(16, 2, 2)
    opts = R.make_options(rank=3, world=4)
    assert R.shard_rows(2, 3, 4) == 0
    frames = [R.make_frame(sc), R.make_frame(sc, seed=5)]
    img, s_rgb8 = R.render_rgb8(sc, opts)
    assert img.shape == (0, 16, 3)
    _, s_frames = R.render_frames(sc, frames, opts)
    rs = R.ResidentScene(sc, opts)
    s_render = rs.render()
    for _ in range(3):
        rs.render_async()
    s_wait = rs.wait()
    buf = torch.zeros(16, dtype=torch.uint8, device="cuda")   # the frames call needs an output, even an empty one
    s_frames_device = rs.render_frames(frames, buf.data_ptr())
    rs.release()
    for st, n in ((s_rgb8, 1), (s_frames, 2), (s_render, 1), (s_wait, 3), (s_frames_device, 2)):
        assert (st["rays"], st["samples"], st["batches"], st["kernel_launches"]) == (0, 0, 0, 0), st
        assert st["frames"] == n and st["gpus_used"] == 1, st
