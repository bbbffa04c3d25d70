"""The work sets of a device on the GPU, against the CPU oracle: lit scenes deep enough to use every buffer of a set, and
renders that overlap on one device. Every comparison is bit-exact: linear f32, RGB8, rays and samples.

A device has two work sets (sample buffer, accumulator, albedo stack, stat block and queue counters, shadow frames, light
terms, frame table), shared by every handle on it. Asynchronous frames of a handle alternate between them; every blocking
render takes set 0. The first part traces lit scenes inside a closed room, where nearly every path runs to max_depth: the
albedo stack past its shared-memory levels (RT_SMEM_STACK = 10) in the lights kernels, next to deep shadow frames. The second
part forces submissions that share a set to overlap on different streams, from one handle or from several."""
import numpy as np
import pytest

import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from synth import mixed_config, _v

pytestmark = pytest.mark.gpu
HOLD = 100_000_000   # clock cycles of torch.cuda._sleep (~50 ms): holds a stream back while the host enqueues behind it


def _room_cfg(n_lights, depth, w=80, h=60, spp=6, seed=31):
    """30 random spheres, the hollow glass shell, the coincident pair and 1-3 lights, closed in by a Lambertian sphere of
    radius 40 so that paths rarely escape to the sky."""
    cfg = mixed_config(w, h, spp, depth, seed=seed, n=30)
    pos = [(0.0, 6.0, 0.0), (-4.0, 3.0, 5.0), (5.0, 2.5, -3.0)]
    for k in range(n_lights):
        cfg["objects"].insert(3 + 5 * k, {"center": _v(*pos[k]), "radius": 1.0 + 0.5 * k, "material": {"Light": {}}})
    cfg["objects"].append({"center": _v(0, 0, 0), "radius": 40.0, "material": {"Lambertian": {"albedo": [0.9, 0.9, 0.9]}}})
    return cfg


def _deep(st, length):
    """Samples of an oracle render whose main path is at least `length` rays long."""
    return sum(st["path_len_hist"][length:])


def _assert_frame(lin, img, want, what):
    assert np.array_equal(lin, want[0]), f"{what}: linear differs in {int((lin != want[0]).any(axis=-1).sum())} pixels, max {np.abs(lin - want[0]).max()}"
    assert np.array_equal(img, want[1]), f"{what}: rgb8 differs"


def _one_shot_vs_oracle(sc, opts=None):
    """render_linear and render_rgb8 of `sc` against the oracle; returns the oracle's stats, the render's and its linear frame."""
    lin_o, img_o, st_o = O.render(sc)
    lin, st = R.render_linear(sc, opts)
    img, st8 = R.render_rgb8(sc, opts)
    _assert_frame(lin, img, (lin_o, img_o), "one-shot")
    assert st["rays"] == st8["rays"] == st_o["rays"] and st["samples"] == st_o["samples"]
    return st_o, st, lin


# ---- 1. lit scenes that use every buffer of a work set ----------------------------------------------------------------

@pytest.mark.parametrize("n_lights,depth", [(1, 10), (2, 11), (3, 50)])
def test_deep_lit_room_matches_the_oracle(n_lights, depth):
    """max_depth 10 and 11 sit on the shared/global boundary of the albedo stack; 50 goes far past it."""
    st_o, _, _ = _one_shot_vs_oracle(R.Scene.from_config(_room_cfg(n_lights, depth)))
    assert _deep(st_o, depth) >= 10_000, st_o["path_len_hist"]              # most paths run to max_depth
    if depth == 50:
        assert _deep(st_o, 30) >= 10_000


@pytest.mark.parametrize("variant", [R.RT_VARIANT_BRUTE_FORCE, R.RT_VARIANT_EXACT_F64], ids=["brute_force", "exact_f64"])
def test_variants_agree_on_the_deep_lit_room(variant):
    sc = R.Scene.from_config(_room_cfg(3, 50))
    lin_t, st_t = R.render_linear(sc, R.make_options(variant=R.RT_VARIANT_FILTERED))
    st_o, st, lin = _one_shot_vs_oracle(sc, R.make_options(variant=variant))
    assert np.array_equal(lin, lin_t) and st["rays"] == st_t["rays"]
    assert _deep(st_o, 30) >= 10_000


def _view(sc, f):
    """The scene with frame f's camera, seed and max_depth (a copy of its C struct, sharing the spheres)."""
    v = R.Scene()
    v.c = R.rt_scene.from_buffer_copy(sc.c)
    v.c.camera = f.camera; v.c.seed = f.seed; v.c.max_depth = f.max_depth
    v._keep = sc
    return v


def _frames_vs_oracle(sc, frames, opts=None):
    img, st = R.render_frames(sc, frames, opts)
    lin, st2 = R.render_frames(sc, frames, opts, linear=True)
    rays = samples = 0
    for i, f in enumerate(frames):
        lin_o, img_o, st_o = O.render(_view(sc, f))
        _assert_frame(lin[i], img[i], (lin_o, img_o), f"frame {i}")
        rays += st_o["rays"]; samples += st_o["samples"]
    assert st["rays"] == st2["rays"] == rays and st["samples"] == samples
    return st


def _room_frames(sc):
    """Three views of the room, each with its own seed."""
    return [R.make_frame(sc, seed=5), R.make_frame(sc, look_from=[-9.0, 3.0, 7.0], seed=6),
            R.make_frame(sc, look_from=[4.0, 8.0, -12.0], look_at=[0.0, 1.0, 0.0], seed=7)]


def test_deep_lit_frames_in_one_launch():
    """The LIGHTS + FRAMES kernel past albedo-stack level 10: three views of the room in one trace launch."""
    sc = R.Scene.from_config(_room_cfg(3, 50))
    st = _frames_vs_oracle(sc, _room_frames(sc))
    assert st["batches"] == 1 and st["frames"] == 3 and st["kernel_launches"] == 1 + 3


def test_deep_lit_sample_batches():
    """A sample buffer of two samples per pixel: three batches accumulate through `accum`."""
    sc = R.Scene.from_config(_room_cfg(2, 50))
    opts = R.make_options(sample_buffer_bytes=2 * 80 * 60 * 16)
    st_o, st, _ = _one_shot_vs_oracle(sc, opts)
    assert st["batches"] == 3 and st["kernel_launches"] == 2 * 3
    assert _deep(st_o, 30) >= 10_000


def _textured_room():
    """The textured test scene (its own light, textured spheres, sky texture) closed in by the room sphere at max_depth 50."""
    cfg = scenes._variant(scenes.test_scene_config(), 80, 60, 4, 50)
    cfg["objects"].append({"center": _v(0, 0, 0), "radius": 40.0, "material": {"Lambertian": {"albedo": [0.9, 0.9, 0.9]}}})
    return R.Scene.from_config(cfg, scenes.SCENES_DIR)


def test_deep_textured_room():
    """Texel codes go onto the albedo stack past its shared-memory levels (a fifth of the paths reach level 13)."""
    st_o, _, _ = _one_shot_vs_oracle(_textured_room())
    assert _deep(st_o, 13) >= 2_000 and st_o["hits"][R.RT_TEXTURE] > 0, st_o["path_len_hist"]


# ---- 2. overlapping renders on one device -------------------------------------------------------------------------------
# Handles A and B hold the same spheres, materials, lights and (no) textures: the 3-light room at max_depth 50, so that the
# albedo stack, shadow frames, light terms, sample buffer and counters of a set are all in use. B has another camera and
# seed, so a frame that picks up work or samples of the other one is wrong. Before anything overlaps, both work sets are
# grown to their final sizes by renders of the same workloads, and the last frames written into both sets are B's: a
# resolve that reads samples another kernel has claimed but not yet written then reads B's, not A's.
#
# Without the ordering of the work sets these overlaps only produce wrong values, never an out-of-bounds access: no buffer is
# freed while in use (nothing grows once the overlaps begin), and every stack code, shadow frame and material index one kernel
# writes and the other reads is valid for both scenes, because their layouts are the same. No test relies on a fault or
# repeats a run.

SIZE = (160, 120, 8)
_ORACLE = {}   # (camera, seed, max_depth) of a view of the overlap scene -> the oracle's linear, rgb8, rays, samples


class _Overlap:
    def __init__(self):
        import torch
        self.torch = torch
        w, h, spp = SIZE
        self.cfg = _room_cfg(3, 50, w, h, spp, seed=31)
        self.sa = R.Scene.from_config(self.cfg); self.sa.seed = 101
        self.sb = R.Scene.from_config(self.cfg); self.sb.seed = 202
        self.sb.set_camera(look_from=_v(-9.0, 3.0, 7.0))
        self.frames_b = [R.make_frame(self.sb, look_from=[4.0, 8.0, -12.0], seed=203), R.make_frame(self.sb, seed=204),
                         R.make_frame(self.sb, look_from=[-6.0, 1.5, -9.0], seed=205)]
        self.n = w * h * 3
        self.a = R.ResidentScene(self.sa)
        self.b = R.ResidentScene(self.sb)
        self.parity = {id(self.a): 0, id(self.b): 0}   # which set the handle's next asynchronous frame takes
        self.streams = [torch.cuda.Stream() for _ in range(3)]
        assert not np.array_equal(self.oracle(self.sa)[1], self.oracle(self.sb)[1])

    def oracle(self, sc, f=None):
        v = sc if f is None else _view(sc, f)
        key = (bytes(v.c.camera), v.c.seed, v.c.max_depth)
        if key not in _ORACLE:
            lin, img, st = O.render(v)
            _ORACLE[key] = (lin, img, st["rays"], st["samples"])
        return _ORACLE[key]

    def bufs(self, k=1):
        t = self.torch
        return t.zeros(k * self.n, dtype=t.uint8, device="cuda"), t.zeros(k * self.n, dtype=t.float32, device="cuda")

    def hold(self, *streams):
        for s in streams:
            with self.torch.cuda.stream(s):
                self.torch.cuda._sleep(HOLD)

    def render_async(self, rs, out, stream):
        self.parity[id(rs)] ^= 1
        rs.render_async(out[0].data_ptr(), out[1].data_ptr(), stream.cuda_stream if stream is not None else 0)

    def even(self, rs):
        """Make the next asynchronous frame of rs take set 0 (the set of every blocking render)."""
        if self.parity[id(rs)]:
            out = self.bufs()
            self.render_async(rs, out, None)
            rs.wait()

    def b_last_in_both_sets(self):
        """The last samples written into both sets are B's (module comment)."""
        self.even(self.b)
        out = [self.bufs(), self.bufs()]
        for o in out:
            self.render_async(self.b, o, None)
        st = self.b.wait()
        self.torch.cuda.synchronize()
        for o in out:
            self.check(o, self.sb, "B filling the sets")
        assert st["rays"] == self.oracle(self.sb)[2]

    def grow(self):
        """Both sets at their final sizes: every workload of the overlaps once, without overlap."""
        o = self.bufs(3)
        self.b.render_frames(self.frames_b, o[0].data_ptr(), o[1].data_ptr())   # set 0, the multi-frame launch
        for rs in (self.a, self.b):
            rs.render(o[0].data_ptr(), o[1].data_ptr())                         # set 0
            for _ in range(2):
                self.render_async(rs, o, None)                                  # sets 0 and 1
            rs.wait()
        R.render_linear(self.sb)                                                # a one-shot render of B's scene
        self.b_last_in_both_sets()

    def check(self, out, sc, what, f=None, k=0):
        want = self.oracle(sc, f)
        lin = out[1].cpu().numpy().reshape(-1, SIZE[1], SIZE[0], 3)[k]
        img = out[0].cpu().numpy().reshape(-1, SIZE[1], SIZE[0], 3)[k]
        _assert_frame(lin, img, want, what)

    def check_stats(self, st, sc, frames, what, f=None):
        want = self.oracle(sc, f)
        assert (st["rays"], st["samples"], st["frames"]) == (want[2], want[3], frames), (what, st["rays"], want[2])

    def release(self):
        self.a.release(); self.b.release()


@pytest.fixture
def ov():
    import torch
    o = _Overlap()
    o.grow()
    yield o
    torch.cuda.synchronize()
    o.release()


def test_one_handle_on_three_streams_round_robin(ov):
    """Frame k on stream k mod 3: frames 0 and 2 share set 0 on two streams, frames 1 and 5 set 1."""
    ov.even(ov.a)
    outs = [ov.bufs() for _ in range(6)]
    ov.hold(*ov.streams)
    for k in range(6):
        ov.render_async(ov.a, outs[k], ov.streams[k % 3])
    st = ov.a.wait()
    ov.torch.cuda.synchronize()
    for k in range(6):
        ov.check(outs[k], ov.sa, f"frame {k}")
    ov.check_stats(st, ov.sa, 6, "wait")


def test_one_handle_on_s1_s1_s2_s2(ov):
    """Frames 0 and 2 share set 0 and start together on S1 and S2; frames 1 and 3 share set 1."""
    ov.even(ov.a)
    s1, s2 = ov.streams[:2]
    outs = [ov.bufs() for _ in range(4)]
    ov.hold(s1, s2)
    for k, s in enumerate((s1, s1, s2, s2)):
        ov.render_async(ov.a, outs[k], s)
    st = ov.a.wait()
    ov.torch.cuda.synchronize()
    for k in range(4):
        ov.check(outs[k], ov.sa, f"frame {k}")
    ov.check_stats(st, ov.sa, 4, "wait")


def test_blocking_renders_of_another_handle_while_frames_are_in_flight(ov):
    """A's asynchronous frame on S1 and B's blocking render_device, then render_frames_device, on S2: all set 0."""
    s1, s2 = ov.streams[:2]
    for blocking in ("render", "render_frames"):
        ov.even(ov.a)
        oa = ov.bufs()
        ob = ov.bufs(3 if blocking == "render_frames" else 1)
        ov.hold(s1, s2)
        ov.render_async(ov.a, oa, s1)
        if blocking == "render":
            stb = ov.b.render(ob[0].data_ptr(), ob[1].data_ptr(), s2.cuda_stream)
            ov.check_stats(stb, ov.sb, 1, "B render")
        else:
            stb = ov.b.render_frames(ov.frames_b, ob[0].data_ptr(), ob[1].data_ptr(), s2.cuda_stream)
            assert stb["batches"] == 1 and stb["frames"] == 3
            want = [ov.oracle(ov.sb, f) for f in ov.frames_b]
            assert (stb["rays"], stb["samples"]) == (sum(w[2] for w in want), sum(w[3] for w in want)), "B render_frames"
        sta = ov.a.wait()
        ov.torch.cuda.synchronize()
        ov.check(oa, ov.sa, f"A beside B's {blocking}")
        ov.check_stats(sta, ov.sa, 1, f"A's wait beside B's {blocking}")
        if blocking == "render":
            ov.check(ob, ov.sb, "B render")
        else:
            for k, f in enumerate(ov.frames_b):
                ov.check(ob, ov.sb, f"B frame {k}", f, k)


@pytest.mark.parametrize("call", ["render_linear", "render_rgb8", "render_rgb8_multi"])
def test_one_shot_render_while_frames_are_in_flight(ov, call):
    """A's asynchronous frame runs (no hold) while a one-shot render of B's scene, on the library's stream, takes set 0."""
    ov.even(ov.a)
    oa = ov.bufs()
    lin_o, img_o, rays_o, samples_o = ov.oracle(ov.sb)
    ov.torch.cuda.synchronize()
    ov.render_async(ov.a, oa, ov.streams[0])
    if call == "render_linear":
        out, st = R.render_linear(ov.sb)
        assert np.array_equal(out, lin_o), "B's one-shot linear frame differs"
    elif call == "render_rgb8":
        out, st = R.render_rgb8(ov.sb)
        assert np.array_equal(out, img_o), "B's one-shot rgb8 frame differs"
    else:
        out, st = R.render_rgb8_multi(ov.sb, 1, R.make_options(device=ov.torch.cuda.current_device()))
        assert np.array_equal(out, img_o) and st["gpus_used"] == 1, "B's multi-GPU frame differs"
    assert (st["rays"], st["samples"]) == (rays_o, samples_o), "B's one-shot stats"
    sta = ov.a.wait()
    ov.torch.cuda.synchronize()
    ov.check(oa, ov.sa, f"A beside {call}")
    ov.check_stats(sta, ov.sa, 1, f"A's wait beside {call}")


def test_two_handles_with_frames_in_flight(ov):
    """A on S1 and B on S2, two frames each: A's and B's first frames share set 0, their second frames set 1."""
    ov.even(ov.a); ov.even(ov.b)
    s1, s2 = ov.streams[:2]
    oa = [ov.bufs() for _ in range(2)]
    ob = [ov.bufs() for _ in range(2)]
    ov.hold(s1, s2)
    for k in range(2):
        ov.render_async(ov.a, oa[k], s1)
        ov.render_async(ov.b, ob[k], s2)
    sta = ov.a.wait()
    stb = ov.b.wait()
    ov.torch.cuda.synchronize()
    for k in range(2):
        ov.check(oa[k], ov.sa, f"A frame {k}")
        ov.check(ob[k], ov.sb, f"B frame {k}")
    ov.check_stats(sta, ov.sa, 2, "A's wait")
    ov.check_stats(stb, ov.sb, 2, "B's wait")
