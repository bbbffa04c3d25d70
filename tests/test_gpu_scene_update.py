"""Moving the spheres of a resident scene on the GPU (rtb200_scene_update_spheres / _geometry_device): after an update every
render of the handle is bit-identical, in linear f32, RGB8 and ray count, to the CPU oracle of the edited scene and to a fresh
upload of it; the device's arrays equal the numpy restatement of tests/test_scene_update_cpu.py; updates are ordered after the
frames enqueued before them and before the frames enqueued after them; refused updates leave the scene unchanged."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O
import rtb200 as R
from rtb200 import scenes
from synth import mixed_config, _v
from test_scene_update_cpu import refit, same_bits

pytestmark = pytest.mark.gpu
INVALID, UNSUPPORTED = -1, -4


def _render(rs):
    import torch
    w = rs.scene.c.width
    n = rs.rows * w * 3
    d8 = torch.zeros(n, dtype=torch.uint8, device="cuda")
    dl = torch.zeros(n, dtype=torch.float32, device="cuda")
    st = rs.render(d8.data_ptr(), dl.data_ptr())
    return d8.cpu().numpy().reshape(rs.rows, w, 3), dl.cpu().numpy().reshape(rs.rows, w, 3), st["rays"]


def _fresh(sc, opts=None):
    rs = R.ResidentScene(sc, opts)
    try:
        return _render(rs)
    finally:
        rs.release()


def _assert_same(got, want, what):
    assert np.array_equal(got[1], want[1]), f"{what}: linear differs, max {np.abs(got[1] - want[1]).max()}"
    assert np.array_equal(got[0], want[0]), f"{what}: rgb8 differs"
    assert got[2] == want[2], f"{what}: rays {got[2]} != {want[2]}"


def _check(rs, sc, oracle=True, what="render"):
    got = _render(rs)
    _assert_same(got, _fresh(sc, rs.opts), what + " vs a fresh upload")
    if oracle:
        lin_o, img_o, st_o = O.render(sc)
        _assert_same(got, (img_o, lin_o, st_o["rays"]), what + " vs the oracle")
    return got


def _jitter(sc, rng, count, scale=0.3, skip=()):
    """Move `count` random spheres (not those in `skip`); returns the indices and the edited records."""
    cand = [i for i in range(sc.n_spheres) if i not in skip]
    idx = sorted(int(i) for i in rng.choice(cand, size=min(count, len(cand)), replace=False))
    recs = []
    for i in idx:
        s = sc._spheres[i]
        recs.append(sc.set_sphere(i, center=[s.center.x + rng.normal() * scale, s.center.y + abs(rng.normal()) * scale, s.center.z + rng.normal() * scale]))
    return idx, recs


def _light_scene(n_lights, depth, seed):
    cfg = mixed_config(48, 36, 3, depth, seed=seed, n=30)
    pos = [(0.0, 6.0, 0.0), (-4.0, 3.0, 5.0)]
    for k in range(n_lights):
        cfg["objects"].insert(3 + 5 * k, {"center": _v(*pos[k]), "radius": 1.0 + 0.5 * k, "material": {"Light": {}}})
    return R.Scene.from_config(cfg)


def test_cover_scene_edits_match_the_oracle_and_a_fresh_upload():
    sc = scenes.cover_scene(64, 48, 4)
    rs = R.ResidentScene(sc)
    rng = np.random.default_rng(1)
    idx, recs = _jitter(sc, rng, 40, skip={0})
    idx += [0, 5, 7]
    recs += [sc.set_sphere(0, center=[0.0, -1000.3, 0.2]),                                            # the ground moves too
             sc.set_sphere(5, material={"Metal": {"albedo": [0.9, 0.8, 0.7], "fuzz": 0.1}}, radius=0.3),
             sc.set_sphere(7, material={"Glass": {"index_of_refraction": 1.5}})]
    rs.update_spheres(idx, recs)
    _check(rs, sc, what="cover")
    rs.release()


@pytest.mark.parametrize("n_lights,depth", [(1, 1), (2, 2), (1, 6), (2, 6)])
def test_moving_lights_in_a_mixed_material_scene(n_lights, depth):
    sc = _light_scene(n_lights, depth, seed=40 + depth)
    rs = R.ResidentScene(sc)
    lights = [i for i in range(sc.n_spheres) if sc._spheres[i].kind == R.RT_LIGHT]
    assert len(lights) == n_lights
    rng = np.random.default_rng(depth)
    idx, recs = _jitter(sc, rng, 8, skip=set(lights))
    for k, i in enumerate(lights):
        s = sc._spheres[i]
        recs.append(sc.set_sphere(i, center=[s.center.x + 1.0, s.center.y - 0.5 * k, s.center.z - 1.5], radius=s.radius * 0.8))
        idx.append(i)
    rs.update_spheres(idx, recs)
    _check(rs, sc, what=f"{n_lights} lights, depth {depth}")
    rs.release()


def test_switch_to_a_texture_material():
    sc = R.Scene.from_config(scenes._variant(scenes.test_scene_config(), 64, 48, 2, 6), scenes.SCENES_DIR)
    assert sc.c.n_textures >= 1
    rs = R.ResidentScene(sc)
    i = next(k for k in range(sc.n_spheres) if sc._spheres[k].kind in (R.RT_LAMBERTIAN, R.RT_METAL, R.RT_GLASS))
    s = sc._spheres[i]
    rec = sc.set_sphere(i, center=[s.center.x, s.center.y + 0.1, s.center.z],
                        material={"Texture": {"albedo": [1.0, 1.0, 1.0], "h_offset": 0.25, "texture": 0}})
    rs.update_spheres([i], [rec])
    _check(rs, sc, what="texture")
    rs.release()


@pytest.mark.parametrize("variant", [R.RT_VARIANT_FILTERED, R.RT_VARIANT_EXACT_F64, R.RT_VARIANT_BRUTE_FORCE])
def test_variants(variant):
    sc = R.Scene.from_config(mixed_config(48, 36, 3, 8, seed=9))
    rs = R.ResidentScene(sc, R.make_options(variant=variant))
    idx, recs = _jitter(sc, np.random.default_rng(variant), 30, scale=1.0)
    recs[0] = sc.set_sphere(idx[0], material={"Lambertian": {"albedo": [0.2, 0.9, 0.2]}})
    rs.update_spheres(idx, recs)
    _check(rs, sc, what=f"variant {variant}")
    rs.release()


def test_an_animation_of_successive_updates():
    sc = scenes.cover_scene(48, 36, 2, depth=10)
    rs = R.ResidentScene(sc)
    base = [(sc._spheres[i].center.x, sc._spheres[i].center.y, sc._spheres[i].center.z) for i in range(sc.n_spheres)]
    movers = list(range(1, sc.n_spheres, 5))
    for step in range(8):
        recs = []
        for i in movers:                                     # a bounce: each mover has its own phase
            x, y, z = base[i]
            recs.append(sc.set_sphere(i, center=[x + 0.05 * step, y + 0.4 * abs(np.sin(0.7 * step + i)), z]))
        rs.update_spheres(movers, recs)
        _check(rs, sc, what=f"step {step}")
    rs.release()


def test_render_frames_after_an_update():
    import torch
    sc = scenes.cover_scene(48, 36, 2)
    rs = R.ResidentScene(sc)
    idx, recs = _jitter(sc, np.random.default_rng(3), 60)
    rs.update_spheres(idx, recs)
    frames = [R.make_frame(sc, seed=5), R.make_frame(sc, look_from=[11.0, 3.0, 6.0], seed=6), R.make_frame(sc, seed=7, max_depth=3)]
    want, _ = R.render_frames(sc, frames)
    want_lin, st_want = R.render_frames(sc, frames, linear=True)
    n = 3 * 48 * 36 * 3
    out = torch.zeros(n, dtype=torch.uint8, device="cuda"); lin = torch.zeros(n, dtype=torch.float32, device="cuda")
    st = rs.render_frames(frames, out.data_ptr(), lin.data_ptr())
    assert np.array_equal(out.cpu().numpy().reshape(want.shape), want)
    assert np.array_equal(lin.cpu().numpy().reshape(want_lin.shape), want_lin) and st["rays"] == st_want["rays"]
    rs.release()


def test_row_band_shards():
    sc = scenes.cover_scene(48, 40, 2)
    handles = [R.ResidentScene(sc, R.make_options(rank=r, world=3, band_rows=2)) for r in range(3)]
    idx, recs = _jitter(sc, np.random.default_rng(4), 50, scale=0.5)
    img_o, rays = O.render(sc)[1], 0
    for r, rs in enumerate(handles):
        rs.update_spheres(idx, recs)
        got = _check(rs, sc, oracle=False, what=f"shard {r}")
        assert np.array_equal(got[0], img_o[R.shard_row_indices(40, r, 3, 2)])
        rays += got[2]
        rs.release()
    assert rays == _fresh(sc)[2]


def _positions(sc):
    return np.array([[s.center.x, s.center.y, s.center.z] for s in sc._spheres[: sc.n_spheres]]), \
        np.array([s.radius for s in sc._spheres[: sc.n_spheres]])


@pytest.mark.parametrize("variant", [R.RT_VARIANT_FILTERED, R.RT_VARIANT_BRUTE_FORCE])
def test_device_arrays_equal_the_restatement(variant):
    sc = R.Scene.from_config(mixed_config(32, 24, 1, 4, seed=12, n=120))
    b0 = R.bvh_records(sc)
    rs = R.ResidentScene(sc, R.make_options(variant=variant))
    up = rs.bvh_records()
    if variant == R.RT_VARIANT_FILTERED:
        for key in ("lo", "hi", "leaf_rec"):
            assert same_bits(up[key], b0[key]), key
    rng = np.random.default_rng(variant)
    idx, recs = _jitter(sc, rng, 80, scale=2.0)
    recs[1] = sc.set_sphere(idx[1], center=[1e16, 0.0, 0.0])        # leaves the f32 frame
    recs[2] = sc.set_sphere(idx[2], center=[np.nan, 0.0, 0.0])
    recs[3] = sc.set_sphere(idx[3], radius=-0.3)
    rs.update_spheres(idx, recs)
    c, r = _positions(sc)
    got, want = rs.bvh_records(), refit(b0, c, r)
    assert np.array_equal(got["geo"][:, :3], c, equal_nan=True) and np.array_equal(got["geo"][:, 3], r)
    keys = ("lo", "hi", "leaf_rec") if variant == R.RT_VARIANT_FILTERED else ("flat",)
    for key in keys:
        assert same_bits(got[key], want[key]), key
    rs.release()


def test_moving_back_restores_the_upload_exactly():
    sc = scenes.cover_scene(32, 24, 1)
    rs = R.ResidentScene(sc)
    before = rs.bvh_records()
    idx = list(range(sc.n_spheres))
    orig = [R.rt_sphere.from_buffer_copy(sc._spheres[i]) for i in idx]
    rng = np.random.default_rng(8)
    moved = []
    for s in orig:
        m = R.rt_sphere.from_buffer_copy(s)
        m.center.x += rng.normal() * 3.0; m.center.z += rng.normal() * 3.0; m.radius *= 1.5
        moved.append(m)
    rs.update_spheres(idx, moved)
    assert not same_bits(rs.bvh_records()["lo"], before["lo"])
    rs.update_spheres(idx, orig)
    after = rs.bvh_records()
    for key in ("lo", "hi", "child", "leaf_rec"):
        assert same_bits(after[key], before[key]), key
    assert np.array_equal(after["geo"], before["geo"])
    rs.release()


def test_out_of_frame_and_nan_spheres_render_like_the_oracle():
    sc = scenes.cover_scene(48, 36, 2, depth=8)
    rs = R.ResidentScene(sc)
    edits = {3: dict(center=[1e16, 0.0, 0.0]), 4: dict(center=[np.inf, 1.0, 0.0]), 5: dict(center=[0.0, np.nan, 0.0]),
             6: dict(radius=np.nan), 7: dict(radius=-0.2), 8: dict(radius=0.0), 9: dict(center=[2.0, 0.5, 9e14])}
    recs = [sc.set_sphere(i, **e) for i, e in edits.items()]
    rs.update_spheres(list(edits), recs)
    _check(rs, sc, what="out of frame")
    rs.release()


HOLD = 100_000_000   # clock cycles of torch.cuda._sleep (~50 ms): holds a stream back while the host enqueues behind it


class _StreamSpy:
    """The library, recording the stream handle each rtb200_scene_update_geometry_device call passes."""

    def __init__(self, L):
        self.L, self.streams = L, []

    def __getattr__(self, name):
        return getattr(self.L, name)

    def rtb200_scene_update_geometry_device(self, h, p, s):
        self.streams.append(s.value)
        return self.L.rtb200_scene_update_geometry_device(h, p, s)


def test_update_geometry_from_a_tensor_equals_the_host_form(monkeypatch):
    import torch
    spy = _StreamSpy(R.lib())
    monkeypatch.setattr(R, "_lib", spy)
    sc = scenes.cover_scene(48, 36, 2)
    a, b = R.ResidentScene(sc), R.ResidentScene(sc)
    c, r = _positions(sc)
    g = torch.tensor(np.concatenate([c, r[:, None]], axis=1), dtype=torch.float64, device="cuda")
    jitter = torch.tensor([0.2, 0.1, 0.2, 0.0], device="cuda", dtype=torch.float64)
    rng = torch.Generator(device="cuda").manual_seed(2)
    s = torch.cuda.Stream()
    for step, stream in enumerate((None, s)):
        torch.cuda.synchronize()
        with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
            torch.cuda._sleep(HOLD)                        # t is written only after the sleep: the update must wait for it
            t = g + torch.randn(g.shape, generator=rng, device="cuda", dtype=torch.float64) * jitter
            a.update_geometry(t)                           # on torch's current stream, right after t was computed
            want_stream = torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY
        assert spy.streams[-1] == want_stream, (step, spy.streams)
        torch.cuda.synchronize()                           # t was written on `stream`; the host copy below runs on another
        new = t.cpu().numpy()
        recs = [sc.set_sphere(i, center=new[i, :3].tolist(), radius=float(new[i, 3])) for i in range(sc.n_spheres)]
        b.update_spheres(list(range(sc.n_spheres)), recs)
        ra, rb = a.bvh_records(), b.bvh_records()
        assert np.array_equal(ra["geo"], new)
        for key in ("lo", "hi", "leaf_rec", "geo"):
            assert np.array_equal(ra[key], rb[key]), (step, key)
        got = _render(a)
        _assert_same(got, _render(b), f"step {step}: device form vs host form")
        _assert_same(got, _fresh(sc), f"step {step}: device form vs a fresh upload")
    assert spy.streams[0] == R.CUDA_STREAM_LEGACY                      # torch's default stream is handle 0, not the library's stream
    with pytest.raises(ValueError):
        a.update_geometry(t.float())
    with pytest.raises(ValueError):
        a.update_geometry(t[:-1])
    with pytest.raises(ValueError):
        a.update_geometry(t.cpu())
    a.release(); b.release()


def test_updates_are_ordered_between_the_frames_around_them():
    """Streams are held back with a sleep kernel so that, without the ordering, the update would run before the frames
    enqueued ahead of it (first part) or after the frames enqueued behind it (second part)."""
    import torch
    sc = scenes.cover_scene(64, 48, 4)
    old = _fresh(sc)
    rs = R.ResidentScene(sc)
    n = 64 * 48 * 3
    s1, s2, s3 = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    bufs = [torch.zeros(n, dtype=torch.uint8, device="cuda") for _ in range(4)]
    torch.cuda.synchronize()
    # 1. frames 0 and 1 wait behind sleeps; the host form enqueued after them on s3 must wait for them
    for st in (s1, s2):
        with torch.cuda.stream(st):
            torch.cuda._sleep(HOLD)
    rs.render_async(bufs[0].data_ptr(), 0, s1.cuda_stream)      # frame k on stream k mod 2: the work sets alternate with them
    rs.render_async(bufs[1].data_ptr(), 0, s2.cuda_stream)
    idx, recs = _jitter(sc, np.random.default_rng(6), 100, scale=0.6)
    rs.update_spheres(idx, recs, s3.cuda_stream)
    rs.wait()
    torch.cuda.synchronize()
    mid = _fresh(sc)
    assert not np.array_equal(old[0], mid[0])
    for k in range(2):
        assert np.array_equal(bufs[k].cpu().numpy().reshape(48, 64, 3), old[0]), f"frame {k}"
    # 2. the device form waits behind a sleep on s3; frames 2 and 3 enqueued after it must wait for it
    _jitter(sc, np.random.default_rng(7), 100, scale=0.6)
    c, r = _positions(sc)
    t = torch.tensor(np.concatenate([c, r[:, None]], axis=1), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s3):
        torch.cuda._sleep(HOLD)
    rs.update_geometry(t, s3)
    rs.render_async(bufs[2].data_ptr(), 0, s1.cuda_stream)
    rs.render_async(bufs[3].data_ptr(), 0, s2.cuda_stream)
    rs.wait()
    torch.cuda.synchronize()
    new = _fresh(sc)
    assert not np.array_equal(mid[0], new[0])
    for k in (2, 3):
        assert np.array_equal(bufs[k].cpu().numpy().reshape(48, 64, 3), new[0]), f"frame {k}"
    # a blocking frames call after an update on another stream
    out = torch.zeros(n, dtype=torch.uint8, device="cuda")
    idx2, recs2 = _jitter(sc, np.random.default_rng(8), 50, scale=0.6)
    with torch.cuda.stream(s3):
        torch.cuda._sleep(HOLD)
    rs.update_spheres(idx2, recs2, s3.cuda_stream)
    rs.render_frames([R.make_frame(sc)], out.data_ptr(), 0)
    assert np.array_equal(out.cpu().numpy().reshape(48, 64, 3), _fresh(sc)[0])
    rs.release()


def test_refused_updates_leave_the_scene_unchanged():
    sc = _light_scene(1, 4, seed=77)
    rs = R.ResidentScene(sc)
    ref = _render(rs)
    light = next(i for i in range(sc.n_spheres) if sc._spheres[i].kind == R.RT_LIGHT)
    other = (light + 1) % sc.n_spheres
    lam = R.rt_sphere.from_buffer_copy(sc._spheres[other]); lam.kind = R.RT_LAMBERTIAN; lam.center.y += 1.0
    as_light = R.rt_sphere.from_buffer_copy(lam); as_light.kind = R.RT_LIGHT
    tex = R.rt_sphere.from_buffer_copy(lam); tex.kind = R.RT_TEXTURE; tex.texture = 0     # the scene has no textures
    bad_kind = R.rt_sphere.from_buffer_copy(lam); bad_kind.kind = 9
    L = R.lib()
    cases = [([sc.n_spheres], [lam], INVALID), ([other, 2, other], [lam, lam, lam], INVALID), ([light], [lam], UNSUPPORTED),
             ([other], [as_light], UNSUPPORTED), ([other], [tex], INVALID), ([other], [bad_kind], INVALID),
             ([other, 1, light], [lam, lam, lam], UNSUPPORTED)]           # one bad record refuses the whole call
    for idx, recs, code in cases:
        arr = (R.rt_sphere * len(recs))(*recs)
        ids = (C.c_uint32 * len(idx))(*idx)
        assert L.rtb200_scene_update_spheres(rs.h, ids, arr, len(idx), None) == code, (idx, L.rtb200_last_error())
        _assert_same(_render(rs), ref, f"after the refused update {idx}")
    host = np.zeros((sc.n_spheres, 4))
    assert L.rtb200_scene_update_geometry_device(rs.h, C.c_void_p(host.ctypes.data), None) == INVALID
    _assert_same(_render(rs), ref, "after the refused device update")
    assert L.rtb200_scene_update_spheres(rs.h, None, None, 0, None) == 0                       # n == 0: a no-op
    rs.release()
