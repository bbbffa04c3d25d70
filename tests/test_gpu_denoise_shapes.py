"""Both à-trous filters on long, thin images (rtb200_denoise[_device], rtb200_denoise_var[_device]; DESIGN.md §4.15, §4.18): single
columns and rows of up to 134 M pixels, narrow strips, at the iteration counts where the grid of every h * h residue class passed
gridDim.x's limit and one pixel short of them, each held bit for bit to the numpy restatements on windows of the image.

After L iterations a pixel depends only on the pixels within R = 2 (2^L - 1) of it along each axis (the variance filter's 3 x 3
prefilter reaches one pixel further per iteration: R + L), so the restatement of a window [a - R, b + R) of the long axis,
clipped to the image, gives [a, b) exactly. The windows take in both ends of the image, where its edge and the last tiles are,
and random interior stretches. Windows do not prove that every pixel was written, so the outputs start as a NaN payload the
filters cannot produce (the RGB8 output, which has no such value, is compared with a second call's that started from another
fill), and no pixel may keep it. Inputs are made on the device from a seeded generator, with non-finite pixels, negative
variances and non-finite guides; only the windows are copied back."""
import ctypes as C
import traceback

import numpy as np
import pytest

import denoise_restatement as DR
import denoise_var_restatement as V
import rtb200 as R
from test_denoise_cpu import assert_bits_equal
from test_denoise_shapes_cpu import OVERFLOWED, one_shorter
from test_gpu_intersect import _torch

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FA5A5A5   # a quiet NaN whose payload no f32 operation makes and no input holds: an output nobody wrote
EDGE = 3000             # the window at each end of the long axis
INTERIOR = 1000         # the length of each random interior window

KW = {"denoise": dict(color_weight=16.0, albedo_weight=4.0, normal_weight=1.0),
      "denoise_var": dict(color_weight=R.DENOISE_VAR_COLOR_WEIGHT, albedo_weight=R.DENOISE_VAR_ALBEDO_WEIGHT,
                          normal_weight=R.DENOISE_VAR_NORMAL_WEIGHT, variance_floor=R.DENOISE_VAR_VARIANCE_FLOOR)}

# (width, height, iterations, what)
SHAPES = ([(w, h, L, "overflowed") for w, h, L in OVERFLOWED]
          + [(*one_shorter(w, h), L, "one_shorter") for w, h, L in OVERFLOWED]
          + [(w, h, L, "same_shape") for w, h, _ in OVERFLOWED for L in (1, 3)]
          + [(20_000_003, 2, 10, "two_rows"), (8, 5_000_011, 10, "eight_columns"), (3, 2_000_003, 10, "grid_was_legal")])


def _stream():
    torch = _torch()
    return torch.cuda.current_stream().cuda_stream or R.CUDA_STREAM_LEGACY


def _inputs(kernel, w, h, seed):
    """color, variance (None for denoise), albedo and normal as CUDA tensors [h, w, 3]. The normal guide is the albedo's buffer
    one pixel on (inputs may overlap; it saves a plane). About one colour value in 2000 is non-finite, one variance in 1000 is
    non-finite or negative, and one guide value in 8000 is non-finite."""
    torch = _torch()
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = w * h

    def scatter(t, values, every):
        flat = t.view(-1)
        idx = torch.randint(0, flat.numel(), (max(4, flat.numel() // every),), generator=g, device="cuda")
        pick = torch.randint(0, len(values), idx.shape, generator=g, device="cuda")
        flat[idx] = torch.tensor(values, dtype=torch.float32, device="cuda")[pick]

    color = torch.rand((h, w, 3), generator=g, device="cuda").pow_(3).mul_(2)
    scatter(color, [float("nan"), float("inf"), -float("inf")], 2000)
    var = None
    if kernel == "denoise_var":
        var = torch.rand((h, w, 3), generator=g, device="cuda").pow_(4).mul_(0.1)
        scatter(var, [float("nan"), float("inf"), -0.5, -1e-30], 1000)
    guides = torch.rand((n + 1) * 3, generator=g, device="cuda")
    scatter(guides, [float("nan"), float("inf")], 8000)
    return color, var, guides[: 3 * n].view(h, w, 3), guides[3:].view(h, w, 3)


def _call(kernel, w, h, L, ins, outs, scratch):
    """The device form through the C ABI into the caller's outputs (linear, rgb8, variance; any may be None)."""
    ptr = lambda t: None if t is None else t.data_ptr()
    color, var, albedo, normal = ins
    kw = KW[kernel]
    if kernel == "denoise":
        p = R.rt_denoise_params(w, h, L, 0, kw["color_weight"], kw["albedo_weight"], kw["normal_weight"], 0.0)
        rc = R.lib().rtb200_denoise_device(0, C.byref(p), ptr(color), ptr(albedo), ptr(normal), ptr(scratch), ptr(outs[0]),
                                           ptr(outs[1]), _stream())
    else:
        p = R.rt_denoise_var_params(w, h, L, 0, kw["color_weight"], kw["albedo_weight"], kw["normal_weight"], kw["variance_floor"])
        rc = R.lib().rtb200_denoise_var_device(0, C.byref(p), ptr(color), ptr(var), ptr(albedo), ptr(normal), ptr(scratch),
                                               ptr(outs[0]), ptr(outs[1]), ptr(outs[2]), _stream())
    R._check(rc)


def _windows(n, seed):
    """[a, b) windows of a long axis of length n: both ends and three random interior stretches."""
    rng = np.random.default_rng(seed)
    ws = [(0, min(n, EDGE)), (max(0, n - EDGE), n)]
    for _ in range(3):
        a = int(rng.integers(0, max(1, n - INTERIOR)))
        ws.append((a, min(n, a + INTERIOR)))
    return ws


def _restate(kernel, L, cut):
    """The restatement of the host arrays `cut` (color, var, albedo, normal): linear, variance (None for denoise)."""
    color, var, albedo, normal = cut
    if kernel == "denoise":
        return DR.denoise(color, albedo, normal, iterations=L, **KW[kernel]), None
    return V.denoise_var(color, var, albedo, normal, iterations=L, **KW[kernel])


def _reach(kernel, L):
    return 2 * ((1 << L) - 1) + (L if kernel == "denoise_var" else 0)


def check_windows(kernel, w, h, L, ins, outs, seed):
    """Each window's interior against the restatement of the window widened by the filter's reach, bit for bit."""
    along_y = h >= w   # the long axis
    n = h if along_y else w
    reach = _reach(kernel, L)

    def cut(t, a, b):
        return None if t is None else (t[a:b] if along_y else t[:, a:b]).cpu().numpy()

    for a, b in _windows(n, seed):
        lo, hi = max(0, a - reach), min(n, b + reach)
        want, want_v = _restate(kernel, L, [cut(t, lo, hi) for t in ins])
        sl = (slice(a - lo, b - lo), slice(None)) if along_y else (slice(None), slice(a - lo, b - lo))
        what = f"{kernel} {w}x{h} L={L} window [{a}, {b})"
        assert_bits_equal(cut(outs[0], a, b), want[sl], f"{what} linear")
        assert np.array_equal(cut(outs[1], a, b), DR.quantise(want[sl])), f"{what} rgb8"
        if want_v is not None:
            assert_bits_equal(cut(outs[2], a, b), want_v[sl], f"{what} variance")


def _freeing(fn, *args):
    """fn(*args), with the device memory of its tensors freed before the next case, also when it fails: a failure's traceback
    would otherwise keep its frames' tensors, up to 20 GiB, alive until pytest drops it."""
    torch = _torch()
    try:
        return fn(*args)
    except BaseException as e:
        traceback.clear_frames(e.__traceback__)
        raise
    finally:
        torch.cuda.empty_cache()


def _run(kernel, w, h, L, seed):
    """The device form with every output, checked on windows and for every pixel written; returns (ins, outs) on the device."""
    torch = _torch()
    assert w * h < 2**31
    ins = _inputs(kernel, w, h, seed)
    bytes_ = (R.lib().rtb200_denoise_scratch_bytes if kernel == "denoise" else R.lib().rtb200_denoise_var_scratch_bytes)(w, h)
    scratch = torch.empty(int(bytes_), dtype=torch.uint8, device="cuda")
    sentinel = lambda: torch.full((h, w, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    outs = [sentinel(), torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda"),
            sentinel() if kernel == "denoise_var" else None]
    _call(kernel, w, h, L, ins, outs, scratch)
    torch.cuda.synchronize()
    for name, t in zip(("linear", "variance"), (outs[0], outs[2])):
        if t is not None:
            left = int((t.view(torch.int32) == SENTINEL).sum())
            assert left == 0, f"{kernel} {w}x{h} L={L}: {left} {name} values were not written"
    check_windows(kernel, w, h, L, ins, outs, seed)
    # the RGB8 output: a second call that starts from another fill gives the same bytes, so every byte was written by both
    rgb8 = torch.full((h, w, 3), 255, dtype=torch.uint8, device="cuda")
    _call(kernel, w, h, L, ins, [None, rgb8, None], scratch)
    torch.cuda.synchronize()
    assert torch.equal(rgb8, outs[1]), f"{kernel} {w}x{h} L={L}: {int((rgb8 != outs[1]).sum())} rgb8 bytes differ between two fills"
    return ins, outs


@pytest.mark.parametrize("kernel", ["denoise", "denoise_var"])
@pytest.mark.parametrize("w,h,L", [s[:3] for s in SHAPES], ids=[f"{w}x{h}-L{L}-{what}" for w, h, L, what in SHAPES])
def test_thin_images(kernel, w, h, L):
    _freeing(_thin_image, kernel, w, h, L)


def _thin_image(kernel, w, h, L):
    _run(kernel, w, h, L, seed=w * 7919 + h * 31 + L)


@pytest.mark.parametrize("kernel", ["denoise", "denoise_var"])
def test_host_form_on_the_first_overflowing_column(kernel):
    """The host form on 1 x 33,550,337 at L = 10 writes every pixel (its outputs start as the sentinel) and equals the device
    form's bytes, which the windows and the sentinel hold to the restatement."""
    _freeing(_host_form, kernel)


def _host_form(kernel):
    torch = _torch()
    w, h, L = OVERFLOWED[0]
    ins, outs = _run(kernel, w, h, L, seed=5)
    host_in = [None if t is None else t.cpu().numpy() for t in ins]
    dev_out = [None if t is None else t.cpu().numpy() for t in outs]
    del ins, outs
    torch.cuda.empty_cache()
    got = [np.full((h, w, 3), SENTINEL, np.uint32).view(np.float32), np.zeros((h, w, 3), np.uint8),
           np.full((h, w, 3), SENTINEL, np.uint32).view(np.float32) if kernel == "denoise_var" else None]
    ptr = lambda a: None if a is None else a.ctypes.data
    st = R.rt_stats()
    kw = KW[kernel]
    color, var, albedo, normal = host_in
    if kernel == "denoise":
        p = R.rt_denoise_params(w, h, L, 0, kw["color_weight"], kw["albedo_weight"], kw["normal_weight"], 0.0)
        R._check(R.lib().rtb200_denoise(-1, C.byref(p), ptr(color), ptr(albedo), ptr(normal), ptr(got[0]), ptr(got[1]),
                                        C.byref(st)))
        assert st.as_dict()["kernel_launches"] == L + 1
    else:
        p = R.rt_denoise_var_params(w, h, L, 0, kw["color_weight"], kw["albedo_weight"], kw["normal_weight"], kw["variance_floor"])
        R._check(R.lib().rtb200_denoise_var(-1, C.byref(p), ptr(color), ptr(var), ptr(albedo), ptr(normal), ptr(got[0]),
                                            ptr(got[1]), ptr(got[2]), C.byref(st)))
        assert st.as_dict()["kernel_launches"] == 2 * L + 1
    for k, name in ((0, "linear"), (2, "variance")):
        if got[k] is not None:
            assert not (got[k].view(np.uint32) == SENTINEL).any(), f"host {name}: pixels were not written"
            assert_bits_equal(got[k], dev_out[k], f"host vs device {name}")
    assert np.array_equal(got[1], dev_out[1]), "host vs device rgb8"
