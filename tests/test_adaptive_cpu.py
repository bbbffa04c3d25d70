"""Adaptive rendering (rtb200_adaptive_*, rtb200_render_adaptive) on the host side: the rt_adaptive_params layout, argument
checks before any device is touched, and the numpy restatement of the rule (tests/adaptive_restatement.py) against the CPU
oracle and on hand-made sums at the edges of the rule. No GPU needed."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import adaptive_restatement as A
import oracle_py as O
import rtb200 as R
from rtb200 import scenes

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, NO_DEVICE = -1, -2
NEW_SYMBOLS = ["rtb200_adaptive_begin", "rtb200_adaptive_step", "rtb200_adaptive_resolve", "rtb200_render_adaptive"]


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_rt_adaptive_params_layout_matches_the_header():
    assert C.sizeof(R.rt_adaptive_params) == 24
    txt = open(os.path.join(REPO, "include", "rtb200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} rt_adaptive_params;", txt).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    ctypes_of = {"uint32_t": C.c_uint32, "float": C.c_float}
    decl = []
    for d in body.strip().rstrip(";").split(";"):
        t, names = d.split(None, 1)
        decl += [(ctypes_of[t], n.strip()) for n in names.split(",")]
    assert decl == [(t, n) for n, t in R.rt_adaptive_params._fields_]
    assert [getattr(R.rt_adaptive_params, n).offset for n, _ in R.rt_adaptive_params._fields_] == [0, 4, 8, 12, 16, 20]


def test_new_symbols_are_exported_and_listed():
    L = R.lib()
    for s in NEW_SYMBOLS:
        assert s in R.ABI_SYMBOLS and hasattr(L, s), s
        assert re.search(rf"\b{s}\(", open(os.path.join(REPO, "include", "rtb200.h")).read()), s


def _bad_params():
    good = dict(samples_per_round=4, max_samples=0, min_samples=4, reserved=0, abs_tol=0.0, rel_tol=0.1)
    cases = {"samples_per_round": dict(good, samples_per_round=0), "min_samples": dict(good, min_samples=0),
             "reserved": dict(good, reserved=1), "NaN": dict(good, abs_tol=math.nan), "NaN ": dict(good, rel_tol=math.nan)}
    return {k: R.rt_adaptive_params(**v) for k, v in cases.items()}


def test_null_arguments_are_refused():
    L = R.lib()
    p = R.make_adaptive(0.1)
    st = R.rt_stats(); active = C.c_uint32()
    assert L.rtb200_adaptive_begin(None, C.byref(p), None) == INVALID
    assert L.rtb200_adaptive_begin(None, None, None) == INVALID
    assert L.rtb200_adaptive_step(None, 1, None, C.byref(active), C.byref(st)) == INVALID
    assert L.rtb200_adaptive_resolve(None, None, None, None, None) == INVALID
    sc = scenes.cover_scene(16, 12, 4)
    out = np.zeros((12, 16, 3), np.uint8)
    assert L.rtb200_render_adaptive(None, None, C.byref(p), out.ctypes.data, None, None, C.byref(st)) == INVALID
    assert L.rtb200_render_adaptive(C.byref(sc.c), None, None, out.ctypes.data, None, None, C.byref(st)) == INVALID
    assert b"null" in L.rtb200_last_error()


@pytest.mark.parametrize("what", list(_bad_params()))
def test_bad_params_are_refused_before_any_device(what):
    L = R.lib()
    sc = scenes.cover_scene(16, 12, 4)
    st = R.rt_stats()
    assert L.rtb200_render_adaptive(C.byref(sc.c), None, C.byref(_bad_params()[what]), None, None, None, C.byref(st)) == INVALID
    assert what.strip().encode() in L.rtb200_last_error()


def test_round_size_limits_are_refused_before_any_device():
    L = R.lib()
    st = R.rt_stats()
    sc = scenes.cover_scene(16, 12, 4)
    p = R.make_adaptive(0.1, samples_per_round=4)
    opts = R.make_options(sample_buffer_bytes=4 * 16 * 12 * 16 - 1)   # one byte short of a round
    assert L.rtb200_render_adaptive(C.byref(sc.c), C.byref(opts), C.byref(p), None, None, None, C.byref(st)) == INVALID
    assert b"sample-buffer cap" in L.rtb200_last_error()
    big = scenes.cover_scene(46341, 46340, 1)   # 2147441940 pixels: two samples per round are 2^31 work ids or more
    p2 = R.make_adaptive(0.1, samples_per_round=2, min_samples=2)
    assert L.rtb200_render_adaptive(C.byref(big.c), None, C.byref(p2), None, None, None, C.byref(st)) == INVALID
    assert b"2^31" in L.rtb200_last_error()
    sc.c.samples_per_pixel = 0   # an invalid scene is still refused as such
    assert L.rtb200_render_adaptive(C.byref(sc.c), None, C.byref(p), None, None, None, C.byref(st)) == INVALID
    assert b"samples_per_pixel" in L.rtb200_last_error()


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_valid_adaptive_render_without_gpu_reports_no_device():
    with pytest.raises(R.RtError) as e:
        R.render_adaptive(scenes.cover_scene(16, 12, 4), R.make_adaptive(0.1, samples_per_round=2, min_samples=2))
    assert e.value.code == NO_DEVICE


# ---- the restatement against the oracle -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def cover():
    sc = scenes.cover_scene(40, 30, 12, depth=8)
    x, rays = A.render_samples(sc, 0, 12)
    return sc, x, rays


def test_render_samples_sum_to_the_oracle_render(cover):
    sc, x, rays = cover
    lin, img, st = O.render(sc)
    S = np.zeros(x.shape[1:], np.float32)
    for s in range(12):
        S = S + x[s]
    assert np.array_equal(np.float32(1.0) / np.float32(12) * S, lin)
    assert int(rays.astype(np.uint64).sum()) == st["rays"]


@pytest.mark.parametrize("m", [4, 5, 12], ids=["m_divides_N", "m_does_not_divide_N", "one_round"])
def test_negative_tolerances_give_the_one_shot_render(cover, m):
    sc, x, rays = cover
    want_lin, want_img, st = O.render(sc)
    got = A.run(x, rays, m, 12, 1, -1e-30, -0.5)
    assert (got["counts"] == 12).all() and got["rounds"] == -(-12 // m)
    assert np.array_equal(got["linear"].view(np.uint32), want_lin.view(np.uint32))
    assert np.array_equal(got["rgb8"], want_img)
    assert got["rays"] == st["rays"] and got["samples"] == st["samples"]


def test_each_pixel_equals_the_oracle_at_its_own_count(cover):
    sc, x, rays = cover
    got = A.run(x, rays, 2, 12, 4, 0.002, 0.05)
    counts = np.unique(got["counts"])
    assert len(counts) >= 3 and counts[0] == 4 and counts[-1] == 12, counts
    for n in counts:
        sc.c.samples_per_pixel = int(n)
        lin, img, _ = O.render(sc)
        at = got["counts"] == n
        assert np.array_equal(got["linear"][at].view(np.uint32), lin[at].view(np.uint32)), n
        assert np.array_equal(got["rgb8"][at], img[at]), n
    sc.c.samples_per_pixel = 12
    assert got["rays"] == sum(int(rays[: got["counts"][y, xx], y, xx].astype(np.uint64).sum()) for y in range(30) for xx in range(40))


# ---- hand-made sums at the edges of the rule --------------------------------------------------------------------------

def _const(v, n):
    S = np.float32(0); Q = np.float32(0)
    for _ in range(n):
        S = np.float32(S + np.float32(v)); Q = np.float32(Q + np.float32(v) * np.float32(v))
    return np.full(3, S, np.float32), np.full(3, Q, np.float32)


def test_zero_variance_stops_at_tolerance_zero():
    S, Q = _const(0.5, 8)
    assert A.leaves(8, S, Q, 100, 8, 0.0, 0.0)
    assert not A.leaves(8, S, Q, 100, 8, -1e-30, 0.0)      # a negative tolerance never stops a pixel early
    assert not A.leaves(8, S, Q, 100, 9, 0.0, 0.0)         # min_samples not reached
    assert A.leaves(100, S, Q, 100, 101, -1.0, -1.0)       # n == N always stops


def test_negative_variance_from_rounding_counts_as_zero():
    found = None
    for v in np.linspace(0.01, 0.99, 99, dtype=np.float32):
        for n in (3, 5, 7, 11, 13):
            S, Q = _const(v, n)
            inv = np.float32(1) / np.float32(n)
            mean = inv * S[0]
            if inv * Q[0] - mean * mean < 0:
                found = (v, n, S, Q)
                break
        if found:
            break
    assert found, "no constant sample sequence with a negative rounded variance"
    v, n, S, Q = found
    assert A.leaves(n, S, Q, 100, 1, 0.0, 0.0)             # err = sqrt(max(var, 0) * inv) = 0 <= 0


@pytest.mark.parametrize("bad", [math.nan, math.inf, -math.inf])
def test_non_finite_sums_run_to_max_samples(bad):
    S, Q = _const(0.5, 8)
    S[1] = bad
    assert not A.leaves(8, S, Q, 16, 1, math.inf, math.inf)
    assert A.leaves(16, S, Q, 16, 1, math.inf, math.inf)
    S, Q = _const(0.5, 8)
    Q[2] = bad
    assert not A.leaves(8, S, Q, 16, 1, math.inf, math.inf)


def test_rounds_when_m_does_not_divide_N():
    """Four pixels: constant (stops at min_samples), a NaN sample (runs to N), an infinite one (runs to N), noisy (in between)."""
    N, m = 10, 4
    x = np.full((N, 1, 4, 3), 0.25, np.float32)
    x[5, 0, 1, 0] = np.nan
    x[1, 0, 2, 2] = np.inf
    rng = np.random.default_rng(3)
    x[:, 0, 3, :] = rng.uniform(0, 1, (N, 3)).astype(np.float32)
    rays = np.ones((N, 1, 4), np.uint32)
    got = A.run(x, rays, m, N, 8, 0.0, 0.0)
    assert got["counts"].tolist() == [[8, 10, 10, 10]]
    assert got["rounds"] == 3 and got["rays"] == 38 and got["samples"] == 38
    assert np.isnan(got["linear"][0, 1, 0]) and np.isinf(got["linear"][0, 2, 2])
    part = A.run(x, rays, m, N, 8, 0.0, 0.0, rounds=1)
    assert part["counts"].tolist() == [[4, 4, 4, 4]] and part["active"] == 4
    two = A.run(x, rays, m, N, 8, 0.0, 0.0, rounds=2)
    assert two["counts"].tolist() == [[8, 8, 8, 8]] and two["active"] == 3
    lin, img = A.resolve(np.zeros((1, 2), np.uint32), np.ones((1, 2, 3), np.float32))
    assert not lin.any() and not img.any()                  # n == 0 resolves to 0
