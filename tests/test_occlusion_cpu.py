"""Occlusion queries without a GPU (rtb200_scene_occluded[_device], DESIGN.md §4.11): the exported entry points, the argument
checks that run before any device work, and a float32 emulation of the pruned traversal. The emulation extends
tests/test_bvh_cpu.py's `_traverse` by the one thing the any-hit kind adds to the node step, the per-ray bound T~ on the
distance along d^: a child is entered iff max(t_near, 0) <= min(t_far, T~). It checks, on that file's scenes (one offset to
7e6) and ray families, with |d| from 1e-10 to 1e10 and bounds at and around the exact roots, that no sphere the exact test
accepts below T is ever pruned, and that the bound does prune short segments."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

import rtb200 as R
from test_bvh_cpu import LEAF, SCENES, U, _exact_hits, _fma, _spheres, _traverse

f32 = np.float32
MAX = float(np.finfo(np.float64).max)


def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_scene_occluded_device", "rtb200_scene_occluded"):
        assert name in R.ABI_SYMBOLS
        assert getattr(L, name) is not None


def test_bad_arguments_are_refused_before_any_device_work():
    """A NULL handle, NULL rays, a NULL origin or direction and a NULL output are refused with RT_ERR_INVALID. The checks
    come before the handle is used, so a stand-in handle that is never dereferenced shows the order."""
    L = R.lib()
    o = np.zeros((1, 3)); d = np.ones((1, 3)); occ = np.full(1, 7, np.uint8)
    rays = R.rt_rays(o.ctypes.data, d.ctypes.data, None)
    st = R.rt_stats()
    assert L.rtb200_scene_occluded(None, C.byref(rays), 1, occ.ctypes.data, C.byref(st)) == -1
    assert b"handle" in L.rtb200_last_error()
    assert L.rtb200_scene_occluded_device(None, C.byref(rays), 1, occ.ctypes.data, None) == -1
    assert b"handle" in L.rtb200_last_error()
    fake = C.c_void_p(C.addressof(C.create_string_buffer(64)))
    cases = [(None, occ.ctypes.data, b"rays"),
             (R.rt_rays(None, d.ctypes.data, None), occ.ctypes.data, b"origin"),
             (R.rt_rays(o.ctypes.data, None, None), occ.ctypes.data, b"direction"),
             (rays, None, b"occluded")]
    for r, out, what in cases:
        rp = C.byref(r) if r is not None else None
        assert L.rtb200_scene_occluded(fake, rp, 1, out, C.byref(st)) == -1
        assert what in L.rtb200_last_error()
        assert L.rtb200_scene_occluded_device(fake, rp, 1, out, None) == -1
        assert what in L.rtb200_last_error()
    assert occ[0] == 7


def _up(x: float, exact: Fraction) -> float:
    """x if it is >= the exact value, else the next double up: x rounded to nearest becomes the value rounded up."""
    return x if Fraction(x) >= exact else float(np.nextafter(x, np.inf))


def tcap(t: float, d) -> f32:
    """The kernel's T~: __double2float_ru(__dmul_ru(__dmul_ru(T, __dsqrt_ru(|d|^2)), 1 + 2^-40)), |d|^2 as rtd::dot."""
    a = float(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
    s = float(np.sqrt(a))
    s = s if Fraction(s) ** 2 >= Fraction(a) else float(np.nextafter(s, np.inf))
    m = 1.0 + 2.0 ** -40
    if not np.isfinite(t * s * m):
        return f32(np.inf)
    p = _up(t * s, Fraction(t) * Fraction(s))
    q = _up(p * m, Fraction(p) * Fraction(m))
    if not np.isfinite(q):
        return f32(np.inf)
    with np.errstate(over="ignore"):
        f = f32(q)
    if np.isfinite(f) and float(f) < q:
        f = np.nextafter(f, f32(np.inf))
    return f32(f)


def _bounded(b, o, d, tc):
    """The any-hit node step in emulated float32: `_traverse`'s per-ray constants and tests, with t_far capped by tc."""
    g = b["recentre"]
    of = (o - g).astype(f32)
    df = d.astype(f32)
    s = _fma(df[0], df[0], _fma(df[1], df[1], f32(df[2] * df[2])))
    oo = _fma(of[0], of[0], _fma(of[1], of[1], f32(of[2] * of[2])))
    assert 1e-30 < s < 1e30 and oo < 1e30
    dn = (df * f32(1.0 / np.sqrt(np.float64(s)))).astype(f32)
    nod = f32(-_fma(of[0], dn[0], _fma(of[1], dn[1], f32(of[2] * dn[2]))))
    thr = f32(np.nextafter(f32(oo * f32(1.0 - 96.0 * U)), f32(-np.inf)))
    ax = np.where(np.abs(dn) < f32(1e-20), np.copysign(f32(1e-20), dn), dn).astype(f32)
    inv = (f32(1.0) / ax).astype(f32)
    mray = f32(np.nextafter(f32(f32(1.9073486328125e-6) * f32(np.nextafter(np.sqrt(oo, dtype=f32), f32(np.inf)))), f32(np.inf)))
    sm = np.copysign(mray, inv).astype(f32)
    cn = ((of + sm).astype(f32) * (-inv)).astype(f32)
    cf = ((of - sm).astype(f32) * (-inv)).astype(f32)
    neg = np.signbit(inv)
    cands, stack, visited = [], [0], 0
    while stack:
        node = stack.pop(); visited += 1
        lo, hi = b["lo"][node], b["hi"][node]
        near = np.where(neg[:, None], hi, lo); far = np.where(neg[:, None], lo, hi)
        tn = np.stack([_fma(near[a], inv[a], cn[a]) for a in range(3)]).max(axis=0)
        tf = np.stack([_fma(far[a], inv[a], cf[a]) for a in range(3)]).min(axis=0)
        hit = np.maximum(tn, f32(0)) <= np.minimum(tf, tc)
        for k in np.nonzero(hit)[0]:
            ref = int(b["child"][node][k])
            if ref & LEAF:
                leaf = ref & 0x7FFFFFFF
                rec = b["leaf_rec"][leaf]
                cx = np.stack([rec[:, 0, 0], rec[:, 0, 1]], 1).ravel(); cy = np.stack([rec[:, 0, 2], rec[:, 0, 3]], 1).ravel()
                cz = np.stack([rec[:, 1, 0], rec[:, 1, 1]], 1).ravel(); nk = np.stack([rec[:, 1, 2], rec[:, 1, 3]], 1).ravel()
                bb = _fma(cx, dn[0], _fma(cy, dn[1], _fma(cz, dn[2], nod)))
                tt = _fma(cx, f32(2) * of[0], _fma(cy, f32(2) * of[1], _fma(cz, f32(2) * of[2], nk)))
                with np.errstate(invalid="ignore", over="ignore"):
                    D = _fma(bb, bb, tt)
                ids = b["leaf_id"][leaf]
                cands.extend(ids[(D >= thr) & (ids != 0xFFFFFFFF)].tolist())
            else:
                stack.append(ref)
    return set(cands) | set(b["always"].tolist()), visited


def _roots(c, r, o, d):
    """Each sphere's root under f64::MAX (sphere.rs:46-58, t_min 0.001), NaN where it accepts none."""
    oc = o - c
    a = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
    hb = oc @ d
    cc = (oc * oc).sum(axis=1) - r * r
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        disc = hb * hb - a * cc
        sq = np.sqrt(np.where(disc >= 0, disc, 0.0))
        r1, r2 = (-hb - sq) / a, (-hb + sq) / a
    root = np.where((disc >= 0) & (r1 > 0.001) & (r1 < MAX), r1, np.where((disc >= 0) & (r2 > 0.001) & (r2 < MAX), r2, np.nan))
    return root


def _rays(sc, c, r, rng, k):
    """test_bvh_cpu's families: primary-like from the camera, scattered from surfaces, grazing and axis-parallel; |d| spans
    1e-10 to 1e10."""
    cam = np.array([sc.c.camera.origin.x, sc.c.camera.origin.y, sc.c.camera.origin.z])
    out = []
    for i in range(k):
        j = int(rng.integers(len(r)))
        if i % 4 == 0:
            o = cam
            d = (c[j] + rng.normal(size=3) * abs(r[j]) * 0.7) - o
        else:
            nrm = rng.normal(size=3); nrm /= np.linalg.norm(nrm)
            o = c[j] + nrm * abs(r[j])
            d = nrm + rng.normal(size=3) * 0.8
            if i % 8 == 1:
                d = d * np.array([1.0, 1e-9, 1.0])
            if i % 16 == 3:
                d = np.array([0.0, 0.0, 1.0]) * (1 if i % 32 == 3 else -1)
        out.append((o, d * 10.0 ** rng.uniform(-10, 10)))
    return out


@pytest.mark.parametrize("mk", SCENES[:4])
def test_the_bound_never_prunes_a_sphere_the_exact_test_accepts_below_it(mk):
    sc = mk()
    b = R.bvh_records(sc)
    c, r = _spheres(sc)
    rng = np.random.default_rng(23)
    checked = 0
    for o, d in _rays(sc, c, r, rng, 120):
        root = _roots(c, r, o, d)
        acc = np.flatnonzero(~np.isnan(root))
        assert sorted(acc.tolist()) == sorted(_exact_hits(c, r, o, d).tolist())
        # the unbounded emulation is test_bvh_cpu's own traversal
        assert _bounded(b, o, d, f32(np.inf)) == _traverse(b, o, d)
        rs = root[acc] if len(acc) else np.array([1.0])
        r0 = float(rs[rng.integers(len(rs))])
        u = np.nextafter(0.001, 1.0)
        bounds = [r0, np.nextafter(r0, np.inf), np.nextafter(r0, -np.inf), r0 * rng.uniform(0, 1), r0 * rng.uniform(1, 4),
                  0.001, u, np.nextafter(u, 1.0), MAX]
        for t in bounds:
            t = float(t)
            want = set(acc[root[acc] < t].tolist())
            if not t > 0.001:
                assert not want   # an accepted root is > 0.001: such a ray does not enter the traversal
                continue
            cand, _ = _bounded(b, o, d, tcap(t, d))
            missing = want - cand
            assert not missing, (o, d, t, sorted(missing))
            checked += len(want)
    assert checked > 150


def test_tcap_rounds_up_and_saturates():
    rng = np.random.default_rng(5)
    for _ in range(2000):
        d = rng.normal(size=3) * 10.0 ** rng.uniform(-10, 10)
        t = float(10.0 ** rng.uniform(-3, 300))
        tc = tcap(t, d)
        exact = Fraction(t) * Fraction(float(np.linalg.norm(d)))
        assert tc == np.inf or Fraction(float(tc)) >= exact * (1 - Fraction(1, 2 ** 50))
        assert tc == np.inf or Fraction(float(tc)) <= exact * (1 + Fraction(1, 2 ** 20))
    assert tcap(MAX, np.array([1.0, 0.0, 0.0])) == np.inf


@pytest.mark.parametrize("mk", [SCENES[0], SCENES[2]])
def test_the_bound_prunes_short_segments(mk):
    """Segments of length <= 0.5 from surface points (t_max 1): the pruned traversal visits fewer nodes than the unbounded
    one on the same rays. The 8-wide trees are 3-4 levels deep and a segment still visits the path down to its own sphere's
    leaf, so the saving is the part of the tree beyond the segment: 7 % here (365 of 392 and 467 of 501 nodes)."""
    sc = mk()
    b = R.bvh_records(sc)
    c, r = _spheres(sc)
    rng = np.random.default_rng(29)
    pruned = full = 0
    for _ in range(150):
        j = int(rng.integers(len(r)))
        nrm = rng.normal(size=3); nrm /= np.linalg.norm(nrm)
        o = c[j] + nrm * abs(r[j])
        g = nrm + rng.normal(size=3); g /= np.linalg.norm(g)
        d = g * rng.uniform(0.01, 0.5)
        full += _traverse(b, o, d)[1]
        pruned += _bounded(b, o, d, tcap(1.0, d))[1]
    assert pruned < 0.95 * full, (pruned, full)
