"""Point queries without a GPU (rtb200_scene_nearest[_device], rtb200_scene_overlaps[_device], DESIGN.md §4.19): the exported
entry points, the argument checks that run before any device work, the numpy restatement against a plain-Python loop on the
contract's edge cases, and a float32 emulation of the kernel's pruned traversal with its directed roundings. The emulation
checks the soundness lemma of §4.19 directly (L~ <= dist_j for every sphere under every child it bounds), on test_bvh_cpu.py's
scenes (one offset to 7e6) and on points in the box, near and inside spheres, far away and on box faces; that the pruned
answers equal the restatement's for both kinds; and that with D~ = +inf every leaf is visited."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

import distance_restatement as DR
import rtb200 as R
from test_bvh_cpu import EMPTY, LEAF, SCENES, _spheres

f32 = np.float32
INF, NAN = float("inf"), float("nan")
FMAX = float(np.finfo(np.float32).max)
KMAX_DEPTH = 21


def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_scene_nearest_device", "rtb200_scene_nearest", "rtb200_scene_overlaps_device", "rtb200_scene_overlaps"):
        assert name in R.ABI_SYMBOLS
        assert getattr(L, name) is not None


def test_bad_arguments_are_refused_before_any_device_work():
    """A NULL handle, q, q->point or output, an rt_nearest with both outputs NULL and overlaps without q->bound are refused
    with RT_ERR_INVALID. The checks come before the handle is used, so a stand-in handle that is never dereferenced shows it."""
    L = R.lib()
    p = np.zeros((1, 3)); b = np.ones(1)
    dist = np.full(1, 7.0); sph = np.full(1, 7, np.uint32); ov = np.full(1, 7, np.uint8)
    q = R.rt_points(p.ctypes.data, b.ctypes.data)
    out = R.rt_nearest(dist.ctypes.data, sph.ctypes.data)
    st = R.rt_stats()
    assert L.rtb200_scene_nearest(None, C.byref(q), 1, C.byref(out), C.byref(st)) == -1
    assert b"handle" in L.rtb200_last_error()
    assert L.rtb200_scene_nearest_device(None, C.byref(q), 1, C.byref(out), None) == -1
    assert b"handle" in L.rtb200_last_error()
    assert L.rtb200_scene_overlaps(None, C.byref(q), 1, ov.ctypes.data, C.byref(st)) == -1
    assert L.rtb200_scene_overlaps_device(None, C.byref(q), 1, ov.ctypes.data, None) == -1
    assert b"handle" in L.rtb200_last_error()
    fake = C.c_void_p(C.addressof(C.create_string_buffer(64)))
    nearest = [(None, out, b"q or out"), (q, None, b"q or out"), (R.rt_points(None, b.ctypes.data), out, b"q->point"),
               (R.rt_points(p.ctypes.data, None), R.rt_nearest(None, None), b"every output")]
    for qq, oo, what in nearest:
        qp = C.byref(qq) if qq is not None else None
        op = C.byref(oo) if oo is not None else None
        assert L.rtb200_scene_nearest(fake, qp, 1, op, C.byref(st)) == -1
        assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
        assert L.rtb200_scene_nearest_device(fake, qp, 1, op, None) == -1
        assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
    overlaps = [(None, ov.ctypes.data, b"q or out"), (R.rt_points(None, b.ctypes.data), ov.ctypes.data, b"q->point"),
                (R.rt_points(p.ctypes.data, None), ov.ctypes.data, b"q->bound"), (q, None, b"overlaps is null")]
    for qq, o, what in overlaps:
        qp = C.byref(qq) if qq is not None else None
        assert L.rtb200_scene_overlaps(fake, qp, 1, o, C.byref(st)) == -1
        assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
        assert L.rtb200_scene_overlaps_device(fake, qp, 1, o, None) == -1
        assert what in L.rtb200_last_error(), (what, L.rtb200_last_error())
    assert dist[0] == 7.0 and sph[0] == 7 and ov[0] == 7


# ---- the restatement against the contract as a plain loop ----

def _loop(p, c, r, b):
    """The contract with Python floats (IEEE double, round to nearest, left to right): (sphere or -1, distance)."""
    best, bd = -1, INF
    for j in range(len(r)):
        x, y, z = float(p[0]) - float(c[j][0]), float(p[1]) - float(c[j][1]), float(p[2]) - float(c[j][2])
        s = math.sqrt((x * x + y * y) + z * z)
        d = s - abs(float(r[j]))
        if d < b and (best < 0 or d < bd):
            best, bd = j, d
    return best, bd


def _edge_spheres():
    c = [(0, 0, 0), (0, 0, 0), (2, 0, 0), (-2, 0, 0), (0, 3, 0), (0, -3, 0), (5, 5, 5), (1, 1, 1), (0, 0, 1000.5),
         (7, 0, 0), (INF, 0, 0), (0, NAN, 0), (0, 0, -4), (0, 0, -9), (1e15, 0, 0), (3, 3, 0), (-1e-300, 0, 0)]
    r = [1.0, 1.0, 0.5, 0.5, -1.0, 1.0, 0.0, -0.0, 1000.0, NAN, 1.0, 1.0, INF, -INF, 1e15 - 5.0, 2.0, 5e-324]
    return np.array(c, np.float64), np.array(r, np.float64)


def _edge_points(c, r, rng):
    pts = [(0, 0, 0), (2, 0, 0), (2.5, 0, 0), (0, 2, 0), (1, 0, 0), (-1, 0, 0), (0, 0, 0.5), (5, 5, 5), (1, 1, 1), (0, 0, 0.5),
           (NAN, 0, 0), (INF, 0, 0), (-INF, 1, 1), (0, 0, INF), (1e300, 0, 0), (-1e300, -1e300, 1e300), (0, 0, 1e-300),
           (-0.0, -0.0, -0.0), (3, 0, 0), (3, 3, 2), (1e15, 0, 0)]
    for j in range(len(r)):   # at the centre, and exactly on the surface along each axis
        if np.isfinite(c[j]).all():
            pts.append(tuple(c[j]))
            if np.isfinite(r[j]):
                for a in range(3):
                    q = c[j].copy(); q[a] += abs(r[j]); pts.append(tuple(q))
    pts += [tuple(x) for x in rng.normal(size=(40, 3)) * 4]
    return np.array(pts, np.float64)


@pytest.mark.parametrize("drop", [None, "lights_and_nonfinite", "all"])
def test_the_restatement_is_the_contract(drop):
    c, r = _edge_spheres()
    if drop == "lights_and_nonfinite":
        keep = np.isfinite(c).all(axis=1) & np.isfinite(r)
        c, r = c[keep], r[keep]
    elif drop == "all":
        c, r = c[:0], r[:0]
    rng = np.random.default_rng(3)
    p = _edge_points(*_edge_spheres(), rng)
    bounds = [None, 0.0, -0.0, -1.0, 0.5, 1.0, INF, -INF, NAN, float(np.finfo(np.float64).max), 1e-300]
    seen_tie = seen_none = seen_inside = 0
    for b in bounds:
        bv = np.full(len(p), INF if b is None else b)
        sph, dist = DR.nearest(p, c, r, None if b is None else bv)
        for i in range(len(p)):
            j, d = _loop(p[i], c, r, bv[i])
            assert sph[i] == j, (b, p[i], sph[i], j)
            assert np.float64(dist[i]).tobytes() == np.float64(d).tobytes(), (b, p[i], dist[i], d)
            seen_none += j < 0
            seen_inside += j >= 0 and d < 0
        ov = DR.overlaps(p, bv, c, r)
        assert np.array_equal(ov, (sph >= 0).astype(np.uint8))
    if drop != "all":
        # ties: the duplicate spheres 0 and 1 and the mirrored 2 and 3 answer with the lower index
        s, d = DR.nearest(np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 0.1]]), c[:4], r[:4])
        assert s[0] == 0 and s[1] == 0 and d[0] == -1.0
        s, _ = DR.nearest(np.array([[0.0, 10.0, 0.0]]), c[2:4], r[2:4])
        assert s[0] == 0
        seen_tie = 1
    assert seen_none and (drop == "all" or (seen_inside and seen_tie))


def test_nonfinite_points_and_bounds_give_none():
    c, r = _edge_spheres()
    p = np.array([[NAN, 0, 0], [0, 0, 0], [0, 0, 0]])
    s, d = DR.nearest(p, c, r, np.array([1.0, NAN, -INF]))
    assert (s == -1).all() and np.isinf(d).all() and (d > 0).all()


# ---- the float32 emulation of the pruned traversal ----

def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _to32(x, e, up):
    """x + e (float64 x, a TwoSum error e) rounded down (or up) to float32."""
    with np.errstate(over="ignore"):
        f = f32(x)
        if up:
            if float(f) < x or (float(f) == x and e > 0):
                f = np.nextafter(f, f32(INF))
        else:
            if float(f) > x or (float(f) == x and e < 0):
                f = np.nextafter(f, f32(-INF))
    return f32(f)


def sub32(a, b, up=False):
    return _to32(*_two_sum(float(a), -float(b)), up)


def add32(a, b, up=False):
    return _to32(*_two_sum(float(a), float(b)), up)


def mul32(a, b, up=False):
    return _to32(float(a) * float(b), 0.0, up)   # the product of two float32 is exact in float64


def sqrt32(a, up=False):
    f = f32(math.sqrt(float(a)))
    if up:
        if float(f) * float(f) < float(a):
            f = np.nextafter(f, f32(INF))
    elif float(f) * float(f) > float(a):
        f = np.nextafter(f, f32(-INF))
    return f32(f)


def rn32(x: Fraction) -> f32:
    """The exact value x rounded to the nearest float32, ties to even (+-inf past FLT_MAX + half an ulp)."""
    if x == 0:
        return f32(0.0)
    if abs(x) >= Fraction(FMAX) + Fraction(2) ** 103:
        return f32(INF if x > 0 else -INF)
    with np.errstate(over="ignore"):
        f = f32(float(x))                        # within one float32 step of the answer (float() rounds once more)
    if not np.isfinite(f):
        f = f32(FMAX if x > 0 else -FMAX)
    near = [g for g in (np.nextafter(f, f32(-INF)), f, np.nextafter(f, f32(INF))) if np.isfinite(g)]
    return f32(min(near, key=lambda g: (abs(Fraction(float(g)) - x), int(np.array(g).view(np.uint32)) & 1)))


def fma32(a, b, c) -> f32:
    """fmaf(a, b, c): the exact a*b + c rounded once to the nearest float32."""
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        with np.errstate(over="ignore", invalid="ignore"):
            return f32(float(a) * float(b) + float(c))
    return rn32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def oo32(pf) -> f32:
    """The kernel's |pf|^2: fmaf(ofx, ofx, fmaf(ofy, ofy, ofz * ofz)), one rounding per FMA (a float64 sum rounded to float32
    rounds twice and can land on the other side of a float32 midpoint)."""
    with np.errstate(over="ignore"):
        zz = f32(pf[2]) * f32(pf[2])
    return fma32(pf[0], pf[0], fma32(pf[1], pf[1], zz))


def d_up(x: float) -> f32:
    """__double2float_ru."""
    if math.isnan(x):
        return f32(NAN)
    if x == -INF:
        return f32(-INF)
    if x < -FMAX:
        return f32(-FMAX)
    return _to32(x, 0.0, True)


def slack_of(pf):
    nrm = sqrt32(add32(add32(mul32(pf[0], pf[0], True), mul32(pf[1], pf[1], True), True), mul32(pf[2], pf[2], True), True), True)
    return add32(mul32(f32(2.0 ** -23), nrm, True), f32(1e-30), True)


def lower_bound(pf, lo, hi, slack):
    """The kernel's L~ of one child box: the distance from pf rounded down, minus the slack; -inf when it is not positive."""
    e = [max(max(sub32(lo[a], pf[a]), sub32(pf[a], hi[a])), f32(0)) for a in range(3)]
    s = add32(add32(mul32(e[0], e[0]), mul32(e[1], e[1])), mul32(e[2], e[2]))
    lv = sub32(sqrt32(s), slack)
    return lv if lv > 0 else f32(-INF)


def _subtrees(b):
    """Member spheres under each (node, child)."""
    memo = {}

    def under(ref):
        if ref & LEAF:
            ids = b["leaf_id"][ref & 0x7FFFFFFF]
            return ids[ids != EMPTY].tolist()
        if ref not in memo:
            memo[ref] = [j for k in b["child"][ref] if k != EMPTY for j in under(int(k))]
        return memo[ref]
    return under


def emulate(b, c, r, p, bound, any_, stop=True, under=None, d_all=None, info=None):
    """The kernel of one point in emulated float32 and exact float64. Returns (sphere or -1, distance, evaluated spheres, leaves
    visited). With `under` and `d_all` it also asserts L~ <= dist_j for every sphere under every child it bounds; a dict
    `info` receives "stack", the most entries the traversal stack held, and "tree", whether the point walked the tree."""
    g = b["recentre"]
    best, bj = bound, -1
    evald, leaves = [], 0

    def ev(j):
        nonlocal best, bj
        d = d_all[j]
        evald.append(j)
        if any_:
            if d < bound:
                bj = j
        elif d < best or (d == best and bj >= 0 and j < bj):
            best, bj = d, j

    if not bound > -INF:
        return bj, INF, evald, leaves
    pf = np.array([f32(p[a] - g[a]) for a in range(3)])
    tree = bool(oo32(pf) < f32(1e30))
    if info is not None:
        info["stack"], info["tree"] = 0, tree
    if not tree:
        for j in range(len(r)):
            ev(j)
            if any_ and stop and bj >= 0:
                break
        return bj, (best if bj >= 0 else INF), evald, leaves
    for j in b["always"].tolist():
        if any_ and stop and bj >= 0:
            break
        ev(j)
    slack = slack_of(pf)
    stack = [(0, f32(-INF))] if b["n_nodes"] and not (any_ and stop and bj >= 0) else []
    while stack:
        assert len(stack) <= 7 * KMAX_DEPTH + 1
        ref, lt = stack.pop()
        dt = d_up(best) if not any_ else d_up(bound)
        if lt > dt:
            continue
        if ref & LEAF:
            leaves += 1
            for j in b["leaf_id"][ref & 0x7FFFFFFF].tolist():
                if j != EMPTY and not (any_ and stop and bj >= 0):
                    ev(j)
            if any_ and stop and bj >= 0:
                break
            continue
        lo, hi = b["lo"][ref], b["hi"][ref]
        kept = []
        for k in range(8):
            child = int(b["child"][ref][k])
            if child == EMPTY:
                continue
            lv = lower_bound(pf, lo[:, k], hi[:, k], slack)
            if under is not None:
                ds = d_all[under(child)]
                ds = ds[~np.isnan(ds)]
                assert len(ds) == 0 or float(lv) <= ds.min(), (p, child, lv, ds.min())
            if not lv > dt:
                kept.append((lv, k, child))
        kept.sort(key=lambda t: (t[0], t[1]), reverse=True)   # the nearest child on top
        stack.extend((child, lv) for lv, _, child in kept)
        assert len(stack) <= 7 * KMAX_DEPTH + 1
        if info is not None:
            info["stack"] = max(info["stack"], len(stack))
    return bj, (best if bj >= 0 else INF), evald, leaves


def _families(sc, b, c, r, rng, k):
    """Points uniform in the box of the centres, near surfaces, inside spheres, far away and on the faces of child boxes."""
    fin = np.isfinite(c).all(axis=1) & np.isfinite(r)
    cc, rr = c[fin], np.abs(r[fin])
    lo, hi = cc.min(axis=0), cc.max(axis=0)
    ext = float(np.max(hi - lo)) + 1.0
    u = rng.normal(size=(k, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    j = rng.integers(0, len(rr), size=k)
    box = lo + rng.uniform(size=(k, 3)) * (hi - lo)
    near = cc[j] + u * (rr[j] * (1 + rng.uniform(-1e-6, 1e-6, size=k)) + rng.uniform(-1e-3, 1e-3, size=k))[:, None]
    inside = cc[j] + u * (rr[j] * rng.uniform(0, 0.999, size=k))[:, None]
    far = (lo + hi) / 2 + u * ext * 10.0 ** rng.uniform(1, 6, size=k)[:, None]
    faces = []
    g = b["recentre"]
    for _ in range(k):
        node = int(rng.integers(b["n_nodes"]))
        ks = [q for q in range(8) if b["child"][node][q] != EMPTY]
        q = ks[int(rng.integers(len(ks)))]
        blo, bhi = b["lo"][node][:, q].astype(np.float64), b["hi"][node][:, q].astype(np.float64)
        pt = blo + rng.uniform(size=3) * (bhi - blo)
        a = int(rng.integers(3))
        pt[a] = blo[a] if rng.uniform() < 0.5 else bhi[a]
        faces.append(pt + g)
    return {"box": box, "near": near, "inside": inside, "far": far, "faces": np.array(faces)}


@pytest.mark.parametrize("mk", SCENES[:4])
def test_the_pruned_traversal_never_prunes_an_answer(mk):
    sc = mk()
    b = R.bvh_records(sc)
    c, r = _spheres(sc)
    under = _subtrees(b)
    rng = np.random.default_rng(41)
    checked_inside = checked_ov = 0
    for fam, pts in _families(sc, b, c, r, rng, 24).items():
        d_pts = DR.distances(pts, c, r)
        for i, p in enumerate(pts):
            d_all = d_pts[i]
            # nearest, unbounded and under a bound just above the answer, at it and below it
            want_j, want_d = DR.nearest(p[None], c, r)
            got = emulate(b, c, r, p, INF, False, under=under, d_all=d_all)
            assert (got[0], got[1]) == (want_j[0], want_d[0]), (fam, p, got[:2], want_j, want_d)
            checked_inside += want_d[0] < 0
            dstar = float(want_d[0])
            for bound in (np.nextafter(dstar, INF), dstar, np.nextafter(dstar, -INF), abs(dstar) * 2 + 0.1, 0.0):
                wj, wd = DR.nearest(p[None], c, r, np.array([bound]))
                got = emulate(b, c, r, p, float(bound), False, d_all=d_all)
                assert (got[0], got[1]) == (wj[0], wd[0]), (fam, p, bound)
            # overlaps: without the early stop every sphere with dist_j < r is evaluated; with it the answer is the restatement's
            for rad in (0.0, max(dstar, 0.0) * 1.5 + 1e-3, np.nextafter(max(dstar, 0.0), INF)):
                want = {j for j in range(len(r)) if d_all[j] < rad}
                got = emulate(b, c, r, p, float(rad), True, stop=False, d_all=d_all)
                assert want <= set(got[2]), (fam, p, rad, sorted(want - set(got[2])))
                assert (emulate(b, c, r, p, float(rad), True, d_all=d_all)[0] >= 0) == bool(want)
                checked_ov += bool(want)
    assert checked_inside > 10 and checked_ov > 50


@pytest.mark.parametrize("mk", [SCENES[0], SCENES[3]])
def test_without_a_bound_every_leaf_is_visited(mk):
    """D~ = +inf (an overlaps query of radius +inf without its early stop) prunes nothing: every leaf and every sphere."""
    sc = mk()
    b = R.bvh_records(sc)
    c, r = _spheres(sc)
    rng = np.random.default_rng(42)
    for p in _families(sc, b, c, r, rng, 4)["box"]:
        _, _, evald, leaves = emulate(b, c, r, p, INF, True, stop=False, d_all=DR.distances(p[None], c, r)[0])
        assert leaves == b["n_leaves"]
        assert sorted(evald) == list(range(sc.n_spheres))


def test_the_directed_roundings_are_exact():
    """sub32, add32, mul32, sqrt32 (the kernel's __f*_rd / __f*_ru) and d_up (__double2float_ru) against exact rationals: the
    result is on the right side of the exact value and one float32 step back is on the wrong side."""
    rng = np.random.default_rng(7)
    vals = np.concatenate([rng.normal(size=300) * 10.0 ** rng.uniform(-30, 15, size=300), [0.0, 1.0, 3.0, 1e15, 7e6, 1e-30]])
    xs = vals.astype(f32)
    for k in range(len(xs) - 1):
        a, bb = xs[k], xs[k + 1]
        for up in (False, True):
            for f, exact in ((sub32(a, bb, up), Fraction(float(a)) - Fraction(float(bb))),
                             (add32(a, bb, up), Fraction(float(a)) + Fraction(float(bb))),
                             (mul32(a, bb, up), Fraction(float(a)) * Fraction(float(bb)))):
                if not np.isfinite(f):
                    continue
                back = np.nextafter(f, f32(-INF) if up else f32(INF))
                if up:
                    assert Fraction(float(f)) >= exact and Fraction(float(back)) < exact
                else:
                    assert Fraction(float(f)) <= exact and Fraction(float(back)) > exact
            s = abs(a)
            q = sqrt32(s, up)
            back = np.nextafter(q, f32(-INF) if up else f32(INF))
            if up:
                assert Fraction(float(q)) ** 2 >= Fraction(float(s)) and (q == 0 or Fraction(float(back)) ** 2 < Fraction(float(s)))
            else:
                assert Fraction(float(q)) ** 2 <= Fraction(float(s)) and Fraction(float(back)) ** 2 > Fraction(float(s))
    for x in list(rng.normal(size=500) * 10.0 ** rng.uniform(-40, 40, size=500)) + [0.0, -0.0, 1e39, -1e39, 1e300, -1e300, 5e-324]:
        f = d_up(float(x))
        assert Fraction(float(f)) >= Fraction(x) if np.isfinite(f) else f > 0
        if np.isfinite(f) and f > -FMAX:
            assert Fraction(float(np.nextafter(f, f32(-INF)))) < Fraction(x)
    assert d_up(INF) == INF and d_up(float(np.finfo(np.float64).max)) == INF and d_up(-INF) == -INF


def test_oo_rounds_once_per_fma():
    """oo32 is the kernel's fmaf chain: on random points it is the exact sum of squares rounded once per FMA, and at a float32
    midpoint it differs from a float64 sum rounded to float32. pf_y^2 = 2^2k (1 + 2^-11 + 2^-24) lies exactly half way between
    two float32 values; pf_z^2 = 2^(2k-80) lifts it above, which the float64 sum loses before its rounding to float32."""
    rng = np.random.default_rng(9)
    for pf in (rng.normal(size=(300, 3)) * 10.0 ** rng.uniform(-20, 18, size=(300, 3))).astype(f32):
        zz = pf[2] * pf[2]
        inner = rn32(Fraction(float(pf[1])) ** 2 + Fraction(float(zz)))
        assert oo32(pf) == rn32(Fraction(float(pf[0])) ** 2 + Fraction(float(inner)))
    for k in (0, 49):                                      # 2^49 (1 + 2^-12) is about 5.6e14: |pf|^2 near 1e30
        pf = np.array([0.0, 2.0 ** k * (1 + 2.0 ** -12), 2.0 ** (k - 40)], f32)
        twice = f32(float(pf[1]) * float(pf[1]) + float(f32(float(pf[2]) * float(pf[2]))))
        assert float(oo32(pf)) == 4.0 ** k * (1 + 2.0 ** -11 + 2.0 ** -23) and float(twice) == 4.0 ** k * (1 + 2.0 ** -11)


def test_lower_bound_is_a_lower_bound_of_the_box_distance():
    """L~ against the exact distance from the unrounded point to the stored box, for random boxes and points: L~ <= it, and
    L~ = -inf when the point is inside the box."""
    rng = np.random.default_rng(8)
    for _ in range(3000):
        s = 10.0 ** rng.uniform(-3, 7)
        lo = (rng.normal(size=3) * s).astype(f32)
        hi = (lo.astype(np.float64) + rng.uniform(0, s, size=3)).astype(f32)
        hi = np.maximum(hi, lo)
        q = rng.normal(size=3) * s * rng.choice([0.1, 1.0, 3.0])
        pf = q.astype(f32)
        lv = lower_bound(pf, lo, hi, slack_of(pf))
        gap = [max(Fraction(float(lo[a])) - Fraction(q[a]), Fraction(q[a]) - Fraction(float(hi[a])), Fraction(0)) for a in range(3)]
        sq = sum(x * x for x in gap)
        inside = all(lo[a] <= pf[a] <= hi[a] for a in range(3))
        if inside:
            assert lv == -INF
        elif lv != -INF:
            assert Fraction(float(lv)) ** 2 <= sq
