"""Point families where the pruning of the point queries (rtb200_scene_nearest / rtb200_scene_overlaps, DESIGN.md §4.19) is
tight, shared by tests/test_distance_far_cpu.py, tests/test_gpu_distance_far.py and tests/distance_far_worker.py. Everything
is deterministic: the scenes are fixed by their names, the families by their scene, the records they aim at and a seed.

Families (families(sc, recs, seed)): name -> {"p": float64 [n, 3], and what the family's reach check reads}:
  box_face    points whose recentred f32 coordinate lies on a stored child plane or 1-4 f32 ulps either side of it, and points
              whose f64 p - g lies 1/8 .. 3/8 of an f32 ulp off the plane while fl32(p - g) rounds onto it
  near_tie    points far out (10x .. 1e6x the pair's extent) on the bisector of two spheres under different children of a node
              (or of the root), nudged by f64 ulps, whose two f64 distances are the least of the scene and differ by 0 to 4 ulps
  inside      points inside spheres of two children of one node, deeper inside one in the later-visited slot than the
              earlier slot's least distance, which is below -delta
  oo_side     points whose f32 |pf|^2 (fmaf(ofx, ofx, fmaf(ofy, ofy, ofz * ofz))) is 0 to 12 f32 ulps either side of 1e30f,
              certified exactly ("side" +1: below, the tree; -1: the all-spheres scan)

ties_scene() holds exact ties across leaves: integer centres at equal-norm integer offsets with equal radii, every member
followed by a blob of 40 farther spheres so that the members of a tie sit in different leaves at every leaf size, in both
index orders, near the recentre and 2.9e7 out of it (where p - g is no float32 value), and two ties between a tree sphere and an
always-list sphere of radius about 6e14 whose f64 distance is made equal by search ulp by ulp. tie_points() gives the tie
points and their neighbours one ulp off."""
from fractions import Fraction

import numpy as np

import intersect_rays as IR
from f32_frame_cases import _child_members
from test_bvh_cpu import EMPTY
from test_distance_cpu import oo32, slack_of

f32 = np.float32
U32 = 2.0 ** -24
OO_HI = f32(1e30)
NEAR_TIE_ULPS = 4


def _pf(p, g):
    """The kernel's recentred point: fl32(fl64(p - g)) per axis."""
    with np.errstate(over="ignore"):
        return (np.asarray(p, np.float64) - g).astype(f32)


def _in_frame(c, r, g):
    with np.errstate(all="ignore"):
        return np.isfinite(c).all(axis=1) & np.isfinite(r) & (np.abs(c - g).max(axis=1) + np.abs(r) < 1e15)


def _children(recs, node):
    return [k for k in range(8) if int(recs["child"][node][k]) != EMPTY]


# ---- box faces ----

def box_face(sc, recs, rng, k=40):
    """Points on the stored plane of a child box (lo or hi of axis `axis`) in the recentred f32 frame, `ulps` f32 steps off it
    (outward positive), the other two coordinates at a member sphere's centre; and with `sub` = j in +-1..3, points whose
    f64 p - g is j/8 of an f32 ulp off the plane (outward positive) and whose f32 value is the plane."""
    c, r = IR.spheres_of(sc)
    g = recs["recentre"]
    inf32 = f32(np.inf)
    pts, node_, child_, axis_, side_, ulps_, sub_ = [], [], [], [], [], [], []
    nodes = [n for n in range(recs["n_nodes"]) if _children(recs, n)]
    for _ in range(20 * k):
        if len(node_) >= 15 * k or not nodes:
            break
        node = int(rng.choice(nodes))
        kk = int(rng.choice(_children(recs, node)))
        lo, hi = recs["lo"][node][:, kk], recs["hi"][node][:, kk]
        if not (np.isfinite(lo).all() and np.isfinite(hi).all()):
            continue
        m = _child_members(recs, node, kk)
        m = m[_in_frame(c[m], r[m], g)]
        if len(m) == 0:
            continue
        j = int(rng.choice(m))
        ax = int(rng.integers(3))
        side = -1 if rng.uniform() < 0.5 else 1
        plane = lo[ax] if side < 0 else hi[ax]
        base = c[j] - g
        for u in range(-4, 5):
            v = plane
            for _ in range(abs(u)):
                v = np.nextafter(v, inf32 if u * side > 0 else -inf32)
            q = base.copy(); q[ax] = float(v)
            pts.append(g + q); node_.append(node); child_.append(kk); axis_.append(ax); side_.append(side); ulps_.append(u); sub_.append(0)
        step = float(np.spacing(np.abs(plane))) if plane != 0 else 2.0 ** -149
        for jj in (-3, -2, -1, 1, 2, 3):
            q = base.copy(); q[ax] = float(plane) + side * jj * step / 8
            pts.append(g + q); node_.append(node); child_.append(kk); axis_.append(ax); side_.append(side); ulps_.append(0); sub_.append(jj)
    a = lambda x: np.array(x, np.int64)
    return {"p": np.array(pts, np.float64).reshape(-1, 3), "node": a(node_), "child": a(child_), "axis": a(axis_),
            "side": a(side_), "ulps": a(ulps_), "sub": a(sub_)}


def face_offsets(fam, recs):
    """(f32 ulps of pf off the plane, outward positive; sign of the f64 p - g off the plane, outward positive) per point."""
    g = recs["recentre"]
    pf = _pf(fam["p"], g)
    n = len(fam["p"])
    i = np.arange(n)
    plane = np.where(fam["side"] < 0, recs["lo"][fam["node"], fam["axis"], fam["child"]], recs["hi"][fam["node"], fam["axis"], fam["child"]])
    got = pf[i, fam["axis"]]
    apart = (_ordered(got) - _ordered(plane)) * fam["side"]
    exact = (fam["p"][i, fam["axis"]] - g[fam["axis"]]) - plane.astype(np.float64)
    return apart, np.sign(exact) * fam["side"]


def _ordered(x):
    """float32 -> integers in the order of the floats (one step per ulp, -0 == +0)."""
    b = np.asarray(x, f32).view(np.int32).astype(np.int64)
    return np.where(b < 0, -(b & 0x7FFFFFFF), b)


# ---- near-ties at far points ----

def _bisector(ci, ri, cj, rj, u, T):
    """The point m + s w + T u (w from ci to cj, u perpendicular to w) with |q - ci| - |ri| == |q - cj| - |rj| exactly: the
    branch of the hyperbola with foci ci, cj."""
    h = np.linalg.norm(cj - ci) / 2
    w = (cj - ci) / (2 * h)
    a = (abs(ri) - abs(rj)) / 2
    b = np.sqrt(h * h - a * a)
    s = a * np.sqrt(1.0 + (T / b) ** 2)
    return (ci + cj) / 2 + s * w + T * u, w


def near_tie(sc, recs, rng, k=40):
    """Pairs (i, j) under different children of one node (half of them of the root), the far-field nearest of the node's
    subtree along a random direction and the nearest under another child; points on their bisector at T = 10 .. 1e6 times the
    pair's extent and nudged by -3 .. 3 f64 ulps along w. Kept where i and j are the two least distances of the scene and
    differ by at most NEAR_TIE_ULPS ulps."""
    import distance_restatement as DR
    c, r = IR.spheres_of(sc)
    g = recs["recentre"]
    ok = _in_frame(c, r, g)
    nodes = [n for n in range(recs["n_nodes"]) if len(_children(recs, n)) >= 2]
    pts, pair, node_ = [], [], []
    for t in range(60 * k):
        if len(pair) >= 6 * k or not nodes:
            break
        node = 0 if t % 2 == 0 else int(rng.choice(nodes))
        if len(_children(recs, node)) < 2:
            continue
        under = {kk: _child_members(recs, node, kk) for kk in _children(recs, node)}
        dirn = rng.normal(size=3); dirn /= np.linalg.norm(dirn)
        sup = (c - g) @ dirn + np.abs(r)
        cand = [(sup[m[ok[m]]].max(), kk, int(m[ok[m]][np.argmax(sup[m[ok[m]]])])) for kk, m in under.items() if ok[m].any()]
        if len(cand) < 2:
            continue
        cand.sort(reverse=True)
        i, j = cand[0][2], cand[1][2]
        h = np.linalg.norm(c[j] - c[i]) / 2
        if h == 0 or abs(abs(r[i]) - abs(r[j])) >= 1.98 * h:
            continue
        ext = 2 * h + abs(r[i]) + abs(r[j])
        u = dirn - (c[j] - c[i]) * ((c[j] - c[i]) @ dirn) / (4 * h * h)
        u /= np.linalg.norm(u)
        T = ext * 10.0 ** rng.uniform(1, 6)
        if np.abs((c[i] + c[j]) / 2 - g).max() + T > 4e14:
            continue
        q, w = _bisector(c[i], r[i], c[j], r[j], u, T)
        step = float(np.spacing(np.abs(q).max()))
        cands = np.array([q + kk * step * w for kk in range(-3, 4)])
        d = DR.distances(cands, c, r)
        for row, p in zip(d, cands):
            o = np.argsort(row, kind="stable")
            if {int(o[0]), int(o[1])} != {i, j} or not np.isfinite(row[[i, j]]).all():
                continue
            if abs(row[i] - row[j]) > NEAR_TIE_ULPS * np.spacing(max(abs(row[i]), abs(row[j]))):
                continue
            if len(o) > 2 and row[o[2]] == row[o[1]]:
                continue
            pts.append(p); pair.append((i, j)); node_.append(node)
    return {"p": np.array(pts, np.float64).reshape(-1, 3), "pair": np.array(pair, np.int64).reshape(-1, 2),
            "node": np.array(node_, np.int64)}


# ---- inside overlapping spheres under different children ----

def inside(sc, recs, rng, k=60):
    """Points inside a sphere i under slot k1 and deeper inside a sphere j under a later slot k2 of the same node, both
    stored boxes holding the point, the least distance under k1 below -delta and the answer of the scene under k2."""
    import distance_restatement as DR
    c, r = IR.spheres_of(sc)
    g = recs["recentre"]
    ok = _in_frame(c, r, g)
    pts, meta = [], []
    order = rng.permutation(recs["n_nodes"])
    for node in order:
        kids = _children(recs, int(node))
        under = {kk: _child_members(recs, int(node), kk) for kk in kids}
        for a in range(len(kids)):
            for b in range(a + 1, len(kids)):
                k1, k2 = kids[a], kids[b]
                m1, m2 = under[k1][ok[under[k1]]], under[k2][ok[under[k2]]]
                for i in m1:
                    for j in m2:
                        D = np.linalg.norm(c[i] - c[j])
                        ri, rj = abs(r[i]), abs(r[j])
                        if D == 0 or D >= ri + rj:
                            continue
                        lo_t, hi_t = 1.0 - ri / D, (D + rj - ri) / (2 * D)
                        lo_t = max(lo_t, 0.0)
                        if not lo_t < hi_t:
                            continue
                        p = c[j] + (c[i] - c[j]) * ((lo_t + hi_t) / 2)
                        pts.append(p); meta.append((int(node), k1, k2))
                        if len(pts) >= 40 * k:
                            break
                    if len(pts) >= 40 * k:
                        break
    keep = []
    if pts:
        P = np.array(pts)
        d = DR.distances(P, c, r)
        ans = DR.nearest(P, c, r)[0]
        for t, (p, (node, k1, k2)) in enumerate(zip(P, meta)):
            if inside_ok(recs, c, r, p, d[t], ans[t], node, k1, k2):
                keep.append(t)
    keep = keep[:: max(1, len(keep) // k)][:k]
    return {"p": np.array([pts[t] for t in keep], np.float64).reshape(-1, 3), "where": np.array([meta[t] for t in keep], np.int64).reshape(-1, 3)}


def inside_ok(recs, c, r, p, d, ans, node, k1, k2):
    """The reach of one inside point: both stored boxes of node hold pf, the least distance under k1 is below -slack, and the
    scene's answer lies under k2 with a smaller distance."""
    g = recs["recentre"]
    pf = _pf(p, g)
    for kk in (k1, k2):
        lo, hi = recs["lo"][node][:, kk], recs["hi"][node][:, kk]
        if not ((lo <= pf) & (pf <= hi)).all():
            return False
    m1, m2 = _child_members(recs, node, k1), _child_members(recs, node, k2)
    best1 = np.nanmin(d[m1]) if len(m1) else np.inf
    return bool(best1 < -float(slack_of(pf)) and ans in set(m2.tolist()) and d[ans] < best1)


# ---- both sides of oo < 1e30f ----

def oo_side(g, rng, k=24):
    """Points g + u * sqrt(1e30) * (1 + j 2^-24) for j in -12 .. 12 along k random and the three axis directions, and points on
    the axes whose f32 coordinate is the f32 values nearest 1e15 (|pf|^2 rounding to 1e30f itself among them). "oo" is the
    kernel's |pf|^2, "side" +1 (below 1e30f: the tree) or -1 (the scan)."""
    dirs = list(np.eye(3)) + list(-np.eye(3))
    for _ in range(k):
        u = rng.normal(size=3); dirs.append(u / np.linalg.norm(u))
    pts = []
    for u in dirs:
        for j in range(-12, 13):
            pts.append(g + u * (np.sqrt(1e30) * (1.0 + j * 2.0 ** -24)))
    x0 = f32(1e15)
    for a in range(3):
        x = x0
        for _ in range(4):
            x = np.nextafter(x, f32(0))
        for _ in range(9):
            e = np.zeros(3); e[a] = float(x)
            pts.append(g + e)
            x = np.nextafter(x, f32(np.inf))
    p = np.array(pts, np.float64)
    oo = np.array([oo32(q) for q in _pf(p, g)], f32)
    return {"p": p, "oo": oo, "side": np.where(oo < OO_HI, 1, -1)}


def oo_certified(fam, g):
    """The exact |pf|^2 of each point against 1e30f, and its one-rounding fmaf chain: (ulps of oo from 1e30f, whether the
    rounding of each FMA was checked against Fraction arithmetic)."""
    pf = _pf(fam["p"], g)
    out = []
    for q in pf:
        F = [Fraction(float(x)) for x in q]
        zz = f32(q[2]) * f32(q[2])
        assert Fraction(float(zz)) - F[2] * F[2] <= Fraction(float(np.spacing(zz))) / 2
        inner = oo32(np.array([0.0, q[1], q[2]], f32))
        outer = oo32(q)
        for got, exact in ((inner, F[1] * F[1] + Fraction(float(zz))), (outer, F[0] * F[0] + Fraction(float(inner)))):
            half = Fraction(float(np.spacing(got))) / 2
            assert abs(Fraction(float(got)) - exact) <= half, (q, got)
        out.append(int(_ordered(outer) - _ordered(OO_HI)))
    return np.array(out, np.int64)


# ---- exact ties across leaves ----

NORM9 = [((4, 4, 7), (0, 0, 9)), ((8, 4, 1), (-1, -4, -8)), ((1, 4, 8), (-4, 7, -4)), ((7, -4, 4), (-8, 1, 4))]
FAR_S = 262_145                         # the far ties' scale: p - g about 2.9e7, odd, past float32's integers
R_ALWAYS, D_ALWAYS = 6.0e14, 6.0e7      # the always-list spheres: radius, and how far their surfaces pass from the origin


def _far(axis, sign):
    """A far tie: members ca and cb = ca + FAR_S (w), p = ca + FAR_S va with |va| = |vb| = 111 (110^2 + 10^2 + 11^2 = 111^2),
    110 along the axis: ca is the scene's extreme sphere in the direction of p."""
    o = [a for a in range(3) if a != axis]
    va, vb = np.zeros(3), np.zeros(3)
    va[axis] = vb[axis] = 110.0 * sign
    va[o[0]], va[o[1]], vb[o[0]], vb[o[1]] = 10.0, 11.0, 11.0, 10.0
    ca = np.zeros(3); ca[axis] = 1502.0 * sign
    p = ca + FAR_S * va
    return p, ca, p - FAR_S * vb


def _blob(c, p, r_member, n=40):
    """n spheres of radius 0.5 on the even grid around c, farther from p than the member's surface by at least 1."""
    v = np.arange(-4, 5, 2)
    grid = np.array([(a, b, e) for a in v for b in v for e in v if (a, b, e) != (0, 0, 0)], np.float64)
    pos = c + grid
    far = np.linalg.norm(pos - p, axis=1) - 0.5 >= np.linalg.norm(c - p) - r_member + 1.0
    pos = pos[far]
    return pos[np.argsort(np.linalg.norm(pos - c, axis=1), kind="stable")[:n]]


def _contract(p, c, r):
    """dist_j of the contract in Python floats."""
    x, y, z = p[0] - c[0], p[1] - c[1], p[2] - c[2]
    return float(np.sqrt((x * x + y * y) + z * z)) - abs(r)


def ties_scene():
    """(Scene, ties): ties is a list of {"p", "members" (two sphere indices, the lower first), "dist", "always" (the member on
    the always-list or -1)}."""
    objs, ties = [], []

    def add(c, r):
        objs.append(IR.sphere(c, r))
        return len(objs) - 1

    def pair(p, ca, cb, r, swap):
        """Two members (and their blobs); with swap the second member gets the lower index."""
        first, second = (cb, ca) if swap else (ca, cb)
        ia = add(first, r)
        for b in _blob(np.array(first), np.array(p), r):
            add(b, 0.5)
        ib = add(second, r)
        for b in _blob(np.array(second), np.array(p), r):
            add(b, 0.5)
        return ia, ib

    for s, (va, vb) in enumerate(NORM9):
        for swap in (False, True):
            p = np.array([160.0 * (2 * s + swap), 0.0, 0.0])
            ia, ib = pair(p, p + va, p + vb, 1.0, swap)
            ties.append({"p": p, "members": sorted((ia, ib)), "dist": 8.0, "always": -1})
    for t, (axis, sign) in enumerate(((0, 1.0), (0, -1.0))):   # members near the recentre, p 2.9e7 out
        p, ca, cb = _far(axis, sign)
        ia, ib = pair(p, ca, cb, 1.0, t % 2 == 1)
        ties.append({"p": p, "members": sorted((ia, ib)), "dist": 111.0 * FAR_S - 1.0, "always": -1})
    # a tree member at distance 8 and an always-list sphere of radius about 6e14 whose surface passes 8 from p, D_ALWAYS out;
    # the always sphere comes first (lower index) at one site and last at the other
    for t, (ax, p, v) in enumerate(((2, np.array([0.0, 3.0, 8.0 - D_ALWAYS]), np.array([4.0, 4.0, 7.0])),
                                    (1, np.array([3.0, 8.0 - D_ALWAYS, 0.0]), np.array([4.0, 7.0, 4.0])))):
        ca = np.zeros(3); ca[ax] = -(R_ALWAYS + D_ALWAYS)
        ra = _always_radius(p, ca, 8.0)
        ia = add(ca, ra) if t == 0 else None
        it = add(p + v, 1.0)
        for b in _blob(p + v, p, 1.0):
            add(b, 0.5)
        if ia is None:
            ia = add(ca, ra)
        ties.append({"p": p, "members": sorted((ia, it)), "dist": 8.0, "always": ia})
    return IR.scene_of(objs)[0], ties


def _always_radius(p, ca, want):
    """The radius, searched ulp by ulp from fl(|p - ca|) - want, at which the contract's dist of p is exactly `want`."""
    ra = _contract(p, ca, 0.0) - want
    for k in range(64):
        for cand in (ra + k * np.spacing(ra), ra - k * np.spacing(ra)):
            if _contract(p, ca, cand) == want:
                return cand
    raise AssertionError("no radius gives the tie")


def tie_points(ties):
    """The tie points, and each tie point moved one f64 ulp along each axis (the neighbours, where the tie may break)."""
    pts, tie = [], []
    for t, x in enumerate(ties):
        p = x["p"]
        pts.append(p); tie.append(t)
        for a in range(3):
            for sgn in (-1, 1):
                q = p.copy(); q[a] = np.nextafter(q[a], sgn * np.inf); pts.append(q); tie.append(-1)
    return {"p": np.array(pts, np.float64), "tie": np.array(tie, np.int64)}


def tie_certified(ties, c, r):
    """Each tie's two distances in Fraction arithmetic (the member on the always-list through the contract's f64 steps, which
    round) equal each other and the f64 contract's."""
    for x in ties:
        p = x["p"]
        ds = []
        for j in x["members"]:
            if j == x["always"]:
                ds.append(Fraction(_contract(p, c[j], r[j])))
                continue
            sq = sum((Fraction(float(p[a])) - Fraction(float(c[j][a]))) ** 2 for a in range(3))
            root = Fraction(int(round(float(sq) ** 0.5)))
            assert root * root == sq, (p, c[j])             # a perfect square: the f64 steps are exact
            ds.append(root - Fraction(abs(float(r[j]))))
            assert Fraction(_contract(p, c[j], r[j])) == ds[-1]
        assert ds[0] == ds[1] == Fraction(x["dist"]), (x, ds)
    return True


def leaf_of(recs, j):
    """The leaf holding sphere j, or -1 (always-list)."""
    hit = np.nonzero(recs["leaf_id"] == j)[0]
    return int(hit[0]) if len(hit) else -1


def nested_scene():
    """300 spheres of radius 1 .. 6 with centres in a cube of side 40: most points inside one sphere are inside several, under
    different children of a node (the inside family's scene)."""
    rng = np.random.default_rng(19)
    c = rng.uniform(-20, 20, size=(300, 3))
    r = rng.uniform(1, 6, size=300)
    return IR.scene_of([IR.sphere(c[i], r[i]) for i in range(300)])[0]


# ---- D~'s edges ----

FMAX = float(np.finfo(np.float32).max)
FIXED_BOUNDS = {"min_sub": 5e-324, "neg_min_sub": -5e-324, "tiny": 1e-300, "neg_tiny": -1e-300, "f32_sub": 1e-40,
                "f32_min_sub": float(np.finfo(np.float32).smallest_subnormal), "f32_min": float(np.finfo(np.float32).tiny),
                "below_fmax": float(np.nextafter(FMAX, 0.0)), "fmax": FMAX, "above_fmax": float(np.nextafter(FMAX, np.inf)),
                "fmax_half_ulp": FMAX + 2.0 ** 103}


def edge_bounds(d):
    """The bounds of every point around its unbounded answer d (1.0 for none): at d and one f64 ulp either side, and the fixed
    values of FIXED_BOUNDS: +-2^-1074, +-1e-300, f32-subnormal, FLT_MIN, FLT_MAX and the doubles next to it, and FLT_MAX
    plus half its ulp (where __double2float_ru gives +inf and round-to-nearest would not)."""
    f = np.where(np.isfinite(d), d, 1.0)
    out = {"at": f, "above": np.nextafter(f, np.inf), "below": np.nextafter(f, -np.inf)}
    for name, v in FIXED_BOUNDS.items():
        out[name] = np.full_like(f, v)
    return out


# ---- every family of one scene ----

def families(sc, recs, seed, small=False):
    """Every point family of the module docstring on scene `sc` whose hierarchy is `recs` (R.bvh_records or
    ResidentScene.bvh_records). `small` takes fewer points (the CPU emulation)."""
    rng = np.random.default_rng(seed)
    k = 6 if small else 40
    return {"box_face": box_face(sc, recs, rng, k), "near_tie": near_tie(sc, recs, rng, k), "inside": inside(sc, recs, rng, k),
            "oo_side": oo_side(recs["recentre"], rng, 4 if small else 24)}


def concat(fams):
    """All families as one point set: (p, family name of each point)."""
    names = np.concatenate([np.full(len(f["p"]), k, dtype=object) for k, f in fams.items()])
    return np.concatenate([f["p"] for f in fams.values()]), names
