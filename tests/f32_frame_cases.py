"""Scenes and ray families where the margins of the closest-hit stage's f32 tests are tight (DESIGN.md §4.2, §4.11), shared by
tests/test_gpu_f32_frame.py, tests/f32_frame_worker.py and tests/test_f32_frame_cpu.py. Everything is deterministic: the
scenes are fixed by their names, the families by their scene, the records they aim at and a seed.

Scenes (SCENES, each made with intersect_rays.scene_of):
  spread_X   a cluster at the origin and equal clusters at +-X (0.8, 0.36, -0.48), X in SPREAD, so that the recentre stays
             at the origin and the outer clusters sit about X out in the f32 frame; radii log-uniform in 1e-3 .. max(10,
             1e-6 X), coincident and negative-radius copies, Lambertian, Metal, Glass and Light spheres
  huge       a sphere of radius 1e14 near the origin with unit spheres on its surface and inside it
  threshold  spheres whose max|c - g| + |r| is one f64 ulp below 1e15 (in the f32 frame, B about 1e15), exactly 1e15 and one
             ulp above (on the always-list), next to unit spheres

Families (families(sc, recs, seed)): name -> {"o", "d" [n, 3] float64, "group" [n] (siblings of one grazing or box-face ray,
-1: none), "target" [n] (the sphere a grazing or box-face ray is aimed at, -1: none), "side" [n] (+1: the ray passes the
flag test of the f32 frame and takes the tree, -1: it fails it and takes the f64 path, 0: not decided here)}."""
import numpy as np

import intersect_rays as IR
from test_bvh_cpu import EMPTY, LEAF, _fma

f32 = np.float32
SPREAD = (1e4, 1e8, 1e12, 4e14)
AXIS = np.array([0.8, 0.36, -0.48])      # a unit vector with no zero component
K = np.arange(-8, 9)                     # the ulp offsets of a grazing or box-face group
S_LO, S_HI, OO_HI = f32(1e-30), f32(1e30), f32(1e30)   # the flag test of closest_hit: s > S_LO && s < S_HI && oo < OO_HI


def _materials():
    return [{"Lambertian": {"albedo": [0.7, 0.4, 0.2]}}, {"Metal": {"albedo": [0.8, 0.8, 0.9], "fuzz": 0.3}},
            {"Metal": {"albedo": [0.9, 0.6, 0.6], "fuzz": 0.0}}, {"Glass": {"index_of_refraction": 1.5}}]


LIGHT = {"Light": {}}   # one per cluster: the oracle's light recursion needs fewer than 10 lights


def _cluster(rng, centre, n, rmax, mats):
    out = []
    spread = 4.0 * rmax
    for i in range(n):
        c = centre + rng.uniform(-spread, spread, size=3)
        r = float(np.exp(rng.uniform(np.log(1e-3), np.log(rmax))))
        out.append(IR.sphere(c, r, LIGHT if i == 0 else mats[i % len(mats)]))
    # a coincident copy (the tie rule) and a negative-radius copy (a hollow shell) of the cluster's largest sphere
    big = max(out, key=lambda s: s["radius"])
    out.append(dict(big, material=mats[(len(out) + 1) % len(mats)]))
    out.append(dict(big, radius=-big["radius"], material=mats[3]))
    return out


def spread_scene(x, n=20):
    rng = np.random.default_rng(int(np.log10(x) * 10))
    rmax = max(10.0, 1e-6 * x)
    mats = _materials()
    objs = _cluster(rng, np.zeros(3), n, rmax, mats)
    objs += _cluster(rng, x * AXIS, n, rmax, mats)
    objs += _cluster(rng, -x * AXIS, n, rmax, mats)
    return IR.scene_of(objs)[0]


def huge_scene():
    rng = np.random.default_rng(7)
    mats = _materials()
    c0 = np.array([3.0, -2.0, 1.0])
    objs = [IR.sphere(c0, 1e14, mats[0])]
    for i in range(16):                                   # unit spheres on the big sphere's surface
        n = rng.normal(size=3); n /= np.linalg.norm(n)
        objs.append(IR.sphere(c0 + 1e14 * n, 1.0, LIGHT if i == 0 else mats[i % 4]))
    for i in range(24):                                   # and inside it, near its centre and far out
        p = rng.normal(size=3) * (10.0 if i % 2 else 1e12)
        objs.append(IR.sphere(c0 + p, float(rng.uniform(0.5, 2.0)), LIGHT if i == 0 else mats[i % 4]))
    return IR.scene_of(objs)[0]


LIMIT = 1e15
STEP = float(np.spacing(LIMIT))          # one f64 ulp at 1e15 (0.125)
# (offset axis, sign, radius, max|c - g| + |r| - 1e15 in ulps): -1 lives in the f32 frame, 0 and +1 go on the always-list
THRESHOLD = [(0, +1, 0.5, -1), (0, -1, 0.5, 0), (1, +1, 1e14, -1), (1, -1, 1e14, +1), (2, +1, 4e14, -1), (2, -1, 4e14, +1),
             (0, +1, 2e14, +1), (2, -1, 0.5, -1)]


def threshold_scene():
    """Unit spheres with centres on a 1/8 grid (so that c - g is exact), and the spheres of THRESHOLD placed from the recentre
    g of the whole scene; g is found by iterating the placement until it stops changing."""
    import rtb200 as R
    rng = np.random.default_rng(8)
    mats = _materials()
    units = [IR.sphere(np.round(rng.uniform(-6, 6, size=3) * 8) / 8, 1.0, LIGHT if i == 0 else mats[i % 4]) for i in range(25)]
    g = np.zeros(3)
    for _ in range(4):
        objs = list(units)
        for k, (ax, sign, r, ulps) in enumerate(THRESHOLD):
            c = g.copy()
            c[ax] += sign * ((LIMIT + ulps * STEP) - r)
            objs.append(IR.sphere(c, r, mats[k % 4]))
        sc = IR.scene_of(objs)[0]
        g2 = R.bvh_records(sc)["recentre"]
        if np.array_equal(g2, g):
            return sc
        g = g2
    raise AssertionError("the recentre of the threshold scene does not settle")


def threshold_ids():
    """Sphere indices of the threshold scene's THRESHOLD spheres, and which of them must be on the always-list."""
    ids = np.arange(25, 25 + len(THRESHOLD))
    return ids, np.array([u >= 0 for _, _, _, u in THRESHOLD])


def spread_name(x):
    m, e = f"{x:.0e}".split("e")
    return f"spread_{m}e{int(e)}"


SCENES = {**{spread_name(x): (lambda x=x: spread_scene(x)) for x in SPREAD}, "huge": huge_scene, "threshold": threshold_scene}


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _perp(rng, v):
    """A random unit vector perpendicular to each row of v."""
    a = rng.normal(size=v.shape)
    a -= v * np.sum(a * v, axis=1, keepdims=True) / np.sum(v * v, axis=1, keepdims=True)
    return _unit(a)


def _ulp(c, r):
    """The spacing a grazing offset is counted in: one ulp of the sphere's largest coordinate (offsets in ulps of a small r
    are lost to the rounding of the coordinates far out), or of r when that is larger."""
    return np.maximum(np.spacing(np.abs(c).max(axis=1)), np.spacing(np.abs(r)))


def targets(sc, k, rng):
    """k spheres to aim at: finite, of non-zero radius, inside the f32 frame (|c| < 1e15), drawn over the whole list."""
    c, r = IR.spheres_of(sc)
    ok = np.flatnonzero(np.isfinite(c).all(axis=1) & np.isfinite(r) & (np.abs(r) > 0) & (np.abs(c).max(axis=1) + np.abs(r) < 1e15))
    return np.sort(rng.choice(ok, size=min(k, len(ok)), replace=False))


def grazing_far(sc, g, rng, k=24):
    """Rays tangent to k target spheres at distance |r| + j ulp(|c|), j in K, from origins 3|r|, 1e3|r| and |c - g| back
    along a random direction, and from the point of the line nearest g (the line aimed past g: |o - g| is about |r|)."""
    c, r = IR.spheres_of(sc)
    t = targets(sc, k, rng)
    os_, ds, gs, ts = [], [], [], []
    grp = 0
    for j in t:
        cj, rj = c[j][None], abs(r[j])
        u = float(_ulp(cj, np.array([rj]))[0])
        toward = cj - g
        for kind in range(4):
            if kind < 3:
                d = _unit(rng.normal(size=(1, 3)))
                a = _perp(rng, d)
                back = (3.0 * rj, 1e3 * rj, max(float(np.linalg.norm(toward)), 3.0 * rj))[kind]
            else:   # aimed from next to g: a perpendicular to c - g, d along c - g
                if np.linalg.norm(toward) < 10 * rj:
                    continue
                d = _unit(toward)
                a = _perp(rng, d)
                back = float(np.linalg.norm(toward))
            p = cj + a * (rj + K[:, None] * u)
            os_.append(p - d * back)
            ds.append(np.repeat(d, len(K), axis=0))
            gs.append(np.full(len(K), grp)); ts.append(np.full(len(K), j))
            grp += 1
    return np.concatenate(os_), np.concatenate(ds), np.concatenate(gs), np.concatenate(ts)


def _child_members(recs, node, k):
    ref = int(recs["child"][node][k])
    if ref & LEAF:
        ids = recs["leaf_id"][ref & 0x7FFFFFFF]
        return ids[ids != EMPTY].astype(np.int64)
    out = []
    for kk in range(8):
        if int(recs["child"][ref][kk]) != EMPTY:
            out.extend(_child_members(recs, ref, kk).tolist())
    return np.array(out, np.int64)


def faces(sc, recs, rng, k=40):
    """Up to k (node, child, axis, side, sphere) faces of the hierarchy `recs`: the member sphere whose exact box (c - g) +- |r|
    reaches the child's box face on that axis and side (spheres on the always-list and infinite boxes left out)."""
    c, r = IR.spheres_of(sc)
    g = recs["recentre"]
    out = []
    for node in range(recs["n_nodes"]):
        for kk in range(8):
            if int(recs["child"][node][kk]) == EMPTY:
                continue
            m = _child_members(recs, node, kk)
            m = m[np.isfinite(c[m]).all(axis=1) & (np.abs(c[m] - g).max(axis=1) + np.abs(r[m]) < 1e15) & (np.abs(r[m]) > 0)]
            if len(m) == 0 or not np.isfinite(recs["lo"][node][:, kk]).all():
                continue
            for ax in range(3):
                lo = (c[m, ax] - g[ax]) - np.abs(r[m])
                hi = (c[m, ax] - g[ax]) + np.abs(r[m])
                out.append((node, kk, ax, -1, int(m[np.argmin(lo)])))
                out.append((node, kk, ax, +1, int(m[np.argmax(hi)])))
    if len(out) > k:
        out = [out[i] for i in np.sort(rng.choice(len(out), size=k, replace=False))]
    return out


def box_face(sc, recs, rng, k=40):
    """For each face of faces(): rays in the face plane through the member sphere's tangent point P = c + side |r| e_axis,
    shifted along the axis by j ulp(P) for j in K (j < 0 inside the sphere), from 3|r| and |P - g| back; the same rays tilted
    out of the plane by j ulp; and rays lying exactly in the stored, inflated f32 plane of the child's box (g + plane)."""
    c, r = IR.spheres_of(sc)
    g = recs["recentre"]
    os_, ds, gs, ts = [], [], [], []
    grp = 0
    for node, kk, ax, side, j in faces(sc, recs, rng, k):
        P = c[j].copy()
        P[ax] += side * abs(r[j])
        u = float(np.spacing(np.abs(P).max()))
        d = rng.normal(size=3); d[ax] = 0.0; d = _unit(d)
        for back in (3.0 * abs(r[j]), max(float(np.linalg.norm(P - g)), 3.0 * abs(r[j]))):
            o = np.repeat((P - d * back)[None], len(K), axis=0)
            o[:, ax] = P[ax] + side * K * u                      # shifted: j < 0 cuts the sphere, j > 0 passes outside
            os_.append(o); ds.append(np.repeat(d[None], len(K), axis=0)); gs.append(np.full(len(K), grp)); ts.append(np.full(len(K), j))
            grp += 1
            dt = np.repeat(d[None], len(K), axis=0)
            dt[:, ax] = K * np.finfo(np.float64).eps            # tilted through P
            os_.append(P - dt * back); ds.append(dt); gs.append(np.full(len(K), -1)); ts.append(np.full(len(K), j))
        plane = float(recs["lo"][node][ax, kk] if side < 0 else recs["hi"][node][ax, kk])
        for back in (3.0 * abs(r[j]), max(float(np.linalg.norm(P - g)), 3.0 * abs(r[j]))):
            o = P - d * back
            o[ax] = g[ax] + plane                                 # in the stored plane: t_near == t_far on that axis
            os_.append(o[None]); ds.append(d[None]); gs.append(np.full(1, -1)); ts.append(np.full(1, -1))
    if not os_:
        return np.zeros((0, 3)), np.zeros((0, 3)), np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(os_), np.concatenate(ds), np.concatenate(gs), np.concatenate(ts)


def f32_s(d):
    """closest_hit's s = |d|^2 in f32 (fmaf(dfx, dfx, fmaf(dfy, dfy, dfz * dfz))), emulated."""
    df = np.asarray(d, np.float64).astype(f32)
    with np.errstate(over="ignore", under="ignore"):
        return np.array([_fma(x[0], x[0], _fma(x[1], x[1], f32(x[2] * x[2]))) for x in df], f32)


def f32_oo(o, g):
    """closest_hit's oo = |o - g|^2 in f32, emulated."""
    of = (np.asarray(o, np.float64) - g).astype(f32)
    with np.errstate(over="ignore", under="ignore"):
        return np.array([_fma(x[0], x[0], _fma(x[1], x[1], f32(x[2] * x[2]))) for x in of], f32)


def _ulps_apart(a, b):
    """Signed distance a - b in f32 ulps (both positive and finite)."""
    return a.view(np.int32).astype(np.int64) - np.asarray(b, f32).view(np.int32).astype(np.int64)


def sides(o, d, g):
    """+1 where the emulated flag test passes (the ray takes the tree), -1 where it fails (the f64 path over every sphere), 0
    where s or oo is within 2 f32 ulps of a threshold (the emulation may round twice, the kernel's rsqrtf-free s and oo do not)."""
    s, oo = f32_s(d), f32_oo(o, g)
    ok = (s > S_LO) & (s < S_HI) & (oo < OO_HI)
    with np.errstate(over="ignore", invalid="ignore"):
        near = ((np.abs(_ulps_apart(s, S_LO)) < 2) | (np.abs(_ulps_apart(s, S_HI)) < 2) | (np.abs(_ulps_apart(oo, OO_HI)) < 2))
    return np.where(near, 0, np.where(ok, 1, -1))


def d_sweep(o, d, g, rng):
    """The rays (o, d) with d scaled by 2^k, k drawn from [-49, 49] (the ends always among them), and copies of them scaled so
    that the f32 s lands 3 to 12 f32 ulps either side of 1e-30 and of 1e30 (side +1: inside, the tree; -1: the f64 path)."""
    n = len(o)
    k = rng.integers(-49, 50, size=n)
    k[: min(n, 8)] = np.resize([-49, 49], min(n, 8))
    ds = d * np.ldexp(1.0, k)[:, None]
    pick = rng.choice(n, size=min(n, 600), replace=False)
    oo, dd, side = [o], [ds], [sides(o, ds, g)]
    for thr in (S_LO, S_HI):
        base = d[pick] / np.linalg.norm(d[pick], axis=1, keepdims=True) * np.sqrt(float(thr))
        for j in (-12, -6, -3, 3, 6, 12):
            scaled = base * (1.0 + j * 2.0 ** -24)
            s = f32_s(scaled)
            apart = _ulps_apart(s, thr)
            # keep the rays whose emulated s is at least 2 ulps from the threshold (the emulation may round twice)
            ok = np.abs(apart) >= 2
            inside = (apart > 0) if thr == S_LO else (apart < 0)
            side.append(np.where(inside[ok] & (f32_oo(o[pick][ok], g) < OO_HI), 1, -1))
            oo.append(o[pick][ok]); dd.append(scaled[ok])
    return np.concatenate(oo), np.concatenate(dd), np.concatenate(side)


def o_sweep(sc, g, rng, k=8):
    """Rays through k target spheres near g (centre plus a random offset inside |r|, or grazing at |r|) from origins at
    |o - g| from 1e3 to 1e15, and at distances whose f32 oo is 3 to 12 ulps either side of 1e30 (side as in d_sweep)."""
    c, r = IR.spheres_of(sc)
    t = targets(sc, 4 * k, rng)
    t = t[np.argsort(np.abs(c[t] - g).max(axis=1))][:k]        # the targets nearest g
    os_, ds, side = [], [], []
    for j in t:
        for q in range(4):
            u = _unit(rng.normal(size=(1, 3)))
            a = _perp(rng, u)
            p = c[j] + a[0] * abs(r[j]) * (0.5, 1.0, 1.0 - 1e-9, 1.0 + 1e-9)[q]   # aimed inside, at and around the rim
            dists = np.concatenate([10.0 ** np.arange(3.0, 15.1, 1.0), [9.9e14]])
            base = g + u * np.sqrt(float(OO_HI))
            near = [base + u * (np.sqrt(float(OO_HI)) * j2 * 2.0 ** -24) for j2 in (-12, -6, -3, 3, 6, 12)]
            o = np.concatenate([g + u * dists[:, None], np.concatenate(near)])
            oo = f32_oo(o, g)
            apart = _ulps_apart(oo, OO_HI)
            keep = np.abs(apart) >= 2
            os_.append(o[keep]); ds.append(_unit(p - o[keep])); side.append(np.where(apart[keep] < 0, 1, -1))
    return np.concatenate(os_), np.concatenate(ds), np.concatenate(side)


def component_edges(sc, g, rng, k=16):
    """Axis-major directions (|d| = 1 on the axis, so d^ equals f32(d)) whose other components sit either side of the 1e-20
    clamp of the slab constants (+-1e-20 (1 +- 2^-20)), are f32-subnormal (1e-40, 1e-45), round to 0 in f32 (1e-50) or are
    -0.0, from origins 3|r| back from k target spheres, aimed inside, at and just outside their rims."""
    c, r = IR.spheres_of(sc)
    tiny = np.array([1e-20 * (1 + 2.0 ** -20), 1e-20 * (1 - 2.0 ** -20), -1e-20 * (1 + 2.0 ** -20), -1e-20 * (1 - 2.0 ** -20),
                     1e-40, -1e-40, 1e-45, -1e-45, 1e-50, -1e-50, -0.0, 0.0])
    os_, ds = [], []
    for j in targets(sc, k, rng):
        for ax in range(3):
            for sgn in (1.0, -1.0):
                e = np.zeros(3); e[ax] = sgn
                others = [a for a in range(3) if a != ax]
                for q in range(len(tiny)):
                    d = e.copy()
                    d[others[0]] = tiny[q]
                    d[others[1]] = tiny[rng.integers(len(tiny))]
                    off = np.zeros(3)
                    off[others[0]] = abs(r[j]) * (0.5, 1.0, 1.0 + 4 * np.finfo(np.float64).eps)[q % 3]
                    os_.append(c[j] + off - d * 3.0 * abs(r[j]))
                    ds.append(d)
    return np.array(os_), np.array(ds)


def segments(sc, rng, k=400):
    """Segments o = a, d = b - a, t_max = 1 between points on spheres of the scene, most of them the far ones."""
    c, r = IR.spheres_of(sc)
    t = targets(sc, 10 ** 6, rng)
    w = np.abs(c[t]).max(axis=1) + 1.0
    a = t[rng.choice(len(t), size=k, p=w / w.sum())]
    b = t[rng.choice(len(t), size=k, p=w / w.sum())]
    na = _unit(rng.normal(size=(k, 3))); nb = _unit(rng.normal(size=(k, 3)))
    pa = c[a] + na * np.abs(r[a])[:, None]
    pb = c[b] + nb * np.abs(r[b])[:, None]
    return pa, pb - pa, np.ones(k)


def families(sc, recs, seed):
    """Every family of the module docstring on scene `sc` whose hierarchy is `recs` (R.bvh_records or ResidentScene.bvh_records)."""
    rng = np.random.default_rng(seed)
    g = recs["recentre"]
    out = {}

    def put(name, o, d, group=None, target=None, side=None):
        n = len(o)
        none = np.full(n, -1, np.int64)
        out[name] = {"o": np.ascontiguousarray(o, np.float64), "d": np.ascontiguousarray(d, np.float64),
                     "group": none if group is None else group, "target": none if target is None else target,
                     "side": np.zeros(n, np.int64) if side is None else side}

    put("grazing_far", *grazing_far(sc, g, rng))
    put("box_face", *box_face(sc, recs, rng))
    both = np.concatenate([out["grazing_far"]["o"], out["box_face"]["o"]]), np.concatenate([out["grazing_far"]["d"], out["box_face"]["d"]])
    o, d, side = d_sweep(*both, g, rng)
    put("d_sweep", o, d, side=side)
    o, d, side = o_sweep(sc, g, rng)
    put("o_sweep", o, d, side=side)
    put("component_edges", *component_edges(sc, g, rng))
    return out


def concat(fams):
    """All families as one ray set: (o, d, name of each ray's family)."""
    names = np.concatenate([np.full(len(f["o"]), k, dtype=object) for k, f in fams.items()])
    return np.concatenate([f["o"] for f in fams.values()]), np.concatenate([f["d"] for f in fams.values()]), names


def edge_bounds(un):
    """The bounds of the occlusion tests around each ray's unbounded root r* (1.0 for a miss): r*, the next and previous f64
    values, and test_gpu_occlusion.t_edges's fixed edges."""
    f = np.where(np.isfinite(un["t"]), un["t"], 1.0)
    return [f, np.nextafter(f, np.inf), np.nextafter(f, -np.inf), np.full_like(f, 0.001), np.full_like(f, np.nextafter(0.001, 0.0)),
            np.full_like(f, np.nextafter(0.001, 1.0)), np.full_like(f, 0.0), np.full_like(f, np.inf), np.full_like(f, np.nan),
            np.full_like(f, IR.MAX), np.full_like(f, -np.inf)]


def flip_share(hit, group):
    """Share of the groups (group >= 0) in which `hit` (the oracle's closest sphere is the group's target) holds for some
    siblings and not for others."""
    gs = group[group >= 0]
    h = hit[group >= 0]
    if len(gs) == 0:
        return 0.0, 0
    ids = np.unique(gs)
    anyh = np.zeros(ids.max() + 1, bool); allh = np.ones(ids.max() + 1, bool)
    np.logical_or.at(anyh, gs, h); np.logical_and.at(allh, gs, h)
    return float(np.mean(anyh[ids] & ~allh[ids])), len(ids)
