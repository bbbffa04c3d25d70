"""Scenes and rays at which a decision of the reference's Sphere::hit, hit_world or first shading step turns on an exact
equality (TEST INFRASTRUCTURE): there `<` and `<=` take different paths, and random or ulp-jittered rays reach such a point
with probability zero.

    E1  tangency: disc == 0, d·n == 0 (front_face false, the normal flips), at every material: Metal fuzz 0 absorbs
        (scattered·n == 0), Glass cannot refract at ir 1.5, can at ir exactly 1 (1·1 > 1 is false) and then reflects
        (reflectance(0, 1) == 1), Texture at its pole (v == 1); and the same rays moved off tangency by the fewest ulps of o_y
        that show, up (a miss) and down (two roots)
    E2  a root exactly at t_min = 0.001: root_a == t_min is rejected and root_b taken; root_a == next(t_min) is accepted;
        root_b == t_min from inside misses the sphere
    E3  exact ties between different spheres: internally and externally tangent pairs, both index orders, the pair in
        different leaves of the hierarchy, and one member on the always-list (the traversal/always-list merge)
    E4  the refraction limit: fl(ratio·sin_theta) == 1.0 from inside (ratio = ir) and from outside at ir < 1 (ratio = 1/ir)
    E5  the cos clamp: -unit_direction·n above 1 at normal incidence

Every case carries its certificate (`claims`): the reference's expressions evaluated op by op in Python floats (IEEE f64,
never contracted, the reference's operation order, sphere.rs:46-78 and materials.rs:176-199) by `Chain`, which also records
every operation whose result differs from the exact rational one (`fractions.Fraction`). Where a case is built from dyadic
numbers the claim is that nothing was rounded, so the f64 equality is the exact one. Where the equality needs rounding to land
(E2, E4) the value was found by searching ulp by ulp in that same order, and the case also holds its two neighbours.
tests/test_exact_edges_cpu.py checks the claims, a vectorised numpy evaluation of the same expressions, and the oracle's
decisions; tests/test_gpu_exact_edges.py holds every GPU variant to the oracle on these rays."""
import math
from fractions import Fraction as Q

import numpy as np

from synth import _v, base_config

T_MIN = 0.001
MAX = 1.7976931348623157e308
P = 2.0 ** 20
LIGHTS = 2                                   # lights of the lit form of every scene


def up(x):
    return float(np.nextafter(x, math.inf))


def down(x):
    return float(np.nextafter(x, -math.inf))


# ---- the reference's f64 expressions, op by op, with a record of what was rounded ----------------------------------------
class Chain:
    """IEEE f64 operations in the reference's order. `rounded` names every operation whose result is not the exact rational
    result of its (already rounded) operands."""

    def __init__(self):
        self.rounded = []

    def _r(self, name, r, exact):
        if not math.isfinite(r) or Q(r) != exact:
            self.rounded.append(name)
        return r

    def add(self, a, b, name="+"):
        return self._r(name, a + b, Q(a) + Q(b))

    def sub(self, a, b, name="-"):
        return self._r(name, a - b, Q(a) - Q(b))

    def mul(self, a, b, name="*"):
        return self._r(name, a * b, Q(a) * Q(b))

    def div(self, a, b, name="/"):
        return self._r(name, a / b, Q(a) / Q(b))

    def sqrt(self, a, name="sqrt"):
        r = math.sqrt(a)
        if Q(r) * Q(r) != Q(a):
            self.rounded.append(name)
        return r

    def dot(self, a, b, name="dot"):            # point3d.rs: x*x' + y*y' + z*z', left to right
        return self.add(self.add(self.mul(a[0], b[0], name), self.mul(a[1], b[1], name), name), self.mul(a[2], b[2], name), name)

    def vsub(self, a, b, name="vsub"):
        return tuple(self.sub(a[k], b[k], name) for k in range(3))

    def unit(self, a, name="unit"):              # point3d.rs:52-70: length() of a - 0, then three divisions
        z = tuple(self.sub(a[k], 0.0, name) for k in range(3))
        ln = self.sqrt(self.dot(z, z, name), name)
        return tuple(self.div(a[k], ln, name) for k in range(3))


def sphere_hit(ch, c, r, o, d, t_min=T_MIN, t_max=MAX):
    """Sphere::hit (sphere.rs:46-78) in `ch`: every intermediate and, for an accepted root, which root, t, p, the normal as
    stored (flipped when front_face is false) and front_face."""
    oc = ch.vsub(o, c, "oc")
    a = ch.dot(d, d, "a")
    hb = ch.dot(oc, d, "half_b")
    cc = ch.sub(ch.dot(oc, oc, "c"), ch.mul(r, r, "c"), "c")
    disc = ch.sub(ch.mul(hb, hb, "disc"), ch.mul(a, cc, "disc"), "disc")
    out = {"oc": oc, "a": a, "half_b": hb, "c": cc, "disc": disc, "which": None}
    if disc >= 0.0:
        sq = ch.sqrt(disc, "sqrtd")
        ra = ch.div(ch.sub(-hb, sq, "root_a"), a, "root_a")
        rb = ch.div(ch.add(-hb, sq, "root_b"), a, "root_b")
        out.update(sqrtd=sq, root_a=ra, root_b=rb)
        for which, t in (("a", ra), ("b", rb)):
            if t < t_max and t > t_min:
                p = tuple(ch.add(o[k], ch.mul(d[k], t, "p"), "p") for k in range(3))
                n = tuple(ch.div(ch.sub(p[k], c[k], "n"), r, "n") for k in range(3))
                dn = ch.dot(d, n, "d.n")
                front = dn < 0.0
                out.update(which=which, t=t, p=p, raw_normal=n, dn=dn, front=front, normal=n if front else tuple(-x for x in n))
                break
    return out


def glass_limit(ch, h, d, ir):
    """materials.rs:182-188 at hit record h: ratio, cos_theta before and after min(1.0), sin_theta, ratio·sin_theta."""
    ratio = ch.div(1.0, ir, "ratio") if h["front"] else ir
    ud = ch.unit(d, "ud")
    raw = ch.dot(tuple(-x for x in ud), h["normal"], "cos")
    cos = min(raw, 1.0)
    sin = ch.sqrt(ch.sub(1.0, ch.mul(cos, cos, "sin"), "sin"), "sin")
    return {"ratio": ratio, "ud": ud, "cos_raw": raw, "cos": cos, "sin": sin, "ratio_sin": ch.mul(ratio, sin, "ratio*sin")}


def reflectance(cosine, ref_idx):            # materials.rs:151-155, powi(5) = x * (x^2)^2
    r0 = (1.0 - ref_idx) / (1.0 + ref_idx)
    r0 = r0 * r0
    x = 1.0 - cosine
    x2 = x * x
    return r0 + (1.0 - r0) * (x * (x2 * x2))


def np_sphere_hit(c, r, o, d):
    """The same expressions, vectorised over rays in numpy float64: (disc, root_a, root_b) with NaN roots where disc < 0."""
    c, o, d = (np.asarray(v, np.float64) for v in (c, o, d))
    oc = o - c
    a = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    hb = (oc[:, 0] * d[:, 0] + oc[:, 1] * d[:, 1]) + oc[:, 2] * d[:, 2]
    cc = ((oc[:, 0] * oc[:, 0] + oc[:, 1] * oc[:, 1]) + oc[:, 2] * oc[:, 2]) - np.asarray(r, np.float64) * np.asarray(r, np.float64)
    disc = hb * hb - a * cc
    with np.errstate(invalid="ignore"):
        sq = np.sqrt(disc)
    return disc, (-hb - sq) / a, (-hb + sq) / a


# ---- cases ---------------------------------------------------------------------------------------------------------------
def sphere(c, r, material):
    return {"center": _v(*c), "radius": float(r), "material": material}


def lam(r, g, b):
    return {"Lambertian": {"albedo": [r, g, b]}}


TEX = {"Texture": {"albedo": [0.0, 0.0, 0.0], "h_offset": 0.0, "width": 5, "height": 3, "pixels": "tex"}}
TEX_SIZE = (5, 3)


class Case:
    """One scene and its rays. `objects` has no lights; `lights` are the LIGHTS light spheres of the lit form. Ray i probes
    sphere target[i]; want[i] is what hit_world must report: {"sphere", "which" (root a/b or None), "t", "front"}.
    `claims` is the certificate: (statement, holds) pairs."""

    def __init__(self, name, objects, lights, o, d, target, want, claims, depth=8):
        self.name, self.objects, self.lights, self.depth = name, objects, lights, depth
        self.o = np.array(o, np.float64).reshape(-1, 3)
        self.d = np.array(d, np.float64).reshape(-1, 3)
        self.target, self.want, self.claims = list(target), list(want), list(claims)
        assert len(self.o) == len(self.d) == len(self.target) == len(self.want)

    def config(self, n_lights=0):
        objs = self.objects + self.lights[:n_lights]
        return base_config(4, 3, 1, self.depth, objs, look_from=(0, 0, 8), look_at=(0, 0, 0), vfov=60.0)

    def sphere_of(self, i):
        s = self.objects[i]
        return (s["center"]["x"], s["center"]["y"], s["center"]["z"]), s["radius"]


def _hit(sphere_idx, h):
    return {"sphere": sphere_idx, "which": h["which"], "t": h["t"], "front": h["front"]}


MISS = {"sphere": -1, "which": None, "t": None, "front": None}


# E1 ------------------------------------------------------------------------------------------------------------------------
E1_MATERIALS = [("lambertian", lam(0.7, 0.4, 0.2)), ("metal_fuzz0", {"Metal": {"albedo": [0.9, 0.8, 0.7], "fuzz": 0.0}}),
                ("metal_fuzz0.3", {"Metal": {"albedo": [0.6, 0.8, 0.9], "fuzz": 0.3}}),
                ("glass_1.5", {"Glass": {"index_of_refraction": 1.5}}), ("glass_1", {"Glass": {"index_of_refraction": 1.0}}),
                ("glass_0.5", {"Glass": {"index_of_refraction": 0.5}}), ("texture", TEX), ("light", {"Light": {}})]
E1_RADII = [2.0 ** -20, 1.0, P]
E1_SPEEDS = [2.0 ** -20, 1.0, P]
E1_CENTRES = [(0.0, 0.0, 0.0), (3.0 * 2 ** 18, -5.0 * 2 ** 16, 2.0 ** 19)]


def _nudge(c, r, o, d, step):
    """o_y moved by the fewest ulps (1 where it shows) that take disc off 0: one ulp of o_y vanishes in |oc|^2 = 17R^2 when
    ulp(o_y) is below 2^-50 R, as it is at c_y = 0."""
    y = o[1]
    for _ in range(64):
        y = step(y)
        if sphere_hit(Chain(), c, r, (o[0], y, o[2]), d)["disc"] != 0.0:
            return y
    raise AssertionError((c, r, o, d))


def e1(R, sign, c0):
    """One sphere of each material at c0 + (0, 0, 64 R k), radius sign·R; for each, o = c + (-4R, R, 0) and d = (s, 0, 0) for
    every s, then o_y the fewest ulps above (a miss) and below (two roots) that take disc off 0."""
    objs, o, d, target, want, claims = [], [], [], [], [], []
    for k, (mname, mat) in enumerate(E1_MATERIALS):
        c = (c0[0], c0[1], c0[2] + 64.0 * R * k)
        objs.append(sphere(c, sign * R, mat))
        for s in E1_SPEEDS:
            oo = (c[0] - 4.0 * R, c[1] + R, c[2])
            for tag, oy in (("tangent", oo[1]), ("+ulp", _nudge(c, sign * R, oo, (s, 0.0, 0.0), up)), ("-ulp", _nudge(c, sign * R, oo, (s, 0.0, 0.0), down))):
                ray_o, ray_d = (oo[0], oy, oo[2]), (s, 0.0, 0.0)
                ch = Chain()
                h = sphere_hit(ch, c, sign * R, ray_o, ray_d)
                what = f"{mname} s={s!r} {tag}"
                if tag == "tangent":
                    t = 4.0 * R / s
                    claims += [(f"{what}: nothing rounded", not ch.rounded), (f"{what}: disc == 0", h["disc"] == 0.0),
                               (f"{what}: root_a == root_b == 4R/s", h["root_a"] == h["root_b"] == t)]
                    if t > T_MIN:
                        claims += [(f"{what}: p == c + (0, R, 0)", h["p"] == (c[0], c[1] + R, c[2])),
                                   (f"{what}: d·n == 0, front_face false", h["dn"] == 0.0 and h["front"] is False)]
                        claims += _e1_shading(what, mname, mat, h, ray_d, c)
                    else:
                        claims.append((f"{what}: the root 4R/s is below t_min", h["which"] is None))
                elif tag == "+ulp":
                    claims.append((f"{what}: disc < 0, a miss", h["disc"] < 0.0 and h["which"] is None))
                else:
                    claims.append((f"{what}: disc > 0, two roots", h["disc"] > 0.0 and h["root_a"] < h["root_b"]))
                    if h["which"] is not None:
                        claims.append((f"{what}: the near root", h["which"] == "a"))
                o.append(ray_o); d.append(ray_d); target.append(k)
                want.append(_hit(k, h) if h["which"] else MISS)
    # the lights sit at -z, clear of every row of spheres and of the rays along x
    lights = [sphere((c0[0], c0[1] + 16.0 * R, c0[2] - 48.0 * R), 4.0 * R, {"Light": {}}),
              sphere((c0[0] + 24.0 * R, c0[1] - 8.0 * R, c0[2] - 40.0 * R), 4.0 * R, {"Light": {}})]
    name = f"E1_tangent_R{_p2(R)}_{'neg' if sign < 0 else 'pos'}_c{'0' if c0 == (0.0, 0.0, 0.0) else 'off'}"
    return Case(name, objs, lights, o, d, target, want, claims)


def _p2(x):
    e = int(math.log2(x))
    assert 2.0 ** e == x
    return f"2^{e}"


def _e1_shading(what, mname, mat, h, d, c):
    """The first shading step at a tangent hit: the claims that put it on its equality."""
    out = []
    n = h["normal"]
    if mname.startswith("metal"):
        # reflected = d - n·2(d·n) = d; scattered·n == fuzz·(rand·n), which is 0 (hence absorbed) exactly when fuzz is 0
        out.append((f"{what}: d·normal == 0, so fuzz 0 scatters along d with scattered·n == 0 (absorbed)", Chain().dot(d, n) == 0.0))
    elif mname.startswith("glass"):
        ch = Chain()
        ir = mat["Glass"]["index_of_refraction"]
        g = glass_limit(ch, h, d, ir)
        out.append((f"{what}: ratio = ir (back face), cos == 0, sin == 1, exactly", not ch.rounded and g["ratio"] == ir and g["cos"] == 0.0 and g["sin"] == 1.0))
        if ir == 1.5:
            out.append((f"{what}: 1.5·1 > 1: cannot refract", g["ratio_sin"] > 1.0))
        elif ir == 1.0:
            out.append((f"{what}: 1·1 == 1, not > 1: may refract, and reflectance(0, 1) == 1 reflects", g["ratio_sin"] == 1.0 and reflectance(0.0, 1.0) == 1.0))
        else:
            out.append((f"{what}: 0.5·1 < 1: may refract", g["ratio_sin"] == 0.5))
    elif mname == "texture":
        ch = Chain()
        nu = ch.unit(ch.vsub(h["p"], c))
        out.append((f"{what}: the pole, v == 1", not ch.rounded and nu[1] * 0.5 + 0.5 == 1.0))
    return out


# E2 ------------------------------------------------------------------------------------------------------------------------
def _search(f, x0, goal, span=4096):
    """The x nearest x0, ulp by ulp, with f(x) == goal."""
    lo = hi = x0
    for _ in range(span):
        if f(lo) == goal:
            return lo
        if f(hi) == goal:
            return hi
        lo, hi = down(lo), up(hi)
    raise AssertionError(f"no value near {x0!r} gives {goal!r}")


def _roots(xc, r):
    """(root_a, root_b) of o = 0, d = (1, 0, 0) against the sphere at (xc, 0, 0) of radius r, in the reference's order."""
    h = sphere_hit(Chain(), (xc, 0.0, 0.0), r, (0.0, 0.0, 0.0), (1.0, 0.0, 0.0), -MAX, MAX)
    return h.get("root_a", math.nan), h.get("root_b", math.nan)


def _step(f, x, step):
    """The nearest x' beyond x, ulp by ulp, with f(x') != f(x)."""
    y, fx = step(x), f(x)
    while f(y) == fx:
        y = step(y)
    return y


E2_RA = 2.0 ** -12                           # the radius of the spheres whose near root is probed (outside, 0.001 + r ahead)
E2_RB = 2.0 ** -10                           # the radius of the sphere whose far root is probed (origin inside, 0.001 - r ahead)


def e2_centres():
    """{label: centre x}: root_a == t_min, root_a == next(t_min), root_b == t_min, each found by search."""
    xa = _search(lambda x: _roots(x, E2_RA)[0], T_MIN + E2_RA, T_MIN)
    xn = _search(lambda x: _roots(x, E2_RA)[0], up(T_MIN) + E2_RA, up(T_MIN))
    xb = _search(lambda x: _roots(x, E2_RB)[1], T_MIN - E2_RB, T_MIN)
    return {"root_a=t_min": (xa, E2_RA), "root_a=next(t_min)": (xn, E2_RA), "root_b=t_min": (xb, E2_RB)}


def e2(mname, mat):
    """Rows at y = 4j: the probed sphere (centre found by search, and its two neighbours) ahead of o = (0, 4j, 0), d = (1, 0,
    0), and a Lambertian backstop of radius 1 at (3, 4j, 0) that catches a ray which passes the probed sphere."""
    objs, o, d, target, want, claims = [], [], [], [], [], []
    row = 0
    for label, (x0, r) in e2_centres().items():
        probe = (lambda x: _roots(x, r)[0]) if label.startswith("root_a") else (lambda x: _roots(x, r)[1])
        for tag, xc in (("found", x0), ("next", _step(probe, x0, up)), ("prev", _step(probe, x0, down))):
            y = 4.0 * row
            row += 1
            i = len(objs)
            objs.append(sphere((xc, y, 0.0), r, mat))
            objs.append(sphere((3.0, y, 0.0), 1.0, lam(0.2, 0.5, 0.8)))
            ro, rd = (0.0, y, 0.0), (1.0, 0.0, 0.0)
            h = sphere_hit(Chain(), (xc, y, 0.0), r, ro, rd)
            hb = sphere_hit(Chain(), (3.0, y, 0.0), 1.0, ro, rd)
            what = f"{label} {tag}"
            ra, rb = h["root_a"], h["root_b"]
            if tag == "found":
                if label == "root_a=t_min":
                    claims += [(f"{what}: root_a == 0.001 exactly, rejected; root_b taken, back face", ra == T_MIN and h["which"] == "b" and not h["front"])]
                elif label == "root_a=next(t_min)":
                    claims += [(f"{what}: root_a == next(0.001), accepted, front face", ra == up(T_MIN) and h["which"] == "a" and h["front"])]
                else:
                    claims += [(f"{what}: root_a < 0 and root_b == 0.001: a miss", ra < 0.0 and rb == T_MIN and h["which"] is None)]
            else:
                claims.append((f"{what}: the nearest centre whose root moves, one double away", probe(xc) in (up(probe(x0)), down(probe(x0)))))
            o.append(ro); d.append(rd); target.append(i)
            want.append(_hit(i, h) if h["which"] else _hit(i + 1, hb))
    lights = [sphere((1.0, -6.0, -3.0), 0.5, {"Light": {}}), sphere((-2.0, 4.0 * row + 2.0, 1.5), 0.5, {"Light": {}})]
    return Case(f"E2_t_min_{mname}", objs, lights, o, d, target, want, claims)


# E3 ------------------------------------------------------------------------------------------------------------------------
MAT_A, MAT_B = lam(0.9, 0.2, 0.1), {"Metal": {"albedo": [0.1, 0.3, 0.9], "fuzz": 0.1}}


def _tie(name, pair, rays, order, extra=(), lights=(), k_want=None):
    """The pair (geometry, material) in `order`, then `extra`; every ray must see both members at one root, the first index
    winning."""
    objs = [pair[j] for j in order] + list(extra)
    o, d, target, want, claims = [], [], [], [], []
    for ro, rd in rays:
        hs, chs = [None, None], []
        for j in (0, 1):
            ch = Chain()
            hs[j] = sphere_hit(ch, *_cr(objs[j]), ro, rd)
            chs.append(ch)
        what = f"o={ro} d={rd}"
        claims += [(f"{what}: nothing rounded", not chs[0].rounded and not chs[1].rounded),
                   (f"{what}: both members hit at one root", hs[0]["which"] is not None and hs[0]["t"] == hs[1]["t"])]
        o.append(ro); d.append(rd); target.append(0); want.append(_hit(0, hs[0]))
    return Case(name, objs, list(lights), o, d, target, want, claims)


def _cr(s):
    return (s["center"]["x"], s["center"]["y"], s["center"]["z"]), s["radius"]


def _rays_along_x(origins, speeds):
    return [((x, 0.0, 0.0), (-s, 0.0, 0.0)) for x in origins for s in speeds]


N_DISTRACT = 48                              # spheres per cluster: more than the largest leaf (32) holds


def distractors():
    """Two mirrored clusters of N_DISTRACT spheres of the pair's radius 1 beside the externally tangent pair A (centre 0) and B
    (centre (2, 0, 0)), centred at x <= -0.25 and x >= 2.25: boxes of one size on either side of the contact, so that the
    builder splits the scene between A's side and B's. They reach x = 0.75 and 1.25 at most, so the rays through the contact,
    which run in the plane x = 1, never meet them."""
    pts = [(x, y, z) for x in (-0.25, -1.0, -1.75, -2.5) for y in (-2.25, -1.5, -0.75, 0.0, 0.75, 1.5, 2.25) for z in (-1.5, 0.0, 1.5)]
    side = [sphere(p, 1.0, lam(0.3, 0.3, 0.3)) for p in pts[:N_DISTRACT]]
    return side + [sphere((2.0 - p[0], p[1], p[2]), 1.0, lam(0.4, 0.4, 0.2)) for p in pts[:N_DISTRACT]]


def e3_cases():
    out = []
    lights = [sphere((0.0, 24.0, -16.0), 2.0, {"Light": {}}), sphere((-20.0, -16.0, 6.0), 2.0, {"Light": {}})]
    # internally tangent: A (0, R 1) and B ((0.5, 0, 0), R 0.5) touch at (1, 0, 0); rays along -x see both at t = (x - 1)/s
    inner = (sphere((0.0, 0.0, 0.0), 1.0, MAT_A), sphere((0.5, 0.0, 0.0), 0.5, MAT_B))
    for order in ((0, 1), (1, 0)):
        out.append(_tie(f"E3_internal_{order[0]}{order[1]}", inner, _rays_along_x((4.0, 3.0, 65.0), (1.0, 0.5, 2.0 ** 10)), order, lights=lights))
    # externally tangent: A (0, R 1) and B ((2, 0, 0), R 1); rays along y through the contact (1, 0, 0), tangent to both
    outer = (sphere((0.0, 0.0, 0.0), 1.0, MAT_A), sphere((2.0, 0.0, 0.0), 1.0, MAT_B))
    rays = [((1.0, -y, 0.0), (0.0, s, 0.0)) for y in (4.0, 0.5) for s in (1.0, 0.25, 8.0)] + [((1.0, 0.0, 3.0), (0.0, 0.0, -1.0))]
    for order in ((0, 1), (1, 0)):
        c = _tie(f"E3_external_{order[0]}{order[1]}", outer, rays, order, lights=lights)
        c.claims += [(f"o={ro} d={rd}: disc == 0 and d·n == 0 for both", all(sphere_hit(Chain(), *_cr(c.objects[j]), ro, rd)["disc"] == 0.0
                                                                            and sphere_hit(Chain(), *_cr(c.objects[j]), ro, rd)["dn"] == 0.0 for j in (0, 1)))
                     for ro, rd in rays]
        out.append(c)
    # the external pair with distractors that put A and B in different leaves (checked on the built hierarchies); the lights
    # lie far out along x, so that x stays the widest centroid axis where the builder falls back to median splits
    for order in ((0, 1), (1, 0)):
        out.append(_tie(f"E3_leaves_{order[0]}{order[1]}", outer, rays, order, extra=distractors(),
                        lights=[sphere((-30.0, 4.0, -3.0), 2.0, {"Light": {}}), sphere((32.0, -4.0, 3.0), 2.0, {"Light": {}})]))
    # one member on the always-list: A of radius 2^50 (|c - g| + r >= 1e15) at (2^50, 0, 0) and B of radius 2^22 at (2^22, 0, 0)
    # touch at the origin; from (-2^24, 0, 0) along +x both roots are 2^24, every product exact (2^100 + 2^75 + 2^48 has 53 bits)
    huge = (sphere((2.0 ** 50, 0.0, 0.0), 2.0 ** 50, MAT_A), sphere((2.0 ** 22, 0.0, 0.0), 2.0 ** 22, MAT_B))
    tree = [sphere((2.0 ** 22 + 2.0 ** 20 * (i % 4), 2.0 ** 23 * (1 + i // 4), 0.0), 2.0 ** 19, lam(0.3, 0.3, 0.3)) for i in range(12)]
    for order in ((0, 1), (1, 0)):
        out.append(_tie(f"E3_always_{order[0]}{order[1]}", huge, [((-2.0 ** 24, 0.0, 0.0), (s, 0.0, 0.0)) for s in (1.0, 2.0 ** 10, 2.0 ** -4)],
                        order, extra=tree, lights=[sphere((0.0, -2.0 ** 26, 2.0 ** 25), 2.0 ** 21, {"Light": {}}),
                                                   sphere((-2.0 ** 25, 2.0 ** 24, -2.0 ** 25), 2.0 ** 21, {"Light": {}})]))
    return out


def always_member(case):
    """The index of the always-list member of an E3_always case."""
    return next(i for i in (0, 1) if case.objects[i]["radius"] == 2.0 ** 50)


# E4 ------------------------------------------------------------------------------------------------------------------------
E4_OFFSETS = [0.75, 0.5]


def _limit_of(h_off, inside):
    """fl(ratio·sin_theta) at the first hit of the ray at height h_off through the unit sphere at the origin, from inside (o =
    (0, h_off, 0)) or outside (o = (-4, h_off, 0)), as a function of ir."""
    o = (0.0, h_off, 0.0) if inside else (-4.0, h_off, 0.0)
    h = sphere_hit(Chain(), (0.0, 0.0, 0.0), 1.0, o, (1.0, 0.0, 0.0))
    return o, h, (lambda ir: glass_limit(Chain(), h, (1.0, 0.0, 0.0), ir)["ratio_sin"])


def e4():
    """Glass spheres of radius 1 in rows at y = 4j, each with the ir (found by search, and its two neighbours) at which
    fl(ratio·sin_theta) == 1.0 for its ray: from inside (back face, ratio = ir > 1) and from outside (ratio = 1/ir, ir < 1)."""
    objs, o, d, target, want, claims = [], [], [], [], [], []
    for inside in (True, False):
        for h_off in E4_OFFSETS:
            ro0, h, f = _limit_of(h_off, inside)
            sin = glass_limit(Chain(), h, (1.0, 0.0, 0.0), 1.0)["sin"]
            ir0 = _search(f, 1.0 / sin if inside else sin, 1.0)
            for tag, ir in (("found", ir0), ("next", up(ir0)), ("prev", down(ir0))):
                y = 4.0 * len(objs)
                i = len(objs)
                objs.append(sphere((0.0, y, 0.0), 1.0, {"Glass": {"index_of_refraction": ir}}))
                ro, rd = (ro0[0], y + h_off, 0.0), (1.0, 0.0, 0.0)
                hh = sphere_hit(Chain(), (0.0, y, 0.0), 1.0, ro, rd)
                g = glass_limit(Chain(), hh, rd, ir)
                what = f"{'inside' if inside else 'outside'} h={h_off} ir {tag}={ir!r}"
                claims.append((f"{what}: front_face {not inside}", hh["which"] is not None and hh["front"] == (not inside)))
                if tag == "found":
                    claims.append((f"{what}: fl(ratio·sin_theta) == 1.0 exactly, not > 1 (may refract)", g["ratio_sin"] == 1.0))
                claims.append((f"{what}: the row's ray sees what the search saw", g["ratio_sin"] == f(ir)))
                o.append(ro); d.append(rd); target.append(i); want.append(_hit(i, hh))
    lights = [sphere((-6.0, -5.0, -4.0), 1.0, {"Light": {}}), sphere((6.0, 4.0 * len(objs) + 2.0, 4.0), 1.0, {"Light": {}})]
    return Case("E4_refraction_limit", objs, lights, o, d, target, want, claims, depth=12)


# E5 ------------------------------------------------------------------------------------------------------------------------
# o = (0, y, 0), d = (1, 0, 0), the sphere at (X, y, 0) of radius R with 2^-53 < R^2 < 2^-52 <= ulp(X^2): c = fl(X^2 - R^2)
# rounds down to X^2 - 2^-52, so disc == 2^-52 exactly, sqrtd == 2^-26 > R and the normal (p - c)/R has length 2^-26/R > 1.
# At normal incidence -unit_direction·n is then that length: well above 1, where an unclamped cos_theta moves reflectance
# (x = 1 - cos_theta < 0) and sin_theta is NaN. (A dot product that rounds to 1 + 1 ulp is clamped to the same decisions
# as an unclamped one: sin_theta NaN and 0 both fail `> 1.0`, and reflectance(1 + 1 ulp) rounds to reflectance(1).) Behind
# each ray's origin a Lambertian backstop at (-4, y, 0) catches the reflected ray, while the refracted one goes on to the sky,
# so that the reflect/refract draw shows in the radiance (both directions are horizontal, where the gradient sky is one colour).
E5_SPHERES = [(1.0 + 2.0 ** -20, 3.0 * 2.0 ** -28), (1.25, 23.0 * 2.0 ** -31), (1.0 + 2.0 ** -10, 3.0 * 2.0 ** -28)]
E5_INDICES = [1.5, 2.5]


def e5():
    objs, o, d, target, want, claims = [], [], [], [], [], []
    for X, R in E5_SPHERES:
        for ir in E5_INDICES:
            y = 4.0 * len(objs)
            i = len(objs)
            objs.append(sphere((X, y, 0.0), R, {"Glass": {"index_of_refraction": ir}}))
            objs.append(sphere((-4.0, y, 0.0), 1.0, lam(0.9, 0.1, 0.5)))
            ro, rd = (0.0, y, 0.0), (1.0, 0.0, 0.0)
            ch = Chain()
            h = sphere_hit(ch, (X, y, 0.0), R, ro, rd)
            g = glass_limit(Chain(), h, rd, ir)
            what = f"X={X!r} R={R!r} ir={ir}"
            claims += [(f"{what}: 2^-53 < R^2 < 2^-52 exactly", Q(2) ** -53 < Q(R) ** 2 < Q(2) ** -52),
                       (f"{what}: c rounds down, disc == 2^-52 exactly, only n rounds after", ch.rounded == ["c", "n"] and h["disc"] == 2.0 ** -52),
                       (f"{what}: front face, -ud·n > 1.3, clamped to 1, sin_theta == 0", h["front"] and g["cos_raw"] > 1.3 and g["cos"] == 1.0 and g["sin"] == 0.0),
                       (f"{what}: unclamped, reflectance drops by more than 0.003", reflectance(1.0, 1.0 / ir) - reflectance(g["cos_raw"], 1.0 / ir) > 0.003)]
            o.append(ro); d.append(rd); target.append(i); want.append(_hit(i, h))
    lights = [sphere((0.5, -3.0, -2.0), 0.5, {"Light": {}}), sphere((0.5, 4.0 * len(objs) + 1.0, 2.0), 0.5, {"Light": {}})]
    return Case("E5_cos_clamp", objs, lights, o, d, target, want, claims, depth=12)


def cases():
    """Every case, in a fixed order."""
    out = [e1(R, sign, c0) for R in E1_RADII for sign in (1.0, -1.0) for c0 in E1_CENTRES]
    out += [e2("lambertian", lam(0.8, 0.3, 0.3)), e2("glass", {"Glass": {"index_of_refraction": 1.5}})]
    out += e3_cases()
    out += [e4(), e5()]
    return out


def by_name():
    return {c.name: c for c in cases()}
