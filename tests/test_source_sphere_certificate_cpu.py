"""The source-sphere certificate of the closest-hit stage (no GPU).

A secondary ray starts on the sphere it just left. Before the traversal, the kernel evaluates `leaves_sphere`
(csrc/rtb200_device.cuh) for that sphere; when it holds, the leaf step leaves the sphere out of the ray's exact-test
candidates. That is only sound if the exact f64 test (sphere_root, t_min 0.001) would reject the sphere. This test restates
both in numpy float64, whose element-wise operations are correctly rounded like the kernel's __d*_rn intrinsics. Over more
than 10^6 rays leaving sphere surfaces it checks that the certificate never holds for a sphere the exact test accepts, and
that it holds for nearly every ray leaving a surface outwards (DESIGN.md §4.2)."""
import numpy as np

from rtb200 import scenes
from synth import mixed_config

T_MIN = 0.001
DBL_MAX = np.finfo(np.float64).max


def _dot(ax, ay, az, bx, by, bz):
    return (ax * bx + ay * by) + az * bz                                   # dot(): ((x*x' + y*y') + z*z'), each op rounded


def _exact_accepts(c, r, o, d):
    """sphere_root(c, r, o, d, length_squared(d), 0.001, DBL_MAX) in the kernel's operation order; arrays of shape [n, 3]."""
    ocx, ocy, ocz = o[:, 0] - c[:, 0], o[:, 1] - c[:, 1], o[:, 2] - c[:, 2]
    hb = _dot(ocx, ocy, ocz, d[:, 0], d[:, 1], d[:, 2])
    cc = _dot(ocx, ocy, ocz, ocx, ocy, ocz) - r * r
    a = _dot(d[:, 0], d[:, 1], d[:, 2], d[:, 0], d[:, 1], d[:, 2])
    disc = hb * hb - a * cc
    ok = disc >= 0.0
    sq = np.sqrt(np.where(ok, disc, 0.0))
    ra, rb = (-hb - sq) / a, (-hb + sq) / a
    return ok & (((ra < DBL_MAX) & (ra > T_MIN)) | ((rb < DBL_MAX) & (rb > T_MIN)))


def _certified(c, r, o, d):
    """leaves_sphere(c, r, o, d, length_squared(d))."""
    ocx, ocy, ocz = o[:, 0] - c[:, 0], o[:, 1] - c[:, 1], o[:, 2] - c[:, 2]
    hb = _dot(ocx, ocy, ocz, d[:, 0], d[:, 1], d[:, 2])
    cc = _dot(ocx, ocy, ocz, ocx, ocy, ocz) - r * r
    a = _dot(d[:, 0], d[:, 1], d[:, 2], d[:, 0], d[:, 1], d[:, 2])
    lo, hi = 2.0 ** -300, 2.0 ** 300
    guard = (hb >= lo) & (hb <= hi) & (a >= lo) & (a <= hi)
    with np.errstate(invalid="ignore", over="ignore"):                 # NaN / inf lanes fail the guard anyway
        inside = (cc <= -lo) & (cc >= -hi) & ((a * -cc + 2.0 ** -48 * (hb * hb)) <= (0.0018 * a) * hb)
    return guard & ((cc >= 0.0) | inside)


def _unit(v):
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _spheres(cfg):
    objs = cfg["objects"]
    c = np.array([[s["center"]["x"], s["center"]["y"], s["center"]["z"]] for s in objs], np.float64)
    r = np.array([s["radius"] for s in objs], np.float64)
    return c, r


def _special_spheres():
    """Zero and negative radii, radius 1000, and spheres far from the origin."""
    c = np.array([[0.0, 0.0, 0.0], [1.0, 2.0, 3.0], [0.0, -1000.0, 0.0], [7.0e6, -3.0e6, 7.0e6], [-7.0e6, 1.0e3, 7.0e6],
                  [7.0e6, 7.0e6, 7.0e6], [3.0, 0.5, -2.0], [1e-3, 1e-3, 1e-3]], np.float64)
    r = np.array([0.0, -0.5, 1000.0, 0.2, -3.0, 1000.0, 1e-4, -1e-3], np.float64)
    return c, r


def _rays(c, r, kind, rng):
    """Rays leaving the surfaces of the spheres (c, r) like the shade stage writes them: o = the hit point, rounded near
    the surface (on either side), d = the scattered / reflected / shadow direction, unnormalised."""
    n = len(r)
    nrm = _unit(rng.normal(size=(n, 3)))                                   # geometric outward unit normal
    incoming = _unit(rng.normal(size=(n, 3)))
    incoming = np.where((np.sum(incoming * nrm, axis=1) > 0)[:, None], -incoming, incoming)   # arrives from outside
    t = 2.0 + 10.0 * rng.random(n)
    prev = (c + nrm * np.abs(r)[:, None]) - incoming * t[:, None]          # the previous origin, outside the sphere
    pd = incoming * t[:, None]
    o = prev + pd                                                          # ray.at(t): rounded onto, inside or outside
    # hit_record's normal: (p - c) / r, flipped to face the incoming ray (negative radii point inwards geometrically)
    out = (o - c) / np.where(r == 0.0, 1.0, r)[:, None]
    front = np.sum(pd * out, axis=1) < 0
    normal = np.where(front[:, None], out, -out)
    rs = rng.uniform(-1.0, 1.0, size=(n, 3))
    rs = rs[np.sum(rs * rs, axis=1) < 1.0]
    rs = np.resize(rs, (n, 3))
    if kind == "diffuse":                                                  # target = p + (normal + rs); d = target - p
        d = (o + (normal + rs)) - o
    elif kind == "metal":                                                  # reflect(d, n) + fuzz * rs
        dn = np.sum(pd * normal, axis=1)
        d = (pd - normal * (2.0 * dn)[:, None]) + rs * rng.uniform(0.0, 1.0, n)[:, None]
    elif kind == "grazing":                                                # n.d down to 1e-12 of |d|
        tang = _unit(np.cross(nrm, rng.normal(size=(n, 3))))
        eps = 10.0 ** rng.uniform(-12.0, -2.0, n) * rng.choice([-1.0, 1.0], n)
        d = tang + nrm * eps[:, None]
    elif kind == "inward":                                                 # refraction / a light behind the surface
        d = -nrm + 0.5 * rs
    elif kind == "axis":                                                   # zero direction components
        ax = rng.integers(0, 3, n)
        d = np.zeros((n, 3)); d[np.arange(n), ax] = rng.choice([-1.0, 1.0], n)
    else:
        raise ValueError(kind)
    d = d * rng.uniform(0.2, 5.0, n)[:, None]
    return o, d, np.sum(d * nrm * np.sign(np.where(r == 0.0, 1.0, r))[:, None], axis=1) > 0   # leaves the ball outwards


def test_certificate_never_holds_for_an_accepted_source_sphere():
    rng = np.random.default_rng(2024)
    scene_spheres = {
        "cover": _spheres(scenes.cover_config()),
        "10k": _spheres(scenes.rtiow_config(50)),
        "offset 7e6": _spheres(mixed_config(8, 6, 1, 2, seed=4, n=60, offset=(-3.0e6, 1.0e3, 7.0e6))),
        "special": _special_spheres(),
    }
    total = 0
    outward_diffuse = certified_diffuse = 0
    for name, (c_all, r_all) in scene_spheres.items():
        for kind in ("diffuse", "metal", "grazing", "inward", "axis"):
            m = 60_000
            j = rng.integers(0, len(r_all), m)
            c, r = c_all[j], r_all[j]
            o, d, outward = _rays(c, r, kind, rng)
            cert = _certified(c, r, o, d)
            accepted = _exact_accepts(c, r, o, d)
            bad = np.nonzero(cert & accepted)[0]
            assert bad.size == 0, (name, kind, [(c[i].tolist(), float(r[i]), o[i].tolist(), d[i].tolist()) for i in bad[:3]])
            total += m
            if kind == "diffuse" and name != "special":
                outward_diffuse += int(outward.sum()); certified_diffuse += int((cert & outward).sum())
            if kind == "inward":
                assert not np.any(cert & ~outward & (np.abs(r) > 0))    # rays into the ball are never certified
    assert total >= 1_000_000
    rate = certified_diffuse / outward_diffuse
    print(f"certificate holds for {rate:.4f} of {outward_diffuse} outward diffuse rays")
    assert rate > 0.95


def test_certificate_edge_cases():
    c = np.zeros((6, 3)); r = np.ones(6)
    o = np.array([[1.0, 0.0, 0.0]] * 6)
    d = np.array([[1.0, 0.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [np.nan, 0.0, 0.0], [np.inf, 0.0, 0.0], [1e-200, 0.0, 0.0]])
    cert = _certified(c, r, o, d)
    assert cert.tolist() == [True, False, False, False, False, False]   # outward; inward; tangent (half_b = 0); NaN; inf; tiny
    # just inside (cc < 0): certified while the far root stays below 0.0009, never once it could exceed t_min
    o_in = np.array([[np.nextafter(1.0, 0.0), 0.0, 0.0]])
    assert _certified(c[:1], r[:1], o_in, d[:1])[0] and not _exact_accepts(c[:1], r[:1], o_in, d[:1])[0]
    o_deep = np.array([[0.9995, 0.0, 0.0]])                                # far root 0.0005: rejected, but outside the bound's proof
    assert not _exact_accepts(c[:1], r[:1], o_deep, d[:1])[0]
    o_deeper = np.array([[0.998, 0.0, 0.0]])                               # far root 0.002: accepted, so never certified
    assert _exact_accepts(c[:1], r[:1], o_deeper, d[:1])[0] and not _certified(c[:1], r[:1], o_deeper, d[:1])[0]
