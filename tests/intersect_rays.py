"""Ray sets and comparisons of the closest-hit query tests (tests/test_intersect_cpu.py, tests/test_gpu_intersect.py,
tests/intersect_worker.py). Every set is (origin [n, 3], direction [n, 3]) float64."""
import numpy as np

import oracle_hit_world as OH
import rtb200 as R

MAX = float(np.finfo(np.float64).max)
FIELDS = [f[0] for f in R.HIT_FIELDS]


def scene_of(objects, w=32, h=24):
    """A resident-scene-ready Scene (and its config) holding `objects` under the cover scene's camera."""
    from rtb200 import scenes
    cfg = scenes._variant(scenes.cover_config(), w, h, 1, 4)
    cfg["objects"] = objects
    return R.Scene.from_config(cfg), cfg


def sphere(c, r, material=None):
    return {"center": {"x": float(c[0]), "y": float(c[1]), "z": float(c[2])}, "radius": float(r),
            "material": material or {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}}


def spheres_of(sc):
    """(centres [n, 3], radii [n]) of a Scene."""
    n = sc.n_spheres
    c = np.array([sc._spheres[i].center.tup() for i in range(n)], np.float64).reshape(n, 3)
    r = np.array([sc._spheres[i].radius for i in range(n)], np.float64)
    return c, r


def camera_rays(sc, w, h):
    """Camera::get_ray (camera.rs:79-84) through the centre of every pixel of a w x h grid, top row first."""
    cam = sc.c.camera
    o = np.array(cam.origin.tup()); llc = np.array(cam.lower_left_corner.tup())
    hor = np.array(cam.horizontal.tup()); ver = np.array(cam.vertical.tup())
    y, x = np.mgrid[0:h, 0:w]
    u = ((x + 0.5) / (w - 1.0)).reshape(-1, 1)
    v = ((h - (y + 0.5)) / (h - 1.0)).reshape(-1, 1)
    d = ((llc + hor * u) + ver * v) - o
    return np.broadcast_to(o, d.shape).copy(), np.ascontiguousarray(d)


def secondary_rays(hits, rng):
    """From every hit point: a diffuse direction (normal + a random unit vector) and the mirror direction of a random one."""
    m = hits["sphere"] >= 0
    p, nrm = hits["point"][m], hits["normal"][m]
    k = len(p)
    g = rng.normal(size=(k, 3))
    diffuse = nrm + g / np.linalg.norm(g, axis=1, keepdims=True)
    v = rng.normal(size=(k, 3))
    mirror = v - nrm * (2.0 * np.sum(v * nrm, axis=1, keepdims=True))
    return np.concatenate([p, p]), np.concatenate([diffuse, mirror])


def surface_rays(sc, rng, k):
    """k rays that start on random spheres' surfaces (centre + radius * unit vector), in random directions."""
    c, r = spheres_of(sc)
    j = rng.integers(0, len(r), size=k)
    g = rng.normal(size=(k, 3))
    g /= np.linalg.norm(g, axis=1, keepdims=True)
    return c[j] + g * r[j, None], rng.normal(size=(k, 3))


def box_rays(sc, rng, k, box=None):
    """k rays with origins uniform in the box of the sphere centres (or `box` = (lo, hi)) and random directions."""
    if box is None:
        c, _ = spheres_of(sc)
        c = c[np.isfinite(c).all(axis=1) & (np.abs(c) < 1e6).all(axis=1)]
        box = (c.min(axis=0), c.max(axis=0)) if len(c) else (np.full(3, -1.0), np.full(3, 1.0))
    lo, hi = box
    return lo + rng.random((k, 3)) * (hi - lo), rng.normal(size=(k, 3))


def grazing_rays(sc, rng, k):
    """Rays that pass a random sphere at a distance of its radius, scaled by 1 + {-4..4} ulp (tangent and just inside or
    outside), in a random direction perpendicular to the offset."""
    c, r = spheres_of(sc)
    ok = np.isfinite(r) & (np.abs(r) > 0) & np.isfinite(c).all(axis=1)
    idx = np.flatnonzero(ok)[rng.integers(0, ok.sum(), size=k)]
    d = rng.normal(size=(k, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    a = rng.normal(size=(k, 3))
    a -= d * np.sum(a * d, axis=1, keepdims=True)
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    scale = 1.0 + rng.integers(-4, 5, size=k) * np.finfo(np.float64).eps
    o = c[idx] + a * (np.abs(r[idx]) * scale)[:, None] - d * (3.0 * np.abs(r[idx]))[:, None]
    return o, d


def axis_rays(sc, rng, k):
    """Axis-parallel directions (some with a 1e-30 component: the slab test's clamped reciprocals) from box origins."""
    o, _ = box_rays(sc, rng, k)
    axes = np.concatenate([np.eye(3), -np.eye(3)])
    d = axes[rng.integers(0, 6, size=k)].copy()
    tiny = rng.random(k) < 0.5
    d[tiny] += rng.choice([-1e-30, 1e-30, 0.0], size=(int(tiny.sum()), 3))
    return o, d


def scaled_rays(sc, rng, k, scale):
    """Camera-like rays whose directions have length ~scale (1e-20 and 1e20 take the kernel out of its f32 frame)."""
    o, d = box_rays(sc, rng, k)
    return o, d * scale


def degenerate_rays(sc, rng):
    """Zero directions, and non-finite origins or directions."""
    o, d = box_rays(sc, rng, 16)
    inf, nan = np.inf, np.nan
    bad = [(0, 0, 0), (-0.0, 0, 0), (inf, 0, 0), (0, -inf, 0), (nan, 0, 0), (0, 0, nan), (inf, inf, inf), (1e308, 1e308, 1e308),
           (5e-324, 0, 0), (1e-300, -1e-300, 0)]
    oo, dd = [], []
    for b in bad:
        oo.append(o[0]); dd.append(b)            # odd directions from a good origin
        oo.append(b); dd.append(d[1])            # odd origins with a good direction
    oo.append((0.0, 0.0, 0.0)); dd.append((0.0, 0.0, 0.0))
    return np.array(oo, np.float64), np.array(dd, np.float64)


def assert_hits_equal(got, want, what="", fields=FIELDS):
    """Every field bit for bit; two NaNs count as equal whatever their payloads."""
    for k in fields:
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert a.shape == b.shape and a.dtype == b.dtype, (what, k, a.shape, b.shape, a.dtype, b.dtype)
        if a.dtype == np.float64:
            nan = np.isnan(a) & np.isnan(b)
            diff = (a.view(np.uint64) != b.view(np.uint64)) & ~nan
        else:
            diff = a != b
        if diff.any():
            i = int(np.argwhere(diff.reshape(len(a), -1).any(axis=1))[0][0])
            raise AssertionError(f"{what}: {k} differs for {int(diff.reshape(len(a), -1).any(axis=1).sum())} of {len(a)} rays, "
                                 f"first ray {i}: got {a[i]!r}, want {b[i]!r} (sphere {got['sphere'][i] if 'sphere' in got else '?'} vs {want['sphere'][i]})")


def oracle(sc, o, d, t_max=None):
    return OH.hit_world(sc, o, d, t_max)


def filtered(unbounded, t_max):
    """What hit_world under t_max must give, from the unbounded answer: the hit when its root is below t_max (a bound above
    f64::MAX counts as f64::MAX), else a miss."""
    tm = np.minimum(t_max, MAX)   # NaN stays NaN
    keep = (unbounded["sphere"] >= 0) & (unbounded["t"] < tm)
    out = {}
    miss = {"t": np.inf, "sphere": -1, "point": 0.0, "normal": 0.0, "uv": 0.0, "front_face": 0}
    for k in FIELDS:
        a = unbounded[k].copy()
        sel = ~keep
        a[sel] = miss[k]
        out[k] = a
    return out
