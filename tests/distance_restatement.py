"""The point queries' contract (include/rtb200.h, DESIGN.md §4.19) in numpy float64, chunked over the spheres: the brute-force
truth that the GPU tests hold every variant of rtb200_scene_nearest and rtb200_scene_overlaps to, bit for bit.

dist_j = fl(fl(sqrt(fl(fl(fl(x*x) + fl(y*y)) + fl(z*z)))) - |R|) with x = fl(p.x - c.x) and so on: numpy evaluates each
operation of that expression in float64 with one rounding, in this order."""
import numpy as np

NONE = -1
CHUNK = 1 << 22   # points x spheres per block


def sphere_arrays(scene):
    """(centres float64 [n, 3], radii float64 [n]) of a Scene's current list."""
    sp = scene._spheres[: scene.n_spheres]
    c = np.array([[s.center.x, s.center.y, s.center.z] for s in sp], np.float64).reshape(-1, 3)
    r = np.array([s.radius for s in sp], np.float64)
    return c, r


def distances(p, c, r):
    """dist_j of every point of p [m, 3] to every sphere: float64 [m, n]."""
    with np.errstate(invalid="ignore", over="ignore"):
        x = p[:, None, 0] - c[None, :, 0]
        y = p[:, None, 1] - c[None, :, 1]
        z = p[:, None, 2] - c[None, :, 2]
        s = np.sqrt((x * x + y * y) + z * z)
        return s - np.abs(r)[None, :]


def nearest(points, c, r, bound=None):
    """(sphere int32 [m] (-1: none), distance float64 [m] (+inf: none)): the j with dist_j < bound and the least dist_j, the
    lowest index among equal distances."""
    points = np.asarray(points, np.float64).reshape(-1, 3)
    m, n = len(points), len(r)
    b = np.full(m, np.inf) if bound is None else np.asarray(bound, np.float64)
    sphere = np.full(m, NONE, np.int32)
    dist = np.full(m, np.inf)
    if n == 0 or m == 0:
        return sphere, dist
    step = max(1, CHUNK // n)
    for a in range(0, m, step):
        d = distances(points[a:a + step], c, r)
        with np.errstate(invalid="ignore"):
            ok = d < b[a:a + step, None]              # NaN and +inf never qualify
        dd = np.where(ok, d, np.inf)
        j = np.argmin(dd, axis=1)                     # the first of equal minima; -0.0 == 0.0
        hit = ok[np.arange(len(j)), j]
        sphere[a:a + step] = np.where(hit, j, NONE)
        dist[a:a + step] = np.where(hit, d[np.arange(len(j)), j], np.inf)
    return sphere, dist


def overlaps(centers, radii, c, r):
    """uint8 [m]: 1 iff some sphere has dist_j < radii[i]."""
    return (nearest(centers, c, r, radii)[0] != NONE).astype(np.uint8)
