"""The temporal accumulation contract of include/rtb200.h (rtb200_temporal[_device], DESIGN.md §4.16) restated twice in numpy,
which rounds every float64 and float32 operation to nearest and never fuses two: `temporal` vectorised over the image, one tap
at a time, and `temporal_scalar` with per-pixel Python loops over np.float64 / np.float32 scalars. The CPU tests hold the two
equal bit for bit; the GPU tests hold the kernel to `temporal`.

A camera is an rt_camera or a tuple (origin, lower_left_corner, horizontal, vertical) of 3-vectors. `prev` is None or a dict of
the previous frame's "color", "length", "sphere", "point" and "camera"."""
import numpy as np

F32, F64 = np.float32, np.float64
MISS = 0xFFFFFFFF


def camera_arrays(cam):
    if hasattr(cam, "lower_left_corner"):
        return tuple(np.array([v.x, v.y, v.z], F64) for v in (cam.origin, cam.lower_left_corner, cam.horizontal, cam.vertical))
    return tuple(np.asarray(v, F64) for v in cam)


def u32(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.int32 else a.astype(np.uint32)


def check(max_history, depth_tol):
    if max_history < 1:
        raise ValueError("max_history must be >= 1")
    if not (np.isfinite(depth_tol) and depth_tol >= 0):
        raise ValueError("depth_tol must be finite and >= 0")


# ---- vectorised ------------------------------------------------------------------------------------------------------------

def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _project(cam, d):
    o, llc, h, vt = cam
    a = llc - o
    cn = _cross(h, vt)
    den = _dot(cn, d)
    front = _dot(cn, a) / den
    u = _dot(_cross(vt, a), d) / den
    v = _dot(_cross(a, h), d) / den
    return u, v, (den != 0) & (front > 0) & np.isfinite(u) & np.isfinite(v)


def temporal(color, sphere, point, camera, prev=None, *, motion=None, max_history, depth_tol):
    """The new history (color float32 [h, w, 3], length uint32 [h, w])."""
    check(max_history, depth_tol)
    c = np.asarray(color, F32)
    H, W, _ = c.shape
    out_c, out_n = c.copy(), np.ones((H, W), np.uint32)
    if prev is None or H * W == 0:
        return out_c, out_n
    sph, P = u32(sphere), np.asarray(point, F64)
    cam, pcam = camera_arrays(camera), camera_arrays(prev["camera"])
    hc, hn, hs, hp = np.asarray(prev["color"], F32), u32(prev["length"]), u32(prev["sphere"]), np.asarray(prev["point"], F64)
    mot = np.zeros((0, 3), F64) if motion is None else np.asarray(motion, F64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        hit = sph != MISS
        moved = hit & (sph < len(mot))
        Pp = np.where(moved[..., None], P - mot[np.where(moved, sph, 0).astype(np.int64)], P) if len(mot) else P
        y, x = np.meshgrid(np.arange(H, dtype=F64), np.arange(W, dtype=F64), indexing="ij")
        u = (x + F64(0.5)) / (F64(W) - F64(1))
        v = (F64(H) - (y + F64(0.5))) / (F64(H) - F64(1))
        o, llc, hh, vt = cam
        miss_d = ((llc + hh * u[..., None]) + vt * v[..., None]) - o
        dc = np.where(hit[..., None], P - cam[0], miss_d)
        dp = np.where(hit[..., None], Pp - pcam[0], miss_d)
        uc, vc, okc = _project(cam, dc)
        up, vp, okp = _project(pcam, dp)
        fx = x + (up - uc) * (F64(W) - F64(1))
        fy = y - (vp - vc) * (F64(H) - F64(1))
        base = np.isfinite(c).all(axis=2) & okc & okp & np.isfinite(fx) & np.isfinite(fy)
        x0, y0 = np.floor(fx), np.floor(fy)
        ax, ay = (fx - x0).astype(F32), (fy - y0).astype(F32)
        bx, by = F32(1) - ax, F32(1) - ay
        weights = (bx * by, ax * by, bx * ay, ax * ay)
        lim = (F64(depth_tol) * F64(depth_tol)) * _dot(dp, dp)
        s = np.zeros((H, W), F32)
        num = np.zeros((H, W, 3), F32)
        L = np.full((H, W), MISS, np.uint32)
        for k in range(4):
            tx, ty = x0 + F64(k & 1), y0 + F64(k >> 1)
            w = weights[k]
            inside = base & (w > 0) & (tx >= 0) & (tx < W) & (ty >= 0) & (ty < H)
            qx, qy = np.where(inside, tx, 0).astype(np.int64), np.where(inside, ty, 0).astype(np.int64)
            hcq = hc[qy, qx]
            e = hp[qy, qx] - Pp
            valid = (inside & (hn[qy, qx] >= 1) & (hs[qy, qx] == sph) & np.isfinite(hcq).all(axis=2)
                     & (~hit | (_dot(e, e) <= lim)))
            s = np.where(valid, s + w, s)
            num = np.where(valid[..., None], num + w[..., None] * hcq, num)
            L = np.where(valid, np.minimum(L, hn[qy, qx]), L)
        n = (np.minimum(L.astype(np.uint64), np.uint64(max_history - 1)) + np.uint64(1))
        blend = (s != 0) & (n >= 2)
        g = num / np.where(blend, s, F32(1))[..., None]
        alpha = F32(1) / n.astype(F64).astype(F32)
        res = g + alpha[..., None] * (c - g)
        out_c = np.where(blend[..., None], res, c).astype(F32)
        out_n = np.where(blend, n, 1).astype(np.uint32)
    return out_c, out_n


# ---- scalar ----------------------------------------------------------------------------------------------------------------

def temporal_scalar(color, sphere, point, camera, prev=None, *, motion=None, max_history, depth_tol):
    """The same contract pixel by pixel over np.float64 / np.float32 scalars, in the header's words."""
    check(max_history, depth_tol)
    c = np.asarray(color, F32)
    H, W, _ = c.shape
    out_c, out_n = c.copy(), np.ones((H, W), np.uint32)
    if prev is None:
        return out_c, out_n
    sph, P = u32(sphere), np.asarray(point, F64)
    cam, pcam = camera_arrays(camera), camera_arrays(prev["camera"])
    hc, hn, hs, hp = np.asarray(prev["color"], F32), u32(prev["length"]), u32(prev["sphere"]), np.asarray(prev["point"], F64)
    mot = [] if motion is None else np.asarray(motion, F64).reshape(-1, 3)

    def vec(a):
        return [F64(a[0]), F64(a[1]), F64(a[2])]

    def sub(a, b):
        return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]

    def dot(a, b):
        return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]

    def cross(a, b):
        return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]

    def project(cm, d):
        o, llc, h, vt = (vec(t) for t in cm)
        a = sub(llc, o)
        cn = cross(h, vt)
        den = dot(cn, d)
        if den == 0:
            return None
        if not dot(cn, a) / den > 0:
            return None
        u, v = dot(cross(vt, a), d) / den, dot(cross(a, h), d) / den
        return (u, v) if np.isfinite(u) and np.isfinite(v) else None

    with np.errstate(all="ignore"):
        for py in range(H):
            for px in range(W):
                cp = [c[py, px, k] for k in range(3)]
                if not all(np.isfinite(t) for t in cp):
                    continue
                j = int(sph[py, px])
                if j != MISS:
                    Pv = vec(P[py, px])
                    Pprev = sub(Pv, vec(mot[j])) if j < len(mot) else Pv
                    d_cur, d_prev = sub(Pv, vec(cam[0])), sub(Pprev, vec(pcam[0]))
                else:
                    u = (F64(px) + F64(0.5)) / (F64(W) - F64(1))
                    v = (F64(H) - (F64(py) + F64(0.5))) / (F64(H) - F64(1))
                    o, llc, h, vt = (vec(t) for t in cam)
                    d_cur = d_prev = [((llc[k] + h[k] * u) + vt[k] * v) - o[k] for k in range(3)]
                pc, pp = project(cam, d_cur), project(pcam, d_prev)
                if pc is None or pp is None:
                    continue
                fx = F64(px) + (pp[0] - pc[0]) * (F64(W) - F64(1))
                fy = F64(py) - (pp[1] - pc[1]) * (F64(H) - F64(1))
                if not (np.isfinite(fx) and np.isfinite(fy)):
                    continue
                x0, y0 = np.floor(fx), np.floor(fy)
                ax, ay = F32(fx - x0), F32(fy - y0)
                taps = [(x0, y0, (F32(1) - ax) * (F32(1) - ay)), (x0 + 1, y0, ax * (F32(1) - ay)),
                        (x0, y0 + 1, (F32(1) - ax) * ay), (x0 + 1, y0 + 1, ax * ay)]
                s, num, L = F32(0), [F32(0)] * 3, None
                for tx, ty, w in taps:
                    if not (w > 0 and 0 <= tx < W and 0 <= ty < H):
                        continue
                    qx, qy = int(tx), int(ty)
                    if hn[qy, qx] < 1 or int(hs[qy, qx]) != j:
                        continue
                    hq = [hc[qy, qx, k] for k in range(3)]
                    if not all(np.isfinite(t) for t in hq):
                        continue
                    if j != MISS:
                        e = sub(vec(hp[qy, qx]), Pprev)
                        if not dot(e, e) <= (F64(depth_tol) * F64(depth_tol)) * dot(d_prev, d_prev):
                            continue
                    s = s + w
                    num = [num[k] + w * hq[k] for k in range(3)]
                    L = int(hn[qy, qx]) if L is None else min(L, int(hn[qy, qx]))
                if s == 0:
                    continue
                n = min(L, max_history - 1) + 1
                if n < 2:
                    continue
                alpha = F32(1) / F32(n)
                for k in range(3):
                    g = num[k] / s
                    out_c[py, px, k] = g + alpha * (cp[k] - g)
                out_n[py, px] = n
    return out_c, out_n
