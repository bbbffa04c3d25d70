"""The variance of each pixel's mean through the temporal accumulation (rtb200_temporal_var[_device], include/rtb200.h step 8;
DESIGN.md §4.21) restated twice in numpy, which rounds every float64 and float32 operation to nearest and never fuses two:
`temporal` vectorised over the image and `temporal_scalar` with per-pixel Python loops over np.float64 / np.float32 scalars. The
CPU tests hold the two equal bit for bit; the GPU tests hold both kernels to `temporal`.

Step 8 reads the taps, weights, s and n of steps 5-6, so steps 1-7 are restated here once more, operation for operation as
tests/temporal_restatement.py and tests/temporal_clamp_restatement.py state them and with their helpers; the CPU tests hold the
colour and length to tests/temporal_clamp_restatement.py's. Both functions return (color float32 [h, w, 3], length uint32
[h, w], variance float32 [h, w, 3]); `variance` is this frame's and prev's "variance" the previous call's."""
import numpy as np

from temporal_clamp_restatement import check_clamp, window_bounds
from temporal_restatement import F32, F64, MISS, _dot, _project, camera_arrays, check, u32


def _check_prev(prev):
    if prev is not None and "variance" not in prev:
        raise ValueError("prev holds the previous call's variance")


# ---- vectorised ------------------------------------------------------------------------------------------------------------

def temporal(color, variance, sphere, point, camera, prev=None, *, motion=None, max_history, depth_tol, clamp=None, clamp_radius=1):
    """The new history (color, length, variance)."""
    check(max_history, depth_tol)
    gamma = None if clamp is None else check_clamp(clamp, clamp_radius)
    _check_prev(prev)
    c, v = np.asarray(color, F32), np.asarray(variance, F32)
    H, W, _ = c.shape
    out_c, out_n, out_v = c.copy(), np.ones((H, W), np.uint32), v.copy()
    if prev is None or H * W == 0:
        return out_c, out_n, out_v
    sph, P = u32(sphere), np.asarray(point, F64)
    cam, pcam = camera_arrays(camera), camera_arrays(prev["camera"])
    hc, hn, hs, hp = np.asarray(prev["color"], F32), u32(prev["length"]), u32(prev["sphere"]), np.asarray(prev["point"], F64)
    hv = np.asarray(prev["variance"], F32)
    mot = np.zeros((0, 3), F64) if motion is None else np.asarray(motion, F64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        # steps 1-6, as temporal_restatement.temporal
        hit = sph != MISS
        moved = hit & (sph < len(mot))
        Pp = np.where(moved[..., None], P - mot[np.where(moved, sph, 0).astype(np.int64)], P) if len(mot) else P
        y, x = np.meshgrid(np.arange(H, dtype=F64), np.arange(W, dtype=F64), indexing="ij")
        u = (x + F64(0.5)) / (F64(W) - F64(1))
        vv = (F64(H) - (y + F64(0.5))) / (F64(H) - F64(1))
        o, llc, hh, vt = cam
        miss_d = ((llc + hh * u[..., None]) + vt * vv[..., None]) - o
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
        vnum = np.zeros((H, W, 3), F32)                                    # step 8: sum of w * prev_variance over the same taps
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
            vnum = np.where(valid[..., None], vnum + w[..., None] * hv[qy, qx], vnum)
            L = np.where(valid, np.minimum(L, hn[qy, qx]), L)
        n = (np.minimum(L.astype(np.uint64), np.uint64(max_history - 1)) + np.uint64(1))
        blend = (s != 0) & (n >= 2)
        sd = np.where(blend, s, F32(1))[..., None]
        g = num / sd
        # step 7: h' = h < lo ? lo : (h > hi ? hi : h); Vh is not clamped
        if gamma is not None:
            lo, hi = window_bounds(c, gamma, clamp_radius)
            g = np.where(g < lo, lo, np.where(g > hi, hi, g))
        alpha = F32(1) / n.astype(F64).astype(F32)
        res = g + alpha[..., None] * (c - g)
        # step 8: (b * b) * Vh + (a * a) * v
        b = F32(1) - alpha
        rv = (b * b)[..., None] * (vnum / sd) + (alpha * alpha)[..., None] * v
        out_c = np.where(blend[..., None], res, c).astype(F32)
        out_n = np.where(blend, n, 1).astype(np.uint32)
        out_v = np.where(blend[..., None], rv, v).astype(F32)
    return out_c, out_n, out_v


# ---- scalar ----------------------------------------------------------------------------------------------------------------

def temporal_scalar(color, variance, sphere, point, camera, prev=None, *, motion=None, max_history, depth_tol, clamp=None,
                    clamp_radius=1):
    """The same contract pixel by pixel over np.float64 / np.float32 scalars, in the header's words."""
    check(max_history, depth_tol)
    gamma = None if clamp is None else check_clamp(clamp, clamp_radius)
    _check_prev(prev)
    c, v = np.asarray(color, F32), np.asarray(variance, F32)
    H, W, _ = c.shape
    out_c, out_n, out_v = c.copy(), np.ones((H, W), np.uint32), v.copy()
    if prev is None:
        return out_c, out_n, out_v
    sph, P = u32(sphere), np.asarray(point, F64)
    cam, pcam = camera_arrays(camera), camera_arrays(prev["camera"])
    hc, hn, hs, hp = np.asarray(prev["color"], F32), u32(prev["length"]), u32(prev["sphere"]), np.asarray(prev["point"], F64)
    hv = np.asarray(prev["variance"], F32)
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
        u, vv = dot(cross(vt, a), d) / den, dot(cross(a, h), d) / den
        return (u, vv) if np.isfinite(u) and np.isfinite(vv) else None

    def clamped(py, px, h):
        """Step 7 for pixel (px, py): the window's moments in window order, then the clamp of each channel."""
        r = clamp_radius
        S, Q, m = [F32(0)] * 3, [F32(0)] * 3, 0
        for qy in range(py - r, py + r + 1):
            for qx in range(px - r, px + r + 1):
                if not (0 <= qy < H and 0 <= qx < W):
                    continue
                cq = [c[qy, qx, k] for k in range(3)]
                if not all(np.isfinite(t) for t in cq):
                    continue
                S = [S[k] + cq[k] for k in range(3)]
                Q = [Q[k] + cq[k] * cq[k] for k in range(3)]
                m += 1
        out = []
        for k in range(3):
            mean = S[k] / F32(m)
            var = Q[k] / F32(m) - mean * mean
            sd = np.sqrt(F32(0) if var < 0 else var)
            lo, hi = mean - gamma * sd, mean + gamma * sd
            out.append(lo if h[k] < lo else (hi if h[k] > hi else h[k]))
        return out

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
                    vv = (F64(H) - (F64(py) + F64(0.5))) / (F64(H) - F64(1))
                    o, llc, h, vt = (vec(t) for t in cam)
                    d_cur = d_prev = [((llc[k] + h[k] * u) + vt[k] * vv) - o[k] for k in range(3)]
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
                s, num, vnum, L = F32(0), [F32(0)] * 3, [F32(0)] * 3, None
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
                    vnum = [vnum[k] + w * hv[qy, qx, k] for k in range(3)]   # a non-finite tap variance propagates
                    L = int(hn[qy, qx]) if L is None else min(L, int(hn[qy, qx]))
                if s == 0:
                    continue
                n = min(L, max_history - 1) + 1
                if n < 2:
                    continue
                a = F32(1) / F32(n)
                b = F32(1) - a
                g = [num[k] / s for k in range(3)]
                if gamma is not None:
                    g = clamped(py, px, g)
                for k in range(3):
                    out_c[py, px, k] = g[k] + a * (cp[k] - g[k])
                    out_v[py, px, k] = (b * b) * (vnum[k] / s) + (a * a) * v[py, px, k]
                out_n[py, px] = n
    return out_c, out_n, out_v
