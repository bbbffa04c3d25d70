"""The variance-guided denoise contract of include/rtb200.h (rtb200_denoise_var[_device], DESIGN.md §4.18) restated twice in
float32 numpy, which rounds every operation and never fuses two: `denoise_var` vectorised over the image, one tap at a time, and
`denoise_var_scalar` with per-pixel Python loops over np.float32 scalars. The CPU tests hold the two equal bit for bit; the GPU
tests hold the kernels to `denoise_var`. Also `render_variance`, the variance of a render's pixel means from its samples."""
import numpy as np

F32 = np.float32
B = (F32(1 / 16), F32(1 / 4), F32(3 / 8), F32(1 / 4), F32(1 / 16))   # every B[i] * B[j] is exact in f32
G = (F32(1 / 4), F32(1 / 2), F32(1 / 4))                               # the variance prefilter's 3 x 3 kernel
TAPS = [(dx, dy) for dy in range(-2, 3) for dx in range(-2, 3)]
PRE_TAPS = [(dx, dy) for dy in range(-1, 2) for dx in range(-1, 2)]


def check(albedo, normal, iterations, color_weight, albedo_weight, normal_weight, variance_floor):
    """The host's refusals of the parameters, as ValueError."""
    if not 1 <= iterations <= 10:
        raise ValueError("iterations must be in [1, 10]")
    for name, lam in (("color", color_weight), ("albedo", albedo_weight), ("normal", normal_weight)):
        lam = F32(lam)
        if not np.isfinite(lam) or lam < 0:
            raise ValueError(f"{name}_weight must be finite and >= 0")
    eps = F32(variance_floor)
    if not np.isfinite(eps) or not eps > 0:
        raise ValueError("variance_floor must be finite and > 0")
    if (albedo is None and albedo_weight != 0) or (normal is None and normal_weight != 0):
        raise ValueError("a nonzero weight for an absent guide")


def _guides(albedo, normal, albedo_weight, normal_weight):
    given = [np.asarray(g, F32) for g in (albedo, normal) if g is not None]
    on = [(np.asarray(g, F32), F32(lam)) for g, lam in ((albedo, albedo_weight), (normal, normal_weight)) if g is not None and lam != 0]
    return given, on


def _window(ox, oy, h, w):
    """q = p + (ox, oy): the source window of q and the destination window of p, both inside the image (None when empty)."""
    ys, yd = slice(max(oy, 0), h + min(oy, 0)), slice(max(-oy, 0), h + min(-oy, 0))
    xs, xd = slice(max(ox, 0), w + min(ox, 0)), slice(max(-ox, 0), w + min(-ox, 0))
    if ys.start >= ys.stop or xs.start >= xs.stop:
        return None
    return ys, xs, yd, xd


def _dist(e):
    return (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]


def denoise_var(color, variance, albedo=None, normal=None, *, iterations, color_weight, albedo_weight=0.0, normal_weight=0.0,
                variance_floor):
    """(colour, variance), [h, w, 3] float32 each, vectorised: for each tap every pixel's sums take one step."""
    check(albedo, normal, iterations, color_weight, albedo_weight, normal_weight, variance_floor)
    c = np.array(color, F32, copy=True)
    var = np.array(variance, F32, copy=True)
    h, w, _ = c.shape
    given, on = _guides(albedo, normal, albedo_weight, normal_weight)
    guides_ok = np.ones((h, w), bool)
    for g in given:
        guides_ok &= np.isfinite(g).all(axis=2)
    lam_c, eps = F32(color_weight), F32(variance_floor)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        for i in range(iterations):
            step = 1 << i
            ok = guides_ok & np.isfinite(c).all(axis=2) & np.isfinite(var).all(axis=2) & (var >= 0).all(axis=2)
            v = (var[..., 0] + var[..., 1]) + var[..., 2]
            sv = np.zeros((h, w), F32)
            sw = np.zeros((h, w), F32)
            for dx, dy in PRE_TAPS:
                win = _window(dx, dy, h, w)
                if win is None:
                    continue
                ys, xs, yd, xd = win
                k = G[dx + 1] * G[dy + 1]
                valid = ok[ys, xs]
                sw[yd, xd] = np.where(valid, sw[yd, xd] + k, sw[yd, xd])
                sv[yd, xd] = np.where(valid, sv[yd, xd] + k * v[ys, xs], sv[yd, xd])
            scale = eps + sv / np.where(ok, sw, F32(1))   # eps + vbar_p, once per pixel
            num = np.zeros((h, w, 3), F32)
            den = np.zeros((h, w), F32)
            nv = np.zeros((h, w, 3), F32)
            for dx, dy in TAPS:
                win = _window(dx * step, dy * step, h, w)
                if win is None:
                    continue
                ys, xs, yd, xd = win
                valid = ok[yd, xd] & ok[ys, xs]
                f = None
                if lam_c != 0:
                    f = F32(1) + lam_c * (_dist(c[ys, xs] - c[yd, xd]) / scale[yd, xd])
                for g, lam in on:
                    fac = F32(1) + lam * _dist(g[ys, xs] - g[yd, xd])
                    f = fac if f is None else f * fac
                k = B[dx + 2] * B[dy + 2]
                wt = np.full(valid.shape, k, F32) if f is None else k / f
                num[yd, xd] = np.where(valid[..., None], num[yd, xd] + wt[..., None] * c[ys, xs], num[yd, xd])
                den[yd, xd] = np.where(valid, den[yd, xd] + wt, den[yd, xd])
                nv[yd, xd] = np.where(valid[..., None], nv[yd, xd] + (wt * wt)[..., None] * var[ys, xs], nv[yd, xd])
            d = np.where(ok, den, F32(1))
            c = np.where(ok[..., None], num / d[..., None], c).astype(F32)
            var = np.where(ok[..., None], nv / (d * d)[..., None], var).astype(F32)
    return c, var


def denoise_var_scalar(color, variance, albedo=None, normal=None, *, iterations, color_weight, albedo_weight=0.0,
                       normal_weight=0.0, variance_floor):
    """The same contract pixel by pixel and tap by tap over np.float32 scalars, with the ok flag carried as the header states
    it (ok' = ok && both results are finite) rather than recomputed."""
    check(albedo, normal, iterations, color_weight, albedo_weight, normal_weight, variance_floor)
    c = np.array(color, F32, copy=True)
    var = np.array(variance, F32, copy=True)
    h, w, _ = c.shape
    given, on = _guides(albedo, normal, albedo_weight, normal_weight)
    lam_c, eps = F32(color_weight), F32(variance_floor)

    def fin(img, y, x):
        return all(np.isfinite(img[y, x, k]) for k in range(3))

    ok = [[fin(c, y, x) and all(fin(g, y, x) for g in given) and fin(var, y, x) and all(var[y, x, k] >= 0 for k in range(3))
           for x in range(w)] for y in range(h)]

    def dist(img, y, x, py, px):
        e = [img[y, x, k] - img[py, px, k] for k in range(3)]
        return (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]

    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        for i in range(iterations):
            step = 1 << i
            nc, nvar = c.copy(), var.copy()
            nok = [row[:] for row in ok]
            for py in range(h):
                for px in range(w):
                    if not ok[py][px]:
                        continue
                    sw, sv = F32(0), F32(0)
                    for dy in range(-1, 2):
                        for dx in range(-1, 2):
                            qy, qx = py + dy, px + dx
                            if 0 <= qy < h and 0 <= qx < w and ok[qy][qx]:
                                k = G[dx + 1] * G[dy + 1]
                                sw = sw + k
                                sv = sv + k * ((var[qy, qx, 0] + var[qy, qx, 1]) + var[qy, qx, 2])
                    vbar = sv / sw
                    num, nv, den = [F32(0)] * 3, [F32(0)] * 3, F32(0)
                    for dy in range(-2, 3):
                        for dx in range(-2, 3):
                            qy, qx = py + step * dy, px + step * dx
                            if not (0 <= qy < h and 0 <= qx < w) or not ok[qy][qx]:
                                continue
                            f = None
                            if lam_c != 0:
                                f = F32(1) + lam_c * (dist(c, qy, qx, py, px) / (eps + vbar))
                            for g, lam in on:
                                fac = F32(1) + lam * dist(g, qy, qx, py, px)
                                f = fac if f is None else f * fac
                            k = B[dx + 2] * B[dy + 2]
                            wt = k if f is None else k / f
                            for ch in range(3):
                                num[ch] = num[ch] + wt * c[qy, qx, ch]
                            den = den + wt
                            for ch in range(3):
                                nv[ch] = nv[ch] + (wt * wt) * var[qy, qx, ch]
                    for ch in range(3):
                        nc[py, px, ch] = num[ch] / den
                        nvar[py, px, ch] = nv[ch] / (den * den)
                    nok[py][px] = fin(nc, py, px) and fin(nvar, py, px)
            c, var, ok = nc, nvar, nok
    return c, var


def render_variance(samples):
    """The variance of each pixel's mean from its samples x[n, ..., 3] (float32, in sample order), as the header states it:
    S_c and Q_c the f32 sums of x_c and x_c * x_c in sample order, inv = 1 / n, mean_c = inv * S_c, d_c = inv * Q_c -
    mean_c * mean_c, var_c = (d_c < 0 ? 0 : d_c) * inv (a NaN d_c stays NaN; n = 0 gives 0)."""
    x = np.asarray(samples, F32)
    if x.shape[0] == 0:
        return np.zeros(x.shape[1:], F32)
    S = np.zeros(x.shape[1:], F32)
    Q = np.zeros(x.shape[1:], F32)
    with np.errstate(all="ignore"):
        for s in range(x.shape[0]):
            S = S + x[s]
            Q = Q + x[s] * x[s]
        return variance_of_sums(S, Q, np.full(x.shape[1:-1], x.shape[0], np.uint32))


def variance_of_sums(S, Q, n):
    """var_c of sums S, Q [..., 3] over n [...] samples (0 where n = 0)."""
    S, Q = np.asarray(S, F32), np.asarray(Q, F32)
    n = np.asarray(n, np.uint32)
    with np.errstate(all="ignore"):
        inv = (F32(1) / n.astype(F32))[..., None]
        mean = inv * S
        d = inv * Q - mean * mean
        var = np.where(d < 0, F32(0), d) * inv
    return np.where(n[..., None] == 0, F32(0), var).astype(F32)
