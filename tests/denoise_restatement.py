"""The denoise contract of include/rtb200.h (rtb200_denoise[_device], DESIGN.md §4.15) restated twice in float32 numpy, which
rounds every operation and never fuses two: `denoise` vectorised over the image, one tap at a time, and `denoise_scalar` with
per-pixel Python loops over np.float32 scalars. The CPU tests hold the two equal bit for bit; the GPU tests hold the kernel to
`denoise`."""
import numpy as np

F32 = np.float32
B = (F32(1 / 16), F32(1 / 4), F32(3 / 8), F32(1 / 4), F32(1 / 16))   # every B[i] * B[j] is exact in f32
TAPS = [(dx, dy) for dy in range(-2, 3) for dx in range(-2, 3)]


def _guides(albedo, normal, albedo_weight, normal_weight):
    """The guides that were given (they take part in the finite test) and those that are on (they weigh the taps)."""
    given = [g for g in (albedo, normal) if g is not None]
    on = [(np.asarray(g, F32), F32(lam)) for g, lam in ((albedo, albedo_weight), (normal, normal_weight)) if g is not None and lam != 0]
    return [np.asarray(g, F32) for g in given], on


def check(color, albedo, normal, iterations, color_weight, albedo_weight, normal_weight):
    """The host's refusals of the parameters, as ValueError."""
    if not 1 <= iterations <= 10:
        raise ValueError("iterations must be in [1, 10]")
    for name, lam in (("color", color_weight), ("albedo", albedo_weight), ("normal", normal_weight)):
        lam = F32(lam)
        if not np.isfinite(lam) or lam < 0:
            raise ValueError(f"{name}_weight must be finite and >= 0")
    with np.errstate(over="ignore"):
        if not np.isfinite(F32(color_weight) * F32(4.0 ** (iterations - 1))):
            raise ValueError("color_weight * 4^(iterations - 1) overflows")
    if (albedo is None and albedo_weight != 0) or (normal is None and normal_weight != 0):
        raise ValueError("a nonzero weight for an absent guide")


def denoise(color, albedo=None, normal=None, *, iterations, color_weight, albedo_weight=0.0, normal_weight=0.0):
    """The filtered image, [h, w, 3] float32, vectorised: for each tap every pixel's num and den take one step."""
    check(color, albedo, normal, iterations, color_weight, albedo_weight, normal_weight)
    c = np.array(color, F32, copy=True)
    h, w, _ = c.shape
    given, on = _guides(albedo, normal, albedo_weight, normal_weight)
    guides_ok = np.ones((h, w), bool)
    for g in given:
        guides_ok &= np.isfinite(g).all(axis=2)
    lam_c0 = F32(color_weight)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        for i in range(iterations):
            step = 1 << i
            lam_c = lam_c0 * F32(4 ** i)
            ok = guides_ok & np.isfinite(c).all(axis=2)
            num = np.zeros((h, w, 3), F32)
            den = np.zeros((h, w), F32)
            for dx, dy in TAPS:
                ox, oy = dx * step, dy * step
                # q = p + (ox, oy): the source window of q and the destination window of p, both inside the image
                ys, yd = slice(max(oy, 0), h + min(oy, 0)), slice(max(-oy, 0), h + min(-oy, 0))
                xs, xd = slice(max(ox, 0), w + min(ox, 0)), slice(max(-ox, 0), w + min(-ox, 0))
                if ys.start >= ys.stop or xs.start >= xs.stop:
                    continue
                valid = ok[yd, xd] & ok[ys, xs]
                f = None
                for lam, g in ([(lam_c, c)] if lam_c != 0 else []) + [(l, g) for g, l in on]:
                    e = g[ys, xs] - g[yd, xd]
                    d = (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]
                    fac = F32(1) + lam * d
                    f = fac if f is None else f * fac
                k = B[dx + 2] * B[dy + 2]
                wt = np.full(valid.shape, k, F32) if f is None else k / f
                cq = c[ys, xs]
                num[yd, xd] = np.where(valid[..., None], num[yd, xd] + wt[..., None] * cq, num[yd, xd])
                den[yd, xd] = np.where(valid, den[yd, xd] + wt, den[yd, xd])
            out = num / np.where(ok, den, F32(1))[..., None]
            c = np.where(ok[..., None], out, c).astype(F32)
    return c


def denoise_scalar(color, albedo=None, normal=None, *, iterations, color_weight, albedo_weight=0.0, normal_weight=0.0):
    """The same contract pixel by pixel and tap by tap over np.float32 scalars, as the issue of the contract states it."""
    check(color, albedo, normal, iterations, color_weight, albedo_weight, normal_weight)
    c = np.array(color, F32, copy=True)
    h, w, _ = c.shape
    given, on = _guides(albedo, normal, albedo_weight, normal_weight)

    def finite(img, y, x):
        if not all(np.isfinite(img[y, x, k]) for k in range(3)):
            return False
        return all(np.isfinite(g[y, x, k]) for g in given for k in range(3))

    def dist(img, y, x, py, px):
        e = [img[y, x, k] - img[py, px, k] for k in range(3)]
        return (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]

    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        for i in range(iterations):
            step = 1 << i
            lam_c = F32(color_weight) * F32(4 ** i)
            nxt = c.copy()
            for py in range(h):
                for px in range(w):
                    if not finite(c, py, px):
                        continue
                    num = [F32(0), F32(0), F32(0)]
                    den = F32(0)
                    for dy in range(-2, 3):
                        for dx in range(-2, 3):
                            qy, qx = py + step * dy, px + step * dx
                            if not (0 <= qy < h and 0 <= qx < w) or not finite(c, qy, qx):
                                continue
                            f = None
                            if lam_c != 0:
                                f = F32(1) + lam_c * dist(c, qy, qx, py, px)
                            for g, lam in on:
                                fac = F32(1) + lam * dist(g, qy, qx, py, px)
                                f = fac if f is None else f * fac
                            k = B[dx + 2] * B[dy + 2]
                            wt = k if f is None else k / f
                            for ch in range(3):
                                num[ch] = num[ch] + wt * c[qy, qx, ch]
                            den = den + wt
                    for ch in range(3):
                        nxt[py, px, ch] = num[ch] / den
            c = nxt
    return c


def quantise(linear):
    """The render's RGB8 of a linear image: sqrt, then min(x * 255, 255) + 2^23 and its low mantissa bits (rtb200_probe_quantise)."""
    x = np.asarray(linear, F32)
    with np.errstate(invalid="ignore"):
        s = np.sqrt(x).astype(F32)
        scaled = np.fmin(s * F32(255), F32(255)).astype(F32)
    bits = (scaled + F32(8388608)).astype(F32).view(np.uint32)
    return np.where(bits >= 0x4B000000, bits - 0x4B000000, 0).astype(np.uint8)
