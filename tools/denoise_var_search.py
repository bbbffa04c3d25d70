"""The CPU grid search behind the variance-guided denoise's defaults (DESIGN.md §4.18): the oracle's cover render at 64x48 from
its per-sample radiances at 2, 4, 8, 16 and 32 spp under two seeds, each spp's variance (the render's formula) and oracle AOV
guides, filtered by the float32 restatement (tests/denoise_var_restatement.py) over a grid of parameters and scored as MSE
against the oracle's 256-spp render of the view. Prints every row and the best; a second edge-stopping form, the squared
rational 1 / (1 + (lc * d_c / (eps + vbar))^2), is scored beside it.

    python tools/denoise_var_search.py [--max-spp 32] [--seeds 2]
"""
import argparse
import itertools
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(REPO, "tests"), os.path.join(REPO, "oracle"), os.path.join(REPO, "rust-raytracer_b200")]

import adaptive_restatement as AR  # noqa: E402
import denoise_restatement as DR  # noqa: E402
import denoise_var_restatement as V  # noqa: E402
import oracle_aov as OA  # noqa: E402
import oracle_py  # noqa: E402
import rtb200 as R  # noqa: E402
from rtb200 import scenes  # noqa: E402

SPPS = (2, 4, 8, 16, 32)
SEED2 = 0x5EED0002


def mse(a, b):
    return float(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))


def inputs(max_spp=32, seeds=2):
    """{(seed index, spp): (mean, variance, albedo, normal)} and the 256-spp truth."""
    truth = oracle_py.render(scenes.cover_scene(64, 48, 256), rgb8=False)[0].reshape(48, 64, 3)
    out = {}
    for si in range(seeds):
        sc = scenes.cover_scene(64, 48, max_spp)
        if si:
            sc.seed = SEED2
        x, _ = AR.render_samples(sc, 0, max_spp)
        for spp in (s for s in SPPS if s <= max_spp):
            mean = render_mean(x[:spp])
            aov = OA.aov(sc, spp, 0)
            out[si, spp] = (mean, V.render_variance(x[:spp]), aov["albedo"], aov["normal"])
    return out, truth


def render_mean(x):
    """The render's linear mean: (1 / n) * the f32 sum in sample order."""
    S = np.zeros(x.shape[1:], np.float32)
    for s in range(x.shape[0]):
        S = S + x[s]
    return np.float32(1) / np.float32(x.shape[0]) * S


def squared(color, variance, albedo, normal, *, iterations, color_weight, albedo_weight, normal_weight, variance_floor):
    """The squared rational form: the colour factor 1 + (lc * d_c / (eps + vbar))^2, in float32 numpy (not the contract)."""
    c, var = np.array(color, np.float32), np.array(variance, np.float32)
    h, w, _ = c.shape
    with np.errstate(all="ignore"):
        for i in range(iterations):
            step = 1 << i
            v = (var[..., 0] + var[..., 1]) + var[..., 2]
            pad = np.pad(v, 1, mode="edge")
            g = np.array([0.25, 0.5, 0.25], np.float32)
            vbar = sum(g[dy] * g[dx] * pad[dy:dy + h, dx:dx + w] for dy in range(3) for dx in range(3))
            num, den, nv = np.zeros_like(c), np.zeros((h, w), np.float32), np.zeros_like(c)
            for dx, dy in V.TAPS:
                win = V._window(dx * step, dy * step, h, w)
                if win is None:
                    continue
                ys, xs, yd, xd = win
                r = np.float32(color_weight) * (V._dist(c[ys, xs] - c[yd, xd]) / (np.float32(variance_floor) + vbar[yd, xd]))
                f = (1 + r * r) * (1 + np.float32(albedo_weight) * V._dist(albedo[ys, xs] - albedo[yd, xd])) \
                    * (1 + np.float32(normal_weight) * V._dist(normal[ys, xs] - normal[yd, xd]))
                wt = V.B[dx + 2] * V.B[dy + 2] / f
                num[yd, xd] += wt[..., None] * c[ys, xs]
                den[yd, xd] += wt
                nv[yd, xd] += (wt * wt)[..., None] * var[ys, xs]
            c, var = num / den[..., None], nv / (den * den)[..., None]
    return c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-spp", type=int, default=32)
    ap.add_argument("--seeds", type=int, default=2)
    a = ap.parse_args()
    data, truth = inputs(a.max_spp, a.seeds)
    spps = sorted({k[1] for k in data})
    raw = {k: mse(d[0], truth) for k, d in data.items()}
    old = {k: mse(DR.denoise(d[0], d[2], d[3], iterations=R.DENOISE_ITERATIONS, color_weight=R.DENOISE_COLOR_WEIGHT,
                             albedo_weight=R.DENOISE_ALBEDO_WEIGHT, normal_weight=R.DENOISE_NORMAL_WEIGHT), truth)
           for k, d in data.items()}
    print("spp: " + " ".join(f"{s:>9}" for s in spps) + "   (mean over seeds)")
    print("raw: " + " ".join(f"{np.mean([raw[si, s] for si in range(a.seeds)]):9.6f}" for s in spps))
    print("old: " + " ".join(f"{np.mean([old[si, s] for si in range(a.seeds)]):9.6f}" for s in spps))
    rows = []
    for form, fn in (("rational", V.denoise_var), ("squared", squared)):
        for L, lc, la, ln, eps in itertools.product((2, 3, 4), (0.5, 1.0, 2.0), (4.0,), (1.0,), (1e-5, 1e-4, 1e-3)):
            kw = dict(iterations=L, color_weight=lc, albedo_weight=la, normal_weight=ln, variance_floor=eps)
            m = {k: mse(fn(d[0], d[1], d[2], d[3], **kw) if fn is squared else fn(*d, **kw)[0], truth) for k, d in data.items()}
            # the score: the mean over every spp and seed of log(MSE / raw MSE)
            score = float(np.mean([np.log(m[k] / raw[k]) for k in data]))
            rows.append((score, form, kw, {s: np.mean([m[si, s] for si in range(a.seeds)]) for s in spps}))
    rows.sort(key=lambda r: r[0])
    for score, form, kw, m in rows[:25]:
        print(f"{score:+.4f} {form:8s} L={kw['iterations']} lc={kw['color_weight']} la={kw['albedo_weight']} "
              f"ln={kw['normal_weight']} eps={kw['variance_floor']:g}: " + " ".join(f"{m[s]:9.6f}" for s in spps))


if __name__ == "__main__":
    main()
