"""Adaptive rendering restated in numpy float32 from per-sample radiances of the CPU oracle (render_samples, one call of the
oracle's per-sample routine oracle_sample per pixel and sample), independently of the CUDA code (rtb200_adaptive.cu,
DESIGN.md §4.9).

The rule (include/rtb200.h): every pixel still on the list traces samples [n, min(n + m, N)) per round and adds them to its
f32 sums S_c and Q_c (of x_c * x_c) in sample order; then, with inv = 1/n, mean_c = inv*S_c, var_c = inv*Q_c - mean_c^2,
err_c = sqrt(max(var_c, 0)*inv) and tol_c = abs_tol + rel_tol*mean_c, it leaves the list if n == N, or if n >= min_samples,
every S_c and Q_c is finite and err_c <= tol_c in all three channels. numpy's float32 operations round to nearest and are never
fused, as the kernel's __f*_rn are."""
import ctypes as C

import numpy as np

import oracle_py as O

F = np.float32
_sample = None


def render_samples(scene, s0, s1):
    """Samples [s0, s1) of every pixel, each alone, by the oracle's oracle_sample (the routine oracle_render runs per sample
    and sums in sample order). Returns (float32 radiance [s1-s0, h, w, 3], uint32 rays [s1-s0, h, w])."""
    global _sample
    if _sample is None:
        O.lib()   # builds liboracle.so when it is missing or stale
        fn = C.CDLL(O.LIB_PATH).oracle_sample   # a function object of our own: it takes raw addresses into numpy arrays
        fn.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        fn.restype = C.c_int
        _sample = fn
    h, w = int(scene.c.height), int(scene.c.width)
    out = np.zeros((s1 - s0, h, w, 3), dtype=F)
    rays = np.zeros((s1 - s0, h, w), dtype=np.uint64)
    sc = C.addressof(scene.c)
    o0, r0 = out.ctypes.data, rays.ctypes.data
    for k, s in enumerate(range(s0, s1)):
        for y in range(h):
            for x in range(w):
                i = (k * h + y) * w + x
                _sample(sc, x, y, s, o0 + 12 * i, r0 + 8 * i, None)
    return out, rays.astype(np.uint32)


def leaves(n, S, Q, N, min_samples, abs_tol, rel_tol):
    """The stopping rule for pixels with n samples and sums S, Q ([..., 3] float32): True where the pixel leaves the list."""
    n = np.asarray(n, dtype=np.uint32)
    S = np.asarray(S, dtype=F); Q = np.asarray(Q, dtype=F)
    with np.errstate(all="ignore"):
        inv = (F(1.0) / n.astype(F))[..., None]
        mean = inv * S
        var = inv * Q - mean * mean
        err = np.sqrt(np.where(var > F(0.0), var, F(0.0)) * inv)
        tol = F(abs_tol) + F(rel_tol) * mean
        ok = np.isfinite(S).all(-1) & np.isfinite(Q).all(-1) & (err <= tol).all(-1)
    return (n >= N) | ((n >= min_samples) & ok)


def quantise(mean):
    """RGB8 of linear means: the one-shot render's quantisation, as the oracle computes it (oracle_quantise)."""
    mean = np.ascontiguousarray(mean, dtype=F)
    out = np.zeros(mean.shape, dtype=np.uint8)
    O.lib().oracle_quantise(mean.ctypes.data, mean.size, out.ctypes.data)
    return out


def resolve(n, S):
    """linear and RGB8 of pixels with n samples and sums S; a pixel with n == 0 is 0."""
    with np.errstate(all="ignore"):
        inv = F(1.0) / np.maximum(n, 1).astype(F)
        mean = np.where((n > 0)[..., None], inv[..., None] * S, F(0.0)).astype(F)
    return mean, quantise(mean)


def run(samples, rays, m, N, min_samples, abs_tol, rel_tol, rounds=None):
    """Adaptive render of the per-sample radiances samples[s] ([>= N, h, w, 3] float32) with rays[s] ([>= N, h, w]).
    `rounds`: stop after that many rounds (None: until no pixel is active). Returns a dict: counts [h, w] (uint32), S, Q,
    linear, rgb8, rays (the rays of every sample taken), samples (taken), active (pixels still on the list), rounds (run),
    and per round run: list_sizes (the pixels on its list), list_runs (the runs of consecutive pixels, in raster order, that
    its list is made of) and list_samples (the samples it took of each of them)."""
    h, w = samples.shape[1:3]
    n = np.zeros((h, w), dtype=np.uint32)
    S = np.zeros((h, w, 3), dtype=F); Q = np.zeros((h, w, 3), dtype=F)
    active = np.ones((h, w), dtype=bool)
    taken_rays = 0
    r = 0
    sizes, runs, counts = [], [], []
    with np.errstate(all="ignore"):
        while active.any() and (rounds is None or r < rounds):
            listed = np.flatnonzero(active)
            sizes.append(len(listed))
            runs.append(1 + int((np.diff(listed) != 1).sum()))
            s0 = int(n[active][0])
            assert (n[active] == s0).all(), "every listed pixel has the same n"
            s1 = min(s0 + m, N)
            counts.append(s1 - s0)
            for s in range(s0, s1):
                x = samples[s][active]
                S[active] = S[active] + x
                Q[active] = Q[active] + x * x
                taken_rays += int(rays[s][active].astype(np.uint64).sum())
            n[active] = s1
            active &= ~leaves(n, S, Q, N, min_samples, abs_tol, rel_tol)
            r += 1
    lin, img = resolve(n, S)
    return {"counts": n, "S": S, "Q": Q, "linear": lin, "rgb8": img, "rays": taken_rays, "samples": int(n.astype(np.uint64).sum()),
            "active": int(active.sum()), "rounds": r, "list_sizes": sizes, "list_runs": runs, "list_samples": counts}


def of_scene(scene, params, N=None, rounds=None):
    """run() on the oracle's per-sample radiances of `scene` with rt_adaptive_params `params` (N: the resolved max_samples)."""
    N = N or params.max_samples or scene.c.samples_per_pixel
    x, rays = render_samples(scene, 0, N)
    return run(x, rays, params.samples_per_round, N, params.min_samples, params.abs_tol, params.rel_tol, rounds)
