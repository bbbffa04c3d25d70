"""The launch geometry of both à-trous step kernels without a GPU (rt_denoise_step_kernel, rt_denoise_var_step_kernel; AtrousTiles
in csrc/rtb200_kernels.cuh, DESIGN.md §4.15), restated in Python: the 1-D grid of one step and the decode of a CTA's index into
its tile and residue class. Held to cover every pixel exactly once per iteration on every image up to 70 x 70 at every
iteration count, and to launch at most width * height <= 2^31 - 1 CTAs over the filters' whole domain, where the grid of every
h * h residue class exceeded gridDim.x's limit on long, thin images."""
import os
import re

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "rust-raytracer_b200", "csrc")
GRID_MAX = 2**31 - 1   # gridDim.x
NPIX_MAX = 2**31 - 1   # the filters accept width * height < 2^31


def _tile(src, bx, by):
    with open(os.path.join(CSRC, src)) as f:
        m = re.search(rf"constexpr int {bx} = (\d+), {by} = (\d+);", f.read())
    return int(m.group(1)), int(m.group(2))


# the CTA tile of each step kernel, read from its source so that the model cannot drift from it
TILES = {"denoise": _tile("rtb200_denoise.cu", "kDenoiseBX", "kDenoiseBY"),
         "denoise_var": _tile("rtb200_denoise_var.cu", "kVarBX", "kVarBY")}

# (width, height, iterations): the first shapes at which the grid of all h * h residue classes passed 2^31 - 1 in some iteration;
# one pixel fewer on the long side stayed under it
OVERFLOWED = [(1, 33_550_337, 10), (4, 33_550_337, 10), (134_201_345, 1, 10), (1, 67_106_817, 9), (1, 134_216_705, 8)]


def one_shorter(w, h):
    return (w, h - 1) if h > w else (w - 1, h)


def geometry(w, h, step, bx, by):
    """AtrousTiles: (tiles_x, tiles_y, res_x, res_y) of step `step` on a w x h image."""
    return (-(-(-(-w // step)) // bx), -(-(-(-h // step)) // by), min(step, w), min(step, h))


def grid(w, h, step, bx, by):
    tx, ty, rx, ry = geometry(w, h, step, bx, by)
    return tx * ty * rx * ry


def grid_every_class(w, h, step, bx, by):
    """The grid before only the residue classes that hold a pixel were launched: every one of the step * step."""
    tx, ty, _, _ = geometry(w, h, step, bx, by)
    return tx * ty * step * step


def decode(b, w, h, step, bx, by):
    """CTA index b (an array) -> (tile x, tile y, rx, ry), as AtrousTiles::decode does it in uint32 arithmetic."""
    tx, ty, rx_n, _ = geometry(w, h, step, bx, by)
    b = np.asarray(b, np.uint64)
    tix = b % tx; b = b // tx
    tiy = b % ty; b = b // ty
    return tix, tiy, b % rx_n, b // rx_n


def axis_hits(n, tiles, res, block, step):
    """How often each coordinate in [0, n) is the pixel of a thread of the kernel along one axis: residue r, tile t and lane
    l give r + (t * block + l) * step, and a thread past the image's edge writes nothing."""
    r, t, l = np.meshgrid(np.arange(res), np.arange(tiles), np.arange(block), indexing="ij")
    x = (r + (t * block + l) * step).ravel()
    return np.bincount(x[x < n], minlength=n)


def test_the_model_reads_both_kernels_tiles():
    assert TILES["denoise"] == (32, 8) and TILES["denoise_var"] == (32, 8)


@pytest.mark.parametrize("kernel", list(TILES))
def test_every_pixel_is_written_once_per_iteration_up_to_70x70(kernel):
    """For every w, h <= 70 and every step of L <= 10: the decode maps [0, grid) one to one onto tiles x residue classes (so a
    CTA's pixels are the product of its x and y lanes'), and along each axis the lanes of the launched tiles and classes hit
    every coordinate exactly once. Together: every pixel exactly once."""
    bx, by = TILES[kernel]
    for step in (1 << i for i in range(10)):
        hits_x = {w: axis_hits(w, *geometry(w, 1, step, bx, by)[::2], bx, step) for w in range(1, 71)}
        hits_y = {h: axis_hits(h, geometry(1, h, step, bx, by)[1], geometry(1, h, step, bx, by)[3], by, step) for h in range(1, 71)}
        for n in range(1, 71):
            assert (hits_x[n] == 1).all(), (kernel, step, "x", n, np.flatnonzero(hits_x[n] != 1)[:8])
            assert (hits_y[n] == 1).all(), (kernel, step, "y", n, np.flatnonzero(hits_y[n] != 1)[:8])
        for w in range(1, 71):
            for h in range(1, 71):
                g = geometry(w, h, step, bx, by)
                tix, tiy, rx, ry = decode(np.arange(grid(w, h, step, bx, by)), w, h, step, bx, by)
                assert (tix < g[0]).all() and (tiy < g[1]).all() and (rx < g[2]).all() and (ry < g[3]).all(), (w, h, step)
                key = ((ry * g[2] + rx) * g[1] + tiy) * g[0] + tix
                assert np.array_equal(np.sort(key), np.arange(g[0] * g[1] * g[2] * g[3], dtype=np.uint64)), (w, h, step)


@pytest.mark.parametrize("kernel", list(TILES))
def test_every_pixel_is_written_once_by_whole_threads_on_small_images(kernel):
    """The same without the product argument: every thread of every launched CTA, its pixel in 2-D, on images up to 24 x 24."""
    bx, by = TILES[kernel]
    lx, ly = np.meshgrid(np.arange(bx), np.arange(by))
    for w in range(1, 25):
        for h in range(1, 25):
            for step in (1 << i for i in range(10)):
                tix, tiy, rx, ry = (a.astype(np.int64)[:, None, None] for a in
                                    decode(np.arange(grid(w, h, step, bx, by)), w, h, step, bx, by))
                x = (rx + (tix * bx + lx) * step).ravel()
                y = (ry + (tiy * by + ly) * step).ravel()
                keep = (x < w) & (y < h)
                hits = np.bincount(y[keep] * w + x[keep], minlength=w * h)
                assert (hits == 1).all(), (kernel, w, h, step, np.flatnonzero(hits != 1)[:8])


def _domain():
    """Shapes over the filters' domain: the rows and columns at the overflow thresholds and one shorter, width * height just
    under 2^31 at several aspect ratios, and powers of two +- 1 on either side."""
    shapes = set()
    for w, h, _ in OVERFLOWED:
        for a, b in ((w, h), one_shorter(w, h)):
            shapes |= {(a, b), (b, a)}
    for n in (1, 2, 3, 4, 7, 8, 9, 31, 32, 33, 299, 511, 512, 513, 1080, 1920, 46340, 46341, 65535, 65536):
        shapes |= {(n, NPIX_MAX // n), (NPIX_MAX // n, n)}
    for k in range(32):
        for d in (-1, 0, 1):
            n = (1 << k) + d
            if n < 1:
                continue
            for m in (1, 2, 3, 8, 33, 600, 1080):
                if n * m <= NPIX_MAX:
                    shapes |= {(n, m), (m, n)}
            if n <= NPIX_MAX:
                shapes |= {(n, NPIX_MAX // n), (NPIX_MAX // n, n)}
    return sorted(shapes)


@pytest.mark.parametrize("kernel", list(TILES))
def test_the_grid_stays_under_the_limit_over_the_domain(kernel):
    bx, by = TILES[kernel]
    shapes = _domain()
    assert len(shapes) > 500
    for w, h in shapes:
        assert 1 <= w * h <= NPIX_MAX, (w, h)
        for step in (1 << i for i in range(10)):
            g = grid(w, h, step, bx, by)
            assert 1 <= g <= w * h and g <= GRID_MAX, (kernel, w, h, step, g)


@pytest.mark.parametrize("kernel", list(TILES))
@pytest.mark.parametrize("block", ["x", "y"])
def test_each_axis_factor_is_at_most_its_length(kernel, block):
    """grid = (tiles_x * res_x) * (tiles_y * res_y), and each factor is at most the axis's length n (DESIGN.md §4.15): every n
    up to 2^20 and every n within 2^12 of a power of two up to 2^31, at every step."""
    b = TILES[kernel][0 if block == "x" else 1]
    n = np.unique(np.concatenate([np.arange(1, 1 << 20)] + [np.arange(max(1, (1 << k) - 4096), min(NPIX_MAX, (1 << k) + 4096) + 1)
                                                           for k in range(20, 32)])).astype(np.int64)
    for step in (1 << i for i in range(10)):
        factor = -(-(-(-n // step)) // b) * np.minimum(step, n)
        assert (factor <= n).all(), (kernel, block, step, n[factor > n][:8])


@pytest.mark.parametrize("kernel", list(TILES))
def test_the_grid_is_unchanged_where_the_step_fits_the_image(kernel):
    """Where h <= min(w, h) every residue class holds a pixel and the grid is the one of all h * h classes; among them 800x600
    and 1920x1080 at every iteration count."""
    bx, by = TILES[kernel]
    seen = 0
    for w, h in _domain() + [(800, 600), (1920, 1080), (401, 300), (65, 33)] + [(w, h) for w in range(1, 71) for h in range(1, 71)]:
        for step in (1 << i for i in range(10)):
            if step <= min(w, h):
                assert grid(w, h, step, bx, by) == grid_every_class(w, h, step, bx, by), (w, h, step)
                seen += 1
    assert seen > 5000
    for w, h in ((800, 600), (1920, 1080)):
        assert all(1 << i <= min(w, h) for i in range(10))


@pytest.mark.parametrize("kernel", list(TILES))
def test_the_overflowing_shapes(kernel):
    """The grid of every class passed 2^31 - 1 at the table's shapes and not one pixel shorter; the grid of the classes that hold a
    pixel stays under w * h at both."""
    bx, by = TILES[kernel]
    for w, h, L in OVERFLOWED:
        steps = [1 << i for i in range(L)]
        assert w * h <= NPIX_MAX
        assert max(grid_every_class(w, h, s, bx, by) for s in steps) > GRID_MAX, (w, h, L)
        assert max(grid_every_class(*one_shorter(w, h), s, bx, by) for s in steps) <= GRID_MAX, (w, h, L)
        for a, b in ((w, h), one_shorter(w, h)):
            assert max(grid(a, b, s, bx, by) for s in steps) <= min(a * b, GRID_MAX)
