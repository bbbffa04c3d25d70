"""Moving the spheres of a resident scene (rtb200_scene_update_*) on the host side, no GPU: a numpy float64 restatement of the
refit (rtb200_refit.cu) on the topology of the uploaded scene's hierarchy. With unchanged spheres it must reproduce the host
builder's arrays bit for bit, which pins it to the builder's rounding; on moved scenes the float32 traversal emulation of
test_bvh_cpu must still reach every sphere the exact f64 test accepts (DESIGN.md §4.7). The GPU tests compare the device's
arrays with this restatement."""
import ctypes as C

import numpy as np
import pytest

import rtb200 as R
from rtb200 import scenes
from synth import base_config, mixed_config, _v
from test_bvh_cpu import SCENES, _exact_hits, _spheres, _traverse

U = 2.0 ** -24
EMPTY, LEAF = 0xFFFFFFFF, 0x80000000
INVALID = -1


def _f32_up(x):
    """rtbvh::f32_up: the smallest float32 >= x."""
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) < x, np.nextafter(f, np.float32(np.inf)), f)


def _f32_down(x):
    """rtbvh::f32_down: the largest float32 <= x."""
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(-np.inf)), f)


def sphere_records(c, r, g):
    """rtbvh::sphere_record of every sphere, float32 [n, 4] {x, y, z, nk}; a sphere outside the f32 frame is (0, 0, 0, +inf)."""
    with np.errstate(all="ignore"):
        x = c - g
        r2 = r * r
        c2 = (x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2]
        es = ((96.0 * U) * c2 + (16.0 * U) * r2) + 1e-30
        nkd = -(c2 - r2) + es
        rec = np.empty((len(r), 4), np.float32)
        rec[:, :3] = x.astype(np.float32)
        fin = np.isfinite(nkd)
        rec[:, 3] = np.where(fin, _f32_up(np.where(fin, nkd, 0.0)), np.float32(np.inf))
        ok = np.isfinite(rec[:, :3]).all(axis=1) & fin & (c2 < 1e30)
    rec[~ok] = (0.0, 0.0, 0.0, np.inf)
    return rec


def sphere_boxes(c, r, g):
    """Exact box (c - g) +- |r| of every sphere; infinite when the host builder would send it to the always-list."""
    with np.errstate(all="ignore"):
        x = c - g
        ra = np.abs(r)
        fin = np.isfinite(x).all(axis=1) & np.isfinite(ra)
        ext = np.where(fin, np.abs(np.where(fin[:, None], x, 0.0)).max(axis=1) + ra, np.inf)
        inside = (fin & (ext < 1e15))[:, None]
        return np.where(inside, x - ra[:, None], -np.inf), np.where(inside, x + ra[:, None], np.inf)


def refit(b, c, r):
    """The refit of rtb200_refit.cu for spheres (c, r) on the topology and recentring of b (bvh_records of the uploaded
    scene): the same dict with new lo / hi / leaf_rec / flat."""
    g, k = b["recentre"], b["leaf_size"]
    rec, (slo, shi) = sphere_records(c, r, g), sphere_boxes(c, r, g)
    out = dict(b)
    n = len(r)
    flat = b["flat"].copy().reshape(-1, 8)
    i = np.arange(n); pp, kk = i // 2, i % 2
    for q in range(4):
        flat[pp, 2 * q + kk] = rec[:, q]
    out["flat"] = flat.reshape(b["flat"].shape)
    nl = b["n_leaves"]
    lr = b["leaf_rec"].copy().reshape(nl, k // 2, 8)
    leaf, slot = np.nonzero(b["leaf_id"] != EMPTY)
    ids = b["leaf_id"][leaf, slot].astype(np.int64)
    for q in range(4):
        lr[leaf, slot // 2, 2 * q + slot % 2] = rec[ids, q]
    out["leaf_rec"] = lr.reshape(b["leaf_rec"].shape)
    llo = np.full((nl, 3), np.inf); lhi = np.full((nl, 3), -np.inf)
    np.minimum.at(llo, leaf, slo[ids]); np.maximum.at(lhi, leaf, shi[ids])
    nn = b["n_nodes"]
    nlo = np.full((nn, 3), np.inf); nhi = np.full((nn, 3), -np.inf)
    lo, hi = b["lo"].copy(), b["hi"].copy()
    for node in range(nn - 1, -1, -1):          # children have larger indices than their parent
        for s, ref in enumerate(b["child"][node]):
            if ref == EMPTY:
                continue
            if ref & LEAF:
                blo, bhi = llo[ref & 0x7FFFFFFF], lhi[ref & 0x7FFFFFFF]
            else:
                assert ref > node
                blo, bhi = nlo[ref], nhi[ref]
            bmax = max(np.abs(blo).max(), np.abs(bhi).max())
            m = (32.0 * U) * bmax + 1e-30
            with np.errstate(all="ignore"):
                lo[node][:, s] = _f32_down(blo - m); hi[node][:, s] = _f32_up(bhi + m)
            nlo[node] = np.minimum(nlo[node], blo); nhi[node] = np.maximum(nhi[node], bhi)
    out["lo"], out["hi"] = lo, hi
    return out


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _degenerate():
    objs = [{"center": _v(0.1 * i, 0, 0), "radius": 0.5, "material": {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}} for i in range(30)]
    objs += [{"center": _v(1, 0, 0), "radius": 0.0, "material": {"Glass": {"index_of_refraction": 1.5}}},
             {"center": _v(2, 0, 0), "radius": -0.4, "material": {"Glass": {"index_of_refraction": 1.5}}},
             {"center": _v(float("inf"), 0, 0), "radius": 1.0, "material": {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}},
             {"center": _v(1e20, 0, 0), "radius": 1.0, "material": {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}}]
    return R.Scene.from_config(base_config(8, 6, 1, 2, objs))


@pytest.mark.parametrize("mk", SCENES + [_degenerate])
def test_refit_of_the_uploaded_spheres_is_the_host_build(mk):
    sc = mk()
    b = R.bvh_records(sc)
    c, r = _spheres(sc)
    f = refit(b, c, r)
    for key in ("lo", "hi", "leaf_rec", "flat"):
        assert same_bits(f[key], b[key]), key


def _moved(sc, how, rng):
    c, r = _spheres(sc)
    c, r = c.copy(), r.copy()
    if how == "jitter":
        c += rng.normal(size=c.shape) * 0.3
    elif how == "permuted":                     # every leaf now spans the scene: the worst tree
        c = c[rng.permutation(len(r))]
    elif how == "far":
        c += np.array([1.0e6, -2.0e5, 1.0e6])
    elif how == "out_of_frame":
        k = len(r)
        c[1] = (1e16, 0.0, 0.0); c[2] = (np.inf, 0.0, 0.0); c[3] = (0.0, np.nan, 0.0); r[4] = np.nan; r[5] = np.inf
        c[6] = (1e15, 1.0, 1.0)
        r[7:k:5] = -r[7:k:5]; r[9:k:7] = 0.0
        c[8:k:3] += rng.normal(size=c[8:k:3].shape) * 0.2
    return c, r


def _rays(c, r, cam, rng, count):
    """Primary rays from the camera towards a sphere and rays leaving a sphere's surface (finite, in-frame spheres only)."""
    ok = np.nonzero(np.isfinite(c).all(axis=1) & np.isfinite(r) & (np.abs(c).max(axis=1) < 1e14))[0]
    for i in range(count):
        j = int(ok[rng.integers(len(ok))])
        if i % 3 == 0:
            o = cam
            d = (c[j] + rng.normal(size=3) * abs(r[j]) * 0.7) - o
        else:
            nrm = rng.normal(size=3); nrm /= np.linalg.norm(nrm)
            o = c[j] + nrm * abs(r[j])
            d = nrm + rng.normal(size=3) * 0.8
            if i % 7 == 1:
                d = d * np.array([1.0, 1e-9, 1.0])
        if not np.any(d):
            d = np.array([0.0, 0.0, 1.0])
        yield o, d * float(rng.uniform(0.2, 5.0))


@pytest.mark.parametrize("how", ["jitter", "permuted", "far", "out_of_frame"])
@pytest.mark.parametrize("mk", [SCENES[0], SCENES[1], SCENES[3]])
def test_traversal_of_refit_records_never_drops_a_sphere_the_exact_test_accepts(mk, how):
    sc = mk()
    b = R.bvh_records(sc)
    rng = np.random.default_rng(5)
    c, r = _moved(sc, how, rng)
    f = refit(b, c, r)
    cam = np.array([sc.c.camera.origin.x, sc.c.camera.origin.y, sc.c.camera.origin.z])
    n_exact = 0
    for i, (o, d) in enumerate(_rays(c, r, cam, rng, 240)):
        with np.errstate(all="ignore"):
            exact = _exact_hits(c, r, o, d)
        cand, _ = _traverse(f, o, d)
        missing = set(exact.tolist()) - cand
        assert not missing, (i, sorted(missing))
        n_exact += len(exact)
    assert n_exact > 100
    if how == "out_of_frame":   # spheres that left the f32 frame are candidates of every ray, like always-list spheres
        o, d = cam, -cam
        cand, _ = _traverse(f, o, d)
        assert {1, 2, 3, 4, 5} <= cand


def test_out_of_frame_members_get_infinite_boxes():
    sc = R.Scene.from_config(mixed_config(16, 12, 1, 2, seed=1, n=20))
    b = R.bvh_records(sc)
    c, r = _spheres(sc)
    c = c.copy(); c[4] = (np.nan, 0.0, 0.0)
    f = refit(b, c, r)
    leaf = int(np.nonzero((b["leaf_id"] == 4).any(axis=1))[0][0])
    node, slot = [(int(n), int(s)) for n, s in zip(*np.nonzero(b["child"] == (LEAF | leaf)))][0]
    assert np.all(f["lo"][node][:, slot] == -np.inf) and np.all(f["hi"][node][:, slot] == np.inf)
    assert np.all(f["lo"][0] <= b["lo"][0])   # the infinite box reaches the root
    assert np.any(f["lo"][0] == -np.inf)


def test_set_sphere_edits_the_host_scene():
    sc = scenes.cover_scene(16, 12, 1)
    old = R.rt_sphere.from_buffer_copy(sc._spheres[3])
    s = sc.set_sphere(3, center=[1.0, 2.0, 3.0], radius=0.25, material={"Metal": {"albedo": [0.1, 0.2, 0.3], "fuzz": 0.5}})
    assert (s.center.x, s.center.y, s.center.z, s.radius, s.kind, s.param, s.texture) == (1.0, 2.0, 3.0, 0.25, R.RT_METAL, 0.5, -1)
    assert list(s.albedo) == [np.float32(0.1), np.float32(0.2), np.float32(0.3)]
    assert bytes(sc._spheres[3]) == bytes(s)                               # the scene holds the edit; s is a copy
    s.radius = 9.0
    assert sc._spheres[3].radius == 0.25
    sc.set_sphere(3, material=old)                                         # material copied from a record; geometry stays
    assert sc._spheres[3].kind == old.kind and sc._spheres[3].radius == 0.25
    with pytest.raises(IndexError):
        sc.set_sphere(sc.n_spheres, radius=1.0)


def test_argument_errors_need_no_device():
    L = R.lib()
    sp = (R.rt_sphere * 1)()
    idx = (C.c_uint32 * 1)(0)
    assert L.rtb200_scene_update_spheres(None, idx, sp, 1, None) == INVALID
    assert b"null scene handle" in L.rtb200_last_error()
    assert L.rtb200_scene_update_spheres(None, None, sp, 1, None) == INVALID
    assert b"index or spheres is null" in L.rtb200_last_error()
    assert L.rtb200_scene_update_spheres(None, idx, None, 1, None) == INVALID
    assert b"index or spheres is null" in L.rtb200_last_error()
    assert L.rtb200_scene_update_spheres(None, None, None, 0, None) == INVALID      # n == 0 still needs a handle
    assert L.rtb200_scene_update_geometry_device(None, None, None) == INVALID
    assert b"is null" in L.rtb200_last_error()
    info = (C.c_uint32 * 8)()
    assert L.rtb200_scene_debug_records(None, info, None, 0, None, 0, None, 0, None, 0) == INVALID
