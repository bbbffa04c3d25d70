"""Inserting and removing spheres of a resident scene without a GPU (rtb200_scene_edit_spheres, DESIGN.md §4.13): the export
and its signature in a C program compiled from the header, the refusals that come before the handle is used, make_sphere, and
Scene.edited, which the GPU tests upload fresh and hand to the oracle, against an independent restatement of the index rule:
a kept old sphere i lands at kept(< i) + #{k : at[k] <= i} and insert k at kept(< at[k]) + k."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import rtb200 as R
from synth import base_config, mixed_config


def test_the_entry_point_is_exported():
    assert "rtb200_scene_edit_spheres" in R.ABI_SYMBOLS
    assert getattr(R.lib(), "rtb200_scene_edit_spheres") is not None


def test_the_signature_matches_the_header(repo, tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "sig.c"
    src.write_text('#include "rtb200.h"\n'
                   '_Static_assert(RTB200_ABI_VERSION == 2, "the ABI version stays 2");\n'
                   'int (*edit)(rtb200_scene_handle, const uint32_t*, uint32_t, const uint32_t*, const rt_sphere*, uint32_t, void*)\n'
                   '    = rtb200_scene_edit_spheres;\n')
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Werror", "-I", os.path.join(repo, "include"), "-c", str(src),
                           "-o", str(tmp_path / "sig.o")])


def test_null_handle_and_null_arrays_are_refused_before_the_handle_is_used():
    """A stand-in handle that is never dereferenced shows that the argument checks come first; an edit of nothing is a no-op
    that does not touch the handle either."""
    L = R.lib()
    rem = np.array([0], np.uint32)
    ins = (R.rt_sphere * 1)(R.make_sphere([0, 0, 0], 1.0, {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}))
    assert L.rtb200_scene_edit_spheres(None, rem.ctypes.data, 1, None, ins, 1, None) == -1
    assert b"handle" in L.rtb200_last_error()
    fake = C.c_void_p(C.addressof(C.create_string_buffer(64)))
    assert L.rtb200_scene_edit_spheres(fake, None, 1, None, ins, 1, None) == -1
    assert b"remove is null" in L.rtb200_last_error()
    assert L.rtb200_scene_edit_spheres(fake, rem.ctypes.data, 1, None, None, 2, None) == -1
    assert b"insert is null" in L.rtb200_last_error()
    assert L.rtb200_scene_edit_spheres(fake, None, 0, None, None, 0, None) == 0


def test_make_sphere_takes_the_materials_set_sphere_takes():
    sc = R.Scene.from_config(mixed_config(8, 6, 1, 2, n=4))
    mats = [{"Lambertian": {"albedo": [0.1, 0.2, 0.3]}}, {"Metal": {"albedo": [0.9, 0.8, 0.7], "fuzz": 0.25}},
            {"Glass": {"index_of_refraction": 1.5}}, {"Texture": {"albedo": [1, 1, 1], "h_offset": 0.5, "texture": 0}}, {"Light": {}}]
    for m in mats:
        got = R.make_sphere([1.0, 2.0, 3.0], -0.5, m)
        want = sc.set_sphere(2, center=[1.0, 2.0, 3.0], radius=-0.5, material=m)
        assert bytes(got) == bytes(want), m
    assert bytes(R.make_sphere([1.0, 2.0, 3.0], -0.5, got)) == bytes(got)   # an rt_sphere's material is copied
    with pytest.raises(ValueError):
        R.make_sphere([0, 0, 0], 1.0, {"Plasma": {}})


def _tagged(n):
    """A scene of n spheres whose radius is 1 + index, so that every sphere of an edited list names where it came from."""
    objs = [{"center": {"x": float(i), "y": 0.5, "z": 0.0}, "radius": 1.0 + i, "material": {"Lambertian": {"albedo": [0.5, 0.5, 0.5]}}}
            for i in range(n)]
    return R.Scene.from_config(base_config(8, 6, 1, 2, objs))


def _inserts(m):
    """m inserts tagged by a negative radius -(1 + k), with alternating materials (lights among them)."""
    mats = [{"Metal": {"albedo": [0.8, 0.8, 0.8], "fuzz": 0.1}}, {"Light": {}}, {"Glass": {"index_of_refraction": 1.5}}]
    return [R.make_sphere([0.0, 2.0 + k, 1.0], -(1.0 + k), mats[k % 3]) for k in range(m)]


def restated(n, remove, m, at):
    """The edited list as tags (old sphere i: 1 + i, insert k: -(1 + k)), placed by the position formulas."""
    gone = set(remove)
    at = [n] * m if at is None else list(at)
    kept_below = lambda j: sum(1 for i in range(j) if i not in gone)   # noqa: E731
    out = [None] * (n - len(gone) + m)
    for i in range(n):
        if i not in gone:
            p = kept_below(i) + sum(1 for a in at if a <= i)
            assert out[p] is None
            out[p] = 1.0 + i
    for k in range(m):
        p = kept_below(at[k]) + k
        assert out[p] is None
        out[p] = -(1.0 + k)
    assert None not in out
    return out


def _check(sc, remove, m, at):
    ins = _inserts(m)
    e = sc.edited(remove, ins, at)
    want = restated(sc.n_spheres, remove, m, at)
    got = [e._spheres[j].radius for j in range(e.n_spheres)]
    assert got == want, (remove, at)
    for j in range(e.n_spheres):   # every record is the old sphere's or the insert's, byte for byte
        r = e._spheres[j].radius
        src = sc._spheres[int(r) - 1] if r > 0 else ins[int(-r) - 1]
        assert bytes(e._spheres[j]) == bytes(src)
    assert bytes(e.c.camera) == bytes(sc.c.camera) and e.c.width == sc.c.width and e.c.seed == sc.c.seed
    assert e.c.n_textures == sc.c.n_textures and e.c.sky.mode == sc.c.sky.mode
    return e


def test_edited_follows_the_index_rule_on_random_edits():
    rng = np.random.default_rng(3)
    for trial in range(200):
        n = int(rng.integers(0, 40))
        remove = [int(i) for i in rng.permutation(n)[: int(rng.integers(0, n + 1))]]
        m = int(rng.integers(0, 12))
        at = None if rng.uniform() < 0.2 else sorted(int(j) for j in rng.integers(0, n + 1, size=m))
        _check(_tagged(n), remove, m, at)


def test_edited_edge_cases():
    sc = _tagged(10)
    assert _check(sc, list(range(10)), 0, None).n_spheres == 0                  # remove everything
    assert _check(_tagged(0), [], 4, [0, 0, 0, 0]).n_spheres == 4               # insert into an empty list
    _check(_tagged(0), [], 3, None)
    _check(sc, [3, 4, 5], 4, [3, 4, 4, 5])                                      # at names removed spheres
    _check(sc, [], 5, [2, 2, 2, 7, 7])                                          # equal at keep their order
    _check(sc, [0, 9], 3, None)                                                 # at = NULL appends
    _check(sc, [9], 3, [10, 10, 10])                                            # at = n_old appends too
    _check(sc, [0], 2, [0, 0])                                                  # before a removed first sphere
    _check(sc, list(range(10)), 3, [0, 5, 10])                                  # everything removed, inserts anywhere


def test_edited_refuses_what_the_library_refuses():
    sc = _tagged(5)
    for remove, m, at in (([5], 0, None), ([1, 1], 0, None), ([], 2, [3, 2]), ([], 1, [6]), ([], 2, [1])):
        with pytest.raises(ValueError):
            sc.edited(remove, _inserts(m), at)
