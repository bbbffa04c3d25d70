"""Rebuilding the hierarchy of a resident scene (rtb200_scene_rebuild / rtb200_scene_debug_topology): argument errors are
reported before any device is touched, so they need no GPU."""
import ctypes as C

import rtb200 as R

INVALID = -1


def test_the_entry_points_are_exported():
    L = R.lib()
    for name in ("rtb200_scene_rebuild", "rtb200_scene_debug_topology"):
        assert name in R.ABI_SYMBOLS and hasattr(L, name)
    assert L.rtb200_abi_version() == 2


def test_argument_errors_need_no_device():
    L = R.lib()
    assert L.rtb200_scene_rebuild(None, None) == INVALID
    assert b"null scene handle" in L.rtb200_last_error()
    g = (C.c_double * 3)()
    info = (C.c_uint32 * 8)()
    assert L.rtb200_scene_debug_topology(None, g, info, None, 0, None, 0, None, 0, None, 0, None, 0) == INVALID
    assert b"null argument" in L.rtb200_last_error()
