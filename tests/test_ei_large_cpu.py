"""CPU-side argument checks of the large-set calls (no GPU needed): the size bounds are tested before the handle or the
device is touched, so they hold on any machine."""
import ctypes
import os
import re


def _ei_large(lib, q, p, num_mc=16, nc=1):
    info = ctypes.c_int(0)
    return lib.cmoe_ei_eval_large(None, None, nc, q, None, p, num_mc, ctypes.c_double(0.0), ctypes.c_uint64(0), None,
                                  None, None, ctypes.byref(info))


def test_ei_eval_large_bounds():
    from cornell_moe_b200 import capi
    lib = capi.lib()
    assert _ei_large(lib, 8000, 193) == capi.ERR_BOUNDS  # U = 8193
    assert _ei_large(lib, 8193, 0) == capi.ERR_BOUNDS
    assert _ei_large(lib, 0, 5) == capi.ERR_BOUNDS
    assert _ei_large(lib, 5, -1) == capi.ERR_BOUNDS
    assert _ei_large(lib, 5, 0, num_mc=0) == capi.ERR_BOUNDS
    assert _ei_large(lib, 5, 0, nc=0) == capi.ERR_BOUNDS


def test_posterior_large_needs_a_handle():
    from cornell_moe_b200 import capi
    info = ctypes.c_int(0)
    rc = capi.lib().cmoe_gp_posterior_large(None, None, 1, 97, None, 0, None, None, None, ctypes.byref(info))
    assert rc == capi.ERR_INVALID_VALUE


def test_limits_are_public():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "include", "cmoe_b200.h")).read()
    assert re.search(r"#define CMOE_MAX_SET_ROWS 96\b", src)
    assert re.search(r"#define CMOE_MAX_LARGE_SET_ROWS 8192\b", src)
