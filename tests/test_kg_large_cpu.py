"""CPU-side argument checks of cmoe_kg_eval_large (no GPU needed): the size bounds are tested before the handle or the
device is touched, so they hold on any machine."""
import ctypes
import os
import re


def _kg_large(lib, q, p, num_mc=16, nc=1):
    from cornell_moe_b200 import capi
    inner = capi.GDParams.from_seq([1, 0, 1, 1, 0.0, 1.0, 1.0, 1e-10])
    info = ctypes.c_int(0)
    return lib.cmoe_kg_eval_large(None, 0, ctypes.byref(inner), None, None, 0, None, nc, q, None, p, num_mc,
                                  ctypes.c_double(0.0), ctypes.c_uint64(0), None, None, None, None, ctypes.byref(info))


def test_kg_eval_large_bounds():
    from cornell_moe_b200 import capi
    lib = capi.lib()
    assert _kg_large(lib, 1000, 25) == capi.ERR_BOUNDS  # Q = 1025
    assert _kg_large(lib, 1025, 0) == capi.ERR_BOUNDS
    assert _kg_large(lib, 0, 5) == capi.ERR_BOUNDS
    assert _kg_large(lib, 5, -1) == capi.ERR_BOUNDS
    assert _kg_large(lib, 5, 0, num_mc=0) == capi.ERR_BOUNDS
    assert _kg_large(lib, 5, 0, nc=0) == capi.ERR_BOUNDS
    assert _kg_large(lib, 5, 0, num_mc=65535 * 64 + 1) == capi.ERR_BOUNDS  # past the scan product's grid


def test_kg_eval_large_needs_a_handle():
    from cornell_moe_b200 import capi
    assert _kg_large(capi.lib(), 1000, 24) == capi.ERR_INVALID_VALUE  # Q = 1024 passes the size bounds


def test_kg_large_limit_is_public():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "include", "cmoe_b200.h")).read()
    assert re.search(r"#define CMOE_MAX_KG_LARGE_ROWS 1024\b", src)
    assert "int cmoe_kg_eval_large(" in src
