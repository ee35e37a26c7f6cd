"""CPU-side argument checks of the ensemble q-KG / q-EI calls past the per-set bounds (no GPU needed): a union past the
large paths' limits is refused before any handle is read or any device work is done, so it holds on any machine."""
import ctypes


def _kg_mcmc(lib, q, p, num_gp=3):
    from cornell_moe_b200 import capi
    inner = capi.GDParams.from_seq([1, 0, 1, 1, 0.0, 1.0, 1.0, 1e-10])
    info = ctypes.c_int(0)
    return lib.cmoe_kg_eval_mcmc(None, num_gp, 0, ctypes.byref(inner), None, None, 0, None, 1, q, None, p, 16, None,
                                 ctypes.c_uint64(0), None, None, None, ctypes.byref(info))


def _ei_mcmc(lib, q, p, num_gp=3):
    info = ctypes.c_int(0)
    return lib.cmoe_ei_eval_mcmc(None, num_gp, None, 1, q, None, p, 16, None, ctypes.c_uint64(0), None, 0, None, None,
                                 ctypes.byref(info))


def test_kg_mcmc_refuses_past_1024_rows_before_the_handles():
    from cornell_moe_b200 import capi
    lib = capi.lib()
    assert _kg_mcmc(lib, 1000, 25) == capi.ERR_BOUNDS  # Q >= q + p = 1025
    assert _kg_mcmc(lib, 1025, 0) == capi.ERR_BOUNDS
    assert b"1024" in lib.cmoe_last_error()


def test_ei_mcmc_refuses_past_8192_rows_before_the_handles():
    from cornell_moe_b200 import capi
    lib = capi.lib()
    assert _ei_mcmc(lib, 8000, 193) == capi.ERR_BOUNDS  # q + p = 8193
    assert _ei_mcmc(lib, 8193, 0) == capi.ERR_BOUNDS
    assert b"8192" in lib.cmoe_last_error()


def test_ensemble_members_in_flight_option():
    from cornell_moe_b200 import capi
    capi.set_option("ensemble_members_in_flight", 1)
    capi.set_option("ensemble_members_in_flight", 0)
    try:
        capi.set_option("ensemble_members_in_flight", -1)
    except capi.InvalidValueError:
        pass
    else:
        raise AssertionError("a negative member count must be refused")
