"""CPU checks of the (start, goal) pair entry points (isdf_frontend_path_pairs[_device], isdf_frontend_path_fields_device,
isdf_plan_pairs): each refuses a NULL context with ISDF_ERR_INVALID, writes no path output and needs no device."""
import ctypes as C
import numpy as np
import isdf_b200 as I


def test_null_context_is_refused():
    lib = I.load_library()
    ip, u8p = C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
    starts, goals = np.zeros((2, 3)), np.ones((2, 3))
    xyz, rp = np.full((8, 3), 7.0), np.full((8, 2), 7.0)
    off, cost, found = np.full(3, -7, dtype=np.int32), np.full(2, 7.0), np.full(2, 7, dtype=np.uint8)
    assert lib.isdf_frontend_path_pairs(None, 2, I._dp(starts), I._dp(goals), None, 0, 8, I._dp(xyz), I._dp(rp), off.ctypes.data_as(ip),
                                        I._dp(cost), found.ctypes.data_as(u8p)) == -1
    assert b"NULL" in lib.isdf_last_error()
    assert (off == -7).all() and (xyz == 7.0).all() and (cost == 7.0).all() and (found == 7).all()
    dummy = C.c_void_p(16)   # never dereferenced: the context is checked before any device pointer is used
    assert lib.isdf_frontend_path_pairs_device(None, 2, dummy, dummy, None, 0, 8, dummy, dummy, dummy, dummy, dummy, None) == -1
    assert lib.isdf_frontend_path_fields_device(None, 2, I._dp(starts), None, dummy, None) == -1
    p = I.PlanParams()
    assert lib.isdf_plan_default_params(None, C.byref(p)) == 0
    po, pf = np.full(3, -7, dtype=np.int32), np.full(3, -7, dtype=np.int32)
    T, Cc = np.zeros(4), np.zeros(72)
    res, cs, ds = (I.PlanResult * 2)(), (I.CertifySummary * 2)(), (I.DynamicsSummary * 2)()
    assert lib.isdf_plan_pairs(None, 2, I._dp(starts), I._dp(goals), C.byref(p), 0, 8, pf.ctypes.data_as(ip), I._dp(xyz), 4,
                               po.ctypes.data_as(ip), I._dp(T), I._dp(Cc), res, cs, ds) == -1
    assert b"NULL" in lib.isdf_last_error()
    assert (pf == -7).all() and (po == -7).all() and all(r.stage == I.PLAN_FAILED for r in res)
