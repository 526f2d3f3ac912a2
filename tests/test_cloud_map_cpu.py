"""CPU checks of the point-cloud map path (isdf_set_map_cloud): the serial C++ and numpy restatements against the reference-compiled
voxelisation (or its committed outputs), the isdf_map_info layout, and every argument refusal without a device."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
import cloud_oracle as CO
import isdf_b200 as I
import oracle_lib as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = CO.load_fixture()


def _check(r, f, thr):
    assert r["dims"] == f["dims"]
    assert np.array_equal(r["bmin"], f["bmin"]) and np.array_equal(r["bmax"], f["bmax"])
    assert np.array_equal(r["occ"], f["occ"][thr])


def test_fixture_covers_the_cases():
    assert set(FIX) == set(CO.cloud_cases())
    for name, (raw, stride, res) in CO.cloud_cases().items():
        f = FIX[name]
        assert f["stride"] == stride and f["res"] == res and np.array_equal(f["raw"], raw), name   # the seeds still make the stored inputs
    assert {f["stride"] for f in FIX.values()} >= {12, 16, 32} and {f["res"] for f in FIX.values()} >= {1.0, 0.1, 0.4}
    # the HUGE_NUMBER start survives on one axis of two cases; the top layer is reached by a maximum at an exact multiple of res
    assert FIX["huge_x_r1_xyz16"]["bmin"][0] == 999999999.0 and FIX["huge_negz_r05_xyz12"]["bmax"][2] == -999999999.0
    f = FIX["faces_r1_xyz16"]
    assert np.array_equal((f["bmax"] - f["bmin"]) / f["res"], f["dims"]) and f["occ"][1][-1, :, :].any()
    for f in FIX.values():   # the thresholds split the voxels
        counts = [int(f["occ"][t].sum()) for t in CO.THRESHOLDS]
        assert counts[0] == np.prod(f["dims"]) and counts == sorted(counts, reverse=True) and counts[4] > 0, counts
    assert sum(len({int(f["occ"][t].sum()) for t in CO.THRESHOLDS}) == 5 for f in FIX.values()) >= 3


@pytest.mark.parametrize("thr", CO.THRESHOLDS)
@pytest.mark.parametrize("name", sorted(CO.cloud_cases()))
def test_serial_and_numpy_match_the_reference(name, thr):
    f = FIX[name]
    _check(CO.serial(f["raw"], f["stride"], f["res"], thr), f, thr)
    _check(CO.numpy_map(f["raw"], f["stride"], f["res"], thr), f, thr)
    if os.path.exists(O.REF_GRID):
        _check(CO.ref_map(f["raw"], f["stride"], f["res"], thr), f, thr)


def test_non_finite_records_are_skipped_by_the_restatements():
    f = FIX["uniform_r04_stride32"]
    rec = f["raw"].view(np.float32).reshape(-1, 8).copy()
    bad = np.zeros((4, 8), dtype=np.float32)
    bad[0, 0], bad[1, 1], bad[2, 2], bad[3, :3] = np.nan, np.inf, -np.inf, [1e30, np.nan, 0]
    raw = np.concatenate([bad[:2], rec, bad[2:]]).view(np.uint8).reshape(-1)
    for fn in (CO.serial, CO.numpy_map):
        r = fn(raw, 32, f["res"], 2)
        _check(r, f, 2)
        assert r["skipped"] == 4


def test_map_info_layout_matches_the_header():
    assert C.sizeof(I.MapInfo) == 96
    offs = {n: getattr(I.MapInfo, n).offset for n, _ in I.MapInfo._fields_}
    assert offs == dict(X=0, Y=4, Z=8, reserved_=12, res=16, bmin=24, bmax=48, occupied_voxels=72, points_used=80, points_skipped=88)
    src = ('#include "isdf.h"\n#include <stddef.h>\n'
           'typedef char a[sizeof(isdf_map_info) == 96 ? 1 : -1];\n'
           'typedef char b[offsetof(isdf_map_info, res) == 16 && offsetof(isdf_map_info, bmax) == 48 ? 1 : -1];\n'
           'typedef char c[offsetof(isdf_map_info, occupied_voxels) == 72 && offsetof(isdf_map_info, points_skipped) == 88 ? 1 : -1];\n'
           'int main(void) { return 0; }\n')
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-Wno-unused-local-typedefs", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c", "-"],
                       input=src.encode(), capture_output=True)
    assert r.returncode == 0, r.stderr.decode()


def test_cloud_entry_points_refuse_bad_arguments_without_a_device():
    lib = I.load_library()
    pts = np.zeros((8, 4), dtype=np.float32)
    p = pts.ctypes.data_as(C.c_void_p)
    err = lambda: lib.isdf_last_error().decode()   # noqa: E731
    for fn, extra in ((lib.isdf_set_map_cloud, ()), (lib.isdf_set_map_cloud_device, (None,))):
        assert fn(None, None, 8, 16, 1.0, 1, *extra) == -1 and "points is NULL" in err()
        assert fn(None, p, 0, 16, 1.0, 1, *extra) == -1 and "point count" in err()
        assert fn(None, p, -5, 16, 1.0, 1, *extra) == -1 and "point count" in err()
        assert fn(None, p, 1 << 32, 16, 1.0, 1, *extra) == -1 and "point count" in err()
        assert fn(None, p, 8, 8, 1.0, 1, *extra) == -1 and "stride_bytes" in err()
        assert fn(None, p, 8, 14, 1.0, 1, *extra) == -1 and "stride_bytes" in err()
        assert fn(None, C.c_void_p(pts.ctypes.data + 2), 7, 16, 1.0, 1, *extra) == -1 and "aligned" in err()
        for res in (0.0, -1.0, float("nan"), float("inf")):
            assert fn(None, p, 8, 16, res, 1, *extra) == -1 and "res" in err()
        assert fn(None, p, 8, 16, 1.0, 1, *extra) == -1 and "ctx is NULL" in err()
    assert lib.isdf_get_map_info(None, None) == -1
    assert lib.isdf_get_map_u8(None, None, 0) == -1 and lib.isdf_get_map_f64(None, None, 0) == -1


def test_python_binding_rejects_other_dtypes():
    ev = I.Evaluator.__new__(I.Evaluator)   # no context: the dtype check comes first
    for bad in (np.zeros((4, 3)), np.zeros((4, 3), dtype=np.float16), np.zeros((4, 3), dtype=np.int32), np.zeros((4, 2), dtype=np.float32)):
        with pytest.raises((TypeError, ValueError)):
            ev.set_map_cloud(bad, 1.0)
