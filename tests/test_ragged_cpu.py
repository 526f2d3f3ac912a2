"""CPU-side checks of ragged batches (include/isdf.h): the Python layout helper round-trips every array, isdf_path_waypoints' offsets are
the ragged waypoint rows, the ragged entry points refuse a NULL context and poison their outputs, and a g++ probe compiles a call to each
declaration."""
import ctypes as C
import os
import subprocess
import tempfile
import numpy as np
import isdf_b200 as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PIECES = [3, 1, 17, 2, 64, 1, 290, 3]


def test_layout_helper_round_trips():
    L = I.Ragged(PIECES)
    rng = np.random.default_rng(0)
    assert L.B == len(PIECES) and L.P == sum(PIECES) and list(L.piece_off) == list(np.concatenate([[0], np.cumsum(PIECES)]))
    xs = [rng.normal(size=4 * n - 3) for n in PIECES]
    x = L.pack_x(xs)
    assert x.size == 4 * L.P - 3 * L.B
    for b, n in enumerate(PIECES):
        assert np.array_equal(x[4 * L.piece_off[b] - 3 * b:4 * L.piece_off[b + 1] - 3 * (b + 1)], xs[b])
    assert all(np.array_equal(a, b) for a, b in zip(L.unpack_x(x), xs))
    Ts = [rng.normal(size=n) for n in PIECES]
    T = L.pack_T(Ts)
    assert all(np.array_equal(T[L.piece_off[b] + i], Ts[b][i]) for b in range(L.B) for i in range(PIECES[b]))
    assert all(np.array_equal(a, b) for a, b in zip(L.unpack_T(T), Ts))
    Cs = [rng.normal(size=18 * n) for n in PIECES]
    Cc = L.pack_coeffs(Cs).reshape(3, 6 * L.P)                     # one 6P x 3 column-major block
    for b, n in enumerate(PIECES):
        own = Cs[b].reshape(3, 6 * n)                               # the problem's own 6N x 3 column-major block
        assert np.array_equal(Cc[:, 6 * L.piece_off[b]:6 * L.piece_off[b + 1]], own)
    assert all(np.array_equal(a, b) for a, b in zip(L.unpack_coeffs(Cc.reshape(-1)), Cs))
    wps = [rng.normal(size=(n - 1, 3)) for n in PIECES]
    wp = L.pack_waypoints(wps).reshape(-1, 3)
    assert len(wp) == L.P - L.B
    for b in range(L.B):
        assert np.array_equal(wp[L.wp_off[b]:L.wp_off[b + 1]], wps[b])
    # the uniform batch is the case piece_off[b] = b N0
    U = I.Ragged([5] * 4)
    assert list(U.piece_off) == [0, 5, 10, 15, 20] and list(U.x_off) == [0, 17, 34, 51, 68]


def test_path_waypoints_offsets_are_the_ragged_waypoint_rows():
    lib = I.load_library()
    rng = np.random.default_rng(3)
    paths = [np.cumsum(rng.integers(-1, 2, size=(S, 3)), axis=0) + 0.5 for S in (1, 2, 3, 9, 40, 130, 5)]
    off = np.zeros(len(paths) + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(p) for p in paths])
    xyz = np.ascontiguousarray(np.concatenate(paths), dtype=np.float64)
    cap = int(off[-1])
    wp, wo, pieces = np.zeros((cap, 3)), np.zeros(len(paths) + 1, dtype=np.int32), np.zeros(len(paths), dtype=np.int32)
    ip, dp = C.POINTER(C.c_int32), C.POINTER(C.c_double)
    assert lib.isdf_path_waypoints(len(paths), off.ctypes.data_as(ip), xyz.ctypes.data_as(dp), 1.0, 3.0, cap, wp.ctypes.data_as(dp),
                                   wo.ctypes.data_as(ip), pieces.ctypes.data_as(ip)) == 0
    L = I.Ragged(pieces)
    assert np.array_equal(L.wp_off, wo)
    wps, _ = I.path_waypoints(paths, 1.0, 3.0)
    assert np.array_equal(L.pack_waypoints(wps).reshape(-1, 3), wp[:wo[-1]])


def test_ragged_entry_points_refuse_a_null_context():
    lib = I.load_library()
    B = 3
    off = (C.c_int32 * (B + 1))(0, 2, 3, 7)
    X = 4 * 7 - 3 * B
    h, t = (C.c_double * 27)(), (C.c_double * 27)()
    x, g, T, Cc = (C.c_double * X)(), (C.c_double * X)(), (C.c_double * 7)(), (C.c_double * (18 * 7))()
    wp = (C.c_double * (3 * 4))()
    ret, it, ev, rounds = (C.c_int32 * B)(), (C.c_int32 * B)(), (C.c_int32 * B)(), C.c_int32()
    lp, mp = I.LbfgsParams(), I.MidendParams()
    lib.isdf_lbfgs_default_params(C.byref(lp))
    lib.isdf_midend_default_params(C.byref(mp))
    cost = (C.c_double * B)(1.0, 2.0, 3.0)
    assert lib.isdf_callback_batch_ragged(None, B, off, h, t, 1, 20.0, x, cost, g) == -1
    assert all(np.isnan(v) for v in cost)
    f = (C.c_double * B)(1.0, 2.0, 3.0)
    assert lib.isdf_lbfgs_batch_ragged(None, B, off, h, t, 1, 20.0, C.byref(lp), x, f, ret, it, ev, C.byref(rounds)) == -1
    assert all(np.isnan(v) for v in f)
    cost = (C.c_double * B)(1.0, 2.0, 3.0)
    assert lib.isdf_midend_callback_batch_ragged(None, B, off, h, t, 1, C.byref(mp), wp, x, cost, g) == -1
    assert all(np.isnan(v) for v in cost)
    f = (C.c_double * B)(1.0, 2.0, 3.0)
    assert lib.isdf_midend_batch_ragged(None, B, off, h, t, 1, C.byref(mp), wp, x, T, Cc, f, ret, it, ev, C.byref(rounds)) == -1
    assert all(np.isnan(v) for v in f)
    assert lib.isdf_callback_batch_ragged_device(None, B, off, None, None, 1, 20.0, None, None, None, None) == -1
    assert lib.isdf_lbfgs_batch_ragged_device(None, B, off, None, None, 1, 20.0, C.byref(lp), None, None, None, None, None, None, None) == -1
    assert lib.isdf_midend_batch_ragged_device(None, B, off, None, None, 1, C.byref(mp), None, None, None, None, None, None, None, None, None,
                                               None) == -1


def test_probe_compiles_a_call_to_each_declaration():
    src = r'''#include "isdf.h"
int main() {
    isdf_ctx *c = 0; const int32_t off[3] = {0, 2, 5}; double d[64] = {0}; int32_t i[8] = {0}, r = 0;
    isdf_lbfgs_params lp; isdf_midend_params mp;
    isdf_lbfgs_default_params(&lp); isdf_midend_default_params(&mp);
    int s = 0;
    s += isdf_callback_batch_ragged(c, 2, off, d, d, 0, 20.0, d, d, d);
    s += isdf_callback_batch_ragged_device(c, 2, off, d, d, 0, 20.0, d, d, d, (void *)0);
    s += isdf_lbfgs_batch_ragged(c, 2, off, d, d, 0, 20.0, &lp, d, d, i, i, i, &r);
    s += isdf_lbfgs_batch_ragged_device(c, 2, off, d, d, 0, 20.0, &lp, d, d, i, i, i, &r, (void *)0);
    s += isdf_midend_callback_batch_ragged(c, 2, off, d, d, 0, &mp, d, d, d, d);
    s += isdf_midend_batch_ragged(c, 2, off, d, d, 0, &mp, d, d, d, d, d, i, i, i, &r);
    s += isdf_midend_batch_ragged_device(c, 2, off, d, d, 0, &mp, d, d, d, d, d, i, i, i, &r, (void *)0);
    return s == -7 ? 0 : 1;
}
'''
    with tempfile.TemporaryDirectory() as d:
        path, exe = os.path.join(d, "probe.cpp"), os.path.join(d, "probe")
        open(path, "w").write(src)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        lib_dir = os.path.dirname(I.LIB_PATH)
        subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", exe, path, "-L", lib_dir,
                               "-lisdf_b200", "-Wl,-rpath," + lib_dir])
        assert subprocess.run([exe]).returncode == 0
