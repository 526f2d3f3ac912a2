"""TEST INFRASTRUCTURE: CPU restatements that isdf_frontend_path is held against (tests/frontpath_serial.cpp, built by build() next to
the library objects), and a brute-force Bellman-Ford that the serial Dijkstra is held against.

  dijkstra(trav, src)           the exact FP64 cost-to-come field of include/isdf.h
  path(g, src, t)               the parent rule of include/isdf.h on a field: (n, 3) voxel indices, start first
  ref_astar(occ, masks, ...)    the reference's A* with its quirks (front_end_Astar.hpp), for comparison only
  bellman_ford(trav, src)       relax every edge until nothing changes (numpy; tiny grids)"""
import ctypes as C
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "frontpath_serial.cpp")
LIB = os.path.join(ROOT, "implicit-sdf-planner_b200", "build", "libfrontpath_serial.so")
OFFSETS = [(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1) if (i, j, k) != (0, 0, 0)]


def build(force=False):
    if force or not os.path.exists(LIB) or os.path.getmtime(SRC) > os.path.getmtime(LIB):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", LIB, SRC])


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        dp, ip, u8p, i64p = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_uint8), C.POINTER(C.c_int64)
        L.fp_dijkstra.argtypes = [u8p, C.c_int, C.c_int, C.c_int, ip, dp]
        L.fp_dijkstra.restype = C.c_int64
        L.fp_path.argtypes = [dp, C.c_int, C.c_int, C.c_int, ip, ip, ip, C.c_int64]
        L.fp_path.restype = C.c_int64
        L.fp_ref_astar.argtypes = [u8p, C.POINTER(C.c_uint32), C.c_int, C.c_int, C.c_int, ip, ip, C.c_int, C.c_int, C.c_double, C.c_double,
                                   C.c_double, dp, ip, dp, C.c_int64, i64p, i64p]
        L.fp_ref_astar.restype = C.c_int
        _lib = L
    return _lib


def _i3(v):
    return np.ascontiguousarray(v, dtype=np.int32).reshape(3)


def dijkstra(trav, src):
    trav = np.ascontiguousarray(trav, dtype=np.uint8)
    X, Y, Z = trav.shape
    g = np.empty((X, Y, Z))
    s = _i3(src)
    lib().fp_dijkstra(trav.ctypes.data_as(C.POINTER(C.c_uint8)), X, Y, Z, s.ctypes.data_as(C.POINTER(C.c_int32)), g.ctypes.data_as(C.POINTER(C.c_double)))
    return g


def path(g, src, t):
    g = np.ascontiguousarray(g, dtype=np.float64)
    X, Y, Z = g.shape
    s, tt = _i3(src), _i3(t)
    ip = C.POINTER(C.c_int32)
    n = lib().fp_path(g.ctypes.data_as(C.POINTER(C.c_double)), X, Y, Z, s.ctypes.data_as(ip), tt.ctypes.data_as(ip), None, 0)
    assert n > 0, "no parent found: not a field of the definition"
    out = np.zeros((n, 3), dtype=np.int32)
    lib().fp_path(g.ctypes.data_as(C.POINTER(C.c_double)), X, Y, Z, s.ctypes.data_as(ip), tt.ctypes.data_as(ip), out.ctypes.data_as(ip), n)
    return out


def ref_astar(occ, masks, src, goal, xk, yk, max_roll=45.0, max_pitch=45.0, ang_res=9.0):
    """-> dict(found, cost, path (n, 3), roll_pitch (n, 2), expanded); masks: (X*Y*Z, 4) free attitudes"""
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y, Z = occ.shape
    masks = np.ascontiguousarray(masks, dtype=np.uint32).reshape(-1, 4)
    s, g = _i3(src), _i3(goal)
    ip = C.POINTER(C.c_int32)
    cost, n, ex = C.c_double(0), C.c_int64(0), C.c_int64(0)
    args = [occ.ctypes.data_as(C.POINTER(C.c_uint8)), masks.ctypes.data_as(C.POINTER(C.c_uint32)), X, Y, Z, s.ctypes.data_as(ip), g.ctypes.data_as(ip),
            xk, yk, max_roll, max_pitch, ang_res, C.byref(cost)]
    found = lib().fp_ref_astar(*args, None, None, 0, C.byref(n), C.byref(ex))
    p, rp = np.zeros((max(n.value, 1), 3), dtype=np.int32), np.zeros((max(n.value, 1), 2))
    lib().fp_ref_astar(*args, p.ctypes.data_as(ip), rp.ctypes.data_as(C.POINTER(C.c_double)), n.value, C.byref(n), C.byref(ex))
    return dict(found=bool(found), cost=cost.value, path=p[:n.value], roll_pitch=rp[:n.value], expanded=ex.value)


def bellman_ford(trav, src):
    """every round offers g(u) + w to all 26 neighbours at once (each sum adds one edge to a path sum, left to right); until no change"""
    trav = np.asarray(trav, dtype=bool)
    X, Y, Z = trav.shape
    g = np.full((X, Y, Z), np.inf)
    g[tuple(src)] = 0.0
    P = np.full((X + 2, Y + 2, Z + 2), np.inf)
    while True:
        P[1:-1, 1:-1, 1:-1] = g
        new = g.copy()
        for i, j, k in OFFSETS:
            # v = u + (i, j, k): g(u) is P at v - (i, j, k)
            gu = P[1 - i:1 - i + X, 1 - j:1 - j + Y, 1 - k:1 - k + Z]
            cand = gu + np.sqrt(float(i * i + j * j + k * k))
            new = np.where(trav & (cand < new), cand, new)
        if np.array_equal(new, g):
            return g
        g = new


def traversable(occ, masks):
    """include/isdf.h's Traversable: free voxel with a non-zero feasibility mask"""
    X, Y, Z = occ.shape
    return (np.asarray(masks).reshape(X, Y, Z, 4).any(axis=3)) & (np.asarray(occ) == 0)


def check_path(nodes, trav, src):
    """26-adjacent steps, start first, every node after the start traversable"""
    nodes = np.asarray(nodes)
    assert tuple(nodes[0]) == tuple(src)
    if len(nodes) > 1:
        assert (np.abs(np.diff(nodes, axis=0)).max(axis=1) == 1).all()
    for v in nodes[1:]:
        assert trav[tuple(v)]
