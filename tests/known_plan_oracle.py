"""TEST INFRASTRUCTURE: restatements of planning through what has been seen (include/isdf.h, DESIGN §3.23) that the device is held against.

  dijkstra(trav, known, src, w)      the front end's field with the surcharge w on unknown voxels (tests/known_plan_serial.cpp)
  path(g, known, src, t, w)          the parent rule on such a field, w(u, v) read at v
  waypoint_gap(S, res, parlength)    isdf_path_waypoints' gap g of a path of S nodes (waypoint row j is path node (j + 1) g)
  known_rows(nodes, known, g, N)     ISDF_PLAN_KNOWN_PREFIX's rows: k* = the first node not known, rows j < N - 1 with (j + 1) g < k*
  gather(occ, known, ..., rows)      isdf_gather_obstacle_points_batch_known for one plan, in numpy"""
import ctypes as C
import math
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "known_plan_serial.cpp")
LIB = os.path.join(ROOT, "implicit-sdf-planner_b200", "build", "libknown_plan_serial.so")


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
        dp, ip, u8p = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
        L.kp_dijkstra.argtypes = [u8p, u8p, C.c_int, C.c_int, C.c_int, ip, C.c_double, dp]
        L.kp_dijkstra.restype = C.c_int64
        L.kp_path.argtypes = [dp, u8p, C.c_int, C.c_int, C.c_int, ip, ip, C.c_double, ip, C.c_int64]
        L.kp_path.restype = C.c_int64
        _lib = L
    return _lib


def _u8(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.uint8)


def _ptr(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def dijkstra(trav, known, src, unknown_weight):
    """known: (X, Y, Z) bools or None (nothing known)"""
    trav, known = _u8(trav), _u8(known)
    X, Y, Z = trav.shape
    g = np.empty((X, Y, Z))
    s = np.ascontiguousarray(src, dtype=np.int32).reshape(3)
    lib().kp_dijkstra(_ptr(trav, C.c_uint8), _ptr(known, C.c_uint8), X, Y, Z, _ptr(s, C.c_int32), 1.0 + float(unknown_weight), _ptr(g, C.c_double))
    return g


def path(g, known, src, t, unknown_weight):
    g, known = np.ascontiguousarray(g, dtype=np.float64), _u8(known)
    X, Y, Z = g.shape
    s, tt = np.ascontiguousarray(src, dtype=np.int32).reshape(3), np.ascontiguousarray(t, dtype=np.int32).reshape(3)
    args = [_ptr(g, C.c_double), _ptr(known, C.c_uint8), X, Y, Z, _ptr(s, C.c_int32), _ptr(tt, C.c_int32), 1.0 + float(unknown_weight)]
    n = lib().kp_path(*args, None, 0)
    assert n > 0, "no parent found: not a field of the definition"
    out = np.zeros((n, 3), dtype=np.int32)
    lib().kp_path(*args, _ptr(out, C.c_int32), n)
    return out


def waypoint_gap(S, res, parlength):
    """k_wp_count's gap of a path of S nodes (0 for S <= 2: no waypoint)"""
    if S <= 2:
        return 0
    pl = parlength
    gp = math.ceil(pl / res)
    while gp >= S - 1:
        pl /= 1.5
        gp = math.ceil(pl / res)
    return int(gp)


def first_unknown(nodes, known):
    """k*: the index of the first node whose voxel is not known, len(nodes) when every node is (known None: 0)"""
    if known is None:
        return 0
    for m, v in enumerate(np.asarray(nodes)):
        if not known[tuple(v)]:
            return m
    return len(nodes)


def known_rows(nodes, known, gap, N):
    ks = first_unknown(nodes, known)
    return sum(1 for j in range(N - 1) if (j + 1) * gap < ks)


def _axis(coord, lo, hi, res, size):
    c = min(max(coord, lo), hi)
    return min(max(int(math.floor((c - lo) / res)), 0), size - 1)


def gather(occ, known, bmin, bmax, res, wps, half, offset=(0.0, 0.0, 0.0), rows=0):
    """one plan's list: for every waypoint j in order, the voxels of box(wp_j + offset, half) outside box(wp_{j-1}, half) (999 before the
    first) that are set in row j's grid (blocked = occ | ~known for j < rows, else occ), in x -> y -> z order, each voxel only in the first
    box of the plan that includes it (tested on that box's own grid)"""
    occ = np.asarray(occ, dtype=bool)
    blocked = occ | ~np.asarray(known, dtype=bool) if known is not None else np.ones_like(occ)
    dims = occ.shape
    wps = np.asarray(wps, dtype=np.float64).reshape(-1, 3)
    boxes = []
    for j, w in enumerate(wps):
        c = [w[a] + offset[a] for a in range(3)]
        l = wps[j - 1] if j else [999.0] * 3
        boxes.append(([_axis(c[a] - half, bmin[a], bmax[a], res, dims[a]) for a in range(3)],
                      [_axis(c[a] + half, bmin[a], bmax[a], res, dims[a]) for a in range(3)],
                      [_axis(l[a] - half, bmin[a], bmax[a], res, dims[a]) for a in range(3)],
                      [_axis(l[a] + half, bmin[a], bmax[a], res, dims[a]) for a in range(3)]))

    def includes(j, I, J, K):
        a0, a1, l0, l1 = boxes[j]
        grid = blocked if j < rows else occ
        inb = (I >= a0[0]) & (I <= a1[0]) & (J >= a0[1]) & (J <= a1[1]) & (K >= a0[2]) & (K <= a1[2])
        inl = (I >= l0[0]) & (I <= l1[0]) & (J >= l0[1]) & (J <= l1[1]) & (K >= l0[2]) & (K <= l1[2])
        return inb & ~inl & grid[np.clip(I, 0, dims[0] - 1), np.clip(J, 0, dims[1] - 1), np.clip(K, 0, dims[2] - 1)]

    out = []
    for j, (a0, a1, _, _) in enumerate(boxes):
        I, J, K = np.meshgrid(np.arange(a0[0], a1[0] + 1), np.arange(a0[1], a1[1] + 1), np.arange(a0[2], a1[2] + 1), indexing="ij")
        I, J, K = I.reshape(-1), J.reshape(-1), K.reshape(-1)
        emit = includes(j, I, J, K)
        for p in range(j):
            emit &= ~includes(p, I, J, K)
        out.append(np.stack([(I[emit] + 0.5) * res + bmin[0], (J[emit] + 0.5) * res + bmin[1], (K[emit] + 0.5) * res + bmin[2]], axis=1))
    return np.concatenate(out) if out else np.zeros((0, 3))
