"""TEST INFRASTRUCTURE: CPU restatements of the reference's point-cloud voxelisation (PCSmapManager::rcvGlobalMapHandler,
PCSmap_manager.cpp:111-181) that isdf_set_map_cloud is held against, and the seeded fixture clouds of tests/golden/cloud_reference.npz.

  serial()     the serial C++ loop on the oracle's grid (tests/cloud_map_serial.cpp, built by build() next to the library objects);
  numpy_map()  an independent vectorised restatement;
  ref_map()    the reference-compiled index arithmetic (oracle/_ref/libref_grid.so: createGridMap, getGridIndex) under a restated
               bounds / count / threshold glue; used to write the fixture where the reference tree exists.

All three skip records with a non-finite coordinate, as the library does (undefined behaviour in the reference)."""
import ctypes as C
import math
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cloud_map_serial.cpp")
LIB = os.path.join(ROOT, "implicit-sdf-planner_b200", "build", "libcloud_map_serial.so")
FIXTURE = os.path.join(ROOT, "tests", "golden", "cloud_reference.npz")
HUGE = 999999999.0
THRESHOLDS = (0, 1, 2, 3, 7)


def build(force=False):
    deps = [SRC, os.path.join(ROOT, "oracle", "oracle_planner.hpp"), os.path.join(ROOT, "oracle", "oracle_math.hpp")]
    if force or not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        # the reference's flags (planner_algorithm/CMakeLists.txt:4: -O3, no -march); no contraction, as in the oracle
        subprocess.check_call([gxx, "-O3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", LIB, SRC])


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.cloud_map_serial.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_double, C.c_int32, C.c_int, C.POINTER(C.c_int32),
                                       C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64), C.POINTER(C.c_uint8)]
        _lib = L
    return _lib


def as_records(raw, stride):
    """(n, 3) float64 view of x, y, z of n records of `stride` bytes (raw: uint8 buffer or float32 (n, k) array)"""
    b = np.ascontiguousarray(raw).view(np.uint8).reshape(-1)
    n = b.size // stride
    return np.ndarray((n, 3), dtype=np.float32, buffer=b, strides=(stride, 4)).astype(np.float64)


def serial(raw, stride, res, thr, dims_only=False):
    """-> dict(dims, bmin, bmax, skipped, occ (X, Y, Z) uint8 or None); None for no finite point / a degenerate extent"""
    b = np.ascontiguousarray(raw).view(np.uint8).reshape(-1)
    n = b.size // stride
    dims, bmin, bmax, sk = np.zeros(3, dtype=np.int32), np.zeros(3), np.zeros(3), C.c_int64(0)
    args = (b.ctypes.data_as(C.c_void_p), n, stride, float(res), int(thr))
    dp = C.POINTER(C.c_double)
    if lib().cloud_map_serial(*args, 1, dims.ctypes.data_as(C.POINTER(C.c_int32)), bmin.ctypes.data_as(dp), bmax.ctypes.data_as(dp), C.byref(sk), None) != 0:
        return None
    occ = None
    if not dims_only:
        occ = np.zeros(tuple(int(d) for d in dims), dtype=np.uint8)
        lib().cloud_map_serial(*args, 0, dims.ctypes.data_as(C.POINTER(C.c_int32)), bmin.ctypes.data_as(dp), bmax.ctypes.data_as(dp), C.byref(sk),
                               occ.ctypes.data_as(C.POINTER(C.c_uint8)))
    return dict(dims=tuple(int(d) for d in dims), bmin=bmin, bmax=bmax, skipped=int(sk.value), occ=occ)


def frame(p):
    """bounds from the HUGE_NUMBER start with strict updates (:111-143) and createGridMap's sizes, over the finite rows of p (float64)"""
    bmin, bmax = np.full(3, HUGE), np.full(3, -HUGE)
    for a in range(3):
        lo, hi = p[:, a].min(), p[:, a].max()
        if lo < bmin[a]:
            bmin[a] = lo
        if hi > bmax[a]:
            bmax[a] = hi
    return bmin, bmax


def _finite(raw, stride):
    p = as_records(raw, stride)
    ok = np.isfinite(p).all(axis=1)
    return p[ok], int((~ok).sum())


def _occupancy(addr, nvox, thr):
    cnt = np.bincount(addr, minlength=nvox)
    return (cnt >= thr).astype(np.uint8)


def numpy_map(raw, stride, res, thr):
    p, skipped = _finite(raw, stride)
    bmin, bmax = frame(p)
    X, Y, Z = (int(math.ceil((bmax[a] - bmin[a]) / res)) for a in range(3))
    q = np.floor((p - bmin) / res).astype(np.int64)       # getGridIndex (Gridmap3D.cpp:135-175)
    ix, iy, iz = q[:, 0].copy(), q[:, 1].copy(), q[:, 2].copy()
    ix[ix < 0] = 0
    ix[ix >= X] = X - 1
    ix[iy < 0] = 0          # sic (quirk Q6)
    iy[iy >= Y] = Y - 1
    ix[iz < 0] = 0          # sic
    iz[iz >= Z] = Z - 1
    occ = _occupancy((ix * Y + iy) * Z + iz, X * Y * Z, thr).reshape(X, Y, Z)
    return dict(dims=(X, Y, Z), bmin=bmin, bmax=bmax, skipped=skipped, occ=occ)


def ref_map(raw, stride, res, thr):
    """the reference-compiled getGridIndex on every record. ref_grid_index builds its grid with createGridMap(bmin, bmin + X*res): it asserts
    that this reproduces X (so createGridMap's own ceil agrees) and that every record is inside it, so the indices are those the reference's
    grid over (bmin, cloud max) returns (getGridIndex reads boundary_xyzmax only through isInMap)."""
    import oracle_lib as O
    p, skipped = _finite(raw, stride)
    bmin, bmax = frame(p)
    dims = tuple(int(math.ceil((bmax[a] - bmin[a]) / res)) for a in range(3))
    idx, _, inmap = O.RefGrid().index(dims, bmin, res, p)
    assert inmap.all(), "a record lies outside createGridMap(bmin, bmin + X*res)"
    X, Y, Z = dims
    idx = idx.astype(np.int64)
    occ = _occupancy((idx[:, 0] * Y + idx[:, 1]) * Z + idx[:, 2], X * Y * Z, thr).reshape(dims)
    return dict(dims=dims, bmin=bmin, bmax=bmax, skipped=skipped, occ=occ)


# ---- the fixture clouds ------------------------------------------------------------------------------------------------
def _records(xyz, stride, rng):
    """float32 records of `stride` bytes with x, y, z at 0, 4, 8 and filler after (NaN and noise: the library must read only x, y, z)"""
    n = xyz.shape[0]
    rec = np.zeros((n, stride // 4), dtype=np.float32)
    rec[:, :3] = xyz
    if stride // 4 > 3:
        rec[:, 3:] = rng.standard_normal((n, stride // 4 - 3)).astype(np.float32)
        rec[::3, 3] = np.nan
    return rec.view(np.uint8).reshape(-1)


def _dup(xyz, rng):
    """each point 1..8 times (so thresholds 2, 3 and 7 split the voxels), in random order"""
    rep = rng.integers(1, 9, size=xyz.shape[0])
    out = np.repeat(xyz, rep, axis=0)
    return out[rng.permutation(out.shape[0])]


def cloud_cases():
    """name -> (records as uint8, stride, res). Seeded; tests/golden/make_cloud_golden.py stores inputs and reference outputs."""
    cases = {}
    rng = np.random.default_rng(20261015)
    # res 1.0, points on voxel faces (integers and half-integers), the maxima at exact multiples of res on every axis (top-layer clamp),
    # negative and fractional origin; PointXYZ records (stride 16)
    g = np.stack(np.meshgrid(np.arange(-3.0, 9.5, 0.5), np.arange(-2.5, 6.0, 0.5), np.arange(0.25, 6.5, 1.0), indexing="ij"), -1).reshape(-1, 3)
    g = g[rng.random(g.shape[0]) < 0.4]
    g = np.concatenate([g, [[-3.0, -2.5, 0.25], [9.0, 5.5, 6.25], [9.0, -2.5, 3.25], [0.0, 5.5, 6.25]]])
    cases["faces_r1_xyz16"] = (_records(_dup(g.astype(np.float32), rng), 16, rng), 16, 1.0)
    # res 0.1 (not representable): coordinates float32(k * 0.1 + o), right on the nominal faces; packed xyz (stride 12)
    k = rng.integers(0, 40, size=(900, 3))
    f = (k * 0.1 + np.array([-1.3, 0.7, 2.2])).astype(np.float32)
    cases["faces_r01_xyz12"] = (_records(_dup(f, rng), 12, rng), 12, 0.1)
    # res 0.4, uniform points with a fractional origin; 32-byte records carrying extra fields (NaN among them)
    u = (rng.random((1500, 3)) * np.array([5.3, 3.1, 2.5]) + np.array([-2.17, 0.31, -0.93])).astype(np.float32)
    cases["uniform_r04_stride32"] = (_records(_dup(u, rng), 32, rng), 32, 0.4)
    # x beyond +999999999 (float32 steps of 64 there): the bounds keep the HUGE_NUMBER start as min x; res 1.0
    h = np.stack([1.0e9 + 64.0 * rng.integers(0, 12, 600), rng.random(600) * 4.0 - 1.0, rng.random(600) * 3.0], -1).astype(np.float32)
    cases["huge_x_r1_xyz16"] = (_records(_dup(h, rng), 16, rng), 16, 1.0)
    # z below -999999999: the max z stays -999999999; res 0.5
    hz = np.stack([rng.random(500) * 3.0, rng.random(500) * 2.0, -1.0e9 - 64.0 * rng.integers(0, 3, 500)], -1).astype(np.float32)
    cases["huge_negz_r05_xyz12"] = (_records(_dup(hz, rng), 12, rng), 12, 0.5)
    return cases


def load_fixture():
    """name -> dict(raw, stride, res, dims, bmin, bmax, occ{thr: (X, Y, Z) uint8})"""
    z = np.load(FIXTURE)
    out = {}
    for name in z["names"]:
        name = str(name)
        dims = tuple(int(d) for d in z[name + "_dims"])
        occ = {}
        for thr in THRESHOLDS:
            bits = z[f"{name}_occ_t{thr}"]
            occ[thr] = np.unpackbits(bits, count=int(np.prod(dims))).reshape(dims)
        out[name] = dict(raw=z[name + "_raw"], stride=int(z[name + "_stride"]), res=float(z[name + "_res"]), dims=dims,
                         bmin=z[name + "_bmin"], bmax=z[name + "_bmax"], occ=occ)
    return out
