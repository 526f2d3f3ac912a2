"""The map's distance field (include/isdf.h, isdf_map_esdf) restated exactly, and the reference-compiled one — TEST INFRASTRUCTURE.

  exact_d2(sites)                     the exact integer squared voxel distance to the nearest site (scipy's nearest-site indices, int64 d2);
                                      None when there is no site
  field(sites, res)                   res * sqrt((double)d2), res * sqrt(DBL_MAX) without a site: POSITIVE with sites = occupied, NEGATIVE
                                      with sites = free
  signed(pos, neg, res)               ISDF_ESDF_SIGNED: pos, plus (-neg + res) where neg > 0
  query(values, bmin, bmax, res, pts) getSDFValueWithGrad / getSDFValue (GridMap3D.h:114-193) restated in numpy float64, operation for
                                      operation (numpy contracts nothing, so it rounds like the reference's no-FMA x86-64 build)
  ref_esdf / ref_query                oracle/_ref/libref_esdf.so (oracle/esdf.mk): the reference's own generateESDF3d and queries
  load_golden()                       tests/golden/esdf_reference.npz (tests/golden/make_esdf_golden.py), reference outputs for hosts
                                      without the reference tree
"""
import ctypes as C
import os
import subprocess
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_DIR = os.path.join(os.path.dirname(HERE), "oracle")
REF_ESDF = os.path.join(ORACLE_DIR, "_ref", "libref_esdf.so")
GOLDEN = os.path.join(HERE, "golden", "esdf_reference.npz")
FIELDS = {"positive": 0, "negative": 1, "signed": 2}
DBL_MAX = np.finfo(np.float64).max


def build(force=False):
    """make's own dependency check decides (oracle/esdf.mk); without the reference tree it keeps whatever library exists"""
    subprocess.call(["make", "-C", ORACLE_DIR, "-f", "esdf.mk"] + (["-B"] if force else []), stdout=subprocess.DEVNULL)


def exact_d2(sites):
    from scipy import ndimage
    sites = np.asarray(sites, dtype=bool)
    if not sites.any():
        return None
    idx = ndimage.distance_transform_edt(~sites, return_distances=False, return_indices=True)
    g = np.indices(sites.shape)
    return sum((idx[k].astype(np.int64) - g[k]) ** 2 for k in range(3))


def field_from_d2(d2, shape, res):
    if d2 is None:
        return np.full(shape, res * np.sqrt(DBL_MAX))
    return res * np.sqrt(d2.astype(np.float64))


def field(sites, res):
    return field_from_d2(exact_d2(sites), np.shape(sites), res)


def signed(pos, neg, res):
    v = pos.copy()
    m = neg > 0.0
    v[m] += (-neg[m] + res)
    return v


def fields(occ, res):
    """{"positive", "negative", "signed"} of an occupancy grid"""
    occ = np.asarray(occ) != 0
    pos, neg = field(occ, res), field(~occ, res)
    return {"positive": pos, "negative": neg, "signed": signed(pos, neg, res)}


def query(values, bmin, bmax, res, pts, grad=True):
    """getSDFValueWithGrad (grad=True: (dist, grad)) or getSDFValue (dist) on one field's X x Y x Z values; finite points only"""
    values = np.asarray(values, dtype=np.float64)
    X, Y, Z = values.shape
    dims = np.array([X, Y, Z])
    bmin, bmax = np.asarray(bmin, dtype=np.float64), np.asarray(bmax, dtype=np.float64)
    p = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    pm = p - 0.5 * res * 1.0
    inside = np.all(~(pm < bmin) & ~(pm > bmax), axis=1)
    # getGridIndex: floor, clamped to the top index; its "iy < 0 => ix = 0" branches cannot fire for pm >= bmin
    with np.errstate(invalid="ignore"):
        idx = np.floor((pm - bmin) / res).astype(np.int64)
    idx = np.minimum(idx, dims - 1)
    idx[~inside] = 0
    centre = (idx + 0.5) * res + bmin
    inv = 1.0 / res
    diff = (p - centre) * inv
    v = np.zeros((p.shape[0], 2, 2, 2))
    for x in range(2):
        for y in range(2):
            for z in range(2):
                j = idx + np.array([x, y, z])
                ok = np.all(j < dims, axis=1)
                jj = np.minimum(j, dims - 1)
                v[:, x, y, z] = np.where(ok, values[jj[:, 0], jj[:, 1], jj[:, 2]], 0.0)
    d0, d1, d2 = diff[:, 0], diff[:, 1], diff[:, 2]
    v00 = (1 - d0) * v[:, 0, 0, 0] + d0 * v[:, 1, 0, 0]
    v01 = (1 - d0) * v[:, 0, 0, 1] + d0 * v[:, 1, 0, 1]
    v10 = (1 - d0) * v[:, 0, 1, 0] + d0 * v[:, 1, 1, 0]
    v11 = (1 - d0) * v[:, 0, 1, 1] + d0 * v[:, 1, 1, 1]
    v0 = (1 - d1) * v00 + d1 * v10
    v1 = (1 - d1) * v01 + d1 * v11
    dist = (1 - d2) * v0 + d2 * v1
    if not grad:
        return dist
    g = np.empty((p.shape[0], 3))
    g[:, 2] = (v1 - v0) * inv
    g[:, 1] = ((1 - d2) * (v10 - v00) + d2 * (v11 - v01)) * inv
    g0 = (1 - d2) * (1 - d1) * (v[:, 1, 0, 0] - v[:, 0, 0, 0])
    g0 = g0 + (1 - d2) * d1 * (v[:, 1, 1, 0] - v[:, 0, 1, 0])
    g0 = g0 + d2 * (1 - d1) * (v[:, 1, 0, 1] - v[:, 0, 0, 1])
    g0 = g0 + d2 * d1 * (v[:, 1, 1, 1] - v[:, 0, 1, 1])
    g[:, 0] = g0 * inv
    return dist, g


# ---- the reference-compiled field (oracle/_ref/libref_esdf.so) ----
_lib = None


def ref_available():
    return os.path.exists(REF_ESDF)


def _ref():
    global _lib
    if _lib is None:
        L = C.CDLL(REF_ESDF)
        u8, dp = C.POINTER(C.c_uint8), C.POINTER(C.c_double)
        L.ref_grid_esdf.argtypes = [u8, C.c_int, C.c_int, C.c_int, dp, dp, C.c_double, dp, dp, dp]
        L.ref_grid_sdf_query.argtypes = [u8, C.c_int, C.c_int, C.c_int, dp, dp, C.c_double, C.c_int, C.c_int, dp, dp, dp]
        _lib = L
    return _lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None else None


def _frame(occ, bmin, bmax, res):
    occ = np.ascontiguousarray(np.asarray(occ) != 0, dtype=np.uint8)
    bmin = np.ascontiguousarray(bmin, dtype=np.float64).reshape(3)
    bmax = (bmin + np.array(occ.shape) * res) if bmax is None else np.ascontiguousarray(bmax, dtype=np.float64).reshape(3)
    return occ, bmin, np.ascontiguousarray(bmax, dtype=np.float64)


def ref_esdf(occ, bmin, res, bmax=None):
    """(grid_esdf, grid_map_buffer_neg, grid_map_buffer_all) of the reference's generateESDF3d; bmax defaults to bmin + dims * res"""
    occ, bmin, bmax = _frame(occ, bmin, bmax, res)
    X, Y, Z = occ.shape
    pos, neg, al = np.empty(occ.shape), np.empty(occ.shape), np.empty(occ.shape)
    r = _ref().ref_grid_esdf(occ.ctypes.data_as(C.POINTER(C.c_uint8)), X, Y, Z, _dp(bmin), _dp(bmax), float(res), _dp(pos), _dp(neg), _dp(al))
    assert r == 0, "createGridMap(bmin, bmax) does not give back the map's dimensions"
    return pos, neg, al


def ref_query(occ, bmin, res, field, pts, grad=True, bmax=None):
    occ, bmin, bmax = _frame(occ, bmin, bmax, res)
    X, Y, Z = occ.shape
    p = np.ascontiguousarray(pts, dtype=np.float64).reshape(-1, 3)
    n = p.shape[0]
    dist = np.empty(n)
    g = np.empty((n, 3)) if grad else None
    r = _ref().ref_grid_sdf_query(occ.ctypes.data_as(C.POINTER(C.c_uint8)), X, Y, Z, _dp(bmin), _dp(bmax), float(res), FIELDS[field], n,
                                  _dp(p), _dp(dist), _dp(g))
    assert r == 0
    return (dist, g) if grad else dist


def load_golden():
    """{case name: dict(occ, bmin, bmax, res, positive, negative, all, pts, and per field f: f_dist, f_grad, f_value)}"""
    z = np.load(GOLDEN)
    names = [str(s) for s in z["names"]]
    out = {}
    for nm in names:
        d = {k[len(nm) + 1:]: z[k] for k in z.files if k.startswith(nm + "/")}
        d["occ"] = np.unpackbits(d.pop("occ_bits"), count=int(np.prod(d["dims"]))).reshape(tuple(d["dims"])).astype(np.uint8)
        d["res"] = float(d["res"])
        out[nm] = d
    return out
