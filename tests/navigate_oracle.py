"""Restatements of the closed-loop navigation calls (include/isdf.h): isdf_map_fuse_cloud's inside test, voxel index and counts on a 0 / 1
grid, and isdf_trajectory_shift's piece location and re-expansion, operation for operation in FP64 (Python floats round as the library's
-fmad=false unit does), so the library's bits can be compared exactly."""
from fractions import Fraction
from math import comb
import numpy as np


def grid_index(p, bmin, res, dims):
    """getGridIndex for points inside the frame (the library's grid_index): floor(((double)c - bmin) / res) clamped to the top index;
    the quirky "iy < 0 => ix = 0" branches cannot fire for such points"""
    idx = np.floor((np.asarray(p, dtype=np.float64) - np.asarray(bmin)) / res).astype(np.int64)
    return np.minimum(idx, np.asarray(dims) - 1)


def fuse(occ, bmin, bmax, res, cloud):
    """occ (X, Y, Z) 0 / 1 after fusing cloud ((n, k >= 3) float32) -> (new occ, dict of isdf_fuse_info counts)"""
    occ = np.array(occ, dtype=np.uint8, copy=True)
    c = np.asarray(cloud, dtype=np.float32)[:, :3]
    fin = np.all(np.isfinite(c), axis=1)
    cd = c.astype(np.float64)
    with np.errstate(invalid="ignore"):
        inside = fin & np.all((cd >= np.asarray(bmin)) & (cd <= np.asarray(bmax)), axis=1)
    idx = grid_index(cd[inside], bmin, res, occ.shape)
    before = int(occ.sum())
    occ[idx[:, 0], idx[:, 1], idx[:, 2]] = 1
    return occ, dict(points_used=int(inside.sum()), points_outside=int((fin & ~inside).sum()), points_skipped=int((~fin).sum()),
                     voxels_added=int(occ.sum()) - before)


def locate(T, t):
    """locatePieceIdx: (piece, local time) by sequential subtraction with a strict '>', clamped into the last piece"""
    i = 0
    while i < len(T) and t > T[i]:
        t -= T[i]
        i += 1
    if i == len(T):
        i -= 1
        t += T[i]
    return i, t


def _block(Cc, N):
    """one trajectory's 6N x 3 column-major block -> (N, 3, 6): piece, axis, coefficient of t^k"""
    return np.asarray(Cc, dtype=np.float64).reshape(3, N, 6).transpose(1, 0, 2)


def _unblock(c):
    return np.ascontiguousarray(np.asarray(c).transpose(1, 0, 2)).reshape(-1)


def reexpand(c, tau):
    """d_k = sum_{j=k..5} (C(j,k) c_j) tau^(j-k), accumulated from 0 in ascending j, tau^m the running product"""
    pw = [1.0]
    for m in range(1, 6):
        pw.append(pw[-1] * tau)
    out = []
    for k in range(6):
        d = 0.0
        for j in range(k, 6):
            d += (float(comb(j, k)) * float(c[j])) * pw[j - k]
        out.append(d)
    return out


def shift_one(T, Cc, t0):
    """isdf_trajectory_shift of one trajectory (T (N,), its 6N x 3 block) -> (T', block')"""
    T = [float(x) for x in T]
    N = len(T)
    D = 0.0
    for x in T:
        D += x
    if N == 0 or not (t0 >= 0.0 and t0 < D):
        return np.zeros(0), np.zeros(0)
    i, tau = locate(T, float(t0))
    blk = _block(Cc, N)
    pieces, durs = [], []
    if T[i] - tau > 0.0:
        pieces.append([reexpand(blk[i, a], tau) for a in range(3)])
        durs.append(T[i] - tau)
    for k in range(i + 1, N):
        pieces.append(blk[k])
        durs.append(T[k])
    if not pieces:
        return np.zeros(0), np.zeros(0)
    return np.array(durs), _unblock(np.array(pieces))


def shift(off, T, Cc, t0):
    """the ragged form: (out_off, T', coeffs')"""
    off = np.asarray(off, dtype=np.int64)
    oT, oC, oo = [], [], [0]
    for b in range(len(off) - 1):
        a, e = off[b], off[b + 1]
        tb, cb = shift_one(np.asarray(T)[a:e], np.asarray(Cc)[18 * a:18 * e], float(np.asarray(t0)[b]))
        oT.append(tb)
        oC.append(cb)
        oo.append(oo[-1] + len(tb))
    return np.array(oo, dtype=np.int32), np.concatenate(oT) if oT else np.zeros(0), np.concatenate(oC) if oC else np.zeros(0)


def reexpand_exact(c, tau):
    """the same re-expansion in exact rational arithmetic"""
    t = Fraction(tau)
    return [sum(comb(j, k) * Fraction(float(c[j])) * t ** (j - k) for j in range(k, 6)) for k in range(6)]


def log_to_init(records):
    """isdf_simulate log records (..., 21: t pos vel quat omega rpm cmd_pos) -> initial states (..., 17: pos vel quat omega rpm)"""
    return np.asarray(records)[..., 1:18]
