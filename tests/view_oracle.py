"""The view gain (include/isdf.h, isdf_view_gain) restated in numpy — TEST INFRASTRUCTURE.

  in_view(pos, quat, cam, bmin, res, dims)          (b) for one camera: isdf_map_observe's rules 2, 1 and 3 (observe_oracle.observe on an
                                                    image where nothing is seen, whose rule 4 then always holds), with sense_oracle's
                                                    transform of the pose
  line(s, v)                                        the voxels strictly between s and v on (c)'s integer line
  line_clear(occ, s, vox)                           (c) for the voxels vox (n, 3): no occupied in-map voxel on the line from s
  view_set(occ, known, pos, quat, cams, bmin, res)  the voxels that count toward the gain of one pose: (a), (b) for some camera, (c)
  gain(...)                                         their number
  pose_voxel(pos, bmin, res)                        s = floor((pos - bmin) / res) in FP64
"""
import numpy as np
import observe_oracle as OO
import sense_oracle as SO

NOTHING_SEEN = 999999


def pose_voxel(pos, bmin, res):
    return np.floor((np.asarray(pos, dtype=np.float64) - np.asarray(bmin, dtype=np.float64)) / res).astype(np.int64)


def in_view(pos, quat, cam, bmin, res, dims):
    # with every pixel at 999999, rule 4 holds for every corner depth below ~999 m: the rule reduces to rules 2, 1 and 3
    assert cam.sensing_horizon < 900.0 and np.isfinite(cam.sensing_horizon)
    _, cw = SO.pose(np.asarray(pos, dtype=np.float64), np.asarray(quat, dtype=np.float64), np.array(cam.cam_to_body[:]))
    img = np.full((cam.height, cam.width), NOTHING_SEEN, dtype=np.int32)
    return OO.observe(img, cw, np.asarray(pos, dtype=np.float64), cam, np.asarray(bmin, dtype=np.float64), res, tuple(dims))


def _floordiv(a, b):
    return np.floor_divide(a, b)   # numpy's integer floor division rounds toward -inf, as the definition asks


def line(s, v):
    """the voxels s + floor((2 k d + m) / (2 m)), k = 1 .. m - 1, d = v - s, m = max |d_a|: (m - 1, 3) int64"""
    s, v = np.asarray(s, dtype=np.int64), np.asarray(v, dtype=np.int64)
    d = v - s
    m = int(np.abs(d).max())
    k = np.arange(1, m, dtype=np.int64)[:, None]
    return s + _floordiv(2 * k * d + m, 2 * m) if m > 1 else np.zeros((0, 3), dtype=np.int64)


def line_clear(occ, s, vox):
    occ = np.asarray(occ).astype(bool)
    s, vox = np.asarray(s, dtype=np.int64), np.asarray(vox, dtype=np.int64).reshape(-1, 3)
    d = vox - s
    m = np.abs(d).max(axis=1) if len(vox) else np.zeros(0, dtype=np.int64)
    ok = np.ones(len(vox), dtype=bool)
    mm = np.maximum(m, 1)
    for k in range(1, int(m.max()) if len(vox) else 0):
        live = k < m
        p = s + _floordiv(2 * k * d + mm[:, None], 2 * mm[:, None])
        inside = live & np.all((p >= 0) & (p < np.array(occ.shape)), axis=1)
        hit = np.zeros(len(vox), dtype=bool)
        q = p[inside]
        hit[inside] = occ[q[:, 0], q[:, 1], q[:, 2]]
        ok &= ~hit
    return ok


def view_set(occ, known, pos, quat, cams, bmin, res):
    occ = np.asarray(occ).astype(bool)
    known = np.zeros_like(occ) if known is None else np.asarray(known).astype(bool)
    cams = list(cams) if isinstance(cams, (list, tuple)) else [cams]
    seen = np.zeros(occ.shape, dtype=bool)
    for cam in cams:
        seen |= in_view(pos, quat, cam, bmin, res, occ.shape)
    cand = seen & ~occ & ~known
    vox = np.argwhere(cand)
    out = np.zeros(occ.shape, dtype=bool)
    if len(vox):
        ok = line_clear(occ, pose_voxel(pos, bmin, res), vox)
        out[tuple(vox[ok].T)] = True
    return out


def gain(occ, known, pos, quat, cams, bmin, res):
    return int(view_set(occ, known, pos, quat, cams, bmin, res).sum())


def gains(occ, known, pos, quat, cams, bmin, res):
    """the gains of Q poses (pos (Q, 3), quat (Q, 4)) -> (Q,) int64"""
    pos, quat = np.asarray(pos, dtype=np.float64).reshape(-1, 3), np.asarray(quat, dtype=np.float64).reshape(-1, 4)
    return np.array([gain(occ, known, p, q, cams, bmin, res) for p, q in zip(pos, quat)], dtype=np.int64)
