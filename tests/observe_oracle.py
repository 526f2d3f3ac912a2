"""Known space (include/isdf.h, isdf_map_observe / isdf_map_mark_known) restated in numpy — TEST INFRASTRUCTURE.

  voxel_span(bmin, res, i)                     the padded closed cube of index i on one axis (lo, hi)
  mip(img)                                     the min-mip of one depth image: a list of levels, level 0 the image
  observe(img, cw, body, p, bmin, res, dims)   the voxels pose's image marks known (X, Y, Z) bool; cw: the render's camera-from-world as
                                               sense_oracle.pose returns it (FP32 entries widened to double[16])
  mark_boxes(boxes, bmin, res, dims)           the voxels isdf_map_mark_known marks (their unpadded cubes inside a box)

Every FP64 operation is the kernel's, in the kernel's order (numpy rounds each one, nothing is contracted), so the results are the same bits.
"""
import numpy as np


def voxel_span(bmin, res, i):
    i = np.asarray(i, dtype=np.float64)
    pad = 1e-12 * (abs(bmin) + (i + 1.0) * res)
    return (bmin + i * res) - pad, (bmin + (i + 1.0) * res) + pad


def mip(img):
    levels = [np.asarray(img, dtype=np.int64)]
    while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
        a = levels[-1]
        h, w = a.shape
        b = np.full((h + (h & 1), w + (w & 1)), np.iinfo(np.int64).max, dtype=np.int64)
        b[:h, :w] = a
        levels.append(b.reshape(b.shape[0] // 2, 2, b.shape[1] // 2, 2).min(axis=(1, 3)))
    return levels


def box_lo(body, horizon, bmin, res):
    return int(max(-2147483000.0, min(2147483000.0, np.floor(((body - horizon) - bmin) / res) - 1.0)))


def observe(img, cw, body, p, bmin, res, dims):
    """the four-part rule for every voxel of the map in the pose's horizon box"""
    h = float(p.sensing_horizon)
    W, H = int(p.width), int(p.height)
    fx, fy, cx, cy = (float(np.float32(v)) for v in (p.fx, p.fy, p.cx, p.cy))
    cw = np.asarray(cw, dtype=np.float64).reshape(4, 4)
    r, t = cw[:3, :3], cw[:3, 3]
    D = int(np.ceil(2.0 * h / res)) + 3
    out = np.zeros(dims, dtype=bool)
    rng = []
    for a in range(3):
        lo = box_lo(float(body[a]), h, float(bmin[a]), res)
        rng.append(np.arange(max(lo, 0), min(lo + D, dims[a])))
    if any(len(x) == 0 for x in rng):
        return out
    I = np.meshgrid(*rng, indexing="ij")
    lo, hi = [], []
    for a in range(3):
        l_, h_ = voxel_span(float(bmin[a]), res, I[a].astype(np.float64))
        lo.append(l_); hi.append(h_)
    with np.errstate(all="ignore"):
        ok = np.ones(I[0].shape, dtype=bool)
        corners = [[(hi[0] if k & 1 else lo[0]), (hi[1] if k & 2 else lo[1]), (hi[2] if k & 4 else lo[2])] for k in range(8)]
        for c in corners:
            d0, d1, d2 = c[0] - body[0], c[1] - body[1], c[2] - body[2]
            ok &= np.sqrt((d0 * d0 + d1 * d1) + d2 * d2) <= h
        M = np.zeros(I[0].shape)
        for a in range(3):
            M = np.maximum(M, np.maximum(np.abs(lo[a]), np.abs(hi[a])))
        E = []
        for i in range(3):
            e = 1e-6 * (((abs(r[i, 0]) + abs(r[i, 1])) + abs(r[i, 2])) * M + abs(t[i])) + 1e-30
            ok &= e < 1e24
            E.append(e)
        cam = [[((r[i, 0] * c[0] + r[i, 1] * c[1]) + r[i, 2] * c[2]) + t[i] for i in range(3)] for c in corners]
        z = np.stack([cc[2] for cc in cam])
        zmin, zmax = z.min(axis=0), z.max(axis=0)
        ok &= zmin > E[2]
        qx = np.stack([cc[0] / cc[2] for cc in cam])
        qy = np.stack([cc[1] / cc[2] for cc in cam])
        u, v = qx * fx + cx, qy * fy + cy
        a_, b_ = np.abs(qx).max(axis=0), np.abs(qy).max(axis=0)
        zl = zmin - E[2]
        dqx, dqy = (E[0] + a_ * E[2]) / zl, (E[1] + b_ * E[2]) / zl
        eu = (fx * dqx + 1.2e-7 * ((a_ + dqx) * fx + abs(cx))) + 1e-9 * (1.0 + (a_ * fx + abs(cx)))
        ev = (fy * dqy + 1.2e-7 * ((b_ + dqy) * fy + abs(cy))) + 1e-9 * (1.0 + (b_ * fy + abs(cy)))
        fx0, fx1 = np.floor((u.min(axis=0) - eu) + 0.5), np.floor((u.max(axis=0) + eu) + 0.5)
        fy0, fy1 = np.floor((v.min(axis=0) - ev) + 0.5), np.floor((v.max(axis=0) + ev) + 0.5)
        ok &= (fx0 >= 0.0) & (fx1 <= W - 1) & (fy0 >= 0.0) & (fy1 <= H - 1)
    idx = np.nonzero(ok)
    if len(idx[0]) == 0:
        return out
    x0, x1, y0, y1 = (a[idx].astype(np.int64) for a in (fx0, fx1, fy0, fy1))
    levels = mip(img)
    lvl = np.full(x0.shape, -1)
    for l in range(len(levels)):
        fit = (lvl < 0) & ((x1 >> l) - (x0 >> l) <= 1) & ((y1 >> l) - (y0 >> l) <= 1)
        lvl[fit] = l
    dmin = np.empty(x0.shape, dtype=np.int64)
    for l, L in enumerate(levels):
        m = lvl == l
        if not m.any():
            continue
        i0, i1, j0, j1 = x0[m] >> l, x1[m] >> l, y0[m] >> l, y1[m] >> l
        dmin[m] = np.minimum(np.minimum(L[j0, i0], L[j0, i1]), np.minimum(L[j1, i0], L[j1, i1]))
    zx, e2 = zmax[idx], E[2][idx]
    d = (1000.0 * e2 + 0.5) + 1.2e-7 * (1000.0 * (zx + e2) + 1.0)
    known = dmin.astype(np.float64) > 1000.0 * zx + d
    sel = tuple(I[a][idx][known] for a in range(3))
    out[sel] = True
    return out


def observe_many(images, cws, bodies, p, bmin, res, dims):
    out = np.zeros(dims, dtype=bool)
    for img, cw, body in zip(images, cws, bodies):
        out |= observe(img, cw, body, p, bmin, res, dims)
    return out


def tested(bodies, horizon, bmin, res, dims):
    """info.voxels_tested: the in-map voxels of every pose's index box"""
    D = int(np.ceil(2.0 * horizon / res)) + 3
    n = 0
    for body in bodies:
        k = 1
        for a in range(3):
            lo = box_lo(float(body[a]), horizon, float(bmin[a]), res)
            k *= max(0, min(lo + D, dims[a]) - max(lo, 0))
        n += k
    return n


def mark_boxes(boxes, bmin, res, dims):
    out = np.zeros(dims, dtype=bool)
    spans = [(bmin[a] + np.arange(dims[a], dtype=np.float64) * res, bmin[a] + (np.arange(dims[a], dtype=np.float64) + 1.0) * res) for a in range(3)]
    for b in np.asarray(boxes, dtype=np.float64).reshape(-1, 6):
        ins = [(spans[a][0] >= b[a]) & (spans[a][1] <= b[3 + a]) for a in range(3)]
        out |= ins[0][:, None, None] & ins[1][None, :, None] & ins[2][None, None, :]
    return out
