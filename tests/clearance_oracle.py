"""Serial FP64 restatement of the trajectory clearance check (include/isdf.h, isdf_trajectory_clearance) — TEST INFRASTRUCTURE.

Brute force: every pose sample is tested against EVERY occupied voxel of the map with the body-frame box test |R^T (c - x)|_inf <= H,
so nothing here shares the kernel's windowing (rotated-box AABB, map clipping, bit-grid scan) or its culls and bounded searches. Poses
are the oracle's (grazing.sample_poses: the piece polynomial evaluated directly, the oracle's flatness map, Eigen's quaternion formula);
SDFs are the oracle's shapes (getonlySDF), or any callable sdf(prel) -> values (the library's own unculled isdf_shape_query for
winding-sign meshes, whose hierarchical winding number the oracle does not replicate)."""
import ctypes as C
import numpy as np
import oracle_lib as O
import grazing as G


def poses(ocfg, T, coeffs, K_c):
    """(pos (S,3), R (S,3,3)) of the N*(K_c+1) samples, sample i*(K_c+1)+j"""
    oc = O.OrcConfig()
    C.memmove(C.byref(oc), C.byref(ocfg), C.sizeof(oc))
    oc.integral_intervs = int(K_c)
    pos, R, _, _ = G.sample_poses(oc, T, coeffs)
    return pos, R


def occupied(occ, bmin, res):
    """flat addresses (ix*Y*Z + iy*Z + iz) and centres (getGridCubeCenter) of every occupied voxel"""
    occ = np.asarray(occ)
    ids = np.flatnonzero(occ.reshape(-1))
    I3 = np.stack(np.unravel_index(ids, occ.shape), axis=1)
    return ids.astype(np.int64), (I3 + 0.5) * res + np.asarray(bmin, float)


def clearance(ocfg, occ, bmin, res, sdf, T, coeffs, K_c, reach, margin, N0=0, keep_candidates=False):
    """sdf: an oracle Shape (getonlySDF) or a callable prel (n,3) -> sdf (n,). Returns dict(clear, voxel, summary[, candidates]):
    per-sample clearance and witness, one summary dict per trajectory, and with keep_candidates the (addresses, sdf) of every
    sample's candidates."""
    f = sdf if callable(sdf) else (lambda p: sdf.query(p, what=0)[0])
    T = np.asarray(T, float).reshape(-1)
    N, K = T.size, int(K_c)
    H = ocfg.kernel_size * ocfg.occupancy_resolution / 2 + reach
    pos, R = poses(ocfg, T, coeffs, K)
    ids, ctr = occupied(occ, bmin, res)
    S = N * (K + 1)
    clear, voxel, cands = np.full(S, float(reach)), np.full(S, -1, dtype=np.int64), []
    for s in range(S):
        prel = (ctr - pos[s]) @ R[s]                              # R^T (c - x), row-vector form
        m = ~np.any(np.abs(prel) > H, axis=1)
        cid, v = ids[m], (f(prel[m]) if m.any() else np.zeros(0))
        if keep_candidates:
            cands.append((cid, v))
        if v.size and v.min() < reach:
            clear[s] = v.min()
            voxel[s] = cid[v == v.min()].min()
    out = dict(clear=clear, voxel=voxel, summary=summaries(T, clear, voxel, K, margin, N0))
    if keep_candidates:
        out["candidates"] = cands
    return out


def summaries(T, clear, voxel, K, margin, N0=0):
    """per-trajectory summary from per-sample results, in (piece, j) order"""
    T = np.asarray(T, float).reshape(-1)
    N = T.size
    N0 = N if N0 == 0 else N0
    per = N0 * (K + 1)
    out = []
    for b in range(N // N0):
        c = clear[b * per:(b + 1) * per]

        def ttime(k):
            p, j = divmod(int(k), K + 1)
            t = 0.0
            for q in range(p):
                t += T[b * N0 + q]
            return t + j * (T[b * N0 + p] * (1.0 / K))
        m = int(np.argmin(c))                                     # first attaining sample
        hit = np.flatnonzero(c < margin)
        out.append(dict(min_clearance=float(c[m]), t_min=ttime(m), first_hit=ttime(hit[0]) if hit.size else -1.0,
                        voxel_min=int(voxel[b * per + m]), piece_min=m // (K + 1), sample_min=m % (K + 1),
                        colliding_samples=int(hit.size), collision_free=int(hit.size == 0)))
    return out
