"""Candidate-list lengths and list passes per mesh query of the discrete scan: for the full cell lists (every triangle within
d_c + 2 hd of the cell centre) and for the sub-box filtered lists the scan walks, the Lipschitz rule applied on k^3 sub-boxes of each
cell (k_mesh_disc_lists, k = DISC_LIST_K = 4 in the library; DESIGN §3.1).

A numpy restatement on the CPU, no GPU needed: the mesh, its cell grid and both list rules are recomputed from bench.py's workload
(the 3900-triangle rounded cone at bench.py's pose and safety margin), and the list pass of list_closest_pre is replayed for a seeded
sample of body-frame query points. The bench's queries are occupied voxel centres (5 % Bernoulli occupancy) seen from poses spread
over the whole map, so in the body frame they are close to uniform; the sample is uniform over the box every query can come from
(the mesh AABB inflated by the safety margin), culled as the scan culls (cell-centre distance minus ghd at least safety_hor). The
map's wall slabs are not modelled. Lists are computed only for the cells the sample lands in.

With --device the mesh is also built by the library on cuda:0, and the cells the sample lands in are compared with the library's
cell distances, list lengths and lower bounds (the restatement of the unfiltered lists is exact when all three agree).

Prints one JSON line per k (sub-boxes per cell edge; k = 1 is the unfiltered rule): list-length histograms over the sampled cells,
mean passes (32 candidates each) and candidate records tested per query answered from a list, and the number of queries answered
from the tree (cells whose list exceeds the cap; with k > 1 such a cell is listed when its filtered list fits under the cap).
Writes nothing."""
import argparse
import json
import os
import sys

import numpy as np

sys.dont_write_bytecode = True   # the imports of bench.py and workloads.py below leave no cache in the tree
ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))

CAP, CAP_DISCRETE = 160, 512   # MESH_LIST_CAP, MESH_LIST_CAP_DISCRETE
FILTER_MIN = 32                 # lists this short take one pass already: not filtered


def tri_dist2(P, A, AB, AC):
    """squared distance of every point P[i] to every triangle (A[j], A[j] + AB[j], A[j] + AC[j]): Ericson's regions, as tri_closest"""
    ap = P[:, None, :] - A[None]
    bp, cp = ap - AB[None], ap - AC[None]
    dot = lambda u, v: np.einsum("...k,...k->...", u, v)
    ab, ac = AB[None], AC[None]
    d1, d2, d3, d4, d5, d6 = dot(ab, ap), dot(ac, ap), dot(ab, bp), dot(ac, bp), dot(ab, cp), dot(ac, cp)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    e43, e56 = d4 - d3, d5 - d6
    with np.errstate(divide="ignore", invalid="ignore"):
        den = 1.0 / (va + vb + vc)
        s, t = vb * den, vc * den
        tab, tac, tbc = d1 / (d1 - d3), d2 / (d2 - d6), e43 / (e43 + e56)
    for cond, ss, tt in [((va <= 0) & (e43 >= 0) & (e56 >= 0), 1.0 - tbc, tbc), ((vb <= 0) & (d2 >= 0) & (d6 <= 0), 0.0, tac),
                         ((d6 >= 0) & (d5 <= d6), 0.0, 1.0), ((vc <= 0) & (d1 >= 0) & (d3 <= 0), tab, 0.0),
                         ((d3 >= 0) & (d4 <= d3), 1.0, 0.0), ((d1 <= 0) & (d2 <= 0), 0.0, 0.0)]:
        s, t = np.where(cond, ss, s), np.where(cond, tt, t)
    q = A[None] + s[..., None] * ab + t[..., None] * ac
    e = P[:, None, :] - q
    return dot(e, e)


def winding(P, A, B, C):
    """generalised winding number of the closed mesh at each point (exact solid-angle sum)"""
    a, b, c = A[None] - P[:, None], B[None] - P[:, None], C[None] - P[:, None]
    la, lb, lc = (np.linalg.norm(x, axis=2) for x in (a, b, c))
    num = np.einsum("ijk,ijk->ij", a, np.cross(b, c))
    den = la * lb * lc + np.einsum("ijk,ijk->ij", a, b) * lc + np.einsum("ijk,ijk->ij", b, c) * la + np.einsum("ijk,ijk->ij", c, a) * lb
    return (2.0 * np.arctan2(num, den)).sum(axis=1) / (4.0 * np.pi)


def f32_down(x):
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(-np.inf)), f)


class Grid:
    def __init__(self, V, F, sf):
        self.A, B, C = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
        self.B, self.C = B, C
        self.AB, self.AC = B - self.A, C - self.A
        self.sf = sf
        blo, bhi = V.min(0), V.max(0)
        pad = 2.0 * sf + 0.1
        ext = float(np.max(bhi - blo + 2 * pad))
        self.gcell = max(0.1, ext / 160.0)
        self.glo = blo - pad
        self.gdim = np.ceil((bhi - blo + 2 * pad) / self.gcell).astype(int) + 1
        self.hd = 0.5 * np.sqrt(3.0) * self.gcell
        self.ghd = self.hd * (1.0 + 1e-6) + 1e-5 * max(1.0, ext)
        self.blo, self.bhi = blo, bhi
        self.sign_radius = sf if 2.0 * self.hd < 0.9 * sf else 0.0
        self.cells = {}

    def centre(self, ijk):
        return self.glo + (np.asarray(ijk) + 0.5) * self.gcell

    def cell(self, ijk, k):
        """(cell distance, full list, filtered list); a list is (triangle ids, float lower bounds), None = no list"""
        key = (tuple(ijk), k)
        if key in self.cells:
            return self.cells[key]
        c = self.centre(ijk)
        d2 = tri_dist2(c[None], self.A, self.AB, self.AC)[0]
        dmag = np.sqrt(d2.min())
        inside = winding(c[None], self.A, self.B, self.C)[0] > 0.5
        dc = float(np.float32(-dmag if inside else dmag))
        R = (abs(dc) + (self.ghd - self.hd) + 2.0 * self.hd) * (1.0 + 1e-9) + 1e-12
        hit = np.nonzero(d2 <= R * R)[0]
        order = hit[np.lexsort((hit, d2[hit]))]
        cap = CAP_DISCRETE if dc + self.ghd < self.sf else CAP
        full = filt = None
        lst = (order, f32_down(np.maximum(np.sqrt(d2[order]) * (1.0 - 1e-9) - 1e-12, 0.0)))
        if len(order) <= cap:
            full = filt = lst
        if k > 1 and len(order) > FILTER_MIN and (full is not None or cap == CAP_DISCRETE):
            # a cell past the discrete cap gets a filtered list when the result fits under it
            keep = self.keep(c, order, k)
            if keep.sum() <= cap:
                filt = (lst[0][keep], lst[1][keep])
        self.cells[key] = (dc, full, filt)
        return self.cells[key]

    def keep(self, c, ids, k):
        """the sub-box rule: keep T if d(y, T) <= dmin(y) + 2 delta for some sub-box centre y (with the build's slack)"""
        he = self.gcell / (2 * k) * (1.0 + 1e-9) + 1e-12
        delta = np.sqrt(3.0) * he
        u = (np.arange(k) + 0.5) / k - 0.5
        Y = c + self.gcell * np.stack(np.meshgrid(u, u, u, indexing="ij"), -1).reshape(-1, 3)
        D = np.sqrt(tri_dist2(Y, self.A[ids], self.AB[ids], self.AC[ids]))
        dmin = D.min(axis=1, keepdims=True)
        keep = (D <= (dmin + 2.0 * delta) * (1.0 + 1e-9) + 1e-12).any(axis=0)
        keep[0] = True
        return keep


def replay(G, p, ijk, lst, bound2):
    """list_closest_pre's passes and tested records for query p on list (ids, lbs)"""
    ids, lbs = lst
    c = G.centre(ijk)
    r_up = np.linalg.norm(p - c) * (1.0 + 1e-9) + 1e-12
    dd = tri_dist2(p[None], G.A[ids], G.AB[ids], G.AC[ids])[0]
    prunes = lambda lb, best: (lb - r_up > 0.0) & ((lb - r_up) ** 2 > best)
    ub = float(lbs[0]) * (1.0 + 1e-6) + 1e-9 + r_up
    best = min(bound2, ub * ub)
    passes = recs = 0
    n = len(ids)
    for base in range(0, n, 32):
        lb = lbs[base:base + 32].astype(np.float64)
        test = ~prunes(lb, best)
        passes += 1
        recs += int(test.sum())
        if test.any():
            best = min(best, float(dd[base:base + 32][test].min()))
        if base + 32 < n and prunes(float(lbs[base + 32]), best):
            break
    return passes, recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=4000)
    ap.add_argument("--ks", default="1,2,3,4")
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--device", action="store_true", help="also build the mesh on cuda:0 and compare the sampled cells' distances and "
                    "lists with the library's (isdf_dbg_mesh_grid / isdf_dbg_mesh_lists)")
    a = ap.parse_args()
    import workloads as W
    import bench as B
    import isdf_b200 as I
    w = B.WORKLOAD
    V0, F = W.rounded_cone_mesh()
    R, t = W.rotation_from_poly_params(w["poly_params"])
    V = np.asarray(V0, dtype=np.float64) @ np.asarray(R).T + np.asarray(t)
    F = np.asarray(F)
    sf = I.default_config_values().safety_hor
    G = Grid(V, F, sf)
    rng = np.random.default_rng(a.seed)
    lo, hi = G.blo - sf, G.bhi + sf
    # sample until enough queries survive the cull (deep cells, d_c + ghd <= -sf, search unbounded: bound2 = 1e300)
    queries = []
    while len(queries) < a.queries:
        p = lo + (hi - lo) * rng.random(3)
        ijk = np.floor((p - G.glo) / G.gcell).astype(int)
        dc = G.cell(ijk, 1)[0]
        if dc - G.ghd >= sf:
            continue
        bounded = G.sign_radius > 0.0 and sf >= G.sign_radius
        deep = dc + G.ghd <= -sf
        queries.append((p, ijk, sf * sf if bounded and not deep else 1e300))
    for k in [int(x) for x in a.ks.split(",")]:
        P, Rc, tree, seen = [], [], 0, {}
        for p, ijk, b2 in queries:
            dc, full, filt = G.cell(ijk, k)
            if filt is None:
                tree += 1
                continue
            seen[tuple(ijk)] = len(filt[0])
            ps, rs = replay(G, p, ijk, filt, b2)
            P.append(ps); Rc.append(rs)
        lens = list(seen.values())
        edges = [0, 32, 64, 128, 160, 256, 384, 512]
        hist = np.histogram(lens, bins=edges + [10 ** 6])[0].tolist()
        print(json.dumps({"k": k, "queries": len(queries), "tree_queries": tree, "passes_per_query": float(np.mean(P)),
                          "one_pass_share": float(np.mean(np.asarray(P) == 1)),
                          "records_per_query": float(np.mean(Rc)), "cells": len(lens), "mean_list_len": float(np.mean(lens)),
                          "list_len_hist": dict(zip([f">={e}" for e in edges], hist))}))
    if a.device:
        ev = I.Evaluator(I.default_config_values(), device=0)
        ev.set_shape_mesh(V0, F, w["poly_params"])
        grid, lists = ev.dbg_mesh_grid(), ev.dbg_mesh_lists()
        ev.close()
        geom_ok = bool(np.allclose(grid["glo"], G.glo, rtol=0, atol=1e-12) and grid["gcell"] == G.gcell and grid["gdim"] == tuple(G.gdim))
        cells = {tuple(ijk): G.cell(ijk, 1) for _, ijk, _ in queries}   # the cells queries land in
        cnt_diff, dc_diff, lb_diff = 0, 0.0, 0.0
        for ijk, (dc, full, _) in cells.items():
            dc_diff = max(dc_diff, abs(float(grid["cell_dist"][ijk]) - dc))
            n = int(grid["cell_cnt"][ijk])
            if n != (0 if full is None else len(full[0])):
                cnt_diff += 1
            elif n:
                off = int(lists["cell_off"][ijk])
                lb_diff = max(lb_diff, float(np.max(np.abs(lists["cand_lb"][off:off + n].astype(np.float64) - full[1]) / np.maximum(full[1], 1e-6))))
        print(json.dumps({"device_check": {"grid_equal": geom_ok, "cells": len(cells), "cells_with_other_count": cnt_diff,
                                           "max_cell_dist_diff": dc_diff, "max_lb_rel_diff": lb_diff}}))


if __name__ == "__main__":
    main()
