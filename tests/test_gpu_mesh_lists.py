"""The mesh's per-cell candidate lists as the pruned list pass relies on them (DESIGN §3.1): every list sorted by distance from its cell
centre, its first entry the triangle nearest to the centre, and every cand_lb a lower bound of that distance that is tight to float
precision. The distances are recomputed here in numpy FP64, independently of the library's closest-point test. A bound rounded to
nearest instead of down, or without its slack, exceeds the distance for about half the candidates and fails the bound check."""
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W

pytestmark = pytest.mark.gpu
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]      # the bench robot's poly_params


def pair_dist(P, A, B, Cv):
    """distance of point P[i] to triangle (A[i], B[i], Cv[i]), all (n, 3): Ericson's Voronoi-region closest point, vectorised"""
    dot = lambda x, y: np.einsum("ij,ij->i", x, y)
    ab, ac = B - A, Cv - A
    ap, bp, cp = P - A, P - B, P - Cv
    d1, d2, d3, d4, d5, d6 = dot(ap, ab), dot(ap, ac), dot(bp, ab), dot(bp, ac), dot(cp, ab), dot(cp, ac)
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    safe = lambda a: np.where(a == 0, 1.0, a)
    den = 1.0 / safe(va + vb + vc)
    q = A + (vb * den)[:, None] * ab + (vc * den)[:, None] * ac
    e43, e56 = d4 - d3, d5 - d6
    regions = [((va <= 0) & (e43 >= 0) & (e56 >= 0), B + (e43 / safe(e43 + e56))[:, None] * (Cv - B)),
               ((vb <= 0) & (d2 >= 0) & (d6 <= 0), A + (d2 / safe(d2 - d6))[:, None] * ac),
               ((d6 >= 0) & (d5 <= d6), Cv),
               ((vc <= 0) & (d1 >= 0) & (d3 <= 0), A + (d1 / safe(d1 - d3))[:, None] * ab),
               ((d3 >= 0) & (d4 <= d3), B),
               ((d1 <= 0) & (d2 <= 0), A)]
    for m, val in regions:                                       # later regions take priority
        q[m] = val[m]
    return np.linalg.norm(P - q, axis=1)


@pytest.mark.parametrize("mesh", ["bench", "coarse"])
def test_candidate_lists_sorted_with_lower_bounds(mesh):
    V, F = W.rounded_cone_mesh() if mesh == "bench" else W.rounded_cone_mesh(n_theta=16, n_prof=12)
    cfg = I.default_config_values()
    ev = I.Evaluator(cfg, device=0)
    try:
        ev.set_shape_mesh(V, F, PP)
        grid = ev.dbg_mesh_grid()
        L = ev.dbg_mesh_lists()
    finally:
        ev.close()
    cnt, off, cand, lb, tris = grid["cell_cnt"], L["cell_off"], L["cand"], L["cand_lb"], L["tris"]
    assert len(cand) == int(cnt.astype(np.int64).sum()) > 0 and len(lb) == len(cand)
    listed = np.argwhere(cnt > 0)
    rng = np.random.default_rng(7)
    cells = listed[rng.choice(len(listed), size=min(len(listed), 600), replace=False)]
    ctr = grid["glo"] + (cells + 0.5) * grid["gcell"]
    n = cnt[tuple(cells.T)].astype(np.int64)
    o = off[tuple(cells.T)].astype(np.int64)
    owner = np.repeat(np.arange(len(cells)), n)                  # every candidate of the sampled cells, list by list
    idx = np.concatenate([np.arange(a, a + k) for a, k in zip(o, n)])
    t = cand[idx].astype(np.int64)
    d = pair_dist(ctr[owner], tris[t, 0], tris[t, 1], tris[t, 2])
    b = lb[idx].astype(np.float64)
    # a lower bound of the distance, tight to float precision
    assert np.all(b <= d), f"{int(np.sum(b > d))} of {len(d)} bounds exceed the distance (worst by {np.max(b - d):.3e})"
    assert np.all(b >= d * (1.0 - 1e-6) - 1e-9), f"bounds looser than float rounding: worst {np.max(d - b):.3e}"
    # sorted by distance; bounds non-decreasing along each list
    same = owner[1:] == owner[:-1]
    assert np.all(b[1:][same] >= b[:-1][same])
    assert np.all(d[1:][same] >= d[:-1][same] - 1e-12)
    # the first entry is the triangle nearest to the cell centre among all of the mesh's triangles
    first = np.concatenate([[0], np.cumsum(n)[:-1]])
    nearest = np.full(len(cells), np.inf)
    for k in range(len(tris)):
        nearest = np.minimum(nearest, pair_dist(ctr, *[np.broadcast_to(tris[k, j], ctr.shape) for j in range(3)]))
    assert np.all(d[first] <= nearest + 1e-12), f"worst {np.max(d[first] - nearest):.3e}"
