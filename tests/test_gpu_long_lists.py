"""Long candidate lists for the cells the discrete scan answers everywhere, and the skipped bounded search in deep cells (DESIGN §3.1).

A cell whose every point lies within safety_hor of the mesh or inside it (d_c + ghd < safety_hor) keeps its exact candidate list up to
MESH_LIST_CAP_DISCRETE = 512 entries; every other cell keeps the cap MESH_LIST_CAP = 160. Only the discrete scan reads the longer lists:
the swept-volume term, the certificates and the clearance check take such a cell as unlisted and search the tree as before.
  * the long lists of the bench robot equal the exact sets recomputed in numpy, and no cell outside the rule has more than 160;
  * the discrete cost and gradient match the oracle at the 1e-6 parity bar on a scene with many pairs in long-list cells and in deep
    cells (d_c + ghd <= -safety_hor), where the scan skips the bounded search that cannot succeed;
  * the swept-volume term and the clearance check give bit-identical outputs to the build before the long lists existed, stored in
    tests/golden/long_lists_reference.npz (produced on an H100 by that build with long_lists_outputs below)."""
import os
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import grazing as G
from common import rel_l2
from test_gpu_mesh_lists import pair_dist

pytestmark = pytest.mark.gpu
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]      # the bench robot's poly_params
CAP, CAP_DISCRETE = 160, 512
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "long_lists_reference.npz")


def bench_robot():
    V, F = W.rounded_cone_mesh()
    return V, F


def long_lists_outputs(Imod):
    """the swept-volume term and the clearance check of the bench robot on a small dense scene (Imod: the isdf_b200 module to run)"""
    cfg = Imod.default_config_values()
    cfg.flags = Imod.WITH_DYNAMICS | Imod.WITH_COLLISION
    cfg.integral_intervs = 16
    occ = W.random_map(40, 40, 40, p=0.08, seed=2, slabs=0)
    T, Cc, wp = W.make_trajectory(4, [0, 0, 0], [40, 40, 40], seed=7, jitter=0.2)
    V, F = bench_robot()
    ev = Imod.Evaluator(cfg, device=0)
    try:
        ev.set_map_u8(occ, [0, 0, 0], 1.0)
        ev.set_shape_mesh(V, F, PP)
        pts = W.gather_obstacle_points(occ, [0, 0, 0], 1.0, wp, cfg.kernel_size * cfg.occupancy_resolution / 3.0)
        ev.set_points(pts)
        c, gC, gT = ev.eval_swept(T, Cc)
        tstar, sdf, grel = ev.swept_results()
        clear, vox, summ = ev.trajectory_clearance(T, Cc, 8, 3.0, cfg.safety_hor)
    finally:
        ev.close()
    return dict(sv_cost=np.array([c]), sv_gC=gC, sv_gT=gT, sv_tstar=tstar, sv_sdf=sdf, sv_grel=grel, clear=clear, clear_vox=vox,
                clear_colliding=np.array([s["colliding_samples"] for s in summ]))


def test_long_lists_are_exact():
    cfg = I.default_config_values()
    V, F = bench_robot()
    ev = I.Evaluator(cfg, device=0)
    try:
        ev.set_shape_mesh(V, F, PP)
        grid = ev.dbg_mesh_grid()
        L = ev.dbg_mesh_lists()
    finally:
        ev.close()
    dc, cnt = grid["cell_dist"].astype(np.float64), grid["cell_cnt"].astype(np.int64)
    rule = (dc + grid["ghd"] < cfg.safety_hor) & (np.abs(dc) <= grid["list_reach"])
    assert np.all(cnt[~rule] <= CAP), "a cell outside the discrete rule carries a list past the old cap"
    assert np.all(cnt <= CAP_DISCRETE)
    check = np.argwhere(rule & ((cnt > CAP) | (cnt == 0)))       # long lists, and the cells that still have none
    n_long = int((cnt > CAP).sum())
    print(f"\n{n_long} lists longer than {CAP} ({int(cnt[cnt > CAP].sum())} candidates), {int((rule & (cnt == 0)).sum())} rule cells without one")
    assert n_long >= 1000
    hd = 0.5 * np.sqrt(3.0) * grid["gcell"]
    tris, off, cand = L["tris"], L["cell_off"].astype(np.int64), L["cand"].astype(np.int64)
    nt = tris.shape[0]
    for s in range(0, len(check), 64):
        cells = check[s:s + 64]
        ctr = grid["glo"] + (cells + 0.5) * grid["gcell"]
        d = pair_dist(np.repeat(ctr, nt, axis=0), np.tile(tris[:, 0], (len(cells), 1)), np.tile(tris[:, 1], (len(cells), 1)),
                      np.tile(tris[:, 2], (len(cells), 1))).reshape(len(cells), nt)
        adc = np.abs(dc[tuple(cells.T)])
        R = (adc + (grid["ghd"] - hd) + 2.0 * hd) * (1.0 + 1e-9) + 1e-12
        for k, c in enumerate(cells):
            n = cnt[tuple(c)]
            sure, maybe = d[k] <= R[k] * (1.0 - 1e-9), d[k] <= R[k] * (1.0 + 1e-9)   # a hair of slack for the FP64 rounding of both sides
            if n == 0:
                assert maybe.sum() > CAP_DISCRETE, f"cell {c}: no list, but only {int(sure.sum())}..{int(maybe.sum())} candidates"
                continue
            got = cand[off[tuple(c)]:off[tuple(c)] + n]
            assert len(np.unique(got)) == n and np.all(maybe[got]) and sure.sum() <= n, f"cell {c}: list differs from the exact set"
            dd = d[k][got]
            assert np.all(dd[1:] >= dd[:-1] - 1e-12), f"cell {c}: list not sorted by distance"


def test_discrete_parity_in_long_list_and_deep_cells():
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = 32
    occ = W.random_map(40, 40, 40, p=0.3, seed=4, slabs=0)
    T, Cc, _ = W.make_trajectory(8, [0, 0, 0], [40, 40, 40], seed=5, jitter=0.2)
    V, F = bench_robot()
    ev = I.Evaluator(cfg, device=0)
    try:
        ev.set_map_u8(occ, [0, 0, 0], 1.0)
        ev.set_shape_mesh(V, F, PP)
        got = ev.eval_discrete(T, Cc)
        pairs = ev.stats().last_pairs
        grid = ev.dbg_mesh_grid()
    finally:
        ev.close()
    oc = O.config_from(cfg)
    exp = O.eval_discrete(oc, occ, [0, 0, 0], 1.0, O.Shape.mesh(V, F, PP), T, Cc, use_omp=True)
    assert pairs == exp[3]
    relc = abs(got[0] - exp[0]) / abs(exp[0])
    relg = rel_l2(np.concatenate([got[1], got[2]]), np.concatenate([exp[1], exp[2]]))
    assert relc <= 1e-6 and relg <= 1e-6, f"cost rel {relc:.3e}, grad rel-L2 {relg:.3e}"
    # the scene reaches both new paths: pairs in cells whose list is past the old cap, and pairs in deep cells
    pos, R, _, _ = G.sample_poses(oc, T, Cc)
    flat = occ.reshape(-1)
    prel = np.concatenate([p[flat[vid] != 0] for _, vid, p, _ in G.window_pairs(oc, [0, 0, 0], 1.0, occ.shape, pos, R)])
    c = np.floor((prel - grid["glo"]) * (1.0 / grid["gcell"])).astype(np.int64)
    inside = np.all((c >= 0) & (c < np.array(grid["gdim"])), axis=1)
    ci = tuple(c[inside].T)
    n_long = int((grid["cell_cnt"][ci] > CAP).sum())
    n_deep = int((grid["cell_dist"][ci].astype(np.float64) + grid["ghd"] <= -cfg.safety_hor).sum())
    print(f"\ncost rel {relc:.1e} grad rel {relg:.1e}; {n_long} pairs in long-list cells, {n_deep} in deep cells")
    assert n_long >= 200 and n_deep >= 20


def test_swept_and_clearance_unchanged():
    ref = np.load(GOLDEN)
    got = long_lists_outputs(I)
    for k in ref.files:
        assert got[k].shape == ref[k].shape and np.array_equal(got[k], ref[k]), f"{k} differs from the reference outputs"
