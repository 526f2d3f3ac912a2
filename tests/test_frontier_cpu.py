"""CPU checks of the frontier restatement (tests/frontier_oracle.py, DESIGN §3.24) on hand-built cases: F against a brute-force
neighbour test, labels and the cluster table, the selection rule (GOAL, FRONTIER, NONE, the tie to the smaller voxel index,
min_cluster_voxels, a start on a voxel outside T_b, an empty T_b), and the mirrors and defaults of the new structs."""
import ctypes as C
import numpy as np
import pytest
import frontier_oracle as FR
import isdf_b200 as I

BMIN, RES = np.array([0.0, 0.0, 0.0]), 1.0


def _brute_frontier(To, Tb):
    X, Y, Z = To.shape
    F = np.zeros_like(Tb)
    for v in np.argwhere(Tb):
        for d in np.ndindex(3, 3, 3):
            u = v + np.array(d) - 1
            if (u >= 0).all() and (u < (X, Y, Z)).all() and To[tuple(u)] and not Tb[tuple(u)]:
                F[tuple(v)] = True
    return F


@pytest.mark.parametrize("seed", range(3))
def test_frontier_is_the_neighbour_rule(seed):
    rng = np.random.default_rng(seed)
    To = rng.random((7, 6, 9)) > 0.3
    Tb = To & (rng.random(To.shape) > 0.5)
    F = FR.frontier(To, Tb)
    assert np.array_equal(F, _brute_frontier(To, Tb)) and F.any()
    lab, table = FR.clusters(F, BMIN, RES)
    assert (lab[F] >= 0).all() and (lab[~F] == -1).all()
    flat = np.arange(F.size).reshape(F.shape)
    assert [c["id"] for c in table] == sorted(set(lab[F].tolist()))
    for c in table:
        m = lab == c["id"]
        assert flat[m].min() == c["id"] and m.sum() == c["size"]
        assert np.array_equal(np.argwhere(m).min(0), c["bmin"]) and np.array_equal(np.argwhere(m).max(0), c["bmax"])


def test_labels_join_diagonal_neighbours_only_when_touching():
    F = np.zeros((6, 6, 6), dtype=bool)
    F[0, 0, 0] = F[1, 1, 1] = True        # corner-adjacent: one cluster
    F[3, 3, 3] = F[5, 5, 5] = True        # two apart: two clusters
    lab, table = FR.clusters(F, BMIN, RES)
    assert lab[1, 1, 1] == 0 and len(table) == 3
    assert [c["size"] for c in table] == [2, 1, 1]
    assert np.allclose(table[0]["centroid"], [1.0, 1.0, 1.0])


def _corridor():
    """a known corridor along x at y = z = 1 (x 0..4) ending in a T (x = 5, y = 0 and 2), with unseen traversable space at (5, 1, 1) and
    beyond x = 5: T_o is the corridor, the T, (5, 1, 1) and the whole box x >= 6; T_b the corridor and the T. F is the corridor's last
    voxel and the T, one cluster"""
    To = np.ones((10, 3, 3), dtype=bool)
    To[0:6] = False
    To[0:6, 1, 1] = To[5, 0, 1] = To[5, 2, 1] = True
    Tb = np.zeros_like(To)
    Tb[0:5, 1, 1] = Tb[5, 0, 1] = Tb[5, 2, 1] = True
    return To, Tb


def test_goal_frontier_and_none():
    To, Tb = _corridor()
    F = FR.frontier(To, Tb)
    assert np.array_equal(np.argwhere(F), [[4, 1, 1], [5, 0, 1], [5, 2, 1]])
    lab, table = FR.clusters(F, BMIN, RES)
    assert len(table) == 1 and table[0]["id"] == 40 and table[0]["size"] == 3
    g = FR.field(Tb, (0, 1, 1))
    goal = np.array([9.5, 1.5, 1.5])
    # the goal in known space: GOAL
    r = FR.select(g, F, lab, table, [3.5, 1.5, 1.5], (3, 1, 1), BMIN, RES)
    assert r["kind"] == FR.GOAL and r["g"] == 3.0 and r["score"] == 3.0
    # the goal beyond: FRONTIER at the corridor's end, 4 + 5
    r = FR.select(g, F, lab, table, goal, (9, 1, 1), BMIN, RES)
    assert r["kind"] == FR.FRONTIER and r["voxel"] == 40 and r["score"] == 9.0 and r["cluster"] == 40
    assert np.array_equal(r["point"], [4.5, 1.5, 1.5])
    # a heavier goal term moves it to the T, whose two arms tie: the smaller voxel index wins
    r = FR.select(g, F, lab, table, goal, (9, 1, 1), BMIN, RES, goal_weight=2.0)
    assert r["voxel"] == 5 * 9 + 0 * 3 + 1 and r["score"] == (4.0 + np.sqrt(2.0)) + 2.0 * np.sqrt(17.0)
    # min_cluster_voxels: the cluster of 3 passes 3, not 4 (then NONE)
    assert FR.select(g, F, lab, table, goal, (9, 1, 1), BMIN, RES, min_cluster_voxels=3)["kind"] == FR.FRONTIER
    r = FR.select(g, F, lab, table, goal, (9, 1, 1), BMIN, RES, min_cluster_voxels=4)
    assert r["kind"] == FR.NONE and r["voxel"] == -1 and np.isinf(r["score"]) and np.array_equal(r["point"], goal)


def test_start_outside_tb_and_empty_tb():
    To, Tb = _corridor()
    F = FR.frontier(To, Tb)
    lab, table = FR.clusters(F, BMIN, RES)
    # a start on a voxel outside T_b (and T_o) beside the corridor: its field still enters the corridor
    g = FR.field(Tb, (0, 0, 1))
    assert g[0, 0, 1] == 0.0 and g[0, 1, 1] == 1.0
    r = FR.select(g, F, lab, table, [9.5, 1.5, 1.5], (9, 1, 1), BMIN, RES)
    assert r["kind"] == FR.FRONTIER and r["voxel"] == 40 and r["g"] == g[4, 1, 1]
    # nothing known: no frontier, NONE unless the start voxel is the goal voxel
    Tb0 = np.zeros_like(Tb)
    F0 = FR.frontier(To, Tb0)
    assert not F0.any()
    lab0, table0 = FR.clusters(F0, BMIN, RES)
    g0 = FR.field(Tb0, (2, 1, 1))
    assert FR.select(g0, F0, lab0, table0, [9.5, 1.5, 1.5], (9, 1, 1), BMIN, RES)["kind"] == FR.NONE
    assert FR.select(g0, F0, lab0, table0, [2.5, 1.5, 1.5], (2, 1, 1), BMIN, RES)["kind"] == FR.GOAL


def test_struct_mirrors_and_defaults():
    assert C.sizeof(I.FrontierCluster) == 64 and C.sizeof(I.FrontierGoal) == 64
    assert C.sizeof(I.FrontierParams) == 16 and C.sizeof(I.FrontierInfo) == 72
    assert I.FRONTIER_GOAL_DTYPE.itemsize == 64 and I.FRONTIER_CLUSTER_DTYPE.itemsize == 64
    for name, off in (("kind", 0), ("voxel", 8), ("cluster", 16), ("g", 24), ("score", 32), ("point", 40)):
        assert getattr(I.FrontierGoal, name).offset == off and I.FRONTIER_GOAL_DTYPE.fields[name][1] == off
    for name, off in (("id", 0), ("size", 8), ("bmin", 16), ("bmax", 28), ("centroid", 40)):
        assert getattr(I.FrontierCluster, name).offset == off and I.FRONTIER_CLUSTER_DTYPE.fields[name][1] == off
    assert I.FrontierInfo.field_ms.offset == 56 and I.FrontierInfo.select_ms.offset == 64
    lib = I.load_library()
    p = I.FrontierParams(goal_weight=7.0, min_cluster_voxels=9, reserved_=3)
    assert lib.isdf_frontier_default_params(C.byref(p)) == 0
    assert (p.goal_weight, p.min_cluster_voxels, p.reserved_) == (1.0, 1, 0)
    assert lib.isdf_frontier_default_params(None) == -1
    assert I.PLAN_KNOWN_ONLY == 16 and (I.FRONTIER_NONE, I.FRONTIER_GOAL, I.FRONTIER_FRONTIER) == (0, 1, 2)


def test_entry_points_refuse_without_a_context():
    lib = I.load_library()
    assert lib.isdf_map_frontiers(None, 0, None, None, 0, None, None) == -1
    assert lib.isdf_map_frontiers_device(None, 0, None, None, 0, None, None, None) == -1
    assert lib.isdf_frontier_goals(None, 1, None, None, None, 0, None, None) == -1
    assert lib.isdf_frontier_goals_device(None, 1, None, None, None, 0, None, None, None) == -1
