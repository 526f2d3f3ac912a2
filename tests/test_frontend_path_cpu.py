"""The CPU restatements behind the front-end path search (tests/frontpath_serial.cpp): the serial Dijkstra is the exact field of
include/isdf.h (bit for bit against a brute-force Bellman-Ford), the parent rule walks it back to the start, and the reference's A*
restatement finds a path exactly when Dijkstra does, at a cost no lower than the optimum."""
import numpy as np
import pytest

import frontpath_oracle as FO


def _random_case(seed, shape, p_block):
    rng = np.random.default_rng(seed)
    trav = (rng.random(shape) >= p_block).astype(np.uint8)
    src = tuple(int(rng.integers(0, d)) for d in shape)
    return rng, trav, src


@pytest.mark.parametrize("seed,shape,p", [(1, (6, 5, 7), 0.1), (2, (8, 8, 3), 0.3), (3, (5, 9, 6), 0.45), (4, (1, 12, 9), 0.2), (5, (7, 1, 1), 0.0)])
def test_dijkstra_equals_bellman_ford_bit_for_bit(seed, shape, p):
    _, trav, src = _random_case(seed, shape, p)
    trav[src] = seed % 2          # the source is expanded whether it is traversable or not
    g = FO.dijkstra(trav, src)
    bf = FO.bellman_ford(trav, src)
    assert np.array_equal(g.view(np.uint64), bf.view(np.uint64))
    assert g[src] == 0.0 and np.isinf(g[(trav == 0)][g[trav == 0] != 0.0]).all()
    # every reachable voxel walks back to the source by the parent rule, through traversable voxels, at its field value
    for v in zip(*np.nonzero(np.isfinite(g))):
        nodes = FO.path(g, src, v)
        FO.check_path(nodes, trav.astype(bool), src)
        s = 0.0
        for a, b in zip(nodes[:-1], nodes[1:]):
            s = s + np.sqrt(float(((b - a) ** 2).sum()))
        assert s == g[v]


def test_path_of_unreachable_target_is_the_start():
    trav = np.ones((4, 4, 4), dtype=np.uint8)
    trav[2, 2, 2] = 0
    g = FO.dijkstra(trav, (0, 0, 0))
    assert np.isinf(g[2, 2, 2])
    assert FO.path(g, (0, 0, 0), (2, 2, 2)).tolist() == [[0, 0, 0]]
    assert FO.path(g, (0, 0, 0), (0, 0, 0)).tolist() == [[0, 0, 0]]


@pytest.mark.parametrize("seed", range(6))
def test_reference_astar_finds_a_path_iff_dijkstra_does_at_no_lower_cost(seed):
    """masks: random free-attitude sets (the level pose among them or not), occupancy separate; the A* restatement sees the map as the
    reference does (occupied, then checkKernelValue), Dijkstra sees include/isdf.h's traversability"""
    rng = np.random.default_rng(100 + seed)
    X, Y, Z = 9, 8, 7
    xk = yk = 5
    occ = (rng.random((X, Y, Z)) < 0.15 + 0.05 * seed).astype(np.uint8)
    free = rng.random((X * Y * Z, xk * yk)) < 0.08
    masks = np.zeros((X * Y * Z, 4), dtype=np.uint32)
    for a in range(xk * yk):
        masks[:, a >> 5] |= (free[:, a].astype(np.uint32) << np.uint32(a & 31))
    trav = FO.traversable(occ, masks)
    ratios = []
    for q in range(12):
        src = tuple(int(rng.integers(0, d)) for d in (X, Y, Z))
        goal = tuple(int(rng.integers(0, d)) for d in (X, Y, Z))
        if q == 0:
            goal = src
        g = FO.dijkstra(trav.astype(np.uint8), src)
        ref = FO.ref_astar(occ, masks, src, goal, xk, yk, 20.0, 20.0, 10.0)
        assert ref["found"] == bool(np.isfinite(g[goal])), (src, goal)
        if ref["found"]:
            assert ref["cost"] >= g[goal]
            FO.check_path(ref["path"], trav, src)
            assert tuple(ref["path"][-1]) == goal
            ratios.append(ref["cost"] / g[goal] if g[goal] > 0 else 1.0)
    print("reference A* cost / optimum:", np.round(ratios, 4))
