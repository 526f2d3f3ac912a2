"""CPU checks of the restatements that planning through what has been seen is held against (tests/known_plan_oracle.py, DESIGN §3.23):
the weighted Dijkstra at weight 0 is frontpath_oracle.dijkstra bit for bit, and at any weight a brute-force Bellman-Ford; on an L-shaped
known corridor beside a straight unknown route the path goes straight below the detour ratio and through the corridor above it; the
known-prefix rows and the gather rule on constructed cases; and the mirrors of isdf_frontpath_params / isdf_plan_params."""
import ctypes as C
import numpy as np
import pytest
import frontpath_oracle as FO
import known_plan_oracle as KO
import oracle_lib as O
import isdf_b200 as I
from test_plan_cpu import _fields, _probe


def _bellman_ford(trav, known, src, w):
    """every round offers g(u) + w(u, v) to all 26 neighbours at once (w read at v); until no change"""
    trav = np.asarray(trav, dtype=bool)
    X, Y, Z = trav.shape
    cw = 1.0 + w
    g = np.full((X, Y, Z), np.inf)
    g[tuple(src)] = 0.0
    P = np.full((X + 2, Y + 2, Z + 2), np.inf)
    while True:
        P[1:-1, 1:-1, 1:-1] = g
        new = g.copy()
        for i, j, k in FO.OFFSETS:
            e = np.sqrt(float(i * i + j * j + k * k))
            wv = np.where(known, e, e * cw) if known is not None else np.full(trav.shape, e * cw)
            cand = P[1 - i:1 - i + X, 1 - j:1 - j + Y, 1 - k:1 - k + Z] + wv
            new = np.where(trav & (cand < new), cand, new)
        if np.array_equal(new, g):
            return g
        g = new


def _grid(seed, shape=(9, 8, 7)):
    rng = np.random.default_rng(seed)
    return rng.random(shape) > 0.25, rng.random(shape) > 0.5


@pytest.mark.parametrize("seed", range(4))
def test_weight_zero_is_the_unweighted_field(seed):
    trav, known = _grid(seed)
    src = (1, 2, 3)
    ref = FO.dijkstra(trav, src)
    for k in (known, None):
        assert np.array_equal(KO.dijkstra(trav, k, src, 0.0), ref)
    t = tuple(np.argwhere(np.isfinite(ref))[-1])
    assert np.array_equal(KO.path(ref, known, src, t, 0.0), FO.path(ref, src, t))


@pytest.mark.parametrize("seed,w", [(0, 0.5), (1, 2.0), (2, 7.25), (3, 1e-3)])
def test_weighted_dijkstra_equals_bellman_ford(seed, w):
    trav, known = _grid(seed)
    src = (4, 0, 6)
    g = KO.dijkstra(trav, known, src, w)
    assert np.array_equal(g, _bellman_ford(trav, known, src, w))
    assert np.array_equal(KO.dijkstra(trav, None, src, w), _bellman_ford(trav, None, src, w))
    # the parent rule walks every reachable voxel back to the source over traversable nodes
    for t in np.argwhere(np.isfinite(g))[::17]:
        p = KO.path(g, known, src, t, w)
        FO.check_path(p, trav, src)
        assert tuple(p[-1]) == tuple(t)


def _corridor(L=12, H=3):
    """z = 1 slice: the straight row y = 0 from S = (0, 0) to T = (L, 0), unknown between them; an L-shaped known corridor up x = 0, along
    y = H and down x = L to T, which is known. Nothing else is traversable."""
    trav = np.zeros((L + 1, H + 1, 1), dtype=bool)
    known = np.zeros_like(trav)
    trav[:, 0] = True
    trav[0, :] = trav[:, H] = trav[L, :] = True
    known[0, 1:] = known[:, H] = known[L, :] = True
    return trav, known, (0, 0, 0), (L, 0, 0)


def test_l_corridor_switches_at_the_detour_ratio():
    trav, known, S, T = _corridor()
    L = T[0]
    detour = FO.dijkstra(trav & (known | (np.arange(L + 1) == 0)[:, None, None]), S)[T]   # the corridor alone, unweighted
    # straight: L - 1 unknown voxels and the known goal, (L - 1) c + 1; corridor: every voxel known, so its length whatever c is
    rho = (detour - 1.0) / (L - 1)
    assert 1.0 < rho < np.inf
    for c, straight in ((1.0, True), (rho * 0.99, True), (rho * 1.01, False), (4 * rho, False)):
        g = KO.dijkstra(trav, known, S, c - 1.0)
        p = KO.path(g, known, S, T, c - 1.0)
        if straight:
            assert (p[:, 1] == 0).all() and len(p) == L + 1
            s = 0.0
            for _ in range(L - 1):
                s += c
            assert g[T] == s + 1.0   # the left-to-right sum along the row
        else:
            assert all(known[tuple(v)] for v in p[1:]), "the path left the known corridor"
            assert g[T] == detour


def test_known_rows_rule():
    known = np.zeros((10, 1, 1), dtype=bool)
    nodes = np.array([[i, 0, 0] for i in range(10)])
    assert KO.first_unknown(nodes, None) == 0 and KO.known_rows(nodes, None, 2, 5) == 0
    assert KO.known_rows(nodes, known, 2, 5) == 0                 # node 0 unknown: k* = 0
    known[:5] = True                                               # k* = 5: nodes 2 and 4 are known, node 6 is not
    assert KO.first_unknown(nodes, known) == 5 and KO.known_rows(nodes, known, 2, 5) == 2
    known[:] = True                                                # k* = 10: every row
    assert KO.known_rows(nodes, known, 2, 5) == 4 and KO.known_rows(nodes, known, 3, 3) == 2
    assert KO.waypoint_gap(10, 1.0, 3.0) == 3 and KO.waypoint_gap(2, 1.0, 3.0) == 0


def test_gather_rule_on_constructed_cases():
    rng = np.random.default_rng(5)
    dims, bmin, res = (16, 12, 10), np.zeros(3), 1.0
    bmax = bmin + np.array(dims) * res
    occ = rng.random(dims) > 0.85
    wps = np.array([[3.5, 5.5, 4.5], [5.5, 6.5, 4.5], [8.5, 6.5, 5.5], [11.5, 5.5, 4.5]])
    h = 2.0
    ref, n = O.gather_obstacle_points(occ.astype(np.uint8), bmin, res, wps, h)
    # no known rows: the occupancy gather, in the reference's order
    assert np.array_equal(KO.gather(occ, np.ones(dims, bool), bmin, bmax, res, wps, h, rows=0), ref[:n])
    # everything known: blocked == occ, whatever the rows
    for rows in (1, 2, 4, 9):
        assert np.array_equal(KO.gather(occ, np.ones(dims, bool), bmin, bmax, res, wps, h, rows=rows), ref[:n])
    # nothing known and every row known: every voxel of the union of the boxes, once
    every = KO.gather(occ, None, bmin, bmax, res, wps, h, rows=4)
    allbox = O.gather_obstacle_points(np.ones(dims, np.uint8), bmin, res, wps, h)
    assert np.array_equal(every, allbox[0][:allbox[1]])
    # one unknown free voxel inside the first two boxes: listed by known row 0 only; with rows = 0 by none
    known = np.ones(dims, bool)
    occ2 = occ.copy()
    v = (4, 6, 4)
    occ2[v] = False
    known[v] = False
    c = (np.array(v) + 0.5) * res + bmin
    one = KO.gather(occ2, known, bmin, bmax, res, wps, h, rows=1)
    assert (np.all(one == c, axis=1)).sum() == 1
    assert not np.all(KO.gather(occ2, known, bmin, bmax, res, wps, h, rows=0) == c, axis=1).any()
    # a known row lists blocked voxels the occupancy rows after it would not: rows = 1 adds exactly the unknown free voxels of box 0
    base = KO.gather(occ2, known, bmin, bmax, res, wps, h, rows=0)
    assert len(one) == len(base) + 1


def test_struct_mirrors_match_the_header():
    structs = [("isdf_frontpath_params", I.FrontPathParams), ("isdf_plan_params", I.PlanParams)]
    got = _probe(structs)
    for cname, py in structs:
        size, offs = got[cname]
        assert size == C.sizeof(py) and offs == dict(_fields(py)), cname
    assert C.sizeof(I.FrontPathParams) == 16
    assert I.PLAN_KNOWN_PREFIX == 8


def test_plan_defaults_leave_the_front_end_unweighted():
    lib = I.load_library()
    p = I.PlanParams()
    assert lib.isdf_plan_default_params(None, C.byref(p)) == 0
    assert p.frontpath.unknown_weight == 0.0 and list(p.frontpath.reserved_) == [0, 0]
    assert not p.flags & I.PLAN_KNOWN_PREFIX
