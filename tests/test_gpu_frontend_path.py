"""The front-end path search (isdf_frontend_path*, include/isdf.h) against the CPU restatements of tests/frontpath_serial.cpp: the
traversability grid equals (feasibility mask != 0) & free, the FP64 field equals a serial Dijkstra bit for bit on every voxel, paths and
costs follow the parent rule exactly, attitudes are isdf_frontend_check_batch chained along the path, and the reference's A* (restated
with its quirks) finds a path exactly when the product does, at a cost no lower."""
import numpy as np
import pytest

import isdf_b200 as I
import workloads as W
import frontpath_oracle as FO
from common import small_case, MESHES

pytestmark = pytest.mark.gpu

BMIN = np.array([-3.25, 1.5, 0.125])


def _setup(occ, robot, ks, bmin=BMIN, safeh=0.0):
    cfg, _, _, _, _ = small_case(N=2, K=4, seed=3, kernel_size=ks)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, bmin, cfg.occupancy_resolution)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        ev.set_shape_mesh(V, F, [0.1, 0.0, -0.1, 120.0, 10.0, 0.0])
    else:
        ev.set_shape_named(robot)
    ev.frontend_build_kernels(45.0, 45.0, 9.0, safeh)
    return ev


def _centre(idx, bmin=BMIN, res=1.0):
    idx = np.asarray(idx, dtype=np.float64)
    return (idx + 0.5) * res + bmin


def _index(xyz, bmin=BMIN, res=1.0):
    return np.floor((np.asarray(xyz) - bmin) / res).astype(np.int64)


def _field(ev, start, shape):
    import torch
    d_g = torch.empty(int(np.prod(shape)), dtype=torch.float64, device="cuda")
    ev.frontend_path_field_device(start, d_g.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d_g.cpu().numpy().reshape(shape)


CASES = {
    # name: (occupancy, robot, kernel_size, front_end_safeh)
    "random24_ball": (lambda: W.random_map(24, 24, 24, p=0.05, seed=3, slabs=1), "Ball", 5, 0.0),
    "random30pct_point_ks1": (lambda: (np.random.default_rng(4).random((30, 26, 33)) < 0.30).astype(np.uint8), "Point", 1, 0.0),
    "slits_40x36x28_capped_cone": (lambda: W.three_slit_map(40, 36, 28, noise=0.003, seed=5), "CappedCone", 13, 0.0),
    "random_64_mesh": (lambda: (np.random.default_rng(6).random((64, 40, 37)) < 0.05).astype(np.uint8), "mesh", 9, 0.8),
    "thin_axis_48x20x1": (lambda: (np.random.default_rng(7).random((48, 20, 1)) < 0.15).astype(np.uint8), "Torus", 9, 0.8),
}


@pytest.mark.parametrize("case", list(CASES))
def test_path_field_and_attitudes_match_the_oracle(case):
    mk, robot, ks, safeh = CASES[case]
    occ = mk()
    X, Y, Z = occ.shape
    ev = _setup(occ, robot, ks, safeh=safeh)
    xk, yk = ev.fe_dims
    masks = ev.frontend_feasibility(X, Y, Z)
    trav = FO.traversable(occ, masks)
    assert trav.any() and not trav.all()
    rng = np.random.default_rng(sum(map(ord, case)))
    cand = np.argwhere(trav)
    src = tuple(int(v) for v in cand[rng.integers(0, len(cand))])
    start = _centre(src) + rng.uniform(-0.45, 0.45, 3)
    goals_idx = [cand[rng.integers(0, len(cand))] for _ in range(14)] + [np.array(src), np.argwhere(occ)[0]]
    goals = np.array([_centre(g) + rng.uniform(-0.45, 0.45, 3) for g in goals_idx])
    res = ev.frontend_path_batch(start, goals)
    # traversability grid of the product against the product's own feasibility masks
    assert np.array_equal(ev.dbg_frontpath_traversable(), trav)
    # the field, bit for bit, on every voxel
    g = _field(ev, start, (X, Y, Z))
    ref = FO.dijkstra(trav.astype(np.uint8), src)
    assert np.array_equal(g.view(np.uint64), ref.view(np.uint64)), f"{(g.view(np.uint64) != ref.view(np.uint64)).sum()} voxels differ"
    info = ev.frontend_path_info()
    assert info["rounds"] >= 1 and info["field_bytes"] == 8 * X * Y * Z
    ratios = []
    for b, t in enumerate(goals_idx):
        t = tuple(int(v) for v in t)
        p, rp = res["paths"][b], res["roll_pitch"][b]
        nodes = _index(p)
        assert np.array_equal(p, _centre(nodes))                    # cube centres, exactly
        want = FO.path(ref, src, t)
        assert np.array_equal(nodes, want)
        assert res["found"][b] == bool(np.isfinite(ref[t]))
        assert res["costs"][b] == ref[t] or (np.isinf(res["costs"][b]) and np.isinf(ref[t]))
        FO.check_path(nodes, trav, src)
        if res["found"][b]:
            assert tuple(nodes[-1]) == t
            s = 0.0
            for a, c in zip(nodes[:-1], nodes[1:]):
                s = s + np.sqrt(float(((c - a) ** 2).sum()))
            assert s == res["costs"][b]
        # attitudes: node 0 level, then isdf_frontend_check_batch from each node's attitude into the next node
        assert rp[0].tolist() == [0.0, 0.0]
        if len(nodes) > 1:
            child, ok = ev.frontend_check_batch(nodes[1:].astype(np.int32), rp[:-1])
            assert ok.all() and np.array_equal(child, rp[1:])
        # batch result == a call with this goal alone
        if b % 5 == 0:
            p1, rp1, c1, f1 = ev.frontend_path(start, goals[b])
            assert np.array_equal(p1, p) and np.array_equal(rp1, rp) and f1 == res["found"][b]
            assert np.float64(c1).view(np.uint64) == res["costs"][b].view(np.uint64)
        # the reference's A* (restated with its quirks): same verdict, cost no lower
        ra = FO.ref_astar(occ, masks, src, t, xk, yk, 45.0, 45.0, 9.0)
        assert ra["found"] == res["found"][b], (case, t)
        if ra["found"]:
            assert res["costs"][b] <= ra["cost"]
            ratios.append(ra["cost"] / res["costs"][b] if res["costs"][b] > 0 else 1.0)
    assert res["found"].sum() >= 3
    print(f"{case}: reference A* cost / exact cost over {len(ratios)} found paths: max {max(ratios):.4f}, mean {np.mean(ratios):.4f}")
    ev.close()


def test_runs_entry_points_and_batches_agree_bit_for_bit():
    import torch
    occ = W.three_slit_map(40, 36, 28, noise=0.01, seed=8)
    ev = _setup(occ, "Ball", 5)
    X, Y, Z = occ.shape
    trav = FO.traversable(occ, ev.frontend_feasibility(X, Y, Z))
    cand = np.argwhere(trav)
    rng = np.random.default_rng(12)
    start = _centre(cand[0])
    goals = np.array([_centre(cand[i]) for i in rng.integers(0, len(cand), 64)])
    a = ev.frontend_path_batch(start, goals)
    b = ev.frontend_path_batch(start, goals)
    for k in ("xyz", "rp", "offsets", "costs", "found"):
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k
    # device entry point on a side stream
    n = int(a["offsets"][-1])
    dev = torch.device("cuda", 0)
    d_goals = torch.from_numpy(goals.reshape(-1)).to(dev)
    d_xyz, d_rp = torch.zeros(3 * n, dtype=torch.float64, device=dev), torch.zeros(2 * n, dtype=torch.float64, device=dev)
    d_off, d_cost = torch.zeros(65, dtype=torch.int32, device=dev), torch.zeros(64, dtype=torch.float64, device=dev)
    d_found = torch.zeros(64, dtype=torch.uint8, device=dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ev.frontend_path_batch_device(start, 64, d_goals.data_ptr(), n, d_xyz.data_ptr(), d_rp.data_ptr(), d_off.data_ptr(), d_cost.data_ptr(),
                                      d_found.data_ptr(), side.cuda_stream)
    side.synchronize()
    assert np.array_equal(d_off.cpu().numpy(), a["offsets"])
    assert np.array_equal(d_xyz.cpu().numpy().reshape(-1, 3), a["xyz"]) and np.array_equal(d_rp.cpu().numpy().reshape(-1, 2), a["rp"])
    assert np.array_equal(d_cost.cpu().numpy().view(np.uint64), a["costs"].view(np.uint64))
    assert np.array_equal(d_found.cpu().numpy().astype(bool), a["found"])
    # every goal alone
    for i in (0, 17, 63):
        p, rp, c, f = ev.frontend_path(start, goals[i])
        assert np.array_equal(p, a["paths"][i]) and np.array_equal(rp, a["roll_pitch"][i]) and f == a["found"][i]
    ev.close()


def test_edges_and_errors():
    occ = np.zeros((20, 18, 22), dtype=np.uint8)
    occ[10, 9, 11] = 1                                                 # an occupied voxel
    occ[3:8, 3:8, 3:8] = 1                                             # a shell around (5, 5, 5)
    occ[4:7, 4:7, 4:7] = 0
    ev = _setup(occ, "Ball", 3)
    s_occ = _centre((10, 9, 11))
    # start == goal on an occupied voxel: found, one node
    p, rp, c, f = ev.frontend_path(s_occ, s_occ)
    assert f and c == 0.0 and np.array_equal(p, [_centre((10, 9, 11))]) and rp.tolist() == [[0.0, 0.0]]
    start = _centre((15, 15, 15))
    # goal occupied, goal enclosed in a shell: not found, the start alone, cost +inf
    for goal in (s_occ, _centre((5, 5, 5))):
        p, rp, c, f = ev.frontend_path(start, goal)
        assert not f and np.isinf(c) and np.array_equal(p, [_centre((15, 15, 15))])
    # a reachable goal
    p, rp, c, f = ev.frontend_path(start, _centre((1, 1, 1)))
    need = len(p)
    assert f and need > 14 and c == FO.dijkstra(FO.traversable(occ, ev.frontend_feasibility(*occ.shape)).astype(np.uint8), (15, 15, 15))[1, 1, 1]
    # on the map's faces: bmin and bmax are inside (isInMap), a hair beyond is not
    bmax = BMIN + np.array(occ.shape)
    p, rp, c, f = ev.frontend_path(BMIN, bmax)
    assert f and np.array_equal(_index(p[0]), [0, 0, 0]) and np.array_equal(_index(p[-1]), np.array(occ.shape) - 1)
    for bad_s, bad_g in ((BMIN - [1e-9, 0, 0], start), (start, bmax + [0, 0, 1e-9]), ([np.nan, 0, 0], start), (start, [0, np.inf, 0])):
        with pytest.raises(I.IsdfError) as e:
            ev.frontend_path(bad_s, bad_g)
        assert e.value.code == -1
    # cap too small: ISDF_ERR_INVALID with the needed length reported
    r, n = ev.frontend_path_raw(start, _centre((1, 1, 1)), need - 1)
    assert r == -1 and n == need
    r, n = ev.frontend_path_raw(start, _centre((1, 1, 1)), need)
    assert r == 0 and n == need
    # sharded context
    ev.set_shard(0, 2)
    with pytest.raises(I.IsdfError) as e:
        ev.frontend_path(start, start)
    assert e.value.code == -4
    ev.set_shard(0, 1)
    # kernels given up by a new shape, and never built
    ev.set_shape_named("Torus")
    with pytest.raises(I.IsdfError) as e:
        ev.frontend_path(start, start, cap=4)
    assert e.value.code == -2
    ev.close()
    cfg, _, _, _, _ = small_case(N=2, K=4, seed=3, kernel_size=3)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_named("Ball")
    with pytest.raises(I.IsdfError) as e:
        ev.frontend_path(start, start, cap=4)
    assert e.value.code == -2
    ev.close()


def test_a_replaced_map_is_searched_not_the_old_one():
    occ = np.zeros((24, 24, 24), dtype=np.uint8)
    ev = _setup(occ, "Ball", 3)
    start, goal = _centre((2, 12, 12)), _centre((21, 12, 12))
    p0, _, c0, f0 = ev.frontend_path(start, goal)
    assert f0 and c0 == 19.0
    wall = occ.copy()
    wall[12, :, :] = 1
    wall[12, 0, 0] = 0                                                 # one hole in a corner
    ev.set_map_u8(wall, BMIN, 1.0)
    p1, _, c1, f1 = ev.frontend_path(start, goal)
    trav = FO.traversable(wall, ev.frontend_feasibility(24, 24, 24))
    ref = FO.dijkstra(trav.astype(np.uint8), (2, 12, 12))
    assert f1 == bool(np.isfinite(ref[21, 12, 12])) and (c1 == ref[21, 12, 12] or (np.isinf(c1) and np.isinf(ref[21, 12, 12])))
    assert c1 > c0
    assert np.array_equal(_index(p1), FO.path(ref, (2, 12, 12), (21, 12, 12)))
    ev.close()


def test_full_size_benchmark_map():
    """one far-apart query on the 512^3 benchmark map of bench.py: the path is valid on the product's traversability grid and its cost is
    the left-to-right sum of its steps, which equals the device field at the goal"""
    X = 512
    occ = W.random_map(X, X, X, p=0.05, seed=1, slabs=3)
    cfg, _, _, _, _ = small_case(N=2, K=4, seed=3, kernel_size=5)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    bm = np.zeros(3)
    src, goal = far_apart_pair(ev, X)
    p, rp, c, f = ev.frontend_path(_centre(src, bm), _centre(goal, bm))
    trav = ev.dbg_frontpath_traversable()
    info = ev.frontend_path_info()
    print("512^3 path:", len(p), "nodes, cost", c, info)
    nodes = _index(p, bm)
    assert f and tuple(nodes[-1]) == goal and len(p) > X // 2
    FO.check_path(nodes, trav, src)
    s = 0.0
    for a, b in zip(nodes[:-1], nodes[1:]):
        s = s + np.sqrt(float(((b - a) ** 2).sum()))
    assert s == c
    child, ok = ev.frontend_check_batch(nodes[1:].astype(np.int32), rp[:-1])
    assert ok.all() and np.array_equal(child, rp[1:])
    assert info["rounds"] >= 1 and info["field_bytes"] == 8 * X ** 3
    ev.close()


def far_apart_pair(ev, X):
    """a traversable start near the (0, 0, 0) corner and the voxel of its component farthest from it (largest finite field value)"""
    import torch
    ev.frontend_path_field_device([0.5, 0.5, 0.5], torch.empty(X ** 3, dtype=torch.float64, device="cuda").data_ptr())   # builds the traversability grid
    trav = ev.dbg_frontpath_traversable()
    cand = np.argwhere(trav)
    cand = cand[np.argsort(cand.sum(axis=1), kind="stable")][:8]
    d_g = torch.empty(X ** 3, dtype=torch.float64, device="cuda")
    best = None
    for v in cand:
        src = tuple(int(a) for a in v)
        ev.frontend_path_field_device(_centre(src, np.zeros(3)), d_g.data_ptr())
        torch.cuda.synchronize()
        fin = torch.where(torch.isfinite(d_g), d_g, torch.full_like(d_g, -1.0))
        far = int(torch.argmax(fin).item())
        if best is None or fin[far].item() > best[2]:
            best = (src, (far // (X * X), (far // X) % X, far % X), fin[far].item())
    del d_g
    return best[0], best[1]
