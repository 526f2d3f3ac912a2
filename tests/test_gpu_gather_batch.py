"""Every plan's obstacle list in one call (isdf_gather_obstacle_points_batch): bit-identical to one isdf_gather_obstacle_points per plan
(points, order, counts) and to the reference-pinned oracle, on dense and cloud-built maps; the sizes reported when cap is too small, by the
batch and by the single call; and set_as_points equal to isdf_set_points_batch with the same lists."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W

pytestmark = pytest.mark.gpu


def _ev(K=16):
    cfg = I.default_config_values()
    cfg.integral_intervs = K
    return I.Evaluator(cfg)


def _plans(seed):
    rng = np.random.default_rng(seed)
    walk = lambda n, s: np.cumsum(rng.normal(size=(n, 3)) * 1.5, axis=0) + s   # noqa: E731  overlapping consecutive boxes
    return [np.zeros((0, 3)),                                                   # no waypoints: gathers nothing
            np.array([[10.3, 20.1, 15.7]]),                                     # one waypoint (its box against the 999 sentinel)
            walk(130, [24.0, 24.0, 17.0]),                                      # 100+ waypoints
            np.repeat([[30.5, 10.5, 8.5]], 4, axis=0),                          # repeated waypoints
            np.array([[-3.0, 2.0, 1.0], [47.0, 50.0, 40.0], [1.0, -2.0, 60.0]]),  # boxes past the map border
            np.concatenate([np.repeat([[20.2, 20.6, 10.4]], 1100, axis=0), walk(5, [21.0, 21.0, 11.0])]),  # > 1024 intersecting earlier boxes
            walk(20, [5.0, 40.0, 30.0])]


def _singles(ev, plans, half, offset):
    out = []
    for w in plans:
        if len(w) == 0:
            out.append(np.zeros((0, 3)))
            continue
        pts, n = ev.gather_obstacle_points(w, half, offset, cap=400000)
        assert len(pts) == n
        out.append(pts)
    return out


@pytest.mark.parametrize("half,offset", [(13.0 / 3.0, (0.0, 0.0, 0.0)), (2.0, (0.3, -0.7, 1.1)), (0.4, (0.0, 0.0, 0.0))])
def test_batch_equals_single_calls_and_the_reference(half, offset):
    occ = W.three_slit_map(48, 48, 48, noise=0.05, seed=7)
    ev = _ev()
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    plans = _plans(3)
    got = ev.gather_obstacle_points_batch(plans, half, offset)
    ref = _singles(ev, plans, half, offset)
    assert sum(len(g) for g in got) > 100
    for b, (g, r) in enumerate(zip(got, ref)):
        assert g.shape == r.shape and np.array_equal(g, r), b
        if len(plans[b]):
            o, n = O.gather_obstacle_points(occ, [0, 0, 0], 1.0, plans[b], half, offset)
            assert n == len(g) and np.array_equal(g, o), b
    perm = [3, 0, 6, 5, 2, 1, 4]                                 # a plan's list depends on its own waypoints only
    got2 = ev.gather_obstacle_points_batch([plans[i] for i in perm], half, offset)
    for k, i in enumerate(perm):
        assert np.array_equal(got2[k], got[i]), i
    ev.close()


def test_batch_on_a_cloud_built_map():
    occ = W.three_slit_map(40, 36, 30, noise=0.04, seed=2)
    idx = np.argwhere(occ)
    rng = np.random.default_rng(4)
    pts = (idx + rng.uniform(0.05, 0.95, size=idx.shape)) * 0.5 + np.array([-3.0, 1.5, 0.25])
    ev = _ev()
    ev.set_map_cloud(pts.astype(np.float32), 0.5)
    info = ev.map_info()
    lo, hi = info["bmin"], info["bmax"]
    plans = [lo + (hi - lo) * rng.uniform(size=(n, 3)) for n in (1, 7, 40, 0, 3)]
    got = ev.gather_obstacle_points_batch(plans, 1.3, (0.1, 0.0, -0.2))
    ref = _singles(ev, plans, 1.3, (0.1, 0.0, -0.2))
    assert sum(len(g) for g in got) > 0
    grid = ev.get_map_u8()                                                 # the oracle on the map the cloud built
    for b, (g, r) in enumerate(zip(got, ref)):
        assert np.array_equal(g, r), b
        if len(plans[b]):
            o, n = O.gather_obstacle_points(grid, lo, info["res"], plans[b], 1.3, (0.1, 0.0, -0.2))
            assert n == len(g) and np.array_equal(g, o), b
    ev.close()


def test_single_call_cap_smaller_than_the_list():
    """isdf_gather_obstacle_points with n > cap: *n is the whole list's size and the first cap points are written (0); with
    set_as_points the same call fails with ISDF_ERR_INVALID"""
    occ = W.three_slit_map(48, 48, 48, noise=0.05, seed=7)
    ev = _ev()
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    wp = np.ascontiguousarray(_plans(3)[2])
    full, n_full = ev.gather_obstacle_points(wp, 13.0 / 3.0)
    assert n_full == len(full) > 10
    ip, dp = C.POINTER(C.c_int32), C.POINTER(C.c_double)
    for cap, set_as_points, code in ((5, 0, 0), (n_full - 1, 0, 0), (5, 1, -1)):
        out, n = np.zeros((cap + 1, 3)), C.c_int(0)
        r = ev.lib.isdf_gather_obstacle_points(ev.h, wp.ctypes.data_as(dp), len(wp), 13.0 / 3.0, None, out.ctypes.data_as(dp), cap, C.byref(n),
                                               set_as_points)
        assert r == code and n.value == n_full, (cap, set_as_points)
        assert np.array_equal(out[:cap], full[:cap]) and not out[cap:].any()
    ev.close()


def test_cap_too_small_reports_the_sizes():
    occ = W.three_slit_map(48, 48, 48, noise=0.05, seed=7)
    ev = _ev()
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    plans = _plans(5)[1:4]
    full = ev.gather_obstacle_points_batch(plans, 13.0 / 3.0)
    sizes = np.cumsum([0] + [len(g) for g in full])
    wo = np.cumsum([0] + [len(w) for w in plans]).astype(np.int32)
    wp = np.ascontiguousarray(np.concatenate(plans))
    ip, dp = C.POINTER(C.c_int32), C.POINTER(C.c_double)
    for cap in (0, int(sizes[-1]) - 1):
        out, pt = np.zeros((max(cap, 1), 3)), np.zeros(len(plans) + 1, dtype=np.int32)
        r = ev.lib.isdf_gather_obstacle_points_batch(ev.h, len(plans), wo.ctypes.data_as(ip), wp.ctypes.data_as(dp), 13.0 / 3.0, None, cap,
                                                     out.ctypes.data_as(dp), pt.ctypes.data_as(ip), 0)
        assert r == -1 and np.array_equal(pt, sizes) and not out.any()
    again = ev.gather_obstacle_points_batch(plans, 13.0 / 3.0, cap=1)   # the binding's retry with the reported total
    assert all(np.array_equal(a, b) for a, b in zip(again, full))
    bad = wo.copy()
    bad[2] = bad[1] - 1
    assert ev.lib.isdf_gather_obstacle_points_batch(ev.h, len(plans), bad.ctypes.data_as(ip), wp.ctypes.data_as(dp), 1.0, None, 0, None,
                                                    pt.ctypes.data_as(ip), 0) == -1
    ev.close()
    fresh = _ev()                                                          # no map
    assert fresh.lib.isdf_gather_obstacle_points_batch(fresh.h, len(plans), wo.ctypes.data_as(ip), wp.ctypes.data_as(dp), 1.0, None, 0, None,
                                                       pt.ctypes.data_as(ip), 0) == -2
    fresh.close()


def test_set_as_points_equals_set_points_batch():
    cfg = I.default_config_values()
    cfg.integral_intervs = 16
    occ = W.three_slit_map(48, 48, 48, noise=0.05, seed=7)
    import test_gpu_lbfgs_device as L
    heads, tails, X = L.problems(4, 5)
    rng = np.random.default_rng(8)
    plans = [np.cumsum(rng.normal(size=(n, 3)), axis=0) + [24.0, 24.0, 17.0] for n in (6, 0, 3, 12)]

    def run(batched):
        ev = I.Evaluator(cfg)
        ev.set_map_u8(occ, [0, 0, 0], 1.0)
        ev.set_shape_named("Ball")
        ev.set_points(np.array([[24.5, 24.5, 17.5], [25.5, 24.5, 17.5]]))
        if batched:
            lists = ev.gather_obstacle_points_batch(plans, 13.0 / 3.0, set_as_points=True)
        else:
            lists = ev.gather_obstacle_points_batch(plans, 13.0 / 3.0)
            ev.set_points_batch(lists)
        out = [ev.callback_batch(heads, tails, 20.0, X) for _ in range(3)]   # t* persists across evaluations
        out.append(ev.swept_results())
        T, Cc, _ = ev.batch_trajectories(4, 5)
        st = ev.lib.isdf_eval_swept(ev.h, 5, T[:5].ctypes.data_as(C.POINTER(C.c_double)), Cc[:90].ctypes.data_as(C.POINTER(C.c_double)),
                                    C.byref(C.c_double(0.0)), np.zeros(90).ctypes.data_as(C.POINTER(C.c_double)),
                                    np.zeros(5).ctypes.data_as(C.POINTER(C.c_double)))
        ev.close()
        return lists, out, st
    la, a, sa = run(True)
    lb, b, sb = run(False)
    assert sum(len(x) for x in la) > 0 and all(np.array_equal(x, y) for x, y in zip(la, lb))
    for (ca, ga), (cb, gb) in zip(a[:3], b[:3]):
        assert np.array_equal(ca, cb) and np.array_equal(ga, gb)
    assert all(np.array_equal(x, y) for x, y in zip(a[3], b[3]))
    assert sa == sb                                                         # the single-problem set is replaced by the lists either way
    assert len(a[3][0]) == sum(len(x) for x in la)


def test_all_empty_batch_switches_the_term_off():
    cfg = I.default_config_values()
    cfg.integral_intervs = 16
    occ = np.zeros((32, 32, 32), dtype=np.uint8)
    import test_gpu_lbfgs_device as L
    heads, tails, X = L.problems(2, 5)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    ev.set_points_batch([np.array([[3.5, 3.5, 3.5]]), np.array([[4.5, 3.5, 3.5]])])
    ev.callback_batch(heads, tails, 20.0, X)
    lists = ev.gather_obstacle_points_batch([np.array([[10.0, 10.0, 10.0]]), np.zeros((0, 3))], 2.0, set_as_points=True)
    assert all(len(x) == 0 for x in lists)
    off = ev.callback_batch(heads, tails, 20.0, X)
    ev.set_points_batch([])
    ref = ev.callback_batch(heads, tails, 20.0, X)
    assert np.array_equal(off[0], ref[0]) and np.array_equal(off[1], ref[1])
    ev.close()
