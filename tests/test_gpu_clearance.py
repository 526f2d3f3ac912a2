"""Trajectory clearance check (isdf_trajectory_clearance) on the GPU against the brute-force restatement of tests/clearance_oracle.py:
per-sample clearance and witness across shapes, maps, resolutions and reach; winding-sign meshes against the library's own unculled
shape query; exact verdicts with clearances placed at margin +- delta and reach +- delta; the motivating case (an obstacle between
waypoints that the gathered obstacle list misses); consistency with the discrete cost; batching, determinism and both entry points;
the empty map and every refusal."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import clearance_oracle as CO

pytestmark = pytest.mark.gpu
TOL = 1e-12                     # DESIGN's SDF bar
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]      # the bench robot's poly_params
ANALYTIC = ["Ball", "Torus", "RoundedCone", "SmoothIntersection", "CSG", "TwistBox", "Box"]
REACHES = [0.15, 0.866, 2.5]
BOX_HALF = [0.9, 0.5, 0.3]


def ref_mesh(name):
    d = np.load(__file__.replace("test_gpu_clearance.py", "golden/ref_meshes.npz"))
    return d[name + "_V"], d[name + "_F"], d[name + "_pp"]


class Robot:
    """one robot on both sides: set_on(ev) for the library, osdf for the oracle"""

    def __init__(self, name):
        self.name = name
        self.mesh = None
        if name == "Box":
            self.osdf = O.Shape.analytic(I.SHAPE_KINDS["BOX"], BOX_HALF)
        elif name == "bench_mesh":
            V, F = W.rounded_cone_mesh()
            self.mesh = (V, F, PP)
        elif name in ("RoundedCone.obj", "Lthick.obj"):
            self.mesh = ref_mesh(name[:-4])
        else:
            self.osdf = O.Shape.named(name)
        if self.mesh is not None:
            self.osdf = O.Shape.mesh(self.mesh[0], self.mesh[1], self.mesh[2], wn_mode=O.WN_BH)

    def set_on(self, ev):
        if self.name == "Box":
            ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], BOX_HALF)
        elif self.mesh is not None:
            ev.set_shape_mesh(*self.mesh)
        else:
            ev.set_shape_named(self.name)


def make_cfg(K=8):
    cfg = I.default_config_values()
    cfg.flags = I.WITH_COLLISION
    cfg.integral_intervs = K
    return cfg


def traj_in(bmin, extent, seed=0, N=3):
    """N pieces through the map's interior, waypoints at random fractions of its extent"""
    rng = np.random.default_rng(seed)
    wp = np.asarray(bmin, float) + extent * (0.3 + 0.4 * rng.random((N + 1, 3)))
    T = 2.0 + rng.random(N)
    return T, W.minco_s3(wp, T)


def maps():
    rnd = W.random_map(24, 24, 24, p=0.05, seed=1, slabs=0)
    slit = W.three_slit_map(64, 64, 64, noise=0.02, seed=1)
    return {"random_1.0": (rnd, [0.0, 0.0, 0.0], 1.0), "slit_1.0": (slit, [0.3, -0.2, 0.15], 1.0),
            "slit_0.4": (slit, [0.3, -0.2, 0.15], 0.4), "slit_0.25": (slit, [0.3, -0.2, 0.15], 0.25)}


def check_parity(robot, occ, bmin, res, reach, K=8, seed=0, margin=None):
    cfg = make_cfg(K)
    T, Cc = traj_in(bmin, np.array(occ.shape) * res, seed=seed)
    margin = reach if margin is None else margin
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, bmin, res)
    robot.set_on(ev)
    clear, vox, summ = ev.trajectory_clearance(T, Cc, K, reach, margin)
    ref = CO.clearance(O.config_from(cfg), occ, bmin, res, robot.osdf, T, Cc, K, reach, margin, keep_candidates=True)
    ev.close()
    compare(clear, vox, ref, reach, TOL)
    return clear, vox, summ, ref


def compare(clear, vox, ref, reach, tol):
    err = np.abs(clear - ref["clear"])
    assert err.max() <= tol, f"clearance differs by {err.max():.3e} at sample {int(err.argmax())}"
    for s, (cid, v) in enumerate(ref["candidates"]):
        below = v < reach - tol
        assert not np.any(np.abs(v - reach) <= tol), "fixture: a candidate sits on the reach cap"
        if vox[s] >= 0:
            hit = np.flatnonzero(cid == vox[s])
            assert hit.size == 1, f"sample {s}: witness {vox[s]} is not a candidate"
            assert abs(v[hit[0]] - v.min()) <= tol, f"sample {s}: witness sdf {v[hit[0]]} vs minimum {v.min()}"
        assert (vox[s] < 0) == (not below.any()), f"sample {s}: witness {vox[s]}, oracle minimum {v.min() if v.size else None}"


# ---- parity: every shape at every reach on the random map; three shapes on every map --------------------------------------------
@pytest.mark.parametrize("reach", REACHES)
@pytest.mark.parametrize("shape", ANALYTIC + ["bench_mesh", "RoundedCone.obj", "Lthick.obj"])
def test_parity_shapes(shape, reach):
    occ, bmin, res = maps()["random_1.0"]
    clear, vox, _, _ = check_parity(Robot(shape), occ, bmin, res, reach)
    assert (vox >= 0).sum() >= 3


@pytest.mark.parametrize("reach", REACHES)
@pytest.mark.parametrize("mapname", ["slit_1.0", "slit_0.4", "slit_0.25"])
@pytest.mark.parametrize("shape", ["Ball", "bench_mesh", "Lthick.obj"])
def test_parity_maps(shape, mapname, reach):
    occ, bmin, res = maps()[mapname]
    check_parity(Robot(shape), occ, bmin, res, reach, seed=2)


# ---- winding sign: every candidate answered, compared with the library's unculled shape query -----------------------------------
def open_box():
    V, F = W.box_mesh(1.2, 0.7, 0.4)
    return V, F[2:]


@pytest.mark.parametrize("reach", [0.15, 2.5])
@pytest.mark.parametrize("mesh", ["open_box", "closed_ico"])
def test_winding_sign_meshes(mesh, reach):
    V, F = open_box() if mesh == "open_box" else W.icosphere(1.3, 2)
    occ, bmin, res = maps()["random_1.0"]
    cfg = make_cfg()
    T, Cc = traj_in(bmin, np.array(occ.shape) * res, seed=4)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, bmin, res)
    ev.set_shape_mesh(V, F, PP, I.MESH_SIGN_WINDING)
    clear, vox, _ = ev.trajectory_clearance(T, Cc, 8, reach, reach)
    ref = CO.clearance(O.config_from(cfg), occ, bmin, res, lambda p: ev.shape_query(p, I.QUERY_SDF)[0], T, Cc, 8, reach, reach,
                       keep_candidates=True)
    ev.close()
    err = np.abs(clear - ref["clear"]).max()
    print(f"    winding {mesh} reach {reach}: max |clearance - unculled query| = {err:.3e}")
    compare(clear, vox, ref, reach, 1e-10)
    assert (vox >= 0).sum() >= 3


# ---- exact verdicts: clearances placed at margin +- delta and reach +- delta ---------------------------------------------------------
DELTA = 1e-3


def verdicts_match(summ, ref):
    for g, e in zip(summ, ref):
        for k in ("collision_free", "colliding_samples", "piece_min", "sample_min", "voxel_min"):
            assert g[k] == e[k], (k, g, e)
        for k in ("min_clearance", "t_min", "first_hit"):
            assert abs(g[k] - e[k]) <= TOL, (k, g, e)
        assert (g["first_hit"] == -1.0) == (e["first_hit"] == -1.0)


@pytest.mark.parametrize("shape", ["Ball", "bench_mesh"])
@pytest.mark.parametrize("where", ["margin-", "margin+", "reach-", "reach+"])
def test_exact_verdicts_at_margin_and_reach(shape, where):
    robot = Robot(shape)
    occ, bmin, res = maps()["random_1.0"]
    cfg = make_cfg(16)
    K, big = 16, 3.0
    T, Cc = traj_in(bmin, np.array(occ.shape) * res, seed=5)
    base = CO.clearance(O.config_from(cfg), occ, bmin, res, robot.osdf, T, Cc, K, big, big)["clear"]
    # a sample clearance c* well inside (0, big): the fixture level is c* -+ delta, and no other sample may sit within 1e-9 of it
    cands = [c for c in np.unique(base) if 0.3 < c < big - 0.5]
    sign = -1.0 if where.endswith("-") else 1.0                   # "-": c* = level - delta (below), "+": c* = level + delta
    for c_star in cands:
        level = c_star - sign * DELTA
        if np.all(np.abs(base - level) > 1e-9):
            break
    reach, margin = (big, level) if where.startswith("margin") else (level, level - 0.2)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, bmin, res)
    robot.set_on(ev)
    clear, vox, summ = ev.trajectory_clearance(T, Cc, K, reach, margin)
    ref = CO.clearance(O.config_from(cfg), occ, bmin, res, robot.osdf, T, Cc, K, reach, margin, keep_candidates=True)
    ev.close()
    assert np.all(np.abs(ref["clear"] - margin) > 1e-9) and np.all(np.abs(ref["clear"][ref["voxel"] >= 0] - reach) > 1e-9)
    compare(clear, vox, ref, reach, TOL)
    assert np.array_equal(vox, ref["voxel"])
    verdicts_match(summ, ref["summary"])
    assert 0 < summ[0]["colliding_samples"] < clear.size


def test_obstacle_between_waypoints_missed_by_the_gathered_list():
    """the motivating case: a voxel next to the middle of a long piece, farther than the gather boxes reach from every waypoint. The
    swept-volume cost over the gathered list is zero; the clearance check reports the collision."""
    cfg = make_cfg(64)
    X = 48
    occ = np.zeros((X, X, X), dtype=np.uint8)
    wp = np.array([[6.0, 6.0, 10.0], [40.0, 6.0, 10.0], [40.0, 40.0, 10.0]])
    T = np.array([5.0, 5.0])
    Cc = W.minco_s3(wp, T)
    mid = W.traj_eval(T, Cc, 2.5).reshape(3)
    occ[tuple(np.floor(mid + [0.0, 0.6, 0.0]).astype(int))] = 1          # beside the path, halfway along piece 0
    occ[43, 2, 13] = 1                                                    # inside waypoint 1's gather box, ~6 m from the path
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    half = cfg.kernel_size * cfg.occupancy_resolution / 3.0
    pts, n = ev.gather_obstacle_points(wp, half, set_as_points=True)
    assert n == 1 and np.allclose(pts[0], [43.5, 2.5, 13.5])             # the mid-piece voxel is not in the list
    cost, _, _ = ev.eval_swept(T, Cc)
    clear, vox, summ = ev.trajectory_clearance(T, Cc, 64, cfg.safety_hor, cfg.safety_hor)
    ev.close()
    ref = CO.clearance(O.config_from(cfg), occ, [0, 0, 0], 1.0, O.Shape.named("Ball"), T, Cc, 64, cfg.safety_hor, cfg.safety_hor)
    verdicts_match(summ, ref["summary"])
    s = summ[0]
    print(f"    swept cost {cost}, min clearance {s['min_clearance']:.4f} at t = {s['t_min']:.3f}, first hit {s['first_hit']:.3f}")
    assert cost == 0.0
    assert s["collision_free"] == 0 and s["colliding_samples"] > 0 and s["min_clearance"] < cfg.safety_hor
    assert s["piece_min"] == 0 and s["voxel_min"] == int(np.ravel_multi_index(tuple(np.floor(mid + [0.0, 0.6, 0.0]).astype(int)), occ.shape))


# ---- consistency with the discrete cost (same samples, same poses) --------------------------------------------------------------
@pytest.mark.parametrize("shape", ["Ball", "bench_mesh"])
def test_consistent_with_discrete_piece_costs(shape):
    robot = Robot(shape)
    cfg = make_cfg(32)
    occ = W.random_map(40, 40, 40, p=0.03, seed=7, slabs=0)
    T, Cc, _ = W.make_trajectory(6, [0, 0, 0], [40, 40, 40], seed=8, jitter=0.2)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    robot.set_on(ev)
    ev.eval_discrete(T, Cc)
    pc = ev.piece_costs(len(T))
    sf, h, K = cfg.safety_hor, cfg.kernel_size * cfg.occupancy_resolution / 2, cfg.integral_intervs
    clear, vox, _ = ev.trajectory_clearance(T, Cc, K, sf, sf)
    ev.close()
    cl = clear.reshape(len(T), K + 1)
    pos, R = CO.poses(O.config_from(cfg), T, Cc, K)
    assert (pc > 0).sum() >= 1
    for i in range(len(T)):
        if pc[i] > 0:
            assert cl[i].min() < sf, f"piece {i}: cost {pc[i]} but no sample closer than safety_hor"
        for j in range(K + 1):
            s = i * (K + 1) + j
            if vox[s] < 0 or clear[s] >= sf:
                continue
            c = (np.array(np.unravel_index(vox[s], occ.shape)) + 0.5) * 1.0
            d = c - pos[s]
            if np.all(np.abs(d) <= h - 1.0) and np.all(np.abs(d @ R[s]) <= h):   # inside the world and the body bd/2 box
                assert pc[i] > 0, f"sample {s}: witness inside both boxes with clearance {clear[s]} but piece {i} costs nothing"


# ---- batching, determinism, both entry points ------------------------------------------------------------------------------------
def device_check(ev, T, Cc, params):
    import torch
    N = len(T)
    S = N * (params.samples_per_piece + 1)
    B = 1 if params.pieces_per_traj == 0 else N // params.pieces_per_traj
    dT, dC = torch.tensor(T, dtype=torch.float64, device="cuda"), torch.tensor(np.asarray(Cc).reshape(-1), dtype=torch.float64, device="cuda")
    dcl, dvx = torch.zeros(S, dtype=torch.float64, device="cuda"), torch.zeros(S, dtype=torch.int64, device="cuda")
    dsum = torch.zeros(B * 6, dtype=torch.float64, device="cuda")      # 48-byte records
    ev.trajectory_clearance_device(N, dT.data_ptr(), dC.data_ptr(), params, dcl.data_ptr(), dvx.data_ptr(), dsum.data_ptr(),
                                   torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    raw = dsum.cpu().numpy().tobytes()
    summ = [I.ClearanceSummary.from_buffer_copy(raw[48 * b:48 * (b + 1)]).as_dict() for b in range(B)]
    return dcl.cpu().numpy(), dvx.cpu().numpy(), summ


def test_batch_alone_repeat_and_device_are_bit_identical():
    robot = Robot("bench_mesh")
    cfg = make_cfg(16)
    occ = W.random_map(48, 48, 48, p=0.002, seed=3, slabs=0)           # sparse: some restarts are collision-free, some are not
    N0, B, K = 3, 8, 16
    trajs = [W.make_trajectory(N0, [0, 0, 0], [48, 48, 48], seed=20 + b, jitter=0.3)[:2] for b in range(B)]
    T = np.concatenate([t for t, _ in trajs])
    Cc = np.concatenate([np.asarray(c).reshape(3, 6 * N0) for _, c in trajs], axis=1).reshape(-1)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    robot.set_on(ev)
    reach, margin = 2.0, 0.866
    c1, v1, s1 = ev.trajectory_clearance(T, Cc, K, reach, margin, N0=N0)
    c2, v2, s2 = ev.trajectory_clearance(T, Cc, K, reach, margin, N0=N0)
    assert c1.tobytes() == c2.tobytes() and np.array_equal(v1, v2) and s1 == s2
    dc, dv, ds = device_check(ev, T, Cc, ev.clearance_params(K, reach, margin, N0))
    assert dc.tobytes() == c1.tobytes() and np.array_equal(dv, v1) and ds == s1
    per = N0 * (K + 1)
    for b, (Tb, Cb) in enumerate(trajs):
        ca, va, sa = ev.trajectory_clearance(Tb, Cb, K, reach, margin)
        assert ca.tobytes() == c1[b * per:(b + 1) * per].tobytes() and np.array_equal(va, v1[b * per:(b + 1) * per]) and sa[0] == s1[b]
    assert sum(s["collision_free"] for s in s1) not in (0, B)             # both verdicts occur in the batch
    ev.close()


def test_lbfgs_batch_trajectories_check_identically_through_either_path():
    cfg = make_cfg(16)
    occ = W.random_map(48, 48, 48, p=0.03, seed=4, slabs=0)
    N0, B = 4, 6
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    Robot("Ball").set_on(ev)
    dim = 4 * N0 - 3
    X0, heads, tails = np.zeros((B, dim)), np.zeros((B, 3, 3)), np.zeros((B, 3, 3))
    for b in range(B):
        wp = W.random_walk_waypoints(N0, [0, 0, 0], [48, 48, 48], seed=300 + b)
        X0[b, :N0] = 1.0
        X0[b, N0:] = wp[1:-1].reshape(-1)
        heads[b, :, 0], tails[b, :, 0] = wp[0], wp[-1]
    ev.lbfgs_batch(heads, tails, 20.0, X0, ev.lbfgs_params(max_iterations=5))
    T, Cc, _ = ev.batch_trajectories(B, N0)
    p = ev.clearance_params(16, 1.5, 0.866, N0)
    c, v, s = ev.trajectory_clearance(T, Cc, 16, 1.5, 0.866, N0=N0)
    dc, dv, ds = device_check(ev, T, Cc, p)
    ev.close()
    assert dc.tobytes() == c.tobytes() and np.array_equal(dv, v) and ds == s
    ref = CO.clearance(O.config_from(cfg), occ, [0, 0, 0], 1.0, O.Shape.named("Ball"), T, Cc, 16, 1.5, 0.866, N0=N0)
    assert np.abs(c - ref["clear"]).max() <= TOL


# ---- edges and refusals ---------------------------------------------------------------------------------------------------------
def test_empty_map_is_clear_everywhere():
    cfg = make_cfg()
    ev = I.Evaluator(cfg)
    ev.set_map_u8(np.zeros((20, 20, 20), dtype=np.uint8), [0, 0, 0], 1.0)
    Robot("bench_mesh").set_on(ev)
    T, Cc = traj_in([0, 0, 0], np.array([20, 20, 20]))
    l0 = ev.stats().kernel_launches
    clear, vox, summ = ev.trajectory_clearance(T, Cc, 8, 1.7, 0.5)
    st = ev.stats()
    ev.close()
    assert np.all(clear == 1.7) and np.all(vox == -1)
    assert summ[0]["collision_free"] == 1 and summ[0]["first_hit"] == -1.0 and summ[0]["voxel_min"] == -1 and summ[0]["colliding_samples"] == 0
    assert st.kernel_launches == l0 + 2 and st.evals_discrete == 0 and st.evals_swept == 0 and st.last_pairs == 0


def test_refusals():
    cfg = make_cfg()
    occ = W.random_map(16, 16, 16, p=0.05, seed=1, slabs=0)
    T, Cc = traj_in([0, 0, 0], np.array([16, 16, 16]))
    ev = I.Evaluator(cfg)
    with pytest.raises(I.IsdfError) as e:
        ev.trajectory_clearance(T, Cc, 8, 1.0, 1.0)
    assert e.value.code == -2                                             # no map
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    with pytest.raises(I.IsdfError) as e:
        ev.trajectory_clearance(T, Cc, 8, 1.0, 1.0)
    assert e.value.code == -2                                             # no shape
    ev.set_shape_named("Ball")
    for K, reach, margin, N0 in [(0, 1.0, 1.0, 0), (8, 0.0, 0.0, 0), (8, -1.0, -1.0, 0), (8, np.inf, 1.0, 0), (8, np.nan, 0.5, 0),
                                 (8, 1.0, 1.5, 0), (8, 1.0, np.nan, 0), (8, 1.0, 1.0, 2), (8, 400.0, 1.0, 0)]:
        with pytest.raises(I.IsdfError) as e:
            ev.trajectory_clearance(T, Cc, K, reach, margin, N0=N0)
        assert e.value.code == -1, (K, reach, margin, N0)
    # the widest window accepted: 2 H sqrt(3) / res + 4 <= 1023
    h = cfg.kernel_size * cfg.occupancy_resolution / 2
    ok = (1019.0 / (2.0 * np.sqrt(3.0))) - h
    ev.trajectory_clearance(T, Cc, 2, ok * (1 - 1e-9), 1.0)
    with pytest.raises(I.IsdfError) as e:
        ev.trajectory_clearance(T, Cc, 2, ok * (1 + 1e-9), 1.0)
    assert e.value.code == -1
    ev.set_shard(0, 2)
    with pytest.raises(I.IsdfError) as e:
        ev.trajectory_clearance(T, Cc, 8, 1.0, 1.0)
    assert e.value.code == -4
    # failed calls poison every summary
    summ = (I.ClearanceSummary * 1)()
    p = ev.clearance_params(8, 1.0, 1.0)
    r = ev.lib.isdf_trajectory_clearance(ev.h, len(T), T.ctypes.data_as(C.POINTER(C.c_double)), np.ascontiguousarray(Cc).ctypes.data_as(C.POINTER(C.c_double)),
                                         C.byref(p), None, None, summ)
    assert r == -4 and np.isnan(summ[0].min_clearance) and summ[0].collision_free == 0
    ev.close()
