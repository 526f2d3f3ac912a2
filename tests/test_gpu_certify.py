"""Continuous clearance certificate (isdf_trajectory_certify) on the GPU: the device motion bound against the dense displacement and the
NumPy restatement (tests/certify_oracle.py); collisions between samples that the sampled check misses; soundness against a dense
clearance across shapes, maps and margins; leaves that partition every piece; agreement with the oracle's refinement; bit identity
(initial samples, alone vs batch, run to run, both entry points); refusals and state isolation."""
import ctypes as C
import math
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import clearance_oracle as CO
import certify_oracle as CE

pytestmark = pytest.mark.gpu
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]      # the bench robot's poly_params
BOX_HALF = [0.9, 0.5, 0.3]
DENSE_K = 2 ** 14


def ref_mesh(name):
    d = np.load(__file__.replace("test_gpu_certify.py", "golden/ref_meshes.npz"))
    return d[name + "_V"], d[name + "_F"], d[name + "_pp"]


class Robot:
    def __init__(self, name):
        self.name, self.mesh = name, None
        if name == "Box":
            self.osdf = O.Shape.analytic(I.SHAPE_KINDS["BOX"], BOX_HALF)
        elif name == "bench_mesh":
            V, F = W.rounded_cone_mesh(n_theta=24, n_prof=16)
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
            ev.set_shape_mesh(self.mesh[0], self.mesh[1], self.mesh[2], I.MESH_SIGN_EXACT)
        else:
            ev.set_shape_named(self.name)


def make_cfg(K=8):
    cfg = I.default_config_values()
    cfg.flags = I.WITH_COLLISION
    cfg.integral_intervs = K
    return cfg


def batch_of(trajs):
    N0 = len(trajs[0][0])
    T = np.concatenate([t for t, _ in trajs])
    Cc = np.concatenate([np.asarray(c).reshape(3, 6 * N0) for _, c in trajs], axis=1).reshape(-1)
    return T, Cc, N0


def dense_min(ev, T, Cc, reach, N0=0):
    clear, _, summ = ev.trajectory_clearance(T, Cc, DENSE_K, reach, 0.0, N0=N0)
    return np.array([s["min_clearance"] for s in summ]), clear


# ---- 1. the bound: sound against the dense displacement, within rounding of the oracle -----------------------------------------------
@pytest.mark.parametrize("shape", ["Ball", "Box", "bench_mesh"])
def test_bound_sound_and_tight(shape):
    cfg = make_cfg()
    ev = I.Evaluator(cfg)
    robot = Robot(shape)
    robot.set_on(ev)
    reach = 2.0
    H = cfg.kernel_size * cfg.occupancy_resolution / 2 + reach
    T, Cc, _ = W.make_trajectory(4, [0, 0, 0], [30, 30, 30], seed=6, jitter=0.4)
    rng = np.random.default_rng(0)
    piece, ta, tb = [], [], []
    for i in range(4):
        for h in (T[i], T[i] / 16, T[i] / 64, 1e-6):
            a = rng.uniform(0, T[i] - h)
            for x, y in ((a, a + h), (T[i] - h, T[i]), (0.0, h)):
                piece.append(i); ta.append(x); tb.append(y)
    D, r = ev.dbg_certify_bound(T, Cc, reach, piece, ta, tb)
    if shape == "Box":
        body = CE.box_corners(BOX_HALF)
    elif shape == "bench_mesh":   # the bound holds for every body point within r: points on that sphere
        u = rng.normal(size=(64, 3))
        body = (r * (1 - 1e-9)) * u / np.linalg.norm(u, axis=1, keepdims=True)
    else:
        body = np.zeros((1, 3))
    ratios = []
    for k in range(len(piece)):
        c = CE.piece_coeffs(Cc, 4, piece[k])
        for e, te in enumerate((ta[k], tb[k])):
            o = CE.bound(cfg, r, H, c, ta[k], tb[k], te)
            assert D[k, e] >= o * (1 - 1e-12), (k, e, D[k, e], o)
            assert D[k, e] <= o * (1 + 1e-9) + CE.eps_pad(cfg, r, H, c, te), (k, e, D[k, e], o)
            if tb[k] - ta[k] < T[piece[k]] / 2:
                dense = CE.displacement(cfg, T, Cc, piece[k], ta[k], tb[k], te, body, n=401)
                assert D[k, e] >= dense, (k, e, D[k, e], dense)
                if abs(tb[k] - ta[k] - T[piece[k]] / 64) < 1e-12 and dense > 0:
                    ratios.append(D[k, e] / dense)
    if shape == "bench_mesh":
        assert r >= 5.1 * 0.99                                                 # the cone is 5.1 m long
    if ratios:
        print(f"    {shape}: bound / dense displacement at h = T_i/64: median {np.median(ratios):.3f}, max {max(ratios):.3f}")
    ev.close()


# ---- 2. missed by sampling, caught here ------------------------------------------------------------------------------------------------
def test_thin_wall_ball():
    cfg = make_cfg(3)
    occ = np.zeros((20, 9, 9), dtype=np.uint8)
    occ[10, :, :] = 1
    wp = np.array([[2.0, 4.5, 4.5], [18.0, 4.5, 4.5]])
    T = np.array([4.0])
    Cc = W.minco_s3(wp, T)
    reach, margin = 2.0, 0.5
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    clear, _, summ = ev.trajectory_clearance(T, Cc, 3, reach, margin)
    assert summ[0]["collision_free"] == 1 and clear.min() >= margin + 0.1
    s = ev.trajectory_certify(T, Cc, 3, reach, margin)[0]
    ev.close()
    t = np.linspace(0, T[0], 40001)
    pos, _ = CE.pose_at(cfg, T, Cc, np.zeros(t.size, int), t)
    inside = t[np.abs(pos[:, 0] - 10.5) < 1.0 + margin]
    print(f"    thin wall: first_hit {s['first_hit']:.4f} in [{inside.min():.4f}, {inside.max():.4f}], samples {s['samples']}")
    assert s["verdict"] == I.COLLIDING and inside.min() <= s["first_hit"] <= inside.max()
    assert s["lower_bound"] <= s["min_clearance"] < margin


def test_bench_mesh_between_samples():
    """seeded random trajectories of the bench mesh: the first one the sampled check passes and the dense check does not"""
    cfg = make_cfg(4)
    occ = W.random_map(40, 40, 40, p=0.004, seed=9, slabs=0)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    Robot("bench_mesh").set_on(ev)
    reach, margin, B = 2.0, 0.3, 64
    trajs = [W.make_trajectory(2, [0, 0, 0], [40, 40, 40], seed=100 + b, jitter=0.6)[:2] for b in range(B)]
    T, Cc, N0 = batch_of(trajs)
    _, _, sampled = ev.trajectory_clearance(T, Cc, 4, reach, margin, N0=N0)
    dmin, dclear = dense_min(ev, T, Cc, reach, N0)
    missed = [b for b in range(B) if sampled[b]["collision_free"] == 1 and dmin[b] < margin]
    assert missed, "no seeded trajectory passes the sampled check while colliding between samples"
    b = missed[0]
    Tb, Cb = trajs[b]
    s = ev.trajectory_certify(Tb, Cb, 4, reach, margin)[0]
    per = N0 * (DENSE_K + 1)
    dc = dclear[b * per:(b + 1) * per]
    ev.close()
    tt = np.concatenate([np.sum(Tb[:i]) + np.arange(DENSE_K + 1) * (Tb[i] / DENSE_K) for i in range(N0)])
    bad = tt[dc < margin]
    print(f"    bench mesh seed {100 + b}: dense min {dmin[b]:.4f}, first_hit {s['first_hit']:.4f}, dense colliding times [{bad.min():.4f}, {bad.max():.4f}]")
    assert s["verdict"] == I.COLLIDING
    assert bad.min() - 1e-3 <= s["first_hit"] <= bad.max() + 1e-3


# ---- 3. soundness sweep, leaves partition every piece, colliding witnesses reproduce in the oracle ----------------------------------
def maps():
    rnd = W.random_map(32, 32, 32, p=0.004, seed=2, slabs=0)
    slit = W.three_slit_map(64, 64, 64, noise=0.002, seed=1)
    return {"random_1.0": (rnd, [0.0, 0.0, 0.0], 1.0), "slit_1.0": (slit, [0.3, -0.2, 0.15], 1.0), "slit_0.4": (slit, [0.3, -0.2, 0.15], 0.4),
            "slit_0.25": (slit, [0.3, -0.2, 0.15], 0.25)}


def check_leaves(leaves, T, N0, B):
    for b in range(B):
        for i in range(N0):
            L = leaves[(leaves["piece"] == b * N0 + i)]
            L = np.sort(L, order="ta")
            assert L.size >= 1 and L["ta"][0] == 0.0 and L["tb"][-1] == T[b * N0 + i], (b, i)
            assert np.array_equal(L["tb"][:-1], L["ta"][1:]), (b, i)            # no gap, no overlap


@pytest.mark.parametrize("shape", ["Ball", "Box", "bench_mesh", "RoundedCone.obj", "Lthick.obj"])
@pytest.mark.parametrize("mapname", ["random_1.0", "slit_1.0", "slit_0.4", "slit_0.25"])
def test_soundness_sweep(shape, mapname):
    robot = Robot(shape)
    occ, bmin, res = maps()[mapname]
    cfg = make_cfg(8)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, bmin, res)
    robot.set_on(ev)
    ext = np.array(occ.shape) * res
    B, reach = 3, 2.0
    trajs = [W.make_trajectory(3, bmin + 0.2 * ext, bmin + 0.8 * ext, seed=40 + b, jitter=0.3, piece_time=2.0)[:2] for b in range(B)]
    T, Cc, N0 = batch_of(trajs)
    dmin, _ = dense_min(ev, T, Cc, reach, N0)
    verdicts = []
    for margin in (0.1, 0.5, 1.2):
        summ = ev.trajectory_certify(T, Cc, 8, reach, margin, N0=N0, max_depth=10, max_samples=1024)
        leaves = ev.dbg_certify_leaves()
        check_leaves(leaves, T, N0, B)
        for b, s in enumerate(summ):
            verdicts.append(s["verdict"])
            assert s["lower_bound"] <= dmin[b], (b, margin, s, dmin[b])
            if s["verdict"] == I.CERTIFIED:
                assert dmin[b] >= s["lower_bound"] >= margin
            if s["verdict"] == I.COLLIDING:       # a colliding endpoint reproduces in the oracle at its (piece, local time)
                L = leaves[(leaves["piece"] // N0 == b) & (leaves["ca"] < margin)]
                assert L.size >= 1
                l = L[0]
                ref, _ = CE._clear_at(cfg, (*CO.occupied(occ, bmin, res), lambda p: robot.osdf.query(p, what=0)[0]), T, Cc, [int(l["piece"])],
                                      [l["ta"]], reach)
                assert abs(ref[0] - l["ca"]) <= 1e-12, (ref[0], l["ca"])
    ev.close()
    print(f"    {shape} {mapname}: verdicts {verdicts}, dense minima {np.round(dmin, 3)}")


# ---- 4. usefulness ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["Ball", "Box"])
def test_clear_trajectories_are_certified_at_the_defaults(shape):
    """dense clearance >= margin + res (capped at the default reach = 2 safety_hor, so the map is fine): CERTIFIED at the defaults"""
    cfg = make_cfg()
    res = 0.25
    occ = np.zeros((64, 64, 64), dtype=np.uint8)
    occ[:, 26, 32] = 1                                                    # a rod of voxels along x at y = 6.625, z = 8.125
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], res)
    Robot(shape).set_on(ev)
    p = ev.certify_params()
    margin, reach = p.clearance.margin, p.clearance.reach
    found = 0
    for seed in range(16):                                                # pieces 2.4 - 3.1 m beside the rod
        rng = np.random.default_rng(seed)
        wp = np.array([[2.0, 4.0, 8.0], [6.0, 3.6, 7.6], [10.0, 4.0, 8.4], [14.0, 3.8, 8.0]]) + 0.2 * rng.standard_normal((4, 3)) * [1, 0.3, 0.3]
        T = 2.0 + rng.random(3)
        Cc = W.minco_s3(wp, T)
        d, _ = dense_min(ev, T, Cc, reach)
        if d[0] < margin + res:
            continue
        found += 1
        s = ev.trajectory_certify(T, Cc, p.clearance.samples_per_piece, reach, margin)[0]
        assert s["verdict"] == I.CERTIFIED and margin <= s["lower_bound"] <= d[0], (seed, d, s)
    print(f"    {shape}: {found} of 16 trajectories with dense clearance >= margin + res, all CERTIFIED")
    assert found >= 1
    ev.close()


def test_near_margin_certified_and_depth_zero_undecided():
    cfg = make_cfg()
    occ = W.random_map(48, 48, 48, p=0.003, seed=12, slabs=0)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    Robot("bench_mesh").set_on(ev)
    reach = 3.0
    for seed in range(20):
        T, Cc, _ = W.make_trajectory(4, [8, 8, 8], [40, 40, 40], seed=seed, jitter=0.3)
        d = dense_min(ev, T, Cc, reach)[0][0]
        if 0.3 < d < reach - 0.5:
            break
    else:
        pytest.fail("no trajectory with a dense minimum in (0.3, reach - 0.5)")
    margin = d - 0.05
    s = ev.trajectory_certify(T, Cc, 16, reach, margin, max_samples=4096)[0]
    print(f"    near margin: dense min {d:.4f}, margin {margin:.4f}: {s}")
    assert s["verdict"] == I.CERTIFIED and margin <= s["lower_bound"] <= d
    s0 = ev.trajectory_certify(T, Cc, 16, reach, margin, max_depth=0)[0]
    assert s0["verdict"] == I.UNDECIDED and s0["lower_bound"] < margin and s0["samples"] == 4 * 17
    ev.close()


# ---- 5. agreement with the oracle's refinement -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["Ball", "Box"])
def test_same_leaves_and_verdicts_as_the_oracle(shape):
    robot = Robot(shape)
    cfg = make_cfg()
    cfg.kernel_size = 7
    occ = W.random_map(14, 14, 14, p=0.01, seed=5, slabs=0)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    robot.set_on(ev)
    trajs = []
    for seed in range(4):
        rng = np.random.default_rng(seed)
        Tt = 1.5 + rng.random(2)
        trajs.append((Tt, W.minco_s3(3.0 + 8.0 * rng.random((3, 3)), Tt)))
    T, Cc, N0 = batch_of(trajs)
    r = ev.dbg_certify_bound(T, Cc, 2.0, [0], [0.0], [0.1])[1]
    for margin in (0.2, 0.6):
        summ = ev.trajectory_certify(T, Cc, 4, 2.0, margin, N0=N0, max_depth=8, max_samples=512)
        leaves = ev.dbg_certify_leaves()
        ref = CE.certify(cfg, occ, [0, 0, 0], 1.0, robot.osdf, r, T, Cc, 4, 2.0, margin, N0=N0, max_depth=8, max_samples=512)
        lbs = [max(ca - Da, cb - Db) for (_, _, _, _, ca, cb, Da, Db, _) in ref["leaves"]]
        assert min(abs(x - margin) for x in lbs) > 1e-9, "fixture: a leaf's lb within 1e-9 of margin"
        got = sorted((int(l["piece"]), float(l["ta"]), float(l["tb"]), int(l["state"])) for l in leaves)
        exp = sorted((b * N0 + i, ta, tb, st) for (b, i, ta, tb, _, _, _, _, st) in ref["leaves"])
        assert got == exp
        for g, e in zip(summ, ref["summary"]):
            assert (g["verdict"], g["samples"], g["undecided_intervals"], g["depth"]) == (e["verdict"], e["samples"], e["undecided_intervals"], e["depth"])
            assert g["lower_bound"] == e["lower_bound"] or abs(g["lower_bound"] - e["lower_bound"]) <= 1e-9   # -inf where a bound is +inf
            assert abs(g["min_clearance"] - e["min_clearance"]) <= 1e-12
    ev.close()


# ---- 6. bit identity ----------------------------------------------------------------------------------------------------------------------
def device_certify(ev, T, Cc, params, B):
    import torch
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        dT = torch.tensor(T, dtype=torch.float64, device="cuda")
        dC = torch.tensor(np.asarray(Cc).reshape(-1), dtype=torch.float64, device="cuda")
        ds = torch.zeros(B * 7, dtype=torch.float64, device="cuda")
        ev.trajectory_certify_device(len(T), dT.data_ptr(), dC.data_ptr(), params, ds.data_ptr(), side.cuda_stream)
    side.synchronize()
    raw = ds.cpu().numpy().tobytes()
    return [I.CertifySummary.from_buffer_copy(raw[56 * b:56 * (b + 1)]).as_dict() for b in range(B)]


def key(summ):
    return [tuple(np.float64(v).tobytes() if isinstance(v, float) else v for v in s.values()) for s in summ]


def test_bit_identity():
    cfg = make_cfg(8)
    occ = W.random_map(48, 48, 48, p=0.002, seed=3, slabs=0)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    Robot("bench_mesh").set_on(ev)
    B, K, reach, margin = 6, 8, 2.5, 0.6
    trajs = [W.make_trajectory(3, [0, 0, 0], [48, 48, 48], seed=20 + b, jitter=0.3)[:2] for b in range(B)]
    T, Cc, N0 = batch_of(trajs)
    for ms in (2048, 5):                                                   # uncapped and capped budgets
        s1 = ev.trajectory_certify(T, Cc, K, reach, margin, N0=N0, max_samples=ms)
        l1 = ev.dbg_certify_leaves()
        s2 = ev.trajectory_certify(T, Cc, K, reach, margin, N0=N0, max_samples=ms)
        assert key(s1) == key(s2) and l1.tobytes() == ev.dbg_certify_leaves().tobytes()
        sd = device_certify(ev, T, Cc, ev.certify_params(K, reach, margin, N0, max_samples=ms), B)
        assert key(sd) == key(s1)
        for b, (Tb, Cb) in enumerate(trajs):
            sa = ev.trajectory_certify(Tb, Cb, K, reach, margin, max_samples=ms)
            la = ev.dbg_certify_leaves()
            assert key(sa) == key([s1[b]]), (ms, b)
            lb_ = l1[l1["piece"] // N0 == b].copy()
            lb_["piece"] -= b * N0
            assert np.array_equal(np.sort(la, order=["piece", "ta"]), np.sort(lb_, order=["piece", "ta"])), (ms, b)
        if ms == 5:
            assert any(s["undecided_intervals"] > 0 for s in s1) or all(s["verdict"] != I.UNDECIDED for s in s1)
    # the initial samples are the clearance check's: every leaf endpoint at a uniform time carries that sample's clearance, bit for bit
    ev.trajectory_certify(T, Cc, K, reach, margin, N0=N0)
    leaves = ev.dbg_certify_leaves()
    clear, _, _ = ev.trajectory_clearance(T, Cc, K, reach, margin, N0=N0)
    seen = 0
    for l in leaves:
        i = int(l["piece"])
        step = T[i] * (1.0 / K)
        for t, c in ((l["ta"], l["ca"]), (l["tb"], l["cb"])):
            j = int(round(t / step))
            if t == j * step or (j == K and t == T[i]):
                assert np.float64(c).tobytes() == np.float64(clear[i * (K + 1) + j]).tobytes()
                seen += 1
    assert seen >= len(T) * K
    ev.close()


# ---- 7. refusals and state ---------------------------------------------------------------------------------------------------------------
def test_refusals_poison_and_leave_the_context_working():
    cfg = make_cfg()
    occ = W.random_map(24, 24, 24, p=0.01, seed=1, slabs=0)
    T, Cc, wp = W.make_trajectory(2, [4, 4, 4], [20, 20, 20], seed=1)
    ev = I.Evaluator(cfg)

    def refused(code, **kw):
        args = dict(K_c=8, reach=2.0, margin=0.5)
        args.update(kw)
        p = ev.certify_params(args["K_c"], args["reach"], args["margin"])
        if "reserved" in kw:
            p.reserved_[1] = 1
        summ = (I.CertifySummary * 1)()
        dp = C.POINTER(C.c_double)
        r = ev.lib.isdf_trajectory_certify(ev.h, len(T), T.ctypes.data_as(dp), np.ascontiguousarray(Cc).ctypes.data_as(dp), C.byref(p), summ)
        assert r == code, (kw, r, ev.lib.isdf_last_error())
        assert summ[0].verdict == 0 and np.isnan(summ[0].lower_bound) and np.isnan(summ[0].min_clearance)

    refused(-2)                                                            # no map
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    refused(-2)                                                            # no shape
    for name in ("Torus", "CSG", "RoundedCone"):
        ev.set_shape_named(name)
        refused(-4)
    ev.set_shape_analytic(I.SHAPE_KINDS["BALL"], [cfg.kernel_size * cfg.occupancy_resolution / 2 + 0.1])
    refused(-4)                                                            # wider than half_bd
    ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], [7.0, 0.5, 0.5])
    refused(-4)
    ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], BOX_HALF, rotate=[[1, 0, 0], [0, 1, 1e-9], [0, 0, 1]])
    refused(-4)                                                            # not orthonormal
    V, F = W.icosphere(1.3, 2)
    ev.set_shape_mesh(V, F, PP, I.MESH_SIGN_WINDING)
    refused(-4)
    ev.set_shape_named("Ball")
    for kw in (dict(margin=-0.1), dict(margin=2.0), dict(margin=2.5), dict(K_c=0), dict(reserved=1)):
        refused(-1, **kw)
    with pytest.raises(I.IsdfError) as e:
        ev.trajectory_certify(T, Cc, 8, 2.0, 0.5, max_depth=65)
    assert e.value.code == -1
    p = ev.certify_params(8, 2.0, 0.5)
    assert ev.lib.isdf_trajectory_certify_device(ev.h, len(T), None, None, C.byref(p), None, None) == -1
    ev.set_shard(0, 2)
    refused(-4)
    ev.set_shard(0, 1)
    # state: a discrete evaluation, the swept-volume results and every statistic but kernel_launches are unchanged by a certificate
    Robot("bench_mesh").set_on(ev)
    c0, g0, t0 = ev.eval_discrete(T, Cc)
    pts = W.gather_obstacle_points(occ, [0, 0, 0], 1.0, wp, 3.0)[:50]
    ev.set_points(pts)
    sv0 = ev.eval_swept(T, Cc)
    st0 = ev.stats()
    ev.trajectory_clearance(T, Cc, 8, 2.0, 0.5)
    counts0 = ev.dbg_clearance_counts()
    st0 = ev.stats()
    s = ev.trajectory_certify(T, Cc, 8, 2.0, 0.5)[0]
    st1 = ev.stats()
    assert s["verdict"] in (-1, 0, 1) and st1.kernel_launches > st0.kernel_launches
    for f in ("evals_discrete", "evals_swept", "last_pairs", "last_sdf_evals", "last_kernel_ms"):
        assert getattr(st1, f) == getattr(st0, f), f
    assert ev.dbg_clearance_counts() == counts0
    c1, g1, t1 = ev.eval_discrete(T, Cc)
    sv1 = ev.eval_swept(T, Cc)
    assert c1 == c0 and np.array_equal(g1, g0) and np.array_equal(t1, t0)
    assert sv1[0] == sv0[0] and np.array_equal(sv1[1], sv0[1])
    ev.close()
