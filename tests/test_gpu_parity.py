"""GPU parity tests (run on an H100 with -m gpu): every call goes through the C-ABI of libisdf_b200.so and is
compared with the oracle on identical seeded inputs.

Tolerances (stated, FP64 path):
  * SDF values: 1e-12 (abs/rel). Arithmetic is FP64 add/mul/div/sqrt with FMA contraction off on both sides; only libm
    (sin/cos/atan2/acos) may differ in the last ulp.
  * FD gradients (getonlyGrad1): 1e-8 — the reference's dx = 5e-6 central difference amplifies 1-ulp SDF differences by 1e5.
  * cost / gradC / gradT: <= 1e-6 relative (cost) and rel-L2 (gradients) — BASELINE.json north_star; typically ~1e-13.
"""
import ctypes as C
import math
import os
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
from common import small_case, rel_l2, BMIN, tilted, MESHES

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-6


def grads(gC, gT):
    return np.concatenate([gC, gT])


def check_eval(got, exp, tol=TOL, what=""):
    c, gC, gT = got
    oc, ogC, ogT = exp[0], exp[1], exp[2]
    if abs(oc) > 0:
        assert abs(c - oc) <= tol * abs(oc), f"{what}: cost {c} vs {oc}"
    else:
        assert c == 0
    r = rel_l2(grads(gC, gT), grads(ogC, ogT))
    assert r <= tol, f"{what}: gradient rel-L2 {r:.3e}"
    return r


# ---- the BasicShape plug-in surface ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", I.NAMED_SHAPES)
def test_shape_query_named(name):
    R, t = tilted()
    ev = I.Evaluator()
    ev.set_shape_named(name, R, t)
    osh = O.Shape.named(name, R, t)
    p = np.random.default_rng(11).uniform(-6, 6, size=(2000, 3))
    s, g = ev.shape_query(p, I.QUERY_SDF_GRAD)
    os_, og = osh.query(p, 2)
    assert np.allclose(s, os_, rtol=1e-12, atol=1e-12), np.abs(s - os_).max()
    bad = np.abs(g - og).max(axis=1) > 1e-8
    assert bad.mean() <= 0.002, (bad.sum(), np.abs(g - og).max())   # FD across a non-smooth seam can flip branch within ±dx
    s0, _ = ev.shape_query(p, I.QUERY_SDF)
    _, g1 = ev.shape_query(p, I.QUERY_GRAD)
    assert np.array_equal(s0, s) and np.array_equal(g1, g)
    ev.close()


def test_shape_query_box_and_golden():
    R, t = tilted()
    ev = I.Evaluator()
    ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], [1.5, 0.15, 0.15], R, t)
    z = np.load(os.path.join(G, "shapes.npz"))
    s, g = ev.shape_query(z["p"])
    assert np.allclose(s, z["Box_sdf"], rtol=1e-12, atol=1e-12) and np.allclose(g, z["Box_grad"], atol=1e-9)
    for name in I.NAMED_SHAPES:
        ev.set_shape_named(name, z["R"], z["t"])
        s, g = ev.shape_query(z["p"])
        assert np.allclose(s, z[f"{name}_sdf"], rtol=1e-12, atol=1e-12), name
    ev.close()


@pytest.mark.parametrize("mesh", list(MESHES))
def test_shape_query_mesh(mesh):
    V, F = MESHES[mesh]()
    pp = [0.2, -0.1, 0.3, 120.0, 10.0, -30.0]
    ev = I.Evaluator()
    ev.set_shape_mesh(V, F, pp)
    osh = O.Shape.mesh(V, F, pp)
    p = np.random.default_rng(5).uniform(-5, 6, size=(3000, 3))
    s, g = ev.shape_query(p)
    os_, og = osh.query(p)
    assert np.array_equal(np.sign(s), np.sign(os_)), "inside/outside classification differs from the exact winding number"
    assert np.allclose(s, os_, rtol=1e-12, atol=1e-12), np.abs(s - os_).max()
    bad = np.abs(g - og).max(axis=1) > 1e-9
    assert bad.mean() <= 0.002   # equidistant-triangle ties
    ev.close()


def test_points_in_aabb_matches_reference_semantics():
    rng = np.random.default_rng(3)
    occ = (rng.random((40, 33, 70)) < 0.2).astype(np.uint8)     # Z > 64: rows span three bit-words
    bmin, res = np.array([-3.0, 1.0, 0.5]), 0.5
    ev = I.Evaluator()
    ev.set_map_u8(occ, bmin, res)
    bmax = bmin + np.array(occ.shape) * res
    for _ in range(40):
        c = bmin + (bmax - bmin) * (rng.random(3) * 1.6 - 0.3)
        half = rng.uniform(0.3, 3.0)
        a, na = ev.points_in_aabb(c, half)
        b, nb = O.points_in_aabb(occ, bmin, res, c, half)
        assert na == nb and np.array_equal(a, b)
    ev.set_map_f64(occ.astype(np.float64) * 3.0, bmin, res)      # reference storage: double per voxel, non-zero = occupied
    a, na = ev.points_in_aabb(bmin + 5, 2.0)
    b, nb = O.points_in_aabb(occ, bmin, res, bmin + 5, 2.0)
    assert na == nb and np.array_equal(a, b)
    ev.close()


# ---- discrete path ------------------------------------------------------------------------------------------------------------
DISCRETE_SHAPES = ["Ball", "Torus_big", "RoundedCone", "CappedCone", "WireframeBox", "BendLinear_big", "TwistBox", "Table", "Trefoil",
                   "SmoothDifference", "SmoothIntersection_big", "CSG"]


@pytest.mark.parametrize("name", DISCRETE_SHAPES)
def test_discrete_parity_analytic(name):
    cfg, occ, T, Cc, _ = small_case(N=4, K=16, seed=3)
    R, t = tilted()
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_named(name, R, t)
    exp = O.eval_discrete(O.config_from(cfg), occ, BMIN, 1.0, O.Shape.named(name, R, t), T, Cc)
    got = ev.eval_discrete(T, Cc)
    r = check_eval(got, exp, what=name)
    assert ev.stats().last_pairs == exp[3]
    print(f"{name}: cost {got[0]:.6g} grad rel-L2 {r:.2e} pairs {exp[3]}")
    ev.close()


def test_discrete_parity_box_shape():
    cfg, occ, T, Cc, _ = small_case(N=3, K=12, seed=8)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], [1.5, 0.3, 0.3])
    exp = O.eval_discrete(O.config_from(cfg), occ, BMIN, 1.0, O.Shape.analytic(I.SHAPE_KINDS["BOX"], [1.5, 0.3, 0.3]), T, Cc)
    check_eval(ev.eval_discrete(T, Cc), exp, what="Box")
    ev.close()


@pytest.mark.parametrize("mesh", list(MESHES))
def test_discrete_parity_mesh(mesh):
    cfg, occ, T, Cc, _ = small_case(N=4, K=16, seed=6)
    V, F = MESHES[mesh]()
    pp = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]        # config_CappedCone.yaml poly_params
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_mesh(V, F, pp)
    exp = O.eval_discrete(O.config_from(cfg), occ, BMIN, 1.0, O.Shape.mesh(V, F, pp), T, Cc)
    got = ev.eval_discrete(T, Cc)
    r = check_eval(got, exp, what=mesh)
    assert got[0] > 0 and ev.stats().last_pairs == exp[3]
    print(f"mesh {mesh}: cost {got[0]:.6g} grad rel-L2 {r:.2e}")
    ev.close()


@pytest.mark.parametrize("case", ["N1", "K1", "res05", "ks17", "ks40", "dense", "outside", "collision_only", "dynamics_only", "empty_map"])
def test_discrete_edge_cases(case):
    N, K, seed, noise, ks, res, flags = 3, 12, 9, 0.03, 13, 1.0, None
    if case == "N1": N = 1
    if case == "K1": K = 1
    if case == "ks17": ks = 17
    if case == "ks40": ks, N, K = 40, 2, 4      # window taller than 32 voxels: exercises the z-chunk loop of the bit scan
    if case == "dense": noise = 0.6
    if case == "collision_only": flags = I.WITH_COLLISION
    if case == "dynamics_only": flags = I.WITH_DYNAMICS
    cfg, occ, T, Cc, wp = small_case(N=N, K=K, seed=seed, noise=noise, flags=flags, kernel_size=ks)
    bmin = list(BMIN)
    if case == "res05":
        res, cfg.occupancy_resolution = 0.5, 0.5
        Cc = Cc * 0.5     # shrink the trajectory into the 32 m map
    if case == "outside":
        bmin = [30.0, -10.0, 5.0]   # most of the trajectory lies outside the map: windows clamp to the border (quirk Q6)
    if case == "empty_map":
        occ = np.zeros_like(occ)
    if case == "dynamics_only":
        cfg.vmax, cfg.omgmax, cfg.thetamax = 0.8, 0.3, 0.2
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, bmin, res)
    ev.set_shape_named("SmoothIntersection")
    exp = O.eval_discrete(O.config_from(cfg), occ, bmin, res, O.Shape.named("SmoothIntersection"), T, Cc)
    got = ev.eval_discrete(T, Cc)
    check_eval(got, exp, what=case)
    assert ev.stats().last_pairs == (exp[3] if (cfg.flags & I.WITH_COLLISION) else 0)
    ev.close()


def test_discrete_accumulates_into_caller_buffers_and_is_deterministic():
    cfg, occ, T, Cc, _ = small_case(N=4, K=16, seed=3)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_named("Torus")
    c1, gC1, gT1 = ev.eval_discrete(T, Cc)
    c2, gC2, gT2 = ev.eval_discrete(T, Cc)
    assert c1 == c2 and np.array_equal(gC1, gC2) and np.array_equal(gT1, gT2)      # bit-reproducible
    c3, gC3, gT3 = ev.eval_discrete(T, Cc, cost=5.0, gradC=np.ones(18 * 4), gradT=2 * np.ones(4))
    assert c3 == 5.0 + c1 and np.array_equal(gC3, 1.0 + gC1) and np.array_equal(gT3, 2.0 + gT1)   # hpp:539-550 semantics
    ev.close()


@pytest.mark.parametrize("world", [2, 3, 8])
def test_discrete_shards_sum_to_full(world):
    cfg, occ, T, Cc, _ = small_case(N=4, K=16, seed=3)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_named("RoundedCone")
    full = ev.eval_discrete(T, Cc)
    acc = [0.0, np.zeros(72), np.zeros(4)]
    for r in range(world):
        ev.set_shard(r, world)
        c, gC, gT = ev.eval_discrete(T, Cc)
        exp = O.eval_discrete(O.config_from(cfg), occ, BMIN, 1.0, O.Shape.named("RoundedCone"), T, Cc, rank=r, world=world)
        check_eval((c, gC, gT), exp, what=f"shard {r}/{world}")
        acc[0] += c; acc[1] += gC; acc[2] += gT
    assert abs(acc[0] - full[0]) <= 1e-12 * abs(full[0]) and rel_l2(grads(acc[1], acc[2]), grads(full[1], full[2])) < 1e-12
    ev.close()


def test_errors_surface_as_status_and_nan_cost():
    cfg, occ, T, Cc, _ = small_case(N=2, K=4)
    ev = I.Evaluator(cfg)
    lib = ev.lib
    c = C.c_double(1.0)
    gC, gT = np.zeros(36), np.zeros(2)
    dp = C.POINTER(C.c_double)
    r = lib.isdf_eval_discrete(ev.h, 2, T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), C.byref(c), gC.ctypes.data_as(dp), gT.ctypes.data_as(dp))
    assert r == -2 and math.isnan(c.value) and b"shape" in lib.isdf_last_error()     # ISDF_ERR_STATE, NaN so the optimiser stops
    ev.set_shape_named("Ball")
    r = lib.isdf_eval_discrete(ev.h, 2, T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), C.byref(c), gC.ctypes.data_as(dp), gT.ctypes.data_as(dp))
    assert r == -2 and b"map" in lib.isdf_last_error()
    with pytest.raises(I.IsdfError):
        ev.set_shape_named("NoSuchShape")
    with pytest.raises(I.IsdfError):
        ev.set_shard(3, 2)
    V, F = W.box_mesh()
    with pytest.raises(I.IsdfError) as e:      # open mesh: the exact ±1 sign needs a closed surface ...
        ev.set_shape_mesh(V, F[:-1], None, I.MESH_SIGN_EXACT)
    assert e.value.code == -4
    with pytest.raises(I.IsdfError) as e:      # ... and a consistently oriented one (one flipped triangle)
        F2 = F.copy(); F2[0] = F2[0][::-1]
        ev.set_shape_mesh(V, F2, None, I.MESH_SIGN_EXACT)
    assert e.value.code == -4
    ev.set_shape_mesh(V, F[:-1])               # the automatic mode accepts both with the winding-number sign (tests/test_gpu_soup.py)
    ev.set_shape_mesh(V, F2)
    ev.close()


def test_discrete_golden_fixture():
    z = np.load(os.path.join(G, "discrete.npz"))
    occ = np.unpackbits(z["occ_bits"])[:np.prod(z["occ_shape"])].reshape(z["occ_shape"]).astype(np.uint8)
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = int(z["K"])
    s = np.load(os.path.join(G, "shapes.npz"))
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    for name in ["Ball", "CSG", "Trefoil", "SmoothIntersection"]:
        ev.set_shape_named(name, s["R"], s["t"])
        check_eval(ev.eval_discrete(z["T"], z["C"]), (float(z[f"{name}_cost"]), z[f"{name}_gradC"], z[f"{name}_gradT"]), what=name)
    V, F = MESHES["lprism"]()
    ev.set_shape_mesh(V, F, [0, 0, 0, 120, 0, 0])
    check_eval(ev.eval_discrete(z["T"], z["C"]), (float(z["mesh_cost"]), z["mesh_gradC"], z["mesh_gradT"]), what="mesh")
    ev.close()


# ---- swept-volume path -----------------------------------------------------------------------------------------------------------
def sv_case(N=4, seed=3, npts=400):
    cfg, occ, T, Cc, wp = small_case(N=N, K=16, seed=seed, noise=0.05)
    pts = W.gather_obstacle_points(occ, BMIN, 1.0, wp, cfg.kernel_size * cfg.occupancy_resolution / 3.0)[:npts]
    return cfg, T, Cc, pts


@pytest.mark.parametrize("name,tilt", [(n, False) for n in ["Ball", "Torus", "RoundedCone", "SmoothIntersection", "CSG", "TwistBox"]] +
                         [("CSG", True), ("TwistBox", True)])
def test_swept_tail_parity_given_tstar(name, tilt):
    """tier T1: chain-rule tail at the oracle's t*, sdf*, g_rel"""
    cfg, T, Cc, pts = sv_case()
    R, t = tilted() if tilt else (None, None)
    osh = O.Shape.named(name, R, t)
    ref = O.eval_swept(O.config_from(cfg), osh, T, Cc, pts)
    assert (ref["sdf"] < 9.99).sum() >= 10
    ev = I.Evaluator(cfg)
    ev.set_shape_named(name, R, t)
    ev.set_points(pts)
    got = ev.eval_swept_given(T, Cc, ref["tstar"], ref["sdf"], ref["grel"])
    check_eval(got, (ref["cost"], ref["gradC"], ref["gradT"]), tol=1e-9, what=f"T1 {name}")
    ev.close()


@pytest.mark.parametrize("tilt", [False, True], ids=["untilted", "tilted"])
@pytest.mark.parametrize("name", I.NAMED_SHAPES + ["Box"])
def test_swept_end_to_end_parity(name, tilt):
    """tier T2: device-side search. Same accept/reject decisions => same hit set, t*, SV-SDF, evaluation count and cost / gradient to
    rounding (strict: t* 1e-12, SV-SDF 1e-10, cost / gradient 1e-9) — for every shape, also TwistBox, BendBox and Trefoil, whose SDFs call
    sin / cos / atan2 (device and glibc results may differ in the last ulp; here that moves SV-SDF values by <= 7e-16, no decision).
    CappedCone has no hit: its SDF grows slowly with distance (0.3 at 3 m, 1.2 at 25 m), so every point stays within range at every coarse
    sample — one open run, dropped — and the test checks exactly that."""
    cfg, T, Cc, pts = sv_case(seed=5)
    R, t = tilted() if tilt else (None, None)
    if name == "Box":
        osh = O.Shape.analytic(I.SHAPE_KINDS["BOX"], [1.5, 0.3, 0.3], R, t)
    else:
        osh = O.Shape.named(name, R, t)
    ref = O.eval_swept(O.config_from(cfg), osh, T, Cc, pts)
    ev = I.Evaluator(cfg)
    if name == "Box":
        ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], [1.5, 0.3, 0.3], R, t)
    else:
        ev.set_shape_named(name, R, t)
    ev.set_points(pts)
    got = ev.eval_swept(T, Cc)
    ts, sd, gr = ev.swept_results()
    hit = ref["sdf"] < 9.99
    dt_all = np.abs(ts - ref["tstar"])
    dt, ds = dt_all[hit], np.abs(sd - ref["sdf"])[hit]
    evals = ev.stats().last_sdf_evals
    rc = abs(got[0] - ref["cost"]) / max(abs(ref["cost"]), 1e-300)
    rg = rel_l2(grads(got[1], got[2]), grads(ref["gradC"], ref["gradT"]))
    first = np.flatnonzero((dt_all > 1e-12) | ((sd < 9.99) != hit))
    print(f"{name} {'tilted' if tilt else 'untilted'}: points {len(pts)} hits {hit.sum()} max|dt*| {dt.max() if dt.size else 0:.1e} "
          f"max|dsdf| {ds.max() if ds.size else 0:.1e} cost rel {rc:.1e} grad rel-L2 {rg:.1e} evals {evals} vs {ref['nsdf']}"
          + (f"; first differing point {first[0]}: t* {ts[first[0]]!r} vs {ref['tstar'][first[0]]!r}, sdf {sd[first[0]]!r} vs {ref['sdf'][first[0]]!r}"
             if first.size else ""))
    assert np.array_equal(sd < 9.99, hit)
    if name == "CappedCone":
        assert hit.sum() == 0 and np.all(sd == 10.0) and got[0] == 0.0
    else:
        assert hit.sum() >= 5
    assert dt_all.max() <= 1e-12 and (ds.max() if ds.size else 0) <= 1e-10
    check_eval(got, (ref["cost"], ref["gradC"], ref["gradT"]), tol=1e-9, what=f"T2 {name}")
    assert evals == ref["nsdf"]
    ev.close()


@pytest.mark.parametrize("mesh,poly", [("lprism", None), ("rcone", None), ("rcone", [0.1, -0.05, 0.0, 120.0, 20.0, -35.0]), ("ico", None)])
def test_swept_end_to_end_mesh(mesh, poly):
    """mesh robots: CTA-per-point kernel (bracket-pruned scans, warp-cooperative searches, parallel step candidates) replays the
    reference's sequential search: same hit set, t*, SV-SDF values, reference-equivalent evaluation count, cost and gradient."""
    cfg, T, Cc, pts = sv_case(seed=7, npts=260)
    V, F = MESHES[mesh]()
    osh = O.Shape.mesh(V, F, poly) if poly is not None else O.Shape.mesh(V, F)
    ref = O.eval_swept(O.config_from(cfg), osh, T, Cc, pts)
    ev = I.Evaluator(cfg)
    ev.set_shape_mesh(V, F, poly)
    ev.set_points(pts)
    got = ev.eval_swept(T, Cc)
    ts, sd, gr = ev.swept_results()
    hit = ref["sdf"] < 9.99
    assert hit.sum() > 20 and np.array_equal(sd < 9.99, hit)
    dt = np.abs(ts - ref["tstar"])[hit]
    assert (dt <= 8e-5).mean() >= 0.99
    assert np.allclose(sd[hit], ref["sdf"][hit], rtol=0, atol=1e-6)
    check_eval(got, (ref["cost"], ref["gradC"], ref["gradT"]), tol=1e-6, what=f"T2 mesh {mesh}")
    assert ev.stats().last_sdf_evals == ref["nsdf"]
    # second evaluation: lastTstar carried over, identical result (the search does not depend on the previous t*)
    again = ev.eval_swept(T, Cc)
    assert again[0] == got[0] and np.array_equal(again[1], got[1]) and np.array_equal(again[2], got[2])
    # point shards (one rank per GPU) sum to the full evaluation
    acc = [0.0, np.zeros_like(got[1]), np.zeros_like(got[2])]
    for r in range(3):
        ev.set_shard(r, 3)
        c, gC, gT = ev.eval_swept(T, Cc)
        acc[0] += c; acc[1] += gC; acc[2] += gT
    assert abs(acc[0] - got[0]) <= 1e-12 * max(abs(got[0]), 1) and rel_l2(grads(acc[1], acc[2]), grads(got[1], got[2])) < 1e-12
    ev.close()


def test_swept_shards_sum_to_full_and_tstar_persists():
    cfg, T, Cc, pts = sv_case(seed=5)
    ev = I.Evaluator(cfg)
    ev.set_shape_named("Torus")
    ev.set_points(pts)
    full = ev.eval_swept(T, Cc)
    t_full, _, _ = ev.swept_results()
    acc = [0.0, np.zeros(72), np.zeros(4)]
    for r in range(3):
        ev.set_shard(r, 3)
        c, gC, gT = ev.eval_swept(T, Cc)
        acc[0] += c; acc[1] += gC; acc[2] += gT
    assert abs(acc[0] - full[0]) <= 1e-12 * max(abs(full[0]), 1) and rel_l2(grads(acc[1], acc[2]), grads(full[1], full[2])) < 1e-12
    t2, _, _ = ev.swept_results()
    assert np.array_equal(t2, t_full)
    ev.close()


def test_swept_golden_fixture():
    z = np.load(os.path.join(G, "swept.npz"))
    cfg, *_ = small_case(N=4, K=16, seed=3)
    ev = I.Evaluator(cfg)
    ev.set_points(z["pts"])
    for name in ["Ball", "Torus", "SmoothIntersection"]:
        ev.set_shape_named(name)
        got = ev.eval_swept(z["T"], z["C"])
        check_eval(got, (float(z[f"{name}_cost"]), z[f"{name}_gradC"], z[f"{name}_gradT"]), what=name)
    ev.close()


# ---- host adapters: the reference's callback / plug-in surface on top of the C ABI ------------------------------------------------
def test_lmbm_callback_matches_oracle_composition():
    """BackEnd::costFunctionLmbm (lmbm_evaluate_t) == forwardT/P -> MINCO -> energy -> swept + time-integral -> propogateGrad ->
    rho*sum(T) -> backwardGradT/P assembled from the oracle's pieces (back_end_optimizer.hpp:358-430)."""
    import ctypes as CT
    import host_lib as H
    cfg, T0, Cc, pts = sv_case(seed=5, npts=300)
    cfg.flags = I.WITH_DYNAMICS                       # the live reference: collision only through the swept-volume term
    cfg.vmax, cfg.omgmax = 1.2, 0.5                   # make the dynamic penalties active
    N = T0.size
    wp = W.random_walk_waypoints(N, [0, 0, 0], [50, 50, 34], seed=5)
    head, tail = np.zeros((3, 3)), np.zeros((3, 3))
    head[:, 0], tail[:, 0] = wp[0], wp[-1]
    rng = np.random.default_rng(1)
    tau = rng.normal(size=N) * 0.5 + 1.0
    x = np.concatenate([tau, wp[1:-1].reshape(-1)])
    rho = 20.0
    # oracle composition
    Tt = np.where(tau > 0, (0.5 * tau + 1) * tau + 1, 1 / ((0.5 * tau - 1) * tau + 1))
    co, energy, gC, gT = O.minco_forward(head, tail, wp[1:-1].T, Tt)
    osh = O.Shape.named("Torus")
    sv = O.eval_swept(O.config_from(cfg), osh, Tt, co, pts)
    di = O.eval_discrete(O.config_from(cfg), None, BMIN, 1.0, None, Tt, co)
    cost = energy + sv["cost"] + di[0] + rho * Tt.sum()
    gp, gt = O.minco_backward(head, tail, wp[1:-1].T, Tt, gC + sv["gradC"] + di[1], gT + sv["gradT"] + di[2])
    gt = gt + rho
    gtau = np.where(tau > 0, gt * (tau + 1), gt * (1 - tau) / ((0.5 * tau - 1) * tau + 1) ** 2)
    g_ref = np.concatenate([gtau, gp.T.reshape(-1)])
    # product
    ev = I.Evaluator(cfg)
    ev.set_shape_named("Torus")
    ev.set_points(pts)
    L = H.lib()
    hh, tt = np.asfortranarray(head), np.asfortranarray(tail)
    be = L.isdf_host_backend_create(ev.h, N, hh.ctypes.data_as(H.dp), tt.ctypes.data_as(H.dp), rho, 1, 1)
    g = np.zeros_like(x)
    c = L.isdf_host_backend_cost(be, x.ctypes.data_as(H.dp), g.ctypes.data_as(H.dp), x.size)
    cp, cother, ctot, st = CT.c_double(), CT.c_double(), CT.c_double(), CT.c_int()
    L.isdf_host_backend_last(be, CT.byref(cp), CT.byref(cother), CT.byref(ctot), CT.byref(st))
    L.isdf_host_backend_destroy(be)
    assert st.value == 0 and ctot.value == c
    assert abs(c - cost) <= 1e-6 * abs(cost), (c, cost)
    assert abs(cp.value - sv["cost"]) <= 1e-6 * max(abs(sv["cost"]), 1.0)
    assert rel_l2(g, g_ref) <= 1e-6
    # the single-point plug-in call goes through the same device SDF
    gr = np.zeros(3)
    p = np.array([1.0, 0.4, -0.2])
    s = L.isdf_host_shape_sdf_grad(ev.h, p.ctypes.data_as(H.dp), gr.ctypes.data_as(H.dp))
    os_, og = osh.query(p[None])
    assert abs(s - os_[0]) < 1e-12 and np.allclose(gr, og[0], atol=1e-8)
    ev.close()


def test_lbfgs_driver_on_gpu_callback_decreases_cost():
    """L-BFGS (reference fork semantics) over the full callback: MINCO -> swept-volume term -> time integral -> adjoint."""
    import ctypes as CT
    import host_lib as H
    cfg, T0, Cc, pts = sv_case(seed=5, npts=300)
    cfg.flags = I.WITH_DYNAMICS
    N = T0.size
    wp = W.random_walk_waypoints(N, [0, 0, 0], [50, 50, 34], seed=5)
    head, tail = np.zeros((3, 3)), np.zeros((3, 3))
    head[:, 0], tail[:, 0] = wp[0], wp[-1]
    x = np.concatenate([np.full(N, 1.2), wp[1:-1].reshape(-1)])
    ev = I.Evaluator(cfg)
    ev.set_shape_named("Torus")
    ev.set_points(pts)
    L = H.lib()
    hh, tt = np.asfortranarray(head), np.asfortranarray(tail)
    be = L.isdf_host_backend_create(ev.h, N, hh.ctypes.data_as(H.dp), tt.ctypes.data_as(H.dp), 20.0, 1, 1)
    g = np.zeros_like(x)
    c0 = L.isdf_host_backend_cost(be, x.ctypes.data_as(H.dp), g.ctypes.data_as(H.dp), x.size)
    fx, it, evs = CT.c_double(0), CT.c_int(0), CT.c_int(0)
    r = L.isdf_host_lbfgs_backend(be, x.ctypes.data_as(H.dp), x.size, CT.byref(fx), 16, 10, 1e-6, 0.0, 60, CT.byref(it), CT.byref(evs))
    L.isdf_host_backend_destroy(be)
    print("lbfgs ret", r, "cost", c0, "->", fx.value, "iterations", it.value, "evaluations", evs.value)
    assert r in (0, 1, -1008) or r <= -1009          # converged / stopped / max iterations / line-search limits: all leave the last iterate
    assert np.isfinite(fx.value) and fx.value < c0 and it.value >= 1 and evs.value >= it.value
    ev.close()


def test_batch_of_trajectories_as_one_concatenated_block():
    """BASELINE configs[4] in miniature: B random-restart trajectories evaluated in ONE call by concatenating their pieces;
    per-trajectory gradients are bit-identical to separate evaluations, per-trajectory costs come from the piece costs."""
    cfg, occ, _, _, _ = small_case(N=4, K=16, seed=3)
    B, N0 = 5, 4
    trajs = [W.make_trajectory(N0, [0, 0, 0], [50, 50, 34], seed=100 + b, jitter=0.3) for b in range(B)]
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    V, F = MESHES["rcone"]()
    ev.set_shape_mesh(V, F, [0, 0, 0, 120, 0, 0])
    singles = [ev.eval_discrete(T, Cc) for (T, Cc, _) in trajs]
    # column-major 6*(B*N0) x 3 block: per axis, the B trajectories' 6*N0 coefficients back to back
    Tall = np.concatenate([T for (T, _, _) in trajs])
    Call = np.concatenate([np.concatenate([Cc.reshape(3, 6 * N0)[ax] for (_, Cc, _) in trajs]) for ax in range(3)])
    c, gC, gT = ev.eval_discrete(Tall, Call)
    pc = ev.piece_costs(B * N0)
    gCm = gC.reshape(3, 6 * B * N0)
    for b in range(B):
        sc, sgC, sgT = singles[b]
        assert np.array_equal(gCm[:, 6 * N0 * b:6 * N0 * (b + 1)].reshape(-1), sgC)
        assert np.array_equal(gT[N0 * b:N0 * (b + 1)], sgT)
        assert abs(pc[N0 * b:N0 * (b + 1)].sum() - sc) <= 1e-12 * max(abs(sc), 1.0)
    assert abs(c - sum(s[0] for s in singles)) <= 1e-12 * abs(c)
    ev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("robot", ["Ball", "mesh"])
def test_batched_device_callback_matches_host_callback(robot):
    """SURVEY 8f row 1: the whole callback (forwardT -> MINCO -> energy -> time-integral term incl. the discrete collision loop ->
    propogateGrad -> rho*sum(T) -> backwardGradT/P) for B problems in one device call == the per-problem host adapter
    (host MINCO port pinned against the oracle) driving the same kernels; trajectories bit-identical to the host MINCO."""
    import host_lib as H
    cfg, occ, _, _, _ = small_case(N=6, K=16, seed=3)
    cfg.vmax, cfg.omgmax = 1.2, 0.5
    B, N0 = 7, 6
    rho = 20.0
    rng = np.random.default_rng(9)
    heads, tails, X = [], [], []
    for b in range(B):
        wp = W.random_walk_waypoints(N0, [0, 0, 0], [50, 50, 34], seed=200 + b)
        h, t = np.zeros((3, 3)), np.zeros((3, 3))
        h[:, 0], t[:, 0] = wp[0], wp[-1]
        h[:, 1] = rng.normal(size=3) * 0.3                          # non-zero boundary velocity
        tau = rng.normal(size=N0) * 0.6 + 0.6                       # both branches of forwardT
        X.append(np.concatenate([tau, (wp[1:-1] + rng.normal(size=(N0 - 1, 3)) * 0.2).reshape(-1)]))
        heads.append(h); tails.append(t)
    X = np.array(X)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        ev.set_shape_mesh(V, F, [0, 0, 0, 120, 0, 0])
    else:
        ev.set_shape_named(robot)
    L = H.lib()
    ref_c, ref_g, ref_co = [], [], []
    for b in range(B):
        hh, tt = np.asfortranarray(heads[b]), np.asfortranarray(tails[b])
        be = L.isdf_host_backend_create(ev.h, N0, hh.ctypes.data_as(H.dp), tt.ctypes.data_as(H.dp), rho, 0, 1)
        g = np.zeros(X.shape[1])
        ref_c.append(L.isdf_host_backend_cost(be, X[b].ctypes.data_as(H.dp), g.ctypes.data_as(H.dp), g.size))
        ref_g.append(g)
        L.isdf_host_backend_destroy(be)
        tau = X[b, :N0]
        Tt = np.where(tau > 0, (0.5 * tau + 1) * tau + 1, 1 / ((0.5 * tau - 1) * tau + 1))
        ref_co.append(H.minco_forward(heads[b], tails[b], X[b, N0:].reshape(-1, 3).T, Tt)[0])
    cost, grad = ev.callback_batch(np.array(heads), np.array(tails), rho, X)
    Tb, Cb, en = ev.batch_trajectories(B, N0)
    Cm = Cb.reshape(3, 6 * B * N0)
    for b in range(B):
        assert np.array_equal(Cm[:, 6 * N0 * b:6 * N0 * (b + 1)].reshape(-1), np.asarray(ref_co[b]).reshape(-1))
        assert abs(cost[b] - ref_c[b]) <= 1e-13 * abs(ref_c[b]), (b, cost[b], ref_c[b])
        assert rel_l2(grad[b], ref_g[b]) <= 1e-12, (b, rel_l2(grad[b], ref_g[b]))
    assert np.all(np.isfinite(cost)) and len(set(np.round(cost, 6))) == B
    # shared boundary conditions: one head/tail pair for the whole batch
    cost2, grad2 = ev.callback_batch(heads[0], tails[0], rho, X[:2])
    assert abs(cost2[0] - ref_c[0]) <= 1e-13 * abs(ref_c[0]) and rel_l2(grad2[0], ref_g[0]) <= 1e-12
    assert np.isfinite(cost2[1])
    ev.close()


def test_obstacle_gather_matches_reference_semantics():
    """plan_manager.cpp:232-254 + getPointsInAABBOutOfLastOne (pcs:182-216): same set, same (waypoint, address) order as the oracle."""
    cfg, occ, T, Cc, wp = small_case(N=6, K=8, seed=4, noise=0.08)
    half = cfg.kernel_size * cfg.occupancy_resolution / 3.0
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    for off in ([0.0, 0.0, 0.0], [0.5, -0.3, 1.2]):
        a, na = ev.gather_obstacle_points(wp[1:-1], half, off)
        b, nb = O.gather_obstacle_points(occ, BMIN, 1.0, wp[1:-1], half, off)
        assert na == nb and na > 50 and np.array_equal(a, b)
        assert len(np.unique(a, axis=0)) == na                     # de-duplicated
    # and it can feed the swept-volume path directly
    pts, n = ev.gather_obstacle_points(wp[1:-1], half, set_as_points=True)
    ev.set_shape_named("Torus")
    got = ev.eval_swept(T, Cc)
    ref = O.eval_swept(O.config_from(cfg), O.Shape.named("Torus"), T, Cc, pts)
    check_eval(got, (ref["cost"], ref["gradC"], ref["gradT"]), what="gather->swept")
    ev.close()


def test_multi_gpu_peer_memory_reduction():
    """isdf_peer_*: the sharded evaluation's sum over ranks through NVLink peer memory, fused into the epilogue kernel — needs >= 2
    GPUs in the box (skipped on the single-GPU test box; run with `gpurun --gpus 2`). See tests/multi_gpu_peer.py."""
    import subprocess, sys, torch
    ng = torch.cuda.device_count()
    if ng < 2:
        pytest.skip("needs at least 2 GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(min(ng, 8)), "--master-addr", "127.0.0.1",
           "--master-port", "29517", os.path.join(here, "multi_gpu_peer.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=240)
    assert r.returncode == 0 and "PEER OK" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


# ---- front end: attitude kernels (SURVEY 8f row 4) -------------------------------------------------------------------------------
@pytest.mark.parametrize("robot,ks", [("CappedCone", 13), ("TwistBox", 13), ("Torus", 9), ("Ball", 5), ("CSG", 13), ("Box", 13), ("mesh", 13), ("tilted", 13)])
def test_frontend_kernels_and_feasibility_bit_exact(robot, ks):
    """robot occupancy kernels per attitude (Shape.hpp:405-461), kernelConv<true> for every voxel x every attitude
    (sw_manager.hpp:821-846), checkKernelValue's first fit in BFS order (:852-941): all integer / boolean -> exact equality."""
    cfg, _, _, _, _ = small_case(N=2, K=4, seed=3, kernel_size=ks)
    X, Y, Z = 40, 36, 28
    occ = W.three_slit_map(X, Y, Z, noise=0.003, seed=5)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], cfg.occupancy_resolution)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        poly = [0.1, 0.0, -0.1, 120.0, 10.0, 0.0]
        ev.set_shape_mesh(V, F, poly); osh = O.Shape.mesh(V, F, poly)
    elif robot == "Box":
        ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], [1.5, 0.9, 0.4]); osh = O.Shape.analytic(I.SHAPE_KINDS["BOX"], [1.5, 0.9, 0.4])
    elif robot == "tilted":
        R, t = tilted()
        ev.set_shape_named("RoundedCone", R, t); osh = O.Shape.named("RoundedCone", R, t)
    else:
        ev.set_shape_named(robot); osh = O.Shape.named(robot)
    safeh = 0.8 if robot in ("Torus", "mesh") else 0.0
    assert ev.frontend_build_kernels(45.0, 45.0, 9.0, safeh) == (11, 11)
    fe = O.FrontEnd(osh, occ, ks=ks, res=cfg.occupancy_resolution, front_end_safeh=safeh)
    K = ev.frontend_kernels(ks)
    assert np.array_equal(K, fe.kernels()), f"{robot}: {(K != fe.kernels()).sum()} kernel voxels differ"
    assert 0 < K[60].sum() < ks ** 3
    masks = ev.frontend_feasibility(X, Y, Z)
    ix, iy, iz = np.meshgrid(np.arange(X), np.arange(Y), np.arange(Z), indexing="ij")
    ind = np.stack([ix, iy, iz], -1).reshape(-1, 3)
    ref = fe.feasibility(ind)
    assert np.array_equal(masks, ref), f"{robot}: {(masks != ref).any(axis=1).sum()} voxels differ"
    nfit = np.array([bin(int(w)).count("1") for w in masks.reshape(-1)]).reshape(-1, 4).sum(axis=1)
    assert (nfit == 0).any() and (nfit > 0).any()
    rng = np.random.default_rng(3)
    n = 3000
    q = ind[rng.integers(0, len(ind), n)]
    father = np.stack([rng.integers(-5, 6, n) * 9.0, rng.integers(-5, 6, n) * 9.0], 1)
    father[:50] += rng.uniform(0, 8.9, (50, 2)) * (father[:50] < 36)           # off-grid fathers truncate like the reference's int cast
    child, ok = ev.frontend_check_batch(q, father)
    rchild, rok = fe.check(q, father)
    assert np.array_equal(ok, rok) and np.array_equal(child, rchild)
    ev.close()


def test_frontend_state_errors():
    cfg, occ, _, _, _ = small_case(N=2, K=4, seed=3)
    ev = I.Evaluator(cfg)
    with pytest.raises(RuntimeError):
        ev.frontend_build_kernels()                        # no shape
    ev.set_shape_named("Torus")
    ev.frontend_build_kernels()
    with pytest.raises(RuntimeError):
        ev.frontend_feasibility(4, 4, 4)                   # no map
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_named("Ball")
    with pytest.raises(RuntimeError):
        ev.frontend_feasibility(*occ.shape)                # kernels are stale after a shape change
    with pytest.raises(RuntimeError):
        ev.frontend_build_kernels(45.0, 45.0, 1.0)         # 91 x 91 attitudes > 128
    ev.frontend_build_kernels()
    with pytest.raises(RuntimeError):
        ev.frontend_check_batch([[0, 0, occ.shape[2]]], [[0.0, 0.0]])   # voxel outside the map
    ev.close()


@pytest.mark.gpu
def test_frontend_two_pass_equals_one_pass_ragged_z():
    """the two-pass feasibility kernels (kernel core first, mask accumulation on the survivors) against the one-pass kernel and the
    oracle, on a map whose z extent is not a multiple of the z-run length and that is dense enough for the core to settle most voxels"""
    import os
    cfg, _, _, _, _ = small_case(N=2, K=4, seed=3, kernel_size=7)
    X, Y, Z = 37, 29, 43                                   # z: one full 32-voxel word + a ragged one, not a multiple of the run length
    occ = W.random_map(X, Y, Z, p=0.04, seed=9, slabs=1)
    V, F = MESHES["rcone"]()
    poly = [0.1, 0.0, -0.1, 120.0, 10.0, 0.0]
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], cfg.occupancy_resolution)
    ev.set_shape_mesh(V, F, poly)
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.8)
    two = ev.frontend_feasibility(X, Y, Z)                 # zero fill + bit-parallel core pass + table-driven accumulation
    os.environ["ISDF_FE_NO_TABLES"] = "1"
    try:
        two_b = ev.frontend_feasibility(X, Y, Z)           # core pass per z-run + offset-mask accumulation
    finally:
        del os.environ["ISDF_FE_NO_TABLES"]
    os.environ["ISDF_FE_ONE_PASS"] = "1"
    try:
        one = ev.frontend_feasibility(X, Y, Z)
    finally:
        del os.environ["ISDF_FE_ONE_PASS"]
    assert np.array_equal(one, two) and np.array_equal(one, two_b)
    fe = O.FrontEnd(O.Shape.mesh(V, F, poly), occ, ks=7, res=cfg.occupancy_resolution, front_end_safeh=0.8)
    ix, iy, iz = np.meshgrid(np.arange(X), np.arange(Y), np.arange(Z), indexing="ij")
    ref = fe.feasibility(np.stack([ix, iy, iz], -1).reshape(-1, 3))
    assert np.array_equal(two, ref)
    settled = (two == 0).all(axis=1).mean()
    assert 0.05 < settled < 1.0
    ev.close()
