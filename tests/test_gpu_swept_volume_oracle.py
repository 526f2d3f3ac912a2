"""Certified swept volume (isdf_swept_volume_*) on the GPU against tests/sweptvol_oracle.py: the kernel decision for decision against the
serial restatement of its refinement (sv_refine) on analytic shapes and an offset box mesh, at the budget, depth, interval-count and band
edges; an enclosure that uses no motion bound for mesh and offset robots in the three mesh-query regimes; grid-versus-point identity on
every node, culled and minimal grids, order independence; the scans beyond one top-level block and the mesh against marching_tets_np."""
import math
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import certify_oracle as CE
import sweptvol_oracle as SO
from test_gpu_swept_volume import box_mesh, line, path_points
from test_certify_cpu import aggressive_pieces

pytestmark = pytest.mark.gpu
BOX_HALF = [0.9, 0.5, 0.3]
ROT = np.linalg.qr(np.random.default_rng(11).normal(size=(3, 3)))[0]
TRANS = np.array([0.31, -0.22, 0.17])
MESH_SHIFT = np.array([1.3, 0.2, -0.1])      # the box mesh's body origin lies outside it
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]        # the bench robot's poly_params
GUARD = 1e-9                                 # no decision of a compared point lies closer than this to its threshold


# ---- shapes -------------------------------------------------------------------------------------------------------------------------
class Robot:
    """a swept-volume shape on the device and its oracle SDF; r_rot / r_body as the library derives them"""

    def __init__(self, name):
        self.name, self.mesh = name, None
        corners = None
        if name == "Point":
            self.osh = O.Shape.named("Point")
        elif name == "Ball":
            self.osh = O.Shape.analytic(I.SHAPE_KINDS["BALL"], [0.7])
        elif name == "Box":
            self.osh, corners = O.Shape.analytic(I.SHAPE_KINDS["BOX"], BOX_HALF), CE.box_corners(BOX_HALF)
        elif name == "BoxRT":
            self.osh = O.Shape.analytic(I.SHAPE_KINDS["BOX"], BOX_HALF, ROT, TRANS)
            corners = CE.box_corners(BOX_HALF, ROT, TRANS)
        else:
            if name == "BoxMesh":
                V, F = box_mesh(BOX_HALF)
                self.mesh = (V + MESH_SHIFT, F, None)
            elif name == "bench_mesh":
                V, F = W.rounded_cone_mesh(n_theta=24, n_prof=16)
                self.mesh = (V, F, PP)
            else:
                d = np.load(__file__.replace("test_gpu_swept_volume_oracle.py", "golden/ref_meshes.npz"))
                self.mesh = (d[name + "_V"], d[name + "_F"], d[name + "_pp"])
            self.osh = O.Shape.mesh(self.mesh[0], self.mesh[1], self.mesh[2], wn_mode=O.WN_EXACT)
            lo, hi = self.mesh[0].min(axis=0), self.mesh[0].max(axis=0)
            corners = [[hi[0] if k & 1 else lo[0], hi[1] if k & 2 else lo[1], hi[2] if k & 4 else lo[2]] for k in range(8)]
        if corners is None:
            self.r_rot, self.r_body = 0.0, (0.7 if name == "Ball" else 0.0) * (1 + 1e-12)
        else:
            self.r_rot = self.r_body = float(np.linalg.norm(np.asarray(corners, float), axis=1).max()) * (1 + 1e-12)

    def set_on(self, ev):
        if self.name == "Point":
            ev.set_shape_named("Point")
        elif self.name == "Ball":
            ev.set_shape_analytic(I.SHAPE_KINDS["BALL"], [0.7])
        elif self.name == "Box":
            ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], BOX_HALF)
        elif self.name == "BoxRT":
            ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], BOX_HALF, ROT.reshape(-1), TRANS)
        else:
            ev.set_shape_mesh(self.mesh[0], self.mesh[1], self.mesh[2], I.MESH_SIGN_EXACT)

    def sdf(self, q):
        return self.osh.query(q, what=0)[0]


# ---- trajectories -------------------------------------------------------------------------------------------------------------------
def concat(*trajs):
    T = np.concatenate([np.asarray(t, float).reshape(-1) for t, _ in trajs])
    Cc = np.concatenate([np.asarray(c, float).reshape(3, -1) for _, c in trajs], axis=1).reshape(-1)
    return T, Cc


def rest(x, Tt):
    c = np.zeros((3, 6))
    c[:, 0] = x
    return np.array([Tt]), c.reshape(-1)


def trajectory(name):
    if name == "traj":
        return W.make_trajectory(3, [0, 0, 0], [6, 4, 3], seed=4, jitter=0.4)[:2]
    if name == "aggressive":   # the 80 degree / large-jerk piece and a random quintic of the certificate's CPU test
        agg = {n: (T, Cc) for n, T, Cc in aggressive_pieces()}
        return concat(agg["tilt80_jerk"], agg["random0"])
    if name == "single":
        return W.make_trajectory(1, [0, 0, 0], [3, 2, 1], seed=2, jitter=0.0)[:2]
    if name == "short":        # a 1e-3 s piece between long ones
        T, Cc = W.make_trajectory(3, [0, 0, 0], [6, 4, 3], seed=5, jitter=0.4)[:2]
        T = np.array(T, float)
        T[1] = 1e-3
        return T, Cc
    if name == "return":       # out, a rest (exact ties: t* is the earliest), and back 0.3 m higher: two windows compete for t*
        a, b = np.array([0.0, 0.0, 0.0]), np.array([3.0, 1.0, 0.5])
        return concat(line(a, b, 1.5), rest(b + [0.0, 0.6, 0.4], 0.5), line(b + [0, 0, 0.3], a + [0, 0, 0.3], 1.5))
    if name == "long":         # 12 pieces: at K = 3 interval 32 (the second 32-lane chunk's first) shares a sample with interval 31
        return W.make_trajectory(12, [0, 0, 0], [12, 8, 6], seed=7, jitter=0.3)[:2]
    raise KeyError(name)


def pos_at(T, Cc, tt):
    toff = np.concatenate([[0.0], np.cumsum(T)[:-1]])
    i = int(np.clip(np.searchsorted(toff, tt, side="right") - 1, 0, len(T) - 1))
    return np.asarray(Cc).reshape(3, -1)[:, 6 * i:6 * i + 6] @ ((tt - toff[i]) ** np.arange(6))


def points_for(robot, T, Cc, band, seed, m=16):
    """path_points, plus points at r_body + band +- 1e-6 from the path"""
    rng = np.random.default_rng(seed)
    P = [path_points(T, Cc, rng, m)]
    for k in range(6):
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        P.append((pos_at(T, Cc, rng.uniform(0, np.sum(T))) + u * (robot.r_body + band + (1e-6 if k % 2 else -1e-6)))[None])
    return np.concatenate(P)


def grid_7x6x5(T, Cc, res, seed):
    """a 7 x 6 x 5 grid (partial bricks in every direction) around a path point"""
    rng = np.random.default_rng(seed)
    g = I.SweptGrid()
    c = pos_at(T, Cc, rng.uniform(0.2, 0.8) * np.sum(T))
    g.bmin[:] = [float(x) for x in c - res * np.array([3.0, 2.5, 2.0]) + rng.uniform(-0.3, 0.3, 3) * res]
    g.res = res
    g.X, g.Y, g.Z = 7, 6, 5
    return g


def make_ev(K=8):
    cfg = I.default_config_values()
    cfg.integral_intervs = K
    return I.Evaluator(cfg), cfg


# ---- 4. the kernel against the restatement ------------------------------------------------------------------------------------------
# (id, robot, trajectory, params, edge): a chosen dozen of K x max_depth x max_samples x tol x band, each with the edge it must reach
CASES = [
    ("point-traj-default", "Point", "traj", dict(K=8), None),
    ("ball-aggressive-K1", "Ball", "aggressive", dict(K=1, tol=1e-3), None),
    ("box-single-depth0", "Box", "single", dict(K=3, max_depth=0, tol=1e-3), "depth"),
    ("boxrt-short-depth1", "BoxRT", "short", dict(K=8, max_depth=1, tol=1e-3), "depth"),
    ("ball-return-ms0", "Ball", "return", dict(K=8, max_samples=0, tol=1e-3), "budget"),
    ("point-return-ms1", "Point", "return", dict(K=3, max_samples=1, tol=1e-3), "partial"),
    ("point-long-ms31", "Point", "long", dict(K=3, max_samples=31, tol=1e-9, band=20.0), "partial"),
    ("point-long-ms32", "Point", "long", dict(K=3, max_samples=32, tol=1e-9, band=20.0), "partial"),
    ("ball-long-ms33", "Ball", "long", dict(K=3, max_samples=33, tol=1e-9, band=20.0), "partial"),
    ("point-long-band20", "Point", "long", dict(K=3, tol=1e-3, band=20.0), "chunk"),
    ("ball-traj-narrow", "Ball", "traj", dict(K=3, tol=1e-3, band=1.5e-3), "inside"),
    # band below the mesh's sign_radius: the mesh query is unbounded, so the device and the oracle both return the exact distance
    ("boxmesh-return-unbounded", "BoxMesh", "return", dict(K=8, tol=1e-3, band=0.5), None),
    ("boxrt-aggressive-tol9", "BoxRT", "aggressive", dict(K=3, tol=1e-9, band=20.0, max_samples=512), None),
]


def refine_all(cfg, robot, T, Cc, prm, P):
    prep = SO.SvPrep(cfg, T, Cc, robot.r_rot, prm)
    return [SO.sv_refine(cfg, T, Cc, p, robot.sdf, robot.r_rot, robot.r_body, prm, prep) for p in P]


def compare(ref, v, lo, ts, dec, what):
    for k, r in enumerate(ref):
        assert r["margin"] > GUARD, (what, k, "fixture: a decision within 1e-9 of its threshold", r["margin"])
        assert bool(dec[k]) == r["decided"], (what, k, r, v[k], lo[k], dec[k])
        assert abs(v[k] - r["value"]) <= 1e-12, (what, k, v[k], r["value"])
        assert lo[k] == r["lower"] or abs(lo[k] - r["lower"]) <= 1e-9, (what, k, lo[k], r["lower"])
        if r["tgap"] > 1e-12:   # the earliest time of the smallest value
            assert ts[k] == r["tstar"], (what, k, ts[k], r["tstar"], r["tgap"])
        else:                   # a sample within rounding of the smallest value (e.g. both sides of a junction)
            assert ts[k] in r["near"], (what, k, ts[k], r["near"])
    assert sum(r["tgap"] > 1e-12 for r in ref) >= 0.5 * len(ref), (what, "fixture: t* mostly compared exactly")


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_kernel_matches_restatement(case):
    name, rname, tname, kw, edge = case
    robot = Robot(rname)
    T, Cc = trajectory(tname)
    ev, cfg = make_ev()
    robot.set_on(ev)
    prm = ev.swept_params(K=kw.get("K"), band=kw.get("band"), tol=kw.get("tol"), max_depth=kw.get("max_depth"),
                          max_samples=kw.get("max_samples"))
    P = points_for(robot, T, Cc, prm.band, seed=len(name))
    ref = refine_all(cfg, robot, T, Cc, prm, P)
    v, lo, ts, dec = ev.swept_volume_sdf(T, Cc, P, prm)
    compare(ref, v, lo, ts, dec, name)
    # the 7 x 6 x 5 grid: every node, and the counters against the restatement's sums
    g = grid_7x6x5(T, Cc, 0.11 if prm.band > 1e-2 else 2e-4, seed=len(name))
    gv, glo, gts, gdec, info = ev.swept_volume_grid(T, Cc, g, prm)
    nodes = I.swept_grid_nodes(g).reshape(-1, 3)
    gref = refine_all(cfg, robot, T, Cc, prm, nodes)
    compare(gref, gv.reshape(-1), glo.reshape(-1), gts.reshape(-1), gdec.reshape(-1), name + " grid")
    assert info["sdf_evals"] == sum(r["evals"] for r in gref), (info, sum(r["evals"] for r in gref))
    assert info["undecided"] == sum(not r["decided"] for r in gref)
    assert info["deepest"] == max(r["deepest"] for r in gref)
    assert info["bricks"] == 2 * 2 * 2
    allr = ref + gref
    # the case reaches its edge
    if edge == "depth":
        assert any(r["depth_cut"] for r in allr)
    elif edge == "budget":
        assert any(r["budget_cut"] for r in allr)
    elif edge == "partial":
        assert any(r["partial"] and r["max_wanting"] > prm.max_samples_per_point for r in allr)
    elif edge == "chunk":   # interval 32, the first of the second 32-lane chunk, reuses interval 31's last sample
        assert any(32 in r["shared"] for r in ref)
    elif edge == "inside":
        assert any(r["value"] < 0 for r in allr) and any(r["tstar"] == -1.0 for r in allr)
    if tname == "return" and robot.mesh is None:   # the rest piece: samples at different times attain value exactly, and t* is compared exactly
        assert any(r["ties"] > 1 and r["tgap"] > 1e-12 for r in ref)
    if robot.mesh is not None:   # a band below sign_radius: the unbounded mesh query, exact at every distance
        assert prm.band < ev.dbg_mesh_grid(arrays=False)["sign_radius"]
    assert any(r["value"] < prm.band for r in allr)
    ev.close()


# ---- 5. an enclosure that uses no motion bound: mesh and offset robots --------------------------------------------------------------
def enclosure(robot, cfg, T, Cc, P, v, lo, ts, dec, prm, n=1001):
    toff = np.concatenate([[0.0], np.cumsum(T)[:-1]])
    for k in range(len(P)):
        d, _ = SO.dense_sv(cfg, T, Cc, P[k], robot.sdf, n=n, polish=40)
        assert lo[k] <= d + 1e-9, (robot.name, k, lo[k], d)
        if v[k] < prm.band:   # value is attained at t*: value >= SV with no appeal to D
            i = int(np.clip(np.searchsorted(toff, ts[k], side="right") - 1, 0, len(T) - 1))
            sd = SO._sd(cfg, T, Cc, [i], [ts[k] - toff[i]], P[k], robot.sdf)[0]
            assert abs(sd - v[k]) <= 1e-9, (robot.name, k, sd, v[k])
        if dec[k]:
            assert v[k] <= d + prm.tol + 1e-9, (robot.name, k, v[k], d)
            if v[k] == prm.band:
                assert d >= prm.band - prm.tol - 1e-9, (robot.name, k, d)


@pytest.mark.parametrize("rname", ["bench_mesh", "Lthick", "RoundedCone", "BoxMesh", "BoxRT"])
def test_enclosure_mesh_and_offset_robots(rname):
    robot = Robot(rname)
    ev, cfg = make_ev()
    robot.set_on(ev)
    T, Cc = W.make_trajectory(2, [0, 0, 0], [6, 4, 3], seed=5, jitter=0.4)[:2]
    bands = [None]
    if robot.mesh is not None:
        gm = ev.dbg_mesh_grid(arrays=False)
        assert 0 < gm["sign_radius"] < gm["gpad"], gm
        bands = [0.5 * gm["sign_radius"], None, gm["gpad"] + 1.0]
    nund = 0
    for band in bands:
        for ms in ((None, 64) if band is None else (None,)):
            prm = ev.swept_params(band=band, max_samples=ms)
            if robot.mesh is not None:   # the regime of the mesh query each band selects
                if band is not None and band < gm["sign_radius"]:
                    assert prm.band < gm["sign_radius"]   # unbounded query
                elif band is None:
                    assert gm["sign_radius"] <= prm.band <= gm["gpad"]
                else:
                    assert prm.band > gm["gpad"]
            P = points_for(robot, T, Cc, prm.band, seed=3, m=14)
            v, lo, ts, dec = ev.swept_volume_sdf(T, Cc, P, prm)
            enclosure(robot, cfg, T, Cc, P, v, lo, ts, dec, prm)
            if ms == 64:
                nund += int(np.sum(dec == 0))
    assert nund > 0, "fixture: the capped runs leave undecided points"
    ev.close()


# ---- 6. grid structure and order independence ------------------------------------------------------------------------------------------
def grid_vs_points(ev, T, Cc, g, prm):
    v, lo, ts, dec, info = ev.swept_volume_grid(T, Cc, g, prm)
    nodes = I.swept_grid_nodes(g).reshape(-1, 3)
    pv, plo, pts_, pdec = ev.swept_volume_sdf(T, Cc, nodes, prm)
    for a, b in ((v, pv), (lo, plo), (ts, pts_), (dec, pdec)):
        assert np.array_equal(a.reshape(-1), b)
    return v, lo, ts, dec, info


def test_grid_equals_points_on_every_node():
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = trajectory("traj")
    prm = ev.swept_params()
    g = I.SweptGrid()
    g.bmin[:] = [-1.0, -1.0, -5.4]
    g.res, g.X, g.Y, g.Z = 0.1, 37, 22, 13
    v, _, _, _, info = grid_vs_points(ev, T, Cc, g, prm)
    assert 0 < info["bricks_culled"] < info["bricks"] and (v < 0).any() and (v == prm.band).any()
    # the cone mesh on a smaller grid
    V, F = W.rounded_cone_mesh(n_theta=16, n_prof=12)
    ev.set_shape_mesh(V, F, None, I.MESH_SIGN_EXACT)
    T2, C2 = W.make_trajectory(2, [0, 0, 0], [6, 4, 3], seed=5, jitter=0.4)[:2]
    g3 = I.swept_grid_for(T2, C2, 2.5, prm.band, 0.7)
    v3, _, _, _, _ = grid_vs_points(ev, T2, C2, g3, ev.swept_params(max_samples=64))
    assert (v3 < 0).any()
    ev.close()


def brick_edges(cfg, n, seed=0):
    """(x0, bmin, res, band) of one-brick grids at the brick cull's threshold: a Point resting at x0 (so D_e is the pose pad alone), the
    brick's nearest corner on the ray from x0 through its centre, and band set to the brick's bound before its slack, where the corner's
    own bound lies below it. Without the slack the brick would drop the interval while the corner node keeps it."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        x0 = rng.uniform(-60, 60, 3) * rng.choice([1e-3, 1.0, 10.0])
        res, dist = float(rng.uniform(0.01, 1.0)), float(rng.uniform(1.0, 10.0))
        sgn = rng.choice([-1.0, 1.0], 3)
        c = np.zeros((3, 6))
        c[:, 0] = x0
        corner = x0 + sgn * dist / math.sqrt(3)
        bmin = [float(corner[a]) if sgn[a] > 0 else float(corner[a] - 3 * res) for a in range(3)]
        p = [bmin[a] + (0.0 if sgn[a] > 0 else 3.0) * res for a in range(3)]
        band = dist
        for _ in range(3):   # D_e depends on band (H = band): iterate to the fixed point
            D = CE.bound(cfg, 0.0, band, c, 0.0, 1.0, 0.0)
            nl, bl = SO.node_cull_bound(p, x0, 0.0, D), SO.brick_cull_bound(bmin, res, (0, 0, 0), (3, 3, 3), x0, 0.0, D)
            if not nl < bl:
                break
            if band == bl:
                assert nl < band <= bl and abs(nl - band) <= 1e-9 * band
                out.append((x0, bmin, res, band, p))
                break
            band = bl
    return out


def test_grid_equals_points_at_the_brick_cull_threshold():
    """one-brick grids whose corner node's cull bound lies within an ulp below band while the brick's bound without its slack reaches
    band: the node keeps the interval, so the brick must keep it too (not culled, SDF evaluations made) and every node must equal its
    point query. At this threshold a node's value and lower bound are band either way, so the brick's decision shows in the counters."""
    ev, cfg = make_ev()
    ev.set_shape_named("Point")
    for x0, bmin, res, band, p in brick_edges(cfg, 24):
        c = np.zeros((3, 6))
        c[:, 0] = x0
        T, Cc = np.array([1.0]), c.reshape(-1)
        prm = ev.swept_params(K=1, band=band)
        g = I.SweptGrid()
        g.bmin[:] = bmin
        g.res, g.X, g.Y, g.Z = res, 4, 4, 4
        v, lo, ts, dec, info = grid_vs_points(ev, T, Cc, g, prm)
        assert info["bricks"] == 1 and info["bricks_culled"] == 0 and info["sdf_evals"] > 0, (x0, bmin, res, band, info)
    ev.close()


def test_all_culled_and_minimal_grids():
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = trajectory("traj")
    prm = ev.swept_params()
    g = I.SweptGrid()
    g.bmin[:] = [40.0, 40.0, 40.0]
    g.res, g.X, g.Y, g.Z = 0.5, 9, 6, 5
    v, lo, ts, dec, info = ev.swept_volume_grid(T, Cc, g, prm)
    assert (v == prm.band).all() and (lo == prm.band).all() and (ts == -1.0).all() and (dec == 1).all()
    assert info["bricks_culled"] == info["bricks"] == 3 * 2 * 2 and info["sdf_evals"] == 0 and info["undecided"] == 0
    # 2 x 2 x 2 across the surface: the restatement's field and mesh
    c = pos_at(T, Cc, 1.0)
    g2 = I.SweptGrid()
    g2.bmin[:] = [float(x) for x in c + [0.55, 0.05, -0.4]]
    g2.res, g2.X, g2.Y, g2.Z = 0.5, 2, 2, 2
    v2, lo2, ts2, dec2, info2 = grid_vs_points(ev, T, Cc, g2, prm)
    assert info2["bricks"] == 1 and (v2 < 0).any() and (v2 > 0).any()
    V, vt, F, _ = ev.swept_volume_mesh(T, Cc, g2, prm)
    RV, Rvt, RF = SO.marching_tets_np(v2, ts2, list(g2.bmin), g2.res)
    assert len(F) > 0 and np.array_equal(V, RV) and np.array_equal(vt, Rvt) and np.array_equal(F, RF)
    ev.close()


def test_order_independence():
    ev, cfg = make_ev()
    V, F = W.rounded_cone_mesh(n_theta=16, n_prof=12)
    ev.set_shape_mesh(V, F, None, I.MESH_SIGN_EXACT)
    T, Cc = W.make_trajectory(2, [0, 0, 0], [6, 4, 3], seed=5, jitter=0.4)[:2]
    prm = ev.swept_params(max_samples=64)
    P = points_for(Robot("bench_mesh"), T, Cc, prm.band, seed=9, m=60)
    base = ev.swept_volume_sdf(T, Cc, P, prm)
    rng = np.random.default_rng(0)
    perm = rng.permutation(len(P))
    sh = ev.swept_volume_sdf(T, Cc, P[perm], prm)
    for a, b in zip(base, sh):
        assert np.array_equal(a[perm], b)
    for chunk in (1, 33):
        parts = [ev.swept_volume_sdf(T, Cc, P[s:s + chunk], prm) for s in range(0, len(P), chunk)]
        for j in range(4):
            assert np.array_equal(np.concatenate([p[j] for p in parts]), base[j])
    ev.close()


# ---- 7. scans and mesh at scale and at edges --------------------------------------------------------------------------------------------
def test_field_scan_beyond_one_top_block():
    """4100 x 4100 x 4 nodes: 1025^2 > 2^20 bricks, so k_sv_scan_top loops; the field through the device entry into torch buffers. Bricks
    are numbered x-major: brick 2^20 is (bx, by) = (1023, 1), so the path runs near x = bmin + 4092 res and live bricks lie on both sides
    of it, and the top loop's second pass carries the offsets of live bricks."""
    import torch
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = line([39.9, -0.9, 0.6], [39.95, 0.6, 0.9], 2.0)
    prm = ev.swept_params(K=4)
    g = I.SweptGrid()
    g.bmin[:] = [-1.0, -1.0, 0.1]
    g.res, g.X, g.Y, g.Z = 0.01, 4100, 4100, 4
    n = g.X * g.Y * g.Z
    dT, dC = torch.from_numpy(np.ascontiguousarray(T)).cuda(), torch.from_numpy(np.ascontiguousarray(Cc)).cuda()
    dv, dt = (torch.empty(n, dtype=torch.float64, device="cuda") for _ in range(2))
    dd = torch.empty(n, dtype=torch.uint8, device="cuda")
    info = ev.swept_volume_grid_device(len(T), dT.data_ptr(), dC.data_ptr(), g, prm, dv.data_ptr(), 0, dt.data_ptr(), dd.data_ptr(),
                                       stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert info["bricks"] == 1025 * 1025 * 1 > 2 ** 20 and 0 < info["bricks_culled"] < info["bricks"]
    below = torch.nonzero(dv < prm.band).reshape(-1)
    rng = np.random.default_rng(4)
    sel = np.concatenate([below.cpu().numpy(), rng.integers(0, n, 10000)])
    v, t, d = dv[torch.from_numpy(sel).cuda()].cpu().numpy(), dt[torch.from_numpy(sel).cuda()].cpu().numpy(), dd[torch.from_numpy(sel).cuda()].cpu().numpy()
    del dv, dt, dd
    torch.cuda.empty_cache()
    ix, r = np.divmod(sel, g.Y * g.Z)
    iy, iz = np.divmod(r, g.Z)
    P = np.stack([g.bmin[0] + ix * g.res, g.bmin[1] + iy * g.res, g.bmin[2] + iz * g.res], 1)
    pv, _, pts_, pdec = ev.swept_volume_sdf(T, Cc, P, prm)
    assert below.numel() > 10000
    live = (ix[:below.numel()] // 4) * 1025 + iy[:below.numel()] // 4   # brick addresses of the nodes below band (BZ = 1)
    assert live.min() < 2 ** 20 <= live.max(), (live.min(), live.max())
    assert np.array_equal(pv, v) and np.array_equal(pts_, t) and np.array_equal(pdec, d)
    ev.close()


def test_mesh_beyond_2_20_nodes():
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = line([0.0, 0.0, 0.0], [4.0, 1.0, 0.5], 2.0)
    prm = ev.swept_params()
    g = I.SweptGrid()
    g.bmin[:] = [-1.6, -1.6, -1.55]
    g.res, g.X, g.Y, g.Z = 0.055, 130, 130, 70
    assert g.X * g.Y * g.Z > 2 ** 20
    v, lo, ts, dec, _ = ev.swept_volume_grid(T, Cc, g, prm)
    V, vt, F, _ = ev.swept_volume_mesh(T, Cc, g, prm)
    RV, Rvt, RF = SO.marching_tets_np(v, ts, list(g.bmin), g.res)
    assert len(F) > 10000 and np.array_equal(V, RV) and np.array_equal(vt, Rvt) and np.array_equal(F, RF)
    ev.close()


def test_mesh_of_a_cut_grid():
    """a grid that cuts through the swept body: bit identity with the restatement, and every edge used by one triangle only lies on the
    grid's outer faces"""
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = trajectory("traj")
    prm = ev.swept_params()
    g = I.swept_grid_for(T, Cc, 1.0, prm.band, 0.3)
    g.X = g.X // 2   # cut across the path
    v, lo, ts, dec, _ = ev.swept_volume_grid(T, Cc, g, prm)
    V, vt, F, _ = ev.swept_volume_mesh(T, Cc, g, prm)
    RV, Rvt, RF = SO.marching_tets_np(v, ts, list(g.bmin), g.res)
    assert np.array_equal(V, RV) and np.array_equal(vt, Rvt) and np.array_equal(F, RF)
    cnt = {}
    for a, b, c in F:
        for u, w in ((a, b), (b, c), (c, a)):
            cnt[(min(u, w), max(u, w))] = cnt.get((min(u, w), max(u, w)), 0) + 1
    open_edges = [e for e, k in cnt.items() if k == 1]
    assert open_edges, "fixture: the grid cuts the surface"
    hi = np.array(g.bmin[:]) + g.res * (np.array([g.X, g.Y, g.Z]) - 1)
    lo_ = np.array(g.bmin[:])
    for e in open_edges:
        for x in V[list(e)]:
            assert np.any(np.abs(x - lo_) <= 1e-9) or np.any(np.abs(x - hi) <= 1e-9), (e, x)
    assert all(k <= 2 for k in cnt.values())
    ev.close()


def test_vtime_with_band_below_res():
    """band < res: an edge between an inside node and a band-capped one takes the t* of the endpoint with the smaller |value|, which is
    the capped node's -1 when band is smaller than the inside value's magnitude (include/isdf.h states that -1 can occur)"""
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = trajectory("traj")
    prm = ev.swept_params(band=0.1)
    g = I.swept_grid_for(T, Cc, 1.0, prm.band, 0.35)
    v, lo, ts, dec, _ = ev.swept_volume_grid(T, Cc, g, prm)
    V, vt, F, _ = ev.swept_volume_mesh(T, Cc, g, prm)
    RV, Rvt, RF = SO.marching_tets_np(v, ts, list(g.bmin), g.res)
    assert np.array_equal(V, RV) and np.array_equal(vt, Rvt) and np.array_equal(F, RF)
    assert (vt == -1.0).any() and (vt >= 0).any(), "fixture: both kinds of vertex time"
    ev.close()
