"""The exact culls and bounded searches of the mesh path, tested where they can go wrong: at the hinge boundary, across safety
margin, mesh scale, map resolution and the pose-window field limit.

Every case evaluates a grazing scene (tests/grazing.py: all occupied voxels within [delta/4, delta] of sdf = safety_hor, on
either side) against the oracle at 1e-9 relative cost / rel-L2 gradient. The fixture's sensitivity figure (the smallest
single-voxel share of the cost) is asserted to be >= 100x that bar, so losing any one grazing voxel fails the case. Per-piece
costs are compared with the oracle run on one-piece slices. A random-map scene at the same config is compared at the 1e-6 bar
of the other parity tests. isdf_dbg_mesh_grid classifies the grazing (and random-scene) pairs by the search branch that
answers them, and each case asserts a minimum count for the branch it targets, so a case cannot silently stop reaching it.

Winding-sign meshes have no distance cull (every voxel in the box is answered) and their sign factor comes from a Barnes-Hut
tree that the oracle does not replicate bit for bit; there the grazing band and the 1e-9 reference use the library's own
unculled isdf_shape_query, and the oracle is checked at the winding-sign bar of test_gpu_soup.py."""
import os
import time
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import grazing as G
from common import rel_l2

pytestmark = pytest.mark.gpu
TOL = 1e-9                 # grazing scenes: legitimate differences are rounding of x >= delta/4 (~1e-12 relative)
TOL_RANDOM = 1e-6          # random maps: the bar of test_gpu_parity.py / test_gpu_configs.py
NTHREADS = max(1, min(len(os.sched_getaffinity(0)), 16))
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]      # the bench robot's poly_params


def make_cfg(safety=0.866, ks=13, eps=1e-2, K=8):
    cfg = I.default_config_values()
    cfg.flags = I.WITH_COLLISION            # collision only: the whole cost is the hinge
    cfg.safety_hor, cfg.kernel_size, cfg.smoothing_eps, cfg.integral_intervs = safety, ks, eps, K
    return cfg


def ocfg_of(cfg):
    oc = O.config_from(cfg)
    oc.threads_num = NTHREADS
    return oc


class Robot:
    """one shape on both sides: the library (set_on) and the oracle (osh); aabb = body-frame vertex box of an exact-sign mesh"""

    def __init__(self, kind, *args, sign_mode=I.MESH_SIGN_AUTO, scale=1.0):
        self.kind, self.args, self.sign_mode, self.aabb = kind, args, sign_mode, None
        if kind == "mesh":
            V, F = args
            self.V, self.F = V * scale, F
            self.osh = O.Shape.mesh(self.V, F, PP, wn_mode=O.WN_RAW if sign_mode == I.MESH_SIGN_WINDING else O.WN_BH)
            R, t = W.rotation_from_poly_params(PP)
            Vb = self.V @ R.T + t
            if sign_mode != I.MESH_SIGN_WINDING:                     # s = 1 - 2 w is no distance function: no shell pre-filter
                self.aabb = (Vb.min(0), Vb.max(0))
        elif kind == "named":
            self.osh = O.Shape.named(args[0])

    def set_on(self, ev):
        if self.kind == "mesh":
            ev.set_shape_mesh(self.V, self.F, PP, self.sign_mode)
        else:
            ev.set_shape_named(self.args[0])

    @property
    def winding(self):
        return self.kind == "mesh" and self.sign_mode == I.MESH_SIGN_WINDING


class DeviceSdf:
    """the library's unculled shape query in the oracle Shape's calling convention"""

    def __init__(self, ev):
        self.ev = ev

    def query(self, p, what=0):
        p = np.asarray(p, float).reshape(-1, 3)
        if p.shape[0] == 0:
            return np.zeros(0), np.zeros((0, 3))
        return self.ev.shape_query(p, I.QUERY_SDF)[0], None


def check(got, exp, tol, what):
    relc = abs(got[0] - exp[0]) / max(abs(exp[0]), 1e-300)
    relg = rel_l2(np.concatenate([got[1], got[2]]), np.concatenate([exp[1], exp[2]]))
    assert relc <= tol and relg <= tol, f"{what}: cost rel {relc:.3e}, grad rel-L2 {relg:.3e} (bar {tol:.0e})"
    return relc, relg


def piece_slice(T, Cc, i):
    N = len(T)
    return T[i:i + 1], np.ascontiguousarray(np.asarray(Cc).reshape(3, 6 * N)[:, 6 * i:6 * i + 6]).reshape(-1)


def random_scene_pairs(cfg, occ, bmin, res, T, Cc):
    """body-frame positions of every (sample, occupied voxel) pair in the box — what the scan kernel culls or answers"""
    oc = O.config_from(cfg)
    pos, R, _, _ = G.sample_poses(oc, T, Cc)
    flat = occ.reshape(-1)
    return np.concatenate([prel[flat[vid] != 0] for _, vid, prel, _ in G.window_pairs(oc, bmin, res, occ.shape, pos, R)])


def run_discrete(what, cfg, robot, T, Cc, bmin, res, dims, delta=1e-3, target=None, scene=None, min_active=20, straddle=False, region=None):
    """grazing scene (1e-9) + optional random scene (1e-6) at one operating point; returns (grid, grazing counts, scene counts)"""
    t0 = time.time()
    N = len(T)
    oc = ocfg_of(cfg)
    ev = I.Evaluator(cfg)
    robot.set_on(ev)
    ref_shape = DeviceSdf(ev) if robot.winding else robot.osh
    g = G.grazing_map(oc, ref_shape, T, Cc, bmin, res, dims, delta=delta, shape_aabb=robot.aabb, region=region,
                      max_voxels=4000 if region is None else 100000)
    assert g["n_active"] >= min_active, f"{what}: only {g['n_active']} active grazing voxels"
    if straddle:                                                     # active pairs on both branches of the smoothed hinge
        x = cfg.safety_hor - g["pairs"]["sdf"]
        below, above = int(((x > 0) & (x <= cfg.smoothing_eps)).sum()), int((x > cfg.smoothing_eps).sum())
        assert below >= 5 and above >= 5, f"{what}: {below} active pairs with x <= mu, {above} with x > mu"
    assert g["sensitivity"] >= 100 * TOL, f"{what}: fixture sensitivity {g['sensitivity']:.2e} cannot resolve one lost voxel at {TOL:.0e}"
    ev.set_map_u8(g["occ"], bmin, res)
    got = ev.eval_discrete(T, Cc)
    pcs = ev.piece_costs(N)
    pairs = ev.stats().last_pairs
    grid, gcounts, scounts = None, None, None
    if robot.kind == "mesh":
        grid = ev.dbg_mesh_grid()
        act = g["pairs"]["sdf"] < cfg.safety_hor
        gcounts = G.branch_counts(grid, g["pairs"]["prel"][act])
    if robot.winding:
        # reference: the unculled device SDF of every box pair through the oracle-form hinge (cost), the oracle at the winding bar
        assert abs(got[0] - g["cost"]) <= TOL * g["cost"], f"{what}: cost {got[0]!r} vs every box pair answered {g['cost']!r}"
        exp = O.eval_discrete(oc, g["occ"], bmin, res, robot.osh, T, Cc, use_omp=True)
        assert pairs == exp[3]                                       # (the oracle's exact winding number moves grazing x itself)
        relc, relg = abs(got[0] - g["cost"]) / g["cost"], float("nan")
        _, _, w, piece = G.sample_poses(oc, T, Cc)
        on = g["pairs"]["sdf"] < cfg.safety_hor
        pexp = np.bincount(piece[g["pairs"]["sample"][on]], weights=w[g["pairs"]["sample"][on]] *
                           G.hinge(cfg.safety_hor - g["pairs"]["sdf"][on], cfg.smoothing_eps), minlength=N)
        assert np.all(np.abs(pcs - pexp) <= TOL * g["cost"]), f"{what}: piece costs {pcs} vs {pexp}"
    else:
        exp = O.eval_discrete(oc, g["occ"], bmin, res, robot.osh, T, Cc, use_omp=True)
        assert abs(exp[0] - g["cost"]) <= TOL * exp[0], f"{what}: fixture's own cost {g['cost']!r} disagrees with the oracle {exp[0]!r}"
        relc, relg = check(got, exp, TOL, what + " grazing")
        assert pairs == exp[3], f"{what}: {pairs} box pairs vs the oracle's {exp[3]}"
        for i in range(N):
            Ti, Ci = piece_slice(T, Cc, i)
            e = O.eval_discrete(oc, g["occ"], bmin, res, robot.osh, Ti, Ci)
            assert abs(pcs[i] - e[0]) <= TOL * max(exp[0], 1e-300), f"{what}: piece {i} cost {pcs[i]!r} vs {e[0]!r}"
    if scene is not None:
        occ_r, bmin_r, res_r = scene
        ev.set_map_u8(occ_r, bmin_r, res_r)
        gr = ev.eval_discrete(T, Cc)
        er = O.eval_discrete(oc, occ_r, bmin_r, res_r, robot.osh, T, Cc, use_omp=True)
        assert ev.stats().last_pairs == er[3]
        if robot.winding:
            assert er[0] > 0 and abs(gr[0] - er[0]) / er[0] < 5e-3
        else:
            assert er[0] > 0
            check(gr, er, TOL_RANDOM, what + " random map")
        if grid is not None:
            scounts = G.branch_counts(grid, random_scene_pairs(cfg, occ_r, bmin_r, res_r, T, Cc))
    geo = "" if grid is None else (f" gcell {grid['gcell']:.4f} ghd {grid['ghd']:.4f} gpad {grid['gpad']:.3f} sign_radius {grid['sign_radius']:.3f} "
                                   f"list_reach {grid['list_reach']:.3f} gdim {grid['gdim']}")
    print(f"\n[{what}] active {g['n_active']} inactive {g['n_inactive']} sensitivity {g['sensitivity']:.2e} cost rel {relc:.1e} grad rel {relg:.1e}"
          f"{geo}\n    grazing active pairs by branch {gcounts}\n    random-scene pairs by branch {scounts}  ({time.time() - t0:.1f} s)")
    if target is not None:
        src, branch, n = target
        counts = gcounts if src == "grazing" else scounts
        assert counts[branch] >= n, f"{what}: {counts[branch]} {src} pairs in {branch} cells, expected >= {n}"
    ev.close()
    return grid, gcounts, scounts, g


def traj(box, seed=3):
    T, Cc, _ = W.make_trajectory(2, [0, 0, 0], [box] * 3, seed=seed, jitter=0.2)
    return T, Cc


def rand_scene(X, res=1.0, p=0.05, seed=1, bmin=(0.0, 0.0, 0.0)):
    return W.random_map(X, X, X, p=p, seed=seed, slabs=0), list(bmin), res


@pytest.fixture(scope="module")
def cone():
    return W.rounded_cone_mesh()


# ---- margin and scale: exact-sign mesh ------------------------------------------------------------------------------
def test_default_margin_listed_cells(cone):
    T, Cc = traj(24)
    grid, gc, _, _ = run_discrete("default", make_cfg(), Robot("mesh", *cone), T, Cc, [0, 0, 0], 0.1, (240,) * 3,
                               scene=rand_scene(24), target=("grazing", "listed", 100))
    assert grid["gcell"] == 0.1 and grid["sign_radius"] > 0


def test_tight_margin_unbounded_searches(cone):
    T, Cc = traj(24)
    grid, gc, sc, _ = run_discrete("tight 0.15", make_cfg(safety=0.15), Robot("mesh", *cone), T, Cc, [0, 0, 0], 0.1, (240,) * 3,
                               scene=rand_scene(24), target=("grazing", "listed", 20))
    assert grid["sign_radius"] == 0.0                                # 2 hd >= 0.9 safety_hor: no sign shortcut, every search unbounded
    assert sc["deep"] >= 5 and gc["overflow"] >= 1                   # unlisted cells: the unbounded tree search answers them


def test_wide_margin_overflow_cells(cone):
    T, Cc = traj(32)
    grid, gc, _, _ = run_discrete("wide 2.5", make_cfg(safety=2.5), Robot("mesh", *cone), T, Cc, [0, 0, 0], 0.1, (320,) * 3,
                               scene=rand_scene(32), target=("grazing", "overflow", 50))
    assert grid["gcell"] > 0.1


def test_large_robot_deep_and_coarse_cells(cone):
    T, Cc = traj(64, seed=4)
    grid, gc, sc, _ = run_discrete("robot x4", make_cfg(ks=45), Robot("mesh", *cone, scale=4.0), T, Cc, [0, 0, 0], 0.25, (256,) * 3,
                                scene=rand_scene(64, p=0.05), target=("random", "deep", 50))
    assert grid["gcell"] > 0.1 and gc["listed"] > 0


def test_concave_corner_needs_the_full_list_radius():
    """Outside a convex body the closest-point map is 1-Lipschitz, so a candidate list of radius |d_c| + hd would already hold the
    closest triangle of every point in the cell; only near a concave edge can the closest triangle of a point lie up to |d_c| + 2 hd
    from the cell centre. The L-shaped prism's inner edge, nearly stationary (every sample sees the same corner), with all grazing
    voxels on the bisector of the two inner faces: some active pairs must be answered by a triangle only the full radius lists."""
    V, F = W.l_prism_mesh()                                          # inner edge at (0.8, 0.8) - (1, 2/3), faces x = and y = const
    robot = Robot("mesh", V, F)
    R, t = W.rotation_from_poly_params(PP)
    corner = np.array([0.8 - 1.0, 0.8 - 2.0 / 3.0, 0.0])

    def region(p):
        q = (p - t) @ R
        a, b = q[:, 0] - corner[0], q[:, 1] - corner[1]
        return (a > 0) & (b > 0) & (np.abs(a - b) <= 0.2)
    cb = np.array([[corner[0] + x, corner[1] + y, z] for x in (-0.3, 1.8) for y in (-0.3, 1.8) for z in (-1.5, 1.5)]) @ R.T + t
    region.box = (cb.min(0), cb.max(0))
    step = 0.05
    wp = np.array([[12, 12, 12], [12 + step, 12 + 0.3 * step, 12 - 0.2 * step], [12 + 2 * step, 12, 12 + 0.1 * step]], float)
    T = np.array([2.5, 2.5])
    Cc = W.minco_s3(wp, T)
    grid, gc, _, g = run_discrete("concave corner", make_cfg(K=32), robot, T, Cc, [8.0, 8.0, 8.0], 0.04, (200,) * 3, delta=0.1,
                                  region=region, target=("grazing", "listed", 1000))
    on = g["pairs"]["sdf"] < 0.866
    crit = G.list_critical(grid, g["pairs"]["prel"][on], (V @ R.T + t)[F])
    print(f"    active pairs whose closest triangle lies beyond |d_c| + ghd of the cell centre: {int(crit.sum())}")
    assert crit.sum() >= 8


# ---- winding sign: no distance cull, every box voxel answered ---------------------------------------------------
def open_box():
    V, F = W.box_mesh(1.2, 0.7, 0.4)
    return V, F[2:]                                                  # one face (two triangles) removed


@pytest.mark.parametrize("safety", [0.15, 2.5])
@pytest.mark.parametrize("mesh", ["open_box", "closed_ico"])
def test_winding_sign_outside_grid(mesh, safety):
    V, F = open_box() if mesh == "open_box" else W.icosphere(1.3, 2)
    T, Cc = traj(24)
    # at the tight margin most box voxels lie outside the cell grid (gpad = 0.4) and are searched with seed -1; at the wide one the
    # 9-voxel window stays inside the grid (gpad = 5.1)
    target = ("random", "outside", 500) if safety < 1 else ("grazing", "listed", 100)
    run_discrete(f"winding {mesh} {safety}", make_cfg(safety=safety, ks=9), Robot("mesh", V, F, sign_mode=I.MESH_SIGN_WINDING),
                 T, Cc, [0, 0, 0], 0.1, (240,) * 3, scene=rand_scene(24), target=target)


# ---- smoothing: the band straddles x = mu (cubic and linear branch of the hinge) -----------------------------------------
@pytest.mark.parametrize("eps", [1e-3, 0.5])
@pytest.mark.parametrize("shape", ["mesh", "Ball", "TwistBox"])
def test_smoothing_both_hinge_branches(shape, eps, cone):
    robot = Robot("mesh", *cone) if shape == "mesh" else Robot("named", shape)
    T, Cc = traj(24)
    res = 0.1 if shape == "mesh" else 0.2
    run_discrete(f"smoothing {eps} {shape}", make_cfg(eps=eps), robot, T, Cc, [0, 0, 0], res, (int(round(24 / res)),) * 3,
                 delta=2 * eps, scene=rand_scene(24), straddle=True)


# ---- map resolution != occupancy_resolution, fractional origin ----------------------------------------------------------
@pytest.mark.parametrize("res", [0.25, 0.4])
@pytest.mark.parametrize("shape", ["mesh", "Ball"])
def test_map_resolution_differs_from_occupancy_resolution(shape, res, cone):
    robot = Robot("mesh", *cone) if shape == "mesh" else Robot("named", shape)
    T, Cc = traj(24)
    bmin = [-0.37, 0.13, -0.71]
    n = int(24 / res)
    h = 6.5
    pos, _, _, _ = G.sample_poses(O.config_from(make_cfg()), T, Cc)
    win = np.floor((pos + h - bmin) / res).astype(int) - np.floor((pos - h - bmin) / res).astype(int) + 1
    # realised windows (inclusive index ranges, every sample and axis): 53 voxels at 0.25 (13 m is exactly 52 voxels), 33 or 34 at 0.4
    assert win.max() == (53 if res == 0.25 else 34) and win.min() == (53 if res == 0.25 else 33), (win.min(), win.max())
    # only voxels on the envelope of the swept robot can graze, so coarse voxels need a wider band (still x <= mu)
    run_discrete(f"map res {res} {shape}", make_cfg(), robot, T, Cc, bmin, res, (n,) * 3, delta=4e-3 if res == 0.25 else 1e-2, min_active=5,
                 scene=(W.random_map(n, n, n, p=0.01, seed=2, slabs=0), bmin, res))


# ---- the pose window at the 10-bit field limit ------------------------------------------------------------------------
I_WINDOW_AXIS_MAX = 1023


def finest_res(cfg):
    """the finest map resolution the library accepts: 2 half_bd / res + 2 <= 1023"""
    return (cfg.kernel_size * cfg.occupancy_resolution) / (I_WINDOW_AXIS_MAX - 2) * (1 + 1e-12)


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("shape", ["Ball", "mesh"])
def test_window_at_the_field_limit(shape, axis, cone):
    cfg = make_cfg()
    res = finest_res(cfg)
    robot = Robot("mesh", *cone) if shape == "mesh" else Robot("named", shape)
    T, Cc = traj(24)
    oc = O.config_from(cfg)
    pos, R, _, _ = G.sample_poses(oc, T, Cc)
    mid = pos[len(pos) // 2]
    dims = [3, 3, 3]
    dims[axis] = 1100
    # a thin rod of voxels centred on the middle sample's position along `axis`, offset sideways to where the robot grazes it
    off = np.full(3, 1.2 if shape == "Ball" else 1.0)
    off[axis] = 0.0
    bmin = mid + off - 0.5 * res * np.array(dims)
    g_lo = np.floor((pos[:, axis] - 6.5 - bmin[axis]) / res).astype(int).clip(0, dims[axis] - 1)
    g_hi = np.floor((pos[:, axis] + 6.5 - bmin[axis]) / res).astype(int).clip(0, dims[axis] - 1)
    assert (g_hi - g_lo + 1).max() >= 1022                           # a realised window at the 10-bit limit of the offset codes
    run_discrete(f"field limit axis {axis} {shape}", cfg, robot, T, Cc, list(bmin), res, tuple(dims), delta=1e-2, min_active=5,
                 scene=((np.random.default_rng(axis).random(dims) < 0.3).astype(np.uint8), list(bmin), res))


def test_resolution_finer_than_the_field_limit_is_refused():
    cfg = make_cfg()
    ev = I.Evaluator(cfg)
    occ = np.zeros((1100, 3, 3), np.uint8)
    ev.set_map_u8(occ, [0, 0, 0], finest_res(cfg))
    with pytest.raises(I.IsdfError) as e:
        ev.set_map_u8(occ, [0, 0, 0], finest_res(cfg) * 0.99)
    assert e.value.code == -4                                        # ISDF_ERR_UNSUPPORTED
    ev.close()


# ---- swept volume: range bound and hinge (closed meshes; winding sign is refused there by design) -------------------------
@pytest.mark.parametrize("what,safety,scale", [("default", 0.866, 1.0), ("tight", 0.03, 1.0), ("wide", 2.5, 1.0), ("robot x4", 0.866, 4.0)])
def test_swept_range_and_hinge_boundaries(what, safety, scale, cone):
    t0 = time.time()
    cfg = make_cfg(safety=safety)
    oc = ocfg_of(cfg)
    robot = Robot("mesh", *cone, scale=scale)
    T, Cc = traj(24)
    pts, sets = G.swept_band_points(oc, robot.osh, T, Cc, robot.aabb, n=2000)
    assert len(sets["range"]) >= 20 and len(sets["active"]) >= 50 and len(sets["inactive"]) >= 50, {k: len(v) for k, v in sets.items()}
    ref = O.eval_swept(oc, robot.osh, T, Cc, pts, use_omp=True)
    # smallest single-point share of the cost, from the hinge values (every point carries the same weight). The swept-volume hinge
    # uses mu = 0.01 literally, not smoothing_eps, as the reference does (oracle_planner.hpp, the SV tail)
    h = G.hinge(safety - ref["sdf"][ref["sdf"] < 9.0], 0.01)
    sens = h[h > 0].min() / h.sum()
    assert sens >= 100 * TOL
    ev = I.Evaluator(cfg)
    robot.set_on(ev)
    ev.set_points(pts)
    got = ev.eval_swept(T, Cc)
    ts, sd, _ = ev.swept_results()
    hit = ref["sdf"] < 9.0
    assert (~hit[sets["above"]]).sum() >= 10                         # just above inf: rejected by the range test
    assert np.array_equal(sd < 9.0, hit)
    assert np.abs(ts[hit] - ref["tstar"][hit]).max() <= 8e-5 and np.abs(sd[hit] - ref["sdf"][hit]).max() <= 1e-9
    assert ev.stats().last_sdf_evals == ref["nsdf"]
    relc, relg = check(got, (ref["cost"], ref["gradC"], ref["gradT"]), TOL, f"swept {what}")
    grid = ev.dbg_mesh_grid(arrays=False)
    if safety < 0.1:
        assert grid["sign_radius"] == 0.0                            # no sign shortcut: the cell brackets alone prune
    print(f"\n[swept {what}] points {len(pts)} hits {hit.sum()} bands {({k: len(v) for k, v in sets.items()})} sensitivity {sens:.2e} "
          f"cost rel {relc:.1e} grad rel {relg:.1e} inf {2 * safety + 0.1:.2f} gcell {grid['gcell']:.4f} ({time.time() - t0:.1f} s)")
    ev.close()
