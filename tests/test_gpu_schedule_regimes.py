"""The discrete evaluation's work-item schedule in every regime its size and K select, and the device entry points in them.

launch_discrete (csrc/isdf_api.cu) changes shape with the number of local samples M and with K = integral_intervs:
  * k_build_items<true> keeps the work values in registers (M <= 24 576), k_build_items<false> re-reads work[rank + world m]
    (24 576 < M <= 98 304), and above 98 304 samples no table is built: the scan runs in natural order;
  * the split threshold THR is raised to a bucket bound when more samples qualify than there are split slots (first_over), and
    saturates (nothing split) when the open-ended top bucket (w >= 8184) alone holds more than MAX_SPLIT_SLOTS samples;
  * k_discrete_epilogue adds a piece's samples in chunks of EPI_THREADS = 288 and carries the running sum across chunks.
Each case first asserts, through isdf_dbg_item_table, that it reached the regime it targets. Then:
  * builder: the table equals the numpy restatement (tests/item_schedule.py) on the work values the builder read;
  * invariance: evaluation 1 (natural order), 3 (work items) and 3 with forced splits give bit-identical cost, gradients, piece
    costs and pair counts; where named, also without window lists, and through isdf_eval_discrete_device on a side stream;
  * oracle: cost and gradient agree with the oracle at 1e-6 (a zero cost exactly), on a sample of pieces run one at a time (the
    discrete term couples no pieces) or on the whole trajectory where that is cheap."""
import os
import numpy as np
import pytest
import torch
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import item_schedule as S
from common import rel_l2, BMIN

pytestmark = pytest.mark.gpu
TOL = 1e-6
NTHREADS = max(1, min(len(os.sched_getaffinity(0)), 16))
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]   # the bench robot's poly_params
FORCE = 50_000_000                      # pretended warp slots: the balanced share drops to SPLIT_WORK_MIN, every heavy sample splits
CACHED_MAX = 24 * 1024                  # ITEMS_CACHE x 1024: the largest M of k_build_items<true>
ITEMS_MAX = 4 * CACHED_MAX              # the largest M that gets a work-item table
WL_DEFAULT = 16                         # default window-list budget, codes per sample


# ---- scenes ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench_map():
    return W.random_map(512, 512, 512, p=0.05, seed=1, slabs=3)


@pytest.fixture(scope="module")
def cone():
    return W.rounded_cone_mesh()


def traj(N, X, seed=11):
    T, Cc, _ = W.make_trajectory(N, [0, 0, 0], [X, X, X], seed=seed, jitter=0.2)
    return T, Cc


def make_cfg(K, safety=None, ks=None):
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = K
    if safety is not None:
        cfg.safety_hor = safety
    if ks is not None:
        cfg.kernel_size = ks
    return cfg


class Robot:
    """the library's and the oracle's view of one robot"""

    def __init__(self, name, cone=None, scale=1.0):
        self.name = name
        if name == "mesh":
            self.V, self.F = cone[0] * scale, cone[1]
            self.osh = O.Shape.mesh(self.V, self.F, PP, wn_mode=O.WN_BH)
        else:
            self.osh = O.Shape.named(name)

    def evaluator(self, cfg, occ):
        ev = I.Evaluator(cfg)
        ev.set_map_u8(occ, BMIN, 1.0)
        if self.name == "mesh":
            ev.set_shape_mesh(self.V, self.F, PP)
        else:
            ev.set_shape_named(self.name)
        return ev


# ---- evaluations -------------------------------------------------------------------------------------------------------------
def result(ev, T, Cc):
    c, gC, gT = ev.eval_discrete(T, Cc)
    return dict(cost=c, grad=np.concatenate([gC, gT]), pieces=ev.piece_costs(len(T)), pairs=ev.stats().last_pairs)


def assert_same(a, b, what):
    assert a["cost"] == b["cost"] and np.array_equal(a["grad"], b["grad"]), f"{what}: cost or gradient differs"
    assert np.array_equal(a["pieces"], b["pieces"]), f"{what}: piece costs differ"
    assert a["pairs"] == b["pairs"], f"{what}: pair count {a['pairs']} vs {b['pairs']}"


def natural(ev, T, Cc):
    """evaluation 1: natural sample order, nothing split, no table built"""
    ev.dbg_schedule(natural_order=True)
    r = result(ev, T, Cc)
    tab = ev.dbg_item_table()
    assert tab["builder"] == "none" and not tab["have_items"]
    return r


def steady(ev, T, Cc, warp_slots=0):
    """evaluation 3 of a schedule learned afresh; returns it and the table it read (built from evaluation 2's work values)"""
    ev.dbg_schedule(warp_slots=warp_slots)
    ev.eval_discrete(T, Cc)
    ev.eval_discrete(T, Cc)
    tab = ev.dbg_item_table()
    r = result(ev, T, Cc)
    after = ev.dbg_item_table()
    assert after["have_items"] == (tab["builder"] != "none"), "the scan did not read the table built for it"
    assert after["builder"] == tab["builder"]
    return r, tab


def check_builder(tab, M, max_split, warp_slots):
    """the table against the restatement; returns the restatement"""
    assert tab["M"] == M and tab["max_split"] == max_split and tab["warp_slots"] == warp_slots, \
        f"builder arguments {dict((k, tab[k]) for k in ('M', 'max_split', 'warp_slots'))}"
    sched = S.schedule(tab["work"], tab["max_split"], tab["warp_slots"])
    S.check_table(sched, tab["items"], tab["max_split"])
    return sched


def regime(tab, sched):
    w = tab["work"]
    return (f"M {tab['M']} builder {tab['builder']} items {tab['item_count']} w>=256: {int((w >= 256).sum())} w>=8184: "
            f"{int((w >= 8184).sum())} THR {sched['thr']} raised at bucket {sched['raised_bucket']} split samples {int(sched['split'].sum())} "
            f"split parts {int(sched['f'][sched['split']].sum())}")


def ocfg_of(cfg):
    oc = O.config_from(cfg)
    oc.threads_num = NTHREADS
    return oc


def check_eval(got, exp, what):
    c, g = got
    if abs(exp[0]) > 0:
        assert abs(c - exp[0]) <= TOL * abs(exp[0]), f"{what}: cost {c!r} vs {exp[0]!r}"
    else:
        assert c == 0, f"{what}: cost {c!r}, the oracle's is zero"
    r = rel_l2(g, np.concatenate([exp[1], exp[2]]))
    assert r <= TOL, f"{what}: gradient rel-L2 {r:.3e}"


def piece_slice(T, Cc, i):
    N = len(T)
    return T[i:i + 1], np.ascontiguousarray(np.asarray(Cc).reshape(3, 6 * N)[:, 6 * i:6 * i + 6]).reshape(-1)


def sampled_pieces(r, N, extra=4):
    """the first and the last piece, the costliest one and `extra` spread between (every piece spans 128-sample range boundaries)"""
    spread = [int(round(k * (N - 1) / (extra + 1))) for k in range(1, extra + 1)]
    return sorted({0, N - 1, int(np.argmax(r["pieces"]))} | set(spread))


def check_pieces(r, cfg, occ, robot, T, Cc, pieces, what, rank=0, world=1):
    """piece cost, 6x3 gradC block and gradT of each sampled piece against the oracle run on that piece alone"""
    N, K = len(T), cfg.integral_intervs
    gC, gT = r["grad"][:18 * N].reshape(3, 6 * N), r["grad"][18 * N:]
    oc = ocfg_of(cfg)
    for i in pieces:
        Ti, Ci = piece_slice(T, Cc, i)
        e = O.eval_discrete(oc, occ, BMIN, 1.0, robot.osh, Ti, Ci, use_omp=True, rank=(rank - i * (K + 1)) % world, world=world)
        check_eval((r["pieces"][i], np.concatenate([gC[:, 6 * i:6 * i + 6].reshape(-1), gT[i:i + 1]])), e, f"{what} piece {i}")


def check_device_entry(ev, T, Cc, ref, what):
    """isdf_eval_discrete_device on a side stream overwrites d_out with what the host entry point adds to zeroed buffers"""
    N = len(T)
    dT = torch.tensor(np.asarray(T, float), device="cuda")
    dC = torch.tensor(np.asarray(Cc, float).reshape(-1), device="cuda")
    out = torch.full((19 * N + 1,), float("nan"), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    ev.eval_discrete_device(N, dT.data_ptr(), dC.data_ptr(), out.data_ptr(), side.cuda_stream)
    side.synchronize()
    o = out.cpu().numpy()
    assert o[0] == ref["cost"] and np.array_equal(o[1:], ref["grad"]), f"{what}: device entry point differs from the host entry point"
    assert np.array_equal(ev.piece_costs(N), ref["pieces"]), f"{what}: piece costs after the device entry point differ"


def invariance(ev, T, Cc, M, max_split, what, no_lists=False):
    """evaluation 1, 3 and 3 with forced splits, each table against the restatement; returns (evaluation 1, tables, restatements)"""
    r1 = natural(ev, T, Cc)
    r3, tab = steady(ev, T, Cc)
    sched = check_builder(tab, M, max_split, tab["warp_slots"])
    assert_same(r1, r3, f"{what}: work items vs natural order")
    rf, tabf = steady(ev, T, Cc, warp_slots=FORCE)
    schedf = check_builder(tabf, M, max_split, FORCE)
    assert_same(r1, rf, f"{what}: forced splits vs natural order")
    if no_lists:
        ev.dbg_window_lists(budget=0)
        rn, _ = steady(ev, T, Cc)
        ev.dbg_window_lists(budget=WL_DEFAULT)
        assert_same(r1, rn, f"{what}: work items without window lists")
    print(f"\n[{what}] {regime(tab, sched)}\n    forced splits: {regime(tabf, schedf)}")
    return r1, (tab, tabf), (sched, schedf)


# ---- k_build_items<false> -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("robot_name", ["mesh", "Ball"])
def test_uncached_builder(bench_map, cone, robot_name):
    """K = 256, 120 pieces: M = 30 840 samples, the builder re-reads the work values"""
    robot = Robot(robot_name, cone)
    cfg = make_cfg(256)
    T, Cc = traj(120, 512)
    M = 120 * 257
    max_split = min(M, S.MAX_SPLIT_SLOTS) if robot_name == "mesh" else 0
    ev = robot.evaluator(cfg, bench_map)
    r1, (tab, tabf), (sched, schedf) = invariance(ev, T, Cc, M, max_split, f"uncached {robot_name}", no_lists=robot_name == "mesh")
    assert CACHED_MAX < M <= ITEMS_MAX and tab["builder"] == tabf["builder"] == "uncached"
    if robot_name == "mesh":
        assert schedf["split"].sum() > 100, "forced splits split next to nothing"
    else:
        assert not sched["split"].any() and not schedf["split"].any()
    check_device_entry(ev, T, Cc, r1, f"uncached {robot_name}")
    check_pieces(r1, cfg, bench_map, robot, T, Cc, sampled_pieces(r1, 120), f"uncached {robot_name}")
    ev.close()


@pytest.mark.parametrize("robot_name", ["mesh", "Ball"])
def test_uncached_builder_sharded(bench_map, cone, robot_name):
    """set_shard(r, 2) over 200 pieces: M = 25 700 local samples per rank, read at work[rank + 2 m]"""
    robot = Robot(robot_name, cone)
    cfg = make_cfg(256)
    N = 200
    T, Cc = traj(N, 512, seed=12)
    ev = robot.evaluator(cfg, bench_map)
    full = natural(ev, T, Cc)
    acc_c, acc_g = 0.0, np.zeros_like(full["grad"])
    for rank in range(2):
        ev.set_shard(rank, 2)
        M = (N * 257 - rank + 1) // 2
        max_split = min(M, S.MAX_SPLIT_SLOTS) if robot_name == "mesh" else 0
        what = f"uncached {robot_name} shard {rank}/2"
        r1, (tab, _), _ = invariance(ev, T, Cc, M, max_split, what, no_lists=robot_name == "mesh")
        assert M == 25700 and tab["builder"] == "uncached" and tab["rank"] == rank and tab["world"] == 2
        check_device_entry(ev, T, Cc, r1, what)
        check_pieces(r1, cfg, bench_map, robot, T, Cc, sampled_pieces(r1, N, extra=2), what, rank=rank, world=2)
        acc_c += r1["cost"]
        acc_g += r1["grad"]
    assert abs(acc_c - full["cost"]) <= 1e-12 * abs(full["cost"]) and rel_l2(acc_g, full["grad"]) <= 1e-12
    ev.close()


# ---- the largest table, and the first launch without one -------------------------------------------------------------------------
@pytest.mark.parametrize("N", [384, 385])
def test_items_boundary(bench_map, cone, N):
    """K = 255: 384 pieces give M = 98 304 (the largest table, uncached builder), 385 give 98 560 (natural order only)"""
    robot = Robot("mesh", cone)
    cfg = make_cfg(255)
    T, Cc = traj(N, 512, seed=13)
    M = N * 256
    ev = robot.evaluator(cfg, bench_map)
    if M <= ITEMS_MAX:
        r1, (tab, tabf), _ = invariance(ev, T, Cc, M, S.MAX_SPLIT_SLOTS, f"boundary N={N}", no_lists=True)
        assert M == ITEMS_MAX and tab["builder"] == tabf["builder"] == "uncached"
    else:
        r1 = natural(ev, T, Cc)
        ev.dbg_schedule()
        for k in range(3):
            r = result(ev, T, Cc)
            tab = ev.dbg_item_table()
            assert tab["M"] == M and tab["builder"] == "none" and not tab["have_items"], f"evaluation {k + 2} of M = {M}: {tab['builder']}"
            assert_same(r1, r, f"boundary N={N}: evaluation {k + 2}")
        ev.dbg_window_lists(budget=0)
        assert_same(r1, result(ev, T, Cc), f"boundary N={N}: without window lists")
        ev.dbg_window_lists(budget=WL_DEFAULT)
    check_device_entry(ev, T, Cc, r1, f"boundary N={N}")
    check_pieces(r1, cfg, bench_map, robot, T, Cc, sampled_pieces(r1, N, extra=3), f"boundary N={N}")
    ev.close()


# ---- THR raised by first_over, THR saturated ------------------------------------------------------------------------------------
def test_split_slots_exhausted(cone):
    """a 15 %-occupancy map: under forced splits more than 16 384 samples reach w >= 256, so first_over raises THR to a bucket
    bound and only the samples above it (at most 16 384) are split"""
    robot = Robot("mesh", cone)
    cfg = make_cfg(256)
    occ = W.random_map(256, 256, 256, p=0.15, seed=5, slabs=0)
    N = 80
    T, Cc = traj(N, 256, seed=14)
    M = N * 257
    ev = robot.evaluator(cfg, occ)
    r1, (_, tabf), (_, schedf) = invariance(ev, T, Cc, M, S.MAX_SPLIT_SLOTS, "split slots exhausted")
    w = tabf["work"]
    assert (w >= S.SPLIT_WORK_MIN).sum() > S.MAX_SPLIT_SLOTS, regime(tabf, schedf)
    assert schedf["raised_bucket"] is not None and schedf["thr"] > S.SPLIT_WORK_MIN and schedf["thr"] != S.THR_SATURATED
    nsplit = int(schedf["split"].sum())
    assert 0 < nsplit <= S.MAX_SPLIT_SLOTS and nsplit == int((w >= schedf["thr"]).sum())
    assert len({int(s) for s in tabf["items"][tabf["items"][:, 2] >= 0, 0]}) == nsplit
    check_pieces(r1, cfg, occ, robot, T, Cc, sampled_pieces(r1, N, extra=2), "split slots exhausted")
    ev.close()


def test_top_bucket_saturated(cone):
    """the bench mesh x4 on a dense map with a wide margin: more than 16 384 samples reach the top bucket (w >= 8184, ~128 mesh
    queries each), THR saturates and nothing is split even under forced splits"""
    robot = Robot("mesh", cone, scale=4.0)
    cfg = make_cfg(256, safety=2.0, ks=45)
    occ = W.random_map(128, 128, 128, p=0.15, seed=6, slabs=0)
    N = 96
    T, Cc = traj(N, 128, seed=15)
    M = N * 257
    ev = robot.evaluator(cfg, occ)
    r1, (tab, tabf), (sched, schedf) = invariance(ev, T, Cc, M, S.MAX_SPLIT_SLOTS, "top bucket saturated")
    for t, s in ((tab, sched), (tabf, schedf)):
        assert (t["work"] >= 8184).sum() > S.MAX_SPLIT_SLOTS, regime(t, s)
        assert s["raised_bucket"] == S.ORDER_BUCKETS - 1 and s["thr"] == S.THR_SATURATED
        assert np.all(t["items"][:, 2] == -1) and t["item_count"] == M
    check_pieces(r1, cfg, occ, robot, T, Cc, sorted({0, int(np.argmax(r1["pieces"])), N - 1}), "top bucket saturated")
    ev.close()


# ---- k_discrete_epilogue over several chunks ----------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [287, 288, 575, 1000])
@pytest.mark.parametrize("robot_name", ["Ball", "mesh"])
def test_multi_chunk_epilogue(cone, robot_name, K):
    """4 pieces of K + 1 samples: one epilogue chunk of 288 at K = 287, two at 288, ... four at 1000; with three shards 96 .. 334
    local samples per piece"""
    robot = Robot(robot_name, cone)
    cfg = make_cfg(K)
    occ = W.three_slit_map(64, 64, 64, noise=0.05, seed=3)
    T, Cc, _ = W.make_trajectory(4, [0, 0, 0], [50, 50, 34], seed=3, jitter=0.3)
    ev = robot.evaluator(cfg, occ)
    oc = ocfg_of(cfg)
    acc_c, acc_g = 0.0, None
    full = None
    for world in (1, 3):
        for rank in range(world):
            ev.set_shard(rank, world)
            M = (4 * (K + 1) - rank + world - 1) // world
            max_split = min(M, S.MAX_SPLIT_SLOTS) if robot_name == "mesh" else 0
            what = f"{robot_name} K={K} shard {rank}/{world}"
            r1, (tab, _), _ = invariance(ev, T, Cc, M, max_split, what)
            assert tab["builder"] == "cached"
            check_device_entry(ev, T, Cc, r1, what)
            e = O.eval_discrete(oc, occ, BMIN, 1.0, robot.osh, T, Cc, use_omp=True, rank=rank, world=world)
            assert r1["pairs"] == e[3], f"{what}: pair count {r1['pairs']} vs the oracle's {e[3]}"
            check_eval((r1["cost"], r1["grad"]), e, what)
            N = 4
            for i in range(N):
                Ti, Ci = piece_slice(T, Cc, i)
                ep = O.eval_discrete(oc, occ, BMIN, 1.0, robot.osh, Ti, Ci, use_omp=True, rank=(rank - i * (K + 1)) % world, world=world)
                assert abs(r1["pieces"][i] - ep[0]) <= TOL * max(abs(e[0]), 1e-300), f"{what}: piece {i} cost {r1['pieces'][i]!r} vs {ep[0]!r}"
            if world == 1:
                full = r1
                assert full["cost"] > 0
            else:
                acc_c += r1["cost"]
                acc_g = r1["grad"] if acc_g is None else acc_g + r1["grad"]
    assert abs(acc_c - full["cost"]) <= 1e-12 * abs(full["cost"]) and rel_l2(acc_g, full["grad"]) <= 1e-12
    ev.close()


# ---- the batched callback in the uncached range and above it ------------------------------------------------------------------
def batch_problems(B, N0, X=512):
    rng = np.random.default_rng(B)
    xs, heads, tails = np.zeros((B, 4 * N0 - 3)), np.zeros((B, 3, 3)), np.zeros((B, 3, 3))
    for b in range(B):
        wp = W.random_walk_waypoints(N0, [0, 0, 0], [X, X, X], seed=1000 + b)
        xs[b, :N0] = 1.0 + 0.2 * rng.normal(size=N0)
        xs[b, N0:] = wp[1:-1].reshape(-1)
        heads[b, :, 0], tails[b, :, 0] = wp[0], wp[-1]
        heads[b, :, 1] = 0.3 * rng.normal(size=3)
    return xs, heads, tails


def device_callback(ev, B, N0, heads, tails, per, rho, xs):
    dh = torch.tensor(I._colmajor(heads), device="cuda")
    dt = torch.tensor(I._colmajor(tails), device="cuda")
    dx = torch.tensor(np.ascontiguousarray(xs).reshape(-1), device="cuda")
    dc = torch.full((B,), float("nan"), dtype=torch.float64, device="cuda")
    dg = torch.full((B * xs.shape[1],), float("nan"), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    ev.callback_batch_device(B, N0, dh.data_ptr(), dt.data_ptr(), per, rho, dx.data_ptr(), dc.data_ptr(), dg.data_ptr(), side.cuda_stream)
    side.synchronize()
    return dc.cpu().numpy(), dg.cpu().numpy().reshape(B, -1)


@pytest.mark.parametrize("B", [5, 6])
def test_batched_callback(bench_map, cone, B):
    """B = 5 restarts of 64 pieces at K = 256 (82 240 samples: uncached builder), B = 6 (98 688: no table)"""
    robot = Robot("mesh", cone)
    cfg = make_cfg(256)
    N0, rho = 64, 20.0
    M = B * N0 * 257
    xs, heads, tails = batch_problems(B, N0)
    ev = robot.evaluator(cfg, bench_map)
    c1, g1 = ev.callback_batch(heads, tails, rho, xs)                # natural order (a fresh context)
    first = ev.dbg_item_table()
    c2, g2 = ev.callback_batch(heads, tails, rho, xs)
    tab = ev.dbg_item_table()
    c3, g3 = ev.callback_batch(heads, tails, rho, xs)
    after = ev.dbg_item_table()
    assert not first["have_items"] and tab["M"] == M
    if M <= ITEMS_MAX:
        assert tab["builder"] == "uncached" and after["have_items"]
        sched = check_builder(tab, M, S.MAX_SPLIT_SLOTS, tab["warp_slots"])
        print(f"\n[batched B={B}] {regime(tab, sched)}")
    else:
        assert tab["builder"] == "none" and not after["have_items"]
    for c, g, k in ((c2, g2, 2), (c3, g3, 3)):
        assert np.array_equal(c, c1) and np.array_equal(g, g1), f"batched B={B}: call {k} differs from call 1"
    dc, dg = device_callback(ev, B, N0, heads, tails, 1, rho, xs)
    assert np.array_equal(dc, c1) and np.array_equal(dg, g1), f"batched B={B}: device callback (per-problem bc) differs from the host callback"
    # one head / tail pair shared by the batch: problem 0's own pair -> problem 0 unchanged
    s_c, s_g = ev.callback_batch(heads[0], tails[0], rho, xs)
    dc0, dg0 = device_callback(ev, B, N0, heads[0], tails[0], 0, rho, xs)
    assert np.array_equal(dc0, s_c) and np.array_equal(dg0, s_g), f"batched B={B}: device callback (shared bc) differs from the host callback"
    assert s_c[0] == c1[0] and np.array_equal(s_g[0], g1[0]), f"batched B={B}: problem 0 under its own bc shared by the batch differs"
    assert np.all(s_c[1:] != c1[1:])
    ev.close()
    oc = ocfg_of(cfg)
    for b in (0, B - 1):
        tau = xs[b, :N0]
        Tt = np.where(tau > 0, (0.5 * tau + 1) * tau + 1, 1 / ((0.5 * tau - 1) * tau + 1))
        inP = xs[b, N0:].reshape(-1, 3).T
        co, energy, gC, gT = O.minco_forward(heads[b], tails[b], inP, Tt)
        di = O.eval_discrete(oc, bench_map, BMIN, 1.0, robot.osh, Tt, co, use_omp=True)
        c_ref = energy + di[0] + rho * Tt.sum()
        gp, gt = O.minco_backward(heads[b], tails[b], inP, Tt, gC + di[1], gT + di[2])
        gt = gt + rho
        gtau = np.where(tau > 0, gt * (tau + 1), gt * (1 - tau) / ((0.5 * tau - 1) * tau + 1) ** 2)
        g_ref = np.concatenate([gtau, gp.T.reshape(-1)])
        relc, relg = abs(c1[b] - c_ref) / abs(c_ref), rel_l2(g1[b], g_ref)
        assert relc <= TOL and relg <= TOL, f"batched B={B} problem {b}: cost rel {relc:.3e}, grad rel-L2 {relg:.3e}"
