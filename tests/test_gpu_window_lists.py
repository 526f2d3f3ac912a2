"""Window lists of the discrete mesh scan (k_discrete_prologue -> k_discrete_mesh).

The prologue computes every local sample's pose and lists the occupied voxels of each run's window (consecutive samples of one
128-sample range with the same window) once; the scan kernel reads the list, or enumerates the window itself when its run did not
fit into the list buffer. Checked here, for the pseudonormal-sign and the winding-sign kernel:
  * the lists read back through isdf_dbg_window_lists equal a numpy enumeration of each sample's window, in canonical order
    (z-chunk of 32, row r = rx * ny + ry, z) and with the run boundaries the prologue must draw: on the bench map, on a map finer
    than the window (z spans several chunks), with windows clamped at the map faces, and with runs crossing 128-sample ranges;
  * results and the pair count are bit-identical with no lists (budget 0), with some runs overflowing and with the default
    budget, for whole samples and for forced split parts, and for sharded launches;
  * the bench workload fits the default budget without overflow."""
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W
from common import BMIN

pytestmark = pytest.mark.gpu
PRO_SAMPLES = 128   # local samples per prologue CTA: every range starts a run
I_DEFAULT = 16      # default list budget, codes per sample of the trajectory
SIGNS = {"pseudonormal": I.MESH_SIGN_AUTO, "winding": I.MESH_SIGN_WINDING}


def windows_of(pos, info, h):
    """window_of (isdf_discrete.cuh) in numpy: n x 6 {ix0, ix1, iy0, iy1, iz0, iz1}"""
    out = np.zeros((len(pos), 6), dtype=np.int64)
    for a in range(3):
        lo, hi, n = info["bmin"][a], info["bmax"][a], info["dims"][a]
        for k, sgn in enumerate((-1.0, 1.0)):
            c = np.clip(pos[:, a] + sgn * h, lo, hi)
            out[:, 2 * a + k] = np.clip(np.floor((c - lo) / info["res"]).astype(np.int64), 0, n - 1)
    return out


def window_codes(occ, w):
    """the window's occupied voxels as codes dx | dy << 10 | dz << 20, in canonical order"""
    sub = occ[w[0]:w[1] + 1, w[2]:w[3] + 1, w[4]:w[5] + 1]
    nx, ny, nz = sub.shape
    parts = []
    for zs in range(0, nz, 32):
        r, z = np.nonzero(sub[:, :, zs:zs + 32].reshape(nx * ny, -1))   # row-major: row ascending, then z
        parts.append((r // ny) | ((r % ny) << 10) | ((z + zs) << 20))
    return np.concatenate(parts).astype(np.uint32)


def check_lists(ev, occ, cfg, T, Cc, rank=0, world=1):
    """the last evaluation's lists against numpy; returns (stats, windows)"""
    L = ev.dbg_window_lists(arrays=True)
    info = ev.map_info()
    K, N = cfg.integral_intervs, len(T)
    M = (N * (K + 1) - rank + world - 1) // world
    assert L["samples"] == M
    s = rank + world * np.arange(M)
    i, j = s // (K + 1), s % (K + 1)
    t = np.concatenate([[0.0], np.cumsum(T)])[i] + j * (T[i] / K)
    pos = L["pose"][:, :3]
    assert np.abs(pos - W.traj_eval(T, Cc, t)).max() <= 1e-9 * max(1.0, np.abs(pos).max())
    win = windows_of(pos, info, cfg.kernel_size * cfg.occupancy_resolution / 2)
    start = np.ones(M, dtype=bool)
    start[1:] = np.any(win[1:] != win[:-1], axis=1)
    start[::PRO_SAMPLES] = True
    starts = np.flatnonzero(start)
    assert L["runs"] == len(starts)
    desc, codes = L["desc"], L["codes"]
    overflow, written, offsets = 0, 0, set()
    for a, b in zip(starts, np.append(starts[1:], M)):
        exp = window_codes(occ, win[a])
        assert np.all(desc[a:b] == desc[a]), f"run {a}..{b}: samples of one run point at different lists"
        off, cnt = int(desc[a, 0]), int(desc[a, 1])
        assert cnt == len(exp), f"run at sample {a}: {cnt} voxels listed, {len(exp)} in the window"
        if off < 0:
            overflow += 1
            continue
        assert off not in offsets or cnt == 0
        offsets.add(off)
        assert np.array_equal(codes[off:off + cnt], exp), f"run at sample {a}: list differs from the window's canonical enumeration"
        written += cnt
    assert L["overflow"] == overflow and L["written"] == written
    return L, win


def evaluate(ev, T, Cc, budget, warp_slots=0):
    """first (natural order) and third (work items; split parts when warp_slots is huge) evaluation under a list budget"""
    ev.dbg_window_lists(budget=budget)
    ev.dbg_schedule(warp_slots=warp_slots)
    a = ev.eval_discrete(T, Cc)
    pa = ev.stats().last_pairs
    ev.eval_discrete(T, Cc)
    b = ev.eval_discrete(T, Cc)
    pb = ev.stats().last_pairs
    return [(a[0], np.concatenate([a[1], a[2]]), pa), (b[0], np.concatenate([b[1], b[2]]), pb)], ev.dbg_window_lists()


def assert_same(x, y, what):
    for (c0, g0, p0), (c1, g1, p1) in zip(x, y):
        assert c0 == c1 and np.array_equal(g0, g1), f"{what}: result differs"
        assert p0 == p1, f"{what}: pair count differs"


def make_ev(cfg, occ, V, F, pp, sign, res=1.0):
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, res)
    ev.set_shape_mesh(V, F, pp, sign_mode=SIGNS[sign])
    return ev


@pytest.fixture(scope="module")
def bench():
    X = 512
    occ = W.random_map(X, X, X, p=0.05, seed=1, slabs=3)
    T, Cc, _ = W.make_trajectory(64, [0, 0, 0], [X, X, X], seed=11, jitter=0.2)
    V, F = W.rounded_cone_mesh()
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = 256
    return cfg, occ, T, Cc, V, F, [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]


@pytest.mark.parametrize("sign", list(SIGNS))
def test_bench_map_lists_and_budgets(bench, sign):
    cfg, occ, T, Cc, V, F, pp = bench
    n = 64 if sign == "pseudonormal" else 8       # the winding-sign kernel answers every voxel in the box: a shorter trajectory
    T, Cc = T[:n].copy(), np.asarray(Cc).reshape(3, 64 * 6)[:, :6 * n].reshape(-1).copy()
    ev = make_ev(cfg, occ, V, F, pp, sign)
    ref, st = evaluate(ev, T, Cc, I_DEFAULT)
    assert st["overflow"] == 0, f"bench workload overflowed {st['overflow']} of {st['runs']} runs at the default budget"
    L, win = check_lists(ev, occ, cfg, T, Cc)
    assert np.any(np.all(win[PRO_SAMPLES::PRO_SAMPLES] == win[PRO_SAMPLES - 1:-1:PRO_SAMPLES], axis=1)), "no run crosses a 128-sample range"
    got, st0 = evaluate(ev, T, Cc, 0)
    assert st0["written"] == 0 and st0["overflow"] == st0["runs"]
    assert_same(ref, got, f"{sign}: no lists vs default budget")
    got, st1 = evaluate(ev, T, Cc, 1)
    assert 0 < st1["overflow"] < st1["runs"], st1
    check_lists(ev, occ, cfg, T, Cc)
    assert_same(ref, got, f"{sign}: overflowing budget vs default budget")
    # forced split parts: every part filters its classes from the list (or from its own enumeration)
    for budget in (I_DEFAULT, 1, 0):
        r, _ = evaluate(ev, T, Cc, budget, warp_slots=50000000)
        assert ev.dbg_item_stats()[1] > 100
        assert_same(ref, r, f"{sign}: forced splits, budget {budget}")
    ev.close()


@pytest.mark.parametrize("sign", list(SIGNS))
def test_fine_map_several_z_chunks(sign):
    """map resolution 0.25 m under 13 m windows: 53 voxels per axis, two z-chunks per window"""
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = 32
    occ = W.random_map(96, 96, 96, p=0.01, seed=4, slabs=1)
    T, Cc, _ = W.make_trajectory(3, [6, 6, 6], [18, 18, 18], seed=5, jitter=0.2)
    V, F = W.rounded_cone_mesh(n_theta=16, n_prof=12)
    ev = make_ev(cfg, occ, V, F, None, sign, res=0.25)
    ref, _ = evaluate(ev, T, Cc, 0)
    got, st = evaluate(ev, T, Cc, 4096)
    assert st["overflow"] == 0
    _, win = check_lists(ev, occ, cfg, T, Cc)
    assert np.all(win[:, 5] - win[:, 4] + 1 > 32), "windows should span more than one z-chunk"
    assert_same(ref, got, f"{sign} fine map: lists vs no lists")
    got, st = evaluate(ev, T, Cc, 200)
    assert 0 < st["overflow"] < st["runs"], st
    check_lists(ev, occ, cfg, T, Cc)
    assert_same(ref, got, f"{sign} fine map: overflowing budget")
    got, _ = evaluate(ev, T, Cc, 4096, warp_slots=50000000)
    assert ev.dbg_item_stats()[1] > 0
    assert_same(ref, got, f"{sign} fine map: forced splits")
    ev.close()


@pytest.mark.parametrize("sign", list(SIGNS))
def test_windows_clamped_at_map_faces(sign):
    """a trajectory through a 20^3 map, partly outside it: windows clamped at the low and the high faces"""
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = 64
    occ = W.random_map(20, 20, 20, p=0.06, seed=7, slabs=1)
    T, Cc, _ = W.make_trajectory(6, [-2, -2, -2], [22, 22, 22], seed=8, jitter=0.2)
    V, F = W.rounded_cone_mesh(n_theta=16, n_prof=12)
    ev = make_ev(cfg, occ, V, F, None, sign)
    ref, _ = evaluate(ev, T, Cc, 0)
    got, st = evaluate(ev, T, Cc, 256)
    assert st["overflow"] == 0
    _, win = check_lists(ev, occ, cfg, T, Cc)
    assert np.any(win[:, 0::2] == 0) and np.any(win[:, 1::2] == 19), "no clamped window"
    assert_same(ref, got, f"{sign} clamped windows: lists vs no lists")
    ev.close()


@pytest.mark.parametrize("sign", list(SIGNS))
def test_sharded_launches_lists_vs_fallback(bench, sign):
    """set_shard(r, 8) on one GPU: each rank's local runs (~54 / 8 samples) against its own enumeration"""
    cfg, occ, T, Cc, V, F, pp = bench
    n = 16 if sign == "pseudonormal" else 4
    T, Cc = T[:n].copy(), np.asarray(Cc).reshape(3, 64 * 6)[:, :6 * n].reshape(-1).copy()
    ev = make_ev(cfg, occ, V, F, pp, sign)
    for r in range(8):
        ev.set_shard(r, 8)
        ref, _ = evaluate(ev, T, Cc, 0)
        got, st = evaluate(ev, T, Cc, I_DEFAULT)
        assert st["overflow"] == 0
        check_lists(ev, occ, cfg, T, Cc, rank=r, world=8)
        assert_same(ref, got, f"{sign} shard {r}/8: lists vs no lists")
    ev.close()
