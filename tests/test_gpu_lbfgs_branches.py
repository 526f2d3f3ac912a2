"""The device lock-step L-BFGS (lbfgs_rounds + k_lbfgs_feed, csrc/isdf_lbfgs.cuh) at every exit and branch of the case catalogue
(tests/lbfgs_cases.py), through isdf_dbg_lbfgs_rounds (the unchanged rounds on a host objective):
  * every case at B = 1 equals the reference-compiled lbfgs.hpp's committed run bit for bit: trace, x, f, return code, evaluations;
  * batches of B = 63, 64, 65 and 1000 mixed exits equal the host sequential driver instance by instance;
  * a round cap (max_rounds) leaves every unfinished instance on its last accepted iterate with LBFGSERR_MAXIMUMITERATION;
and the back end's and the mid-end's entry points around the same rounds."""
import numpy as np
import pytest
import isdf_b200 as I
import host_lib as H
import lbfgs_cases as LC
from common import small_case, BMIN, MESHES
from test_lbfgs_branches_cpu import CASES, NAMES, golden, same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ev():
    e = I.Evaluator()
    yield e
    e.close()


def _params(ev, case, **kw):
    return ev.lbfgs_params(**{**case["params"], **kw})


@pytest.mark.parametrize("name", NAMES)
def test_every_case_equals_reference_golden_at_B1(ev, name):
    k = NAMES.index(name)
    c = CASES[k]
    g = golden(k)
    r = ev.dbg_lbfgs_rounds(c["fun"], c["x0"][None, :], _params(ev, c), cancel_after=c["cancel_after"])
    e = int(r["evaluations"][0])
    assert r["ret"][0] == LC.sequential_ret(c, g["ret"]) and e == g["evaluations"] and r["rounds"] == e, (name, r["ret"][0], e)
    assert np.array_equal(r["trace"][:e, 0], g["trace"]), name             # instance b's trace: its requested points in rounds 1..evaluations
    assert np.array_equal(r["x"][0], g["x"]), name
    if c["f_unwritten"]:
        assert g["f"] == 0.0 and r["f"][0] == LC.one(c["fun"])(r["x"][0])[0], name
    else:
        assert same(r["f"][0], g["f"]), name
    assert c["reached"](dict(ret=int(r["ret"][0]), iterations=int(r["iterations"][0]), evaluations=e, x=r["x"][0], f=r["f"][0], trace=r["trace"][:e, 0]))


# ---- batches: one objective, seeded starts that end in every way (at the start, STOP, NaN in the line search, iteration and line-search caps)
BATCH_PARAMS = dict(LC.DEFAULTS, mem_size=5, past=3, delta=1e-7, g_epsilon=1e-7, max_iterations=30, max_linesearch=6)


def batch_family(B, seed):
    rng = np.random.default_rng(seed)
    c = np.array([1.0, -0.5, 0.25, 2.0, -1.5, 0.75])
    fun = LC.beyond(LC.quad_quartic([0.05, 0.3, 1.0, 3.0, 0.1, 0.6], c, [0.5, 0.1, 2.0, 0.01, 1.0, 0.2]), 4.0, np.nan)
    X0 = c + rng.normal(size=(B, 6)) * rng.choice([0.0, 0.3, 1.0, 2.0], size=(B, 1))
    return fun, X0


def host_sequential(fun, x0, **over):
    kw = {k: BATCH_PARAMS[k] for k in LC.HOST_KEYS}
    kw.update(over)
    r = H.lbfgs_minimize(LC.one(fun), x0, **kw)
    r["trace"] = np.array(r["trace"])
    return r


@pytest.mark.parametrize("B", [63, 64, 65, 1000])
def test_batches_equal_host_sequential_driver(ev, B):
    fun, X0 = batch_family(B, 5 + B)
    r = ev.dbg_lbfgs_rounds(fun, X0, ev.lbfgs_params(**BATCH_PARAMS))
    assert r["rounds"] == r["evaluations"].max() == len(r["trace"])
    assert len(set(r["ret"].tolist())) >= 4, np.unique(r["ret"], return_counts=True)
    assert len(set(r["evaluations"].tolist())) >= 10                          # instances finish in many different rounds
    for b in range(B):
        s = host_sequential(fun, X0[b])
        e = int(r["evaluations"][b])
        assert r["ret"][b] == s["ret"] and r["iterations"][b] == s["iterations"] and e == s["evaluations"], (B, b, r["ret"][b], s["ret"])
        assert np.array_equal(r["trace"][:e, b], s["trace"]), (B, b)
        assert np.array_equal(r["x"][b], s["x"]) and same(r["f"][b], s["f"]), (B, b)
        assert (r["trace"][e:, b] == r["x"][b]).all(), (B, b)                   # finished: its requested point never changes again


def test_round_cap_stops_every_running_instance_on_its_last_accepted_iterate(ev):
    B = 65
    fun, X0 = batch_family(B, 77)
    f1 = LC.one(fun)
    full = ev.dbg_lbfgs_rounds(fun, X0, ev.lbfgs_params(**BATCH_PARAMS))
    R = full["rounds"]
    cache = {}

    def capped_reference(b, k):   # the sequential driver stopped after k accepted iterations; (x0, f(x0)) before the first
        if (b, k) not in cache:
            cache[(b, k)] = (X0[b], f1(X0[b])[0]) if k == 0 else (lambda s: (s["x"], s["f"]))(host_sequential(fun, X0[b], max_iterations=k))
        return cache[(b, k)]
    cut_total = 0
    for rcap in range(1, R + 1):
        r = ev.dbg_lbfgs_rounds(fun, X0, ev.lbfgs_params(**BATCH_PARAMS, max_rounds=rcap))
        assert r["rounds"] == rcap
        running = full["evaluations"] > rcap
        cut_total += int(running.sum())
        for b in range(B):
            if not running[b]:
                assert r["ret"][b] == full["ret"][b] and np.array_equal(r["x"][b], full["x"][b]) and same(r["f"][b], full["f"][b]), (rcap, b)
                assert r["iterations"][b] == full["iterations"][b] and r["evaluations"][b] == full["evaluations"][b], (rcap, b)
                continue
            k = int(r["iterations"][b])
            assert r["ret"][b] == LC.ERR_MAXIMUMITERATION and r["evaluations"][b] == rcap, (rcap, b, r["ret"][b])
            assert k <= full["iterations"][b]
            x_ref, f_ref = capped_reference(b, k)
            assert np.array_equal(r["x"][b], x_ref) and same(r["f"][b], f_ref), (rcap, b, k)
            assert same(f1(r["x"][b])[0], r["f"][b]), (rcap, b)           # f is the objective at the reported x (NaN for a NaN start)
    assert cut_total > B


# ---- the back end: isdf_lbfgs_batch_device and isdf_lbfgs_batch ----------------------------------------------------------------------------
def _backend_ctx(robot):
    cfg, occ, _, _, _ = small_case(N=4, K=16, seed=3)
    cfg.vmax, cfg.omgmax = 1.2, 0.5
    e = I.Evaluator(cfg)
    e.set_map_u8(occ, BMIN, 1.0)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        e.set_shape_mesh(V, F, [0, 0, 0, 120, 0, 0])
    else:
        e.set_shape_named(robot)
    return e


def test_backend_device_entry_point_equals_host_entry_point():
    import torch
    import test_gpu_lbfgs_device as L
    e = _backend_ctx("Ball")
    B, N0, rho = 70, 4, 20.0
    heads, tails, X = L.problems(B, N0, seed=300)
    prm = e.lbfgs_params(max_iterations=10, mem_size=4, past=2, delta=1e-7)
    cm = lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2)).reshape(-1)
    dv = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")
    for per in (0, 1):
        h, t = (heads, tails) if per else (heads[0], tails[0])
        host = e.lbfgs_batch(h, t, rho, X, prm)
        assert host["rounds"] == host["evaluations"].max()
        d_h, d_t, d_x = dv(cm(h)), dv(cm(t)), dv(X.reshape(-1))
        d_f = torch.zeros(B, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            rounds = e.lbfgs_batch_device(B, N0, d_h.data_ptr(), d_t.data_ptr(), per, rho, d_x.data_ptr(), d_f.data_ptr(), None, None, None, prm,
                                          s.cuda_stream)
        s.synchronize()
        assert rounds == host["rounds"], per
        assert np.array_equal(d_x.cpu().numpy().reshape(B, -1), host["x"]) and np.array_equal(d_f.cpu().numpy(), host["f"]), per
    e.close()


@pytest.mark.parametrize("robot", ["Ball", "mesh"])
def test_backend_65_instances_equal_host_sequential_driver(robot):
    import test_gpu_lbfgs_device as L
    e = _backend_ctx(robot)
    B, N0, rho = 65, 4, 20.0
    heads, tails, X = L.problems(B, N0, seed=500)
    kw = dict(mem_size=3, past=2, delta=1e-6, g_epsilon=0.0, max_iterations=8)
    dev = e.lbfgs_batch(heads, tails, rho, X, e.lbfgs_params(**kw))
    assert dev["rounds"] == dev["evaluations"].max()
    for b in range(B):
        def fun(x, b=b):
            c, g = e.callback_batch(heads[b], tails[b], rho, x[None, :])
            return float(c[0]), g[0]
        r = H.lbfgs_minimize(fun, X[b], **kw)
        assert r["ret"] == dev["ret"][b] and r["iterations"] == dev["iterations"][b] and r["evaluations"] == dev["evaluations"][b], (robot, b)
        assert np.array_equal(r["x"], dev["x"][b]) and r["f"] == dev["f"][b], (robot, b)
    e.close()


# ---- the mid-end under a round cap -------------------------------------------------------------------------------------------------
def test_midend_round_cap_reports_cut_off_plans_as_failures():
    import midend_cases as M
    cfg = I.default_config_values()
    cfg.integral_intervs = 64
    e = I.Evaluator(cfg)
    B, N0 = 12, 5
    hs, ts, Qs = zip(*(M.problem(N0, 600 + b) for b in range(B)))
    heads, tails, Q = np.array(hs), np.array(ts), np.array(Qs).reshape(B, N0 - 1, 3)
    full = e.midend_batch(heads, tails, Q)
    assert np.all(full["ret"] >= 0)
    rcap = int(np.median(full["evaluations"]))
    cut = e.midend_batch(heads, tails, Q, e.midend_params(max_rounds=rcap))
    running = full["evaluations"] > rcap
    assert running.any() and not running.all()
    assert np.all(cut["ret"][running] == LC.ERR_MAXIMUMITERATION) and np.array_equal(cut["ret"][~running], full["ret"][~running])
    cost, _ = e.midend_callback_batch(heads, tails, Q, cut["x"])
    assert np.array_equal(cost, cut["f"])                                       # f and x belong together: an evaluated, accepted iterate
    for b in np.flatnonzero(running):
        me = M.HostMidEnd(heads[b], tails[b], Q[b], K=64)
        h = me.optimize(max_iterations=int(cut["iterations"][b])) if cut["iterations"][b] > 0 else None
        if h is not None:
            assert np.array_equal(cut["x"][b], h["x"]) and cut["f"][b] == h["f"], b
    e.close()
