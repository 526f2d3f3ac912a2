"""Device-resident lock-step L-BFGS (isdf_lbfgs_batch, csrc/isdf_lbfgs.cuh) == the host drivers (host/isdf_lbfgs.hpp), bit for bit:
  * every instance against the SEQUENTIAL single-instance driver run on its own problem (callback = the same device kernels with B = 1);
  * the whole batch against the host lock-step driver (one PCIe round trip of all iterates per round), incl. return codes and counters."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W
from common import small_case, BMIN, MESHES

pytestmark = pytest.mark.gpu


def problems(B, N0, seed=200):
    rng = np.random.default_rng(9)
    heads, tails, X = [], [], []
    for b in range(B):
        wp = W.random_walk_waypoints(N0, [0, 0, 0], [50, 50, 34], seed=seed + b)
        h, t = np.zeros((3, 3)), np.zeros((3, 3))
        h[:, 0], t[:, 0] = wp[0], wp[-1]
        h[:, 1] = rng.normal(size=3) * 0.3
        tau = rng.normal(size=N0) * 0.4 + 0.8
        X.append(np.concatenate([tau, (wp[1:-1] + rng.normal(size=(N0 - 1, 3)) * 0.2).reshape(-1)]))
        heads.append(h); tails.append(t)
    return np.array(heads), np.array(tails), np.array(X)


@pytest.mark.parametrize("robot", ["Ball", "mesh"])
def test_device_lockstep_lbfgs_equals_host_drivers(robot):
    import host_lib as H
    cfg, occ, _, _, _ = small_case(N=6, K=16, seed=3)
    cfg.vmax, cfg.omgmax = 1.2, 0.5
    B, N0, rho = 7, 6, 20.0
    heads, tails, X = problems(B, N0)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        ev.set_shape_mesh(V, F, [0, 0, 0, 120, 0, 0])
    else:
        ev.set_shape_named(robot)
    max_it = 14
    prm = ev.lbfgs_params(max_iterations=max_it, mem_size=8, past=3, delta=1e-7)
    dev = ev.lbfgs_batch(heads, tails, rho, X, prm)
    assert set(dev["ret"]) <= {0, 1, -1008, -1009, -1007, -1010, -1004}, dev["ret"]     # stop / convergence / max-iteration / line-search exits
    assert dev["iterations"].max() >= 3 and np.all(dev["evaluations"] >= dev["iterations"])
    c0, _ = ev.callback_batch(heads, tails, rho, X)
    assert np.all(dev["f"] < c0)                                                          # every instance made progress
    # (1) sequential single-instance driver per problem, callback = the same batched entry point with B = 1
    for b in range(B):
        def fun(x, b=b):
            c, g = ev.callback_batch(heads[b], tails[b], rho, x[None, :])
            return float(c[0]), g[0]
        r = H.lbfgs_minimize(fun, X[b], mem_size=8, past=3, delta=1e-7, g_epsilon=0.0, max_iterations=max_it)
        assert r["ret"] == dev["ret"][b] and r["iterations"] == dev["iterations"][b] and r["evaluations"] == dev["evaluations"][b], (b, r["ret"], dev["ret"][b])
        assert np.array_equal(r["x"], dev["x"][b]) and r["f"] == dev["f"][b], (b, np.abs(r["x"] - dev["x"][b]).max())
    # (2) host lock-step driver over the batch
    L = H.lib()
    Xl = np.ascontiguousarray(X).copy().reshape(-1)
    fl, rl = np.zeros(B), np.zeros(B, dtype=np.int32)
    itl, evl, stl = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32), C.c_int()
    ipt = C.POINTER(C.c_int)
    hh = np.ascontiguousarray(np.swapaxes(heads, 1, 2)).reshape(B, 9)
    tt = np.ascontiguousarray(np.swapaxes(tails, 1, 2)).reshape(B, 9)
    rounds = L.isdf_host_lbfgs_batch_backend(ev.h, B, N0, hh.ctypes.data_as(H.dp), tt.ctypes.data_as(H.dp), rho, Xl.ctypes.data_as(H.dp), fl.ctypes.data_as(H.dp),
                                             rl.ctypes.data_as(ipt), 8, 3, 1e-7, 0.0, max_it, itl.ctypes.data_as(ipt), evl.ctypes.data_as(ipt), C.byref(stl))
    assert stl.value == 0 and rounds == dev["rounds"]
    assert np.array_equal(Xl.reshape(B, -1), dev["x"]) and np.array_equal(fl, dev["f"])
    assert np.array_equal(rl, dev["ret"]) and np.array_equal(itl, dev["iterations"]) and np.array_equal(evl, dev["evaluations"])
    ev.close()


def test_lbfgs_batch_argument_validation():
    cfg, occ, _, _, _ = small_case(N=4, K=8, seed=3)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_named("Ball")
    heads, tails, X = problems(2, 4)
    bad = ev.lbfgs_params(mem_size=0)
    with pytest.raises(I.IsdfError) as e:
        ev.lbfgs_batch(heads, tails, 20.0, X, bad)
    assert e.value.code == -1
    # mem_size 1..64 (the history ring's bound); a refused call leaves f NaN
    assert np.all(np.isfinite(ev.lbfgs_batch(heads, tails, 20.0, X, ev.lbfgs_params(mem_size=64, max_iterations=3))["f"]))
    hh = np.ascontiguousarray(np.swapaxes(heads, 1, 2)).reshape(-1)
    tt = np.ascontiguousarray(np.swapaxes(tails, 1, 2)).reshape(-1)
    for p in (ev.lbfgs_params(mem_size=65), bad):
        x, f = np.ascontiguousarray(X).copy(), np.zeros(2)
        r = ev.lib.isdf_lbfgs_batch(ev.h, 2, 4, hh.ctypes.data_as(C.POINTER(C.c_double)), tt.ctypes.data_as(C.POINTER(C.c_double)), 1, 20.0, C.byref(p),
                                    x.ctypes.data_as(C.POINTER(C.c_double)), f.ctypes.data_as(C.POINTER(C.c_double)), None, None, None, None)
        assert r == -1 and np.all(np.isnan(f))
    ev.close()
