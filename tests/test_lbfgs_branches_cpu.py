"""The L-BFGS case catalogue (tests/lbfgs_cases.py) on the host drivers (host/isdf_lbfgs.hpp), CPU only: every case reaches its branch; the
sequential driver equals the reference-compiled utils/lbfgs.hpp's committed run (tests/golden/lbfgs_branches_reference.npz) bit for bit,
and the live reference build where oracle/_ref was built; the lock-step driver equals the sequential one instance by instance."""
import os
import numpy as np
import pytest
import host_lib as H
import oracle_lib as O
import lbfgs_cases as LC

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lbfgs_branches_reference.npz")
CASES = LC.cases()
NAMES = [c["name"] for c in CASES]


def golden(k, pre=""):
    z = np.load(G)
    assert [str(s) for s in z["names"]] == NAMES, "the catalogue changed: regenerate the golden (tests/golden/make_reference_golden.py)"
    return dict(trace=z[f"c{k}_{pre}trace"], x=z[f"c{k}_{pre}x"], f=float(z[f"c{k}_{pre}f"]), ret=int(z[f"c{k}_{pre}ret"]),
                evaluations=int(z[f"c{k}_{pre}evals"]))


def same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def sequential(c):
    return H.lbfgs_minimize(LC.one(c["fun"]), c["x0"], **LC.sequential_kwargs(c))


def assert_run_equal(a, b, what):
    assert a["ret"] == b["ret"], f"{what}: return code {a['ret']} vs {b['ret']}"
    assert a["evaluations"] == b["evaluations"] == len(a["trace"]) == len(b["trace"]), f"{what}: evaluations {a['evaluations']} vs {b['evaluations']}"
    for k, (p, q) in enumerate(zip(a["trace"], b["trace"])):
        assert np.array_equal(p, q), f"{what}: evaluation {k} at different points"
    assert np.array_equal(a["x"], b["x"]) and same(a["f"], b["f"]), what


@pytest.mark.parametrize("name", NAMES)
def test_case_reaches_its_branch(name):
    c = CASES[NAMES.index(name)]
    r = sequential(c)
    r["ret"] = LC.sequential_ret(c, r["ret"])
    assert c["reached"](r), (name, r["ret"], r["iterations"], r["evaluations"], LC.resets(r["trace"]))


@pytest.mark.parametrize("name", NAMES)
def test_sequential_driver_equals_reference_golden(name):
    k = NAMES.index(name)
    c = CASES[k]
    b = sequential(c)
    assert_run_equal(golden(k), dict(b, trace=np.array(b["trace"])), name)


@pytest.mark.skipif(not os.path.exists(O.REF_LBFGS), reason="oracle/_ref not built (needs the reference's sources)")
def test_live_reference_build_equals_golden():
    rl = O.RefLbfgs()
    if not rl.full:
        pytest.skip("oracle/_ref/libref_lbfgs.so was built from an older wrapper without the full parameter set")
    for k, c in enumerate(CASES):
        a = rl.minimize(LC.one(c["fun"]), c["x0"], **LC.sequential_kwargs(c))
        a["trace"] = np.array(a["trace"])
        assert_run_equal(a, golden(k, "ref_" if c["host_pinned"] else ""), c["name"])
        if c["host_pinned"]:   # the recorded divergence: the stand-in's maxCoeff keeps the leading NaN
            assert (a["ret"], golden(k)["ret"]) == (LC.ERR_INVALIDPARAMETERS, LC.CONVERGENCE) and a["evaluations"] == 1


def _lockstep_groups():
    """for every case: a batch of every catalogue objective of its n (its own first), all run with its parameters"""
    out = []
    for c in CASES:
        n = c["x0"].size
        out.append((c, [c] + [d for d in CASES if d is not c and d["x0"].size == n]))
    return out


@pytest.mark.parametrize("name", NAMES)
def test_lockstep_driver_equals_sequential(name):
    c, batch = next(g for g in _lockstep_groups() if g[0]["name"] == name)
    funs = [LC.one(d["fun"]) for d in batch]
    X0 = np.array([d["x0"] for d in batch])
    kw = LC.host_kwargs(c)
    rb = H.lbfgs_minimize_batch(lambda i, x: funs[i](x), X0, cancel_after=c["cancel_after"], **kw)
    assert rb["rounds"] == rb["evaluations"].max()
    for b, d in enumerate(batch):
        rs = H.lbfgs_minimize(funs[b], X0[b], **LC.sequential_kwargs(c))
        what = f"{name}: instance {b} ({d['name']})"
        assert rb["ret"][b] == LC.sequential_ret(c, rs["ret"]), what
        assert rb["iterations"][b] == rs["iterations"] and rb["evaluations"][b] == rs["evaluations"], what
        assert np.array_equal(rb["x"][b], rs["x"]), what
        if rs["ret"] == LC.ERR_INVALID_FUNCVAL and rs["f"] == 0.0 and np.isfinite(rb["f"][b]):
            assert rb["f"][b] == funs[b](rb["x"][b])[0], what   # the direction-norm exit: the sequential driver leaves f unwritten
        else:
            assert same(rb["f"][b], rs["f"]), what
