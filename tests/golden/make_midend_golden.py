"""Writes midend_reference.npz: the reference-form results the mid-end tests compare with where oracle/_ref/ was not built (no reference
tree): OriTraj::costFunction in the reference's form (reference-compiled MINCO + libm pow) on the CPU test's cost cases, the
reference-compiled lbfgs.hpp on the product's host cost for the CPU pin's runs, and one whole reference-form getOriTraj for the GPU test.
Run from the repository root after build(): python tests/golden/make_midend_golden.py"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "implicit-sdf-planner_b200", "py"))
import numpy as np  # noqa: E402
import oracle_lib as O  # noqa: E402
import midend_cases as M  # noqa: E402
import test_midend_cpu as T  # noqa: E402


def main():
    rm, rl = O.RefMinco(), O.RefLbfgs()
    out = {}
    for k, (N, head, tail, Q, x) in enumerate(T._cost_cases()):
        out[f"cost{k}_c"], out[f"cost{k}_g"] = M.ref_form_cost(rm, head, tail, Q, x)
    for k, (kind, N, seed, extra) in enumerate(T._lbfgs_cases() + [("nan", 4, 15, {})]):
        head, tail, Q = M.problem(N, seed)
        if kind == "nan":
            Q = Q.copy(); Q[1, 2] = np.nan
        me = M.HostMidEnd(head, tail, Q, cancel_after=extra.get("cancel_after", 8000))
        kw = dict(M.LB)
        if kind == "cancel":
            kw["max_iterations"] = extra["cancel_after"] + 1
        a = rl.minimize(me.cost, M.start_point(N, Q), **kw)
        out[f"lb{k}_ret"], out[f"lb{k}_evals"], out[f"lb{k}_x"], out[f"lb{k}_f"] = a["ret"], a["evaluations"], a["x"], a["f"]
        out[f"lb{k}_trace_sha256"] = M.trace_digest(a["trace"])
    head, tail, Q = M.ref_run_problem()
    r = M.ref_form_optimize(rm, rl, head, tail, Q)
    out["run_ret"], out["run_f"], out["run_x"], out["run_evals"] = r["ret"], r["f"], r["x"], r["evaluations"]
    np.savez_compressed(os.path.join(HERE, "midend_reference.npz"), **out)
    print("midend_reference.npz written")


if __name__ == "__main__":
    main()
