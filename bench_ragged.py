"""Ragged-batch benchmark: one ragged call over problems of many piece counts against one uniform call per distinct N on the same problems.

Workload: B = 128 and 1024 problems, N drawn uniformly from 2..64 plus one problem of N = 290 (the largest the solver takes), in a seeded
random order.
  mid-end : getOriTraj (isdf_midend_batch_ragged vs isdf_midend_batch per N) on waypoints selected from seeded A*-like paths; default
            parameters except cancel_after (--midend-cancel) so that a run stays short.
  L-BFGS  : the back end (isdf_lbfgs_batch_ragged vs isdf_lbfgs_batch per N) on the time-integral term with collision (Ball robot, the
            three-slit map), max_iterations = --backend-iterations.
Prints one JSON line per (stage, B): wall ms of each arm (host clock around the synchronous host entry points, best of --reps after one
warm-up call), the rounds of the ragged call and the sum of the per-N calls' rounds, the number of groups, and whether every output
(x, f, ret, iterations, evaluations; T and coeffs for the mid-end) is bit-identical between the arms. Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def piece_counts(B, seed):
    rng = np.random.default_rng(seed)
    Ns = list(rng.integers(2, 65, size=B - 1)) + [290]
    return [int(n) for n in rng.permutation(Ns)]


def _same(a, b):
    return bool(np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True))


def _best(fn, reps):
    fn()                                                   # warm-up: allocations, module load
    best, out = None, None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ms = 1e3 * (time.perf_counter() - t0)
        best = ms if best is None else min(best, ms)
    return best, out


def bench_midend(ev, B, seed, reps, cancel):
    import isdf_b200 as I
    import midend_cases as M
    Ns = piece_counts(B, seed)
    paths, heads, tails = [], np.zeros((B, 3, 3)), np.zeros((B, 3, 3))
    for b, N in enumerate(Ns):
        paths.append(M.astar_like_path(3 * (N - 1) + 2, seed + b))
        heads[b, :, 0], tails[b, :, 0] = paths[b][0], paths[b][-1]
    wps, pieces = I.path_waypoints(paths, 1.0)
    assert list(pieces) == Ns
    Q = [np.asarray(w).reshape(-1, 3) for w in wps]
    p = ev.midend_params(cancel_after=cancel)
    groups = sorted(set(Ns))

    def grouped():
        out = {}
        for N in groups:
            idx = [b for b in range(B) if Ns[b] == N]
            out[N] = (idx, ev.midend_batch(heads[idx], tails[idx], np.array([Q[b] for b in idx]).reshape(len(idx), N - 1, 3), p))
        return out
    t_r, r = _best(lambda: ev.midend_batch_ragged(heads, tails, Q, p), reps)
    t_g, g = _best(grouped, reps)
    same = True
    for N, (idx, m) in g.items():
        for q, b in enumerate(idx):
            same &= _same(m["x"][q], r["x"][b]) and _same(m["T"][q], r["T"][b]) and _same(m["coeffs"].reshape(3, -1, 6 * N)[:, q, :].reshape(-1), r["coeffs"][b])
            same &= all(_same(m[k][q], r[k][b]) for k in ("f", "ret", "iterations", "evaluations"))
    return dict(stage="midend", B=B, groups=len(groups), cancel_after=cancel, ragged_ms=round(t_r, 2), grouped_ms=round(t_g, 2),
                speedup=round(t_g / t_r, 3), ragged_rounds=r["rounds"], grouped_rounds_sum=sum(m["rounds"] for _, m in g.values()),
                max_evaluations=int(r["evaluations"].max()), identical=bool(same))


def bench_lbfgs(ev, B, seed, reps, iters):
    import workloads as W
    Ns = piece_counts(B, seed)
    rng = np.random.default_rng(seed)
    heads, tails, xs = np.zeros((B, 3, 3)), np.zeros((B, 3, 3)), []
    for b, N in enumerate(Ns):
        wp = W.random_walk_waypoints(N, [0, 0, 0], [50, 50, 34], seed=seed + b)
        heads[b, :, 0], tails[b, :, 0] = wp[0], wp[-1]
        xs.append(np.concatenate([rng.normal(size=N) * 0.4 + 0.8, (wp[1:-1] + rng.normal(size=(N - 1, 3)) * 0.2).reshape(-1)]))
    prm = ev.lbfgs_params(max_iterations=iters)
    groups = sorted(set(Ns))

    def grouped():
        out = {}
        for N in groups:
            idx = [b for b in range(B) if Ns[b] == N]
            out[N] = (idx, ev.lbfgs_batch(heads[idx], tails[idx], 20.0, np.array([xs[b] for b in idx]), prm))
        return out
    t_r, r = _best(lambda: ev.lbfgs_batch_ragged(heads, tails, 20.0, xs, prm), reps)
    t_g, g = _best(grouped, reps)
    same = True
    for N, (idx, m) in g.items():
        for q, b in enumerate(idx):
            same &= _same(m["x"][q], r["x"][b]) and all(_same(m[k][q], r[k][b]) for k in ("f", "ret", "iterations", "evaluations"))
    return dict(stage="lbfgs", B=B, groups=len(groups), max_iterations=iters, ragged_ms=round(t_r, 2), grouped_ms=round(t_g, 2),
                speedup=round(t_g / t_r, 3), ragged_rounds=r["rounds"], grouped_rounds_sum=sum(m["rounds"] for _, m in g.values()),
                max_evaluations=int(r["evaluations"].max()), identical=bool(same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="128,1024")
    ap.add_argument("--stages", default="midend,lbfgs")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--midend-cancel", type=int, default=500)
    ap.add_argument("--backend-iterations", type=int, default=30)
    a = ap.parse_args()
    import torch
    import isdf_b200 as I
    import workloads as W
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the ragged-batch benchmark measures the GPU")
    gpu = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode().strip()
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = 16
    ev = I.Evaluator(cfg)
    ev.set_map_u8(W.three_slit_map(64, 64, 64, noise=0.03, seed=3), [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    for B in [int(v) for v in a.batches.split(",")]:
        for st in a.stages.split(","):
            row = bench_midend(ev, B, 11 + B, a.reps, a.midend_cancel) if st == "midend" else bench_lbfgs(ev, B, 17 + B, a.reps, a.backend_iterations)
            row["gpu"] = gpu
            print(json.dumps(row), flush=True)
    ev.close()


if __name__ == "__main__":
    main()
