#!/usr/bin/env python
"""bench_dynlimits.py — the dynamic-limit certificate (isdf_trajectory_dynamics) on an H100; prints one JSON line.

  python bench_dynlimits.py --steps K --warmup W [--small] [--no-batch] [--batch-total B] [--lbfgs-iterations I]

Workloads (bench.py's, imported from it so both measure the same inputs), default parameters except K = 64, the reference config's
integral_intervs (bench.py samples 256 per piece): vmax = omgmax = 10, tolerances 1e-3 / 1e-4, max_depth 16, 2048 samples per trajectory:
  single   bench.py's 64-piece trajectory;
  batched  bench.py's batch problems (1024 restarts x 64 pieces) after I device L-BFGS iterations, certified in one call.
One step = one isdf_trajectory_dynamics_device call, timed with CUDA events. Prints ms per call, rounds, samples added, upper - attained per
quantity, the verdict mix and the undecided intervals, with the card's name and power limit read in the same run. Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True      # importing bench.py must leave no __pycache__ behind in a read-only tree

import bench as B   # noqa: E402

SUMMARY_BYTES = 168


def summaries(d_sum, n):
    import isdf_b200 as I
    raw = d_sum.cpu().numpy().tobytes()
    return [I.DynamicsSummary.from_buffer_copy(raw[SUMMARY_BYTES * b:SUMMARY_BYTES * (b + 1)]).as_dict() for b in range(n)]


def run(ev, N, dT, dC, prm, nB, steps, warmup, stream):
    import torch
    import isdf_b200 as I
    d_sum = torch.zeros(SUMMARY_BYTES // 8 * nB, dtype=torch.float64, device="cuda")
    times = []
    l0 = ev.stats().kernel_launches
    for k in range(warmup + steps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ev.trajectory_dynamics_device(N, dT.data_ptr(), dC.data_ptr(), prm, d_sum.data_ptr(), stream)
        e1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            times.append(e0.elapsed_time(e1))
    launches = (ev.stats().kernel_launches - l0) // (warmup + steps)
    summ = summaries(d_sum, nB)
    K, N0 = prm.samples_per_piece, N // nB
    gap = np.array([s["upper"] - s["attained"] for s in summ])
    gap_thr_min = np.array([s["thrust_attained_min"] - s["thrust_lower"] for s in summ])
    return {"ms_per_call": statistics.mean(times), "ms_min": min(times), "ms_max": max(times), "rounds": int((launches - 2) // 2),
            "kernel_launches_per_call": int(launches), "initial_samples": N * (K + 1),
            "samples_added": int(sum(s["samples"] - N0 * (K + 1) for s in summ)),
            "verdicts": {"feasible": sum(s["verdict"] == I.FEASIBLE for s in summ), "violating": sum(s["verdict"] == I.VIOLATING for s in summ),
                         "undecided": sum(s["verdict"] == 0 for s in summ)},
            "max_upper_minus_attained": dict(zip(I.DYN_QUANTITIES, [float(x) for x in np.nanmax(gap, axis=0)])),
            "max_thrust_attained_min_minus_lower": float(np.nanmax(gap_thr_min)),
            "undecided_intervals": int(sum(s["undecided_intervals"] for s in summ)), "max_depth_reached": max(s["depth"] for s in summ),
            "trajectories_at_sample_cap": int(sum(s["samples"] - N0 * (K + 1) >= prm.max_samples_per_traj for s in summ)),
            "first_summary": {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in summ[0].items()} if nB == 1 else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--small", action="store_true", help="tiny workload for plumbing checks (not a bench value)")
    ap.add_argument("--no-batch", action="store_true")
    ap.add_argument("--batch-total", type=int, default=1024)
    ap.add_argument("--lbfgs-iterations", type=int, default=8)
    args = ap.parse_args()

    import torch
    import isdf_b200 as I
    w, cfg, occ, T, Cc, V, F = B.make_workload(args.small)
    N = w["pieces"]
    ev = I.Evaluator(cfg, device=0)
    stream = torch.cuda.current_stream().cuda_stream
    dT, dC = torch.from_numpy(np.ascontiguousarray(T)).cuda(), torch.from_numpy(np.ascontiguousarray(Cc)).cuda()
    K = 64
    prm = ev.dynamics_params(K=K)
    line = {"metric": "dynamics_ms_per_trajectory", "value": None, "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "higher_is_better": False, "dtype": "f64", "data": "synthetic",
            "config": {"workload": B.workload_name(w) + "; one step = isdf_trajectory_dynamics_device over the whole trajectory",
                       "K": prm.samples_per_piece, "vmax": prm.vmax, "omgmax": prm.omgmax, "thetamax": prm.thetamax,
                       "tol": [prm.tol_v, prm.tol_a, prm.tol_omg, prm.tol_theta, prm.tol_thrust], "max_depth": prm.max_depth,
                       "max_samples_per_traj": prm.max_samples_per_traj}}
    try:
        line["gpu"] = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        line["gpu"] = None
    line["single"] = run(ev, N, dT, dC, prm, 1, args.steps, args.warmup, stream)
    line["value"] = line["single"]["ms_per_call"]
    if not args.no_batch:
        ev.set_map_u8(occ, [0, 0, 0], 1.0)
        ev.set_shape_mesh(V, F, w["poly_params"], I.MESH_SIGN_EXACT)
        Bt, N0 = (64 if args.small else args.batch_total), w["pieces"]
        xs, heads, tails = B.batch_problems(Bt, N0, w["map_dim"])
        hh, tt = heads.reshape(Bt, 3, 3).transpose(0, 2, 1), tails.reshape(Bt, 3, 3).transpose(0, 2, 1)
        t0 = time.perf_counter()
        ev.lbfgs_batch(hh, tt, 20.0, xs, ev.lbfgs_params(max_iterations=args.lbfgs_iterations))
        lb_s = time.perf_counter() - t0
        Tb, Cb, _ = ev.batch_trajectories(Bt, N0)
        dTb, dCb = torch.from_numpy(Tb).cuda(), torch.from_numpy(Cb).cuda()
        line["batched"] = {"restarts": Bt, "pieces_per_restart": N0, "lbfgs_iterations": args.lbfgs_iterations, "lbfgs_seconds": lb_s,
                           **run(ev, Bt * N0, dTb, dCb, ev.dynamics_params(K=K, N0=N0), Bt, max(1, args.steps // 2), 1, stream)}
    print(json.dumps(line))
    ev.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
