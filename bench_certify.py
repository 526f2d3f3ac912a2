#!/usr/bin/env python
"""bench_certify.py — the continuous clearance certificate (isdf_trajectory_certify) on an H100; prints one JSON line.

  python bench_certify.py --steps K --warmup W [--small] [--no-batch] [--batch-total B] [--lbfgs-iterations I]

Workload: bench.py's map (512^3 random voxels), 3900-triangle mesh robot and 64-piece trajectory (imported from bench.py, so both measure
the same inputs), K_c = 16, reach = 3.0. One step = one isdf_trajectory_certify_device call, timed with CUDA events. Lines:
  single  the bench trajectory on the bench map at margin = 0.05 below its dense minimum clearance (isdf_trajectory_clearance at
          K_c = 2^14), or 0 when that minimum is below 0.05 (the trajectory collides: one round decides it);
  carved  the same trajectory on the bench map with every voxel within 6 m of its path removed, at margin = dense minimum - 0.05: the
          refinement has to work near the closest approach;
  batched restarts of bench.py's batch problems after the device-resident L-BFGS, certified in one call at margin = safety_hor.
Prints device time, rounds, samples added and the verdict mix, with the card's name and power limit read in the same run. Writes nothing
to the tree.
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
import workloads as W   # noqa: E402


def timed(n, warmup, call):
    import torch
    times = []
    for k in range(n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call(k)
        e1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            times.append(e0.elapsed_time(e1))
    return times


def summaries(d_sum, n):
    import isdf_b200 as I
    raw = d_sum.cpu().numpy().tobytes()
    return [I.CertifySummary.from_buffer_copy(raw[56 * b:56 * (b + 1)]).as_dict() for b in range(n)]


def run(ev, N, dT, dC, prm, nB, steps, warmup, stream):
    import torch
    d_sum = torch.zeros(7 * nB, dtype=torch.float64, device="cuda")
    l0 = ev.stats().kernel_launches
    times = timed(warmup + steps, warmup, lambda k: ev.trajectory_certify_device(N, dT.data_ptr(), dC.data_ptr(), prm, d_sum.data_ptr(), stream))
    launches = (ev.stats().kernel_launches - l0) // (warmup + steps)
    summ = summaries(d_sum, nB)
    K = prm.clearance.samples_per_piece
    N0 = N // nB
    verdicts = {"certified": sum(s["verdict"] == 1 for s in summ), "colliding": sum(s["verdict"] == -1 for s in summ),
                "undecided": sum(s["verdict"] == 0 for s in summ)}
    added = sum(s["samples"] - N0 * (K + 1) for s in summ)
    # rounds = scan launches: 1 init + per round (scan + 2 interval kernels) - the last round's scan + 1 summary
    rounds = (launches - 2 + 1) // 3
    return {"ms_per_call": statistics.mean(times), "ms_min": min(times), "ms_max": max(times), "rounds": int(rounds),
            "kernel_launches_per_call": int(launches), "initial_samples": N * (K + 1), "samples_added": int(added), "verdicts": verdicts,
            "max_depth_reached": max(s["depth"] for s in summ), "undecided_intervals": sum(s["undecided_intervals"] for s in summ),
            "first_summary": summ[0] if nB == 1 else None}


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
    N, K, reach = w["pieces"], 16, 3.0
    ev = I.Evaluator(cfg, device=0)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_mesh(V, F, w["poly_params"], I.MESH_SIGN_EXACT)
    stream = torch.cuda.current_stream().cuda_stream
    _, _, dsum = ev.trajectory_clearance(T, Cc, 2 ** 14, reach, 0.0)
    dmin = dsum[0]["min_clearance"]
    margin = max(dmin - 0.05, 0.0)
    dT, dC = torch.from_numpy(np.ascontiguousarray(T)).cuda(), torch.from_numpy(np.ascontiguousarray(Cc)).cuda()
    prm = ev.certify_params(K, reach, margin, 0)
    single = run(ev, N, dT, dC, prm, 1, args.steps, args.warmup, stream)
    line = {"metric": "certify_ms_per_trajectory", "value": single["ms_per_call"], "unit": "ms", "n_gpus": 1, "steps": args.steps,
            "warmup": args.warmup, "higher_is_better": False, "dtype": "f64", "data": "synthetic",
            "config": {"workload": B.workload_name(w) + "; one step = isdf_trajectory_certify_device over the whole trajectory", "K_c": K,
                       "reach": reach, "margin": margin, "dense_min_clearance": dmin, "max_depth": prm.max_depth,
                       "max_samples_per_traj": prm.max_samples_per_traj},
            "single": single}
    try:
        line["gpu"] = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        line["gpu"] = None
    # carved: clear a 6 m ball of voxels around path points 0.1 s apart, then certify 0.05 below the new dense minimum
    tt = np.arange(0.0, float(np.sum(T)), 0.1)
    P = W.traj_eval(T, Cc, tt)
    occ_c = occ.copy()
    rad = 6
    off = np.stack(np.meshgrid(*(np.arange(-rad, rad + 1),) * 3, indexing="ij"), -1).reshape(-1, 3)
    off = off[np.linalg.norm(off, axis=1) <= rad]
    for p in P:
        idx = np.floor(p).astype(int) + off
        idx = idx[np.all((idx >= 0) & (idx < np.array(occ.shape)), axis=1)]
        occ_c[idx[:, 0], idx[:, 1], idx[:, 2]] = 0
    ev.set_map_u8(occ_c, [0, 0, 0], 1.0)
    _, _, csum = ev.trajectory_clearance(T, Cc, 2 ** 14, reach, 0.0)
    cmin = csum[0]["min_clearance"]
    prm_c = ev.certify_params(K, reach, max(cmin - 0.05, 0.0), 0)
    line["carved"] = {"dense_min_clearance": cmin, "margin": prm_c.clearance.margin, "carve_radius_m": rad,
                      **run(ev, N, dT, dC, prm_c, 1, args.steps, args.warmup, stream)}
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    if not args.no_batch:
        Bt, N0 = (64 if args.small else args.batch_total), w["pieces"]
        xs, heads, tails = B.batch_problems(Bt, N0, w["map_dim"])
        hh, tt = heads.reshape(Bt, 3, 3).transpose(0, 2, 1), tails.reshape(Bt, 3, 3).transpose(0, 2, 1)
        t0 = time.perf_counter()
        ev.lbfgs_batch(hh, tt, 20.0, xs, ev.lbfgs_params(max_iterations=args.lbfgs_iterations))
        lb_s = time.perf_counter() - t0
        Tb, Cb, _ = ev.batch_trajectories(Bt, N0)
        dTb, dCb = torch.from_numpy(Tb).cuda(), torch.from_numpy(Cb).cuda()
        prm_b = ev.certify_params(K, reach, cfg.safety_hor, N0)
        line["batched"] = {"restarts": Bt, "pieces_per_restart": N0, "margin": cfg.safety_hor, "lbfgs_iterations": args.lbfgs_iterations,
                           "lbfgs_seconds": lb_s, **run(ev, Bt * N0, dTb, dCb, prm_b, Bt, max(1, args.steps // 4), 1, stream)}
    print(json.dumps(line))
    ev.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
