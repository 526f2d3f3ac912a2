#!/usr/bin/env python
"""bench_clearance.py — the trajectory clearance check (isdf_trajectory_clearance) on an H100; prints one JSON line.

  python bench_clearance.py --steps K --warmup W [--no-cpu-baseline] [--no-batch] [--batch-total B] [--lbfgs-iterations I]

Workload: the BASELINE configs[2] trajectory and map of bench.py (imported from it, so both measure the same inputs): 512^3 random
voxel map, 64-piece MINCO trajectory, 3900-triangle mesh robot, K_c = 256 samples per piece (S = 64 x 257 pose samples). One step = one
isdf_trajectory_clearance_device call over the whole trajectory, timed with CUDA events, L2 flushed before every check, a different
iterate every step; at reach = safety_hor and at reach = 3.0. Then a batched line: the 1024 restarts of configs[4] after the
device-resident L-BFGS, read back with isdf_get_batch_trajectories and checked in one call. Parity: the brute-force oracle
(tests/clearance_oracle.py) on a subset of the samples. Writes nothing to the tree.
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

import bench as B   # noqa: E402  (workload, iterates, clock sampler, restart problems: the same inputs as bench.py)


def timed_checks(ev, flush, n, call, warmup):
    import torch
    times = []
    for k in range(n):
        flush.zero_()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call(k)
        e1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            times.append(e0.elapsed_time(e1))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--small", action="store_true", help="tiny workload for plumbing checks (not a bench value)")
    ap.add_argument("--no-cpu-baseline", action="store_true", help="skip the parity check against the brute-force oracle")
    ap.add_argument("--no-batch", action="store_true", help="skip the batched line (1024 restarts after isdf_lbfgs_batch)")
    ap.add_argument("--batch-total", type=int, default=1024)
    ap.add_argument("--lbfgs-iterations", type=int, default=8)
    args = ap.parse_args()

    import torch
    import isdf_b200 as I
    w, cfg, occ, T, Cc, V, F = B.make_workload(args.small)
    N, K = w["pieces"], w["samples_per_piece"]
    S = N * (K + 1)
    dev = torch.device("cuda", 0)
    ev = I.Evaluator(cfg, device=0)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_mesh(V, F, w["poly_params"])
    stream = torch.cuda.current_stream().cuda_stream
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2 (H100)
    n_it = args.warmup + args.steps
    iters = B.make_iterates(w, T, Cc, n_it)
    d_T = torch.from_numpy(np.ascontiguousarray(T)).to(dev)
    d_C = [torch.from_numpy(np.ascontiguousarray(c)).to(dev) for c in iters]
    d_cl = torch.zeros(S, dtype=torch.float64, device=dev)
    d_vx = torch.zeros(S, dtype=torch.int64, device=dev)
    d_sm = torch.zeros(6, dtype=torch.float64, device=dev)          # one 48-byte isdf_clearance_summary
    sampler = B.ClockSampler(0)
    res = {}
    for reach in (cfg.safety_hor, 3.0):
        prm = ev.clearance_params(K, reach, min(cfg.safety_hor, reach), 0)
        times = timed_checks(ev, flush, n_it, lambda k: ev.trajectory_clearance_device(N, d_T.data_ptr(), d_C[k].data_ptr(), prm, d_cl.data_ptr(),
                                                                                        d_vx.data_ptr(), d_sm.data_ptr(), stream), args.warmup)
        pairs, searches = ev.dbg_clearance_counts()
        summ = I.ClearanceSummary.from_buffer_copy(d_sm.cpu().numpy().tobytes()).as_dict()
        res[reach] = {"ms_per_check": statistics.mean(times), "ms_min": min(times), "ms_max": max(times), "candidate_pairs": pairs,
                      "exact_searches": searches, "summary_last": summ}
    clocks = sampler.stop()
    line = {"metric": "clearance_checks_per_s", "value": 1e3 / res[cfg.safety_hor]["ms_per_check"], "unit": "checks/s", "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": res[cfg.safety_hor]["ms_per_check"], "higher_is_better": True,
            "dtype": "f64", "data": "synthetic",
            "config": {"workload": B.workload_name(w) + "; one step = isdf_trajectory_clearance_device over the whole trajectory", "samples": S,
                       "K_c": K, "margin": cfg.safety_hor, "l2": "flushed (512 MiB write) before every check",
                       "iterates": "distinct (trajectory moved ~1 cm per step)"},
            "clocks": clocks, "reach": {str(r): v for r, v in res.items()}}
    try:
        line["gpu"] = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        line["gpu"] = None
    # parity on a subset: the brute-force oracle tests every occupied voxel of the map for every sample (~0.5 s per sample at 512^3)
    if not args.no_cpu_baseline:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import oracle_lib as O
        import clearance_oracle as CO
        osh = O.Shape.mesh(V, F, w["poly_params"], wn_mode=O.WN_BH)
        pieces, Ks = [0, N // 2], 8
        Cm = np.asarray(iters[-1]).reshape(3, 6 * N)
        Ts = np.ascontiguousarray(T[pieces])
        Cs = np.ascontiguousarray(np.concatenate([Cm[:, 6 * i:6 * i + 6] for i in pieces], axis=1)).reshape(-1)
        par = {}
        for reach in (cfg.safety_hor, 3.0):
            clear, vox, _ = ev.trajectory_clearance(Ts, Cs, Ks, reach, min(cfg.safety_hor, reach))
            ref = CO.clearance(O.config_from(cfg), occ, [0, 0, 0], 1.0, osh, Ts, Cs, Ks, reach, min(cfg.safety_hor, reach))
            par[str(reach)] = {"max_abs_clearance_diff": float(np.abs(clear - ref["clear"]).max()), "witness_equal": bool(np.array_equal(vox, ref["voxel"]))}
        line["parity"] = {"against": "brute-force oracle (tests/clearance_oracle.py), last iterate", "tolerance": 1e-12,
                          "sample": f"pieces {pieces} of {N} at K_c = {Ks} ({len(pieces) * (Ks + 1)} samples): the oracle tests all "
                                    f"{int(occ.sum())} occupied voxels per sample", **par}
    # batched line: the restarts of configs[4] after the device-resident L-BFGS, read back and checked in one call
    if not args.no_batch:
        Bt, N0 = args.batch_total, w["pieces"]
        xs, heads, tails = B.batch_problems(Bt, N0, w["map_dim"])
        hh, tt = heads.reshape(Bt, 3, 3).transpose(0, 2, 1), tails.reshape(Bt, 3, 3).transpose(0, 2, 1)
        t0 = time.perf_counter()
        ev.lbfgs_batch(hh, tt, 20.0, xs, ev.lbfgs_params(max_iterations=args.lbfgs_iterations))
        lb_s = time.perf_counter() - t0
        Tb, Cb, _ = ev.batch_trajectories(Bt, N0)
        dTb, dCb = torch.from_numpy(Tb).to(dev), torch.from_numpy(Cb).to(dev)
        Sb = Bt * N0 * (K + 1)
        dclb, dvxb = torch.zeros(Sb, dtype=torch.float64, device=dev), torch.zeros(Sb, dtype=torch.int64, device=dev)
        dsmb = torch.zeros(6 * Bt, dtype=torch.float64, device=dev)
        prm = ev.clearance_params(K, cfg.safety_hor, cfg.safety_hor, N0)
        bt = timed_checks(ev, flush, 2 + max(1, args.steps // 4), lambda k: ev.trajectory_clearance_device(Bt * N0, dTb.data_ptr(), dCb.data_ptr(), prm,
                                                                                                            dclb.data_ptr(), dvxb.data_ptr(), dsmb.data_ptr(), stream), 2)
        raw = dsmb.cpu().numpy().tobytes()
        free = sum(I.ClearanceSummary.from_buffer_copy(raw[48 * b:48 * (b + 1)]).collision_free for b in range(Bt))
        ms = statistics.mean(bt)
        line["batched"] = {"value": Bt * 1e3 / ms, "unit": "checks/s", "ms_per_call": ms, "restarts": Bt, "samples_per_call": Sb,
                           "reach": cfg.safety_hor, "collision_free_restarts": int(free), "lbfgs_iterations": args.lbfgs_iterations, "lbfgs_seconds": lb_s,
                           "what": f"{Bt} restarts x {N0} pieces after isdf_lbfgs_batch, isdf_get_batch_trajectories, one isdf_trajectory_clearance_device call (N0 = {N0})"}
    print(json.dumps(line))
    ev.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
