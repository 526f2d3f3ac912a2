#!/usr/bin/env python
"""bench_states.py — executing trajectories (isdf_trajectory_states, isdf_pose_points) on an H100; prints one JSON line.

  python bench_states.py --steps K --warmup W

Trajectories: bench.py's 64-piece benchmark trajectory (imported from bench.py) as trajectory 0, and ragged plans of 2-290 pieces (32 distinct
MINCO trajectories, cycled) as the rest, in isdf_plan_batch's layout, on the device.
  states   isdf_trajectory_states_device at Q = 1e4, 1e6 and 3e6 queries over B = 128 and 1024 trajectories, in playback order (each
           trajectory's queries together, times increasing over [0, duration)). CUDA events around each call, the L2 flushed before it;
           median and spread over K calls after W warm-up calls. GB/s counts the 160-byte records written (the reads, 12 bytes per query plus
           the trajectories, are under 10 %), the fraction is of the H100 SXM data-sheet 3.35 TB/s.
  pose     isdf_pose_points_device: the vertices of bench.py's 3900-triangle mesh robot at 1e3 and 1e4 states (states from the 1e4-query
           run); GB/s counts the Q P 24 bytes written.
  host     wall time of the host forms (Evaluator.trajectory_states / pose_points: staging, copies both ways, kernel) at the largest sizes.
The card's name, power limit and SM clocks are read in the same run. Writes nothing to the tree.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True      # importing bench.py must leave no __pycache__ behind in a read-only tree

import bench as BM   # noqa: E402

PEAK_HBM = 3.35e12
RECORD_BYTES = 160


def timed(torch, fn, steps, warmup, flush):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for i in range(warmup + steps):
        flush.zero_()
        torch.cuda.synchronize()
        ev0.record()
        fn()
        ev1.record()
        ev1.synchronize()
        if i >= warmup:
            out.append(ev0.elapsed_time(ev1))
    return out


def stats_ms(ts):
    return {"median_ms": round(statistics.median(ts), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4), "n": len(ts)}


def trajectories(B):
    """trajectory 0: bench.py's benchmark trajectory; the others cycle through 32 seeded plans of 2-290 pieces"""
    import workloads as W
    w = dict(BM.WORKLOAD)
    X = w["map_dim"]
    T0, C0, _ = W.make_trajectory(w["pieces"], [0, 0, 0], [X, X, X], seed=11, jitter=0.2)
    rng = np.random.default_rng(21)
    pool = []
    for k in range(32):
        n = int(rng.integers(2, 291))
        T, Cc, _ = W.make_trajectory(n, [0, 0, 0], [X, X, X], seed=100 + k, jitter=0.4)
        pool.append((T, Cc))
    trajs = [(T0, C0)] + [pool[b % 32] for b in range(B - 1)]
    off = np.zeros(B + 1, dtype=np.int32)
    off[1:] = np.cumsum([t.size for t, _ in trajs])
    return off, np.concatenate([t for t, _ in trajs]), np.concatenate([np.asarray(c).reshape(-1) for _, c in trajs]), np.array([t.sum() for t, _ in trajs])


def playback(Q, dur):
    """Q queries split evenly over the trajectories, each trajectory's times increasing over [0, duration)"""
    B = dur.size
    traj = (np.arange(Q, dtype=np.int64) * B // Q).astype(np.int32)
    first = np.searchsorted(traj, np.arange(B))
    cnt = np.diff(np.append(first, Q))
    k = np.arange(Q) - first[traj]
    return traj, k / np.maximum(cnt[traj], 1) * dur[traj]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import isdf_b200 as I
    import workloads as W
    dev = torch.device("cuda:0")
    ev = I.Evaluator(I.default_config_values(), device=0)
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2 (H100)
    d = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)   # noqa: E731
    line = {"bench": "states", "l2": "flushed (512 MiB write) before each call", "states": {}, "pose": {}, "host": {}}
    keep = None
    for B in (128, 1024):
        off, T, Cc, dur = trajectories(B)
        d_off, d_T, d_C = d(off, np.int32), d(T, np.float64), d(Cc, np.float64)
        for Q in (10 ** 4, 10 ** 6, 3 * 10 ** 6):
            traj, times = playback(Q, dur)
            d_tr, d_tm = d(traj, np.int32), d(times, np.float64)
            out = torch.empty((Q, 20), dtype=torch.float64, device=dev)
            fn = lambda: ev.trajectory_states_device(B, d_off.data_ptr(), d_T.data_ptr(), d_C.data_ptr(), Q, d_tr.data_ptr(), d_tm.data_ptr(),   # noqa: E731
                                                     out.data_ptr(), 0)
            ts = timed(torch, fn, args.steps, args.warmup, flush)
            med = statistics.median(ts) * 1e-3
            gbs = RECORD_BYTES * Q / med / 1e9
            line["states"][f"B{B}_Q{Q}"] = dict(stats_ms(ts), mrecords_per_s=round(Q / med / 1e6, 1), gb_per_s_written=round(gbs, 1),
                                                frac_of_3_35_tb_s=round(gbs * 1e9 / PEAK_HBM, 3), pieces=int(off[-1]))
            if B == 1024 and Q == 3 * 10 ** 6:
                t0 = time.perf_counter()
                host = ev.trajectory_states((off, T, Cc), traj, times)
                line["host"][f"states_B{B}_Q{Q}_s"] = round(time.perf_counter() - t0, 4)
                t0 = time.perf_counter()
                ev.trajectory_states((off, T, Cc), traj, times)
                line["host"][f"states_B{B}_Q{Q}_s_again"] = round(time.perf_counter() - t0, 4)
                line["host"]["states_host_equals_device"] = bool(np.array_equal(host, out.cpu().numpy(), equal_nan=True))
                del host
            if B == 128 and Q == 10 ** 4:
                keep = out.clone()
            del out, d_tr, d_tm
    V, _ = W.rounded_cone_mesh()
    V = np.ascontiguousarray(V, dtype=np.float64)
    P = V.shape[0]
    d_V = d(V, np.float64)
    for Q in (10 ** 3, 10 ** 4):
        st = keep[:Q].contiguous()
        out = torch.empty((Q, P, 3), dtype=torch.float64, device=dev)
        fn = lambda: ev.pose_points_device(Q, st.data_ptr(), P, d_V.data_ptr(), out.data_ptr(), 0)   # noqa: E731
        ts = timed(torch, fn, args.steps, args.warmup, flush)
        med = statistics.median(ts) * 1e-3
        gbs = 24.0 * Q * P / med / 1e9
        line["pose"][f"Q{Q}"] = dict(stats_ms(ts), vertices=P, mpoints_per_s=round(Q * P / med / 1e6, 1), gb_per_s_written=round(gbs, 1),
                                     frac_of_3_35_tb_s=round(gbs * 1e9 / PEAK_HBM, 3))
        if Q == 10 ** 4:
            sh = st.cpu().numpy()
            t0 = time.perf_counter()
            host = ev.pose_points(sh, V)
            line["host"][f"pose_Q{Q}_s"] = round(time.perf_counter() - t0, 4)
            t0 = time.perf_counter()
            ev.pose_points(sh, V)
            line["host"][f"pose_Q{Q}_s_again"] = round(time.perf_counter() - t0, 4)
            line["host"]["pose_host_equals_device"] = bool(np.array_equal(host, out.cpu().numpy(), equal_nan=True))
            del host
        del out
    ev.close()
    try:
        line["gpu"] = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                               "--format=csv,noheader"], text=True).strip()
    except Exception:
        line["gpu"] = torch.cuda.get_device_name(0)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
