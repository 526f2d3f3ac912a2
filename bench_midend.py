"""Mid-end benchmark: getOriTraj for B plans at once on the device (isdf_midend_batch_device) against the sequential host driver
(host/isdf_midend.hpp) on the same problems.

Workload: B = 1, 64, 1024 plans at N0 = 16 and 64 pieces; every plan's waypoints are selected (isdf_path_waypoints) from a seeded
random walk of one-voxel steps shaped like A* output; default parameters (isdf_midend_default_params). Prints one JSON line per
(B, N0): rounds, iterations (mean, max), the return-code histogram, device ms per call and per round (CUDA events around the call on
its stream), plans/s, and the CPU arm (ms per plan, the same iterates: its results are checked equal to the device's). Writes nothing
to the tree."""
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


def plans(B, N0, seed):
    import isdf_b200 as I
    import midend_cases as M
    paths = [M.astar_like_path(3 * (N0 - 1) + 2, seed + b) for b in range(B)]
    wps, pieces = I.path_waypoints(paths, 1.0)
    assert np.all(pieces == N0)
    heads, tails = np.zeros((B, 3, 3)), np.zeros((B, 3, 3))
    for b, p in enumerate(paths):
        heads[b, :, 0], tails[b, :, 0] = p[0], p[-1]
    return heads, tails, np.array(wps).reshape(B, N0 - 1, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,64,1024")
    ap.add_argument("--pieces", default="16,64")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-plans", type=int, default=16, help="plans timed on the CPU arm per (B, N0)")
    a = ap.parse_args()
    import torch
    import isdf_b200 as I
    import midend_cases as M
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the mid-end benchmark measures the GPU")
    gpu = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"]).decode().strip()
    ev = I.Evaluator(I.default_config_values())
    p = ev.midend_params()
    for N0 in [int(v) for v in a.pieces.split(",")]:
        for B in [int(v) for v in a.batches.split(",")]:
            heads, tails, Q = plans(B, N0, 100 * N0)
            dv = lambda x: torch.tensor(np.ascontiguousarray(x), dtype=torch.float64, device="cuda")
            cm = lambda x: np.ascontiguousarray(np.swapaxes(x, -1, -2)).reshape(-1)
            d_h, d_t, d_q = dv(cm(heads)), dv(cm(tails)), dv(Q.reshape(-1))
            d_x, d_T, d_C, d_f = (torch.zeros(n, dtype=torch.float64, device="cuda") for n in (B * (4 * N0 - 3), B * N0, 18 * B * N0, B))
            d_i = torch.zeros(3 * B, dtype=torch.int32, device="cuda")
            s = torch.cuda.Stream()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ms = []
            for rep in range(a.reps + 1):                        # the first call warms up (allocations, module load)
                with torch.cuda.stream(s):
                    e0.record(s)
                    rounds = ev.midend_batch_device(B, N0, d_h.data_ptr(), d_t.data_ptr(), 1, d_q.data_ptr(), d_x.data_ptr(), d_T.data_ptr(), d_C.data_ptr(),
                                                    d_f.data_ptr(), d_i.data_ptr(), d_i.data_ptr() + 4 * B, d_i.data_ptr() + 8 * B, p, s.cuda_stream)
                    e1.record(s)
                s.synchronize()
                if rep:
                    ms.append(e0.elapsed_time(e1))
            i = d_i.cpu().numpy()
            ret, it, evs = i[:B], i[B:2 * B], i[2 * B:]
            x = d_x.cpu().numpy().reshape(B, -1)
            # CPU arm: the sequential host driver on the first plans, timed per plan; its results must be the device's
            nc = min(B, a.cpu_plans)
            t0 = time.perf_counter()
            host = [M.HostMidEnd(heads[b], tails[b], Q[b], cancel_after=p.cancel_after).optimize(p.init_time) for b in range(nc)]
            cpu_ms = (time.perf_counter() - t0) * 1e3 / nc
            same = all(np.array_equal(h["x"], x[b]) and h["ret"] == ret[b] and h["evaluations"] == evs[b] for b, h in enumerate(host))
            med = float(np.median(ms))
            hist = {int(k): int(v) for k, v in zip(*np.unique(ret, return_counts=True))}
            print(json.dumps(dict(bench="midend", B=B, N0=N0, rounds=rounds, iterations_mean=float(it.mean()), iterations_max=int(it.max()),
                                  ret_hist=hist, device_ms_per_call=med, device_ms_all=ms, device_ms_per_round=med / rounds, plans_per_s=B / (med * 1e-3),
                                  cpu_ms_per_plan=cpu_ms, cpu_plans=nc, cpu_equals_device=bool(same), gpu=gpu)), flush=True)
            if not same:
                raise SystemExit("CPU arm differs from the device")
    ev.close()


if __name__ == "__main__":
    main()
