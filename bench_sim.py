"""Closed-loop rollouts (isdf_simulate_device) of a 64-piece trajectory: device time, rollout-steps per second, the spread of dopri5
tries per simulation step, the serial restatement (tests/sim_serial.cpp) on one core for the speed-up, and the whole-body clearance of
the logged poses (isdf_pose_clearance_device, bench mesh robot, 64 x 64 x 48 random map at 1 m).
    python bench_sim.py [--R 1 128 1024 8192] [--t_end 10] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time
import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import isdf_b200 as I   # noqa: E402
import workloads as W   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--R", type=int, nargs="+", default=[1, 128, 1024, 8192])
    ap.add_argument("--t_end", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import sim_oracle as S
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    T, Cc, _ = W.make_trajectory(64, [0, 0, 0], [50, 50, 34], seed=3, jitter=0.3)
    off = np.array([0, 64], dtype=np.int32)
    T, Cc = np.asarray(T, dtype=np.float64), np.asarray(Cc, dtype=np.float64).reshape(-1)
    p = I.sim_default_params(floor=0, t_end=a.t_end, log_every=10, diverge_dist=1e3)
    ev = I.Evaluator(device=0)
    dv = torch.device("cuda:0")
    d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dv)
    occ = W.random_map(64, 64, 48, p=0.05, seed=1, slabs=0)
    ev.set_map_u8(occ, [-7.0, -7.0, -7.0], 1.0)
    V, F = W.rounded_cone_mesh()
    ev.set_shape_mesh(V, F, [0.0, 0.0, 0.0, 120.0, 0.0, 0.0])
    pc = ev.pose_clearance_params(2.0, 0.866)

    def inputs(R, seed):
        rng = np.random.default_rng(seed)
        traj = np.zeros(R, dtype=np.int32)
        init = I.sim_init_from_trajectories(off, Cc, traj)
        init[:, :3] += rng.normal(scale=0.1, size=(R, 3))
        dist = np.zeros((R, 6))
        dist[:, :3] = rng.normal(scale=0.3, size=(R, 3))
        return traj, init, dist

    # serial restatement on one core: the same kind of perturbed rollouts as the device arm, best of reps per rollout, 4 rollouts
    tr4, in4, di4 = inputs(4, 99)
    serial = []
    for r in range(4):
        best = 1e30
        for _ in range(a.reps):
            t0 = time.perf_counter()
            S.simulate(off, T, Cc, tr4[r:r + 1], in4[r:r + 1], di4[r:r + 1], p)
            best = min(best, time.perf_counter() - t0)
        serial.append(best)
    serial_s = float(np.mean(serial))
    steps = int(round(a.t_end * p.sim_rate))
    for R in a.R:
        traj, init, dist = inputs(R, R)
        args = [d(off), d(T), d(Cc), d(traj), d(init), d(dist)]
        ev.simulate_device(*args, params=p)   # warm-up
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = ev.simulate_device(*args, params=p)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        s = I.decode_sim_summaries(out["summary"])
        acc = np.array([x["accepted"] for x in s], dtype=np.float64) / steps
        rej = np.array([x["rejected"] for x in s], dtype=np.float64) / steps
        best = min(ms)
        # whole-body clearance of every logged pose, read in place from the log (pos at 1, quat at 7, 21 doubles per record)
        lg = out["log"]
        Q = lg.shape[0] * lg.shape[1]
        dc, dvx = torch.empty(Q, dtype=torch.float64, device=dv), torch.empty(Q, dtype=torch.int64, device=dv)
        dsm = torch.empty((1, 48), dtype=torch.uint8, device=dv)
        base = lg.data_ptr()
        pose = lambda: ev.pose_clearance_device(Q, base + 8, base + 56, I.SIM_DOUBLES, pc, dc.data_ptr(), dvx.data_ptr(), dsm.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream)
        pose()
        torch.cuda.synchronize()
        pms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); pose(); e1.record()
            torch.cuda.synchronize()
            pms.append(e0.elapsed_time(e1))
        print(json.dumps(dict(gpu=gpu, R=R, sim_seconds=a.t_end, steps_per_rollout=steps, device_ms=[round(m, 2) for m in ms],
                              rollout_steps_per_s=R * steps / (best / 1e3), accepted_per_step_mean=acc.mean(), accepted_per_step_max=acc.max(),
                              rejected_per_step_mean=rej.mean(), rejected_per_step_max=rej.max(), diverged=int(sum(x["diverged"] for x in s)),
                              serial_ms_per_rollout=serial_s * 1e3, speedup_vs_serial=R * serial_s * 1e3 / best,
                              pose_clearance_poses=Q, pose_clearance_ms=[round(m, 3) for m in pms],
                              poses_per_s=Q / (min(pms) / 1e3))), flush=True)
    ev.close()


if __name__ == "__main__":
    main()
