#!/usr/bin/env python
"""bench_brake.py — time isdf_trajectory_brake_device (Evaluator.trajectory_brake_device, DESIGN §3.21) on remaining trajectories that
a certificate has just found colliding; prints one JSON line.

  python bench_brake.py [--vehicles 16,64,1024] [--reps R] [--seed N]

World and robot: bench_navigate.py's (mockamap's box world, seed 511, in a 40 x 40 x 10 m frame at 1 m; the Ball robot, kernel size 11,
vmax 3 m/s). The remaining trajectories are plan_pairs_device plans between bench_navigate.py's seeded start / goal pairs made in an
EMPTY map of that frame, so many of them run through boxes; the whole world's certificate then cuts them: t_stop_max is first_hit for a
COLLIDING trajectory and +inf otherwise. Brake parameters: brake_params() (8 candidates of 4 pieces, the certificates' defaults).
Per B: milliseconds per call (CUDA events around each call, mean / min over R calls after two warm-up calls), the stops' statuses, and,
from one torch.profiler run of its own, how the call's kernel time splits between setup + MINCO (k_brake_setup, k_minco_forward), the
two certificates, and select + scan + write. Prints the card's name and power limit. Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True


def _group(name):
    if "k_brake_setup" in name or "k_minco_forward" in name:
        return "setup_minco"
    if "k_brake_select" in name or "k_brake_write" in name or "Scan" in name:
        return "select_write"
    return "certificates"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vehicles", default="16,64,1024")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import torch
    import isdf_b200 as I
    import bench_navigate as BN
    if not torch.cuda.is_available():
        raise SystemExit("bench_brake.py measures the GPU path and needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    cfg = I.default_config_values()
    cfg.integral_intervs, cfg.kernel_size, cfg.vmax = 16, 11, 3.0
    st = torch.cuda.current_stream()
    truth = I.Evaluator(cfg)
    truth.set_shape_named("Ball")
    scene = BN.world(truth)
    truth.set_map_u8(np.zeros(BN.DIMS, np.uint8), BN.BMIN, BN.RES)
    truth.map_fuse_cloud_device(scene, stream=st.cuda_stream)
    occ = truth.get_map_u8()
    sizes = [int(v) for v in args.vehicles.split(",")]
    # the remaining trajectories: plans made without knowing the world
    blind = I.Evaluator(cfg)
    blind.set_shape_named("Ball")
    blind.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    blind.set_map_u8(np.zeros(BN.DIMS, np.uint8), BN.BMIN, BN.RES)
    starts, goals = BN.pairs(occ, max(sizes), args.seed)
    pl = blind.plan_pairs_device(torch.as_tensor(starts, device="cuda"), torch.as_tensor(goals, device="cuda"),
                                 params=blind.plan_params(flags=I.PLAN_CERTIFY, backend_max_iterations=200))
    po = pl["piece_off"].cpu().numpy().astype(np.int64)
    n = np.diff(po)
    have = np.nonzero(n > 0)[0]
    blind.close()
    out = dict(bench="brake", gpu=gpu, world="mockamap boxes seed 511, 40 x 40 x 10 m, 20 boxes; 1 m frame", plans=int(have.size), runs=[])
    bp = truth.brake_params()
    out["candidates"], out["pieces"] = int(bp.candidates), int(bp.pieces)
    for B in sizes:
        sel = have[np.arange(B) % have.size]
        counts = n[sel]
        off = np.zeros(B + 1, dtype=np.int64)
        off[1:] = np.cumsum(counts)
        idx = np.concatenate([np.arange(po[b], po[b + 1]) for b in sel])
        T = pl["T"][torch.as_tensor(idx, device="cuda")].contiguous()
        Cc = pl["coeffs"][(18 * torch.as_tensor(idx, device="cuda")[:, None] + torch.arange(18, device="cuda")[None]).reshape(-1)].contiguous()
        d_off = torch.as_tensor(off.astype(np.int32), device="cuda")
        # the world's certificate of each, one call per piece count
        ts = np.full(B, np.inf)
        verdicts = np.zeros(B, dtype=np.int64)
        cp = I.CertifyParams.from_buffer_copy(bytes(bp.certify))
        for N in sorted(set(counts.tolist())):
            grp = np.nonzero(counts == N)[0]
            base = torch.as_tensor(off[grp], device="cuda")
            gT = T[(base[:, None] + torch.arange(N, device="cuda")[None]).reshape(-1)].contiguous()
            gC = Cc[(18 * base[:, None] + torch.arange(18 * N, device="cuda")[None])].reshape(len(grp), 3, 6 * N).permute(1, 0, 2).contiguous()
            summ = torch.empty((len(grp), 56), dtype=torch.uint8, device="cuda")
            cp.clearance.pieces_per_traj = int(N)
            truth.trajectory_certify_device(len(grp) * int(N), gT.data_ptr(), gC.data_ptr(), cp, summ.data_ptr(), st.cuda_stream)
            v = I._field(summ, I.CertifySummary, "verdict").cpu().numpy()
            fh = I._field(summ, I.CertifySummary, "first_hit").cpu().numpy()
            verdicts[grp] = v
            ts[grp] = np.where(v == I.COLLIDING, fh, np.inf)
        d_ts = torch.as_tensor(ts, device="cuda")
        for _ in range(2):
            r = truth.trajectory_brake_device(d_off, T, Cc, d_ts, params=bp)
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            r = truth.trajectory_brake_device(d_off, T, Cc, d_ts, params=bp)
            e1.record(st)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        status = [s["status"] for s in I.decode_brake_summaries(r["summary"])]
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            truth.trajectory_brake_device(d_off, T, Cc, d_ts, params=bp)
            torch.cuda.synchronize()
        split = {"setup_minco": 0.0, "certificates": 0.0, "select_write": 0.0}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0.0)
            if t and e.key and not e.key.startswith("cuda") and "Memcpy" not in e.key and "Memset" not in e.key:
                split[_group(e.key)] += t / 1000.0
        out["runs"].append(dict(trajectories=B, pieces=int(off[-1]), colliding=int((verdicts == I.COLLIDING).sum()),
                                certified=int((verdicts == I.CERTIFIED).sum()), ms_per_call=round(float(np.mean(ms)), 3),
                                ms_min=round(float(np.min(ms)), 3), braked=status.count(I.BRAKED), none=status.count(I.BRAKE_NONE),
                                no_input=status.count(I.BRAKE_NO_INPUT), kernel_ms=({k: round(v, 3) for k, v in split.items()})))
    truth.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
