#!/usr/bin/env python
"""bench_frontier.py — frontier extraction (isdf_map_frontiers) and frontier-goal selection (isdf_frontier_goals) on an H100; prints one
JSON line.

  python bench_frontier.py --steps K --warmup W [--small] [--profile DIR]

Workloads:
  navigate  bench_navigate.py's box world (mockamap boxes, seed 511) in its 40 x 40 x 10 frame at 1 m, Ball robot, kernel size 11: the
            scene fused into the map, then observed from 64 seeded poses of the reference camera (horizon 15 m), so that the known space is
            what depth images prove; goals: 16 pairs of bench_navigate.py's seeded start / goal sets.
  half512   bench_frontpath.py's 512^3 random map (p = 0.05, 3 wall slabs, seed 1), Ball robot at kernel size 5, with the half x < 256 marked
            known (isdf_map_mark_known); goals: bench_frontpath.py's start near the (0, 0, 0) corner to 16 seeded goals in the unknown half.
Per workload: the device time of the stages (CUDA events, isdf_frontier_info: both feasibility passes, F and its list, labelling and the
cluster table, the fields over T_b and the selection), the wall time of each call, |T_b|, |F| and the cluster count. --profile DIR writes a
torch.profiler trace of one extraction and one goal call per workload under DIR, with the per-kernel device time split, in a run of its own.
Writes nothing to the tree.
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
sys.dont_write_bytecode = True


def timed(call, steps, warmup):
    rows = []
    for k in range(warmup + steps):
        t0 = time.perf_counter()
        info = call()
        wall = (time.perf_counter() - t0) * 1e3
        if k >= warmup:
            rows.append((wall, info))
    keys = ("traversability_ms", "frontier_ms", "cluster_ms", "field_ms", "select_ms")
    out = {"wall_ms": round(statistics.mean(r[0] for r in rows), 3), "wall_ms_min": round(min(r[0] for r in rows), 3)}
    out.update({k: round(statistics.mean(r[1][k] for r in rows), 3) for k in keys})
    out.update({k: rows[-1][1][k] for k in ("traversable_blocked", "frontier_voxels", "clusters")})
    return out


def navigate_world():
    import torch
    import isdf_b200 as I
    import bench_navigate as BN
    cfg = I.default_config_values()
    cfg.integral_intervs, cfg.kernel_size, cfg.vmax = 16, 11, 3.0
    ev = I.Evaluator(cfg)
    ev.set_shape_named("Ball")
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    scene = BN.world(ev)
    ev.set_map_u8(np.zeros(BN.DIMS, np.uint8), BN.BMIN, BN.RES)
    ev.map_fuse_cloud_device(scene, stream=torch.cuda.current_stream().cuda_stream)
    occ = ev.get_map_u8()
    starts, goals = BN.pairs(occ, 16, 23)
    rng = np.random.default_rng(3)
    pos = np.concatenate([starts, BN.pairs(occ, 48, 31)[0]]) + rng.uniform(-0.4, 0.4, (64, 3))
    yaw = rng.uniform(0, 2 * np.pi, 64)
    rec = np.zeros((64, 7))
    rec[:, :3] = pos
    rec[:, 3], rec[:, 6] = np.cos(yaw / 2), np.sin(yaw / 2)
    ev.set_sense_cloud_device(scene, stream=torch.cuda.current_stream().cuda_stream)
    ev.map_observe(rec, params=I.sense_params(sensing_horizon=15.0))
    return ev, starts, goals, "mockamap boxes seed 511, 40 x 40 x 10 frame at 1 m, 64 observed poses"


def half512(X):
    import isdf_b200 as I
    import workloads as W
    occ = W.random_map(X, X, X, p=0.05, seed=1, slabs=3)
    cfg = I.default_config_values()
    cfg.kernel_size = 5
    ev = I.Evaluator(cfg, device=0)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_frontend_path import far_apart_pair   # noqa: E402  (bench_frontpath.py's start: near the corner, in a large component)
    start = np.array(far_apart_pair(ev, X)[0]) + 0.5
    ev.map_mark_known([[0.0, 0.0, 0.0, X / 2, X, X]])
    rng = np.random.default_rng(5)
    goals = np.column_stack([rng.uniform(X / 2 + 1, X, 16), rng.uniform(0, X, 16), rng.uniform(0, X, 16)])
    return ev, np.repeat([start], 16, 0), goals, f"random {X}^3 (p=0.05, 3 wall slabs, seed 1), half x < {X // 2} known"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--small", action="store_true", help="128^3 instead of 512^3 for the second workload (plumbing checks, not a bench value)")
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_frontier.py measures the GPU path and needs a CUDA device")
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = dict(bench="frontier", gpu=gpu, steps=args.steps, warmup=args.warmup, workloads={})
    for name, make in (("navigate", navigate_world), ("half512", lambda: half512(128 if args.small else 512))):
        ev, starts, goals, desc = make()
        extract = timed(lambda: ev.map_frontiers()["info"], args.steps, args.warmup)
        recs = [None]

        def goals_call():
            recs[0], info = ev.frontier_goals(starts, goals)
            return info
        select = timed(goals_call, args.steps, args.warmup)
        kinds = np.bincount(recs[0]["kind"], minlength=3)
        out["workloads"][name] = dict(map=desc, dims=list(ev.map_info()["dims"]), pairs=len(starts), extract=extract, goals=select,
                                      kinds=dict(none=int(kinds[0]), goal=int(kinds[1]), frontier=int(kinds[2])))
        if args.profile:
            from torch.profiler import profile, ProfilerActivity
            os.makedirs(args.profile, exist_ok=True)
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                ev.map_frontiers()
                ev.frontier_goals(starts, goals)
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(args.profile, f"frontier_{name}.pt.trace.json"))
            split = {}
            for e in prof.key_averages():
                if getattr(e, "self_device_time_total", 0) > 0:   # kernels and copies
                    split[e.key[:60]] = round(e.self_device_time_total / 1e3, 3)
            out["workloads"][name]["kernel_ms"] = dict(sorted(split.items(), key=lambda kv: -kv[1])[:16])
        ev.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
