#!/usr/bin/env python
"""bench_view.py — the view gain (isdf_view_gain) and frontier goals that need something left to see (isdf_frontier_goals_view) on an H100;
prints one JSON line.

  python bench_view.py --steps K --warmup W [--small] [--profile DIR]

Workloads (bench_frontier.py's maps):
  navigate  bench_navigate.py's box world in its 40 x 40 x 10 frame at 1 m, observed from 64 seeded poses (horizon 15 m). View gain for
            B = 16 and 64 vehicles x 4 sensed records each, with navigate's rigs (bench_navigate.py: the reference camera, horizon 15 m, and
            four of them at yaw 0, 90, 180, 270 deg), poses at the vehicles' seeded starts, tilted by up to 0.3 rad.
  half512   the 512^3 random map with the half x < 256 known: 256 poses near the boundary x = 256, level, seeded yaw, one camera.
Frontier goals: bench_frontier.py's pairs on both maps through isdf_frontier_goals and through isdf_frontier_goals_view with one camera
and with four (min_gain 0, so that the three select alike and the difference is the gains' cost).
Per call: the mean and minimum wall time of a host call (which returns when the result is on the host). --profile DIR: in a run of its
own, a torch.profiler trace per workload under DIR, and the device time of each kernel, so that k_view_gain's share of a call shows.
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
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True


def timed(call, steps, warmup):
    ms = []
    for k in range(warmup + steps):
        t0 = time.perf_counter()
        call()
        if k >= warmup:
            ms.append((time.perf_counter() - t0) * 1e3)
    return dict(wall_ms=round(statistics.mean(ms), 3), wall_ms_min=round(min(ms), 3))


def poses(centres, n, seed, tilt):
    """n poses per centre: jittered positions, seeded yaw, roll and pitch up to tilt rad -> (len(centres) n, 7) records"""
    rng = np.random.default_rng(seed)
    c = np.repeat(np.asarray(centres, dtype=np.float64), n, 0)
    yaw, roll, pitch = rng.uniform(-np.pi, np.pi, len(c)), rng.uniform(-tilt, tilt, len(c)), rng.uniform(-tilt, tilt, len(c))
    cy, sy, cr, sr, cp, sp = np.cos(yaw / 2), np.sin(yaw / 2), np.cos(roll / 2), np.sin(roll / 2), np.cos(pitch / 2), np.sin(pitch / 2)
    q = np.column_stack([cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy])
    return np.column_stack([c + rng.uniform(-0.4, 0.4, c.shape), q])


def profile_split(prof):
    split = {}
    for e in prof.key_averages():
        if getattr(e, "self_device_time_total", 0) > 0:   # kernels and copies
            split[e.key[:60]] = round(e.self_device_time_total / 1e3, 3)
    return dict(sorted(split.items(), key=lambda kv: -kv[1])[:12])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--small", action="store_true", help="128^3 instead of 512^3 for the second workload (plumbing checks, not a bench value)")
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_view.py measures the GPU path and needs a CUDA device")
    import bench_frontier as BF
    import bench_navigate as BN
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = dict(bench="view", gpu=gpu, steps=args.steps, warmup=args.warmup, workloads={})
    rigs = {1: [BN.rig(1)], 4: BN.rig(4)}
    for name, make in (("navigate", BF.navigate_world), ("half512", lambda: BF.half512(128 if args.small else 512))):
        ev, starts, goals, desc = make()
        X = ev.map_info()["dims"][0]
        w = dict(map=desc, dims=list(ev.map_info()["dims"]), known_voxels=int(ev.get_map_known_u8().sum()), view_gain=[], frontier_goals={})
        if name == "navigate":
            cases = [(B, k, poses(BN.pairs(ev.get_map_u8(), B, 7 + B)[0], 4, B, 0.3)) for B in (16, 64) for k in (1, 4)]
        else:
            rng = np.random.default_rng(4)
            centres = np.column_stack([rng.uniform(X / 2 - 8, X / 2 - 1, 256), rng.uniform(8, X - 8, 256), rng.uniform(8, X - 8, 256)])
            cases = [(None, 1, poses(centres, 1, 5, 0.0))]
        for B, k, rec in cases:
            gains = ev.view_gain(rec, params=rigs[k])
            row = dict(poses=len(rec), cameras=k, pose_camera_pairs=len(rec) * k, mean_gain=round(float(gains.mean()), 1),
                       **timed(lambda: ev.view_gain(rec, params=rigs[k]), args.steps, args.warmup))
            if B is not None:
                row["vehicles"] = B
            w["view_gain"].append(row)
        recs = {}
        for label, kw in (("plain", {}), ("view_1cam", dict(cams=rigs[1])), ("view_4cam", dict(cams=rigs[4]))):
            def call():
                recs[label], info = ev.frontier_goals(starts, goals, **kw)
                return info
            w["frontier_goals"][label] = timed(call, args.steps, args.warmup)
        same = True
        for label in ("view_1cam", "view_4cam"):   # min_gain 0: the same records but for the gain field
            r = recs[label].copy()
            r["gain"] = 0
            same &= bool(np.array_equal(r.view(np.uint8), recs["plain"].view(np.uint8)))
        w["frontier_goals"]["same_records"] = same
        w["frontier_goals"]["pairs"] = len(starts)
        w["frontier_goals"]["frontier_voxels"] = int(ev.map_frontiers()["info"]["frontier_voxels"])
        if args.profile:
            from torch.profiler import profile, ProfilerActivity
            os.makedirs(args.profile, exist_ok=True)
            rec = cases[-1][2]
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                ev.view_gain(rec, params=rigs[cases[-1][1]])
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(args.profile, f"view_gain_{name}.pt.trace.json"))
            w["view_gain"][-1]["kernel_ms"] = profile_split(prof)
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                ev.frontier_goals(starts, goals, cams=rigs[4])
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(args.profile, f"frontier_goals_view_{name}.pt.trace.json"))
            w["frontier_goals"]["view_4cam"]["kernel_ms"] = profile_split(prof)
        out["workloads"][name] = w
        ev.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
