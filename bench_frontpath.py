#!/usr/bin/env python
"""bench_frontpath.py — the front-end path search (isdf_frontend_path*) on an H100; prints one JSON line.

  python bench_frontpath.py --steps K --warmup W [--small] [--unknown-weight U]

Workload: the 512^3 random voxel map of bench.py (p = 0.05, wall slabs, seed 1) and the Ball robot with kernel_size 5 and 121 attitudes
(+-45 deg at 9 deg). The shipped CappedCone at kernel_size 13 fits nowhere on that map. One far-apart query (a traversable start near the (0, 0, 0) corner,
the goal the voxel of its component with the largest cost-to-come) and one call with B = 64 goals from the same start (that goal and 63
uniform random points, most of them unreachable or blocked). Per call: device time of the traversability build, of the field (relaxation rounds, host
flag reads included) and of the path walk + attitude replay (CUDA events, isdf_frontend_path_info), the wall time of the whole call, the
relaxation rounds and the bytes of the FP64 field. --unknown-weight U marks the half of the map with x < X/2 known (isdf_map_mark_known)
and runs both calls with the surcharge U on unknown voxels (DESIGN §3.23); without it the output is what it always was. Writes nothing to
the tree.
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


def timed(ev, call, steps, warmup):
    rows = []
    for k in range(warmup + steps):
        t0 = time.perf_counter()
        out = call()
        wall = (time.perf_counter() - t0) * 1e3
        info = ev.frontend_path_info()
        if k >= warmup:
            rows.append((wall, info))
    mean = lambda f: statistics.mean(f(r) for r in rows)   # noqa: E731
    return out, {"wall_ms": mean(lambda r: r[0]), "wall_ms_min": min(r[0] for r in rows),
                 "traversability_ms": mean(lambda r: r[1]["traversability_ms"]), "field_ms": mean(lambda r: r[1]["field_ms"]),
                 "paths_ms": mean(lambda r: r[1]["paths_ms"]), "rounds": rows[-1][1]["rounds"], "field_bytes": rows[-1][1]["field_bytes"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--small", action="store_true", help="128^3 map for plumbing checks (not a bench value)")
    ap.add_argument("--unknown-weight", type=float, default=None, help="surcharge on unknown voxels, with the half x < X/2 known")
    args = ap.parse_args()
    import isdf_b200 as I
    import workloads as W
    X = 128 if args.small else 512
    occ = W.random_map(X, X, X, p=0.05, seed=1, slabs=3)
    cfg = I.default_config_values()
    cfg.kernel_size = 5
    ev = I.Evaluator(cfg, device=0)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    xk, yk = ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.dont_write_bytecode = True
    from test_gpu_frontend_path import far_apart_pair   # noqa: E402  (start near a corner, goal = the farthest voxel it reaches)
    src, dst = far_apart_pair(ev, X)
    start, goal = [a + 0.5 for a in src], [a + 0.5 for a in dst]
    uw = args.unknown_weight
    if uw is not None:
        ev.map_mark_known([[0.0, 0.0, 0.0, X / 2, X, X]])
    (p, rp, c, f), one = timed(ev, lambda: ev.frontend_path(start, goal, unknown_weight=uw), args.steps, args.warmup)
    one.update(found=bool(f), cost=float(c), nodes=int(len(p)))
    rng = np.random.default_rng(5)
    goals = np.concatenate([[goal], rng.uniform(0, X, size=(63, 3))])
    res, batch = timed(ev, lambda: ev.frontend_path_batch(start, goals, unknown_weight=uw), args.steps, args.warmup)
    batch.update(found=int(res["found"].sum()), nodes=int(res["offsets"][-1]), goals=64)
    line = {"metric": "frontend_path_ms", "value": one["wall_ms"], "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "higher_is_better": False, "dtype": "f64", "data": "synthetic",
            "config": {"map": f"random {X}^3 (p=0.05, 3 wall slabs, seed 1), res 1.0", "robot": "Ball", "kernel_size": cfg.kernel_size,
                       "attitudes": xk * yk, "start": start, "goal": goal},
            "single": one, "batch64": batch}
    if uw is not None:
        line["config"].update(unknown_weight=uw, known="x < X/2")
    try:
        line["gpu"] = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                                              text=True).strip()
    except Exception:
        line["gpu"] = None
    print(json.dumps(line))
    ev.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
