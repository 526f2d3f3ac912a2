#!/usr/bin/env python
"""bench_swept_volume.py — the certified swept volume (isdf_swept_volume_grid_device / isdf_swept_volume_mesh) on one GPU; prints one
JSON line.

  python bench_swept_volume.py --steps K --warmup W [--pieces P]

Workload: the first P pieces (default 4) of bench.py's 64-piece trajectory (imported from bench.py, so both use the same inputs; the
whole 512 m trajectory would need a grid of ~10^9 nodes at these resolutions), the 3900-triangle mesh robot in exact-sign mode and the
Ball, at res = occupancy_resolution / 2 and / 4 on the grid sized by isdf_b200.swept_grid_for (bounding box inflated by
r_body + band + res), default parameters. Per case: device ms of the field (one grid_device call, CUDA events) and of the mesh stage,
node count, culled brick share, SDF evaluations per node of a surviving brick, undecided nodes, triangle count. The card's name and power
limit are read in the same run. Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True      # importing bench.py must leave no __pycache__ behind in a read-only tree

import bench as B   # noqa: E402
import workloads as W   # noqa: E402


def case(ev, T, Cc, r_body, res, steps, warmup):
    import torch
    p = ev.swept_params()
    g = __import__("isdf_b200").swept_grid_for(T, Cc, r_body, p.band, res)
    n = g.X * g.Y * g.Z
    dT, dC = torch.from_numpy(np.ascontiguousarray(T)).cuda(), torch.from_numpy(np.ascontiguousarray(Cc)).cuda()
    dv = torch.empty(n, dtype=torch.float64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    times, info = [], None
    for k in range(warmup + steps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        info = ev.swept_volume_grid_device(len(T), dT.data_ptr(), dC.data_ptr(), g, p, dv.data_ptr(), stream=stream, info=(k == warmup + steps - 1))
        e1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            times.append(e0.elapsed_time(e1))
    V, vt, F, minfo = ev.swept_volume_mesh(T, Cc, g, p)
    surv = max(info["bricks"] - info["bricks_culled"], 1)
    return {"res": res, "grid": [g.X, g.Y, g.Z], "nodes": n, "field_ms": statistics.mean(times), "field_ms_min": min(times),
            "field_stage_ms": {k: info[k] for k in ("prep_ms", "cull_ms", "refine_ms")}, "mesh_ms": minfo["mesh_ms"],
            "bricks": info["bricks"], "culled_brick_share": info["bricks_culled"] / max(info["bricks"], 1),
            "sdf_evals": info["sdf_evals"], "sdf_evals_per_surviving_node": info["sdf_evals"] / (64.0 * surv),
            "undecided_nodes": info["undecided"], "deepest": info["deepest"], "vertices": int(len(V)), "triangles": int(len(F))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--pieces", type=int, default=4)
    args = ap.parse_args()
    import isdf_b200 as I
    w, cfg, occ, T, Cc, V, F = B.make_workload(False)
    N = args.pieces
    T, Cc = np.asarray(T)[:N].copy(), np.asarray(Cc).reshape(3, -1)[:, :6 * N].reshape(-1).copy()
    ev = I.Evaluator(cfg, device=0)
    R, t = W.rotation_from_poly_params(w["poly_params"])
    Vb = np.asarray(V) @ R.T + t
    r_mesh = float(np.linalg.norm(np.maximum(np.abs(Vb.min(0)), np.abs(Vb.max(0)))))
    line = {"metric": "swept_volume_field_ms", "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "higher_is_better": False,
            "dtype": "f64", "data": "synthetic",
            "config": {"workload": B.workload_name(w) + f"; first {N} pieces", "K": cfg.integral_intervs, "params": "isdf_swept_default_params"}}
    cases = {}
    ev.set_shape_mesh(V, F, w["poly_params"], I.MESH_SIGN_EXACT)
    for div in (2, 4):
        cases[f"mesh_res_1/{div}"] = case(ev, T, Cc, r_mesh, cfg.occupancy_resolution / div, args.steps, args.warmup)
    ev.set_shape_named("Ball")
    for div in (2, 4):
        cases[f"ball_res_1/{div}"] = case(ev, T, Cc, 1.0, cfg.occupancy_resolution / div, args.steps, args.warmup)
    line["value"] = cases["mesh_res_1/2"]["field_ms"]
    line["cases"] = cases
    try:
        line["gpu"] = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        line["gpu"] = None
    print(json.dumps(line))
    ev.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
