#!/usr/bin/env python
"""bench_esdf.py — the map's distance field (isdf_map_esdf, isdf_esdf_query_device) on an H100; prints one JSON line.

  python bench_esdf.py --steps K --warmup W [--no-cpu-baseline]

Workload: bench.py's 512^3 map (imported from bench.py, as bench_map.py does), res 1.0.
  build    CUDA events around isdf_map_esdf (both fields), L2 flushed before each call; median and spread over K calls after W warm-up
           calls. GB/s counts 40 bytes per voxel (pass z writes 8; passes y and x each read 8 and write 8), the fraction is of the H100
           SXM data-sheet 3.35 TB/s.
  query    isdf_esdf_query_device with gradient on 1 M and 16 M uniform random points in the map, points already on the device.
  memory   the device bytes the field holds after the build (the drop in free memory, so other work on a shared card moves it) and
           the build's peak from its allocation sizes (the two fields plus the pass y / x stack, include/isdf.h and DESIGN §3.15).
  cpu      the reference-compiled generateESDF3d (oracle/_ref/libref_esdf.so) on a 256 x 256 x 128 map, one run, with a bit-for-bit
           check of isdf_map_esdf against it; skipped when that library is absent.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True      # importing bench.py must leave no __pycache__ behind in a read-only tree

import bench as B   # noqa: E402

PEAK_HBM = 3.35e12
BYTES_PER_VOXEL = 40


def timed(torch, fn, steps, warmup, flush=None):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for i in range(warmup + steps):
        if flush is not None:
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    args = ap.parse_args()
    import torch
    import isdf_b200 as I
    dev = torch.device("cuda:0")
    w, _, occ, *_ = B.make_workload()
    X, Y, Z = occ.shape
    nvox = X * Y * Z
    ev = I.Evaluator(I.default_config_values(), device=0)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    ev.map_esdf()
    held = free0 - torch.cuda.mem_get_info(0)[0]
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2 (H100)
    bt = timed(torch, ev.map_esdf, args.steps, args.warmup, flush)
    med = statistics.median(bt) * 1e-3
    gbs = BYTES_PER_VOXEL * nvox / med / 1e9
    props = torch.cuda.get_device_properties(0)
    resident = props.multi_processor_count * 2048          # k_esdf_line: 32 registers, 8 CTAs of 256 per SM
    stack = max(min(X * Z, resident) * Y, min(Y * Z, resident) * X) * 8
    line = {"bench": "esdf", "map": [X, Y, Z], "occupancy": w["occupancy"],
            "build": dict(stats_ms(bt), gb_per_s=round(gbs, 1), frac_of_3_35_tb_s=round(gbs * 1e9 / PEAK_HBM, 3), bytes_per_voxel_model=BYTES_PER_VOXEL),
            "l2": "flushed (512 MiB write) before each build",
            "memory": {"held_after_build_bytes": int(held), "held_bytes_per_voxel": round(held / nvox, 3),
                       "peak_during_build_bytes": int(8 * nvox + stack), "peak_bytes_per_voxel": round((8 * nvox + stack) / nvox, 3)}}
    del flush
    rng = np.random.default_rng(4)
    line["query"] = {}
    for n in (1 << 20, 1 << 24):
        pts = torch.as_tensor(rng.random((n, 3)) * np.array([X, Y, Z]), device=dev)
        dist = torch.empty(n, dtype=torch.float64, device=dev)
        grad = torch.empty((n, 3), dtype=torch.float64, device=dev)
        fn = lambda: ev.lib.isdf_esdf_query_device(ev.h, 0, pts.data_ptr(), n, dist.data_ptr(), grad.data_ptr(), None)
        qt = timed(torch, fn, args.steps, args.warmup)
        line["query"][str(n)] = dict(stats_ms(qt), mpoints_per_s=round(n / (statistics.median(qt) * 1e-3) / 1e6, 1))
        del pts, dist, grad
    ev.close()
    if not args.no_cpu_baseline:
        import esdf_oracle as E
        if E.ref_available():
            small = (np.random.default_rng(3).random((256, 256, 128)) < 0.05).astype(np.uint8)
            t0 = time.perf_counter()
            pos, neg, _ = E.ref_esdf(small, [0, 0, 0], 0.125)
            cpu_s = time.perf_counter() - t0
            ev = I.Evaluator(I.default_config_values(), device=0)
            ev.set_map_u8(small, [0, 0, 0], 0.125)
            ev.map_esdf()
            ok = bool(np.array_equal(ev.get_esdf("positive"), pos) and np.array_equal(ev.get_esdf("negative"), neg))
            gt = timed(torch, ev.map_esdf, max(3, args.steps // 4), 1)
            ev.close()
            line["cpu"] = {"map": [256, 256, 128], "reference_generateESDF3d_s": round(cpu_s, 3), "gpu_median_ms": round(statistics.median(gt), 4),
                           "bit_identical": ok}
        else:
            line["cpu"] = "skipped: oracle/_ref/libref_esdf.so absent"
    try:
        line["gpu"] = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        line["gpu"] = torch.cuda.get_device_name(0)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
