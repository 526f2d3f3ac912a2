#!/usr/bin/env python
"""bench_map.py — the occupancy grid from a point cloud (isdf_set_map_cloud*) on an H100; prints one JSON line.

  python bench_map.py --steps K --warmup W [--no-cpu-baseline]

Workload: bench.py's BASELINE configs[2] map (512^3, imported from bench.py so both measure the same occupancy) turned into a cloud: k = 4
float32 points jittered inside every occupied voxel, in voxel order, plus the two corners (0, 0, 0) and (512, 512, 512) that fix the frame
(the top corner lands in the top layer through getGridIndex's clamp). Records of stride 12 (packed xyz) and 16 (pcl::PointXYZ).
  device   isdf_set_map_cloud_device with the points already on the device, CUDA events around the call, L2 flushed before each call;
           sta_threshold 1 (the bit-setting path) and 3 (the counting path) at stride 12, and 1 at stride 16;
  host     isdf_set_map_cloud from pageable host memory, end to end (H2D copy included), host clock;
  cpu      the serial loop of the reference's handler (tests/cloud_map_serial.cpp on the oracle's grid), one run per threshold.
GB/s counts n * stride bytes of records read plus the X*Y*ceil(Z/32) words of the bit grid written, over the device time; the fraction
is of the H100 SXM data-sheet 3.35 TB/s. Parity: the grid read back with isdf_get_map_u8 against the CPU arm, bit for bit.
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
K_PER_VOXEL = 4


def make_cloud(occ, seed=3):
    rng = np.random.default_rng(seed)
    idx = np.argwhere(occ).astype(np.float32)
    pts = np.repeat(idx, K_PER_VOXEL, axis=0)
    pts += rng.uniform(0.02, 0.98, size=pts.shape).astype(np.float32)          # res 1.0, bmin 0: voxel (i, j, k) is [i, i+1) x ...
    X = occ.shape[0]
    return np.concatenate([pts, np.array([[0, 0, 0], [X, X, X]], dtype=np.float32)])


def with_stride(pts, stride):
    rec = np.zeros((pts.shape[0], stride // 4), dtype=np.float32)
    rec[:, :3] = pts
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    args = ap.parse_args()
    import torch
    import isdf_b200 as I
    if not torch.cuda.is_available():
        raise SystemExit("bench_map.py measures the GPU path and needs a CUDA device")
    w, cfg, occ, *_ = B.make_workload()
    pts12 = make_cloud(occ)
    n = pts12.shape[0]
    dev = torch.device("cuda:0")
    ev = I.Evaluator(cfg, device=0)
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2 (H100)
    stream = torch.cuda.current_stream()

    def device_ms(d_pts, stride, thr):
        for _ in range(args.warmup):
            ev.set_map_cloud_device(d_pts.data_ptr(), n=n, stride_bytes=stride, res=1.0, sta_threshold=thr, stream=stream.cuda_stream)
        times = []
        for _ in range(args.steps):
            flush.zero_()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ev.set_map_cloud_device(d_pts.data_ptr(), n=n, stride_bytes=stride, res=1.0, sta_threshold=thr, stream=stream.cuda_stream)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        return statistics.median(times), min(times)

    info = None
    results, grids = {}, {}
    for stride, thr in ((12, 1), (12, 3), (16, 1)):
        host = pts12 if stride == 12 else with_stride(pts12, stride)
        d_pts = torch.from_numpy(host).to(dev)
        med, best = device_ms(d_pts, stride, thr)
        del d_pts
        info = ev.map_info()
        X, Y, Z = info["dims"]
        nbytes = n * stride + X * Y * ((Z + 31) // 32) * 4
        grids[(stride, thr)] = ev.get_map_u8()
        results[f"device_stride{stride}_thr{thr}"] = {"ms_median": round(med, 3), "ms_min": round(best, 3),
                                                      "GB_per_s": round(nbytes / (med * 1e-3) / 1e9, 1),
                                                      "fraction_of_3.35TB_s": round(nbytes / (med * 1e-3) / PEAK_HBM, 3)}
    # host entry end to end (pageable host records, H2D copy included)
    ht = []
    for k in range(max(2, min(args.steps, 5)) + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev.set_map_cloud(pts12, 1.0, 1)
        ht.append((time.perf_counter() - t0) * 1e3)
    host_ms = statistics.median(ht[1:])
    same_entry = bool(np.array_equal(ev.get_map_u8(), grids[(12, 1)]))
    line = {"metric": "point cloud -> occupancy grid (isdf_set_map_cloud*)",
            "config": {"workload": B.workload_name(w) + f"; cloud: {K_PER_VOXEL} jittered float32 points per occupied voxel + 2 corners, res 1.0",
                       "points": n, "occupied_voxels": int(info["occupied_voxels"]), "dims": info["dims"], "l2": "flushed (512 MiB write) before each call",
                       "steps": args.steps, "warmup": args.warmup},
            **results, "host_stride12_thr1_ms": round(host_ms, 2), "host_equals_device": same_entry,
            "stride16_equals_stride12": bool(np.array_equal(grids[(16, 1)], grids[(12, 1)]))}
    if not args.no_cpu_baseline:
        import cloud_oracle as CO
        for thr in (1, 3):
            t0 = time.perf_counter()
            r = CO.serial(pts12, 12, 1.0, thr)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            line[f"cpu_serial_thr{thr}_ms"] = round(cpu_ms, 1)
            line[f"speedup_device_vs_cpu_thr{thr}"] = round(cpu_ms / results[f"device_stride12_thr{thr}"]["ms_median"], 1)
            line[f"parity_thr{thr}_bits_identical"] = bool(r["dims"] == info["dims"] and np.array_equal(r["occ"], grids[(12, thr)]))
    try:
        line["gpu"] = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        line["gpu"] = torch.cuda.get_device_name(0)
    ev.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
