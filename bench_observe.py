#!/usr/bin/env python
"""bench_observe.py — known space from depth images (isdf_map_observe_device, DESIGN §3.22) alone; prints one JSON line.

  python bench_observe.py [--poses Q] [--horizon H] [--reps R] [--profile]

World: bench_navigate.py's box world (mockamap boxes, seed 511, 40 x 40 x 10 m) as the scene, the reference's 640 x 480 camera with a
horizon of H m (default 15), Q seeded poses (default 768) at x, y in [-18, 18], z in [1, 9] with random yaw and pitch within 0.3 rad. For
each of the 1 m and 0.25 m frames over that box: milliseconds per call (CUDA events around R calls after one warm-up call, each on a
fresh known grid), voxels tested and voxels known. --profile runs one call per frame under torch.profiler instead and reports the
milliseconds of the image stage (k_sense_* and k_obs_mip) and of the voxel stage (k_obs_voxels) separately. The card's name, power limit and
SM clock are read in the same run. Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
sys.dont_write_bytecode = True

BMIN, EXTENT = np.array([-20.0, -20.0, 0.0]), np.array([40.0, 40.0, 10.0])


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                                      text=True).strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception as e:   # the numbers below still stand; say why the card is not named
        return [f"unavailable: {e}"]


def yaw_pitch_quat(yaw, pitch):
    """(w, x, y, z) of R = Rz(yaw) Ry(pitch)"""
    cy, sy, cp, sp = np.cos(yaw / 2), np.sin(yaw / 2), np.cos(pitch / 2), np.sin(pitch / 2)
    return np.array([cy * cp, -sy * sp, cy * sp, sy * cp])


def poses(Q, seed=3):
    rng = np.random.default_rng(seed)
    pos = np.column_stack([rng.uniform(-18, 18, Q), rng.uniform(-18, 18, Q), rng.uniform(1, 9, Q)])
    quat = np.array([yaw_pitch_quat(a, b) for a, b in zip(rng.uniform(-np.pi, np.pi, Q), rng.uniform(-0.3, 0.3, Q))])
    return np.ascontiguousarray(np.column_stack([pos, quat]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=768)
    ap.add_argument("--horizon", type=float, default=15.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    import isdf_b200 as I
    import bench_navigate as BN
    ev = I.Evaluator(I.default_config_values())
    cloud = BN.world(ev)
    ev.set_sense_cloud_device(cloud)
    p = I.sense_params(sensing_horizon=a.horizon)
    rec = torch.from_numpy(poses(a.poses)).cuda()
    out = dict(bench="observe", poses=a.poses, horizon=a.horizon, gpu=gpu_info(), frames={})
    for res in (1.0, 0.25):
        dims = tuple(int(round(e / res)) for e in EXTENT)
        zero = np.zeros(dims, np.uint8)
        ev.set_map_u8(zero, BMIN, res)
        info = ev.map_observe_device(rec, params=p)
        row = dict(dims=dims, voxels_tested=info["voxels_tested"], voxels_known=info["voxels_added"])
        if a.profile:
            from torch.profiler import profile, ProfilerActivity
            ev.set_map_u8(zero, BMIN, res)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ev.map_observe_device(rec, params=p)
                torch.cuda.synchronize()
            img = vox = 0.0
            for e in prof.key_averages():
                t = e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
                if "k_obs_voxels" in e.key:
                    vox += t
                elif "k_sense_" in e.key or "k_obs_mip" in e.key:
                    img += t
            row.update(image_ms=img, voxel_ms=vox)
        else:
            ms = []
            for _ in range(a.reps):
                ev.set_map_u8(zero, BMIN, res)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                ev.map_observe_device(rec, params=p)
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
            row.update(ms=float(np.median(ms)), ms_min=float(np.min(ms)))
        out["frames"][str(res)] = row
    ev.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
