#!/usr/bin/env python
"""bench_sense.py — depth sensing (isdf_sense_*) on an H100 against the reference's own renderer; prints one JSON line.

  python bench_sense.py [--steps K] [--warmup W] [--poses Q]

Scene: bench_map.py's cloud of the benchmark map (bench.py's 512^3 map, 4 jittered points per occupied voxel: 32.7 M points).
Poses (default camera, horizon 5 m for the clouds):
  traj   Q states (default 1024) of the benchmark trajectory at 30 Hz (isdf_trajectory_states; times wrap at its duration);
  wall   64 bodies at free voxel centres facing an occupied voxel one voxel ahead (+x), where the splats dominate.
Arms, CUDA events after warm-up (medians of K steps):
  depth  isdf_sense_depth_device: all Q images into one device tensor;
  cloud  isdf_sense_cloud_device: the sensed points and offsets;
  ref    the reference's DepthRender::render_pose (oracle/_ref/libref_depth.so), one launch per pose over the whole cloud with its image
         copy to the host, as pcl_render_node runs it (one timed pass).
Only poses whose image gets no centre from a point closer than 0.1 m in front of the camera are used (the reference kernel loops over its
whole unclipped splat once a centre is inside); the line reports how many were dropped. Parity: every image of the batched call is
compared with the reference's (images_differing).
Writes nothing to the tree.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True      # importing bench.py must leave no __pycache__ behind in a read-only tree

import bench as B   # noqa: E402
import bench_map as BM   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--poses", type=int, default=1024)
    args = ap.parse_args()
    import torch
    import isdf_b200 as I
    import sense_oracle as SO
    if not torch.cuda.is_available():
        raise SystemExit("bench_sense.py measures the GPU path and needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    w, cfg, occ, T, Cc, *_ = B.make_workload()
    xyz = BM.make_cloud(occ)
    ev = I.Evaluator(cfg, device=0)
    dev = torch.device("cuda:0")
    d_xyz = torch.from_numpy(xyz).to(dev)
    ev.set_sense_cloud_device(d_xyz, stream=torch.cuda.current_stream().cuda_stream)
    p_depth, p_cloud = I.sense_params(), I.sense_params(sensing_horizon=5.0)
    d_xyz64 = d_xyz.double()

    # poses: the trajectory at 30 Hz, and bodies facing walls
    T = np.asarray(T, dtype=np.float64).reshape(-1)
    dur = float(T.sum())
    times = (np.arange(args.poses) / 30.0) % dur
    st = ev.trajectory_states((np.array([0, T.size], np.int32), T, Cc), np.zeros(args.poses, np.int32), times)
    traj = np.column_stack([st[:, 0:3], st[:, 12:16]])
    occb = occ != 0
    cand = np.argwhere(~occb[:-1] & occb[1:])                      # free voxel with an occupied voxel ahead in +x
    rng = np.random.default_rng(7)
    cand = cand[rng.permutation(len(cand))[:4096]]
    wall = np.column_stack([cand + 0.5, np.tile([1.0, 0, 0, 0], (len(cand), 1))])

    def safe(rec):
        """the records whose image would get no centre from a point less than 0.101 m in front of the camera (the reference kernel
        tests the centre before it loops over the splat, so only such points can make its square large)"""
        keep = []
        for r in rec:
            _, cw = SO.pose(r[:3], r[3:7], np.array(p_depth.cam_to_body[:]))
            Tm = torch.tensor(cw.reshape(4, 4), device=dev)
            c = d_xyz64 @ Tm[:3, :3].T + Tm[:3, 3]
            z = c[:, 2]
            near = (z > 0) & (z < SO.MIN_REF_DEPTH + 1e-3)
            u, v = c[near, 0] / z[near] * p_depth.fx + p_depth.cx, c[near, 1] / z[near] * p_depth.fy + p_depth.cy
            keep.append(not bool(((u > -2) & (u < p_depth.width + 2) & (v > -2) & (v < p_depth.height + 2)).any()))
        return np.array(keep)

    k_traj = safe(traj)
    traj = traj[k_traj]
    k_wall = np.zeros(len(wall), bool)
    for i in range(len(wall)):       # the first 64 safe wall poses
        k_wall[i] = safe(wall[i:i + 1])[0]
        if k_wall.sum() == 64:
            break
    wall = wall[k_wall]
    del d_xyz64

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        ms = []
        for _ in range(args.steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
        return statistics.median(ms), ms

    out = dict(gpu=gpu, points=int(xyz.shape[0]), bricks=ev.sense_info()["bricks"])
    ref = SO._reflib() if SO.ref_available() else None
    h = ref.ref_depth_create(p_depth.fx, p_depth.fy, p_depth.cx, p_depth.cy, p_depth.width, p_depth.height,
                             xyz.ctypes.data_as(SO.fp), xyz.shape[0]) if ref else None
    for name, rec, dropped in (("traj", traj, int((~k_traj).sum())), ("wall", wall, None)):
        if len(rec) == 0:
            out[name] = dict(Q=0)
            continue
        d_rec = torch.from_numpy(np.ascontiguousarray(rec)).to(dev)
        Q = len(rec)
        res = {}
        depth_ms, depth_all = timed(lambda: ev.sense_depth_device(d_rec, params=p_depth))
        cloud_ms, cloud_all = timed(lambda: ev.sense_cloud_device(d_rec, params=p_cloud))
        _, off = ev.sense_cloud_device(d_rec, params=p_cloud)
        img = ev.sense_depth_device(d_rec, params=p_depth).cpu().numpy()
        res.update(Q=Q, depth_ms=round(depth_ms, 2), depth_ms_all=[round(m, 2) for m in depth_all], cloud_ms=round(cloud_ms, 2),
                   cloud_ms_all=[round(m, 2) for m in cloud_all], sensed_points=int(off[-1]))
        if dropped is not None:
            res["dropped_unsafe_poses"] = dropped
        if h:
            import time
            Ts = [SO.pose(r[:3], r[3:7], np.array(p_depth.cam_to_body[:]))[1] for r in rec]
            buf = np.empty((p_depth.height, p_depth.width), np.int32)
            ref.ref_depth_render(h, SO._d(np.ascontiguousarray(Ts[0])), buf.ctypes.data_as(SO.ip))   # warm-up
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            refimg = np.empty_like(img)
            t0 = time.perf_counter()
            a.record()
            for q in range(Q):
                ref.ref_depth_render(h, SO._d(np.ascontiguousarray(Ts[q])), refimg[q].ctypes.data_as(SO.ip))
            b.record()
            torch.cuda.synchronize()
            bad = int(sum(not np.array_equal(refimg[q], img[q]) for q in range(Q)))
            res.update(ref_ms=round(a.elapsed_time(b), 2), ref_wall_ms=round(1e3 * (time.perf_counter() - t0), 2), images_differing=bad,
                       speedup_depth=round(a.elapsed_time(b) / depth_ms, 2))
        out[name] = res
    if h:
        ref.ref_depth_destroy(h)
    print(json.dumps(out))
    ev.close()


if __name__ == "__main__":
    main()
