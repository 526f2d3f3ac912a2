#!/usr/bin/env python
"""bench_navigate.py — B vehicles fly to goals through a generated world they only see through the reference's depth camera
(Evaluator.navigate: sense -> fuse -> check -> replan -> fly -> advance, every stage batched over vehicles); prints one JSON line.

  python bench_navigate.py [--vehicles 1,16,64] [--rounds R] [--horizon H] [--sense-every S] [--seed N] [--fallback keep|brake]
                           [--unknown free|occupied] [--cameras 1|4] [--prefer-known W] [--explore] [--min-gain G]

World: mockamap's box world (isdf_world_cloud_device, ISDF_WORLD_BOXES) with seed 511, 40 x 40 x 10 m at 0.5 m (size 80 x 80 x 20,
scale 2), 20 boxes 1.5 to 3 m wide: x and y in [-20, 20] m, z in [0, 10] m. The vehicles' map starts as an empty 1 m frame over that box
(set_map_u8 of zeros) and grows only by fusing what the camera (the reference's 640 x 480 camera, horizon 15 m) sees. Robot: the Ball
shape (radius 1 m), kernel size 11 at 1 m, vmax 3 m/s; planning with PLAN_CERTIFY and 200 back-end iterations; flight with the reference's
simulator for `horizon` seconds per round.
Start / goal pairs are seeded: starts at x in [-17, -12], goals at x in [12, 17], y in [-17, 17], z in [2, 8], all in voxels of the true
map at least 2 voxels from any occupied one. The true map (the whole world fused into the same frame, in a second context) checks every
flown pose with pose_clearance_device.
Per B: per-stage milliseconds per round (mean over the rounds run, CUDA events), rounds run, arrivals, failed replans, and the minimum true
clearance over every flown pose. --fallback brake (navigate's fallback, DESIGN §3.21) adds the stops taken and the rounds held; the
default, keep, prints what it always printed. --unknown occupied (navigate's unknown policy, DESIGN §3.22; needs --fallback brake) seeds
the known space with the 5 x 5 x 5-voxel block around each start (free in the true map by pairs()) and adds the commits taken; --cameras 4
flies a rig of four cameras, cam_to_body = Rz(k 90 deg) cam02body. --prefer-known W plans through what has been seen (DESIGN §3.23):
the front end's surcharge unknown_weight = W on unknown voxels and ISDF_PLAN_KNOWN_PREFIX, so that the back end treats unseen space as
an obstacle along each plan's known prefix. --explore (needs --unknown occupied) flies navigate(explore=True) (DESIGN §3.24): a vehicle
whose goal cannot be reached through seen space plans to the best frontier of what has been seen; it adds the frontier plans taken, and the
frontier-goal call is timed inside the replan stage. --min-gain G (needs --explore) makes that call the view form (DESIGN §3.25): a frontier
is a candidate only when navigate's rig, level at its cube centre, would see at least G unknown voxels; it adds the gains of the frontiers
chosen (a histogram) and, for the vehicles that end held, the gain of the last frontier each was sent to. Either option (also --unknown free) also reports the pose of the minimum true clearance: its
vehicle, round and witness voxel, and whether that voxel is occupied in the vehicles' fused map at the end of the run. Writes nothing to the
tree.
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

DIMS, BMIN, RES = (40, 40, 10), np.array([-20.0, -20.0, 0.0]), 1.0


def world(ev):
    import isdf_b200 as I
    p = I.world_params("boxes", seed=511, size=[80, 80, 20], scale=2.0, obstacle_number=20, width_min=1.5, width_max=3.0)
    return ev.world_cloud_device(p)


def pairs(occ, B, seed):
    """B seeded (start, goal) pairs at voxel centres of the true map at least 2 voxels from any occupied voxel"""
    pad = np.pad(occ, 2)
    near = np.zeros_like(occ, dtype=bool)
    X, Y, Z = occ.shape
    for i in range(5):
        for j in range(5):
            for k in range(5):
                near |= pad[i:i + X, j:j + Y, k:k + Z] > 0
    free = np.argwhere(~near)
    c = free + 0.5 + BMIN
    ok = (c[:, 2] >= 2) & (c[:, 2] <= 8) & (np.abs(c[:, 1]) <= 17)
    st, gl = c[ok & (c[:, 0] >= -17) & (c[:, 0] <= -12)], c[ok & (c[:, 0] >= 12) & (c[:, 0] <= 17)]
    rng = np.random.default_rng(seed)
    return st[rng.choice(len(st), B, replace=len(st) < B)], gl[rng.choice(len(gl), B, replace=len(gl) < B)]


def min_clearance(truth, logs, where=None):
    """the minimum true clearance over every flown pose; where (a dict) receives the log index, vehicle and witness voxel of that pose"""
    import torch
    m = float("inf")
    for k, (vi, lg) in enumerate(logs):
        rec = lg.reshape(-1, lg.shape[-1]).contiguous()
        Q = rec.shape[0]
        clear = torch.empty(Q, dtype=torch.float64, device=rec.device)
        vox = torch.empty(Q, dtype=torch.int64, device=rec.device)
        summ = torch.empty((1, 48), dtype=torch.uint8, device=rec.device)
        base = rec.data_ptr()
        truth.pose_clearance_device(Q, base + 8, base + 56, lg.shape[-1], truth.pose_clearance_params(), clear.data_ptr(), vox.data_ptr(),
                                    summ.data_ptr(), torch.cuda.current_stream().cuda_stream)
        j = int(torch.argmin(clear))
        if float(clear[j]) < m and where is not None:
            where.update(log=k, vehicle=int(vi[j // lg.shape[1]]), voxel=int(vox[j]))
        m = min(m, float(clear.min()))
    return m


def rig(k):
    """k = 1: the reference camera; k = 4: four cameras at yaw 0, 90, 180, 270 deg (cam_to_body = Rz cam02body, exact in FP64)"""
    import isdf_b200 as I
    c0 = np.array([[0, 0, 1, 0], [-1, 0, 0, 0], [0, -1, 0, 0], [0, 0, 0, 1]], dtype=np.float64)
    cams = []
    for c, s in [(1, 0), (0, 1), (-1, 0), (0, -1)][:k]:
        Rz = np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=np.float64)
        cams.append(I.sense_params(sensing_horizon=15.0, cam_to_body=(Rz @ c0).reshape(-1)))
    return cams[0] if k == 1 else cams


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vehicles", default="1,16,64")
    ap.add_argument("--rounds", type=int, default=40)
    ap.add_argument("--horizon", type=float, default=0.5)
    ap.add_argument("--sense-every", type=int, default=25)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--fallback", choices=("keep", "brake"), default="keep")
    ap.add_argument("--unknown", choices=("free", "occupied"), default=None)
    ap.add_argument("--cameras", type=int, choices=(1, 4), default=1)
    ap.add_argument("--prefer-known", type=float, default=None, metavar="W")
    ap.add_argument("--explore", action="store_true")
    ap.add_argument("--min-gain", type=int, default=None, metavar="G")
    args = ap.parse_args()
    if args.unknown == "occupied" and args.fallback != "brake":
        raise SystemExit("--unknown occupied needs --fallback brake")
    if args.explore and args.unknown != "occupied":
        raise SystemExit("--explore needs --unknown occupied")
    if args.min_gain is not None and not args.explore:
        raise SystemExit("--min-gain needs --explore")
    import torch
    import isdf_b200 as I
    if not torch.cuda.is_available():
        raise SystemExit("bench_navigate.py measures the GPU path and needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    cfg = I.default_config_values()
    cfg.integral_intervs, cfg.kernel_size, cfg.vmax = 16, 11, 3.0
    truth = I.Evaluator(cfg)
    truth.set_shape_named("Ball")
    scene = world(truth)
    truth.set_map_u8(np.zeros(DIMS, np.uint8), BMIN, RES)
    truth.map_fuse_cloud_device(scene, stream=torch.cuda.current_stream().cuda_stream)
    occ = truth.get_map_u8()
    out = dict(bench="navigate", gpu=gpu, world="mockamap boxes seed 511, 40 x 40 x 10 m, 20 boxes; 1 m frame", points=int(scene.shape[0]),
               horizon_s=args.horizon, sense_every=args.sense_every, runs=[])
    brake = args.fallback == "brake"
    if brake:
        out["fallback"] = "brake"
    trace = args.unknown is not None or args.cameras != 1
    if trace:
        out.update(unknown=args.unknown or "free", cameras=args.cameras)
    pkw = dict(flags=I.PLAN_CERTIFY, backend_max_iterations=200)
    if args.prefer_known is not None:
        pkw.update(flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_PREFIX, unknown_weight=args.prefer_known)
        out["prefer_known"] = args.prefer_known
    if args.explore:
        out["explore"] = True
    if args.min_gain is not None:
        out["min_gain"] = args.min_gain
    for B in [int(v) for v in args.vehicles.split(",")]:
        starts, goals = pairs(occ, B, args.seed + B)
        ev = I.Evaluator(cfg)
        ev.set_shape_named("Ball")
        ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
        ev.set_map_u8(np.zeros(DIMS, np.uint8), BMIN, RES)
        ev.set_sense_cloud_device(scene, stream=torch.cuda.current_stream().cuda_stream)
        kw = dict(unknown="occupied", known_boxes=np.concatenate([starts - 2.5, starts + 2.5], 1)) if args.unknown == "occupied" else {}
        if args.explore:
            kw["explore"] = True
        if args.min_gain is not None:
            kw["min_gain"] = args.min_gain
        r = ev.navigate(starts, goals, rounds=args.rounds, horizon=args.horizon, sense_every=args.sense_every, tol=1.0,
                        plan_params=ev.plan_params(**pkw),
                        sense_params=rig(args.cameras), fallback=args.fallback, **kw)
        fail = np.isin(r["actions"], [I.NAV_REPLAN_FAILED, I.NAV_BRAKED, I.NAV_HELD]) if brake else r["actions"] == I.NAV_REPLAN_FAILED
        why = {}   # failed replans by (plan stage, certificate verdict); -2: no plan call (a head outside the frame)
        for st, v in zip(r["replan_stages"][fail], r["replan_verdicts"][fail]):
            why[f"{st}/{v}"] = why.get(f"{st}/{v}", 0) + 1
        stages = list(r["times"][0])
        ms = {k: round(float(np.mean([t[k] for t in r["times"]])), 3) for k in stages}
        out["runs"].append(dict(vehicles=B, rounds=len(r["times"]), ms_per_round=ms, ms_round_total=round(sum(ms.values()), 3),
                                arrived=int((r["status"] == I.NAV_ARRIVED).sum()), stopped=int((r["status"] == I.NAV_STOPPED).sum()),
                                diverged=int((r["status"] == I.NAV_DIVERGED).sum()), timeout=int((r["status"] == I.NAV_TIMEOUT).sum()),
                                replans=int(r["replans"].sum()), failed_replans=int(r["failed_replans"].sum()), failed_by_stage_verdict=why,
                                uncertified_rounds=int(r["uncertified_rounds"].sum()), map_voxels=int(ev.map_info()["occupied_voxels"]),
                                min_true_clearance=round(min_clearance(truth, r["logs"], where := {}), 4)))
        if brake:
            out["runs"][-1].update(brakes=int(r["brakes"].sum()), held_rounds=int(r["held_rounds"].sum()))
        if "commits" in r:
            out["runs"][-1].update(commits=int(r["commits"].sum()))
        if "frontier_plans" in r:
            out["runs"][-1].update(frontier_plans=int(r["frontier_plans"].sum()))
        if "frontier_gains" in r:
            fg = r["frontier_gains"]
            chosen = fg[fg >= 0]
            edges = [0, 1, 10, 100, 1000, 10000, 1 << 62]
            hist = np.histogram(chosen, bins=edges)[0] if chosen.size else np.zeros(len(edges) - 1, dtype=int)
            last = {}   # a vehicle that ends held (TIMEOUT): the gain of the last frontier it was sent to
            for b in np.nonzero(r["status"] == I.NAV_TIMEOUT)[0]:
                g = fg[:, b][fg[:, b] >= 0]
                if g.size:
                    last[int(b)] = int(g[-1])
            out["runs"][-1].update(frontier_gain_hist={f"[{a},{b})": int(n) for a, b, n in zip(edges[:-1], edges[1:], hist)},
                                   timeout_last_frontier_gain=last)
        if trace and where:
            flown = [k for k in range(len(r["times"])) if (r["verdicts"][k] != I.NAV_NO_TRAJECTORY).any()]
            v = where["voxel"]
            fused = bool(ev.get_map_u8().reshape(-1)[v]) if v >= 0 else None
            out["runs"][-1].update(min_clearance_at=dict(vehicle=where["vehicle"], round=flown[where["log"]], witness_voxel=v,
                                                         witness_in_fused_map=fused))
        ev.close()
    truth.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
