"""Planning-step benchmark: isdf_plan_batch (generateTraj for one start and B goals in one call) against the Python chain of public calls it
replaces (tests/test_gpu_midend.py::test_generate_traj_chain_end_to_end, with one isdf_gather_obstacle_points per plan).

Workloads: workloads.three_slit_map(128, 128, 128, noise=0.01), the Ball and the RoundedCone mesh (workloads.rounded_cone_mesh), B = 1, 16
and 128 goals drawn from the free voxels with a fixed seed, isdf_plan_default_params (both certificates on) except two caps that keep a run
short: the back end's max_iterations (--backend-iters, 100) and the mid-end's cancel rule (--midend-cancel, 500). With the defaults (10000
back-end iterations) one plan on the Ball takes about 30 000 batched back-end evaluations. Per workload one JSON line:
device ms per stage (isdf_get_plan_info), wall ms of the call, the stage histogram, and wall ms of the Python chain after checking that its
outputs equal the call's bit for bit. A second line per workload times the batched gather of the plans' waypoints against one
isdf_gather_obstacle_points per plan. Writes nothing to the tree."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16,128")
    ap.add_argument("--robots", default="Ball,mesh")
    ap.add_argument("--K", type=int, default=16, help="integral_intervs of the context")
    ap.add_argument("--size", type=int, default=128)
    ap.add_argument("--backend-iters", type=int, default=100, help="isdf_plan_params.backend.max_iterations (the default is 10000)")
    ap.add_argument("--midend-cancel", type=int, default=500, help="isdf_plan_params.midend.cancel_after (the default is 8000)")
    a = ap.parse_args()
    import isdf_b200 as I
    import workloads as W
    from test_gpu_plan import _compose, _check_plan
    occ = W.three_slit_map(a.size, a.size, a.size, noise=0.01, seed=4)
    free = np.argwhere(occ == 0)
    start = free[np.argmin(np.abs(free - [4, 4, 24]).sum(1))] + 0.5
    cfg = I.default_config_values()
    cfg.integral_intervs = a.K
    for robot in a.robots.split(","):
        def make():
            ev = I.Evaluator(cfg)
            ev.set_map_u8(occ, [0, 0, 0], 1.0)
            if robot == "mesh":
                V, F = W.rounded_cone_mesh()
                ev.set_shape_mesh(V, F)
            else:
                ev.set_shape_named(robot)
            ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
            return ev
        ev = make()
        for B in (int(x) for x in a.batches.split(",")):
            goals = free[np.random.default_rng(1000 + B).choice(len(free), B, replace=False)] + 0.5
            p = ev.plan_params(backend_max_iterations=a.backend_iters, midend_cancel_after=a.midend_cancel)
            ev.plan_batch(start, goals, p)                     # warm-up: buffers, kernel images
            t0 = time.perf_counter()
            got, info = ev.plan_batch(start, goals, p)
            wall = (time.perf_counter() - t0) * 1e3
            chain_ev = make()
            _compose(chain_ev, start, goals, p)                # warm-up of the chain's context
            chain_ev.close()
            chain_ev = make()
            t0 = time.perf_counter()
            ref = _compose(chain_ev, start, goals, p)
            chain_wall = (time.perf_counter() - t0) * 1e3
            equal = max((r["duration"] for r in ref), default=0.0) < 300.0
            if equal:
                for b in range(B):
                    _check_plan(got[b], ref[b], b)
            # the gather alone: the plans' waypoints, batched against one call per plan
            wps, _ = I.path_waypoints([g["path"] for g in got], 1.0, p.parlength)
            half = p.half_extent
            ev.gather_obstacle_points_batch(wps, half)
            t0 = time.perf_counter()
            lists = ev.gather_obstacle_points_batch(wps, half)
            g_batch = (time.perf_counter() - t0) * 1e3
            t0 = time.perf_counter()
            singles = [chain_ev.gather_obstacle_points(w, half)[0] if len(w) else np.zeros((0, 3)) for w in wps]
            g_single = (time.perf_counter() - t0) * 1e3
            assert all(np.array_equal(x, y) for x, y in zip(lists, singles))
            chain_ev.close()
            hist = {str(s): int(sum(g["stage"] == s for g in got)) for s in sorted({g["stage"] for g in got})}
            print(json.dumps(dict(workload="plan_batch", robot=robot, map=a.size, B=B, K=a.K, backend_iters=a.backend_iters, midend_cancel=a.midend_cancel, stage_ms={k: round(v, 3) for k, v in info.items() if k.endswith("_ms")},
                                  groups=info["groups"], backend_rounds=info["backend_rounds"], call_wall_ms=round(wall, 2), stages=hist,
                                  chain_wall_ms=round(chain_wall, 2), chain_equal_checked=bool(equal))), flush=True)
            print(json.dumps(dict(workload="gather", robot=robot, B=B, waypoints=int(sum(len(w) for w in wps)), points=int(sum(len(x) for x in lists)),
                                  batched_wall_ms=round(g_batch, 3), single_calls_wall_ms=round(g_single, 3))), flush=True)
        ev.close()


if __name__ == "__main__":
    main()
