"""(start, goal) pairs on an H100: one pairs call against one call per start; one JSON line per workload.

  python bench_pairs.py [--sources 1,4,16] [--batches 16,128] [--robots Ball] [--small]

Front end (isdf_frontend_path_pairs against isdf_frontend_path per pair): the 512^3 random map of bench.py (p = 0.05, 3 wall slabs,
seed 1), the Ball at kernel_size 5 with 121 attitudes (as bench_frontpath.py), S pairs from S distinct traversable starts to traversable
goals drawn with a fixed seed. Per arm: device ms of the field stage and of the traversability builds (isdf_frontend_path_info, summed
over the single calls), relaxation rounds (summed likewise) and wall ms.

Planning (isdf_plan_pairs against isdf_plan_batch per pair): workloads.three_slit_map(128, 128, 128, noise=0.01) of bench_plan.py with its
caps (back-end max_iterations 100, mid-end cancel_after 500), B pairs with B distinct traversable starts and free goals drawn with a fixed
seed. Per arm: device ms per stage (isdf_get_plan_info, summed over the single calls) and wall ms.

Every arm's outputs are checked bit-equal to the other arm's before its line is printed. Each line carries the card's name and power
limit. Each arm runs once after a warm-up call. Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True
import numpy as np  # noqa: E402


def gpu():
    try:
        return subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        return None


def wall(call):
    t0 = time.perf_counter()
    out = call()
    return out, (time.perf_counter() - t0) * 1e3


def frontend(I, W, args, card):
    import frontpath_oracle as FO
    X = 128 if args.small else 512
    occ = W.random_map(X, X, X, p=0.05, seed=1, slabs=3)
    cfg = I.default_config_values()
    cfg.kernel_size = 5
    ev = I.Evaluator(cfg, device=0)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    masks = ev.frontend_feasibility(X, X, X)
    trav = np.argwhere(FO.traversable(occ, masks))
    del masks
    for S in (int(s) for s in args.sources.split(",")):
        rng = np.random.default_rng(100 + S)
        starts = trav[rng.choice(len(trav), S, replace=False)] + 0.5
        goals = trav[rng.choice(len(trav), S, replace=False)] + 0.5
        cap = int(ev.frontend_path_pairs(starts, goals)["offsets"][-1])   # warm-up, and the cap that fits: a too-small cap repeats the call
        res, pw = wall(lambda: ev.frontend_path_pairs(starts, goals, cap=cap))
        pi = ev.frontend_path_info()
        single = dict(wall_ms=0.0, field_ms=0.0, traversability_ms=0.0, rounds=0)
        for b in range(S):
            (p, rp, c, f), w = wall(lambda: ev.frontend_path(starts[b], goals[b]))
            i = ev.frontend_path_info()
            assert np.array_equal(p, res["paths"][b]) and np.array_equal(rp, res["roll_pitch"][b]) and f == res["found"][b]
            assert np.float64(c).view(np.uint64) == res["costs"][b].view(np.uint64)
            single["wall_ms"] += w
            single["field_ms"] += i["field_ms"]
            single["traversability_ms"] += i["traversability_ms"]
            single["rounds"] += i["rounds"]
        line = dict(workload="frontend_pairs", map=f"random {X}^3 (p=0.05, 3 wall slabs, seed 1)", robot="Ball", kernel_size=5, S=S,
                    found=int(res["found"].sum()), nodes=int(res["offsets"][-1]), outputs_bit_equal=True,
                    pairs=dict(wall_ms=round(pw, 2), field_ms=round(pi["field_ms"], 2), traversability_ms=round(pi["traversability_ms"], 2),
                               paths_ms=round(pi["paths_ms"], 2), rounds=pi["rounds"], field_bytes=pi["field_bytes"]),
                    single_calls={k: round(v, 2) if isinstance(v, float) else v for k, v in single.items()},
                    field_speedup=round(single["field_ms"] / pi["field_ms"], 3), wall_speedup=round(single["wall_ms"] / pw, 3), gpu=card)
        print(json.dumps(line), flush=True)
    ev.close()


def planning(I, W, args, card):
    import frontpath_oracle as FO
    from test_gpu_plan import _check_plan
    X = 48 if args.small else 128
    occ = W.three_slit_map(X, X, X, noise=0.01, seed=4)
    free = np.argwhere(occ == 0)
    cfg = I.default_config_values()
    cfg.integral_intervs = 16
    for robot in args.robots.split(","):
        ev = I.Evaluator(cfg)
        ev.set_map_u8(occ, [0, 0, 0], 1.0)
        if robot == "mesh":
            V, F = W.rounded_cone_mesh()
            ev.set_shape_mesh(V, F)
        else:
            ev.set_shape_named(robot)
        ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
        trav = np.argwhere(FO.traversable(occ, ev.frontend_feasibility(X, X, X)))
        p = ev.plan_params(backend_max_iterations=100, midend_cancel_after=500)
        for B in (int(x) for x in args.batches.split(",")):
            rng = np.random.default_rng(2000 + B)
            starts = trav[rng.choice(len(trav), B, replace=False)] + 0.5
            goals = free[rng.choice(len(free), B, replace=False)] + 0.5
            ev.plan_pairs(starts, goals, p)                                # warm-up
            (got, info), pw = wall(lambda: ev.plan_pairs(starts, goals, p))
            single = {k: 0.0 for k in info if k.endswith("_ms")}
            single["wall_ms"] = 0.0
            for b in range(B):
                (alone, ai), w = wall(lambda: ev.plan_batch(starts[b], goals[b:b + 1], p))
                _check_plan(got[b], alone[0], b)
                single["wall_ms"] += w
                for k in ai:
                    if k.endswith("_ms"):
                        single[k] += ai[k]
            hist = {str(s): int(sum(g["stage"] == s for g in got)) for s in sorted({g["stage"] for g in got})}
            line = dict(workload="plan_pairs", robot=robot, map=f"three_slit {X}^3 (noise 0.01, seed 4)", B=B, distinct_starts=B,
                        backend_iters=100, midend_cancel=500, stages=hist, outputs_bit_equal=True,
                        pairs=dict(wall_ms=round(pw, 2), groups=info["groups"], backend_rounds=info["backend_rounds"],
                                   **{k: round(v, 2) for k, v in info.items() if k.endswith("_ms")}),
                        single_calls={k: round(v, 2) for k, v in single.items()}, wall_speedup=round(single["wall_ms"] / pw, 3), gpu=card)
            print(json.dumps(line), flush=True)
        ev.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", default="1,4,16", help="distinct starts of the front-end workloads")
    ap.add_argument("--batches", default="16,128", help="pairs of the planning workloads")
    ap.add_argument("--robots", default="Ball")
    ap.add_argument("--skip", default="", help="frontend and/or planning")
    ap.add_argument("--small", action="store_true", help="128^3 and 48^3 maps for plumbing checks (not a bench value)")
    args = ap.parse_args()
    import isdf_b200 as I
    import workloads as W
    card = gpu()
    if "frontend" not in args.skip:
        frontend(I, W, args, card)
    if "planning" not in args.skip:
        planning(I, W, args, card)
    return 0


if __name__ == "__main__":
    sys.exit(main())
