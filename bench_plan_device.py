"""The planning step in host memory against device memory on an H100: isdf_plan_batch against isdf_plan_batch_device; one JSON line per B.

  python bench_plan_device.py [--batches 16,128,1024] [--reps 3] [--small]

Workload (bench_plan.py's): workloads.three_slit_map(128, 128, 128, noise=0.01, seed 4), the Ball, one start and B free goals drawn with
a fixed seed, back-end max_iterations 100 and mid-end cancel_after 500, both certificates on. Caps are the sizes a warm-up call reported.

Arms, alternated rep by rep after one warm-up call each:
  host    isdf_plan_batch with numpy outputs (the host form stages the pipeline's device outputs and copies them back)
  device  isdf_plan_batch_device with goals and every output in torch CUDA tensors, on torch's current stream
Per arm: wall ms of each rep (a host clock around a call that returns when its outputs are complete; the device arm adds a
torch.cuda.synchronize), the per-stage device ms of isdf_get_plan_info and the transfer counters of isdf_dbg_plan_transfers, both of the
last rep. Every rep's outputs are checked bit-equal between the arms before the line is printed. Each line carries the card's name and
power limit. Writes nothing to the tree."""
import argparse
import ctypes as C
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


def host_arm(I, ev, p, start, goals, cap_nodes, cap_pieces):
    B = len(goals)
    ip = C.POINTER(C.c_int32)
    st, gl = np.ascontiguousarray(start, dtype=np.float64), np.ascontiguousarray(goals, dtype=np.float64)
    pf, po = np.zeros(B + 1, dtype=np.int32), np.zeros(B + 1, dtype=np.int32)
    xyz, T, Cc = np.zeros((cap_nodes, 3)), np.zeros(cap_pieces), np.zeros(18 * cap_pieces)
    res, cs, ds = (I.PlanResult * B)(), (I.CertifySummary * B)(), (I.DynamicsSummary * B)()
    t0 = time.perf_counter()
    r = ev.lib.isdf_plan_batch(ev.h, I._dp(st), B, I._dp(gl), C.byref(p), cap_nodes, pf.ctypes.data_as(ip), I._dp(xyz), cap_pieces,
                               po.ctypes.data_as(ip), I._dp(T), I._dp(Cc), res, cs, ds)
    ms = (time.perf_counter() - t0) * 1e3
    assert r == 0, ev.lib.isdf_last_error().decode()
    n, q = int(pf[B]), int(po[B])
    out = [pf, xyz[:n], po, T[:q], Cc[:18 * q], np.frombuffer(res, np.uint8), np.frombuffer(cs, np.uint8), np.frombuffer(ds, np.uint8)]
    return ms, out


def device_arm(I, torch, ev, p, start, d_goals, cap_nodes, cap_pieces):
    B = d_goals.shape[0]
    dev = d_goals.device
    pf, po = torch.zeros(B + 1, dtype=torch.int32, device=dev), torch.zeros(B + 1, dtype=torch.int32, device=dev)
    xyz = torch.empty((cap_nodes, 3), dtype=torch.float64, device=dev)
    T, Cc = torch.empty(cap_pieces, dtype=torch.float64, device=dev), torch.empty(18 * cap_pieces, dtype=torch.float64, device=dev)
    res = torch.empty((B, C.sizeof(I.PlanResult)), dtype=torch.uint8, device=dev)
    cs = torch.empty((B, C.sizeof(I.CertifySummary)), dtype=torch.uint8, device=dev)
    ds = torch.empty((B, C.sizeof(I.DynamicsSummary)), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = ev.plan_batch_device_raw(start, B, d_goals.data_ptr(), p, cap_nodes, pf.data_ptr(), xyz.data_ptr(), cap_pieces, po.data_ptr(), T.data_ptr(),
                                 Cc.data_ptr(), res.data_ptr(), cs.data_ptr(), ds.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    assert r == 0, ev.lib.isdf_last_error().decode()
    n, q = int(pf[B]), int(po[B])
    out = [pf, xyz[:n], po, T[:q], Cc[:18 * q], res, cs, ds]
    return ms, [t.cpu().numpy().reshape(-1) if t.dim() != 2 or t.shape[1] != 3 else t.cpu().numpy() for t in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="16,128,1024")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--small", action="store_true", help="a 48^3 map and B = 16, 128 for plumbing checks (not a bench value)")
    args = ap.parse_args()
    import torch
    import isdf_b200 as I
    import workloads as W
    card = gpu()
    X = 48 if args.small else 128
    batches = [16, 128] if args.small else [int(b) for b in args.batches.split(",")]
    occ = W.three_slit_map(X, X, X, noise=0.01, seed=4)
    free = np.argwhere(occ == 0)
    start = free[np.argmin(np.abs(free - [4, 4, X // 2]).sum(1))] + 0.5
    cfg = I.default_config_values()
    cfg.integral_intervs = 16
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    p = ev.plan_params(backend_max_iterations=100, midend_cancel_after=500)
    for B in batches:
        goals = free[np.random.default_rng(1000 + B).choice(len(free), B, replace=False)] + 0.5
        d_goals = torch.tensor(goals, dtype=torch.float64, device="cuda")
        got, _ = ev.plan_batch(start, goals, p)                           # warm-up, and the caps
        cap_nodes, cap_pieces = max(sum(g["path_nodes"] for g in got), 1), max(sum(g["T"].size for g in got), 1)
        device_arm(I, torch, ev, p, start, d_goals, cap_nodes, cap_pieces)
        arms = {"host": dict(wall_ms=[]), "device": dict(wall_ms=[])}
        for _ in range(args.reps):
            hm, ho = host_arm(I, ev, p, start, goals, cap_nodes, cap_pieces)
            arms["host"].update(info=ev.plan_info(), transfers=ev.dbg_plan_transfers())
            dm, do = device_arm(I, torch, ev, p, start, d_goals, cap_nodes, cap_pieces)
            arms["device"].update(info=ev.plan_info(), transfers=ev.dbg_plan_transfers())
            for k, (a, b) in enumerate(zip(ho, do)):
                assert np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)), (B, k)
            arms["host"]["wall_ms"].append(round(hm, 2))
            arms["device"]["wall_ms"].append(round(dm, 2))
        for a in arms.values():
            a["info"] = {k: round(v, 2) if isinstance(v, float) else v for k, v in a["info"].items()}
        stages = I.decode_plan_results(torch.from_numpy(do[5].copy()))["stage"].numpy()
        line = dict(workload="plan_batch host vs device", robot="Ball", map=f"three_slit {X}^3 (noise 0.01, seed 4)", B=B, backend_iters=100,
                    midend_cancel=500, stages={str(s): int((stages == s).sum()) for s in sorted(set(stages.tolist()))}, nodes=cap_nodes,
                    pieces=cap_pieces, outputs_bit_equal=True, host=arms["host"], device=arms["device"],
                    wall_ratio_host_over_device=round(float(np.median(arms["host"]["wall_ms"]) / np.median(arms["device"]["wall_ms"])), 3), gpu=card)
        print(json.dumps(line), flush=True)
    ev.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
