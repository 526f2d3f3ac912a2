"""Per-kernel view of the discrete evaluation that bench.py times (BASELINE configs[2], mesh robot, one GPU).

For each window-list budget (default: the library's 16 codes per sample, and 0 = no lists, every window enumerated by the scan
kernel itself) prints one JSON line with
  * ms per step: CUDA events around isdf_eval_discrete_device on distinct iterates, L2 flushed between steps (bench.py's loop);
  * per-kernel device time, mean us per step, from torch.profiler's CUDA activity in a separate run (prologue, scan, epilogue, and
    the work-item builder on the aux stream, which overlaps the caller);
  * the window-list statistics of the last evaluation (runs, codes written, overflowed runs);
  * the card's name, power limit and SM clock, read in the same call.
Writes nothing to the tree."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))

KERNELS = {"prologue": "k_discrete_prologue", "scan": "k_discrete_mesh", "epilogue": "k_discrete_epilogue", "build_items": "k_build_items"}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.check_output(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"]).decode().strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--budgets", default="16,0", help="window-list budgets (codes per sample) to measure, in this order")
    a = ap.parse_args()
    import torch
    import bench as B
    import isdf_b200 as I
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU kernels")
    w, cfg, occ, T, Cc, V, F = B.make_workload()
    N = w["pieces"]
    ev = I.Evaluator(cfg, device=0)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_mesh(V, F, w["poly_params"])
    iters = B.make_iterates(w, T, Cc, a.warmup + a.steps + 1)
    dev = torch.device("cuda", 0)
    d_T, d_Cs = torch.from_numpy(T).to(dev), torch.from_numpy(iters).to(dev)
    d_out = torch.zeros(19 * N + 1, dtype=torch.float64, device=dev)
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def step(k):
        ev.eval_discrete_device(N, d_T.data_ptr(), d_Cs[k].data_ptr(), d_out.data_ptr(), stream)

    timed_ks = range(a.warmup, a.warmup + a.steps)
    for budget in [int(b) for b in a.budgets.split(",")]:
        ev.dbg_window_lists(budget=budget)
        for k in range(a.warmup):
            step(k)
        torch.cuda.synchronize()
        ts = []
        for k in timed_ks:
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(); step(k); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        lists = ev.dbg_window_lists()
        # per-kernel device times in a run of their own (tracing slows the host)
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in timed_ks:
                flush.zero_()
                step(k)
            torch.cuda.synchronize()
        us = {}
        for e in prof.key_averages():
            for short, name in KERNELS.items():
                if name in e.key:
                    us[short] = us.get(short, 0.0) + e.device_time_total / a.steps
        print(json.dumps({"budget_codes_per_sample": budget, "ms_per_step": statistics.mean(ts), "ms_min": min(ts), "ms_max": max(ts),
                          "kernel_us_per_step": us, "lists": lists, "gpu": gpu_info(),
                          "workload": B.workload_name(w)}))
    ev.close()


if __name__ == "__main__":
    main()
