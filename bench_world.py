#!/usr/bin/env python
"""bench_world.py — the world generators (isdf_world_*) on an H100 against the serial restatement and the reference's own generators;
prints one JSON line.

  python bench_world.py [--steps K] [--warmup W] [--no-serial]

Cases: globalmap_gene maps 3 and 10 at 0.1 m and 0.05 m (5.4 M to 1.4e8 points), mockamap's Perlin world at 512 x 512 x 128 (33.5 M
voxels, launch-file noise parameters) and 200 boxes. Arms (medians of K steps after W warm-up calls):
  device_ms   isdf_world_cloud_device into a preallocated CUDA tensor, CUDA events around the call;
  host_ms     isdf_world_cloud into a preallocated numpy array, host clock (includes the device-to-host copy of n x 16 bytes);
  serial_ms   tests/world_serial.cpp (libc rand, std::sort), one timed pass, for the cases up to 0.1 m;
  ref_ms      the reference's own generators (oracle/_ref/libref_world.so, where built), one timed pass, same cases.
Parity: the device cloud is compared byte for byte with the serial one wherever the serial arm runs (differing: false expected).
chain_ms: map 10 at 0.1 m generated and voxelised (isdf_set_map_cloud_device at 0.1 m) without leaving the device, CUDA events.
write_GBps: n x 16 bytes over device_ms, the emission's store rate. Writes nothing to the tree.
"""
import argparse
import ctypes as C
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
sys.dont_write_bytecode = True

CASES = [("gm3_r0.1", "globalmap", dict(map_id=3, cloud_resolution=0.1), True),
         ("gm10_r0.1", "globalmap", dict(map_id=10, cloud_resolution=0.1), True),
         ("gm3_r0.05", "globalmap", dict(map_id=3, cloud_resolution=0.05), False),
         ("gm10_r0.05", "globalmap", dict(map_id=10, cloud_resolution=0.05), False),
         ("perlin_512x512x128", "perlin", dict(size=[512, 512, 128]), True),
         ("boxes_200", "boxes", dict(obstacle_number=200), True)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-serial", action="store_true")
    args = ap.parse_args()
    import torch
    import isdf_b200 as I
    import world_oracle as WO
    if not torch.cuda.is_available():
        raise SystemExit("bench_world.py measures the GPU path and needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    ev = I.Evaluator(I.default_config_values(), device=0)
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    out = {"gpu": gpu, "steps": args.steps, "cases": {}}
    for name, kind, kw, serial in CASES:
        p = I.world_params(kind, **kw)
        n = C.c_int64(-1)
        ev.lib.isdf_world_cloud_device(ev.h, C.byref(p), 0, None, C.byref(n), C.c_void_p(st.cuda_stream))   # size query
        N = n.value
        assert N > 0, name
        t = torch.empty((N, 4), dtype=torch.float32, device=dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dms = []
        for i in range(args.warmup + args.steps):
            e0.record(st)
            assert ev.lib.isdf_world_cloud_device(ev.h, C.byref(p), N, C.c_void_p(t.data_ptr()), C.byref(n), C.c_void_p(st.cuda_stream)) == 0
            e1.record(st)
            e1.synchronize()
            if i >= args.warmup:
                dms.append(e0.elapsed_time(e1))
        h = np.empty((N, 4), dtype=np.float32)
        hms = []
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            assert ev.lib.isdf_world_cloud(ev.h, C.byref(p), N, h.ctypes.data_as(C.c_void_p), C.byref(n)) == 0
            if i >= args.warmup:
                hms.append(1e3 * (time.perf_counter() - t0))
        r = {"n": N, "device_ms": round(statistics.median(dms), 4), "host_ms": round(statistics.median(hms), 2),
             "write_GBps": round(16 * N / (statistics.median(dms) * 1e6), 1),
             "host_equals_device": bool(np.array_equal(h.view(np.uint32), t.cpu().numpy().view(np.uint32)))}
        if serial and not args.no_serial:
            t0 = time.perf_counter()
            s = WO.serial(p)
            r["serial_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
            r["differing"] = not (len(s) == N and s.tobytes() == h.tobytes())
            del s
            if WO.ref_lib() is not None:
                t0 = time.perf_counter()
                f = WO.ref(p)
                r["ref_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
                r["ref_differing"] = not (len(f) == N and f.tobytes() == h.tobytes())
                del f
        out["cases"][name] = r
        del t, h
        torch.cuda.empty_cache()
    # chain: map 10 at 0.1 m generated and voxelised on the device
    p = I.world_params("globalmap", map_id=10, cloud_resolution=0.1)
    n = C.c_int64(0)
    ev.lib.isdf_world_cloud_device(ev.h, C.byref(p), 0, None, C.byref(n), C.c_void_p(st.cuda_stream))
    t = torch.empty((n.value, 4), dtype=torch.float32, device=dev)
    cms = []
    for i in range(args.warmup + args.steps):
        e0.record(st)
        ev.lib.isdf_world_cloud_device(ev.h, C.byref(p), n.value, C.c_void_p(t.data_ptr()), C.byref(n), C.c_void_p(st.cuda_stream))
        ev.set_map_cloud_device(t.data_ptr(), n=n.value, stride_bytes=16, res=0.1, stream=st.cuda_stream)
        e1.record(st)
        e1.synchronize()
        if i >= args.warmup:
            cms.append(e0.elapsed_time(e1))
    out["chain_ms"] = round(statistics.median(cms), 3)
    out["chain_map"] = {k: (list(map(float, v)) if hasattr(v, "__len__") else v) for k, v in ev.map_info().items() if k in ("dims", "occupied_voxels")}
    ev.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
