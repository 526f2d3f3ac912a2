"""Writes tests/golden/navigate_reference.npz: what Evaluator.navigate computes in the five runs of tests/test_gpu_navigate_golden.py
(counts, per-round tables, logged vehicles and SHA-256 digests of the logs, stage names), with the device name and SM count.
Recorded at commit 5f8d440, before navigate's round loop was rebuilt on one ragged trajectory set, on an NVIDIA H100 80GB HBM3
(132 SMs). Every run is made twice and must reproduce before it is written. Needs a GPU; run from the repository root:
python tests/golden/make_navigate_golden.py [out.npz]"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "implicit-sdf-planner_b200", "py"))
import test_gpu_navigate_golden as G  # noqa: E402


def main():
    import torch
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "navigate_reference.npz")
    prop = torch.cuda.get_device_properties(0)
    out = dict(device=np.array(prop.name), sm_count=np.array(prop.multi_processor_count))
    for name, run in G.SCENARIOS.items():
        a, b = G.record(run()), G.record(run())
        bad = [k for k in a if not np.array_equal(a[k], b[k])]
        if bad:
            raise SystemExit(f"{name}: two runs differ in {bad}")
        out.update({f"{name}.{k}": v for k, v in a.items()})
        print(name, {k: v.shape for k, v in a.items()}, flush=True)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes on", prop.name, prop.multi_processor_count, "SMs")


if __name__ == "__main__":
    main()
