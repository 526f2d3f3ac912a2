"""CPU-run invariants of the product's mesh acceleration structures (tests/host_mesh_check.cu compiled with nvcc for the HOST):
the 32-ary tree's leaves partition the triangles, leaf boxes (axis-aligned and oriented) contain their triangles, both box
distances are lower bounds of the exact leaf distance at near and far query points, and the host-compiled closest-triangle search
(the same code the device's lane searches run) equals brute force."""
import os
import shutil
import subprocess
import numpy as np
import pytest
import workloads as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("hm") / "host_mesh_check")
    r = subprocess.run(["nvcc", "-std=c++17", "-O2", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                        os.path.join(ROOT, "tests", "host_mesh_check.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return exe


@pytest.mark.parametrize("mesh", ["rcone", "lprism", "ico", "box"])
def test_mesh_structures_hold_their_invariants(checker, mesh, tmp_path):
    V, F = {"rcone": W.rounded_cone_mesh, "lprism": W.l_prism_mesh, "ico": lambda: W.icosphere(1.3, 2), "box": lambda: W.box_mesh(1.2, 0.7, 0.4)}[mesh]()
    vf, ff = str(tmp_path / "V.bin"), str(tmp_path / "F.bin")
    np.ascontiguousarray(V, dtype=np.float64).tofile(vf)
    np.ascontiguousarray(F, dtype=np.int32).tofile(ff)
    r = subprocess.run([checker, vf, ff, str(len(V)), str(len(F))], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "HOST MESH OK" in r.stdout, (r.stdout, r.stderr)
