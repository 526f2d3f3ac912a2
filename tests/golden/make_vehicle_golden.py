"""Reference outputs at the vehicles of tests/vehicles.py, computed by REFERENCE-COMPILED code. Run where the reference tree exists:
    python tests/golden/make_vehicle_golden.py [REFERENCE_ROOT]
  vehicle_reference.npz — per vehicle tag:
    {tag}_par                          {mass, grav, dh, dv, cp, veps} as FlatnessMap::reset takes them;
    {tag}_v/a/j/pg/vg/qg/og            flatness-map inputs (vehicles.flat_inputs: test_reference_pins.flat_inputs away from the singularities);
    {tag}_quat/omg/back                utils/flatness.hpp's optimizated_forward (quaternion, body rate) and backwardthreadsafe (n x 12) on them,
                                       from oracle/_ref/libref_flat.so (`make -C oracle ref`);
    c{k}_{tag}_att                     the vehicle-dependent columns quat(w, x, y, z) omg thr of SweptVolumeManager::process's state on case k
                                       of states_reference.npz (N = 1, 2, 7, 64, 290 pieces) at its times: FlatnessMap::forward
                                       (flatness.hpp:150-228) at yaw 0, compiled as make_states_golden.py compiles it, on that fixture's
                                       velocity, acceleration and jerk (reference-compiled trajectory.hpp, independent of the vehicle).
The archive is written with fixed member timestamps, so that regenerating it reproduces the committed file byte for byte."""
import ctypes as C
import io
import os
import shutil
import subprocess
import sys
import tempfile
import zipfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
import oracle_lib as O             # noqa: E402
import states_oracle as SO         # noqa: E402
import vehicles as VH              # noqa: E402
from make_states_golden import FLAT_WRAPPER   # noqa: E402

OUT = os.path.join(HERE, "vehicle_reference.npz")
N_FLAT = 256


def save_npz_fixed(path, arrays):
    """np.savez's layout (one .npy member per array) with every member dated 1980-01-01"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[name]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), compress_type=zipfile.ZIP_DEFLATED)


def compute(reference):
    O.build()
    assert O.ref_flat_available(), "oracle/_ref/libref_flat.so is missing: run make -C oracle ref where the reference tree exists"
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    tmp = tempfile.mkdtemp()
    try:
        cpp, so = os.path.join(tmp, "flat.cpp"), os.path.join(tmp, "libflat.so")
        with open(cpp, "w") as f:
            f.write(FLAT_WRAPPER)
        subprocess.check_call([gxx, "-O3", "-std=c++14", "-fPIC", "-ffp-contract=off", "-w", "-I", os.path.join(ROOT, "oracle", "_shim"), "-I",
                               os.path.join(reference, "src", "utils", "include"), "-shared", "-o", so, cpp])
        flat = C.CDLL(so)
        dp = C.POINTER(C.c_double)
        p = lambda a: a.ctypes.data_as(dp)   # noqa: E731
        flat.forward.argtypes = [dp, C.c_int, dp, dp, dp, dp, dp, dp]
        cases, _ = SO.load_golden()
        out = {}
        for t, tag in enumerate(VH.TAGS):
            cfg = VH.config(tag)
            par = VH.par(cfg)
            out[f"{tag}_par"] = par
            v, a, j, pg, vg, qg, og = VH.flat_inputs(cfg, N_FLAT, seed=40 + t)
            ref = O.RefFlat(O.config_from(cfg))
            assert np.array_equal(ref.par, par)
            q, o = ref.forward(v, a, j)
            assert np.array_equal(ref.forward_quat(v, a, j), q)
            out.update({f"{tag}_v": v, f"{tag}_a": a, f"{tag}_j": j, f"{tag}_pg": pg, f"{tag}_vg": vg, f"{tag}_qg": qg, f"{tag}_og": og,
                        f"{tag}_quat": q, f"{tag}_omg": o, f"{tag}_back": ref.backward(v, a, j, pg, vg, qg, og)})
            for k, c in enumerate(cases):
                pvaj = np.ascontiguousarray(c["rec"]["drag"][:, :12])
                n = pvaj.shape[0]
                vv, aa, jj = (np.ascontiguousarray(pvaj[:, s:s + 3]) for s in (3, 6, 9))
                thr, qq, oo = np.zeros(n), np.zeros((n, 4)), np.zeros((n, 3))
                flat.forward(p(par), n, p(vv), p(aa), p(jj), p(thr), p(qq), p(oo))
                out[f"c{k}_{tag}_att"] = np.concatenate([qq, oo, thr[:, None]], axis=1)
        return out
    finally:
        shutil.rmtree(tmp)


def main(reference):
    save_npz_fixed(OUT, compute(reference))
    print(os.path.basename(OUT), "written")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
