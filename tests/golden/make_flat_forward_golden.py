"""Golden vectors of the reference's FlatnessMap::forward (utils/flatness.hpp:150-207) at psi = dpsi = 0, computed by REFERENCE-COMPILED
code: a small C wrapper, written out below, is compiled into a temporary directory against the reference's own flatness.hpp and the
element-access Eigen stand-in oracle/_shim/Eigen/Eigen, with the flags of oracle/Makefile's libref_flat.so (-O3, no -march: no FMA).
Nothing is written outside this directory's fixture. Run where the reference tree exists:
    python tests/golden/make_flat_forward_golden.py [REFERENCE_ROOT]
  flat_forward_reference.npz — per config tag (drag: the default config; nodrag: drag coefficients 0): par {mass, grav, dh, dv, cp, veps},
                               seeded v, a, j, and the reference's thrust, quaternion and body rate. The dynamic-limit certificate's
                               thrust (tests/dynlimits_oracle.py::thrust_exact and the device's, at samples) is held to it."""
import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
import isdf_b200 as I          # noqa: E402

WRAPPER = r"""
#include <utils/flatness.hpp>
extern "C" void forward_thrust(const double *par, int n, const double *vel, const double *acc, const double *jer, double *thr,
                               double *quat, double *omg) {
    flatness::FlatnessMap F; F.reset(par[0], par[1], par[2], par[3], par[4], par[5]);
    for (int i = 0; i < n; i++) {
        Eigen::Vector3d v, a, j, o; Eigen::Vector4d q;
        for (int k = 0; k < 3; k++) { v(k) = vel[3 * i + k]; a(k) = acc[3 * i + k]; j(k) = jer[3 * i + k]; }
        const double psi = 0.0, dpsi = 0.0;
        F.forward(v, a, j, psi, dpsi, thr[i], q, o);
        for (int k = 0; k < 4; k++) quat[4 * i + k] = q(k);
        for (int k = 0; k < 3; k++) omg[3 * i + k] = o(k);
    }
}
"""


def inputs(n, seed):
    rng = np.random.default_rng(seed)
    scale = 10.0 ** rng.uniform(-2, 1.3, size=(n, 1))
    v, a, j = rng.normal(size=(n, 3)) * scale, rng.normal(size=(n, 3)) * scale * 1.5, rng.normal(size=(n, 3)) * scale * 3
    a[:, 2] = np.abs(a[:, 2]) * 0.3 - 2.0   # keeps thrust away from the singular zu = -|zu| e_z
    return v, a, j


def main(reference):
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    tmp = tempfile.mkdtemp()
    try:
        src, lib = os.path.join(tmp, "forward.cpp"), os.path.join(tmp, "libforward.so")
        with open(src, "w") as f:
            f.write(WRAPPER)
        subprocess.check_call([gxx, "-O3", "-std=c++14", "-fPIC", "-ffp-contract=off", "-I", os.path.join(ROOT, "oracle", "_shim"),
                               "-I", os.path.join(reference, "src", "utils", "include"), "-shared", "-o", lib, src])
        L = C.CDLL(lib)
        dp = C.POINTER(C.c_double)
        L.forward_thrust.argtypes = [dp, C.c_int, dp, dp, dp, dp, dp, dp]
        p = lambda a: a.ctypes.data_as(dp)   # noqa: E731
        out = {}
        for tag, drag in (("drag", True), ("nodrag", False)):
            cfg = I.default_config_values()
            if not drag:
                cfg.horiz_drag = cfg.vert_drag = cfg.paras_drag = 0.0
            v, a, j = inputs(256, seed=7 if drag else 8)
            par = np.array([cfg.vehicle_mass, cfg.grav_acc, cfg.horiz_drag, cfg.vert_drag, cfg.paras_drag, cfg.speed_eps])
            thr, q, o = np.zeros(len(v)), np.zeros((len(v), 4)), np.zeros((len(v), 3))
            L.forward_thrust(p(par), len(v), p(v), p(a), p(j), p(thr), p(q), p(o))
            out.update({f"{tag}_par": par, f"{tag}_v": v, f"{tag}_a": a, f"{tag}_j": j, f"{tag}_thr": thr, f"{tag}_quat": q, f"{tag}_omg": o})
    finally:
        shutil.rmtree(tmp)
    np.savez(os.path.join(HERE, "flat_forward_reference.npz"), **out)
    print("flat_forward_reference.npz written")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
