"""Golden records of isdf_trajectory_states, computed by REFERENCE-COMPILED code: SweptVolumeManager::process's state at a time
(sw_manager.hpp:961-971) on trajectories made by the reference's own MINCO. Two small C wrappers, written out below, are compiled into a
temporary directory with the flags of oracle/Makefile (-O3, no -march: no FMA), each against the Eigen stand-in its header needs:
  traj: utils/minco.hpp + utils/trajectory.hpp (oracle/_shim_dyn): MINCO_S3NU::getTrajectory, then Trajectory::getPos / getVel / getAcc /
        getJer (trajectory.hpp:545-593) at each time, each with its own locatePieceIdx, as process() calls them;
  flat: utils/flatness.hpp (oracle/_shim): FlatnessMap::forward(vel, acc, jer, 0.0, 0.0, thr, quat, omg) (flatness.hpp:150-228).
Nothing is written outside this directory's fixture. Run where the reference tree exists:
    python tests/golden/make_states_golden.py [REFERENCE_ROOT]
  states_reference.npz — per case k (N = 1, 2, 7, 64, 290 pieces): c{k}_head / tail (3 x 3, columns pos, vel, acc), c{k}_inPs (3 x N-1),
                         c{k}_T (the reference trajectory's durations), c{k}_coeffs (its coefficients in the library's 6N x 3 column-major
                         ascending-power layout: a pure reordering of getCoeffMat), c{k}_times; per config tag (drag: the default config;
                         nodrag: drag coefficients 0) {tag}_par {mass, grav, dh, dv, cp, veps} and c{k}_{tag}_rec (times x 20 records:
                         pos vel acc jer quat(w, x, y, z) omg thr)."""
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

PIECES = (1, 2, 7, 64, 290)

TRAJ_WRAPPER = r"""
#include <utils/minco.hpp>
// MINCO -> Trajectory<5>: durations N, coefficient matrices N x (3 x 6, column-major, highest power first), total duration; then per time
// getPos, getVel, getAcc, getJer (12 doubles)
extern "C" void traj_states(int N, const double *head, const double *tail, const double *inPs, const double *T, double *durations,
                            double *cmats, double *total, int nt, const double *times, double *out) {
    Eigen::Matrix3d h, t;
    for (int k = 0; k < 9; k++) { h(k) = head[k]; t(k) = tail[k]; }
    Eigen::Matrix3Xd P(3, N - 1);
    for (int k = 0; k < 3 * (N - 1); k++) P(k) = inPs[k];
    Eigen::VectorXd ts(N);
    for (int k = 0; k < N; k++) ts(k) = T[k];
    minco::MINCO_S3NU m;
    m.setConditions(h, t, N);
    m.setParameters(P, ts);
    Trajectory<5> traj;
    m.getTrajectory(traj);
    for (int i = 0; i < N; i++) {
        durations[i] = traj.getPiece(i).getDuration();
        const Trajectory<5>::CoefficientMat &cm = traj.getindexCoeffMat(i);
        for (int k = 0; k < 18; k++) cmats[18 * i + k] = cm(k);
    }
    *total = traj.getTotalDuration();
    for (int q = 0; q < nt; q++) {
        const Eigen::Vector3d p = traj.getPos(times[q]), v = traj.getVel(times[q]), a = traj.getAcc(times[q]), j = traj.getJer(times[q]);
        for (int k = 0; k < 3; k++) { out[12 * q + k] = p(k); out[12 * q + 3 + k] = v(k); out[12 * q + 6 + k] = a(k); out[12 * q + 9 + k] = j(k); }
    }
}
"""

FLAT_WRAPPER = r"""
#include <utils/flatness.hpp>
extern "C" void forward(const double *par, int n, const double *vel, const double *acc, const double *jer, double *thr, double *quat,
                        double *omg) {
    flatness::FlatnessMap F; F.reset(par[0], par[1], par[2], par[3], par[4], par[5]);
    for (int i = 0; i < n; i++) {
        Eigen::Vector3d v, a, j, o; Eigen::Vector4d q;
        for (int k = 0; k < 3; k++) { v(k) = vel[3 * i + k]; a(k) = acc[3 * i + k]; j(k) = jer[3 * i + k]; }
        F.forward(v, a, j, 0.0, 0.0, thr[i], q, o);
        for (int k = 0; k < 4; k++) quat[4 * i + k] = q(k);
        for (int k = 0; k < 3; k++) omg[3 * i + k] = o(k);
    }
}
"""


def cases():
    """seeded MINCO boundary conditions, waypoints and durations"""
    rng = np.random.default_rng(31)
    out = []
    for N in PIECES:
        head = np.stack([rng.normal(size=3) * 5, rng.normal(size=3), rng.normal(size=3) * 0.3], axis=1)
        tail = np.stack([rng.normal(size=3) * 5 + 20, rng.normal(size=3), rng.normal(size=3) * 0.3], axis=1)
        inPs = np.cumsum(rng.normal(size=(3, N - 1)) * 2 + 1.0, axis=1)
        T = rng.uniform(0.2, 2.5, N)
        out.append((N, head, tail, inPs, T))
    return out


def times_for(T, total, rng):
    """0, every junction (left-to-right sums, as locatePieceIdx subtracts), each junction -/+ 1 ulp, uniformly inside, the total duration,
    negative times and times past the end"""
    cs = np.cumsum(T)
    junctions = cs[:-1]
    return np.concatenate([[0.0, -0.0], junctions, np.nextafter(junctions, -np.inf), np.nextafter(junctions, np.inf), rng.uniform(0, total, 64),
                           [total, np.nextafter(total, -np.inf), np.nextafter(total, np.inf), cs[-1], -1e-300, -0.3, -7.0, total + 1e-9, total + 0.7,
                            2 * total]])


def configs():
    out = []
    for tag, drag in (("drag", True), ("nodrag", False)):
        cfg = I.default_config_values()
        if not drag:
            cfg.horiz_drag = cfg.vert_drag = cfg.paras_drag = 0.0
        out.append((tag, cfg, np.array([cfg.vehicle_mass, cfg.grav_acc, cfg.horiz_drag, cfg.vert_drag, cfg.paras_drag, cfg.speed_eps])))
    return out


def compute(reference):
    """every fixture array, from the reference compiled now"""
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    inc = os.path.join(reference, "src", "utils", "include")
    tmp = tempfile.mkdtemp()
    try:
        libs = {}
        for name, src, shim in (("traj", TRAJ_WRAPPER, "_shim_dyn"), ("flat", FLAT_WRAPPER, "_shim")):
            cpp, so = os.path.join(tmp, name + ".cpp"), os.path.join(tmp, "lib" + name + ".so")
            with open(cpp, "w") as f:
                f.write(src)
            subprocess.check_call([gxx, "-O3", "-std=c++14", "-fPIC", "-ffp-contract=off", "-w", "-I", os.path.join(ROOT, "oracle", shim), "-I", inc,
                                   "-shared", "-o", so, cpp])
            libs[name] = C.CDLL(so)
        dp = C.POINTER(C.c_double)
        p = lambda a: a.ctypes.data_as(dp)   # noqa: E731
        libs["traj"].traj_states.argtypes = [C.c_int, dp, dp, dp, dp, dp, dp, dp, C.c_int, dp, dp]
        libs["flat"].forward.argtypes = [dp, C.c_int, dp, dp, dp, dp, dp, dp]
        rng = np.random.default_rng(32)
        out = {}
        for tag, _, par in configs():
            out[f"{tag}_par"] = par
        for k, (N, head, tail, inPs, T) in enumerate(cases()):
            h, t, ip = (np.asfortranarray(x, dtype=np.float64) for x in (head, tail, inPs.reshape(3, -1)))
            dur, cm, total = np.zeros(N), np.zeros(18 * N), C.c_double(0)
            libs["traj"].traj_states(N, p(h), p(t), p(ip), p(T), p(dur), p(cm), C.byref(total), 0, p(np.zeros(1)), p(np.zeros(12)))
            times = times_for(dur, total.value, rng)
            pvaj = np.zeros((times.size, 12))
            libs["traj"].traj_states(N, p(h), p(t), p(ip), p(T), p(dur), p(cm), C.byref(total), times.size, p(times), p(pvaj))
            # column c of piece i's 3 x 6 matrix is power 5 - c: the library's block holds axis a, piece i, power k at a 6N + 6i + k
            coeffs = cm.reshape(N, 6, 3)[:, ::-1, :].transpose(2, 0, 1).reshape(-1).copy()
            out.update({f"c{k}_head": head, f"c{k}_tail": tail, f"c{k}_inPs": inPs, f"c{k}_T": dur, f"c{k}_coeffs": coeffs, f"c{k}_times": times})
            v, a, j = (np.ascontiguousarray(pvaj[:, s:s + 3]) for s in (3, 6, 9))
            for tag, _, par in configs():
                thr, q, o = np.zeros(times.size), np.zeros((times.size, 4)), np.zeros((times.size, 3))
                libs["flat"].forward(p(par), times.size, p(v), p(a), p(j), p(thr), p(q), p(o))
                out[f"c{k}_{tag}_rec"] = np.concatenate([pvaj, q, o, thr[:, None]], axis=1)
        return out
    finally:
        shutil.rmtree(tmp)


def main(reference):
    np.savez(os.path.join(HERE, "states_reference.npz"), **compute(reference))
    print("states_reference.npz written")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
