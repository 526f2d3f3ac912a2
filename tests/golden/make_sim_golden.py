"""Writes tests/golden/sim_reference.npz: the reference's own simulator (oracle/_ref/libref_sim.so, built by oracle/sim.mk from
Quadrotor.cpp, SO3Control.cpp, quadrotor_simulator_so3.cpp's getControl and the vendored odeint) on component cases and short closed-loop
rollouts, with their inputs, so the CPU and GPU tests run without the reference tree. Needs the built library (no GPU); run once from the
repository root: python tests/golden/make_sim_golden.py"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "implicit-sdf-planner_b200", "py"))
import isdf_b200 as I  # noqa: E402
import sim_oracle as S  # noqa: E402


def params_bytes(p):
    return np.frombuffer(bytes(p), dtype=np.uint8).copy()


def params_from(b):
    return I.SimParams.from_buffer_copy(np.asarray(b, dtype=np.uint8).tobytes())


def state(pos=(0, 0, 1), vel=(0, 0, 0), R=np.eye(3), omega=(0, 0, 0), rpm=(15000,) * 4):
    x = np.zeros(22)
    x[0:3], x[3:6], x[15:18], x[18:22] = pos, vel, omega, rpm
    x[6:15] = np.asarray(R, dtype=np.float64).T.reshape(9)   # column-major
    return x


def rot(axis, a):
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def nondefault():
    return I.sim_default_params(mass=1.3, grav=9.79, J=(3.1e-3, 2.2e-3, 5.5e-3), kf=1.1e-8, km=2.0e-10, arm=0.21, motor_tau=0.05,
                                min_rpm=800.0, max_rpm=30000.0, ctrl_mass=1.25, ctrl_grav=9.8, kx=(4.9, 5.3, 6.6), kv=(3.0, 3.7, 4.4),
                                kR=(1.3, 0.8, 1.1), kOm=(0.09, 0.06, 0.12), corrections=(4e-10, 0.01, -0.02), use_external_yaw=0)


def component_cases():
    rng = np.random.default_rng(11)
    pd = I.sim_default_params()
    pn = nondefault()
    out = {}
    # right-hand side: hover, tumbling, inverted, upside down at the floor, near-singular R and a non-orthonormal R (the LLT path)
    hover = np.sqrt(pd.mass * pd.grav / (4 * pd.kf))
    skew = rot(0, 0.3) @ rot(2, 1.1)
    X = [state(rpm=(hover,) * 4),
         state(vel=(1.5, -0.7, 0.4), R=rot(1, 0.8) @ rot(0, -0.5), omega=(40.0, -25.0, 60.0), rpm=(21000, 9000, 30000, 14000)),
         state(pos=(0.3, 0.2, 2.0), vel=(0.0, 0.2, -1.0), R=rot(0, np.pi), omega=(0.5, 0.1, -0.2)),
         state(pos=(0.0, 0.0, 0.0), vel=(0.1, 0.0, -0.5), R=rot(1, np.pi - 1e-3), rpm=(5000, 5000, 6000, 6000)),
         state(R=np.diag([1.0, 1.0, 1e-7]) @ skew, omega=(1.0, 2.0, 3.0)),
         state(R=skew + 0.05 * rng.normal(size=(3, 3)), vel=(0.2, 0.3, -0.1), omega=(-3.0, 2.0, 0.5))]
    RPM = [(hover,) * 4, (21000, 9000, 30000, 14000), (15000, 16000, 14000, 15500), (1200, 35000, 20000, 8000), (15000,) * 4,
           (18000, 12000, 16000, 14000)]
    DIST = [np.zeros(6), np.array([0.2, -0.1, 0.3, 1e-4, -2e-4, 5e-5]), np.zeros(6), np.array([0.0, 0.0, -1.0, 0, 0, 0]), np.zeros(6),
            np.array([1.0, 0.5, 0.0, 1e-3, 0, -1e-3])]
    P = [pd, pd, pd, pd, pn, pn]
    out["rhs/x"], out["rhs/rpm"], out["rhs/dist"] = np.array(X), np.array(RPM, dtype=np.float64), np.array(DIST)
    out["rhs/params"] = np.array([params_bytes(p) for p in P])
    dx = [S.ref_rhs(p, x, r, d) for p, x, r, d in zip(P, X, RPM, DIST)]
    out["rhs/dx"], out["rhs/acc"] = np.array([a for a, _ in dx]), np.array([b for _, b in dx])
    # single steps: smooth, rejection-heavy (|omega| ~ 1e3), far past 1000 tries in all (|omega| ~ 1e6, each try count per accepted step
    # stays below 1000), a floor contact, a NaN rollback (an infinite velocity), and the library's 100000-try bound (|omega| ~ 1e150: each
    # accepted try advances ~1e-152 s), where odeint would go on
    X = [state(vel=(0.5, 0.2, -0.3), omega=(0.3, -0.2, 0.1), rpm=(15000, 15500, 14500, 15200)),
         state(omega=(1000.0, -700.0, 300.0), rpm=(hover,) * 4),
         state(omega=(1e6, -4e5, 2e5), rpm=(hover,) * 4),
         state(pos=(0.0, 0.0, 1e-4), vel=(0.0, 0.0, -0.5), rpm=(0,) * 4),
         state(vel=(np.inf, 0.0, 0.0), rpm=(hover,) * 4),
         state(omega=(1e150, -3e149, 2e149), rpm=(hover,) * 4)]
    RPM = [(16000, 14000, 15000, 15500), (hover,) * 4, (hover,) * 4, (0,) * 4, (hover,) * 4, (hover,) * 4]
    P = [pd, pd, pd, pd, pd, pd]
    out["step/x"], out["step/rpm"] = np.array(X), np.array(RPM, dtype=np.float64)
    out["step/params"] = np.array([params_bytes(p) for p in P])
    res = [S.ref_step(p, x, r) for p, x, r in zip(P, X, RPM)]
    for _, c, ok in res:
        assert c["same"] == 1, (c, ok)
    out["step/status"] = np.array([ok for _, _, ok in res], dtype=np.int32)
    out["step/x_out"] = np.array([x for x, _, _ in res])
    out["step/counts"] = np.array([[c["accepted"], c["rejected"], c["rollbacks"], c["floor"]] for _, c, _ in res], dtype=np.int64)
    # setInput: NaN, under min_rpm, over max_rpm, inside
    U = np.array([[np.nan, 100.0, 4e4, 20000.0], [1199.0, 35001.0, np.nan, 1200.0], [0.0, 35000.0, -5.0, np.inf]])
    out["set_input/rpm"] = U
    out["set_input/params"] = np.array([params_bytes(pd), params_bytes(pd), params_bytes(pn)])
    out["set_input/input"] = np.array([S.ref_set_input(params_from(b), u) for b, u in zip(out["set_input/params"], U)])
    # getControl across the Psi gate (Psi = 0, just under 1, exactly 1, above), with use_external_yaw 1 and 0
    Rs, Om, Cmd, Pg = [], [], [], []
    for ext in (1, 0):
        pg = I.sim_default_params(use_external_yaw=ext)
        for a in (0.0, 1.0, np.pi / 2, 2.0):   # R = rot_x(a), Rd = I: Psi = 1 - cos(a)
            Rs.append(rot(0, a) @ rot(2, 0.4))
            Om.append([0.3, -0.2, 0.5])
            Cmd.append([0.3, -0.2, 9.9, np.cos(0.2), 0.0, 0.0, np.sin(0.2), 0.4 if ext else 0.0])
            Pg.append(pg)
    # Psi exactly 1 in FP32: R = rot_x(pi/2) with no yaw against Rd = I gives trace 1 in float
    Rs.append(rot(0, np.pi / 2)); Om.append([0.0, 0.0, 0.0]); Cmd.append([0.0, 0.0, 9.6, 1.0, 0.0, 0.0, 0.0, 0.0]); Pg.append(pd)
    Rs.append(rot(2, 0.7) @ rot(1, 0.3)); Om.append([2.0, -1.0, 0.5]); Cmd.append([0.5, 0.2, 9.0, 0.9, 0.1, -0.1, 0.2, 0.7]); Pg.append(pn)
    out["get_control/R"], out["get_control/omega"], out["get_control/cmd"] = np.array(Rs), np.array(Om), np.array(Cmd)
    out["get_control/params"] = np.array([params_bytes(p) for p in Pg])
    out["get_control/rpm"] = np.array([S.ref_get_control(p, R, o, c[0:3], c[3:7], c[7]) for p, R, o, c in zip(Pg, Rs, Om, Cmd)])
    # calculateControl on both sides of the limit at theta = pi/2 (force with a positive, zero and negative vertical part) and with an
    # unused desired position
    cases = [([0, 0, 1], [0.1, 0, 0], [0, 0, 0], [0.5, -0.2, 1.3], [0.2, 0.1, 0], [0.1, 0.2, 0.3]),
             ([0, 0, 1], [0, 0, 0], [0, 0, 0], [1.0, 0.0, 1.0], [0, 0, 0], [0, 0, -9.81 - 5.7 / 0.98 * 0 + 0.0]),
             ([0, 0, 3], [0, 0, 2], [0, 0, 0], [0.5, 0.3, 1.0], [0, 0, 0], [0.0, 0.0, -12.0]),
             ([0, 0, 1], [0, 0, 0], [0.1, 0, 0], [np.nan, 0, 0], [1.0, 0, 0], [0.0, 0.0, 0.0]),
             ([2, 1, 1], [0, 0, 0], [0, 0, 0], [2.0, 1.0, 1.0], [0, 0, 0], [4.0, 0.0, -9.81])]
    out["calc/in"] = np.array([np.concatenate([np.asarray(c, dtype=np.float64) for c in cs]) for cs in cases])
    fq = [S.ref_calculate_control(pd, *np.split(v, 6)) for v in out["calc/in"]]
    out["calc/force"], out["calc/quat"] = np.array([f for f, _ in fq]), np.array([q for _, q in fq])
    return out


def rollout_cases():
    """{name: (params, traj, init, dist)} over sim_oracle.line_trajectories(); every case keeps the reference's floor on"""
    off, T, Cc = S.line_trajectories()
    pd = I.sim_default_params
    rng = np.random.default_rng(5)
    traj = np.array([0, 1], dtype=np.int32)

    def start(p, rpm=None, jitter=0.05):
        init = I.sim_init_from_trajectories(off, Cc, traj, p, rpm=rpm)
        init[:, 0:3] += rng.normal(scale=jitter, size=(2, 3))
        return init

    dist = np.zeros((2, 6))
    dist[:, 0:3] = rng.normal(scale=0.1, size=(2, 3))
    dist[:, 3:6] = rng.normal(scale=1e-4, size=(2, 3))
    cases = {}
    p = pd(t_end=2.0, log_every=5)
    cases["default"] = (p, traj, start(p), dist)
    p = nondefault(); p.t_end, p.log_every = 2.0, 3
    cases["vehicle"] = (p, traj, start(p), dist)
    p = pd(sim_rate=100.0, t_end=2.0, log_every=4)
    cases["ratio1"] = (p, traj, start(p), dist)
    p = pd(sim_rate=2000.0, t_end=1.5, log_every=7)
    cases["ratio20"] = (p, traj, start(p), dist)
    p = pd(t_end=1.5, log_every=2, max_rpm=18000.0)   # a low rpm ceiling: the climb off the floor clamps the input
    init = start(p, rpm=0, jitter=0.0)
    init[:, 2], init[:, 5] = 0.0, -0.2   # zero rpm on the floor, moving down: the first steps put it back on the floor
    cases["floor"] = (p, traj, init, np.zeros((2, 6)))
    p = pd(t_end=1.0, diverge_dist=0.5)
    gust = dist.copy(); gust[1, 0] = 50.0
    cases["gust"] = (p, traj, start(p), gust)
    p = pd(t_end=3.0, log_every=10)   # trajectories of 2 s and 1 s: the command holds past their ends
    cases["hold"] = (p, traj, start(p), dist)
    p = pd(t_end=0.3, log_every=1)
    init = start(p)
    init[1, 13:17] = 1e160   # rpm^2 overflows: every step's integrated state has a NaN and step() restores it
    cases["rollback"] = (p, traj, init, dist)
    return (off, T, Cc), cases


def main():
    out = component_cases()
    (off, T, Cc), cases = rollout_cases()
    out["traj/off"], out["traj/T"], out["traj/C"] = off, T, Cc
    for name, (p, traj, init, dist) in cases.items():
        log, summ = S.ref_simulate(off, T, Cc, traj, init, dist, p)
        out[f"roll/{name}/params"], out[f"roll/{name}/traj"], out[f"roll/{name}/init"], out[f"roll/{name}/dist"] = params_bytes(p), traj, init, dist
        out[f"roll/{name}/log"] = log
        out[f"roll/{name}/summary"] = np.array([[s[k] for k in SUMMARY_FIELDS] for s in summ], dtype=np.float64)
        print(name, [(s["accepted"], s["rejected"], s["floor_contacts"], s["clamped_steps"], s["diverged"]) for s in summ])
    out["roll/names"] = np.array(list(cases))
    np.savez_compressed(os.path.join(HERE, "sim_reference.npz"), **out)
    print("wrote", os.path.join(HERE, "sim_reference.npz"))


SUMMARY_FIELDS = [n for n, _ in I.SimSummary._fields_]

if __name__ == "__main__":
    main()
