"""CPU checks of the closed-loop definition (include/isdf.h, isdf_simulate) on its serial restatement tests/sim_serial.cpp, and of the
default parameters the C ABI reports."""
import numpy as np
import isdf_b200 as I
import sim_oracle as S


def hover_state(p, z=1.0):
    x = np.zeros(22)
    x[2] = z
    x[6], x[10], x[14] = 1.0, 1.0, 1.0
    x[18:22] = np.sqrt(p.mass * p.grav / (4 * p.kf))
    return x


def still_trajectory(pos, dur=1.0):
    T = np.array([dur])
    Cc = np.zeros(18)
    Cc[0], Cc[6], Cc[12] = pos
    return np.array([0, 1], dtype=np.int32), T, Cc


def test_default_params_table():
    p = I.sim_default_params()
    assert (p.mass, p.grav, list(p.J), p.kf, p.arm, p.motor_tau, p.min_rpm, p.max_rpm) == \
        (0.98, 9.81, [2.64e-3, 2.64e-3, 4.96e-3], 8.98132e-9, 0.26, 1.0 / 30, 1200, 35000)
    assert p.km == 0.07 * (3 * 0.062) * 8.98132e-9
    assert (p.ctrl_mass, p.ctrl_grav) == (0.98, 9.81)
    assert list(p.kx) == [5.7, 5.7, 6.2] and list(p.kv) == [3.4, 3.4, 4.0]
    assert list(p.kR) == [1.0, 1.0, 1.0] and list(p.kOm) == [0.07, 0.07, 0.1] and list(p.corrections) == [0, 0, 0]
    assert (p.sim_rate, p.cmd_rate, p.t_end, p.log_every, p.use_external_yaw, p.floor, p.reserved_) == (1000, 100, 10, 1, 1, 1, 0)


def test_open_loop_hover_holds_position():
    p = I.sim_default_params()
    x0 = hover_state(p)
    x, cnt, ok = S.open_loop(p, x0, x0[18:22], 10000)
    assert ok and cnt["rollbacks"] == 0 and cnt["rejected"] == 0
    assert np.abs(x[:3] - x0[:3]).max() <= 1e-9


def test_closed_loop_hover_holds_position():
    # the FP32 attitude loop rounds the commanded thrust, so the closed loop holds to its rounding, not to 1e-9
    p = I.sim_default_params(t_end=10.0)
    off, T, Cc = still_trajectory([0.0, 0.0, 1.0])
    init = np.zeros((1, 17)); init[0, 2] = 1.0; init[0, 6] = 1.0; init[0, 13:] = np.sqrt(p.mass * p.grav / (4 * p.kf))
    log, s = S.simulate(off, T, Cc, [0], init, None, p)
    assert s[0]["diverged"] == 0 and s[0]["max_err"] <= 1e-5
    assert np.isfinite(log).all()


def test_constant_force_gives_pd_offset():
    p = I.sim_default_params(t_end=15.0)
    off, T, Cc = still_trajectory([0.0, 0.0, 1.0])
    init = np.zeros((1, 17)); init[0, 2] = 1.0; init[0, 6] = 1.0; init[0, 13:] = np.sqrt(p.mass * p.grav / (4 * p.kf))
    F = np.array([[0.2, -0.1, 0.3, 0.0, 0.0, 0.0]])
    log, s = S.simulate(off, T, Cc, [0], init, F, p)
    offset = log[0, -1, 1:4] - np.array([0.0, 0.0, 1.0])
    pred = F[0, :3] / np.array(list(p.kx))
    assert np.abs(offset - pred).max() <= 2e-4, (offset, pred)


def rk4_reference(p, x0, inp, t_end, h):
    x = x0.copy()
    for _ in range(int(round(t_end / h))):
        k1 = S.rhs(p, x, inp)[0]
        k2 = S.rhs(p, x + 0.5 * h * k1, inp)[0]
        k3 = S.rhs(p, x + 0.5 * h * k2, inp)[0]
        k4 = S.rhs(p, x + h * k3, inp)[0]
        x = x + h / 6 * (k1 + 2 * k2 + 2 * k3 + k4)
    return x


def test_step_controller_rejects_and_stays_accurate():
    p = I.sim_default_params(floor=0)
    x0 = hover_state(p)
    x0[15:18] = [1000.0, -700.0, 300.0]   # a tumbling start: the first tries are rejected
    n = 20
    x, cnt, ok = S.open_loop(p, x0, x0[18:22], n)
    assert ok and cnt["rejected"] > 0 and cnt["accepted"] > n
    ref = rk4_reference(p, x0, x0[18:22], n / p.sim_rate, 1e-5)
    idx = list(range(0, 6)) + list(range(15, 22))
    rel = np.abs(x[idx] - ref[idx]) / np.maximum(1.0, np.abs(ref[idx]))   # |omega| is ~1e3 rad/s here
    assert rel.max() <= 1e-6, rel.max()


def test_floor_clamp():
    p = I.sim_default_params()
    x0 = hover_state(p, z=0.2)
    x, cnt, _ = S.open_loop(p, x0, [0, 0, 0, 0], 1000)
    assert cnt["floor"] > 0 and x[2] == 0.0 and x[5] == 0.0 and cnt["clamped"] == 1000
    p.floor = 0
    x, cnt, _ = S.open_loop(p, x0, [0, 0, 0, 0], 1000)
    assert cnt["floor"] == 0 and x[2] < -1.0


def test_nan_rollback_restores_the_state():
    p = I.sim_default_params(floor=0)
    x0 = hover_state(p)
    x0[3] = np.inf   # inf - inf in the stages gives a NaN state, which the step undoes
    x, cnt, ok = S.open_loop(p, x0, x0[18:22], 1)
    assert ok and cnt["rollbacks"] == 1
    assert np.array_equal(x[:6], x0[:6]) and np.array_equal(x[15:], x0[15:])


def test_get_control_psi_gate_and_clamps():
    p = I.sim_default_params(use_external_yaw=0)
    a = np.deg2rad(120.0)
    R = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    om = np.zeros(3)
    # Psi = 1.5 >= 1: the force is gated off, so the output does not depend on it
    r1 = S.get_control(p, R, om, [0, 0, 9.6], [1, 0, 0, 0])
    r2 = S.get_control(p, R, om, [0, 0, 20.0], [1, 0, 0, 0])
    assert np.array_equal(r1, r2) and (r1 == 0).any()
    # level: Psi = 0, the force passes
    r3 = S.get_control(p, np.eye(3), om, [0, 0, 9.6], [1, 0, 0, 0])
    r4 = S.get_control(p, np.eye(3), om, [0, 0, 20.0], [1, 0, 0, 0])
    assert (r4 > r3).all()
    hover = np.sqrt(9.6 / (4 * p.kf))
    assert np.abs(r3 - hover).max() <= 1e-3 * hover
    # setInput: NaN -> the mean of the limits, then the clamps
    u, cl = S.set_input(p, [np.nan, 1e5, 10.0, 20000.0])
    assert cl and list(u) == [(p.min_rpm + p.max_rpm) / 2, p.max_rpm, p.min_rpm, 20000.0]


def test_drag_lag_on_a_constant_velocity_line():
    # derived from the model alone: at constant velocity v along x the drag 0.1 pi arm^2 v^2 is balanced by the position gain, so the
    # vehicle trails its command by drag / kx (velocity and acceleration errors vanish in steady state)
    p = I.sim_default_params(t_end=12.0, floor=0)
    v = 2.0
    T = np.array([20.0])
    Cc = np.zeros(18)
    Cc[0], Cc[1], Cc[6], Cc[12] = 0.0, v, 0.0, 5.0
    off = np.array([0, 1], dtype=np.int32)
    init = I.sim_init_from_trajectories(off, Cc, [0], p)
    init[0, 3] = v
    log, s = S.simulate(off, T, Cc, [0], init, None, p)
    lag = log[0, -1, 18] - log[0, -1, 1]
    drag = 0.1 * np.pi * p.arm ** 2 * v ** 2
    assert s[0]["diverged"] == 0
    assert abs(lag - drag / p.kx[0]) <= 2e-4 * drag / p.kx[0] + 1e-6, (lag, drag / p.kx[0])
