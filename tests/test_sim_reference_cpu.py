"""The closed loop's serial restatement (tests/sim_serial.cpp, line for line the device code csrc/isdf_sim.cuh) against the reference's own
simulator: Quadrotor.cpp, SO3Control.cpp, getControl and the vendored odeint, compiled by oracle/sim.mk into oracle/_ref/libref_sim.so, or
its stored answers tests/golden/sim_reference.npz where the reference tree is absent.

What can separate the two sides: the reference is compiled against oracle/_shim_sim's restatement of Eigen, whose reductions group
additions as Eigen's SSE2 packets do (the thrust sum of four squares as (s0 + s2) + (s1 + s3), where the restatement adds left to right);
both sides call the same libm and round every operation alike. On these cases that grouping changes no bit: right-hand sides, single steps,
setInput and getControl are equal, and the closed-loop logs differ by at most ~1e-15 (one ulp of a sum, carried through the loop). The
tolerances allow one regrouped sum and nothing more. Counts (accepted and rejected tries, clamped steps, floor contacts, rollbacks,
divergence) are exact."""
import numpy as np
import pytest
import isdf_b200 as I
import sim_oracle as S

SUMMARY_FIELDS = [n for n, _ in I.SimSummary._fields_]
COUNTS = ("accepted", "rejected", "clamped_steps", "floor_contacts", "nan_rollbacks", "diverged")
REL_COMPONENT = 1e-15   # one regrouped sum of four positive squares: a few ulp relative (measured: 0)
LOG_TOL = 1e-13         # closed loop over <= 3 s: such ulps carried through the tracking loop's contraction (measured: <= 1e-15)


def params_from(b):
    return I.SimParams.from_buffer_copy(np.asarray(b, dtype=np.uint8).tobytes())


@pytest.fixture(scope="module")
def golden():
    z = np.load(S.GOLDEN)
    return {k: z[k] for k in z.files}


@pytest.fixture(scope="module", params=["golden", "live"])
def ref(request, golden):
    """the reference's answers: the golden file, or the live library recomputing them (which must reproduce the file bit for bit)"""
    if request.param == "golden":
        return golden
    if not S.ref_available():
        pytest.skip("oracle/_ref/libref_sim.so is absent (no reference tree): the golden file stands in")
    out = dict(golden)
    for i, (b, x, r, d) in enumerate(zip(golden["rhs/params"], golden["rhs/x"], golden["rhs/rpm"], golden["rhs/dist"])):
        dx, acc = S.ref_rhs(params_from(b), x, r, d)
        assert np.array_equal(dx.view(np.uint64), golden["rhs/dx"][i].view(np.uint64)), i
    for i, (b, x, r) in enumerate(zip(golden["step/params"], golden["step/x"], golden["step/rpm"])):
        xo, c, ok = S.ref_step(params_from(b), x, r)
        assert ok == golden["step/status"][i] and c["same"] == 1
        assert [c["accepted"], c["rejected"], c["rollbacks"], c["floor"]] == list(golden["step/counts"][i])
        assert np.array_equal(xo.view(np.uint64), golden["step/x_out"][i].view(np.uint64)), i
    for i, (b, u) in enumerate(zip(golden["set_input/params"], golden["set_input/rpm"])):
        assert np.array_equal(S.ref_set_input(params_from(b), u), golden["set_input/input"][i]), i
    for i, (b, R, om, c) in enumerate(zip(golden["get_control/params"], golden["get_control/R"], golden["get_control/omega"], golden["get_control/cmd"])):
        assert np.array_equal(S.ref_get_control(params_from(b), R, om, c[0:3], c[3:7], c[7]), golden["get_control/rpm"][i]), i
    pd = I.sim_default_params()
    for i, v in enumerate(golden["calc/in"]):
        f, q = S.ref_calculate_control(pd, *np.split(v, 6))
        assert np.array_equal(f, golden["calc/force"][i]) and np.array_equal(q, golden["calc/quat"][i]), i
    for name in golden["roll/names"]:
        k = f"roll/{name}/"
        log, summ = S.ref_simulate(golden["traj/off"], golden["traj/T"], golden["traj/C"], golden[k + "traj"], golden[k + "init"],
                                   golden[k + "dist"], params_from(golden[k + "params"]))
        assert np.array_equal(log.view(np.uint64), golden[k + "log"].view(np.uint64)), name
        rows = np.array([[d[f] for f in SUMMARY_FIELDS] for d in summ], dtype=np.float64)
        assert np.array_equal(rows.view(np.uint64), golden[k + "summary"].view(np.uint64)), name
    return out


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.abs(a - b) / np.maximum(np.abs(b), 1e-300)


def test_rhs(ref):
    worst = 0.0
    for b, x, r, d, dx_ref, acc_ref in zip(ref["rhs/params"], ref["rhs/x"], ref["rhs/rpm"], ref["rhs/dist"], ref["rhs/dx"], ref["rhs/acc"]):
        p = params_from(b)
        dx, acc = S.rhs(p, x, S.set_input(p, r)[0], d)
        assert np.array_equal(np.isnan(dx), np.isnan(dx_ref)) and (dx[dx_ref == 0] == 0).all()
        nz = dx_ref != 0
        e = max(rel(dx[nz], dx_ref[nz]).max(initial=0.0), rel(acc[acc_ref != 0], acc_ref[acc_ref != 0]).max(initial=0.0))
        worst = max(worst, e)
    print("worst relative RHS difference:", worst)
    assert worst <= REL_COMPONENT


def test_single_steps(ref):
    kinds = []
    for b, x, r, x_ref, cnt, status in zip(ref["step/params"], ref["step/x"], ref["step/rpm"], ref["step/x_out"], ref["step/counts"],
                                           ref["step/status"]):
        p = params_from(b)
        xs, c, ok = S.open_loop(p, x, r, 1)
        assert ok == (status == 1)
        assert [c["accepted"], c["rejected"], c["rollbacks"], c["floor"]] == list(cnt)
        kinds.append(cnt)
        if not ok:
            continue   # the step gave up: neither side defines the state it leaves
        d = np.where(xs == x_ref, 0.0, np.abs(xs - x_ref) / np.maximum(np.abs(x_ref), 1.0))   # an infinite velocity restored equals itself
        print("step", list(cnt), "max scaled difference", d.max())
        assert d.max() <= REL_COMPONENT
    kinds = np.array(kinds)
    # the cases reach what they are for: rejections, thousands of tries over one step's accepted substeps, a floor contact, a rollback, and
    # the library's bound of 100000 tries in one step (where odeint has none: the wrapper stops it there)
    assert kinds[1, 1] > 0 and kinds[2, 0] + kinds[2, 1] > 1000 and kinds[3, 3] == 1 and kinds[4, 2] == 1
    assert ref["step/status"][5] == -1 and kinds[5, 0] + kinds[5, 1] == 100000


def test_set_input(ref):
    for b, u, want in zip(ref["set_input/params"], ref["set_input/rpm"], ref["set_input/input"]):
        got, _ = S.set_input(params_from(b), u)
        assert np.array_equal(got, want), (u, got, want)


def test_get_control(ref):
    # FP32 as the reference writes it: equal to the bit, every branch of the Psi gate and the external yaw included
    psi_gated = 0
    for b, R, om, c, want in zip(ref["get_control/params"], ref["get_control/R"], ref["get_control/omega"], ref["get_control/cmd"], ref["get_control/rpm"]):
        got = S.get_control(params_from(b), R, om, c[0:3], c[3:7], c[7])
        assert np.array_equal(got, want), (R, got, want)
        psi_gated += got.min() == 0
    assert psi_gated > 0


def test_calculate_control(ref):
    # the position loop in FP64, the limit at theta = pi/2 (the source's "45 degree" comment notwithstanding) on both sides included: it
    # fires when the commanded force points at or below the horizon and then scales its deviation from m g e3 so that the force lies on
    # the horizon (vertical part 0 up to rounding)
    p = I.sim_default_params()
    mg = p.ctrl_mass * p.ctrl_grav
    limited = []
    for v, f_ref, q_ref in zip(ref["calc/in"], ref["calc/force"], ref["calc/quat"]):
        f, q = S.calculate_control(p, *np.split(v, 6))
        assert np.array_equal(f, f_ref) and np.array_equal(q, q_ref), (f, f_ref, q, q_ref)
        limited.append(bool(abs(f_ref[2]) <= 1e-6 * mg and np.abs(f_ref[:2]).max() > 0))
    assert limited == [False, True, True, False, True]


def summaries(ref, name):
    return [dict(zip(SUMMARY_FIELDS, row)) for row in ref[f"roll/{name}/summary"]]


@pytest.mark.parametrize("name", ["default", "vehicle", "ratio1", "ratio20", "floor", "gust", "hold", "rollback"])
def test_rollouts(ref, name):
    k = f"roll/{name}/"
    p = params_from(ref[k + "params"])
    log, summ = S.simulate(ref["traj/off"], ref["traj/T"], ref["traj/C"], ref[k + "traj"], ref[k + "init"], ref[k + "dist"], p)
    rlog, rsumm = ref[k + "log"], summaries(ref, name)
    assert np.array_equal(np.isnan(log), np.isnan(rlog))
    fin = np.isfinite(rlog)
    err = np.abs(log[fin] - rlog[fin]).max()
    print(name, "max |serial - reference| over the log:", err)
    assert err <= LOG_TOL
    for a, b in zip(summ, rsumm):
        for c in COUNTS:
            assert a[c] == b[c], (c, a[c], b[c])
        for c in ("max_err", "rms_err", "final_err", "max_tilt", "max_omega", "t_max_err", "t_diverged"):
            assert (np.isnan(a[c]) and np.isnan(b[c])) or abs(a[c] - b[c]) <= LOG_TOL, (c, a[c], b[c])
    # each case reaches its branch
    if name == "floor":
        assert all(s["floor_contacts"] > 0 and s["clamped_steps"] > 0 for s in rsumm)
    if name == "rollback":
        assert rsumm[0]["nan_rollbacks"] == 0 and rsumm[1]["nan_rollbacks"] == rsumm[1]["accepted"] > 0 and rsumm[1]["diverged"] == 0
    if name == "gust":
        assert rsumm[1]["diverged"] == 1 and rsumm[0]["diverged"] == 0
    if name == "hold":
        n, d = ref["traj/off"], ref["traj/T"]
        durs = [d[n[b]:n[b + 1]].sum() for b in range(len(n) - 1)]
        assert rlog[0, -1, 0] > max(durs)
