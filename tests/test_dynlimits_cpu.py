"""CPU-only checks of the dynamic-limit certificate's restatement (tests/dynlimits_oracle.py): its enclosures against dense reference
values on aggressive pieces, their convergence, the refinement against exact polynomial maxima of |v| and |a|, the thrust against the
reference-compiled FlatnessMap::forward's golden, and the C ABI's layouts and defaults without a GPU."""
import ctypes as C
import math
import os
import numpy as np
import pytest
import isdf_b200 as I
import dynlimits_oracle as DO
import oracle_lib as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flat_forward_reference.npz")


def cfg_with(drag, veps=1e-4):
    cfg = I.default_config_values()
    if not drag:
        cfg.horiz_drag = cfg.vert_drag = cfg.paras_drag = 0.0
    cfg.speed_eps = veps
    return cfg


def aggressive_pieces():
    """(name, T (1,), coeffs (18,)) single pieces: hover through zero speed, an 80-degree tilt with large jerk, random quintics"""
    g = 9.8
    out = []
    c = np.zeros((3, 6)); c[:, 0] = [1.0, 2.0, 3.0]; c[0, 1] = -1.0; c[0, 2] = 1.0
    out.append(("through_rest", 1.0, c))
    c = np.zeros((3, 6)); c[0, 2] = 0.5 * g * math.tan(math.radians(80.0)); c[0, 3] = 40.0; c[1, 3] = -30.0; c[2, 1] = 1.0
    out.append(("tilt80_jerk", 0.25, c))
    rng = np.random.default_rng(3)
    for k in range(4):
        c = rng.normal(0, 1, (3, 6)) * np.array([5, 4, 3, 2, 1.5, 1.0])
        out.append((f"random{k}", 0.6 + 0.2 * k, c))
    return [(n, np.array([T]), c.reshape(-1)) for n, T, c in out]


def params(**kw):
    p = I.DynamicsParams()
    I.load_library().isdf_dynamics_default_params(None, C.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("drag", [True, False])
@pytest.mark.parametrize("veps", [1e-4, 0.0])
def test_enclosures_contain_dense_reference_values(drag, veps):
    cfg = cfg_with(drag, veps)
    checked = 0
    for name, T, Cc in aggressive_pieces():
        c = DO.piece_coeffs(Cc, 1)
        for K in (8, 32):
            edges = np.linspace(0.0, T[0], K + 1)
            ta, tb = edges[:-1], edges[1:]
            te = ta + 0.5 * (tb - ta)
            h = np.fmax(tb - te, te - ta)
            lo, hi = DO.enclose(cfg, np.repeat(c, K, 0), te, h)
            for k in range(K):
                t = np.linspace(ta[k], tb[k], 2001)
                vals, cz = DO.dense(cfg, T, Cc, 0, t)
                for q in range(5):
                    if not np.isfinite(hi[k, q]):
                        continue
                    tolq = 1e-9 * max(1.0, np.nanmax(np.abs(vals[:, q])))
                    if q == 3:   # acos is ill-conditioned at 0: compare through cos(theta)
                        assert np.all(cz <= math.cos(min(lo[k, 3], math.pi)) + 1e-12), (name, K, k)
                        assert np.all(cz >= math.cos(min(hi[k, 3], math.pi)) - 1e-12), (name, K, k)
                        continue
                    x = vals[np.isfinite(vals[:, q]), q]   # the reference's 0/0 at exactly zero speed with speed_eps = 0 is NaN
                    assert x.size >= 2000 and x.max() <= hi[k, q] + tolq, (name, K, k, q)
                    assert x.min() >= lo[k, q] - tolq, (name, K, k, q)
                    checked += 1
                assert np.nanmin(vals[:, 4]) >= -hi[k, 5] - 1e-9 * max(1.0, np.nanmax(np.abs(vals[:, 4])))
    assert checked >= 900


@pytest.mark.parametrize("drag", [True, False])
def test_enclosure_width_shrinks_at_least_linearly(drag):
    cfg = cfg_with(drag)
    for name, T, Cc in aggressive_pieces():
        c = DO.piece_coeffs(Cc, 1)
        te = np.full(8, 0.37 * T[0])
        h = 0.05 * T[0] * 0.5 ** np.arange(8)
        lo, hi = DO.enclose(cfg, np.repeat(c, 8, 0), te, h)
        w = hi - lo
        for q in range(5):
            if not np.all(np.isfinite(w[:, q])) or w[0, q] < 1e-9:
                continue
            ratio = w[3:, q] / w[2:-1, q]
            assert np.all(ratio <= 0.55), (name, q, ratio)


@pytest.mark.parametrize("drag", [True, False])
def test_refinement_brackets_exact_polynomial_maxima(drag):
    cfg = cfg_with(drag)
    p = params(samples_per_piece=16, max_depth=30, max_samples_per_traj=100000)
    for name, T, Cc in aggressive_pieces():
        summ, _ = DO.certify(cfg, T, Cc, p)
        s = summ[0]
        vm, am = DO.poly_max_va(T, Cc, 0)
        for q, m, tol in ((0, vm, p.tol_v), (1, am, p.tol_a)):
            assert s["attained"][q] <= m * (1 + 1e-14) and m <= s["upper"][q] * (1 + 1e-14), (name, q, s["attained"][q], m, s["upper"][q])
            assert s["upper"][q] - s["attained"][q] <= tol, (name, q)


def test_oracle_thrust_equals_reference_compiled_golden():
    g = np.load(GOLDEN)
    for tag, drag in (("drag", True), ("nodrag", False)):
        cfg = cfg_with(drag)
        par = np.array([cfg.vehicle_mass, cfg.grav_acc, cfg.horiz_drag, cfg.vert_drag, cfg.paras_drag, cfg.speed_eps])
        assert np.array_equal(par, g[f"{tag}_par"])
        v, a, j = (g[f"{tag}_{x}"] for x in "vaj")
        lo, hi = DO.channels(cfg, [DO.Iv(v[:, k]) for k in range(3)], [DO.Iv(a[:, k]) for k in range(3)], [DO.Iv(j[:, k]) for k in range(3)])
        ref = g[f"{tag}_thr"]
        scale = np.maximum(np.abs(ref), 1.0)
        assert np.max(np.abs(lo[:, 4] - ref) / scale) <= 1e-12 and np.max(np.abs(hi[:, 4] - ref) / scale) <= 1e-12
        # the dense reference's thrust is the same function
        assert np.max(np.abs(DO.thrust_exact(cfg, v, a) - ref) / scale) <= 1e-12
        # the golden's body rate is the reference-compiled optimizated_forward's: the fixture and oracle/_ref agree
        _, o = O.RefFlat(cfg).forward(v, a, j)
        assert np.max(np.abs(o - g[f"{tag}_omg"]) / np.maximum(np.abs(g[f"{tag}_omg"]), 1.0)) <= 1e-12


def test_layouts_and_defaults_without_gpu():
    assert C.sizeof(I.DynamicsParams) == 112 and C.sizeof(I.DynamicsSummary) == 168
    assert I.DynamicsParams.vmax.offset == 16 and I.DynamicsParams.tol_v.offset == 64 and I.DynamicsParams.reserved_.offset == 104
    assert I.DynamicsSummary.thrust_lower.offset == 120 and I.DynamicsSummary.verdict.offset == 144 and I.DynamicsSummary.depth.offset == 164
    lib = I.load_library()
    for s in ("isdf_dynamics_default_params", "isdf_trajectory_dynamics", "isdf_trajectory_dynamics_device"):
        assert hasattr(lib, s)
    p = I.DynamicsParams()
    assert lib.isdf_dynamics_default_params(None, C.byref(p)) == 0
    d = I.default_config_values()
    assert (p.samples_per_piece, p.pieces_per_traj, p.max_depth, p.max_samples_per_traj) == (d.integral_intervs, 0, 16, 2048)
    assert (p.vmax, p.omgmax, p.thetamax) == (d.vmax, d.omgmax, d.thetamax)
    assert p.amax == math.inf and p.thrust_max == math.inf and p.thrust_min == -math.inf
    assert (p.tol_v, p.tol_a, p.tol_omg, p.tol_theta, p.tol_thrust) == (1e-3, 1e-3, 1e-3, 1e-4, 1e-3)
    assert list(p.reserved_) == [0, 0]
    assert lib.isdf_dynamics_default_params(None, None) == I.IsdfError(-1, "").code
    # argument checks run before any device work: a NULL context is refused without touching a GPU
    s = (I.DynamicsSummary * 1)()
    T, Cc = np.ones(1), np.zeros(18)
    assert lib.isdf_trajectory_dynamics(None, 1, I._dp(T), I._dp(Cc), C.byref(p), s) == -1
    assert s[0].verdict == 0 and math.isnan(s[0].upper[0]) and s[0].samples == -1
