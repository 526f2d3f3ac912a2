"""CPU checks of the swept-volume references (tests/sweptvol_oracle.py): the marching-tetrahedra restatement on an analytic sphere field
is closed, oriented, of Euler characteristic 2, and its volume converges to 4/3 pi r^3; the root-based SV of a Ball agrees with dense
sampling."""
import math
import numpy as np
import pytest
import workloads as W
import sweptvol_oracle as SO


def sphere_field(res, r=1.0, c=(0.013, -0.021, 0.007)):
    n = int(math.ceil(2.6 * r / res)) + 2
    bmin = np.array(c) - 1.3 * r - res
    ax = [bmin[a] + np.arange(n) * res for a in range(3)]
    P = np.stack(np.meshgrid(*ax, indexing="ij"), -1)
    return np.linalg.norm(P - np.array(c), axis=-1) - r, bmin


def test_mt_sphere_closed_oriented():
    f, bmin = sphere_field(0.25)
    V, vt, F = SO.marching_tets(f, None, bmin, 0.25)
    chk = SO.mesh_checks(V, F)
    assert chk["manifold"] and chk["oriented"] and chk["euler"] == 2, chk
    assert chk["volume"] > 0   # normals toward increasing value: outward


def test_mt_sphere_volume_converges():
    errs = []
    for res in (0.4, 0.2, 0.1):
        f, bmin = sphere_field(res)
        V, _, F = SO.marching_tets(f, None, bmin, res)
        errs.append(abs(SO.mesh_checks(V, F)["volume"] - 4.0 / 3.0 * math.pi))
    assert errs[2] < errs[1] < errs[0] and errs[2] < 0.05, errs


def test_mt_vertex_times_and_positions():
    f, bmin = sphere_field(0.5)
    ts = np.arange(f.size, dtype=float).reshape(f.shape)
    V, vt, F = SO.marching_tets(f, ts, bmin, 0.5)
    assert len(V) == len(vt) and F.max() < len(V)
    # every vertex lies on the sphere up to linear interpolation error
    assert np.abs(np.linalg.norm(V - np.array((0.013, -0.021, 0.007)), axis=1) - 1.0).max() < 0.2


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_ball_exact_matches_dense(seed):
    T, Cc, _ = W.make_trajectory(3, [0, 0, 0], [6, 4, 3], seed=seed, jitter=0.4)
    rng = np.random.default_rng(seed)
    Cm = np.asarray(Cc).reshape(3, -1)
    for _ in range(6):
        i = rng.integers(3)
        t = rng.uniform(0, T[i])
        x = Cm[:, 6 * i:6 * i + 6] @ (t ** np.arange(6))
        p = x + rng.normal(size=3) * rng.choice([0.1, 1.0, 3.0])
        ex = SO.exact_sv_point(T, Cc, p, 0.5)
        dense = math.inf
        for k in range(3):
            tt = np.linspace(0, T[k], 20001)
            X = (Cm[:, 6 * k:6 * k + 6] @ (tt[None, :] ** np.arange(6)[:, None])).T
            dense = min(dense, float(np.linalg.norm(X - p, axis=1).min()) - 0.5)
        assert ex <= dense + 1e-12 and dense - ex < 1e-6, (ex, dense)


# ---- the refinement's restatement (sv_refine) --------------------------------------------------------------------------------------
class Params:
    """the fields of isdf_swept_params that sv_refine reads"""
    def __init__(self, K=8, max_depth=16, max_samples=512, tol=1e-3, band=1.732):
        self.samples_per_piece, self.max_depth, self.max_samples_per_point, self.tol, self.band = K, max_depth, max_samples, tol, band


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_sv_refine_encloses_exact_ball(seed):
    """the restated refinement with the Ball SDF: lower <= SV <= value against the root-based SV, value attained at t*, and decided
    points within tol, on the trajectories of test_ball_exact_matches_dense"""
    import isdf_b200 as I
    import certify_oracle as CE
    T, Cc, _ = W.make_trajectory(3, [0, 0, 0], [6, 4, 3], seed=seed, jitter=0.4)
    cfg = I.default_config_values()
    radius = 0.5
    prm = Params(K=4, tol=1e-3)
    ball = lambda q: np.linalg.norm(q, axis=1) - radius
    prep = SO.SvPrep(cfg, T, Cc, 0.0, prm)
    rng = np.random.default_rng(seed)
    Cm = np.asarray(Cc).reshape(3, -1)
    toff = np.concatenate([[0.0], np.cumsum(T)[:-1]])
    ndec = nin = 0
    for _ in range(12):
        i = rng.integers(3)
        t = rng.uniform(0, T[i])
        p = Cm[:, 6 * i:6 * i + 6] @ (t ** np.arange(6)) + rng.normal(size=3) * rng.choice([0.1, 1.0, 3.0])
        r = SO.sv_refine(cfg, T, Cc, p, ball, 0.0, radius, prm, prep)
        ex = SO.exact_sv_point(T, Cc, p, radius)
        assert r["lower"] <= ex + 1e-9 and r["value"] >= min(ex, prm.band) - 1e-9, (r, ex)
        if r["value"] < prm.band:
            nin += 1
            k = int(np.searchsorted(toff, r["tstar"], side="right") - 1)
            pos, _ = CE.pose_at(cfg, T, Cc, [k], [r["tstar"] - toff[k]])
            assert abs(np.linalg.norm(p - pos[0]) - radius - r["value"]) <= 1e-12
        else:
            assert r["tstar"] == -1.0
        if r["decided"]:
            ndec += 1
            assert r["value"] - r["lower"] <= prm.tol
    assert ndec >= 8 and nin >= 4, (ndec, nin)


# ---- the vectorised marching tetrahedra against the loop ---------------------------------------------------------------------------
def _same_mesh(f, ts, bmin, res):
    a = SO.marching_tets(f, ts, bmin, res)
    b = SO.marching_tets_np(f, ts, bmin, res)
    for x, y in zip(a, b):
        assert x.shape == y.shape and np.array_equal(x, y)
    return a


@pytest.mark.parametrize("res", [0.5, 0.25])
def test_mt_np_matches_loop_on_spheres(res):
    f, bmin = sphere_field(res)
    ts = np.arange(f.size, dtype=float).reshape(f.shape) * 0.01
    V, _, F = _same_mesh(f, ts, bmin, res)
    assert len(F) > 100


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_mt_np_matches_loop_on_random_fields(seed):
    """random fields with exact zeros (outside: value < 0 is inside) and band-capped values whose t* is -1; odd sizes and a cut
    border"""
    rng = np.random.default_rng(seed)
    shp = tuple(int(x) for x in rng.integers(2, 9, 3))
    band = 0.7
    f = rng.normal(size=shp)
    f[rng.random(shp) < 0.2] = 0.0
    f[rng.random(shp) < 0.2] = -0.0
    cap = rng.random(shp) < 0.3
    f[cap] = band
    ts = np.where(cap, -1.0, rng.random(shp) * 10)
    V, vt, F = _same_mesh(f, ts, rng.normal(size=3), 0.37)
    assert F.size == 0 or F.max() < len(V)


# ---- the pose pad at swept-volume distances -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("band", [1.732, 20.0])
def test_pose_pad_covers_swept_volume_distances(band):
    """the swept volume evaluates points up to rho = band + r_body + D_e from x(t_e) with H = band: the position error plus rho times
    the rotation error of the double pose against an extended-precision one stays below eps_e / 1000, on the aggressive pieces of the
    certificate's CPU test, for every initial interval at K in {1, 3, 8, 64} with a finite bound (the bench cone's r_body)"""
    import isdf_b200 as I
    import certify_oracle as CE
    from test_certify_cpu import aggressive_pieces
    cfg = I.default_config_values()
    V, _ = W.rounded_cone_mesh(n_theta=24, n_prof=16)
    lo, hi = V.min(axis=0), V.max(axis=0)
    r = CE.body_radius([[hi[0] if k & 1 else lo[0], hi[1] if k & 2 else lo[1], hi[2] if k & 4 else lo[2]] for k in range(8)])
    far = 0.0
    for name, T, Cc in aggressive_pieces():
        c = CE.piece_coeffs(Cc, 1, 0)
        for K in (1, 3, 8, 64):
            for j in range(K):
                ta, tb = j * (T[0] * (1.0 / K)), (T[0] if j + 1 == K else (j + 1) * (T[0] * (1.0 / K)))
                for te in (ta, tb):
                    D = CE.bound(cfg, r, band, c, ta, tb, te)
                    if not D < math.inf:
                        continue
                    rho = band + r + D
                    p64, R64 = CE.pose_at(cfg, T, Cc, [0], [te])
                    pl, Rl = CE.pose_closed_form(cfg, c, te, np.longdouble)
                    err = float(np.abs(p64[0] - pl.astype(float)).max() + rho * np.abs(R64[0] - Rl.astype(float)).max())
                    assert err * 1e3 <= CE.eps_pad(cfg, r, band, c, te), (name, K, j, te, err)
                    far = max(far, rho / (r + 2 * band))
    assert far >= 10.0, far   # the distances reach well past the r + 2H the pad was derived for
