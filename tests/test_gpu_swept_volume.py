"""Certified swept volume (isdf_swept_volume_*) on the GPU: the enclosure [lower, value] against the exact SV of Point and Ball and the
dense references of Box and a box mesh; bit identity across entry points, grid nodes and repeated calls; the marching-tetrahedra mesh
against its NumPy restatement, closed and oriented on a capsule, near the zero set and of the right volume on a curved path; the
reference's local search against the certified lower bound; refusals and state isolation."""
import ctypes as C
import math
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W
import certify_oracle as CE
import sweptvol_oracle as SO

pytestmark = pytest.mark.gpu
BOX_HALF = [0.9, 0.5, 0.3]


def make_ev(K=8):
    cfg = I.default_config_values()
    cfg.integral_intervs = K
    return I.Evaluator(cfg), cfg


def box_mesh(h):
    V = np.array([[sx * h[0], sy * h[1], sz * h[2]] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], float)
    F = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4],
                  [1, 5, 7], [1, 7, 3]], dtype=np.int32)
    return V, F


def traj(seed=4, n=3):
    return W.make_trajectory(n, [0, 0, 0], [6, 4, 3], seed=seed, jitter=0.4)[:2]


def path_points(T, Cc, rng, m):
    """points on, near and away from the path, and near the junctions"""
    Cm = np.asarray(Cc).reshape(3, -1)
    N = len(T)
    out = []
    for k in range(m):
        i = int(rng.integers(N))
        t = T[i] if k % 5 == 0 else rng.uniform(0, T[i])
        x = Cm[:, 6 * i:6 * i + 6] @ (t ** np.arange(6))
        out.append(x + rng.normal(size=3) * [0.0, 0.05, 0.3, 1.0, 3.0][k % 5])
    return np.array(out)


# ---- exactness: Point and Ball against the root-based SV ----------------------------------------------------------------------------
@pytest.mark.parametrize("shape,radius", [("Point", 0.0), ("Ball", 1.0)])
def test_exact_point_and_ball(shape, radius):
    ev, cfg = make_ev()
    ev.set_shape_named(shape)
    rng = np.random.default_rng(7)
    ndec = 0
    for seed in (4, 5):
        T, Cc = traj(seed)
        P = path_points(T, Cc, rng, 40)
        p = ev.swept_params(tol=1e-4)
        v, lo, ts, dec = ev.swept_volume_sdf(T, Cc, P, p)
        for k in range(len(P)):
            ex = SO.exact_sv_point(T, Cc, P[k], radius)
            assert lo[k] <= ex + 1e-9, (k, lo[k], ex)
            assert v[k] >= min(ex, p.band) - 1e-9, (k, v[k], ex)
            if dec[k]:
                ndec += 1
                assert v[k] - lo[k] <= p.tol, (k, v[k], lo[k])
    assert ndec >= 40


# ---- Box and a closed box mesh of the same geometry: dense references ---------------------------------------------------------------
def test_box_and_box_mesh_dense():
    T, Cc = traj(6)
    rng = np.random.default_rng(3)
    P = path_points(T, Cc, rng, 6)
    res = {}
    for kind in ("box", "mesh"):
        ev, cfg = make_ev()
        if kind == "box":
            ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], BOX_HALF)
        else:
            V, F = box_mesh(BOX_HALF)
            ev.set_shape_mesh(V, F, None, I.MESH_SIGN_EXACT)
        p = ev.swept_params(tol=1e-3)
        res[kind] = ev.swept_volume_sdf(T, Cc, P, p)
    f = SO.box_sdf(BOX_HALF)
    r = CE.body_radius(CE.box_corners(BOX_HALF))
    toff = np.concatenate([[0.0], np.cumsum(T)[:-1]])
    for kind in ("box", "mesh"):
        v, lo, ts, dec = res[kind]
        for k in range(len(P)):
            d, _ = SO.dense_sv(cfg, T, Cc, P[k], f)
            dl = SO.dense_lower(cfg, T, Cc, P[k], f, r, p.band, n=32)
            assert lo[k] <= d + 1e-9 and min(d, p.band) <= v[k] + 1e-9 + (0 if dec[k] else math.inf), (kind, k, lo[k], d, v[k])
            assert min(dl, p.band) <= v[k] + 1e-9, (kind, k, dl, v[k])   # value is capped at band
            if v[k] < p.band:   # value is attained at t*
                i = int(np.searchsorted(toff, ts[k], side="right") - 1)
                sd = SO._sd(cfg, T, Cc, [i], [ts[k] - toff[i]], P[k], f)[0]
                assert abs(sd - v[k]) <= 1e-12, (kind, k, sd, v[k])
    both = res["box"][3].astype(bool) & res["mesh"][3].astype(bool)
    assert both.sum() >= 4
    assert np.abs(res["box"][0] - res["mesh"][0])[both].max() <= p.tol + 1e-9


# ---- consistency ------------------------------------------------------------------------------------------------------------------------
def test_bit_identity_points_grid_device():
    import torch
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = traj(4)
    p = ev.swept_params()
    g = I.swept_grid_for(T, Cc, 1.0, p.band, 0.4)
    v, lo, ts, dec, info = ev.swept_volume_grid(T, Cc, g, p)
    assert info["nodes"] == g.X * g.Y * g.Z and 0 < info["bricks_culled"] < info["bricks"]
    v2, lo2, ts2, dec2, _ = ev.swept_volume_grid(T, Cc, g, p)
    for a, b in ((v, v2), (lo, lo2), (ts, ts2), (dec, dec2)):
        assert np.array_equal(a, b)
    nodes = I.swept_grid_nodes(g).reshape(-1, 3)
    rng = np.random.default_rng(1)
    sel = np.concatenate([np.flatnonzero(v.reshape(-1) < p.band)[::7], rng.integers(0, nodes.shape[0], 200)])
    pv, plo, pts_, pdec = ev.swept_volume_sdf(T, Cc, nodes[sel], p)
    assert np.array_equal(pv, v.reshape(-1)[sel]) and np.array_equal(plo, lo.reshape(-1)[sel])
    assert np.array_equal(pts_, ts.reshape(-1)[sel]) and np.array_equal(pdec, dec.reshape(-1)[sel])
    n = g.X * g.Y * g.Z
    dT, dC = torch.from_numpy(np.ascontiguousarray(T)).cuda(), torch.from_numpy(np.ascontiguousarray(Cc)).cuda()
    dv, dl, dt = (torch.zeros(n, dtype=torch.float64, device="cuda") for _ in range(3))
    dd = torch.zeros(n, dtype=torch.uint8, device="cuda")
    ev.swept_volume_grid_device(len(T), dT.data_ptr(), dC.data_ptr(), g, p, dv.data_ptr(), dl.data_ptr(), dt.data_ptr(), dd.data_ptr(),
                                stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(dv.cpu().numpy(), v.reshape(-1)) and np.array_equal(dl.cpu().numpy(), lo.reshape(-1))
    assert np.array_equal(dt.cpu().numpy(), ts.reshape(-1)) and np.array_equal(dd.cpu().numpy(), dec.reshape(-1))


def test_bit_identity_mesh_robot():
    ev, cfg = make_ev()
    V, F = W.rounded_cone_mesh(n_theta=16, n_prof=12)
    ev.set_shape_mesh(V, F, None, I.MESH_SIGN_EXACT)
    T, Cc = traj(5, 2)
    p = ev.swept_params(max_samples=64)
    g = I.swept_grid_for(T, Cc, 2.5, p.band, 0.5)
    v, lo, ts, dec, _ = ev.swept_volume_grid(T, Cc, g, p)
    v2, lo2, _, _, _ = ev.swept_volume_grid(T, Cc, g, p)
    assert np.array_equal(v, v2) and np.array_equal(lo, lo2)
    assert (v < 0).any() and (lo <= v).all()
    nodes = I.swept_grid_nodes(g).reshape(-1, 3)
    sel = np.flatnonzero(v.reshape(-1) < p.band)[::11]
    pv, plo, _, _ = ev.swept_volume_sdf(T, Cc, nodes[sel], p)
    assert np.array_equal(pv, v.reshape(-1)[sel]) and np.array_equal(plo, lo.reshape(-1)[sel])


# ---- mesh -------------------------------------------------------------------------------------------------------------------------------
def test_mesh_matches_restatement():
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = traj(4, 2)
    p = ev.swept_params()
    g = I.swept_grid_for(T, Cc, 1.0, p.band, 0.6)
    v, lo, ts, dec, _ = ev.swept_volume_grid(T, Cc, g, p)
    V, vt, F, info = ev.swept_volume_mesh(T, Cc, g, p)
    RV, Rvt, RF = SO.marching_tets(v, ts, list(g.bmin), g.res)
    assert len(F) > 0 and info["mesh_ms"] > 0
    assert np.array_equal(V, RV) and np.array_equal(vt, Rvt) and np.array_equal(F, RF)


def line(a, b, Tt):
    """one piece moving from a to b at constant velocity over Tt"""
    c = np.zeros((3, 6))
    c[:, 0] = a
    c[:, 1] = (np.asarray(b, float) - np.asarray(a, float)) / Tt
    return np.array([Tt]), c.reshape(-1)


def test_capsule_closed_oriented():
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = line([0.1, 0.2, 0.3], [4.1, 1.2, 0.8], 2.0)
    p = ev.swept_params()
    g = I.swept_grid_for(T, Cc, 1.0, p.band, 0.25)
    V, vt, F, _ = ev.swept_volume_mesh(T, Cc, g, p)
    chk = SO.mesh_checks(V, F)
    assert chk["manifold"] and chk["oriented"] and chk["euler"] == 2, chk
    L = np.linalg.norm([4.0, 1.0, 0.5])
    exact = math.pi * L + 4.0 / 3.0 * math.pi
    assert abs(chk["volume"] - exact) < 0.05 * exact, (chk["volume"], exact)
    assert (vt >= 0).all() and (vt <= 2.0).all()


def test_curved_mesh_near_zero_and_volume():
    ev, cfg = make_ev()
    ev.set_shape_named("Ball")
    T, Cc = traj(5, 3)
    p = ev.swept_params()
    res = 0.25
    g = I.swept_grid_for(T, Cc, 1.0, p.band, res)
    V, vt, F, _ = ev.swept_volume_mesh(T, Cc, g, p)
    chk = SO.mesh_checks(V, F)
    assert chk["manifold"] and chk["oriented"], chk
    rng = np.random.default_rng(2)
    for k in rng.choice(len(V), size=min(150, len(V)), replace=False):
        assert abs(SO.exact_sv_point(T, Cc, V[k], 1.0)) <= res * math.sqrt(3) + p.tol, k
    # Monte Carlo volume of {SV < 0} in the grid box, from the certified point query
    lo = np.array(g.bmin[:]); hi = lo + res * (np.array([g.X, g.Y, g.Z]) - 1)
    Q = lo + rng.random((200000, 3)) * (hi - lo)
    v, _, _, _ = ev.swept_volume_sdf(T, Cc, Q, p)
    box = float(np.prod(hi - lo))
    frac = float(np.mean(v < 0))
    vmc, sig = frac * box, math.sqrt(frac * (1 - frac) / len(Q)) * box
    P = np.asarray(V); tri = F
    area = 0.5 * np.linalg.norm(np.cross(P[tri[:, 1]] - P[tri[:, 0]], P[tri[:, 2]] - P[tri[:, 0]]), axis=1).sum()
    # linear interpolation of a 1-Lipschitz field moves the surface by at most res: |dV| <= res * area
    print(f"curved: mesh volume {chk['volume']:.4f}, Monte Carlo {vmc:.4f} +- {sig:.4f}, area {area:.3f}")
    assert abs(chk["volume"] - vmc) <= res * area + 4 * sig


# ---- against the reference's local search -------------------------------------------------------------------------------------------
def test_lower_below_reference_search():
    cfg = I.default_config_values()
    cfg.integral_intervs = 16
    ev = I.Evaluator(cfg)
    occ = W.three_slit_map(64, 64, 64, noise=0.03, seed=1)
    T, Cc, wp = W.make_trajectory(4, [0, 0, 0], [50, 50, 34], seed=3, jitter=0.3)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    pts = W.gather_obstacle_points(occ, [0, 0, 0], 1.0, wp, cfg.kernel_size * cfg.occupancy_resolution / 3.0)[:400]
    ev.set_points(pts)
    ev.eval_swept(T, Cc)
    _, sdf, _ = ev.swept_results()
    p = ev.swept_params(band=50.0, tol=1e-6)
    v, lo, ts, dec = ev.swept_volume_sdf(T, Cc, pts, p)
    assert (lo <= sdf + 1e-9).all(), np.max(lo - sdf)
    miss = int(np.sum(sdf > v + p.tol))
    print(f"reference search ends above value + tol at {miss} of {len(pts)} obstacle points")


# ---- contract -----------------------------------------------------------------------------------------------------------------------
def call_sdf(ev, T, Cc, pts, p):
    n = len(pts)
    v = np.zeros(max(n, 1))
    P = np.ascontiguousarray(pts, dtype=np.float64).reshape(-1, 3)
    r = ev.lib.isdf_swept_volume_sdf(ev.h, len(T), I._dp(np.ascontiguousarray(T, float)), I._dp(np.ascontiguousarray(Cc, float)),
                                     C.byref(p) if p is not None else None, n, I._dp(P), I._dp(v), None, None, None)
    return r, v


def test_errors_and_state():
    ev, cfg = make_ev()
    T, Cc = traj(4)
    P = np.zeros((3, 3))
    p = ev.swept_params()
    assert call_sdf(ev, T, Cc, P, p)[0] == -2                     # no shape (and no map: none needed)
    ev.set_shape_named("Torus")
    r, v = call_sdf(ev, T, Cc, P, p)
    assert r == -4 and np.isnan(v).all()
    ev.set_shape_named("Ball")
    assert call_sdf(ev, T, Cc, P, None)[0] == -1
    for field, bad in (("samples_per_piece", 0), ("tol", 0.0), ("band", p.tol), ("max_depth", 65), ("max_samples_per_point", -1),
                       ("reserved_", 1)):
        q = ev.swept_params()
        setattr(q, field, bad)
        assert call_sdf(ev, T, Cc, P, q)[0] == -1, field
    Tb = np.array(T, float); Tb[1] = -1.0
    assert call_sdf(ev, Tb, Cc, P, p)[0] == -1
    Cb = np.array(Cc, float); Cb[5] = np.nan
    assert call_sdf(ev, T, Cb, P, p)[0] == -1
    g = I.swept_grid_for(T, Cc, 1.0, p.band, 0.5)
    for field, bad in (("X", 1), ("res", 0.0), ("reserved_", 2)):
        gb = I.swept_grid_for(T, Cc, 1.0, p.band, 0.5)
        setattr(gb, field, bad)
        with pytest.raises(I.IsdfError) as e:
            ev.swept_volume_grid(T, Cc, gb, p)
        assert e.value.code == -1
    V, F = W.rounded_cone_mesh(n_theta=16, n_prof=12)
    ev.set_shape_mesh(V, F, None, I.MESH_SIGN_WINDING)
    assert call_sdf(ev, T, Cc, P, p)[0] == -4
    ev.set_shape_named("Ball")
    # small caps: INVALID with the counts written
    nV, nF = C.c_int64(0), C.c_int64(0)
    r = ev.lib.isdf_swept_volume_mesh(ev.h, len(T), I._dp(np.ascontiguousarray(T, float)), I._dp(np.ascontiguousarray(Cc, float)),
                                      C.byref(p), C.byref(g), 0, 0, None, None, None, C.byref(nV), C.byref(nF), None)
    assert r == -1 and nV.value > 0 and nF.value > 0
    # state: only kernel_launches moves; the swept-volume term's results stay
    pts = np.array([[1.0, 1.0, 1.0], [2.0, 0.5, 0.2]])
    ev.set_points(pts)
    ev.eval_swept(T, Cc)
    before = ev.swept_results()
    s0 = ev.stats()
    ev.swept_volume_grid(T, Cc, g, p)
    ev.swept_volume_mesh(T, Cc, g, p)
    s1 = ev.stats()
    after = ev.swept_results()
    for a, b in zip(before, after):
        assert np.array_equal(a, b)
    assert s1.kernel_launches > s0.kernel_launches
    for f, _ in I.Stats._fields_:
        if f != "kernel_launches":
            assert getattr(s1, f) == getattr(s0, f), f
    ev.set_shard(0, 2)
    assert call_sdf(ev, T, Cc, P, p)[0] == -4
