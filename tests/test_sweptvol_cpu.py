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
