"""The grazing fixtures (tests/grazing.py) checked against the oracle alone: every occupied voxel's minimum-over-samples SDF lies in
its band, the active count and the fixture's own cost match the oracle, and removing any sampled active voxel moves the oracle cost
by at least 100x the 1e-9 bar the GPU tests hold the kernels to. No GPU needed."""
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import grazing as G
from common import MESHES

TOL = 1e-9
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]


def scene(shape):
    cfg = I.default_config_values()
    cfg.flags, cfg.integral_intervs = I.WITH_COLLISION, 6
    oc = O.config_from(cfg)
    T, Cc, _ = W.make_trajectory(2, [0, 0, 0], [24, 24, 24], seed=3, jitter=0.2)
    aabb = None
    if shape == "mesh":
        V, F = MESHES["rcone"]()
        osh = O.Shape.mesh(V, F, PP, wn_mode=O.WN_BH)
        R, t = W.rotation_from_poly_params(PP)
        Vb = V @ R.T + t
        aabb = (Vb.min(0), Vb.max(0))
    else:
        osh = O.Shape.named(shape)
    bmin, res, dims = [-0.3, 0.2, 0.1], 0.15, (160, 160, 160)
    g = G.grazing_map(oc, osh, T, Cc, bmin, res, dims, shape_aabb=aabb)
    return oc, osh, T, Cc, bmin, res, dims, g


@pytest.fixture(scope="module", params=["mesh", "Ball"])
def case(request):
    return scene(request.param)


def test_every_occupied_voxel_is_in_its_band(case):
    """recomputed without the shell pre-filter: the min over samples of the oracle SDF of every occupied voxel"""
    oc, osh, T, Cc, bmin, res, dims, g = case
    delta, sf = 1e-3, oc.safety_hor
    occ = g["occ"].reshape(-1)
    pos, R, _, _ = G.sample_poses(oc, T, Cc)
    ids = np.flatnonzero(occ)
    mins = np.full(ids.size, np.inf)
    for _, vid, prel, _ in G.window_pairs(oc, bmin, res, dims, pos, R):
        on = occ[vid] != 0
        if on.any():
            s, _ = osh.query(prel[on], what=0)
            k = np.searchsorted(ids, vid[on])
            np.minimum.at(mins, k, s)
    x = sf - mins
    active = (x >= delta / 4) & (x <= delta)
    inactive = (-x >= delta / 4) & (-x <= delta)
    assert np.all(active | inactive), f"{(~(active | inactive)).sum()} occupied voxels outside both bands"
    assert active.sum() == g["n_active"] and inactive.sum() == g["n_inactive"] and g["n_active"] >= 20 and g["n_inactive"] >= 20
    assert np.array_equal(ids[active], g["active_ids"])
    exp = O.eval_discrete(oc, g["occ"], bmin, res, osh, T, Cc)
    assert abs(exp[0] - g["cost"]) <= TOL * exp[0]                       # the fixture's hinge sum is the oracle's cost


def test_losing_any_one_active_voxel_is_visible_at_the_bar(case):
    oc, osh, T, Cc, bmin, res, dims, g = case
    assert g["sensitivity"] >= 100 * TOL
    base = O.eval_discrete(oc, g["occ"], bmin, res, osh, T, Cc)[0]
    rng = np.random.default_rng(0)
    pick = np.unique(np.concatenate([[np.argmin(g["voxel_cost"])], rng.choice(g["active_ids"].size, 9, replace=False)]))
    for k in pick:
        occ = g["occ"].copy().reshape(-1)
        occ[g["active_ids"][k]] = 0
        c = O.eval_discrete(oc, occ.reshape(dims), bmin, res, osh, T, Cc)[0]
        rel = (base - c) / base
        assert rel >= 100 * TOL, f"voxel {g['active_ids'][k]}: removing it moves the cost by only {rel:.2e}"
        assert abs(rel - g["voxel_cost"][k] / g["cost"]) <= 1e-9          # the derived share is the measured one
    # and an inactive voxel contributes exactly nothing
    occ = g["occ"].copy().reshape(-1)
    occ[g["inactive_ids"][:50]] = 0
    assert O.eval_discrete(oc, occ.reshape(dims), bmin, res, osh, T, Cc)[0] == pytest.approx(base, rel=1e-13)


def test_triangle_distance_helper_matches_the_oracle():
    """grazing.tri_dist (used to find pairs that only the full candidate-list radius answers) against the oracle's mesh distance"""
    V, F = W.l_prism_mesh()
    p = np.random.default_rng(4).uniform(-3, 3, (3000, 3))
    d = np.stack([G.tri_dist(p, V[f]) for f in F], 1).min(1)
    s, _ = O.Shape.mesh(V, F).query(p, what=0)
    assert np.abs(d - np.abs(s)).max() <= 1e-12
