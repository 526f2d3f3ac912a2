"""isdf_plan_states / _device: with rest states at the path fronts of an isdf_plan_pairs run every output equals isdf_plan_pairs bit for
bit; with moving heads the trajectories start at the head state; a pair alone equals it in a batch, permutations permute, max_fields and the
two forms change no bit; refusals follow the failure contract and the device form stays within the pairs' transfer bounds."""
import numpy as np
import pytest
import isdf_b200 as I
from test_gpu_plan import _ev, _scene, _params, _same, _summ_same

pytestmark = pytest.mark.gpu


def _plans_same(a, b):
    keys = ("stage", "path_nodes", "pieces", "obstacle_points", "midend_ret", "backend_ret", "backend_iterations", "path_cost", "midend_f",
            "backend_f", "duration", "path", "T", "coeffs")
    return all(_same(x[k], y[k]) for x, y in zip(a, b) for k in keys) and all(_summ_same(x["certify"], y["certify"]) for x, y in zip(a, b))


def _setup(n=6, seed=21):
    occ, start, goals = _scene(n, seed=seed)
    ev = _ev("Ball", occ)
    rng = np.random.default_rng(seed)
    free = np.argwhere(occ == 0)
    starts = free[rng.choice(len(free), n, replace=False)] + rng.uniform(0.1, 0.9, (n, 3))
    return ev, starts, goals


def test_rest_heads_at_path_fronts_equal_plan_pairs():
    ev, starts, goals = _setup()
    p = _params(ev, flags=I.PLAN_CERTIFY)
    ref, _ = ev.plan_pairs(starts, goals, p)
    heads = np.zeros((len(goals), 9))
    heads[:, :3] = [r["path"][0] for r in ref]
    got, _ = ev.plan_states(heads, goals, p)
    assert _plans_same(got, ref)
    ev.close()


def test_moving_heads_start_the_trajectories_and_batches_agree():
    import torch
    ev, starts, goals = _setup(seed=22)
    p = _params(ev, flags=I.PLAN_CERTIFY)
    rng = np.random.default_rng(3)
    heads = np.concatenate([starts, rng.normal(0, 1.5, (len(goals), 3)), rng.normal(0, 2.0, (len(goals), 3))], 1)
    got, _ = ev.plan_states(heads, goals, p)
    have = [b for b, r in enumerate(got) if r["pieces"] > 0]
    assert have
    off, T, Cc = ev.pack_plans([got[b] for b in have])
    st = ev.trajectory_states((off, T, Cc), np.arange(len(have)), np.zeros(len(have)))
    for k, b in enumerate(have):
        assert np.array_equal(st[k, :3], heads[b, :3])
        for lo in (3, 6):
            assert np.abs(st[k, lo:lo + 3] - heads[b, lo:lo + 3]).max() <= 1e-12 * max(np.abs(heads[b, lo:lo + 3]).max(), 1.0)
    # alone, permuted, every max_fields, device form
    for b in (0, len(goals) - 1):
        one, _ = ev.plan_states(heads[b:b + 1], goals[b:b + 1], p)
        assert _plans_same(one, [got[b]])
    perm = np.random.default_rng(4).permutation(len(goals))
    pg, _ = ev.plan_states(heads[perm], goals[perm], p, max_fields=2)
    assert _plans_same(pg, [got[i] for i in perm])
    d = ev.plan_states_device(torch.as_tensor(heads, device="cuda"), torch.as_tensor(goals, device="cuda"), p, max_fields=1)
    res = I.decode_plan_results(d["results"])
    po = d["piece_off"].cpu().numpy()
    for b in range(len(goals)):
        assert int(res["stage"][b]) == got[b]["stage"]
        assert np.array_equal(d["T"][po[b]:po[b + 1]].cpu().numpy(), got[b]["T"])
        assert np.array_equal(d["coeffs"][18 * po[b]:18 * po[b + 1]].cpu().numpy(), got[b]["coeffs"])
    tr = ev.dbg_plan_transfers()
    assert tr["d2h_bytes"] <= 80 * len(goals) + 64
    ev.close()


def test_refusals_follow_the_failure_contract():
    import torch
    ev, starts, goals = _setup(n=3, seed=23)
    p = _params(ev, flags=I.PLAN_CERTIFY)
    heads = np.concatenate([starts, np.zeros((3, 6))], 1)
    for bad in (np.nan, np.inf):
        h = heads.copy()
        h[1, 4 if bad is np.nan else 7] = bad
        with pytest.raises(I.IsdfError) as e:
            ev.plan_states(h, goals, p)
        assert e.value.code == -1 and "starts[1]" in str(e.value)
        # the device form refuses after its check of v and a: one launch more than a pairs call refused at its endpoints
        launches = ev.stats().kernel_launches
        with pytest.raises(I.IsdfError):
            ev.plan_pairs_device(torch.as_tensor(starts, device="cuda"), torch.as_tensor(goals - 100.0, device="cuda"), p)
        base = ev.stats().kernel_launches - launches
        launches = ev.stats().kernel_launches
        with pytest.raises(I.IsdfError) as e:
            ev.plan_states_device(torch.as_tensor(h, device="cuda"), torch.as_tensor(goals, device="cuda"), p)
        assert e.value.code == -1 and "starts[1]" in str(e.value)
        assert ev.stats().kernel_launches - launches == base + 1
    out = heads.copy()
    out[0, :3] = -5.0   # outside the map
    with pytest.raises(I.IsdfError) as e:
        ev.plan_states(out, goals, p)
    assert e.value.code == -1
    noker = _ev("Ball", np.zeros((8, 8, 8), np.uint8), kernels=False)
    with pytest.raises(I.IsdfError) as e:
        noker.plan_states(np.array([[1.5, 1.5, 1.5, 0, 0, 0, 0, 0, 0]]), np.array([[5.5, 5.5, 5.5]]), p)
    assert e.value.code == -2
    ev.close(); noker.close()
