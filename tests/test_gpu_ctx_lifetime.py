"""Context lifetime and state replacement: a context releases every device resource it acquired, and a single obstacle point set
replaces any per-problem sets, whichever entry point sets it."""
import numpy as np
import pytest
import torch
import isdf_b200 as I
import workloads as W
from common import small_case, BMIN

pytestmark = pytest.mark.gpu


def batch_problems(B, N0, occ, seed):
    rng = np.random.default_rng(seed)
    heads, tails, X, wps = [], [], [], []
    for b in range(B):
        wp = W.random_walk_waypoints(N0, [0, 0, 0], [50, 50, 34], seed=seed + b)
        h, t = np.zeros((3, 3)), np.zeros((3, 3))
        h[:, 0], t[:, 0] = wp[0], wp[-1]
        X.append(np.concatenate([rng.normal(size=N0) * 0.3 + 0.9, wp[1:-1].reshape(-1)]))
        heads.append(h); tails.append(t); wps.append(wp)
    return np.array(heads), np.array(tails), np.array(X), wps


def use_every_subsystem(cfg, occ, T, Cc, wp):
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    cloud = np.ascontiguousarray(np.argwhere(occ) + 0.5, dtype=np.float32)
    ev.set_map_cloud(cloud, 1.0)
    d_cloud = torch.from_numpy(cloud).cuda()
    ev.set_map_cloud_device(d_cloud, res=1.0)
    torch.cuda.synchronize()
    del d_cloud
    ev.set_map_u8(occ, BMIN, 1.0)
    V, F = W.rounded_cone_mesh(n_theta=16, n_prof=12)
    ev.set_shape_mesh(V, F)
    for _ in range(2):                                  # the second evaluation runs on the work items the first one built
        ev.eval_discrete(T, Cc)
    ev.gather_obstacle_points(wp, cfg.kernel_size * cfg.occupancy_resolution / 3.0, cap=4096, set_as_points=True)
    ev.eval_swept(T, Cc)
    heads, tails, X, wps = batch_problems(2, 4, occ, seed=40)
    ev.set_points_batch([W.gather_obstacle_points(occ, BMIN, 1.0, w, 2.0)[:30] for w in wps])
    ev.callback_batch(heads, tails, 20.0, X)
    ev.lbfgs_batch(heads, tails, 20.0, X, ev.lbfgs_params(max_iterations=3))
    ev.frontend_build_kernels()
    ev.frontend_feasibility(*occ.shape)
    ev.trajectory_clearance(T, Cc, 8, 2.0, cfg.safety_hor)
    ev.close()


def test_context_releases_its_device_memory():
    cfg, occ, T, Cc, wp = small_case(N=4, K=16, seed=3)
    # one full round first: the kernels' modules are loaded on first use and stay loaded, which is not a leak
    use_every_subsystem(cfg, occ, T, Cc, wp)
    torch.cuda.synchronize(); torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        use_every_subsystem(cfg, occ, T, Cc, wp)
    torch.cuda.synchronize(); torch.cuda.empty_cache()
    free1 = torch.cuda.mem_get_info()[0]
    assert abs(free1 - free0) <= 1 << 20, f"free device memory moved by {(free1 - free0) / 2**20:.1f} MiB over three contexts"


def test_gathered_point_set_replaces_per_problem_sets():
    cfg, occ, _, _, _ = small_case(N=4, K=16, seed=3, flags=I.WITH_DYNAMICS)
    B, N0, rho = 2, 5, 20.0
    heads, tails, X, wps = batch_problems(B, N0, occ, seed=300)
    half = cfg.kernel_size * cfg.occupancy_resolution / 3.0
    psets = []
    for w in wps:
        pts = W.gather_obstacle_points(occ, BMIN, 1.0, w, half)
        psets.append(pts[:: max(1, len(pts) // 40)][:40])
    results = []
    for batch_sets in (psets, []):
        ev = I.Evaluator(cfg)
        ev.set_map_u8(occ, BMIN, 1.0)
        ev.set_shape_analytic(I.SHAPE_KINDS["BALL"], [3.0])   # a body this large reaches the gathered points from the trajectory
        ev.set_points_batch(batch_sets)
        if batch_sets:   # the per-problem sets are in effect before the gather replaces them
            with_sets, _ = ev.callback_batch(heads, tails, rho, X)
        _, n = ev.gather_obstacle_points(wps[0], half, set_as_points=True)
        assert n > 0
        results.append(ev.callback_batch(heads, tails, rho, X))
        ev.close()
    (c_a, g_a), (c_b, g_b) = results
    assert np.any(with_sets != c_b)                      # the swept term was really on, so stale sets would show
    assert np.array_equal(c_a, c_b) and np.array_equal(g_a, g_b)
