"""The discrete scan's sub-box filtered candidate lists (k_mesh_disc_lists, DESIGN §3.1).

  * each filtered list is an ordered subsequence of the cell's full list, with the same first entry and the same lower bounds;
  * at random points of sampled cells, on their faces and corners and one ulp outside them, every triangle exactly tied for nearest
    (brute-force FP64 over all triangles) is in the filtered list;
  * the discrete cost and gradient are bit-identical with the full lists (k = 1) and the filtered ones (the default k): bench robot,
    winding sign, the x4 robot (deep cells), safety 0.15 and 2.5, a sharded launch, and the batched callback."""
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W
from test_gpu_mesh_lists import pair_dist

pytestmark = pytest.mark.gpu
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]      # the bench robot's poly_params
FILTER_MIN = 32    # DISC_FILTER_MIN
DISC_K = 4         # DISC_LIST_K, the library's default


def lists_of(ev):
    grid, full, disc = ev.dbg_mesh_grid(), ev.dbg_mesh_lists(), ev.dbg_disc_lists()
    return grid, full, disc


@pytest.fixture(scope="module")
def bench_lists():
    V, F = W.rounded_cone_mesh()
    ev = I.Evaluator(I.default_config_values(), device=0)
    try:
        ev.set_shape_mesh(V, F, PP)
        grid, full, disc = lists_of(ev)
    finally:
        ev.close()
    return grid, full, disc


def test_filtered_lists_are_subsequences(bench_lists):
    grid, full, disc = bench_lists
    assert disc is not None and disc["k"] > 1
    cnt, off = grid["cell_cnt"].reshape(-1), full["cell_off"].reshape(-1)
    dcnt, doff = disc["cell_cnt"].reshape(-1), disc["cell_off"].reshape(-1)
    assert np.all(dcnt <= cnt) and np.all((dcnt == 0) == (cnt == 0))
    assert np.array_equal(dcnt[cnt <= FILTER_MIN], cnt[cnt <= FILTER_MIN])
    shorter = 0
    for i in np.nonzero(cnt)[0]:
        a, b = full["cand"][off[i]:off[i] + cnt[i]], disc["cand"][doff[i]:doff[i] + dcnt[i]]
        la, lb = full["cand_lb"][off[i]:off[i] + cnt[i]], disc["cand_lb"][doff[i]:doff[i] + dcnt[i]]
        pos, idx = 0, []   # walk the full list in order, matching the filtered list's entries
        for t in b:
            hit = np.nonzero(a[pos:] == t)[0]
            assert len(hit), f"cell {i}: triangle {t} not in order in the full list"
            pos += int(hit[0]); idx.append(pos); pos += 1
        idx = np.array(idx)
        assert idx[0] == 0 and np.array_equal(lb, la[idx])
        shorter += dcnt[i] < cnt[i]
    total, dtotal = int(cnt.sum()), int(dcnt.sum())
    print(f"\nk = {disc['k']}: {dtotal} of {total} candidates kept ({dtotal / total:.1%}), {shorter} lists shortened")
    assert dtotal < total


def test_filtered_lists_keep_every_nearest_triangle(bench_lists):
    grid, full, disc = bench_lists
    tris = full["tris"]
    A, B, Cv = tris[:, 0], tris[:, 1], tris[:, 2]
    glo, gcell, gdim = grid["glo"], grid["gcell"], np.array(grid["gdim"])
    cnt = grid["cell_cnt"]
    rng = np.random.default_rng(11)
    cells = np.argwhere(cnt > FILTER_MIN)
    cells = cells[rng.choice(len(cells), size=min(120, len(cells)), replace=False)]
    checked = 0
    for ijk in cells:
        lo = glo + ijk * gcell
        hi = lo + gcell
        corners = lo + gcell * np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], dtype=np.float64)
        faces = lo + gcell * np.array([[0, .5, .5], [1, .5, .5], [.5, 0, .5], [.5, 1, .5], [.5, .5, 0], [.5, .5, 1]])
        P = np.concatenate([corners, faces, lo + gcell * rng.random((10, 3)),
                            np.nextafter(corners, corners + (corners - (lo + hi) / 2))])   # one ulp outside the box
        flat = int(np.ravel_multi_index(tuple(ijk), tuple(gdim)))
        o, n = int(disc["cell_off"].reshape(-1)[flat]), int(disc["cell_cnt"].reshape(-1)[flat])
        kept = set(disc["cand"][o:o + n].tolist())
        for p in P:
            d = pair_dist(np.broadcast_to(p, A.shape), A, B, Cv)
            tied = np.nonzero(d <= d.min() * (1.0 + 1e-12))[0]   # exact ties and everything within FP64 rounding of them
            assert set(tied.tolist()) <= kept, (tuple(ijk), p, tied)
            checked += 1
    print(f"\n{checked} points in {len(cells)} cells")


def run_discrete(k, V, F, safety=0.866, sign_mode=I.MESH_SIGN_AUTO, shards=1, batch=False, mapdim=40, scale=1.0):
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = 32
    cfg.safety_hor = safety
    occ = W.random_map(mapdim, mapdim, mapdim, p=0.3, seed=4, slabs=0)
    T, Cc, wp = W.make_trajectory(8, [0, 0, 0], [mapdim] * 3, seed=5, jitter=0.2)
    ev = I.Evaluator(cfg, device=0)
    try:
        ev.dbg_disc_k(k)
        ev.set_map_u8(occ, [0, 0, 0], 1.0)
        ev.set_shape_mesh(np.asarray(V) * scale, F, PP, sign_mode=sign_mode)
        assert (ev.dbg_disc_lists() is None) == (k == 1)
        if batch:
            rng = np.random.default_rng(3)
            heads, tails, X = [], [], []
            for b in range(4):
                w = W.random_walk_waypoints(6, [0, 0, 0], [mapdim] * 3, seed=40 + b)
                h, t = np.zeros((3, 3)), np.zeros((3, 3))
                h[:, 0], t[:, 0] = w[0], w[-1]
                heads.append(h); tails.append(t)
                X.append(np.concatenate([rng.normal(size=6) * 0.3 + 0.9, w[1:-1].reshape(-1)]))
            cost, grad = ev.callback_batch(np.array(heads), np.array(tails), 20.0, np.array(X))
            return [cost, grad]
        out = []
        for r in range(shards):
            if shards > 1:
                ev.set_shard(r, shards)
            c, gC, gT = ev.eval_discrete(T, Cc)
            out += [np.array([c]), gC, gT]
        return out
    finally:
        ev.close()


@pytest.mark.parametrize("case", ["bench", "winding", "x4", "safety0.15", "safety2.5", "sharded", "batched"])
def test_discrete_bit_identical(case):
    V, F = W.rounded_cone_mesh()
    kw = {"bench": {}, "winding": dict(sign_mode=I.MESH_SIGN_WINDING), "x4": dict(scale=4.0, mapdim=64), "safety0.15": dict(safety=0.15),
          "safety2.5": dict(safety=2.5), "sharded": dict(shards=8), "batched": dict(batch=True)}[case]
    full = run_discrete(1, V, F, **kw)
    filt = run_discrete(DISC_K, V, F, **kw)
    assert any(np.any(a != 0) for a in full)
    for a, b in zip(full, filt):
        assert a.tobytes() == b.tobytes()
