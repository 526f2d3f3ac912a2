"""Grazing fixtures: scenes whose whole collision cost sits at the hinge boundary sdf = safety_hor.

On a random map the discrete cost is dominated by voxels deep inside the hinge; a cull or bounded search that wrongly drops a
voxel whose SDF is just below safety_hor loses a contribution of order x^3 / mu^2 (x = safety_hor - sdf), far below any
relative tolerance of the total. Here every occupied voxel is placed, by the oracle's own SDF, in a thin band around the
boundary:
  * active:   safety_hor - min_sdf in [delta/4, delta]  (the voxel contributes, but only barely)
  * inactive: min_sdf - safety_hor in [delta/4, delta]  (just outside: it must contribute exactly nothing)
where min_sdf is the minimum over the trajectory's pose samples whose body-frame box holds the voxel. Because |x| >= delta/4 at
every voxel's closest pose, neither FMA contraction nor a one-ulp SDF difference can flip a hinge decision there, so a correct
kernel agrees with the oracle to ~1e-12 and losing any single voxel moves the cost by at least `sensitivity` (relative).

The same idea for the swept-volume path: point sets whose oracle SV-SDF lies near the range bound inf = 2 safety_hor + 0.1
or near the hinge. Everything here is numpy + the oracle (no GPU)."""
import numpy as np
import oracle_lib as O


def sample_poses(ocfg, T, coeffs):
    """every pose sample of the discrete term, as the oracle forms it (oracle_planner.hpp eval_sample): piece i, local time
    j * (T_i / K), the piece polynomial evaluated directly. Returns pos (S,3), R (S,3,3), weight (S,) = weight_p * node * step,
    piece (S,)."""
    T = np.asarray(T, float).reshape(-1)
    N, K = T.size, ocfg.integral_intervs
    Cm = np.asarray(coeffs, float).reshape(3, 6 * N)            # column-major 6N x 3 -> [axis, 6 i + k]
    pos, vel, acc, jer, w, piece = [], [], [], [], [], []
    k = np.arange(6)
    for i in range(N):
        step = T[i] * (1.0 / K)
        c = Cm[:, 6 * i:6 * i + 6]
        for j in range(K + 1):
            s = j * step
            sp = s ** k
            pos.append(c @ sp)
            vel.append(c @ np.array([0, 1, 2 * s, 3 * s ** 2, 4 * s ** 3, 5 * s ** 4]))
            acc.append(c @ np.array([0, 0, 2, 6 * s, 12 * s ** 2, 20 * s ** 3]))
            jer.append(c @ np.array([0, 0, 0, 6, 24 * s, 60 * s ** 2]))
            w.append(ocfg.weight_p * (0.5 if j in (0, K) else 1.0) * step)
            piece.append(i)
    q, _ = O.flat_forward_batch(ocfg, np.array(vel), np.array(acc), np.array(jer))
    return np.array(pos), quat_to_R(q), np.array(w), np.array(piece)


def quat_to_R(q):
    """Eigen::Quaterniond(w, x, y, z).toRotationMatrix() without normalisation, batched"""
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.empty((q.shape[0], 3, 3))
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - w * z); R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y); R[:, 2, 1] = 2 * (y * z + w * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def window_pairs(ocfg, bmin, res, dims, pos, R, keep=None, clip=None):
    """(sample, voxel) pairs whose voxel centre lies in the sample's body-frame box |prel| <= bd/2 (the pairs the oracle answers).
    keep(prel) -> (needs_query, deep): an optional pre-filter in the body frame (shell_filter). Yields per sample
    (flat voxel ids, prel, deep mask); pairs neither queried nor deep are dropped. clip: an optional body-frame (lo, hi) box
    outside which pairs are not generated at all."""
    bmin, dims = np.asarray(bmin, float), np.asarray(dims)
    h = ocfg.kernel_size * ocfg.occupancy_resolution / 2
    for s in range(pos.shape[0]):
        wlo, whi = pos[s] - h, pos[s] + h
        for box in [b for b in (getattr(keep, "box", None), clip) if b is not None]:   # world AABB of a body-frame box bounds the scan
            c, e = 0.5 * (box[0] + box[1]), 0.5 * (box[1] - box[0])
            wc, we = pos[s] + R[s] @ c, np.abs(R[s]) @ e
            wlo, whi = np.maximum(wlo, wc - we - res), np.minimum(whi, wc + we + res)
        lo = np.clip(np.floor((wlo - bmin) / res).astype(int), 0, dims - 1)
        hi = np.clip(np.floor((whi - bmin) / res).astype(int), 0, dims - 1)
        ix, iy, iz = (np.arange(lo[a], hi[a] + 1) for a in range(3))
        I3 = np.stack(np.meshgrid(ix, iy, iz, indexing="ij"), -1).reshape(-1, 3)
        ctr = (I3 + 0.5) * res + bmin
        prel = (ctr - pos[s]) @ R[s]                             # R^T (c - pos), row-vector form
        m = np.all(np.abs(prel) <= h, axis=1)
        deep = np.zeros_like(m)
        if keep is not None:
            q, deep = keep(prel)
            m &= q | deep
        if clip is not None:
            m &= np.all((prel >= clip[0]) & (prel <= clip[1]), axis=1)
        I3, prel, deep = I3[m], prel[m], deep[m]
        yield s, (I3[:, 0] * dims[1] + I3[:, 1]) * dims[2] + I3[:, 2], prel, deep


def hinge(x, mu):
    """smoothedL1 (the reference's hinge): 0 for x < 0, cubic up to mu, linear beyond"""
    x = np.asarray(x, float)
    xd = x / mu
    f = np.where(x > mu, x - 0.5 * mu, (mu - 0.5 * x) * xd ** 3)
    return np.where(x < 0, 0.0, f)


def shell_filter(shape, shape_aabb, sf, delta, spacing=0.2):
    """Exact body-frame pre-filter for a true (1-Lipschitz) distance function whose zero set lies in shape_aabb: the SDF is
    sampled once on a lattice of the given spacing over the AABB padded by sf + delta, and a point p needs a query only if
    |sdf(node) - sf| <= |p - node| + delta at its nearest node; otherwise it is certainly above the band or certainly below it
    ('deep'). Points off the lattice are farther than sf + delta from the AABB. keep(p) -> (needs_query, deep) masks."""
    pad = sf + delta + spacing
    lo, hi = np.asarray(shape_aabb[0], float) - pad, np.asarray(shape_aabb[1], float) + pad
    n = np.ceil((hi - lo) / spacing).astype(int) + 1
    nodes = lo + spacing * np.stack(np.meshgrid(*(np.arange(k) for k in n), indexing="ij"), -1).reshape(-1, 3)
    sn, _ = shape.query(nodes, what=0)
    sn = sn.reshape(tuple(n))

    def keep(p):
        inbox = np.all((p >= lo) & (p <= hi), axis=1)
        k = np.clip(np.rint((p - lo) / spacing).astype(int), 0, n - 1)
        r = np.linalg.norm(p - (lo + spacing * k), axis=1) * (1 + 1e-9) + delta + 1e-9
        dn = sn[k[:, 0], k[:, 1], k[:, 2]] - sf
        return inbox & (np.abs(dn) <= r), inbox & (dn < -r)
    keep.box = (lo, hi)
    return keep


def grazing_map(ocfg, shape, T, coeffs, bmin, res, dims, delta=1e-3, shape_aabb=None, max_voxels=4000, region=None):
    """Occupancy map whose occupied voxels all graze the robot along the trajectory (module docstring).

    shape_aabb: optional body-frame (lo, hi) box holding the zero set of a true distance function (an exact-sign mesh's vertex box):
    only voxels that can lie in the band are queried (shell_filter). Leave it None for shapes whose SDF is not 1-Lipschitz
    (winding-sign meshes, twisted boxes). region(prel) -> bool mask: optionally, only voxels with a near-band pair inside this
    body-frame region are occupied. If it has a .box (body-frame lo, hi), pairs outside that box are not generated: the box must
    hold every pair of every voxel that can become eligible (the oracle comparison of the fixture's cost checks this). Returns a dict:
      occ (uint8 dims), n_active, n_inactive, active_ids / inactive_ids (flat voxel ids), min_sdf (per occupied voxel, id order),
      pairs: dict(sample, vid, prel, sdf) of every (sample, occupied voxel) pair with |sdf - safety| <= delta,
      voxel_cost: the oracle-form cost of every active voxel (sum over its samples of weight * hinge), cost: their sum,
      sensitivity: min(voxel_cost) / cost — the smallest relative change of the cost when one active voxel is lost."""
    sf = ocfg.safety_hor
    pos, R, w, _ = sample_poses(ocfg, T, coeffs)
    keep = shell_filter(shape, shape_aabb, sf, delta, spacing=max(0.2, 2 * res)) if shape_aabb is not None else None
    allv, alls, rec = [], [], []
    for s, vid, prel, deep in window_pairs(ocfg, bmin, res, dims, pos, R, keep, getattr(region, "box", None)):
        if vid.size == 0:
            continue
        sdf = np.full(vid.size, -np.inf)                         # certainly below the band: never a grazing voxel
        sdf[~deep], _ = shape.query(prel[~deep], what=0)
        near = np.abs(sdf - sf) <= delta
        rec.append((np.full(near.sum(), s), vid[near], prel[near], sdf[near]))
        allv.append(vid); alls.append(sdf)
    ids, inv = np.unique(np.concatenate(allv), return_inverse=True)
    mins = np.full(ids.size, np.inf)
    np.minimum.at(mins, inv, np.concatenate(alls))
    x = sf - mins
    act = (x >= delta / 4) & (x <= delta)
    ina = (-x >= delta / 4) & (-x <= delta)
    s_, v_, p_, d_ = (np.concatenate(a) for a in zip(*rec)) if rec else (np.zeros(0, int), np.zeros(0, int), np.zeros((0, 3)), np.zeros(0))
    if region is not None:                                       # only voxels with a near-band pair inside the body-frame region
        eligible = np.isin(ids, v_[region(p_)])
        act &= eligible
        ina &= eligible
    assert act.sum() > 0, "no grazing voxel: the trajectory never brings a voxel centre into the band"
    sel = act | ina
    if sel.sum() > max_voxels:                                   # keep the fixture small: thin both bands evenly
        rng = np.random.default_rng(0)
        drop = np.flatnonzero(sel)[rng.permutation(sel.sum())[max_voxels:]]
        act[drop] = ina[drop] = False
        sel = act | ina
    occ = np.zeros(int(np.prod(dims)), dtype=np.uint8)
    occ[ids[sel]] = 1
    order = np.argsort(ids[sel])
    on = occ[v_] == 1
    pairs = dict(sample=s_[on], vid=v_[on], prel=p_[on], sdf=d_[on])
    # cost of every active voxel over all its pairs (pairs with sdf < safety - delta cannot exist: delta bounds the minimum)
    contrib = w[pairs["sample"]] * hinge(sf - pairs["sdf"], ocfg.smoothing_eps)
    active_ids = np.sort(ids[act])
    vc = np.zeros(active_ids.size)
    np.add.at(vc, np.searchsorted(active_ids, pairs["vid"][pairs["sdf"] < sf]), contrib[pairs["sdf"] < sf])
    return dict(occ=occ.reshape(tuple(dims)), n_active=int(act.sum()), n_inactive=int(ina.sum()), active_ids=active_ids,
                inactive_ids=np.sort(ids[ina]), min_sdf=mins[sel][order], pairs=pairs, voxel_cost=vc, cost=float(vc.sum()),
                sensitivity=float(vc.min() / vc.sum()))


def unravel(vid, dims):
    return np.stack(np.unravel_index(vid, tuple(dims)), axis=1)


# ---- which branch of the mesh search answers a body-frame query point (isdf_dbg_mesh_grid) ------------------------
BRANCHES = ("listed", "overflow", "deep", "far", "outside")


def classify(grid, prel):
    """per point: 'outside' the cell grid, in a cell with a candidate list ('listed'), in an unlisted cell within list_reach
    ('overflow': more than the list cap of candidates -> reach-bounded tree search from the cell's seed), or in an unlisted cell
    beyond list_reach: 'deep' inside the mesh (bounded search, then unbounded when the bound misses) or 'far' outside it
    (culled by the cell's distance bracket in the discrete path)."""
    prel = np.asarray(prel, float).reshape(-1, 3)
    c = np.floor((prel - grid["glo"]) * (1.0 / grid["gcell"])).astype(np.int64)
    g = np.array(grid["gdim"])
    inside = np.all((c >= 0) & (c < g), axis=1)
    out = np.full(prel.shape[0], "outside", dtype=object)
    ci = c[inside]
    dc = grid["cell_dist"][ci[:, 0], ci[:, 1], ci[:, 2]].astype(np.float64)
    cnt = grid["cell_cnt"][ci[:, 0], ci[:, 1], ci[:, 2]]
    lab = np.where(cnt > 0, "listed", np.where(np.abs(dc) <= grid["list_reach"], "overflow", np.where(dc < 0, "deep", "far")))
    out[inside] = lab
    return out


def tri_dist(p, tri):
    """distance of points p (n,3) to one triangle tri (3,3): Ericson's Voronoi-region closest point, vectorised"""
    A, B, Cv = tri
    ab, ac = B - A, Cv - A
    ap, bp, cp = p - A, p - B, p - Cv
    d1, d2, d3, d4, d5, d6 = ap @ ab, ap @ ac, bp @ ab, bp @ ac, cp @ ab, cp @ ac
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    safe = lambda a: np.where(a == 0, 1.0, a)
    den = 1.0 / safe(va + vb + vc)
    q = A + np.outer(vb * den, ab) + np.outer(vc * den, ac)
    regions = [((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0), lambda m: B + np.outer(((d4 - d3) / safe((d4 - d3) + (d5 - d6)))[m], Cv - B)),
               ((vb <= 0) & (d2 >= 0) & (d6 <= 0), lambda m: A + np.outer((d2 / safe(d2 - d6))[m], ac)),
               ((d6 >= 0) & (d5 <= d6), lambda m: Cv),
               ((vc <= 0) & (d1 >= 0) & (d3 <= 0), lambda m: A + np.outer((d1 / safe(d1 - d3))[m], ab)),
               ((d3 >= 0) & (d4 <= d3), lambda m: B),
               ((d1 <= 0) & (d2 <= 0), lambda m: A)]
    for m, f in regions:                                         # later regions take priority, as in the kernels
        q[m] = f(m)
    return np.linalg.norm(p - q, axis=1)


def list_critical(grid, prel, tris):
    """per point: its closest triangle lies farther than |d_c| + ghd from its cell centre, i.e. only a candidate list of the full
    radius |d_c| + 2 hd (every triangle that can be closest to some point of the cell) holds it. tris: (T, 3, 3) body frame."""
    prel = np.asarray(prel, float).reshape(-1, 3)
    c = np.floor((prel - grid["glo"]) * (1.0 / grid["gcell"])).astype(np.int64)
    ctr = grid["glo"] + (c + 0.5) * grid["gcell"]
    dc = np.abs(grid["cell_dist"][c[:, 0], c[:, 1], c[:, 2]].astype(np.float64))
    best = np.argmin(np.stack([tri_dist(prel, t) for t in tris], 1), axis=1)
    dbest = np.stack([tri_dist(ctr, t) for t in tris], 1)[np.arange(prel.shape[0]), best]
    return dbest > dc + grid["ghd"]


def branch_counts(grid, prel):
    lab = classify(grid, prel)
    return {b: int((lab == b).sum()) for b in BRANCHES}


# ---- swept volume ------------------------------------------------------------------------------------------------
def _world_normal(ocfg, T, coeffs, tstar, grel):
    """unit world-frame gradient of the swept-volume SDF at the oracle's t*: R(t*) g_rel"""
    out, _, _, _ = O.traj_eval(T, coeffs, tstar)
    q, _ = O.flat_forward_batch(ocfg, out[:, 3:6], out[:, 6:9], out[:, 9:12])
    n = np.einsum("sij,sj->si", quat_to_R(q), grel)
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def swept_band_points(ocfg, shape, T, coeffs, shape_aabb, n=1200, delta=1e-3, newton=3, seed=0):
    """Obstacle points whose oracle SV-SDF lies (a) within delta below the range bound inf = 2 safety_hor + 0.1 (the range test and
    the cell brackets around it), with a copy of each pushed just above it ('above': mostly never in range), and (b) at the hinge: safety_hor - sdf in [delta/4, delta] (active) or sdf - safety_hor in
    [delta/4, delta] (inactive). Random points around the trajectory are moved onto target levels by Newton steps along the
    oracle's swept-volume gradient. Returns (points, dict of index arrays range / above / active / inactive)."""
    sf = ocfg.safety_hor
    inf = 2 * sf + 0.1
    rng = np.random.default_rng(seed)
    T = np.asarray(T, float)
    t = rng.uniform(0, T.sum(), n)
    out, _, _, _ = O.traj_eval(T, coeffs, t)
    q, _ = O.flat_forward_batch(ocfg, out[:, 3:6], out[:, 6:9], out[:, 9:12])
    lo, hi = np.asarray(shape_aabb[0]) - inf, np.asarray(shape_aabb[1]) + inf
    pts = out[:, 0:3] + np.einsum("sij,sj->si", quat_to_R(q), rng.uniform(lo, hi, (n, 3)))
    u = rng.random(n)
    k = rng.integers(0, 3, n)
    target = np.where(k == 0, inf - delta * (0.25 + 0.5 * u), np.where(k == 1, sf - delta * (0.3 + 0.6 * u), sf + delta * (0.3 + 0.6 * u)))
    for _ in range(newton):
        r = O.eval_swept(ocfg, shape, T, coeffs, pts, use_omp=True)
        hit = r["sdf"] < 9.0
        pts, target = pts[hit], target[hit]
        nrm = _world_normal(ocfg, T, coeffs, r["tstar"][hit], r["grel"][hit])
        pts = pts + (target - r["sdf"][hit])[:, None] * nrm
    r = O.eval_swept(ocfg, shape, T, coeffs, pts, use_omp=True)
    sd = r["sdf"]
    x = sf - sd
    sets = dict(range=np.flatnonzero((sd < inf) & (sd >= inf - delta)), active=np.flatnonzero((x >= delta / 4) & (x <= delta)),
                inactive=np.flatnonzero((-x >= delta / 4) & (-x <= delta)))
    # the other side of the range bound: the points just below inf pushed out along the gradient to inf + [delta/4, 3 delta/4]
    k = sets["range"]
    up = rng.random(k.size)
    above = pts[k] + (inf - sd[k] + delta * (0.25 + 0.5 * up))[:, None] * _world_normal(ocfg, T, coeffs, r["tstar"][k], r["grel"][k])
    sets["above"] = np.arange(pts.shape[0], pts.shape[0] + k.size)
    return np.concatenate([pts, above]), sets
