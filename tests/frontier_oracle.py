"""TEST INFRASTRUCTURE: a restatement of the frontiers of known space and the frontier goals (include/isdf.h, DESIGN §3.24) that the
device is held against.

  traversable(occ, masks)                 T_o (or T_b with the blocked grid and its masks): not occupied and a non-zero feasibility mask
  blocked(occ, known)                     occ | ~known
  frontier(To, Tb)                        F = Tb & dilate26(To & ~Tb), the dilation inside the map
  clusters(F, bmin, res)                  labels (scipy.ndimage.label, 3 x 3 x 3 structure) relabelled to each component's smallest voxel
                                          index, and the cluster table in ascending id
  field(Tb, src)                          g_b: the serial Dijkstra of tests/known_plan_serial.cpp over Tb with cw = 1
  select(g, F, labels, table, ...)        one pair's record (GOAL / FRONTIER / NONE)"""
import numpy as np
import scipy.ndimage as ndi
import known_plan_oracle as KO

NONE, GOAL, FRONTIER = 0, 1, 2


def traversable(occ, masks):
    occ = np.asarray(occ).astype(bool)
    return ~occ & np.asarray(masks).reshape(occ.shape + (4,)).any(axis=-1)


def blocked(occ, known):
    return np.asarray(occ).astype(bool) | ~np.asarray(known).astype(bool)


def frontier(To, Tb):
    To, Tb = np.asarray(To, dtype=bool), np.asarray(Tb, dtype=bool)
    assert not (Tb & ~To).any(), "T_b must be a subset of T_o"
    d = ndi.binary_dilation(To & ~Tb, structure=np.ones((3, 3, 3), dtype=bool), border_value=0)
    return Tb & d


def clusters(F, bmin, res):
    """-> (labels (X, Y, Z) int64, -1 outside F, else the cluster id; table: list of dicts id, size, bmin, bmax, centroid by ascending id)"""
    F = np.asarray(F, dtype=bool)
    lab, n = ndi.label(F, structure=np.ones((3, 3, 3), dtype=int))
    flat = np.arange(F.size, dtype=np.int64).reshape(F.shape)
    out = np.full(F.shape, -1, dtype=np.int64)
    table = []
    for k in range(1, n + 1):
        m = lab == k
        cid = int(flat[m].min())
        out[m] = cid
        idx = np.argwhere(m)
        s = idx.sum(axis=0)
        table.append(dict(id=cid, size=len(idx), bmin=idx.min(axis=0), bmax=idx.max(axis=0),
                          centroid=np.array([bmin[a] + (float(s[a]) / float(len(idx)) + 0.5) * res for a in range(3)])))
    table.sort(key=lambda c: c["id"])
    return out, table


def field(Tb, src):
    return KO.dijkstra(np.asarray(Tb, dtype=np.uint8), None, src, 0.0)


def voxel(p, bmin, res, dims):
    """path_voxel for a point inside the map"""
    i = np.floor((np.asarray(p, dtype=np.float64) - bmin) / res).astype(int)
    return tuple(int(min(max(i[a], 0), dims[a] - 1)) for a in range(3))


def select(g, F, labels, table, goal, t, bmin, res, goal_weight=1.0, min_cluster_voxels=1):
    """the record of one pair: dict(kind, voxel, cluster, g, score, point); g the field from the pair's start, t its goal voxel"""
    X, Y, Z = g.shape
    flat = lambda v: (v[0] * Y + v[1]) * Z + v[2]   # noqa: E731
    goal = np.asarray(goal, dtype=np.float64)
    if np.isfinite(g[t]):
        return dict(kind=GOAL, voxel=flat(t), cluster=-1, g=g[t], score=g[t], point=goal.copy())
    size = {c["id"]: c["size"] for c in table}
    best = None
    for v in np.argwhere(F):   # ascending voxel index: a later voxel wins only with a strictly smaller score
        v = tuple(int(a) for a in v)
        if not np.isfinite(g[v]) or size[int(labels[v])] < min_cluster_voxels:
            continue
        c = np.array([(v[a] + 0.5) * res + bmin[a] for a in range(3)])
        d = c - goal
        sc = g[v] + goal_weight * np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
        if best is None or sc < best[0]:
            best = (sc, v, c)
    if best is None:
        return dict(kind=NONE, voxel=-1, cluster=-1, g=np.inf, score=np.inf, point=goal.copy())
    sc, v, c = best
    return dict(kind=FRONTIER, voxel=flat(v), cluster=int(labels[v]), g=g[v], score=sc, point=c)
