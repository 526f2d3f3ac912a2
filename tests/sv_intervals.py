"""Interval-edge fixtures for the swept-volume search: obstacle point sets whose coarse in-range bitmaps (choiceTInit's 0.2 s loop,
swm:392-421) reach every branch of the bitmap -> interval conversion.

The robot flies a loop around a centre more than once and leaves it outwards at the end, so a point can come within range
(inf = 2 safety_hor + 0.1) several times, stay within range throughout (near the centre), or only at the end. Candidate points are
placed around the robot at every coarse sample, at body-frame distances where the SDF is near inf; the oracle's own coarse loop
(oracle_lib.sv_coarse) classifies each. A point is kept only if every coarse SDF is at least DELTA away from inf, so that no rounding
difference can flip a coarse decision, and then counts in each category its bitmap shows:
  A  a closed run starts at sample 0 (lb clamped at 0)
  B  a run is still open at the last sample (dropped): B_alone without, B_after with an earlier closed run (the open run's entry
     still seeds range_mindis)
  C  a closed run ends exactly at sample nc - 1 (ub clamped to the duration)
  D  a closed run enters at bit 31 or leaves at bit 0 of a 32-bit word
  E  two or more closed runs; E_carried: a later run's fine scan does not improve range_mindis, so its seed is an earlier run's
  F  a closed run of one sample
  G  never in range (SV-SDF 10, t* untouched)
  H  in range at every sample (one open run: SV-SDF 10)
Trajectories have nc = 0 or 1 (mod 32) coarse samples: a full last bitmap word, or a last word holding one sample.
Everything here is numpy + the oracle (no GPU)."""
import functools
import numpy as np
import isdf_b200 as I
import oracle_lib as O
import workloads as W
from common import tilted, MESHES
from grazing import quat_to_R

DELTA = 1e-6
CATEGORIES = ["A", "B_alone", "B_after", "C", "D", "E", "E_carried", "F", "G", "H"]
MESH_PP = [0.1, -0.05, 0.0, 120.0, 20.0, -35.0]
ROBOTS = ["CSG_tilted", "rcone"]


def config():
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = 16
    return cfg


def oracle_robot(robot):
    if robot == "CSG_tilted":
        R, t = tilted()
        return O.Shape.named("CSG", R, t)
    V, F = MESHES[robot]()
    return O.Shape.mesh(V, F, MESH_PP)


def set_robot(ev, robot):
    if robot == "CSG_tilted":
        R, t = tilted()
        ev.set_shape_named("CSG", R, t)
    else:
        V, F = MESHES[robot]()
        ev.set_shape_mesh(V, F, MESH_PP)


def loop_trajectory(nc, radius=2.0, turns=1.3, pieces=9):
    """a loop of `turns` turns around the origin, then out to 1.5 radius; total duration 0.2 nc - 0.1 s, so choiceTInit's loop takes
    exactly nc coarse samples (its running sum stays 0.1 s away from the duration)"""
    a = np.linspace(0.0, 2 * np.pi * turns, pieces)
    wp = np.stack([radius * np.cos(a), radius * np.sin(a), 0.4 * np.sin(2 * a)], 1)
    wp = np.concatenate([wp, [wp[-1] * 1.5]])
    seg = np.linalg.norm(np.diff(wp, axis=0), axis=1)
    T = (0.2 * nc - 0.1) * seg / seg.sum()
    return T, W.minco_s3(wp, T)


def coarse_times(duration):
    t, out = 0.0, []
    while t < duration:
        out.append(t)
        t += 0.2
    return np.array(out)


def in_range(bits, nc):
    k = np.arange(nc)
    return ((bits[:, k >> 5] >> (k & 31).astype(np.uint32)) & 1).astype(bool)


def runs(row):
    """closed runs [(kin, kout)] (kout = first sample out of range again) and the entry of a run still open at the end (or None)"""
    closed, kin = [], None
    for k, v in enumerate(row):
        if v and kin is None:
            kin = k
        elif not v and kin is not None:
            closed.append((kin, k))
            kin = None
    return closed, kin


def classify(bits, nc, carried):
    """category -> boolean mask over the points"""
    inr = in_range(bits, nc)
    cats = {c: np.zeros(len(inr), bool) for c in CATEGORIES}
    for q, row in enumerate(inr):
        closed, open_kin = runs(row)
        cats["A"][q] = any(kin == 0 for kin, _ in closed)
        cats["B_alone"][q] = open_kin is not None and not closed and not row.all()
        cats["B_after"][q] = open_kin is not None and bool(closed)
        cats["C"][q] = any(kout == nc - 1 for _, kout in closed)
        cats["D"][q] = any(kin % 32 == 31 or kout % 32 == 0 for kin, kout in closed)
        cats["E"][q] = len(closed) >= 2
        cats["E_carried"][q] = len(closed) >= 2 and carried[q] >= 1
        cats["F"][q] = any(kout == kin + 1 for kin, kout in closed)
        cats["G"][q] = not row.any()
        cats["H"][q] = row.all()
    return cats


def _candidates(ocfg, osh, T, Cc, times, rng, per_sample):
    """points around the robot at every coarse sample, at body-frame distances where the SDF is inf + s, s in [-0.4, 0.4]; plus points
    near the loop centre (in range throughout) and far away (never)"""
    inf = 2 * ocfg.safety_hor + 0.1
    out, _, _, _ = O.traj_eval(T, Cc, times)
    q, _ = O.flat_forward_batch(ocfg, out[:, 3:6], out[:, 6:9], out[:, 9:12])
    R = quat_to_R(q)
    n = len(times) * per_sample
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    target = inf + rng.uniform(-0.4, 0.4, n)
    lo, hi = np.zeros(n), np.full(n, 12.0)
    for _ in range(40):                                  # bisection along the ray for sdf(r u) = target (first crossing not needed)
        mid = 0.5 * (lo + hi)
        s, _ = osh.query(mid[:, None] * u, what=0)
        below = s < target
        lo, hi = np.where(below, mid, lo), np.where(below, hi, mid)
    body = lo[:, None] * u
    k = np.repeat(np.arange(len(times)), per_sample)
    world = out[k, 0:3] + np.einsum("nij,nj->ni", R[k], body)
    centre = rng.uniform(-1.5, 1.5, (200, 3))
    far = rng.normal(size=(30, 3))
    far = 30.0 * far / np.linalg.norm(far, axis=1, keepdims=True)
    return np.concatenate([world, centre, far])


@functools.lru_cache(maxsize=None)
def fixture(robot, nc_target, quota=5, per_sample=24, seed=0):
    """dict(T, C, pts, nc, cats (category -> indices into pts), margin, carried): up to `quota` points per category, each with coarse
    margin >= DELTA"""
    cfg = config()
    ocfg = O.config_from(cfg)
    osh = oracle_robot(robot)
    T, Cc = loop_trajectory(nc_target)
    times = coarse_times(T.sum())
    rng = np.random.default_rng(seed)
    cand = _candidates(ocfg, osh, T, Cc, times, rng, per_sample)
    nc, bits, margin, carried = O.sv_coarse(ocfg, osh, T, Cc, cand)
    ok = margin >= DELTA
    cats = classify(bits, nc, carried)
    pick = set()
    for c in CATEGORIES:
        idx = np.flatnonzero(cats[c] & ok)
        pick.update(idx[:quota].tolist())
    pick = np.array(sorted(pick))
    pts = cand[pick]
    nc2, bits2, margin2, carried2 = O.sv_coarse(ocfg, osh, T, Cc, pts)
    sel = classify(bits2, nc2, carried2)
    return dict(robot=robot, cfg=cfg, T=T, C=Cc, pts=pts, nc=nc2, margin=margin2, carried=carried2,
                cats={c: np.flatnonzero(m) for c, m in sel.items()})
