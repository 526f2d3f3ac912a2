"""Vehicles other than the default one, and the wrong vehicles each test must tell apart from them — TEST INFRASTRUCTURE.

Every reference config ships one airframe (0.61 kg, drags 0.10 / 0.10 / 0.01, speed_eps 1e-4, dynamic weights all 1000), and at that point
horiz_drag == vert_drag and the three dynamic weights are equal, so a swap among them computes the same numbers. The vehicles below give every
parameter a value no parameter it could be confused with has:
  heavy       every parameter away from the default; dh != dv, mass != 1, grav far enough from 9.8 for the discrete cost to show it
              through its 1e-6 bar (9.81 moves it by only ~60e-6), speed_eps large enough against the squared speeds for its
              hard-coded value to show, the four weights distinct
  vdrag       the default airframe with the vertical drag only (dh = 0: the flatness map no longer sees the mass)
  hdrag_lowg  a light airframe under low gravity, horizontal drag only, no parasitic drag (speed_eps then enters nothing)

wrong(cfg) lists the mistakes a consumer's parameter block could make — dh and dv swapped, the mass read as 1, a hard-coded gravity, the dynamic
weights swapped pairwise, a hard-coded speed_eps — as configs; effective(cfg, reads) says which of them a consumer could see at all."""
import numpy as np
import isdf_b200 as I

PAR_FIELDS = ("vehicle_mass", "grav_acc", "horiz_drag", "vert_drag", "paras_drag", "speed_eps")
VEHICLES = {
    "heavy": dict(vehicle_mass=1.9, grav_acc=9.6, horiz_drag=0.34, vert_drag=0.07, paras_drag=0.12, speed_eps=1.0,
                  weight_v=700.0, weight_omg=1300.0, weight_theta=2100.0, weight_p=3100.0),
    "vdrag": dict(vehicle_mass=0.61, grav_acc=9.8, horiz_drag=0.0, vert_drag=0.25, paras_drag=0.02, speed_eps=1e-4,
                  weight_v=1000.0, weight_omg=1000.0, weight_theta=1000.0, weight_p=4000.0),
    "hdrag_lowg": dict(vehicle_mass=0.45, grav_acc=3.71, horiz_drag=0.2, vert_drag=0.0, paras_drag=0.0, speed_eps=1e-6,
                       weight_v=1500.0, weight_omg=600.0, weight_theta=900.0, weight_p=4000.0),
}
TAGS = tuple(VEHICLES)


def config(tag, base=None):
    """the default config (or a copy of base) with the vehicle's parameters"""
    cfg = I.default_config_values() if base is None else base.copy()
    for k, v in VEHICLES[tag].items():
        setattr(cfg, k, v)
    return cfg


def par(cfg):
    """{mass, grav, dh, dv, cp, veps}: FlatnessMap::reset's arguments"""
    return np.array([getattr(cfg, f) for f in PAR_FIELDS], dtype=np.float64)


def wrong(cfg):
    """[(name, cfg')]: the vehicle with one plumbing mistake each"""
    def w(**kw):
        c = cfg.copy()
        for k, v in kw.items():
            setattr(c, k, v)
        return c
    return [("dh<->dv", w(horiz_drag=cfg.vert_drag, vert_drag=cfg.horiz_drag)),
            ("mass=1", w(vehicle_mass=1.0)),
            ("grav=9.8", w(grav_acc=9.8)),
            ("wv<->womg", w(weight_v=cfg.weight_omg, weight_omg=cfg.weight_v)),
            ("womg<->wtheta", w(weight_omg=cfg.weight_theta, weight_theta=cfg.weight_omg)),
            ("veps=1e-4", w(speed_eps=1e-4))]


# what each consumer reads, as the quantities its kernels are given: the flatness map (quaternion, body rate and their adjoint) sees the mass only
# through dh / mass and speed_eps only through paras_drag * sqrt(|v|^2 + speed_eps); the thrust adds the mass and dv; the penalties the weights
FLAT = ("dh_over_m", "grav", "cp", "veps")
THRUST = FLAT + ("mass", "dv")
WEIGHTS = ("wv", "womg", "wtheta", "wp")


def effective(cfg, reads):
    """the values of the named quantities at cfg; two configs a consumer cannot tell apart have equal tuples"""
    q = dict(dh_over_m=cfg.horiz_drag / cfg.vehicle_mass, grav=cfg.grav_acc, cp=cfg.paras_drag,
             veps=cfg.speed_eps if cfg.paras_drag != 0.0 else None, mass=cfg.vehicle_mass, dv=cfg.vert_drag,
             wv=cfg.weight_v, womg=cfg.weight_omg, wtheta=cfg.weight_theta, wp=cfg.weight_p)
    return tuple(q[k] for k in reads)


def golden(tag):
    """tests/golden/vehicle_reference.npz at one vehicle: par, the flatness inputs and the reference-compiled outputs on them, and the
    reference-compiled process() records (n x 20) of every states_reference.npz case"""
    import os
    import states_oracle as SO
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vehicle_reference.npz"))
    out = {k: z[f"{tag}_{k}"] for k in ("par", "v", "a", "j", "pg", "vg", "qg", "og", "quat", "omg", "back")}
    cases, _ = SO.load_golden()
    out["cases"] = cases
    out["rec"] = [np.concatenate([c["rec"]["drag"][:, :12], z[f"c{k}_{tag}_att"]], axis=1) for k, c in enumerate(cases)]
    return out


def flat_inputs(cfg, n, seed):
    """n rows of test_reference_pins.flat_inputs kept away from the flatness singularities at this vehicle: |zu| >= 1 and 1 + z_z >= 0.2"""
    from test_reference_pins import flat_inputs as draw
    v, a, j, pg, vg, qg, og = draw(4 * n, seed=seed)
    w = (1.0 + cfg.paras_drag * np.sqrt((v * v).sum(1) + cfg.speed_eps))[:, None] * v
    zu = a + (cfg.horiz_drag / cfg.vehicle_mass) * w
    zu[:, 2] += cfg.grav_acc
    nz = np.linalg.norm(zu, axis=1)
    keep = np.flatnonzero((nz >= 1.0) & (1.0 + zu[:, 2] / nz >= 0.2))[:n]
    assert keep.size == n, "fixture: too few inputs away from the singularities"
    return tuple(np.ascontiguousarray(x[keep]) for x in (v, a, j, pg, vg, qg, og))


def sensitivity(cfg, reads, moved, tol, what):
    """for every wrong vehicle the consumer can see: assert that moved(name, cfg') — the checked output's error metric between the reference at
    cfg' and the reference at cfg — is at least 100 tol, and print the margin; wrong vehicles the consumer cannot see are printed as skipped"""
    base = effective(cfg, reads)
    seen = 0
    for name, wc in wrong(cfg):
        if effective(wc, reads) == base:
            print(f"    {what}: {name:14s} skipped (reads none of the changed quantities)")
            continue
        m = moved(name, wc) / tol
        print(f"    {what}: {name:14s} margin {m:.3e}")
        assert m >= 100.0, f"{what}: the wrong vehicle {name} moves the checked output by only {m:.3e} x the tolerance"
        seen += 1
    assert seen >= 1, f"{what}: no wrong vehicle is visible to this consumer"
    return seen
