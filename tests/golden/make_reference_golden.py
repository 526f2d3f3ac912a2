"""Golden vectors computed by REFERENCE-COMPILED code (oracle/_ref/*.so built from /root/reference by `make -C oracle ref`).
Run in the build container (where /root/reference exists):  python tests/golden/make_reference_golden.py
  flat_reference.npz — inputs and outputs of the reference's utils/flatness.hpp (optimizated_forward, backwardthreadsafe);
  ref_meshes.npz     — the robot meshes the reference ships and loads down its mesh Generalshape path (src/plan_manager/shapes/
                       {Lthick,drone,kuang,box,RoundedCone,mybox}.obj; INPUT data, read with the product's OBJ reader), the
                       poly_params of the config that names them, seeded query points, and the winding numbers the
                       reference-compiled igl/FastWindingNumberForSoups.h returns for them (order 2, accuracy scale 2.0: Shape.cpp:86,110);
  minco_reference.npz — outputs of the reference's utils/minco.hpp (MINCO_S3NU forward, energy gradients, propogateGrad) on seeded problems, and
                        of its utils/trajectory.hpp (getPos_Vel_Acc_Jerk, locatePieceIdx, getTotalDuration) on the resulting trajectories;
  lbfgs_reference.npz — what the reference's utils/lbfgs.hpp does on seeded problems: every evaluated point, solution, value, return code;
  grid_reference.npz  — the reference's map_manager/src/Gridmap3D.cpp: grid indices, cube centres, in-map flags and AABB gathers on seeded grids;
  ref_shapes_obj.npz  — the bytes of the OBJ files behind ref_meshes.npz, so that the product's OBJ reader is checked on the files themselves;
  sign_policy_reference.npz — the oracle's discrete cost and gradient with the reference-faithful sign s = 1 - 2 w (w from the reference-compiled
                        FWN header) on the inputs of test_gpu_reference_pins.py::test_sign_policy_deviation_from_reference_faithful_fwn;
  lbfgs_branches_reference.npz — what the reference's utils/lbfgs.hpp does on every case of tests/lbfgs_cases.py: every evaluated point,
                        solution, value, return code and evaluation count (for the one case pinned to the product's host driver, that
                        driver's run, with the reference build's beside it under ref_*).
`python tests/golden/make_reference_golden.py lbfgs_branches` writes only the last file (any of the functions below can be named)."""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "implicit-sdf-planner_b200", "py"))
import isdf_b200 as I          # noqa: E402
import lbfgs_cases as LC       # noqa: E402
import oracle_lib as O         # noqa: E402
from test_reference_pins import flat_inputs, _minco_cases, _lbfgs_problems, _traj_times, _grid_cases   # noqa: E402
from test_gpu_reference_pins import sign_policy_case, SIGN_POLICY_MESHES   # noqa: E402


REF_SHAPES = "/root/reference/src/plan_manager/shapes"
# mesh -> poly_params: config_L.yaml:8-10 (Lthick), config_CappedCone.yaml:8-10 (RoundedCone), config_box.yaml:8-11 (mybox); drone / kuang /
# box are named by no shipped config (sw_manager.hpp:255-275 sends any unknown name down the mesh path): CappedCone's parameters
MESHES = {"Lthick": [0, 0, 0, 0, 0, 0], "RoundedCone": [0, 0, 0, 120, 0, 0], "mybox": [0, 0, 0, 0, 0, 0],
          "drone": [0, 0, 0, 120, 0, 0], "kuang": [0, 0, 0, 120, 0, 0], "box": [0, 0, 0, 120, 0, 0]}


def ref_meshes():
    import host_lib as H
    import workloads as W
    out = {}
    for name, pp in MESHES.items():
        V, F = H.read_obj(os.path.join(REF_SHAPES, name + ".obj"))
        R, t = W.rotation_from_poly_params(pp)
        Vt = V @ R.T + t                                            # Shape.cpp:38-50
        lo, hi = Vt.min(0) - 1.0, Vt.max(0) + 1.0
        rng = np.random.default_rng(abs(hash(name)) % 1000 + 5 if False else sum(map(ord, name)))
        q = lo + (hi - lo) * rng.random((600, 3))
        w = O.RefFwn(Vt, F, order=2).query(q, 2.0)
        out[name + "_V"], out[name + "_F"], out[name + "_pp"], out[name + "_q"], out[name + "_w"] = V, F, np.array(pp, float), q, w
        print(name, V.shape, F.shape, "w range", w.min(), w.max())
    np.savez_compressed(os.path.join(HERE, "ref_meshes.npz"), names=np.array(list(MESHES)), **out)
    print("ref_meshes.npz written")
    raw = {name: np.frombuffer(open(os.path.join(REF_SHAPES, name + ".obj"), "rb").read(), dtype=np.uint8) for name in MESHES}
    np.savez_compressed(os.path.join(HERE, "ref_shapes_obj.npz"), **raw)
    print("ref_shapes_obj.npz written")


def sign_policy_reference():
    out = {}
    for name in SIGN_POLICY_MESHES:
        cfg, occ, T, Cc, V, F, pp = sign_policy_case(name)
        c, gC, gT, _ = O.eval_discrete(O.config_from(cfg), occ, [0, 0, 0], 1.0, O.Shape.mesh(V, F, pp, wn_mode=O.WN_REF), T, Cc)
        out.update({f"{name}_cost": np.array(c), f"{name}_gradC": gC, f"{name}_gradT": gT})
    np.savez_compressed(os.path.join(HERE, "sign_policy_reference.npz"), **out)
    print("sign_policy_reference.npz written")


def lbfgs_branches():
    import host_lib as H
    rl = O.RefLbfgs()
    cs = LC.cases()
    out = {"names": np.array([c["name"] for c in cs])}
    for k, c in enumerate(cs):
        f1, kw = LC.one(c["fun"]), LC.sequential_kwargs(c)
        a = rl.minimize(f1, c["x0"], **kw)
        runs = [("", a)]
        if c["host_pinned"]:
            runs = [("", H.lbfgs_minimize(f1, c["x0"], **kw)), ("ref_", a)]
        for pre, r in runs:
            out.update({f"c{k}_{pre}trace": np.array(r["trace"]).reshape(len(r["trace"]), -1), f"c{k}_{pre}x": r["x"], f"c{k}_{pre}f": np.array(r["f"]),
                        f"c{k}_{pre}ret": np.array(r["ret"]), f"c{k}_{pre}evals": np.array(r["evaluations"])})
        print(c["name"], a["ret"], a["evaluations"])
    np.savez_compressed(os.path.join(HERE, "lbfgs_branches_reference.npz"), **out)
    print("lbfgs_branches_reference.npz written")


def main():
    O.build()
    ref_meshes()
    sign_policy_reference()
    cfg = O.config_from(I.default_config_values())
    ref = O.RefFlat(cfg)
    v, a, j, pg, vg, qg, og = flat_inputs(256, seed=123)
    q, o = ref.forward(v, a, j)
    b = ref.backward(v, a, j, pg, vg, qg, og)
    np.savez(os.path.join(HERE, "flat_reference.npz"), par=ref.par, v=v, a=a, j=j, pg=pg, vg=vg, qg=qg, og=og, quat=q, omg=o, back=b)
    print("flat_reference.npz written")
    rm = O.RefMinco()
    out = {}
    for k, (N, head, tail, inPs, T, gC, gT) in enumerate(_minco_cases()):
        co, e, gc, gt = rm.forward(head, tail, inPs, T)
        gp, gto = rm.backward(head, tail, inPs, T, gC, gT)
        out.update({f"c{k}_coeffs": co, f"c{k}_energy": np.array(e), f"c{k}_gdC": gc, f"c{k}_gdT": gt, f"c{k}_gradP": np.asarray(gp), f"c{k}_gradT": gto})
        times = _traj_times(T, np.random.default_rng(100 + k))
        ev, piece, tloc, total = rm.traj_eval(head, tail, inPs, T, times)
        out.update({f"c{k}_times": times, f"c{k}_pvaj": ev, f"c{k}_piece": piece, f"c{k}_tloc": tloc, f"c{k}_total": np.array(total)})
    np.savez_compressed(os.path.join(HERE, "minco_reference.npz"), ncases=np.array(len(_minco_cases())), **out)
    print("minco_reference.npz written")
    rl = O.RefLbfgs()
    out = {}
    for k, (name, fun, x0, kw) in enumerate(_lbfgs_problems()):
        r = rl.minimize(fun, x0, **kw)
        out.update({f"p{k}_trace": np.array(r["trace"]), f"p{k}_x": r["x"], f"p{k}_f": np.array(r["f"]), f"p{k}_ret": np.array(r["ret"]), f"p{k}_evals": np.array(r["evaluations"])})
        print(name, r["ret"], r["evaluations"])
    np.savez_compressed(os.path.join(HERE, "lbfgs_reference.npz"), nproblems=np.array(len(_lbfgs_problems())), **out)
    print("lbfgs_reference.npz written")
    rg = O.RefGrid()
    out = {}
    for k, (dims, bmin, res, pts, occ, boxes) in enumerate(_grid_cases()):
        idx, ctr, inm = rg.index(dims, bmin, res, pts)
        out.update({f"g{k}_idx": idx, f"g{k}_centre": ctr, f"g{k}_inmap": inm})
        for b, (centre, half) in enumerate(boxes):
            p_, n_ = rg.points_in_aabb(occ, bmin, res, centre, half)
            out.update({f"g{k}_b{b}_pts": p_, f"g{k}_b{b}_n": np.array(n_)})
    np.savez_compressed(os.path.join(HERE, "grid_reference.npz"), **out)
    print("grid_reference.npz written")


if __name__ == "__main__":
    if len(sys.argv) > 1:
        O.build()
        for fn in sys.argv[1:]:
            globals()[fn]()
    else:
        main()
        lbfgs_branches()
