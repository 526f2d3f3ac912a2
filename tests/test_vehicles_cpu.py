"""The oracle and the restatements at vehicles other than the default one (tests/vehicles.py), CPU only.

tests/golden/vehicle_reference.npz holds what the reference's own utils/flatness.hpp computes at those vehicles (made by
tests/golden/make_vehicle_golden.py); every pin below holds where the reference tree is absent. Also: the config's path from Python to the
oracle's orc_config and to the library's isdf_config, field by field, and the helper parameters the restatements derive from it."""
import ctypes as C
import os
import re
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import states_oracle as SO
import certify_oracle as CE
import dynlimits_oracle as DO
import vehicles as VH
from test_reference_pins import relerr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("tag", VH.TAGS)
def test_flatness_oracle_equals_reference_at_vehicle(tag):
    """orc::Flat forward and adjoint against the reference-compiled flatness.hpp at the vehicle, to the tolerances of
    test_flatness_oracle_equals_committed_reference_outputs; where oracle/_ref exists the live library reproduces the fixture bit for bit.
    The flatness map reads neither dv nor the weights (nor the mass when dh = 0, nor speed_eps when cp = 0): those wrong vehicles are skipped."""
    z = VH.golden(tag)
    cfg = VH.config(tag)
    assert np.array_equal(z["par"], VH.par(cfg))
    ins = [z[k] for k in ("v", "a", "j", "pg", "vg", "qg", "og")]
    if O.ref_flat_available():
        ref = O.RefFlat(O.config_from(cfg))
        q, o = ref.forward(*ins[:3])
        assert np.array_equal(q, z["quat"]) and np.array_equal(o, z["omg"]) and np.array_equal(ref.backward(*ins), z["back"])

    def err(c):
        q, o = O.flat_forward_batch(O.config_from(c), *ins[:3])
        b = O.flat_backward_batch(O.config_from(c), *ins)
        return relerr(q, z["quat"]) / 1e-15, relerr(o, z["omg"]) / 1e-12, relerr(b, z["back"]) / 1e-12

    assert max(err(cfg)) <= 1.0, err(cfg)
    VH.sensitivity(cfg, VH.FLAT, lambda _, c: max(err(c)), 1.0, f"oracle flatness [{tag}]")


@pytest.mark.parametrize("tag", VH.TAGS)
def test_states_restatement_equals_reference_at_vehicle(tag):
    """states_oracle.flat_forward_yaw0 (dh / mass in the attitude, dv raw in the thrust) reproduces the reference-compiled process() records'
    attitude, body rate and thrust bit for bit at the vehicle; a wrong vehicle moves them by far more than an ulp"""
    z = VH.golden(tag)
    moved = {name: 0.0 for name, _ in VH.wrong(VH.config(tag))}
    for rec in z["rec"]:
        q, o, thr = SO.flat_forward_yaw0(z["par"], rec[:, 3:6], rec[:, 6:9], rec[:, 9:12])
        assert SO.same_bits(np.concatenate([q, o, thr[:, None]], axis=1), rec[:, 12:20])
        for name, wc in VH.wrong(VH.config(tag)):
            q, o, thr = SO.flat_forward_yaw0(VH.par(wc), rec[:, 3:6], rec[:, 6:9], rec[:, 9:12])
            moved[name] = max(moved[name], relerr(np.concatenate([q, o, thr[:, None]], axis=1), rec[:, 12:20]))
    VH.sensitivity(VH.config(tag), VH.THRUST, lambda name, _: moved[name], 2.0 ** -52, f"states restatement [{tag}]")


def _struct_fields(text, name):
    """field names of a C struct in declaration order"""
    body = re.search(r"struct " + name + r"\s*\{(.*?)\}", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            fields += [f.strip() for f in re.sub(r"^\s*(double|int32_t|int)\s+", "", decl).split(",")]
    return fields


def test_config_reaches_every_same_named_slot():
    """every field of the Python Config set to a distinct value: oracle_lib.config_from carries each to the same-named orc_config slot, and the
    Python mirrors declare the fields of include/isdf.h's isdf_config and oracle_capi.cpp's orc_config in their order"""
    names = [n for n, _ in I.Config._fields_]
    hdr = open(os.path.join(ROOT, "include", "isdf.h")).read()
    orc = open(os.path.join(ROOT, "oracle", "oracle_capi.cpp")).read()
    assert _struct_fields(hdr, "isdf_config") == names
    assert _struct_fields(orc, "orc_config") == names == [n for n, _ in O.OrcConfig._fields_]
    cfg = I.Config()
    for k, (n, t) in enumerate(I.Config._fields_):
        setattr(cfg, n, (k + 1) * 1.25 + 0.125 if t is C.c_double else 100 + k)
    o = O.config_from(cfg)
    for n, _ in I.Config._fields_:
        assert getattr(o, n) == getattr(cfg, n), n
    assert len({getattr(cfg, n) for n in names}) == len(names)


def test_default_config_values_equal_the_library_default():
    lib = I.load_library()
    d = I.Config()
    assert lib.isdf_default_config(C.byref(d)) == 0
    assert bytes(d) == bytes(I.default_config_values())
    for tag in VH.TAGS:   # a vehicle changes only the vehicle and weight fields
        v = VH.config(tag)
        for n, _ in I.Config._fields_:
            if n not in VH.VEHICLES[tag]:
                assert getattr(v, n) == getattr(d, n), (tag, n)


@pytest.mark.parametrize("tag", VH.TAGS)
def test_restatement_helper_parameters_at_vehicle(tag):
    """the restatements derive FlatnessMap::reset's quantities as the reference does (flatness.hpp:36-51): dh_over_m = dh / mass in the
    attitude, dv and mass raw in the thrust"""
    cfg = VH.config(tag)
    z = VH.golden(tag)
    assert CE.flat_params(cfg) == (cfg.horiz_drag / cfg.vehicle_mass, cfg.paras_drag, cfg.speed_eps, cfg.grav_acc)
    for rec in z["rec"][:3]:
        ok = np.isfinite(rec).all(axis=1)
        v, a, j, q, thr = rec[ok, 3:6], rec[ok, 6:9], rec[ok, 9:12], rec[ok, 12:16], rec[ok, 19]
        scale = np.maximum(np.abs(thr), 1.0)
        assert np.max(np.abs(DO.thrust_exact(cfg, v, a) - thr) / scale) <= 1e-12
        # the dynamic-limit enclosure at a point: its thrust channel is the reference thrust to rounding
        lo, hi = DO.channels(cfg, [DO.Iv(v[:, k]) for k in range(3)], [DO.Iv(a[:, k]) for k in range(3)], [DO.Iv(j[:, k]) for k in range(3)])
        assert np.max(np.abs(lo[:, 4] - thr) / scale) <= 1e-12 and np.max(np.abs(hi[:, 4] - thr) / scale) <= 1e-12
        # the certificate's closed-form attitude: z of R(z) is the reference quaternion's body z axis
        for r in range(0, len(thr), max(1, len(thr) // 16)):
            c = np.zeros((3, 6)); c[:, 1], c[:, 2], c[:, 3] = v[r], 0.5 * a[r], j[r] / 6.0
            _, R = CE.pose_closed_form(cfg, c, 0.0)
            w, x, y, zz = q[r]
            zq = np.array([2 * (x * zz + w * y), 2 * (y * zz - w * x), 1 - 2 * (x * x + y * y)])
            assert np.abs(R[:, 2] - zq).max() <= 1e-12
    # the tag's own states config for the two fixture tags still carries the default vehicle
    assert np.array_equal(VH.par(SO.config_for("drag")), VH.par(I.default_config_values()))
