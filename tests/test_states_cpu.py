"""CPU checks of tests/golden/states_reference.npz (the reference-compiled state of process() on reference-MINCO trajectories), which the GPU
test holds isdf_trajectory_states to bit for bit:
  * where the reference tree exists, regenerating the fixture gives the committed bits;
  * everywhere, the oracle's trajectory evaluation (orc::Traj) gives its pos / vel / acc / jer bits, the numpy restatement of
    FlatnessMap::forward at yaw 0 its quat / omg / thr bits, and the oracle's flatness map (optimizated_forward) the same quat and omg values;
  * the new entry points refuse a NULL context without touching the GPU."""
import ctypes as C
import os
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import states_oracle as SO

REFERENCE = "/root/reference"


def test_fixture_covers_the_stated_cases():
    cases, _ = SO.load_golden()
    assert [c["N"] for c in cases] == [1, 2, 7, 64, 290]
    for c in cases:
        cs = np.cumsum(c["T"])
        t = c["times"]
        assert np.isin(cs[:-1], t).all() and np.isin(np.nextafter(cs[:-1], np.inf), t).all() and np.isin(np.nextafter(cs[:-1], -np.inf), t).all()
        assert (t < 0).any() and (t > cs[-1]).any() and 0.0 in t
        for tag in SO.TAGS:
            assert c["rec"][tag].shape == (t.size, 20) and np.isfinite(c["rec"][tag]).all()


@pytest.mark.skipif(not os.path.isfile(os.path.join(REFERENCE, "src", "utils", "include", "utils", "flatness.hpp")), reason="reference tree absent")
def test_fixture_regenerates_from_the_reference():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_states_golden", os.path.join(os.path.dirname(SO.GOLDEN), "make_states_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    live = mk.compute(REFERENCE)
    z = np.load(SO.GOLDEN)
    assert sorted(live) == sorted(z.files)
    for k in z.files:
        assert SO.same_bits(live[k], z[k]), k


def test_fixture_equals_oracle_trajectory_and_flatness_restatement():
    cases, par = SO.load_golden()
    for c in cases:
        pvaj, _, _, total = O.traj_eval(c["T"], c["coeffs"], c["times"])
        assert total == np.cumsum(c["T"])[-1]
        for tag in SO.TAGS:
            rec = c["rec"][tag]
            assert SO.same_bits(pvaj, rec[:, :12]), f"N={c['N']} {tag}: pos/vel/acc/jer"
            v, a, j = rec[:, 3:6], rec[:, 6:9], rec[:, 9:12]
            q, o, thr = SO.flat_forward_yaw0(par[tag], v, a, j)
            assert SO.same_bits(q, rec[:, 12:16]) and SO.same_bits(o, rec[:, 16:19]) and SO.same_bits(thr, rec[:, 19]), f"N={c['N']} {tag}: attitude"
            oq, oo = O.flat_forward_batch(O.config_from(SO.config_for(tag)), v, a, j)
            # optimizated_forward is forward at yaw 0 up to the signs of zero products
            assert np.array_equal(oq, rec[:, 12:16]) and np.array_equal(oo, rec[:, 16:19]), f"N={c['N']} {tag}: oracle flatness"


def test_null_context_is_refused():
    lib = I.load_library()
    ip = C.POINTER(C.c_int32)
    off, T, Cc = np.array([0, 1], dtype=np.int32), np.ones(1), np.zeros(18)
    tr, tm, out = np.zeros(1, dtype=np.int32), np.zeros(1), np.full(20, 7.0)
    assert lib.isdf_trajectory_states(None, 1, off.ctypes.data_as(ip), I._dp(T), I._dp(Cc), 1, tr.ctypes.data_as(ip), I._dp(tm), I._dp(out)) == -1
    assert lib.isdf_trajectory_states_device(None, 1, None, None, None, 1, None, None, None, None) == -1
    assert lib.isdf_pose_points(None, 1, I._dp(out), 1, I._dp(T), I._dp(out)) == -1
    assert lib.isdf_pose_points_device(None, 1, None, 1, None, None, None) == -1
    assert (out == 7.0).all()
