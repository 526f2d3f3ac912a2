"""The map's distance field without a GPU: the reference-compiled generateESDF3d is the exact integer Euclidean distance transform
followed by res * sqrt((double)d2), bit for bit (the definition isdf_map_esdf restates), it is undefined past 46 341 voxels on an axis,
its grid_map_buffer_all adds the occupancy where ISDF_ESDF_SIGNED adds the positive distance, and the restated trilinear query equals
the reference's. The reference-compiled cases need oracle/_ref/libref_esdf.so; the golden cases run from tests/golden alone."""
import os
import numpy as np
import pytest
import esdf_oracle as E

needs_ref = pytest.mark.skipif(not E.ref_available(), reason="oracle/_ref/libref_esdf.so not built (needs the reference tree)")


def _all_patterns(axis):
    """every 16-bit pattern as one line along `axis` of a 256 x 256 x 16 map (in that axis order)"""
    bits = ((np.arange(65536)[:, None] >> np.arange(16)) & 1).astype(np.uint8).reshape(256, 256, 16)
    return np.moveaxis(bits, 2, axis).copy()


def _check_exact(occ, res, bmin=(0.0, 0.0, 0.0)):
    pos, neg, _ = E.ref_esdf(occ, bmin, res)
    assert np.array_equal(pos, E.field(occ != 0, res))
    assert np.array_equal(neg, E.field(occ == 0, res))


@needs_ref
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_reference_is_exact_transform_all_line_patterns(axis):
    _check_exact(_all_patterns(axis), 0.125)


@needs_ref
@pytest.mark.parametrize("dens", [0.001, 0.01, 0.3, 0.7])
def test_reference_is_exact_transform_random(dens):
    rng = np.random.default_rng(int(dens * 1000))
    occ = (rng.random((37, 53, 70)) < dens).astype(np.uint8)
    _check_exact(occ, 0.25, bmin=(-1.0, 2.0, 0.5))


@needs_ref
@pytest.mark.parametrize("case", ["single", "empty", "full"])
def test_reference_is_exact_transform_special(case):
    occ = np.zeros((9, 11, 13), np.uint8)
    if case == "single":
        occ[4, 5, 6] = 1
    if case == "full":
        occ[:] = 1
    _check_exact(occ, 0.5)
    if case != "single":   # one field has no site: res * sqrt(DBL_MAX), not inf
        pos, neg, _ = E.ref_esdf(occ, (0, 0, 0), 0.5)
        assert np.all((pos if case == "empty" else neg) == 0.5 * np.sqrt(np.finfo(np.float64).max))


@needs_ref
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_reference_is_exact_at_46341_voxels(axis):
    rng = np.random.default_rng(46341 + axis)
    shape = [2, 2, 2]
    shape[axis] = 46341
    occ = (rng.random(shape) < 1e-4).astype(np.uint8)
    _check_exact(occ, 1.0)


@needs_ref
def test_reference_differs_past_46341_voxels():
    """fillESDF's int q * q overflows at q = 46341: the negative field of a 2 x 2 x 46342 map is no longer the exact transform, which is
    why isdf_map_esdf refuses such maps"""
    rng = np.random.default_rng(46342)
    occ = (rng.random((2, 2, 46342)) < 1e-4).astype(np.uint8)
    pos, neg, _ = E.ref_esdf(occ, (0, 0, 0), 1.0)
    assert not np.array_equal(neg, E.field(occ == 0, 1.0))


def _golden_cases():
    return E.load_golden() if os.path.exists(E.GOLDEN) else {}


def test_golden_fields_are_exact_transform():
    G = _golden_cases()
    assert G, "tests/golden/esdf_reference.npz missing"
    for nm, d in G.items():
        F = E.fields(d["occ"], d["res"])
        assert np.array_equal(F["positive"], d["positive"]), nm
        assert np.array_equal(F["negative"], d["negative"]), nm


def test_buffer_all_adds_occupancy_where_signed_adds_distance():
    """grid_map_buffer_all = occ + (-neg + res) where neg > 0, occ elsewhere; ISDF_ESDF_SIGNED has the positive distance in occ's place"""
    for nm, d in _golden_cases().items():
        occ, neg, res = d["occ"].astype(np.float64), d["negative"], d["res"]
        expect = occ.copy()
        m = neg > 0.0
        expect[m] += (-neg[m] + res)
        assert np.array_equal(d["all"], expect), nm
        # neg > 0 exactly at occupied voxels (pos = 0 there): buffer_all is 1 + (-neg + res) inside obstacles and 0 in free space, where
        # SIGNED is (-neg + res) inside and the positive distance outside
        assert np.array_equal(m, d["occ"] != 0) and np.all(d["positive"][m] == 0.0), nm
        sgn = E.signed(d["positive"], neg, res)
        assert np.array_equal(sgn[m], -neg[m] + res) and np.array_equal(sgn[~m], d["positive"][~m]), nm
        assert np.all(d["all"][~m] == 0.0) and np.array_equal(d["all"][m], 1.0 + (-neg[m] + res)), nm


@pytest.mark.parametrize("field", list(E.FIELDS))
def test_golden_query_restated(field):
    """the numpy restatement of getSDFValueWithGrad / getSDFValue equals the reference-compiled queries stored in the goldens"""
    for nm, d in _golden_cases().items():
        vals = E.fields(d["occ"], d["res"])[field]
        dist, grad = E.query(vals, d["bmin"], d["bmax"], d["res"], d["pts"])
        assert np.array_equal(dist, d[f"{field}_dist"]), nm
        assert np.array_equal(grad, d[f"{field}_grad"]), nm
        assert np.array_equal(E.query(vals, d["bmin"], d["bmax"], d["res"], d["pts"], grad=False), d[f"{field}_value"]), nm


@needs_ref
@pytest.mark.parametrize("field", list(E.FIELDS))
def test_reference_query_equals_restated(field):
    for nm, d in _golden_cases().items():
        dist, grad = E.ref_query(d["occ"], d["bmin"], d["res"], field, d["pts"], bmax=d["bmax"])
        vals = E.fields(d["occ"], d["res"])[field]
        rd, rg = E.query(vals, d["bmin"], d["bmax"], d["res"], d["pts"])
        assert np.array_equal(dist, rd) and np.array_equal(grad, rg), nm


@needs_ref
def test_goldens_regenerate_identically(tmp_path):
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_esdf_golden", os.path.join(os.path.dirname(E.GOLDEN), "make_esdf_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    fresh = mod.generate()
    old = np.load(E.GOLDEN)
    assert set(fresh) == set(old.files)
    for k in old.files:
        assert np.array_equal(np.asarray(fresh[k]), old[k]), k
