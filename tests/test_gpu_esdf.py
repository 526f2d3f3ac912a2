"""The map's distance field on the GPU (isdf_map_esdf, isdf_get_esdf_f64, isdf_esdf_query(_device)): bit-identity with the
reference-compiled generateESDF3d and queries on every golden case (tests/golden/esdf_reference.npz), with the exact transform
(tests/esdf_oracle.py) on every 16-bit line pattern in each axis order, on 46 341-voxel axes and on a 256^3 map, with exact nearest sites
on sampled voxels of bench.py's 512^3 map, and across the three map setters; then its lifetime, its refusals and its statistics."""
import ctypes as C
import os
import sys
import numpy as np
import pytest
import torch
import esdf_oracle as E
import isdf_b200 as I

pytestmark = pytest.mark.gpu
GOLD = E.load_golden()
FIELDS = list(E.FIELDS)


def evaluator():
    return I.Evaluator(I.default_config_values(), device=0)


def device_query(ev, pts, field, grad=True, stream=None):
    t = torch.as_tensor(np.ascontiguousarray(pts, dtype=np.float64), device="cuda:0")
    if stream is None:
        r = ev.esdf_query_device(t, field=field, grad=grad)
    else:
        with torch.cuda.stream(stream):
            r = ev.esdf_query_device(t, field=field, grad=grad, stream=stream.cuda_stream)
        stream.synchronize()
    torch.cuda.synchronize()
    return (r[0].cpu().numpy(), r[1].cpu().numpy()) if grad else r.cpu().numpy()


@pytest.mark.parametrize("name", sorted(GOLD))
def test_golden_cases_bit_identical(name):
    """every golden map through isdf_set_map_u8: the three readbacks, and both query forms through both entry points. The u8 setter
    frames bmax as bmin + dims * res; where the golden frame differs (the cloud-framed case) the queries are held against the restatement
    on the u8 frame here, and against the golden in test_cloud_framed_queries"""
    d = GOLD[name]
    ev = evaluator()
    ev.set_map_u8(d["occ"], d["bmin"], d["res"])
    ev.map_esdf()
    F = E.fields(d["occ"], d["res"])
    assert np.array_equal(ev.get_esdf("positive"), d["positive"])
    assert np.array_equal(ev.get_esdf("negative"), d["negative"])
    assert np.array_equal(ev.get_esdf("signed"), F["signed"])
    info = ev.map_info()
    same_frame = np.array_equal(info["bmax"], d["bmax"])
    side = torch.cuda.Stream()
    for f in FIELDS:
        if same_frame:
            want_d, want_g, want_v = d[f"{f}_dist"], d[f"{f}_grad"], d[f"{f}_value"]
        else:
            want_d, want_g = E.query(F[f], info["bmin"], info["bmax"], d["res"], d["pts"])
            want_v = E.query(F[f], info["bmin"], info["bmax"], d["res"], d["pts"], grad=False)
        dist, grad = ev.esdf_query(d["pts"], field=f)
        assert np.array_equal(dist, want_d) and np.array_equal(grad, want_g), f
        assert np.array_equal(ev.esdf_query(d["pts"], field=f, grad=False), want_v), f
        dd, dg = device_query(ev, d["pts"], f, stream=side)
        assert np.array_equal(dd, want_d) and np.array_equal(dg, want_g), f
        assert np.array_equal(device_query(ev, d["pts"], f, grad=False), want_v), f
    ev.close()


def test_cloud_framed_queries():
    """a cloud-built map keeps the cloud's maximum as bmax, and the queries' isInMap uses it: the golden cloud case, built from one point
    per occupied voxel plus the two frame corners, against the reference-compiled queries with that bmax"""
    d = GOLD["cloud"]
    res, bmin, bmax = d["res"], d["bmin"], d["bmax"]
    idx = np.argwhere(d["occ"] != 0)
    # a quarter voxel in from each voxel's lower corner: the top layer's points stay at or below bmax, which lies below its centres
    pts = np.concatenate([(idx + 0.25) * res + bmin, [bmin, bmax]]).astype(np.float32)
    ev = evaluator()
    ev.set_map_cloud(pts, res)
    info = ev.map_info()
    assert info["dims"] == tuple(d["occ"].shape) and np.array_equal(info["bmin"], bmin) and np.array_equal(info["bmax"], bmax)
    assert np.array_equal(ev.get_map_u8(), d["occ"])
    ev.map_esdf()
    assert np.array_equal(ev.get_esdf("positive"), d["positive"]) and np.array_equal(ev.get_esdf("negative"), d["negative"])
    for f in FIELDS:
        dist, grad = ev.esdf_query(d["pts"], field=f)
        assert np.array_equal(dist, d[f"{f}_dist"]) and np.array_equal(grad, d[f"{f}_grad"]), f
        dd, dg = device_query(ev, d["pts"], f)
        assert np.array_equal(dd, d[f"{f}_dist"]) and np.array_equal(dg, d[f"{f}_grad"]), f
        assert np.array_equal(ev.esdf_query(d["pts"], field=f, grad=False), d[f"{f}_value"]), f
    ev.close()


def check_exact(ev, occ, res, bmin=(0.0, 0.0, 0.0)):
    ev.set_map_u8(occ, bmin, res)
    ev.map_esdf()
    pos, neg = ev.get_esdf("positive"), ev.get_esdf("negative")
    ep, en = E.field(occ != 0, res), E.field(occ == 0, res)
    assert np.array_equal(pos, ep), f"{int((pos != ep).sum())} positive voxels differ"
    assert np.array_equal(neg, en), f"{int((neg != en).sum())} negative voxels differ"
    return pos, neg


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_all_line_patterns_exact(axis):
    bits = ((np.arange(65536)[:, None] >> np.arange(16)) & 1).astype(np.uint8).reshape(256, 256, 16)
    ev = evaluator()
    check_exact(ev, np.ascontiguousarray(np.moveaxis(bits, 2, axis)), 0.125)
    ev.close()


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_46341_voxel_axes_exact(axis):
    rng = np.random.default_rng(46341 + axis)
    shape = [2, 3, 2]
    shape[axis] = 46341
    ev = evaluator()
    for dens in (1e-4, 0.5):
        check_exact(ev, (rng.random(shape) < dens).astype(np.uint8), 1.0)
    ev.close()


def test_random_256_cubed_exact():
    occ = (np.random.default_rng(256).random((256, 256, 256), dtype=np.float32) < 0.02).astype(np.uint8)
    ev = evaluator()
    check_exact(ev, occ, 0.25, bmin=(-3.0, 1.0, 0.5))
    ev.close()


@pytest.mark.parametrize("case", ["single", "empty", "full", "ragged_z"])
def test_special_maps_exact(case):
    rng = np.random.default_rng(5)
    occ = np.zeros((7, 5, 1100), np.uint8)   # z spans two 1024-voxel chunks of pass z
    if case == "single":
        occ[3, 2, 1099] = 1
    elif case == "full":
        occ[:] = 1
    elif case == "ragged_z":
        occ[:, :, rng.integers(0, 1100, 3)] = 1
        occ[2, :, 1030:1040] = 1
    ev = evaluator()
    check_exact(ev, occ, 0.5)
    ev.close()


def _nearest_d2(occ, site_value, pts):
    """exact squared voxel distance from each (i, j, k) to the nearest voxel with occ == site_value: grow a cube around the voxel until
    the best distance found inside it is at most its half-width (nothing outside the cube can then be closer)"""
    dims = np.array(occ.shape)
    out = np.empty(len(pts), dtype=np.int64)
    for n, p in enumerate(pts):
        r = 1
        while True:
            lo, hi = np.maximum(p - r, 0), np.minimum(p + r + 1, dims)
            win = occ[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] == site_value
            if win.any():
                q = np.argwhere(win) + lo
                best = int(((q - p) ** 2).sum(axis=1).min())
                if best <= r * r or (lo == 0).all() and (hi == dims).all():
                    out[n] = best
                    break
            r *= 2
    return out


def test_bench_map_sampled_exact():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    w, _, occ, *_ = bench.make_workload()
    ev = evaluator()
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.map_esdf()
    rng = np.random.default_rng(512)
    vox = rng.integers(0, occ.shape[0], size=(10000, 3))
    centres = vox + 0.5
    for f, site in (("positive", 1), ("negative", 0)):
        got = device_query(ev, centres, f, grad=False)   # at a voxel centre the query returns that voxel's value exactly
        want = np.sqrt(_nearest_d2(occ, site, vox).astype(np.float64))
        assert np.array_equal(got, want), f"{f}: {int((got != want).sum())} of {len(vox)} sampled voxels differ"
    ev.close()


def test_three_setters_same_field():
    """the same occupancy through isdf_set_map_u8, isdf_set_map_f64 and isdf_set_map_cloud gives the same fields; queries on the cloud
    map use the cloud's bmax (inside the top voxel layer)"""
    rng = np.random.default_rng(9)
    occ = (rng.random((40, 33, 70)) < 0.08).astype(np.uint8)
    occ[0, 0, 0] = occ[-1, -1, -1] = 1   # the cloud's frame corners lie in these voxels
    bmin, res = np.array([0.0, 0.0, 0.0]), 0.5
    F = E.fields(occ, res)
    ev = evaluator()
    top = bmin + (np.array(occ.shape) - 0.25) * res
    pts = np.concatenate([(np.argwhere(occ != 0) + 0.5) * res + bmin, [bmin, top]]).astype(np.float32)
    for name, setter in (("u8", lambda: ev.set_map_u8(occ, bmin, res)), ("f64", lambda: ev.set_map_f64(occ.astype(np.float64), bmin, res)),
                         ("cloud", lambda: ev.set_map_cloud(pts, res))):
        setter()
        assert np.array_equal(ev.get_map_u8(), occ), name
        ev.map_esdf()
        for f in FIELDS:
            assert np.array_equal(ev.get_esdf(f), F[f]), (name, f)
    info = ev.map_info()
    assert np.array_equal(info["bmax"], top)
    q = bmin + rng.random((500, 3)) * (np.array(occ.shape) * res + 1.0) - 0.5
    q[:50, 0] = top[0] + rng.random(50) * 0.25 * res   # between the cloud's bmax and bmin + X * res
    for f in FIELDS:
        dist, grad = ev.esdf_query(q, field=f)
        rd, rg = E.query(F[f], info["bmin"], info["bmax"], res, q)
        assert np.array_equal(dist, rd) and np.array_equal(grad, rg), f
    ev.close()


# ---- lifetime, refusals, statistics -------------------------------------------------------------------------------------------
def _code(fn):
    with pytest.raises(I.IsdfError) as e:
        fn()
    return e.value.code


def test_state_errors():
    ev = evaluator()
    assert _code(ev.map_esdf) == -2
    occ = np.zeros((4, 5, 6), np.uint8)
    occ[1, 2, 3] = 1
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    assert _code(lambda: ev.get_esdf("positive")) == -2
    assert _code(lambda: ev.esdf_query(np.zeros((2, 3)))) == -2
    assert _code(lambda: ev.esdf_query_device(torch.zeros((2, 3), dtype=torch.float64, device="cuda:0"))) == -2
    ev.close()


def test_setters_and_lifetime():
    rng = np.random.default_rng(3)
    occ = (rng.random((10, 12, 14)) < 0.2).astype(np.uint8)
    ev = evaluator()
    ev.set_map_u8(occ, [0, 0, 0], 0.5)
    ev.map_esdf()
    before = [ev.get_esdf(f) for f in FIELDS]
    # refused setters: bad sizes (checked before the device), a cloud without a finite point (refused after its bounds pass)
    L, bmin = ev.lib, np.zeros(3)
    assert L.isdf_set_map_u8(ev.h, occ.ctypes.data_as(C.POINTER(C.c_uint8)), 0, 12, 14, bmin.ctypes.data_as(C.POINTER(C.c_double)), 0.5) == -1
    assert _code(lambda: ev.set_map_cloud(np.full((5, 3), np.nan, np.float32), 0.5)) == -1
    assert _code(lambda: ev.set_map_u8(np.zeros((46342, 1, 1), np.uint8), [0, 0, 0], -1.0)) == -1
    for f, b in zip(FIELDS, before):
        assert np.array_equal(ev.get_esdf(f), b), f
    # rebuilding replaces the field
    ev.map_esdf()
    for f, b in zip(FIELDS, before):
        assert np.array_equal(ev.get_esdf(f), b), f
    # a successful setter gives it up, for every setter
    for setter in (lambda: ev.set_map_u8(occ, [0, 0, 0], 0.5), lambda: ev.set_map_f64(occ.astype(np.float64), [0, 0, 0], 0.5),
                   lambda: ev.set_map_cloud(np.array([[0, 0, 0], [3, 3, 3]], np.float32), 0.5)):
        ev.set_map_u8(occ, [0, 0, 0], 0.5)
        ev.map_esdf()
        setter()
        assert _code(lambda: ev.get_esdf("positive")) == -2
        ev.map_esdf()
        ev.get_esdf("positive")
    ev.close()


def test_unsupported_long_axis():
    ev = evaluator()
    ev.set_map_u8(np.zeros((46342, 1, 1), np.uint8), [0, 0, 0], 1.0)
    with pytest.raises(I.IsdfError) as e:
        ev.map_esdf()
    assert e.value.code == -4 and "int" in str(e.value) and "46341" in str(e.value)
    assert _code(lambda: ev.get_esdf("positive")) == -2
    ev.close()


def test_invalid_arguments():
    ev = evaluator()
    occ = np.zeros((4, 5, 6), np.uint8)
    occ[1, 2, 3] = 1
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.map_esdf()
    L, h = ev.lib, ev.h
    out = np.zeros(occ.size)
    pts, dist, grad = np.zeros((3, 3)), np.zeros(3), np.zeros((3, 3))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    assert L.isdf_map_esdf(None) == -1
    assert L.isdf_get_esdf_f64(None, 0, dp(out), out.size) == -1
    assert L.isdf_get_esdf_f64(h, 0, None, out.size) == -1
    assert L.isdf_get_esdf_f64(h, 0, dp(out), out.size - 1) == -1
    assert L.isdf_get_esdf_f64(h, 0, dp(out), -1) == -1
    for bad in (-1, 3):
        assert L.isdf_get_esdf_f64(h, bad, dp(out), out.size) == -1
        assert L.isdf_esdf_query(h, bad, dp(pts), 3, dp(dist), dp(grad)) == -1
        assert L.isdf_esdf_query_device(h, bad, None, 0, None, None, None) == -1
    assert L.isdf_esdf_query(None, 0, dp(pts), 3, dp(dist), dp(grad)) == -1
    assert L.isdf_esdf_query(h, 0, None, 3, dp(dist), dp(grad)) == -1
    assert L.isdf_esdf_query(h, 0, dp(pts), 3, None, dp(grad)) == -1
    assert L.isdf_esdf_query(h, 0, dp(pts), -1, dp(dist), dp(grad)) == -1
    t = torch.zeros((3, 3), dtype=torch.float64, device="cuda:0")
    td = torch.zeros(3, dtype=torch.float64, device="cuda:0")
    assert L.isdf_esdf_query_device(h, 0, None, 3, C.c_void_p(td.data_ptr()), None, None) == -1
    assert L.isdf_esdf_query_device(h, 0, C.c_void_p(t.data_ptr()), 3, None, None, None) == -1
    assert L.isdf_esdf_query_device(h, 0, C.c_void_p(t.data_ptr()), -1, C.c_void_p(td.data_ptr()), None, None) == -1
    with pytest.raises(ValueError):
        ev.get_esdf("both")
    # nothing above disturbed the field
    assert np.array_equal(ev.get_esdf("positive"), E.field(occ != 0, 1.0))
    ev.close()


def test_non_finite_points_give_nan():
    ev = evaluator()
    ev.set_map_u8(np.ones((3, 3, 3), np.uint8), [0, 0, 0], 1.0)
    ev.map_esdf()
    d, g = ev.esdf_query(np.array([[np.nan, 1, 1], [1, np.inf, 1], [1.5, 1.5, 1.5]]))
    assert np.isnan(d[:2]).all() and np.isnan(g[:2]).all() and np.isfinite(d[2])
    ev.close()


def test_kernel_launches_counted_and_nothing_else():
    ev = evaluator()
    occ = (np.random.default_rng(1).random((20, 21, 22)) < 0.1).astype(np.uint8)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    fields = ["evals_discrete", "evals_swept", "last_pairs", "last_sdf_evals", "last_kernel_ms"]

    def snap():
        s = ev.stats()
        return s.kernel_launches, [getattr(s, k) for k in fields]

    k0, rest0 = snap()
    ev.map_esdf()
    k1, rest1 = snap()
    assert k1 - k0 == 3 and rest1 == rest0
    out = np.empty(occ.size)   # the C call itself: get_esdf asks isdf_get_map_info for the dimensions, which launches a kernel too
    assert ev.lib.isdf_get_esdf_f64(ev.h, 2, out.ctypes.data_as(C.POINTER(C.c_double)), out.size) == 0
    k2, rest2 = snap()
    assert k2 - k1 == 1 and rest2 == rest0
    ev.esdf_query(np.random.default_rng(2).random((100, 3)) * 20, field="negative")
    device_query(ev, np.zeros((5, 3)), "positive")
    k3, rest3 = snap()
    assert k3 - k2 == 2 and rest3 == rest0
    ev.close()
