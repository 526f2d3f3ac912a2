"""World generators on the GPU (isdf_world_*): every case of tests/golden/world_reference.npz (the reference-compiled generators) bit for
bit through the host and the device form, large worlds byte for byte against the serial restatement tests/world_serial.cpp (tens of
millions of glibc draws across many chunk starts, 4 M-voxel Perlin selections, 200 boxes), the size query and the cap, argument errors,
and the chain into the occupancy map and the depth camera."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import world_oracle as WO

pytestmark = pytest.mark.gpu
GOLDEN = WO.load_golden()


def _torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def ev():
    e = I.Evaluator(I.default_config_values())
    yield e
    e.close()


def _check(got, case, name):
    assert len(got) == case["n"], name
    if "full" in case:
        assert np.array_equal(got.view(np.uint32), case["full"].view(np.uint32)), name
    else:
        assert np.array_equal(got[case["idx"]].view(np.uint32), case["rows"].view(np.uint32)), name
        assert WO.digest(got) == case["sha256"], name


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_golden_host_and_device(ev, name):
    case = GOLDEN[name]
    p = I.world_params(case["kind"], **case["overrides"])
    host = ev.world_cloud(p)
    _check(host, case, name)
    dev = ev.world_cloud_device(p).cpu().numpy()
    assert np.array_equal(host.view(np.uint32), dev.view(np.uint32)), name


LARGE = [("globalmap", dict(map_id=2, cloud_resolution=0.1)),
         ("globalmap", dict(map_id=10, cloud_resolution=0.1)),
         ("globalmap", dict(map_id=9, cloud_resolution=0.1)),
         ("globalmap", dict(map_id=3, cloud_resolution=0.13, rand_seed=4242))] + \
        [("globalmap", dict(map_id=m, srand_seed=s, cloud_resolution=r)) for m in (4, 11) for s, r in ((0, 0.6), (1700000123, 0.1),
                                                                                                      (2 ** 32 - 1, 0.25))] + \
        [("perlin", dict(size=[256, 256, 64], fractal=1)),
         ("perlin", dict(size=[256, 256, 64], fractal=3, attenuation=0.5, complexity=0.02, fill=0.45)),
         ("perlin", dict(size=[97, 61, 33], seed=123456, complexity=0.11, fill=0.05)),
         ("boxes", dict(obstacle_number=200)),
         ("boxes", dict(obstacle_number=200, seed=2 ** 31 + 17, size=[300, 200, 40], width_min=0.1, width_max=2.5))]


@pytest.mark.parametrize("kind,kw", LARGE, ids=[f"{k}-{'-'.join(f'{a}{b}' for a, b in kw.items())}" for k, kw in LARGE])
def test_large_equals_serial(ev, kind, kw):
    p = I.world_params(kind, **kw)
    ref = WO.serial(p)
    got = ev.world_cloud_device(p).cpu().numpy()
    assert len(got) == len(ref)
    assert got.tobytes() == ref.tobytes()


def test_runs_repeat_bit_for_bit(ev):
    for kind, kw in [("globalmap", dict(map_id=10, cloud_resolution=0.2)), ("perlin", dict(size=[128, 96, 40])), ("boxes", {})]:
        p = I.world_params(kind, **kw)
        a = ev.world_cloud_device(p).cpu().numpy()
        b = ev.world_cloud(p)
        c = ev.world_cloud_device(p).cpu().numpy()
        assert a.tobytes() == b.tobytes() == c.tobytes()


def _raw(ev, p, cap, points=None, device=False):
    n = C.c_int64(-1)
    if device:
        rc = ev.lib.isdf_world_cloud_device(ev.h, C.byref(p), cap, C.c_void_p(points), C.byref(n), None)
    else:
        rc = ev.lib.isdf_world_cloud(ev.h, C.byref(p), cap, points.ctypes.data_as(C.c_void_p) if points is not None else None, C.byref(n))
    return rc, n.value


@pytest.mark.parametrize("kind", ["globalmap", "perlin", "boxes"])
def test_size_query_and_cap(ev, kind):
    torch = _torch()
    p = I.world_params(kind, map_id=9)
    full = ev.world_cloud(p)
    rc, n = _raw(ev, p, 0)
    assert rc == -1 and n == len(full) > 0   # a size query: *n written, ISDF_ERR_INVALID since the cloud exceeds cap 0
    for cap in (1, len(full) // 3, len(full) - 1):
        out = np.full((cap + 5, 4), -7.0, dtype=np.float32)
        rc, n = _raw(ev, p, cap, out)
        assert rc == -1
        assert n == len(full)
        assert np.array_equal(out[:cap], full[:cap]) and np.all(out[cap:] == -7.0)
        t = torch.full((cap + 5, 4), -7.0, dtype=torch.float32, device="cuda")
        rc, n = _raw(ev, p, cap, t.data_ptr(), device=True)
        torch.cuda.synchronize()
        assert rc == -1 and n == len(full)
        a = t.cpu().numpy()
        assert np.array_equal(a[:cap], full[:cap]) and np.all(a[cap:] == -7.0)
    out = np.empty((len(full), 4), dtype=np.float32)
    assert _raw(ev, p, len(full), out) == (0, len(full))
    assert np.array_equal(out, full)


def test_unaligned_device_output(ev):
    torch = _torch()
    for kind, kw in [("globalmap", dict(map_id=1)), ("perlin", dict(size=[40, 30, 20])), ("boxes", dict(obstacle_number=5))]:
        p = I.world_params(kind, **kw)
        full = ev.world_cloud(p)
        t = torch.zeros(4 * len(full) + 1, dtype=torch.float32, device="cuda")
        rc, n = _raw(ev, p, len(full), t.data_ptr() + 4, device=True)
        torch.cuda.synchronize()
        assert rc == 0 and n == len(full)
        assert np.array_equal(t[1:].cpu().numpy().reshape(-1, 4), full)


BAD = [dict(kind=0), dict(kind=4), dict(kind=1, map_id=0), dict(kind=1, map_id=12), dict(kind=1, cloud_resolution=0.0),
       dict(kind=1, cloud_resolution=-0.5), dict(kind=1, cloud_resolution=float("nan")), dict(kind=1, cloud_resolution=float("inf")),
       dict(kind=1, init=[float("nan"), 1.0, 1.0]), dict(kind=1, reserved_=[1, 0]), dict(kind=3, reserved_=[0, 2]),
       dict(kind=1, map_id=10, cloud_resolution=1e-9),
       dict(kind=2, size=[0, 10, 10]), dict(kind=2, size=[10, -1, 10]), dict(kind=2, size=[2048, 2048, 512]),
       dict(kind=2, scale=0.0), dict(kind=2, scale=float("nan")), dict(kind=2, fractal=0), dict(kind=2, fractal=31),
       dict(kind=2, complexity=float("inf")), dict(kind=2, fill=float("nan")), dict(kind=2, attenuation=float("nan")),
       dict(kind=2, fill=0.0), dict(kind=2, fill=-0.5), dict(kind=2, complexity=1e9),
       dict(kind=3, width_min=2.0, width_max=1.0), dict(kind=3, obstacle_number=-1), dict(kind=3, width_max=float("inf")),
       dict(kind=3, width_min=4.0, width_max=5.0, size=[100, 100, 300]), dict(kind=3, size=[0, 1, 1]), dict(kind=3, scale=-1.0)]


@pytest.mark.parametrize("kw", BAD, ids=[str(i) for i in range(len(BAD))])
def test_argument_errors(ev, kw):
    kw = dict(kw)
    kind = kw.pop("kind")
    p = I.world_params({2: "perlin", 3: "boxes"}.get(kind, "globalmap"))
    p.kind = kind
    for k, v in kw.items():
        if k in ("init", "size", "reserved_"):
            for i, x in enumerate(v):
                getattr(p, k)[i] = x
        else:
            setattr(p, k, v)
    out = np.empty((4, 4), dtype=np.float32)
    assert _raw(ev, p, 4, out) == (-1, -1)   # refused: *n untouched
    assert _raw(ev, p, 0) == (-1, -1)
    assert ev.lib.isdf_world_cloud_device(ev.h, C.byref(p), 0, None, C.byref(C.c_int64()), None) == -1


def test_null_arguments(ev):
    p = I.world_params("globalmap")
    n = C.c_int64()
    assert ev.lib.isdf_world_cloud(None, C.byref(p), 0, None, C.byref(n)) == -1
    assert ev.lib.isdf_world_cloud(ev.h, None, 0, None, C.byref(n)) == -1
    assert ev.lib.isdf_world_cloud(ev.h, C.byref(p), 0, None, None) == -1
    assert ev.lib.isdf_world_cloud(ev.h, C.byref(p), 5, None, C.byref(n)) == -1
    assert ev.lib.isdf_world_cloud(ev.h, C.byref(p), -1, None, C.byref(n)) == -1
    assert ev.lib.isdf_world_default_params(7, C.byref(p)) == -1


def test_launches_counted(ev):
    for kind in ("globalmap", "perlin", "boxes"):
        before = ev.stats().kernel_launches
        ev.world_cloud(I.world_params(kind, map_id=3))
        assert ev.stats().kernel_launches > before


def test_chain_into_map(ev):
    """set_map_cloud_device(world tensor) builds the grid set_map_cloud builds from the golden cloud (map 9's from the host form after
    checking it against the golden hash), maps 9, 7 and 1 at 0.6 m"""
    for name in ("gm9_r0.6", "gm7_r0.6", "gm1_r0.6"):
        case = GOLDEN[name]
        p = I.world_params(case["kind"], **case["overrides"])
        host = case["full"] if "full" in case else ev.world_cloud(p)
        _check(host, case, name)
        t = ev.world_cloud_device(p)
        ev.set_map_cloud_device(t.data_ptr(), n=t.shape[0], stride_bytes=16, res=0.2)
        info_d, grid_d = ev.map_info(), ev.get_map_u8()
        ev.set_map_cloud(host, 0.2)
        info_h, grid_h = ev.map_info(), ev.get_map_u8()
        assert info_d["dims"] == info_h["dims"] and np.array_equal(info_d["bmin"], info_h["bmin"])
        assert np.array_equal(info_d["bmax"], info_h["bmax"]) and info_d["occupied_voxels"] == info_h["occupied_voxels"]
        assert np.array_equal(grid_d, grid_h) and info_d["occupied_voxels"] > 0


def test_chain_into_sense(ev):
    """set_sense_cloud_device(world tensor) then sense_depth equals the same with the golden cloud from the host"""
    case = GOLDEN["gm7_r0.6"]
    p = I.world_params(case["kind"], **case["overrides"])
    t = ev.world_cloud_device(p)
    rec = np.array([[20.0, 30.0, 5.0, 1.0, 0.0, 0.0, 0.0], [25.0, 10.0, 8.0, 0.9238795325112867, 0.0, 0.0, 0.3826834323650898]])
    ev.set_sense_cloud_device(t.data_ptr(), n=t.shape[0], stride_bytes=16)
    a = ev.sense_depth(rec)
    ev.set_sense_cloud(case["full"])
    b = ev.sense_depth(rec)
    assert np.array_equal(a, b) and (a < 999999).sum() > 1000
