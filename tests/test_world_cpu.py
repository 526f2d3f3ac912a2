"""CPU checks of the world generators (include/isdf.h, isdf_world_*): the glibc rand() jump-ahead the library uses (isdf_dbg_world_rand,
the same __host__ __device__ routine the kernels start their chunks from) against libc's own rand(), the serial restatement
tests/world_serial.cpp against tests/golden/world_reference.npz, and both against the reference-compiled generators
(oracle/_ref/libref_world.so) where that library exists."""
import ctypes as C
import os
import numpy as np
import pytest
import isdf_b200 as I
import world_oracle as WO

GOLDEN = WO.load_golden()


def _jump(seed, offsets):
    L = I.load_library()
    L.isdf_dbg_world_rand.argtypes = [C.c_uint32, C.c_void_p, C.c_int64, C.c_void_p]
    off = np.ascontiguousarray(offsets, dtype=np.uint64)
    out = np.empty(len(off), dtype=np.int32)
    assert L.isdf_dbg_world_rand(seed, off.ctypes.data, len(off), out.ctypes.data) == 0
    return out


@pytest.mark.parametrize("seed", [0, 1, 12345])
def test_jump_ahead_equals_libc_rand(seed):
    libc = C.CDLL(None)
    libc.rand.restype = C.c_int
    n = 100001
    libc.srand(seed)
    ref = np.array([libc.rand() for _ in range(n)], dtype=np.int32)
    assert np.array_equal(_jump(seed, np.arange(n)), ref)


@pytest.mark.parametrize("seed", [0, 1, 12345])
def test_jump_ahead_far_offsets(seed):
    offs = [10 ** 7, 10 ** 7 + 30, 10 ** 7 + 31]
    got = _jump(seed, offs)
    assert [int(g) for g in got] == [WO.rand_at(seed, o) for o in offs]


def test_jump_ahead_beyond_2_31():
    o = (1 << 31) + 5
    assert int(_jump(12345, [o])[0]) == WO.rand_at(12345, o)


def test_seed_zero_is_seed_one():
    offs = np.arange(0, 5000, 7)
    assert np.array_equal(_jump(0, offs), _jump(1, offs))


def _params(case):
    return I.world_params(case["kind"], **case["overrides"])


def _check(got, case, name):
    assert got is not None and len(got) == case["n"], name
    if "full" in case:
        assert np.array_equal(got.view(np.uint32), case["full"].view(np.uint32)), name
    else:
        assert np.array_equal(got[case["idx"]].view(np.uint32), case["rows"].view(np.uint32)), name
        assert WO.digest(got) == case["sha256"], name


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_serial_equals_golden(name):
    _check(WO.serial(_params(GOLDEN[name])), GOLDEN[name], name)


def test_golden_params_are_current_defaults():
    """the stored parameter sets are the launch-file defaults with the stored overrides (so a default change shows up here)"""
    for name, case in GOLDEN.items():
        p = _params(case)
        for k, v in case["params"].items():
            got = getattr(p, k)
            assert (list(got) if k in ("init", "size", "reserved_") else got) == v, (name, k)


def test_time_seed_reaches_maps_4_and_11():
    for m in (4, 11):
        a, b = (GOLDEN[f"gm{m}_r0.6_s{s}"]["full"] for s in (0, 1700000000))
        assert len(a) == len(b) and not np.array_equal(a, b)
        assert np.array_equal(a[:10], b[:10])   # the two walls before srand(time(NULL)): 5 points each at 0.6 m


def test_defaults():
    g, p, b = (I.world_params(k) for k in ("globalmap", "perlin", "boxes"))
    assert (g.kind, g.map_id, g.rand_seed, g.cloud_resolution, list(g.init)) == (1, 4, 1, 0.6, [1.0, 1.0, 1.0])
    assert (p.kind, p.seed, list(p.size), p.scale, p.complexity, p.fill, p.fractal, p.attenuation) == \
        (2, 511, [100, 100, 30], 10.0, 0.03, 0.3, 1, 0.1)
    assert (b.kind, b.obstacle_number, b.width_min, b.width_max) == (3, 50, 0.6, 1.5)


@pytest.mark.skipif(not os.path.exists(WO.REF_WORLD), reason="oracle/_ref/libref_world.so not built (needs the reference tree)")
@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_reference_equals_golden_and_serial(name):
    p = _params(GOLDEN[name])
    ref = WO.ref(p)
    _check(ref, GOLDEN[name], name)
    assert np.array_equal(ref.view(np.uint32), WO.serial(p).view(np.uint32))


@pytest.mark.skipif(not os.path.exists(WO.REF_WORLD), reason="oracle/_ref/libref_world.so not built (needs the reference tree)")
def test_reference_equals_serial_beyond_golden():
    for kind, kw in [("globalmap", dict(map_id=4, srand_seed=12345, cloud_resolution=0.3)),
                     ("globalmap", dict(map_id=2, rand_seed=0, init=[14.6, 52.0, 1.0])),
                     ("globalmap", dict(map_id=9, cloud_resolution=0.45)),
                     ("perlin", dict(size=[30, 20, 10], fill=0.9, fractal=2, seed=3)),
                     ("boxes", dict(seed=99, obstacle_number=30, size=[60, 40, 20], scale=5.0))]:
        p = I.world_params(kind, **kw)
        assert np.array_equal(WO.ref(p).view(np.uint32), WO.serial(p).view(np.uint32)), (kind, kw)
