"""World generators (include/isdf.h, isdf_world_*) restated serially, and the reference-compiled generators — TEST INFRASTRUCTURE.

  build()                                  tests/world_serial.cpp -> libworld_serial.so next to the library objects (no contraction)
  rand_at(seed, offset)                    glibc rand() after srand(seed) with offset draws discarded, by libc itself
  serial(p)                                the (n, 4) float32 cloud of isdf_world_params p by the serial restatement (None where tpos is out
                                           of range)
  ref(p)                                   the same by oracle/_ref/libref_world.so (oracle/world.mk): the reference's own globalmap_gene.cpp
                                           and mockamap maps.cpp / perlinnoise.cpp; None when that library is absent
  load_golden()                            tests/golden/world_reference.npz (tests/golden/make_world_golden.py) as {case: dict}
  digest(a)                                SHA-256 of an (n, 4) float32 cloud's records
"""
import ctypes as C
import hashlib
import os
import subprocess
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ORACLE_DIR = os.path.join(ROOT, "oracle")
SRC = os.path.join(HERE, "world_serial.cpp")
LIB = os.path.join(ROOT, "implicit-sdf-planner_b200", "build", "libworld_serial.so")
REF_WORLD = os.path.join(ORACLE_DIR, "_ref", "libref_world.so")
GOLDEN = os.path.join(HERE, "golden", "world_reference.npz")
GLOBALMAP, PERLIN, BOXES = 1, 2, 3
fp, dp = C.POINTER(C.c_float), C.POINTER(C.c_double)


def build(force=False):
    if force or not os.path.exists(LIB) or os.path.getmtime(SRC) > os.path.getmtime(LIB):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", LIB, SRC])
    # the reference-compiled generators: make's dependency check decides; without the reference tree whatever library exists is kept
    subprocess.call(["make", "-C", ORACLE_DIR, "-f", "world.mk"] + (["-B"] if force else []), stdout=subprocess.DEVNULL)


_lib, _ref = None, None


def _bind(L, prefix):
    f = getattr(L, prefix + "globalmap")
    f.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.c_double, dp, fp, C.c_longlong]
    f.restype = C.c_longlong
    f = getattr(L, prefix + "perlin")
    f.argtypes = [C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, fp, C.c_longlong]
    f.restype = C.c_longlong
    f = getattr(L, prefix + "boxes")
    f.argtypes = [C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double, C.c_double, fp, C.c_longlong]
    f.restype = C.c_longlong
    return L


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = _bind(C.CDLL(LIB), "world_serial_")
        _lib.world_serial_rand_at.argtypes = [C.c_uint32, C.c_uint64]
        _lib.world_serial_rand_at.restype = C.c_int32
    return _lib


def ref_lib():
    """oracle/_ref/libref_world.so, or None"""
    global _ref
    if _ref is None and os.path.exists(REF_WORLD):
        _ref = _bind(C.CDLL(REF_WORLD), "ref_world_")
    return _ref


def rand_at(seed, offset):
    return int(lib().world_serial_rand_at(seed, offset))


def _run(L, prefix, p):
    def call(out, cap):
        ptr = out.ctypes.data_as(fp)
        if p.kind == GLOBALMAP:
            init = (C.c_double * 3)(*p.init)
            return getattr(L, prefix + "globalmap")(p.map_id, p.rand_seed, p.srand_seed, p.cloud_resolution, init, ptr, cap)
        if p.kind == PERLIN:
            return getattr(L, prefix + "perlin")(p.seed, p.size[0], p.size[1], p.size[2], p.scale, p.complexity, p.fill, p.attenuation,
                                                  p.fractal, ptr, cap)
        return getattr(L, prefix + "boxes")(p.seed, p.size[0], p.size[1], p.size[2], p.scale, p.obstacle_number, p.width_min, p.width_max,
                                            ptr, cap)
    if p.kind == PERLIN:   # one pass: the voxel count bounds the cloud
        out = np.empty((max(p.size[0] * p.size[1] * p.size[2], 1), 4), dtype=np.float32)
        n = call(out, out.shape[0])
    else:
        n = call(np.empty((1, 4), dtype=np.float32), 0)
        out = np.empty((max(n, 1), 4), dtype=np.float32)
        n = call(out, n)
    return None if n < 0 else out[:n]


def serial(p):
    return _run(lib(), "world_serial_", p)


def ref(p):
    L = ref_lib()
    return None if L is None else _run(L, "ref_world_", p)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def load_golden():
    """{case name: dict(params=dict of isdf_world_params fields, n, sha256, and full (n, 4) or rows + idx)}"""
    import json
    z = np.load(GOLDEN)
    meta = json.loads(str(z["meta"]))
    out = {}
    for name, m in meta.items():
        d = dict(m)
        for k in ("full", "rows", "idx"):
            key = f"{name}/{k}"
            if key in z.files:
                d[k] = z[key]
        out[name] = d
    return out
