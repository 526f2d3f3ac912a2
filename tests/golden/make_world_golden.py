"""Writes tests/golden/world_reference.npz: the reference's own world generators (oracle/_ref/libref_world.so, built by oracle/world.mk
from map_manager/src/globalmap_gene.cpp and mockamap's maps.cpp / perlinnoise.cpp) on the cases of world_oracle-style parameter sets below.
Small clouds are stored whole; larger ones as their size, the SHA-256 of their float32 records and SAMPLED rows at fixed indices. Every
case is also checked against the serial restatement (tests/world_serial.cpp) before it is written. Needs the reference tree; run from the
repository root: python tests/golden/make_world_golden.py"""
import json
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "implicit-sdf-planner_b200", "py"))
import isdf_b200 as I  # noqa: E402
import world_oracle as WO  # noqa: E402

FULL = 10000     # clouds up to this size are stored whole
SAMPLED = 256    # rows stored of a larger cloud


def cases():
    """{name: (kind, overrides)}"""
    c = {}
    for m in range(1, 12):
        if m in (4, 11):
            for s in (0, 1700000000):
                c[f"gm{m}_r0.6_s{s}"] = ("globalmap", dict(map_id=m, srand_seed=s))
        else:
            c[f"gm{m}_r0.6"] = ("globalmap", dict(map_id=m))
    c["gm3_r0.3"] = ("globalmap", dict(map_id=3, cloud_resolution=0.3))
    c["gm9_r0.3"] = ("globalmap", dict(map_id=9, cloud_resolution=0.3))
    c["gm2_r0.6_rand7"] = ("globalmap", dict(map_id=2, rand_seed=7, init=[20.0, 30.0, 1.0]))
    c["perlin_a"] = ("perlin", dict(size=[48, 40, 16]))
    c["perlin_fractal3"] = ("perlin", dict(size=[40, 30, 20], fractal=3, complexity=0.07, attenuation=0.5, fill=0.38))
    c["perlin_seed7"] = ("perlin", dict(seed=7, size=[32, 32, 12], complexity=0.142857, fill=0.2))
    c["perlin_default"] = ("perlin", dict())
    c["boxes_511"] = ("boxes", dict())
    c["boxes_12"] = ("boxes", dict(seed=12, obstacle_number=20, width_min=0.3, width_max=2.0))
    return c


def fields(p):
    return {k: (list(getattr(p, k)) if k in ("init", "size", "reserved_") else getattr(p, k)) for k, _ in p._fields_}


def main():
    meta, arrays = {}, {}
    for name, (kind, kw) in cases().items():
        p = I.world_params(kind, **kw)
        ref = WO.ref(p)
        assert ref is not None, "oracle/_ref/libref_world.so is missing: make -C oracle -f world.mk"
        ser = WO.serial(p)
        assert np.array_equal(ref.view(np.uint32), ser.view(np.uint32)), f"{name}: the serial restatement differs from the reference"
        n = len(ref)
        meta[name] = dict(kind=kind, overrides=kw, params=fields(p), n=n, sha256=WO.digest(ref))
        if n <= FULL:
            arrays[f"{name}/full"] = ref
        else:
            idx = np.unique(np.concatenate([np.linspace(0, n - 1, SAMPLED // 2).astype(np.int64),
                                            np.random.default_rng(len(name)).integers(0, n, SAMPLED // 2)]))
            arrays[f"{name}/idx"], arrays[f"{name}/rows"] = idx, ref[idx]
    path = os.path.join(HERE, "world_reference.npz")
    np.savez_compressed(path, meta=np.array(json.dumps(meta, sort_keys=True)), **arrays)
    print("wrote", path, {k: v["n"] for k, v in meta.items()})


if __name__ == "__main__":
    main()
