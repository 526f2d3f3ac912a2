"""cloud_reference.npz: the occupancy grids the reference's global-map handler (PCSmapManager::rcvGlobalMapHandler,
PCSmap_manager.cpp:111-181) builds from the seeded clouds of tests/cloud_oracle.py::cloud_cases, with the reference-compiled
createGridMap / getGridIndex (oracle/_ref/libref_grid.so, built by `make -C oracle ref`) under the restated bounds / count / threshold glue.
Run where the reference tree exists:  python tests/golden/make_cloud_golden.py
Per case: the records (uint8) and their stride, res, dims, bmin, bmax and, per threshold in cloud_oracle.THRESHOLDS, the occupancy as
np.packbits of the flattened X*Y*Z grid. Writes only this file; the other fixtures are untouched."""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cloud_oracle as CO   # noqa: E402
import oracle_lib as O      # noqa: E402


def main():
    O.build()
    assert os.path.exists(O.REF_GRID), "oracle/_ref/libref_grid.so is missing: run `make -C oracle ref` where the reference tree exists"
    out, names = {}, []
    for name, (raw, stride, res) in CO.cloud_cases().items():
        names.append(name)
        out[name + "_raw"], out[name + "_stride"], out[name + "_res"] = raw, np.int32(stride), np.float64(res)
        for thr in CO.THRESHOLDS:
            r = CO.ref_map(raw, stride, res, thr)
            out[name + "_dims"], out[name + "_bmin"], out[name + "_bmax"] = np.array(r["dims"], np.int32), r["bmin"], r["bmax"]
            out[f"{name}_occ_t{thr}"] = np.packbits(r["occ"].reshape(-1))
            print(name, "n", raw.size // stride, "res", res, "dims", r["dims"], "thr", thr, "occupied", int(r["occ"].sum()))
    np.savez_compressed(CO.FIXTURE, names=np.array(names), **out)
    print("cloud_reference.npz written")


if __name__ == "__main__":
    main()
