"""Writes tests/golden/esdf_reference.npz: the reference-compiled generateESDF3d (grid_esdf, grid_map_buffer_neg, grid_map_buffer_all)
and getSDFValue / getSDFValueWithGrad on every field, for small maps, from oracle/_ref/libref_esdf.so (oracle/esdf.mk).

    python tests/golden/make_esdf_golden.py [out.npz]

Maps have non-cubic dimensions with Z not a multiple of 32, and (dims, res) pairs for which createGridMap(bmin, bmin + X*res) gives X
back (dyadic resolutions). The cloud-framed case has bmax != bmin + X*res, as isdf_set_map_cloud leaves it. Query points: voxel centres,
voxel faces, the first half voxel, the upper faces, points outside on every side and random interior points.
"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import esdf_oracle as E  # noqa: E402


def cases():
    rng = np.random.default_rng(20261017)
    out = []
    for name, dens in (("rand1", 0.01), ("rand30", 0.30), ("rand70", 0.70)):
        out.append((name, rng.random((13, 17, 40)) < dens, [-1.5, 0.25, 2.0], 0.25, None))
    single = np.zeros((9, 11, 35), bool)
    single[4, 7, 33] = True
    out.append(("single", single, [0.0, 0.0, 0.0], 0.5, None))
    out.append(("empty", np.zeros((5, 6, 7), bool), [1.0, -2.0, 0.5], 0.125, None))
    out.append(("full", np.ones((5, 6, 7), bool), [1.0, -2.0, 0.5], 0.125, None))
    # cloud-framed: bmax is the cloud's maximum, inside the top voxel layer (ceil((bmax - bmin) / res) still gives the dims). The frame
    # is exact in float32 and both corner voxels are occupied, so a cloud of the occupied centres plus the points bmin and bmax gives
    # this map back through isdf_set_map_cloud.
    cloud = rng.random((12, 10, 33)) < 0.05
    cloud[0, 0, 0] = cloud[-1, -1, -1] = True
    bmin = np.array([-0.75, 0.5, -1.25])
    bmax = bmin + np.array([11.25, 9.5, 32.375]) * 0.25
    out.append(("cloud", cloud, bmin, 0.25, bmax))
    return out


def points(dims, bmin, bmax, res, rng):
    dims, bmin, bmax = np.array(dims), np.asarray(bmin, float), np.asarray(bmax, float)
    top = bmin + dims * res
    P = []
    idx = rng.integers(0, dims, size=(40, 3))
    centres = (idx + 0.5) * res + bmin
    P.append(centres)                                                       # voxel centres
    faces = centres.copy()
    ax = rng.integers(0, 3, 40)
    faces[np.arange(40), ax] += np.where(rng.random(40) < 0.5, -0.5, 0.5) * res
    P.append(faces)                                                         # voxel faces
    lo = bmin + rng.random((30, 3)) * (dims * res)
    a = rng.integers(0, 3, 30)
    lo[np.arange(30), a] = bmin[a] + rng.random(30) * 0.5 * res
    P.append(lo)                                                            # the first half voxel on one axis
    up = bmin + rng.random((36, 3)) * (dims * res)
    for k in range(36):
        a = k % 3
        up[k, a] = (bmax[a], top[a], top[a] - 0.5 * res, bmax[a] - 0.25 * res)[k // 3 % 4]
    P.append(up)                                                            # the upper faces (both bmax and bmin + dims * res)
    out = []
    for a in range(3):
        for s in (-1, 1):
            q = bmin + rng.random((4, 3)) * (dims * res)
            q[:, a] = (bmin[a] - (0.1 + rng.random(4)) * res * 3) if s < 0 else (bmax[a] + (0.1 + rng.random(4)) * res * 3)
            out.append(q)
    P.append(np.concatenate(out))                                           # outside, every side
    P.append(bmin + rng.random((100, 3)) * (dims * res))                   # random interior
    return np.concatenate(P)


def generate():
    rng = np.random.default_rng(7)
    z = {}
    names = []
    for name, occ, bmin, res, bmax in cases():
        occ = occ.astype(np.uint8)
        bmin = np.asarray(bmin, dtype=np.float64)
        bmax = bmin + np.array(occ.shape) * res if bmax is None else np.asarray(bmax, dtype=np.float64)
        pos, neg, al = E.ref_esdf(occ, bmin, res, bmax=bmax)
        pts = points(occ.shape, bmin, bmax, res, rng)
        names.append(name)
        z[f"{name}/dims"] = np.array(occ.shape, dtype=np.int64)
        z[f"{name}/occ_bits"] = np.packbits(occ.reshape(-1))
        z[f"{name}/bmin"], z[f"{name}/bmax"], z[f"{name}/res"] = bmin, bmax, np.float64(res)
        z[f"{name}/positive"], z[f"{name}/negative"], z[f"{name}/all"] = pos, neg, al
        z[f"{name}/pts"] = pts
        for f in E.FIELDS:
            d, g = E.ref_query(occ, bmin, res, f, pts, grad=True, bmax=bmax)
            z[f"{name}/{f}_dist"], z[f"{name}/{f}_grad"] = d, g
            z[f"{name}/{f}_value"] = E.ref_query(occ, bmin, res, f, pts, grad=False, bmax=bmax)
    z["names"] = np.array(names)
    return z


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else E.GOLDEN
    np.savez_compressed(out, **generate())
    print("wrote", out, os.path.getsize(out), "bytes")
