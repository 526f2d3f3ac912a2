"""isdf_map_fuse_cloud / _device: fusion into a cloud-built map equals the cloud of the union, fusion into an empty frame equals the
restatement (tests/navigate_oracle.py) for any split and order, the counts, the distance field given up and rebuilt, refusals that leave
the map, host = device, and the reference camera's sensed points fused as the restatement fuses their host copy."""
import numpy as np
import pytest
import isdf_b200 as I
import navigate_oracle as NO

pytestmark = pytest.mark.gpu


def _cloud(rng, n, lo, hi):
    return rng.uniform(lo, hi, (n, 3)).astype(np.float32)


def _empty(ev, dims, bmin, res):
    ev.set_map_u8(np.zeros(dims, dtype=np.uint8), bmin, res)
    info = ev.map_info()
    return info["bmin"], info["bmax"]


def test_fuse_into_a_cloud_map_equals_the_union():
    rng = np.random.default_rng(1)
    c1 = _cloud(rng, 4000, [0, 0, 0], [6, 5, 3])
    c1[:2] = [[0, 0, 0], [6, 5, 3]]        # the bounds of C1
    c2 = _cloud(rng, 3000, [0, 0, 0], [6, 5, 3])
    a, b = I.Evaluator(), I.Evaluator()
    a.set_map_cloud(c1, 0.25)
    info0 = a.map_info()
    got = a.map_fuse_cloud(c2)
    b.set_map_cloud(np.concatenate([c1, c2]), 0.25)
    assert np.array_equal(a.get_map_u8(), b.get_map_u8())
    info = a.map_info()
    assert info["dims"] == info0["dims"] and np.array_equal(info["bmax"], info0["bmax"])
    assert info["occupied_voxels"] == info0["occupied_voxels"] + got["voxels_added"] == b.map_info()["occupied_voxels"]
    assert (info["points_used"], info["points_skipped"]) == (info0["points_used"], info0["points_skipped"])
    assert got["points_used"] == len(c2) and got["points_outside"] == got["points_skipped"] == 0
    a.close(); b.close()


def test_fuse_splits_and_permutations_match_the_restatement():
    rng = np.random.default_rng(2)
    dims, bmin, res = (40, 30, 20), np.array([-2.0, 1.0, 0.5]), 0.2
    cloud = _cloud(rng, 20000, bmin - 0.5, bmin + np.array(dims) * res + 0.5)
    cloud[::97] = np.nan
    cloud[5::101, 1] = np.inf
    ev = I.Evaluator()
    lo, hi = _empty(ev, dims, bmin, res)
    ref, cnt = NO.fuse(np.zeros(dims, np.uint8), lo, hi, res, cloud)
    for seed, parts in ((0, 1), (1, 3), (2, 17)):
        _empty(ev, dims, bmin, res)
        perm = cloud[np.random.default_rng(seed).permutation(len(cloud))]
        tot = dict(points_used=0, points_outside=0, points_skipped=0, voxels_added=0)
        for part in np.array_split(perm, parts):
            got = ev.map_fuse_cloud(part)
            for k in tot:
                tot[k] += got[k]
        assert np.array_equal(ev.get_map_u8(), ref), (seed, parts)
        assert tot == cnt and ev.map_info()["occupied_voxels"] == int(ref.sum()) == tot["voxels_added"]
    assert cnt["points_outside"] > 0 and cnt["points_skipped"] > 0
    ev.close()


def test_fuse_gives_up_the_field_and_refusals_leave_the_map():
    rng = np.random.default_rng(3)
    dims, bmin, res = (24, 20, 16), np.zeros(3), 0.5
    ev, fresh = I.Evaluator(), I.Evaluator()
    _empty(ev, dims, bmin, res)
    ev.map_fuse_cloud(_cloud(rng, 500, 0, 8))
    ev.map_esdf()
    ev.map_fuse_cloud(_cloud(rng, 500, 0, 8))
    with pytest.raises(I.IsdfError) as e:
        ev.get_esdf("positive")
    assert e.value.code == -2
    ev.map_esdf()
    fresh.set_map_u8(ev.get_map_u8(), bmin, res)
    fresh.map_esdf()
    for f in ("positive", "negative", "signed"):
        assert np.array_equal(ev.get_esdf(f).view(np.uint64), fresh.get_esdf(f).view(np.uint64)), f
    # refusals: no map, a bad stride, no record; the map and its field stay
    before = ev.get_map_u8()
    with pytest.raises(I.IsdfError) as e:
        ev.map_fuse_cloud(np.zeros(40, dtype=np.float32), stride_bytes=10)
    assert e.value.code == -1
    with pytest.raises(I.IsdfError):
        ev.map_fuse_cloud(np.zeros((0, 3), dtype=np.float32))
    assert np.array_equal(ev.get_map_u8(), before) and ev.get_esdf("positive").size == np.prod(dims)
    empty = I.Evaluator()
    with pytest.raises(I.IsdfError) as e:
        empty.map_fuse_cloud(_cloud(rng, 10, 0, 1))
    assert e.value.code == -2
    ev.close(); fresh.close(); empty.close()


def test_host_and_device_forms_agree():
    import torch
    rng = np.random.default_rng(4)
    dims, bmin, res = (50, 40, 12), np.array([0.0, 0.0, 0.0]), 0.1
    cloud = np.concatenate([_cloud(rng, 30000, -0.2, 5.2), np.ones((30000, 1), np.float32)], 1)   # stride 16 records
    a, b = I.Evaluator(), I.Evaluator()
    _empty(a, dims, bmin, res); _empty(b, dims, bmin, res)
    ha = a.map_fuse_cloud(cloud)
    hb = b.map_fuse_cloud_device(torch.as_tensor(cloud, device="cuda"), stream=torch.cuda.current_stream().cuda_stream)
    assert ha == hb and np.array_equal(a.get_map_u8(), b.get_map_u8())
    a.close(); b.close()


def test_fused_sensed_points_match_the_restatement():
    import torch
    rng = np.random.default_rng(5)
    ev = I.Evaluator()
    scene = _cloud(rng, 60000, [2, -3, 0], [8, 3, 3])
    ev.set_sense_cloud(scene)
    dims, bmin, res = (48, 32, 16), np.array([0.0, -4.0, 0.0]), 0.25
    lo, hi = _empty(ev, dims, bmin, res)
    poses = torch.zeros((3, 7), dtype=torch.float64, device="cuda")
    poses[:, 0] = torch.tensor([0.0, 0.5, 1.0], dtype=torch.float64)
    poses[:, 2] = 1.5
    poses[:, 3] = 1.0
    pts, off = ev.sense_cloud_device(poses, 0, 3)
    got = ev.map_fuse_cloud_device(pts, stream=torch.cuda.current_stream().cuda_stream)
    ref, cnt = NO.fuse(np.zeros(dims, np.uint8), lo, hi, res, pts.cpu().numpy())
    assert pts.shape[0] > 1000 and got == cnt and np.array_equal(ev.get_map_u8(), ref)
    ev.close()
