"""Depth sensing (include/isdf.h, isdf_sense_*) restated serially, and the reference-compiled renderer — TEST INFRASTRUCTURE.

  build()                               tests/sense_serial.cpp -> libsense_serial.so next to the library objects (no contraction)
  pose(pos, quat, cam_to_body)          (cam2world, camera-from-world as the FP32 matrix the render uses, widened to double[16])
  render(rec, T, params)                one depth image (H, W) from a double[16] camera-from-world, and the records skipped
  depth(rec, pos, quat, params)         Q depth images as isdf_sense_depth defines them
  cloud(rec, pos, quat, params)         (points (M, 3) float32, offsets (Q + 1) int64) as isdf_sense_cloud defines them
  ref_render(rec, T, params)            oracle/_ref/libref_depth.so (oracle/depth.mk): the reference's own DepthRender::render_pose
  load_golden()                         tests/golden/sense_reference.npz (tests/golden/make_sense_golden.py)
"""
import ctypes as C
import os
import subprocess
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ORACLE_DIR = os.path.join(ROOT, "oracle")
SRC = os.path.join(HERE, "sense_serial.cpp")
LIB = os.path.join(ROOT, "implicit-sdf-planner_b200", "build", "libsense_serial.so")
REF_DEPTH = os.path.join(ORACLE_DIR, "_ref", "libref_depth.so")
GOLDEN = os.path.join(HERE, "golden", "sense_reference.npz")
dp, fp, ip = C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int32)


def build(force=False):
    deps = [SRC]
    if force or not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", LIB, SRC])
    # the reference-compiled renderer: make's dependency check decides; without the reference tree whatever library exists is kept
    subprocess.call(["make", "-C", ORACLE_DIR, "-f", "depth.mk"] + (["-B"] if force else []), stdout=subprocess.DEVNULL)


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.sense_pose.argtypes = [dp, dp, dp, dp, dp]
        L.sense_render.argtypes = [fp, C.c_longlong, C.c_int, dp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, ip]
        L.sense_render.restype = C.c_longlong
        L.sense_backproject.argtypes = [ip, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, dp, dp, C.c_double, fp]
        L.sense_backproject.restype = C.c_longlong
        _lib = L
    return _lib


def _d(a):
    return a.ctypes.data_as(dp)


def _records(rec):
    """(float32 array, records, stride in floats) of an (n, k >= 3) float32 array"""
    rec = np.ascontiguousarray(rec, dtype=np.float32)
    rec = rec.reshape(rec.shape[0], -1)
    return rec, rec.shape[0], rec.shape[1]


def pose(pos, quat, cam_to_body):
    c2w, cw = np.empty(16), np.empty(16)
    lib().sense_pose(_d(np.ascontiguousarray(pos, dtype=np.float64)), _d(np.ascontiguousarray(quat, dtype=np.float64)),
                     _d(np.ascontiguousarray(cam_to_body, dtype=np.float64).reshape(16)), _d(c2w), _d(cw))
    return c2w, cw


def render(rec, T, p):
    rec, n, s = _records(rec)
    img = np.empty((p.height, p.width), dtype=np.int32)
    sk = lib().sense_render(rec.ctypes.data_as(fp), n, s, _d(np.ascontiguousarray(T, dtype=np.float64).reshape(16)), p.width, p.height,
                            p.fx, p.fy, p.cx, p.cy, img.ctypes.data_as(ip))
    return img, int(sk)


def depth(rec, pos, quat, p):
    pos, quat = np.asarray(pos, dtype=np.float64).reshape(-1, 3), np.asarray(quat, dtype=np.float64).reshape(-1, 4)
    out = np.empty((pos.shape[0], p.height, p.width), dtype=np.int32)
    for q in range(pos.shape[0]):
        _, cw = pose(pos[q], quat[q], np.array(p.cam_to_body[:]))
        out[q] = render(rec, cw, p)[0]
    return out


def backproject(img, c2w, body, p):
    out = np.empty((p.width * p.height, 3), dtype=np.float32)
    m = lib().sense_backproject(np.ascontiguousarray(img, dtype=np.int32).ctypes.data_as(ip), p.width, p.height, p.fx, p.fy, p.cx, p.cy,
                                _d(np.ascontiguousarray(c2w, dtype=np.float64)), _d(np.ascontiguousarray(body, dtype=np.float64)),
                                p.sensing_horizon, out.ctypes.data_as(fp))
    return out[:m]


def cloud(rec, pos, quat, p, images=None):
    """the sensed points of every pose; images: the poses' depth images when already computed"""
    pos, quat = np.asarray(pos, dtype=np.float64).reshape(-1, 3), np.asarray(quat, dtype=np.float64).reshape(-1, 4)
    pts, off = [], [0]
    for q in range(pos.shape[0]):
        c2w, cw = pose(pos[q], quat[q], np.array(p.cam_to_body[:]))
        img = render(rec, cw, p)[0] if images is None else images[q]
        pts.append(backproject(img, c2w, pos[q], p))
        off.append(off[-1] + len(pts[-1]))
    return np.concatenate(pts).reshape(-1, 3), np.array(off, dtype=np.int64)


# ---- the reference-compiled renderer (oracle/_ref/libref_depth.so) ----
_ref = None
MIN_REF_DEPTH = 0.1   # the reference kernel loops over its whole (2r+1)^2 square: at z >= 0.1 m, r <= 222


def ref_available():
    return os.path.exists(REF_DEPTH)


def _reflib():
    global _ref
    if _ref is None:
        L = C.CDLL(REF_DEPTH)
        L.ref_depth_create.argtypes = [C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int, fp, C.c_int]
        L.ref_depth_create.restype = C.c_void_p
        L.ref_depth_render.argtypes = [C.c_void_p, dp, ip]
        L.ref_depth_destroy.argtypes = [C.c_void_p]
        _ref = L
    return _ref


def min_positive_depth(xyz, T):
    """the smallest camera-frame z > 0 of the points under T (FP64), +inf if none"""
    T = np.asarray(T, dtype=np.float64).reshape(4, 4)
    z = np.asarray(xyz, dtype=np.float64).reshape(-1, 3) @ T[2, :3] + T[2, 3]
    z = z[z > 0]
    return float(z.min()) if z.size else np.inf


def check_ref_safe(xyz, transforms):
    """every scene handed to the reference kernel keeps its points at least 0.1 m in front of the camera (finite points only)"""
    for T in transforms:
        zmin = min_positive_depth(xyz, T)
        assert zmin >= MIN_REF_DEPTH + 1e-3, f"a point lies {zmin} m in front of the camera: the reference kernel's splat would be too large"


def ref_render(xyz, transforms, p):
    """the reference kernel's images (len(transforms), H, W) of one finite scene"""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    assert np.isfinite(xyz).all()
    check_ref_safe(xyz, transforms)
    L = _reflib()
    h = L.ref_depth_create(p.fx, p.fy, p.cx, p.cy, p.width, p.height, xyz.ctypes.data_as(fp), xyz.shape[0])
    assert h
    try:
        out = np.empty((len(transforms), p.height, p.width), dtype=np.int32)
        for i, T in enumerate(transforms):
            img = np.empty((p.height, p.width), dtype=np.int32)
            assert L.ref_depth_render(h, _d(np.ascontiguousarray(T, dtype=np.float64).reshape(16)), img.ctypes.data_as(ip)) == 0
            out[i] = img
        return out
    finally:
        L.ref_depth_destroy(h)


def load_golden():
    """{scene name: dict(xyz (n, 3) float32, T (k, 16), depth (k, H, W) int32)}; the default camera"""
    z = np.load(GOLDEN)
    names = [str(s) for s in z["names"]]
    return {nm: {k[len(nm) + 1:]: z[k] for k in z.files if k.startswith(nm + "/")} for nm in names}


# ---- scenes and poses shared by the golden file and the tests ----
def yaw_pitch_quat(yaw, pitch=0.0):
    """(w, x, y, z) of R = Rz(yaw) Ry(pitch)"""
    cy, sy, cp, sp = np.cos(yaw / 2), np.sin(yaw / 2), np.cos(pitch / 2), np.sin(pitch / 2)
    return np.array([cy * cp, -sy * sp, cy * sp, sy * cp])


def room_scene(n, seed, half=5.0, height=3.0):
    """float32 (n, 3): the walls, floor and ceiling of a [-half, half]^2 x [0, height] room sampled at random, and two boxes inside"""
    rng = np.random.default_rng(seed)
    k = n // 8
    out = []
    for a in range(2):
        for s in (-half, half):
            p = np.column_stack([rng.uniform(-half, half, k), rng.uniform(-half, half, k), rng.uniform(0, height, k)])
            p[:, a] = s
            out.append(p)
    for z in (0.0, height):
        out.append(np.column_stack([rng.uniform(-half, half, k), rng.uniform(-half, half, k), np.full(k, z)]))
    m = n - 6 * k
    for c, e in (((2.0, 1.0, 1.0), (0.5, 0.8, 1.0)), ((-1.5, -2.0, 0.6), (0.7, 0.4, 0.6))):
        f = rng.uniform(-1, 1, (m // 2, 3))
        ax = rng.integers(0, 3, m // 2)
        f[np.arange(m // 2), ax] = np.sign(f[np.arange(m // 2), ax])
        out.append(np.array(c) + f * np.array(e))
    return np.concatenate(out).astype(np.float32)[:n]


def room_poses(Q, seed, half=5.0):
    """pos (Q, 3), quat (Q, 4): bodies inside the room at random yaw and small pitch"""
    rng = np.random.default_rng(seed)
    pos = np.column_stack([rng.uniform(-half + 0.5, half - 0.5, Q), rng.uniform(-half + 0.5, half - 0.5, Q), rng.uniform(0.5, 2.5, Q)])
    quat = np.array([yaw_pitch_quat(y, p) for y, p in zip(rng.uniform(-np.pi, np.pi, Q), rng.uniform(-0.3, 0.3, Q))])
    return pos, quat


def golden_cases():
    """{name: (xyz, pos, quat)}: a room seen from inside, near a wall (large splats, points >= 0.15 m ahead), from outside looking away
    (an empty view), and a random cloud; the default camera"""
    room = room_scene(40000, 1)
    pos, quat = room_poses(4, 2)
    near = np.array([[4.85, 0.3, 1.2], [-4.8, -1.0, 1.5]])
    nq = np.array([yaw_pitch_quat(0.0), yaw_pitch_quat(np.pi, 0.1)])
    away = np.array([[8.0, 0.0, 1.5]])
    aq = np.array([yaw_pitch_quat(0.0)])
    rng = np.random.default_rng(3)
    blob = rng.normal(0, 2.0, (20000, 3)).astype(np.float32) + np.float32([6.0, 0, 0])
    cases = {
        "room": (room, np.concatenate([pos, near, away]), np.concatenate([quat, nq, aq])),
        "blob": (blob, np.array([[0.0, 0.0, 0.0], [0.5, 1.0, -0.5]]), np.array([yaw_pitch_quat(0.0), yaw_pitch_quat(0.4, -0.2)])),
    }
    return {k: (keep_ahead(x, ps, qs, 0.15), ps, qs) for k, (x, ps, qs) in cases.items()}


def keep_ahead(xyz, pos, quat, zmin, cam_to_body=(0, 0, 1, 0, -1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 0, 1)):
    """the points of xyz that no pose sees at a camera depth in (0, zmin): what the reference kernel may be given"""
    keep = np.ones(len(xyz), dtype=bool)
    for q in range(len(pos)):
        T = pose(pos[q], quat[q], np.array(cam_to_body, dtype=np.float64))[1].reshape(4, 4)
        z = xyz.astype(np.float64) @ T[2, :3] + T[2, 3]
        keep &= ~((z > 0) & (z < zmin))
    return xyz[keep]
