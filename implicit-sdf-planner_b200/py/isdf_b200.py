"""ctypes binding of libisdf_b200.so (include/isdf.h) used by tests/ and bench.py.

Thin by design: every method is one C-ABI call with host numpy buffers, or device pointers for the
`*_device` variants. There is NO fallback: if the shared library or a CUDA device is missing, loading /
`Evaluator()` raises.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libisdf_b200.so")

# isdf_shape_kind (include/isdf.h)
SHAPE_KINDS = dict(BALL=0, POINT=1, TORUS=2, CAPPED_TORUS=3, CAPPED_CONE=4, ROUNDED_CONE=5, WIREFRAME_BOX=6,
                   BEND_LINEAR=7, TWIST_BOX=8, BEND_BOX=9, TABLE=10, TREFOIL=11, SMOOTH_DIFFERENCE=12,
                   SMOOTH_INTERSECTION=13, CSG=14, BOX=15, MESH=16)
NAMED_SHAPES = ["Ball", "Point", "Torus", "Torus_big", "Cappedtorus", "CappedCone", "RoundedCone", "WireframeBox",
                "BendLinear", "BendLinear_big", "TwistBox", "BendBox", "Table", "Trefoil", "SmoothDifference",
                "SmoothIntersection", "SmoothIntersection_big", "CSG"]
WITH_DYNAMICS, WITH_COLLISION = 1, 2
QUERY_SDF, QUERY_GRAD, QUERY_SDF_GRAD = 0, 1, 2
MESH_SIGN_AUTO, MESH_SIGN_EXACT, MESH_SIGN_WINDING = 0, 1, 2

# every symbol include/isdf.h declares (tests assert the library exports all of them)
ABI_SYMBOLS = ["isdf_default_config", "isdf_create", "isdf_destroy", "isdf_last_error", "isdf_get_stats", "isdf_set_shard",
               "isdf_set_shape_analytic", "isdf_set_shape_named", "isdf_set_shape_mesh", "isdf_set_shape_mesh_ex", "isdf_shape_query",
               "isdf_set_map_u8", "isdf_set_map_f64", "isdf_points_in_aabb", "isdf_eval_discrete",
               "isdf_eval_discrete_device", "isdf_set_points", "isdf_eval_swept", "isdf_eval_swept_device",
               "isdf_get_swept_results", "isdf_eval_swept_given", "isdf_get_piece_costs",
               "isdf_gather_obstacle_points", "isdf_callback_batch", "isdf_callback_batch_device", "isdf_get_batch_trajectories",
               "isdf_lbfgs_default_params", "isdf_lbfgs_batch", "isdf_lbfgs_batch_device", "isdf_set_points_batch",
               "isdf_frontend_build_kernels", "isdf_frontend_get_kernels", "isdf_frontend_feasibility", "isdf_frontend_feasibility_device",
               "isdf_frontend_check_batch", "isdf_peer_export", "isdf_peer_connect", "isdf_peer_allreduce_device", "isdf_peer_status", "isdf_peer_disconnect",
               "isdf_clearance_default_params", "isdf_trajectory_clearance", "isdf_trajectory_clearance_device",
               "isdf_set_map_cloud", "isdf_set_map_cloud_device", "isdf_get_map_info", "isdf_get_map_u8", "isdf_get_map_f64",
               "isdf_frontend_path", "isdf_frontend_path_batch", "isdf_frontend_path_batch_device", "isdf_frontend_path_field_device",
               "isdf_frontend_path_info", "isdf_path_waypoints", "isdf_midend_default_params", "isdf_midend_callback_batch",
               "isdf_midend_batch", "isdf_midend_batch_device", "isdf_certify_default_params", "isdf_trajectory_certify",
               "isdf_trajectory_certify_device"]
CERTIFIED, UNDECIDED, COLLIDING = 1, 0, -1   # isdf_certify_summary.verdict


class KernelConfig(C.Structure):
    """isdf_kernel_config"""
    _fields_ = [(n, C.c_double) for n in ["kernel_max_roll", "kernel_max_pitch", "kernel_ang_res", "front_end_safeh"]]


class Config(C.Structure):
    """isdf_config — same field order as include/isdf.h."""
    _fields_ = [(n, C.c_double) for n in
                ["vehicle_mass", "grav_acc", "horiz_drag", "vert_drag", "paras_drag", "speed_eps", "vmax", "omgmax", "thetamax",
                 "weight_v", "weight_p", "weight_omg", "weight_theta", "smoothing_eps", "safety_hor", "occupancy_resolution"]] + \
               [(n, C.c_int32) for n in ["kernel_size", "integral_intervs", "threads_num", "flags"]]

    def copy(self):
        c = Config()
        C.memmove(C.byref(c), C.byref(self), C.sizeof(Config))
        return c


class LbfgsParams(C.Structure):
    """isdf_lbfgs_params"""
    _fields_ = [(n, C.c_int32) for n in ["mem_size", "past", "max_iterations", "max_linesearch", "max_rounds", "reserved_"]] + \
               [(n, C.c_double) for n in ["g_epsilon", "delta", "min_step", "max_step", "f_dec_coeff", "cautious_factor", "machine_prec"]]


class MidendParams(C.Structure):
    """isdf_midend_params"""
    _fields_ = [("weight_pr", C.c_double), ("rho", C.c_double), ("init_time", C.c_double), ("cancel_after", C.c_int32), ("reserved_", C.c_int32),
                ("lbfgs", LbfgsParams)]


class ClearanceParams(C.Structure):
    """isdf_clearance_params"""
    _fields_ = [("samples_per_piece", C.c_int32), ("pieces_per_traj", C.c_int32), ("reach", C.c_double), ("margin", C.c_double)]


class ClearanceSummary(C.Structure):
    """isdf_clearance_summary (one per trajectory)"""
    _fields_ = [("min_clearance", C.c_double), ("t_min", C.c_double), ("first_hit", C.c_double), ("voxel_min", C.c_int64),
                ("piece_min", C.c_int32), ("sample_min", C.c_int32), ("colliding_samples", C.c_int32), ("collision_free", C.c_int32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class CertifyParams(C.Structure):
    """isdf_certify_params"""
    _fields_ = [("clearance", ClearanceParams), ("max_depth", C.c_int32), ("max_samples_per_traj", C.c_int32), ("reserved_", C.c_int32 * 2)]


class CertifySummary(C.Structure):
    """isdf_certify_summary (one per trajectory)"""
    _fields_ = [("lower_bound", C.c_double), ("min_clearance", C.c_double), ("t_min", C.c_double), ("first_hit", C.c_double),
                ("voxel_min", C.c_int64), ("verdict", C.c_int32), ("samples", C.c_int32), ("undecided_intervals", C.c_int32), ("depth", C.c_int32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


# record of isdf_dbg_certify_leaves (not part of include/isdf.h)
CERT_LEAF_DTYPE = np.dtype([("ta", "<f8"), ("tb", "<f8"), ("ca", "<f8"), ("cb", "<f8"), ("Da", "<f8"), ("Db", "<f8"), ("piece", "<i4"), ("state", "<i4")])


class MapInfo(C.Structure):
    """isdf_map_info"""
    _fields_ = [("X", C.c_int32), ("Y", C.c_int32), ("Z", C.c_int32), ("reserved_", C.c_int32), ("res", C.c_double),
                ("bmin", C.c_double * 3), ("bmax", C.c_double * 3), ("occupied_voxels", C.c_int64), ("points_used", C.c_int64),
                ("points_skipped", C.c_int64)]

    def as_dict(self):
        return dict(dims=(self.X, self.Y, self.Z), res=self.res, bmin=np.array(self.bmin[:]), bmax=np.array(self.bmax[:]),
                    occupied_voxels=self.occupied_voxels, points_used=self.points_used, points_skipped=self.points_skipped)


class FrontPathParams(C.Structure):
    """isdf_frontpath_params"""
    _fields_ = [("reserved_", C.c_int32 * 4)]


class FrontPathInfo(C.Structure):
    """isdf_frontpath_info"""
    _fields_ = [("rounds", C.c_int32), ("reserved_", C.c_int32), ("field_bytes", C.c_int64), ("traversability_ms", C.c_double),
                ("field_ms", C.c_double), ("paths_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved_"}


class Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_int64), ("evals_discrete", C.c_int64), ("evals_swept", C.c_int64),
                ("last_pairs", C.c_int64), ("last_sdf_evals", C.c_int64), ("last_kernel_ms", C.c_double)]


def default_config_values():
    """plan_manager/config/config_CappedCone.yaml — pure python (no library needed)."""
    c = Config()
    c.vehicle_mass, c.grav_acc, c.horiz_drag, c.vert_drag, c.paras_drag, c.speed_eps = 0.61, 9.8, 0.10, 0.10, 0.01, 1e-4
    c.vmax, c.omgmax, c.thetamax = 10, 10, 100.0
    c.weight_v, c.weight_p, c.weight_omg, c.weight_theta = 1000.0, 4000.0, 1000.0, 1000.0
    c.smoothing_eps, c.safety_hor, c.occupancy_resolution = 1e-2, 0.866, 1.0
    c.kernel_size, c.integral_intervs, c.threads_num, c.flags = 13, 64, 30, WITH_DYNAMICS   # discrete collision term: opt-in
    return c


_lib = None


def load_library(path=None):
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise RuntimeError(f"{p} not found: build it with `python __graft_entry__.py build` (no CPU fallback exists)")
    lib = C.CDLL(p)
    dp, ip, vp = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.c_void_p
    lib.isdf_last_error.restype = C.c_char_p
    lib.isdf_default_config.argtypes = [C.POINTER(Config)]
    lib.isdf_create.argtypes = [C.POINTER(Config), C.c_int, C.POINTER(vp)]
    lib.isdf_destroy.argtypes = [vp]
    lib.isdf_get_stats.argtypes = [vp, C.POINTER(Stats)]
    lib.isdf_set_shard.argtypes = [vp, C.c_int, C.c_int]
    lib.isdf_set_shape_analytic.argtypes = [vp, C.c_int, dp, C.c_int, dp, dp]
    lib.isdf_set_shape_named.argtypes = [vp, C.c_char_p, dp, dp]
    lib.isdf_set_shape_mesh.argtypes = [vp, dp, C.c_int, ip, C.c_int, dp]
    lib.isdf_set_shape_mesh_ex.argtypes = [vp, dp, C.c_int, ip, C.c_int, dp, C.c_int]
    lib.isdf_shape_query.argtypes = [vp, dp, C.c_int, dp, dp, C.c_int]
    lib.isdf_set_map_u8.argtypes = [vp, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, dp, C.c_double]
    lib.isdf_set_map_f64.argtypes = [vp, dp, C.c_int, C.c_int, C.c_int, dp, C.c_double]
    lib.isdf_points_in_aabb.argtypes = [vp, dp, C.c_double, dp, C.c_int, C.POINTER(C.c_int)]
    lib.isdf_eval_discrete.argtypes = [vp, C.c_int, dp, dp, dp, dp, dp]
    lib.isdf_eval_discrete_device.argtypes = [vp, C.c_int, vp, vp, vp, vp]
    lib.isdf_set_points.argtypes = [vp, dp, C.c_int]
    lib.isdf_eval_swept.argtypes = [vp, C.c_int, dp, dp, dp, dp, dp]
    lib.isdf_eval_swept_device.argtypes = [vp, C.c_int, vp, vp, vp, vp]
    lib.isdf_get_swept_results.argtypes = [vp, dp, dp, dp]
    lib.isdf_get_piece_costs.argtypes = [vp, dp, C.c_int]
    lib.isdf_gather_obstacle_points.argtypes = [vp, dp, C.c_int, C.c_double, dp, dp, C.c_int, C.POINTER(C.c_int), C.c_int]
    lib.isdf_callback_batch.argtypes = [vp, C.c_int, C.c_int, dp, dp, C.c_int, C.c_double, dp, dp, dp]
    lib.isdf_callback_batch_device.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_int, C.c_double, vp, vp, vp, vp]
    lib.isdf_get_batch_trajectories.argtypes = [vp, dp, dp, dp]
    lib.isdf_set_points_batch.argtypes = [vp, C.c_int, ip, dp]
    lib.isdf_lbfgs_default_params.argtypes = [C.POINTER(LbfgsParams)]
    lib.isdf_lbfgs_batch.argtypes = [vp, C.c_int, C.c_int, dp, dp, C.c_int, C.c_double, C.POINTER(LbfgsParams), dp, dp, ip, ip, ip, ip]
    lib.isdf_lbfgs_batch_device.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_int, C.c_double, C.POINTER(LbfgsParams), vp, vp, vp, vp, vp, ip, vp]
    lib.isdf_frontend_build_kernels.argtypes = [vp, C.POINTER(KernelConfig), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.isdf_frontend_get_kernels.argtypes = [vp, C.POINTER(C.c_uint8), C.c_int]
    lib.isdf_frontend_feasibility.argtypes = [vp, C.POINTER(C.c_uint32)]
    lib.isdf_frontend_feasibility_device.argtypes = [vp, vp, vp]
    lib.isdf_frontend_check_batch.argtypes = [vp, C.c_int, ip, dp, dp, C.POINTER(C.c_uint8)]
    lib.isdf_peer_export.argtypes = [vp, C.c_int, C.c_int, C.c_char_p]
    lib.isdf_peer_connect.argtypes = [vp, C.c_int, C.c_int, C.c_char_p, C.c_int]
    lib.isdf_peer_allreduce_device.argtypes = [vp, vp, C.c_int, vp]
    lib.isdf_peer_status.argtypes = [vp]
    lib.isdf_peer_disconnect.argtypes = [vp]
    lib.isdf_eval_swept_given.argtypes = [vp, C.c_int, dp, dp, dp, dp, dp, dp, dp, dp]
    lib.isdf_clearance_default_params.argtypes = [C.POINTER(ClearanceParams)]
    lib.isdf_trajectory_clearance.argtypes = [vp, C.c_int, dp, dp, C.POINTER(ClearanceParams), dp, C.POINTER(C.c_int64), C.POINTER(ClearanceSummary)]
    lib.isdf_trajectory_clearance_device.argtypes = [vp, C.c_int, vp, vp, C.POINTER(ClearanceParams), vp, vp, vp, vp]
    lib.isdf_certify_default_params.argtypes = [C.POINTER(CertifyParams)]
    lib.isdf_trajectory_certify.argtypes = [vp, C.c_int, dp, dp, C.POINTER(CertifyParams), C.POINTER(CertifySummary)]
    lib.isdf_trajectory_certify_device.argtypes = [vp, C.c_int, vp, vp, C.POINTER(CertifyParams), vp, vp]
    lib.isdf_set_map_cloud.argtypes = [vp, vp, C.c_int64, C.c_int32, C.c_double, C.c_int32]
    lib.isdf_set_map_cloud_device.argtypes = [vp, vp, C.c_int64, C.c_int32, C.c_double, C.c_int32, vp]
    lib.isdf_get_map_info.argtypes = [vp, C.POINTER(MapInfo)]
    lib.isdf_get_map_u8.argtypes = [vp, C.POINTER(C.c_uint8), C.c_int64]
    lib.isdf_get_map_f64.argtypes = [vp, dp, C.c_int64]
    fpp, u8p = C.POINTER(FrontPathParams), C.POINTER(C.c_uint8)
    lib.isdf_frontend_path.argtypes = [vp, dp, dp, fpp, C.c_int, dp, dp, ip, dp, u8p]
    lib.isdf_frontend_path_batch.argtypes = [vp, dp, C.c_int, dp, fpp, C.c_int, dp, dp, ip, dp, u8p]
    lib.isdf_frontend_path_batch_device.argtypes = [vp, dp, C.c_int, vp, fpp, C.c_int, vp, vp, vp, vp, vp, vp]
    lib.isdf_frontend_path_field_device.argtypes = [vp, dp, fpp, vp, vp]
    lib.isdf_frontend_path_info.argtypes = [vp, C.POINTER(FrontPathInfo)]
    mpp = C.POINTER(MidendParams)
    lib.isdf_path_waypoints.argtypes = [C.c_int, ip, dp, C.c_double, C.c_double, C.c_int, dp, ip, ip]
    lib.isdf_midend_default_params.argtypes = [mpp]
    lib.isdf_midend_callback_batch.argtypes = [vp, C.c_int, C.c_int, dp, dp, C.c_int, mpp, dp, dp, dp, dp]
    lib.isdf_midend_batch.argtypes = [vp, C.c_int, C.c_int, dp, dp, C.c_int, mpp, dp, dp, dp, dp, dp, ip, ip, ip, ip]
    lib.isdf_midend_batch_device.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_int, mpp, vp, vp, vp, vp, vp, vp, vp, vp, ip, vp]
    for s in ABI_SYMBOLS:
        if s != "isdf_last_error":
            getattr(lib, s).restype = C.c_int
    if path is None:
        _lib = lib
    return lib


def _colmajor(a):
    """3x3 (or B x 3x3) row-major -> the library's column-major order"""
    return np.ascontiguousarray(np.swapaxes(np.asarray(a, dtype=np.float64), -1, -2)).reshape(-1)


def path_waypoints(paths, res, parlength=3.0):
    """isdf_path_waypoints (plan_manager.cpp:204-245): paths = list of (n_b, 3) arrays -> (list of (N_b - 1, 3) waypoints, pieces N_b).
    Host-only: needs no context or GPU."""
    lib = load_library()
    B = len(paths)
    off = np.zeros(B + 1, dtype=np.int32)
    for b, p in enumerate(paths):
        off[b + 1] = off[b] + len(p)
    xyz = _f64(np.concatenate([np.asarray(p, dtype=np.float64).reshape(-1, 3) for p in paths])) if B else np.zeros((0, 3))
    cap = max(int(off[B]), 1)
    wp, wo, pieces = np.zeros((cap, 3)), np.zeros(B + 1, dtype=np.int32), np.zeros(max(B, 1), dtype=np.int32)
    ip = C.POINTER(C.c_int32)
    r = lib.isdf_path_waypoints(B, off.ctypes.data_as(ip), _dp(xyz), float(res), float(parlength), cap, _dp(wp), wo.ctypes.data_as(ip), pieces.ctypes.data_as(ip))
    if r != 0:
        raise IsdfError(r, lib.isdf_last_error().decode())
    return [wp[wo[b]:wo[b + 1]].copy() for b in range(B)], pieces[:B].copy()


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None else None


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class IsdfError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"isdf error {code}: {msg}")
        self.code = code


class Evaluator:
    """One isdf_ctx. Mirrors the call order of the reference: setParam -> setEnvironment(shape) / setGridMap(map) ->
    cost callbacks (back_end_optimizer.hpp:667-747)."""

    def __init__(self, cfg=None, device=0):
        self.lib = load_library()
        self.cfg = cfg.copy() if cfg is not None else default_config_values()
        h = C.c_void_p()
        self._check(self.lib.isdf_create(C.byref(self.cfg), device, C.byref(h)))
        self.h = h

    def _check(self, r):
        if r != 0:
            raise IsdfError(r, self.lib.isdf_last_error().decode())

    def close(self):
        if getattr(self, "h", None):
            self.lib.isdf_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- shape ----
    def set_shape_named(self, name, rotate=None, trans=None):
        r = _f64(rotate).reshape(9) if rotate is not None else None
        t = _f64(trans).reshape(3) if trans is not None else None
        self._check(self.lib.isdf_set_shape_named(self.h, name.encode(), _dp(r), _dp(t)))

    def set_shape_analytic(self, kind, params, rotate=None, trans=None):
        p = _f64(params).reshape(-1)
        r = _f64(rotate).reshape(9) if rotate is not None else None
        t = _f64(trans).reshape(3) if trans is not None else None
        self._check(self.lib.isdf_set_shape_analytic(self.h, int(kind), _dp(p) if p.size else None, p.size, _dp(r), _dp(t)))

    def set_shape_mesh(self, V, F, poly_params=None, sign_mode=MESH_SIGN_AUTO):
        V = _f64(V).reshape(-1, 3)
        F = np.ascontiguousarray(F, dtype=np.int32).reshape(-1, 3)
        pp = _f64(poly_params).reshape(6) if poly_params is not None else None
        self._check(self.lib.isdf_set_shape_mesh_ex(self.h, _dp(V), V.shape[0], F.ctypes.data_as(C.POINTER(C.c_int32)), F.shape[0], _dp(pp), int(sign_mode)))

    def shape_query(self, p, what=QUERY_SDF_GRAD):
        p = _f64(p).reshape(-1, 3)
        n = p.shape[0]
        sdf = np.zeros(n)
        grad = np.zeros((n, 3))
        self._check(self.lib.isdf_shape_query(self.h, _dp(p), n, _dp(sdf), _dp(grad), what))
        return sdf, grad

    # ---- map ----
    def set_map_u8(self, occ, bmin, res):
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        X, Y, Z = occ.shape
        b = _f64(bmin).reshape(3)
        self._check(self.lib.isdf_set_map_u8(self.h, occ.ctypes.data_as(C.POINTER(C.c_uint8)), X, Y, Z, _dp(b), float(res)))

    def set_map_f64(self, grid, bmin, res):
        grid = _f64(grid)
        X, Y, Z = grid.shape
        b = _f64(bmin).reshape(3)
        self._check(self.lib.isdf_set_map_f64(self.h, _dp(grid), X, Y, Z, _dp(b), float(res)))

    def set_map_cloud(self, points, res, sta_threshold=1, stride_bytes=None):
        """the occupancy grid from a float32 point cloud (PCSmapManager::rcvGlobalMapHandler; see isdf_set_map_cloud in include/isdf.h).
        points: (n, 3) or (n, k >= 3) float32 with x, y, z in the first three columns, or a 1-D float32 / uint8 buffer of n records of
        stride_bytes each (a PointCloud2's data with point_step). Any other dtype raises rather than being rounded silently."""
        pts = np.asarray(points)
        if pts.dtype == np.float32 and pts.ndim == 2:
            if pts.shape[1] < 3:
                raise ValueError("points need at least 3 columns (x, y, z)")
            pts = np.ascontiguousarray(pts)
            stride = pts.shape[1] * 4 if stride_bytes is None else int(stride_bytes)
            if stride != pts.shape[1] * 4:
                raise ValueError("stride_bytes must equal the row size of a 2-D points array")
            n = pts.shape[0]
        elif pts.dtype in (np.float32, np.uint8) and pts.ndim == 1:
            if stride_bytes is None:
                raise ValueError("a flat record buffer needs stride_bytes")
            pts = np.ascontiguousarray(pts)
            stride = int(stride_bytes)
            n = pts.nbytes // stride if stride > 0 else 0
        else:
            raise TypeError(f"points must be float32 (n, k>=3) or a flat float32/uint8 record buffer, got {pts.dtype} {pts.shape}")
        self._check(self.lib.isdf_set_map_cloud(self.h, pts.ctypes.data_as(C.c_void_p) if n else None, n, stride, float(res), int(sta_threshold)))

    def set_map_cloud_device(self, points, n=None, stride_bytes=None, res=1.0, sta_threshold=1, stream=0):
        """points on the context's device: a float32 torch tensor (n, k >= 3), contiguous, or a raw device pointer with n and stride_bytes"""
        if hasattr(points, "data_ptr"):
            if str(points.dtype) != "torch.float32" or points.dim() != 2 or points.shape[1] < 3:
                raise TypeError(f"points must be a float32 (n, k>=3) tensor, got {points.dtype} {tuple(points.shape)}")
            if not points.is_contiguous():
                raise ValueError("points must be contiguous")
            ptr, n, stride = points.data_ptr(), points.shape[0], points.shape[1] * 4
            if stride_bytes is not None and int(stride_bytes) != stride:
                raise ValueError("stride_bytes must equal the row size of a points tensor")
        else:
            if n is None or stride_bytes is None:
                raise ValueError("a raw device pointer needs n and stride_bytes")
            ptr, stride = int(points), int(stride_bytes)
        self._check(self.lib.isdf_set_map_cloud_device(self.h, C.c_void_p(ptr), int(n), stride, float(res), int(sta_threshold), C.c_void_p(stream)))

    def map_info(self):
        """isdf_map_info of the current map as a dict(dims, res, bmin, bmax, occupied_voxels, points_used, points_skipped)"""
        m = MapInfo()
        self._check(self.lib.isdf_get_map_info(self.h, C.byref(m)))
        return m.as_dict()

    def get_map_u8(self):
        X, Y, Z = self.map_info()["dims"]
        out = np.empty((X, Y, Z), dtype=np.uint8)
        self._check(self.lib.isdf_get_map_u8(self.h, out.ctypes.data_as(C.POINTER(C.c_uint8)), out.size))
        return out

    def get_map_f64(self):
        X, Y, Z = self.map_info()["dims"]
        out = np.empty((X, Y, Z), dtype=np.float64)
        self._check(self.lib.isdf_get_map_f64(self.h, _dp(out), out.size))
        return out

    def points_in_aabb(self, centre, half, cap=100000):
        out = np.zeros((cap, 3))
        n = C.c_int(0)
        c = _f64(centre).reshape(3)
        self._check(self.lib.isdf_points_in_aabb(self.h, _dp(c), float(half), _dp(out), cap, C.byref(n)))
        return out[:min(n.value, cap)].copy(), n.value

    # ---- evaluation (host buffers; ACCUMULATES like the reference) ----
    def eval_discrete(self, T, coeffs, cost=0.0, gradC=None, gradT=None):
        T = _f64(T).reshape(-1)
        N = T.size
        Cc = _f64(coeffs).reshape(-1)
        assert Cc.size == 18 * N
        gC = np.zeros(18 * N) if gradC is None else _f64(gradC).reshape(-1)
        gT = np.zeros(N) if gradT is None else _f64(gradT).reshape(-1)
        c = C.c_double(cost)
        self._check(self.lib.isdf_eval_discrete(self.h, N, _dp(T), _dp(Cc), C.byref(c), _dp(gC), _dp(gT)))
        return c.value, gC, gT

    def gather_obstacle_points(self, waypoints, half, offset=(0.0, 0.0, 0.0), cap=1000000, set_as_points=False):
        wp = _f64(waypoints).reshape(-1, 3)
        off = _f64(offset).reshape(3)
        out = np.zeros((cap, 3))
        n = C.c_int(0)
        self._check(self.lib.isdf_gather_obstacle_points(self.h, _dp(wp), wp.shape[0], float(half), _dp(off), _dp(out), cap, C.byref(n), int(set_as_points)))
        if set_as_points:
            self.n_points = n.value
        return out[:min(n.value, cap)].copy(), n.value

    def callback_batch(self, head, tail, rho, X):
        """B decision vectors [tau (N0) | xi (3(N0-1))] -> (cost[B], grad[B, 4*N0-3]); head/tail 3x3 (columns p, v, a), shared (3,3)
        or per problem (B,3,3); passed to the library column-major."""
        X = _f64(X)
        B, dim = X.shape
        N0 = (dim + 3) // 4
        assert 4 * N0 - 3 == dim
        head, tail = np.asarray(head, dtype=np.float64), np.asarray(tail, dtype=np.float64)
        per = int(head.ndim == 3)
        colmajor = (lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2)).reshape(-1))
        h, t = colmajor(head), colmajor(tail)
        cost, grad = np.zeros(B), np.zeros((B, dim))
        Xf = np.ascontiguousarray(X).reshape(-1)
        self._check(self.lib.isdf_callback_batch(self.h, B, N0, _dp(h), _dp(t), per, float(rho), _dp(Xf), _dp(cost), _dp(grad.reshape(-1))))
        return cost, grad

    def callback_batch_device(self, B, N0, d_head, d_tail, per_problem_bc, rho, d_x, d_cost, d_grad, stream=None):
        self._check(self.lib.isdf_callback_batch_device(self.h, B, N0, d_head, d_tail, int(per_problem_bc), float(rho), d_x, d_cost, d_grad, stream))

    def set_points_batch(self, point_sets):
        """per-problem obstacle point sets for the batched callback (list of (P_b, 3) arrays); an empty list switches the batched swept term off"""
        B = len(point_sets)
        off = np.zeros(B + 1, dtype=np.int32)
        for b, p in enumerate(point_sets):
            off[b + 1] = off[b] + len(p)
        pts = _f64(np.concatenate([np.asarray(p, float).reshape(-1, 3) for p in point_sets])) if B and off[B] else np.zeros((0, 3))
        self._check(self.lib.isdf_set_points_batch(self.h, B, off.ctypes.data_as(C.POINTER(C.c_int32)), _dp(pts) if pts.size else None))
        if B:
            self.n_points = int(off[B])       # swept_results() then returns every problem's points, problem-major

    def dbg_batch_swept_out(self, B, N0):
        """the swept-volume term of the last batched callback (isdf_dbg_batch_swept_out, not part of include/isdf.h): (B, 19*N0+1) rows
        [cost | gradC 18*N0 | gradT N0]"""
        out = np.zeros((B, 19 * N0 + 1))
        self.lib.isdf_dbg_batch_swept_out.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_longlong]
        self._check(self.lib.isdf_dbg_batch_swept_out(self.h, _dp(out.reshape(-1)), out.size))
        return out

    def lbfgs_params(self, **kw):
        p = LbfgsParams()
        self._check(self.lib.isdf_lbfgs_default_params(C.byref(p)))
        for k, v in kw.items():
            setattr(p, k, v)
        return p

    def lbfgs_batch(self, head, tail, rho, X, params=None):
        """device-resident lock-step L-BFGS over the batched callback: X (B, 4*N0-3) starting points -> dict(x, f, ret, iterations, evaluations, rounds)"""
        X = _f64(X)
        B, dim = X.shape
        N0 = (dim + 3) // 4
        head, tail = np.asarray(head, dtype=np.float64), np.asarray(tail, dtype=np.float64)
        per = int(head.ndim == 3)
        colmajor = (lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2)).reshape(-1))
        h, t = colmajor(head), colmajor(tail)
        x = np.ascontiguousarray(X).copy().reshape(-1)
        f = np.zeros(B)
        ret, it, evs = (np.zeros(B, dtype=np.int32) for _ in range(3))
        rounds = C.c_int32(0)
        ip = C.POINTER(C.c_int32)
        p = params if params is not None else self.lbfgs_params()
        self._check(self.lib.isdf_lbfgs_batch(self.h, B, N0, _dp(h), _dp(t), per, float(rho), C.byref(p), _dp(x), _dp(f), ret.ctypes.data_as(ip), it.ctypes.data_as(ip),
                                              evs.ctypes.data_as(ip), C.byref(rounds)))
        return dict(x=x.reshape(B, dim), f=f, ret=ret, iterations=it, evaluations=evs, rounds=rounds.value)

    def lbfgs_batch_device(self, B, N0, d_head, d_tail, per_problem_bc, rho, d_x, d_f, d_ret=None, d_iterations=None, d_evaluations=None, params=None,
                           stream=None):
        """isdf_lbfgs_batch_device on raw device pointers (e.g. torch .data_ptr()); returns the rounds"""
        p = params if params is not None else self.lbfgs_params()
        rounds = C.c_int32(0)
        self._check(self.lib.isdf_lbfgs_batch_device(self.h, B, N0, d_head, d_tail, int(per_problem_bc), float(rho), C.byref(p), d_x, d_f, d_ret,
                                                     d_iterations, d_evaluations, C.byref(rounds), stream))
        return rounds.value

    _DBG_LBFGS_EVAL = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))

    def dbg_lbfgs_rounds(self, fun, X0, params=None, cancel_after=0):
        """the device lock-step L-BFGS rounds (lbfgs_rounds + k_lbfgs_feed) on a host objective (isdf_dbg_lbfgs_rounds, not part of
        include/isdf.h). fun(X (B, n)) -> (f (B,), G (B, n)) is called once per round with every instance's requested point, finished
        instances included. Returns dict(x, f, ret, iterations, evaluations, rounds, trace): trace[r] is round r + 1's requested points."""
        X = np.ascontiguousarray(_f64(X0)).copy()
        B, n = X.shape
        trace = []

        def cb(_user, b, nn, xp, fp, gp):
            xs = np.ctypeslib.as_array(xp, shape=(b, nn)).copy()
            trace.append(xs)
            fv, gv = fun(xs.copy())
            np.ctypeslib.as_array(fp, shape=(b,))[:] = fv
            np.ctypeslib.as_array(gp, shape=(b, nn))[:] = gv
        cfn = self._DBG_LBFGS_EVAL(cb)
        ip = C.POINTER(C.c_int32)
        self.lib.isdf_dbg_lbfgs_rounds.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(LbfgsParams), C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_double),
                                                   C.POINTER(C.c_double), ip, ip, ip, ip]
        p = params if params is not None else self.lbfgs_params()
        f = np.zeros(B)
        ret, it, evs = (np.zeros(B, dtype=np.int32) for _ in range(3))
        rounds = C.c_int32(0)
        self._check(self.lib.isdf_dbg_lbfgs_rounds(self.h, B, n, C.byref(p), int(cancel_after), C.cast(cfn, C.c_void_p), None, _dp(X.reshape(-1)), _dp(f),
                                                   ret.ctypes.data_as(ip), it.ctypes.data_as(ip), evs.ctypes.data_as(ip), C.byref(rounds)))
        return dict(x=X, f=f, ret=ret, iterations=it, evaluations=evs, rounds=rounds.value, trace=np.array(trace).reshape(len(trace), B, n))

    # ---- mid-end: warm start of the back end (see include/isdf.h) ----
    def midend_params(self, **kw):
        """isdf_midend_default_params with overrides; keys of isdf_lbfgs_params (mem_size, delta, ...) go to the nested lbfgs block,
        reserved_ to the mid-end's own"""
        p = MidendParams()
        self._check(self.lib.isdf_midend_default_params(C.byref(p)))
        lb = {n for n, _ in LbfgsParams._fields_} - {"reserved_"}
        for k, v in kw.items():
            setattr(p.lbfgs if k in lb else p, k, v)
        return p

    @staticmethod
    def path_waypoints(paths, res, parlength=3.0):
        return path_waypoints(paths, res, parlength)

    @staticmethod
    def _midend_args(head, tail, waypoints, B, N0):
        head, tail = np.asarray(head, dtype=np.float64), np.asarray(tail, dtype=np.float64)
        wp = _f64(waypoints).reshape(-1)
        assert wp.size == 3 * B * (N0 - 1)
        return int(head.ndim == 3), _colmajor(head), _colmajor(tail), (wp if wp.size else np.zeros(1))

    def midend_callback_batch(self, head, tail, waypoints, X, params=None):
        """OriTraj::costFunction for B problems: X (B, 4*N0-3), waypoints (B, N0-1, 3), head / tail (3,3) or (B,3,3) -> (cost[B], grad[B, 4*N0-3])"""
        X = _f64(X)
        B, dim = X.shape
        N0 = (dim + 3) // 4
        assert 4 * N0 - 3 == dim
        per, h, t, wp = self._midend_args(head, tail, waypoints, B, N0)
        p = params if params is not None else self.midend_params()
        cost, grad = np.zeros(B), np.zeros((B, dim))
        self._check(self.lib.isdf_midend_callback_batch(self.h, B, N0, _dp(h), _dp(t), per, C.byref(p), _dp(wp), _dp(X.reshape(-1)), _dp(cost),
                                                        _dp(grad.reshape(-1))))
        return cost, grad

    def midend_batch(self, head, tail, waypoints, params=None):
        """getOriTraj for B problems of N0 pieces: waypoints (B, N0-1, 3) -> dict(x (B, 4*N0-3), T (B, N0), coeffs (18*B*N0, the layout of
        batch_trajectories), f, ret, iterations, evaluations, rounds)"""
        wp3 = _f64(waypoints)
        B, N0 = wp3.shape[0], wp3.shape[1] + 1
        per, h, t, wp = self._midend_args(head, tail, wp3, B, N0)
        p = params if params is not None else self.midend_params()
        x, T, Cc, f = np.zeros((B, 4 * N0 - 3)), np.zeros((B, N0)), np.zeros(18 * B * N0), np.zeros(B)
        ret, it, evs = (np.zeros(B, dtype=np.int32) for _ in range(3))
        rounds = C.c_int32(0)
        ip = C.POINTER(C.c_int32)
        self._check(self.lib.isdf_midend_batch(self.h, B, N0, _dp(h), _dp(t), per, C.byref(p), _dp(wp), _dp(x.reshape(-1)), _dp(T.reshape(-1)), _dp(Cc), _dp(f),
                                               ret.ctypes.data_as(ip), it.ctypes.data_as(ip), evs.ctypes.data_as(ip), C.byref(rounds)))
        return dict(x=x, T=T, coeffs=Cc, f=f, ret=ret, iterations=it, evaluations=evs, rounds=rounds.value)

    def midend_batch_device(self, B, N0, d_head, d_tail, per_problem_bc, d_waypoints, d_x, d_T, d_coeffs, d_f, d_ret, d_iterations, d_evaluations,
                            params=None, stream=None):
        """raw device pointers (e.g. torch .data_ptr()); returns the rounds"""
        p = params if params is not None else self.midend_params()
        rounds = C.c_int32(0)
        self._check(self.lib.isdf_midend_batch_device(self.h, B, N0, d_head, d_tail, int(per_problem_bc), C.byref(p), d_waypoints, d_x, d_T, d_coeffs, d_f,
                                                      d_ret, d_iterations, d_evaluations, C.byref(rounds), stream))
        return rounds.value

    def midend_from_paths(self, fp, res=None, parlength=3.0, params=None):
        """generateTraj's mid-end for the result of frontend_path_batch: waypoints per plan, head = [front, 0, 0], tail = [back, 0, 0], the plans
        grouped by N (one isdf_midend_batch per N). Returns one dict per N: N, idx (problem indices), waypoints (B_g, N-1, 3), head / tail
        (B_g, 3, 3), x (the starting point for lbfgs_batch), T, coeffs, f, ret, iterations, evaluations, rounds. res = None: the map's resolution."""
        if res is None:
            res = self.map_info()["res"]
        paths = fp["paths"]
        wps, pieces = path_waypoints(paths, res, parlength)
        groups = []
        for N in sorted(set(int(n) for n in pieces)):
            idx = np.flatnonzero(pieces == N)
            head, tail = np.zeros((idx.size, 3, 3)), np.zeros((idx.size, 3, 3))
            for q, b in enumerate(idx):
                head[q, :, 0], tail[q, :, 0] = paths[b][0], paths[b][-1]
            wp = np.array([wps[b] for b in idx]).reshape(idx.size, N - 1, 3)
            r = self.midend_batch(head, tail, wp, params)
            groups.append(dict(N=N, idx=idx, waypoints=wp, head=head, tail=tail, **r))
        return groups

    def batch_trajectories(self, B, N0):
        T, Cc, en = np.zeros(B * N0), np.zeros(18 * B * N0), np.zeros(B)
        self._check(self.lib.isdf_get_batch_trajectories(self.h, _dp(T), _dp(Cc), _dp(en)))
        return T, Cc, en

    # ---- trajectory clearance check (see include/isdf.h) ----
    def clearance_params(self, K_c=None, reach=None, margin=None, N0=0):
        p = ClearanceParams()
        self._check(self.lib.isdf_clearance_default_params(C.byref(p)))
        if K_c is not None:
            p.samples_per_piece = int(K_c)
        if reach is not None:
            p.reach = float(reach)
            p.margin = float(reach) if margin is None else p.margin
        if margin is not None:
            p.margin = float(margin)
        p.pieces_per_traj = int(N0)
        return p

    def trajectory_clearance(self, T, coeffs, K_c, reach, margin, N0=0):
        """per-sample clearance (N*(K_c+1)), witness voxel addresses (int64, -1 = nothing within reach) and one summary dict per
        trajectory (pieces b*N0 .. b*N0+N0-1; N0 = 0: a single trajectory)"""
        T = _f64(T).reshape(-1)
        N = T.size
        Cc = _f64(coeffs).reshape(-1)
        assert Cc.size == 18 * N
        p = self.clearance_params(K_c, reach, margin, N0)
        B = 1 if N0 == 0 else max(N // N0, 1)
        clear, vox = np.zeros(N * (int(K_c) + 1)), np.zeros(N * (int(K_c) + 1), dtype=np.int64)
        summ = (ClearanceSummary * B)()
        self._check(self.lib.isdf_trajectory_clearance(self.h, N, _dp(T), _dp(Cc), C.byref(p), _dp(clear), vox.ctypes.data_as(C.POINTER(C.c_int64)), summ))
        return clear, vox, [s.as_dict() for s in summ]

    def trajectory_clearance_device(self, N, d_T, d_coeffs, params, d_clear, d_voxel, d_summary, stream=0):
        """raw device pointers (e.g. torch .data_ptr()); d_summary holds N/N0 isdf_clearance_summary records (48 bytes each)"""
        self._check(self.lib.isdf_trajectory_clearance_device(self.h, N, C.c_void_p(d_T), C.c_void_p(d_coeffs), C.byref(params), C.c_void_p(d_clear),
                                                              C.c_void_p(d_voxel), C.c_void_p(d_summary), C.c_void_p(stream)))

    def dbg_clearance_counts(self):
        """{candidate pairs, exact mesh searches} of the last clearance check (isdf_dbg_clearance_counts, not part of include/isdf.h)"""
        out = (C.c_ulonglong * 2)()
        self.lib.isdf_dbg_clearance_counts.argtypes = [C.c_void_p, C.POINTER(C.c_ulonglong)]
        self._check(self.lib.isdf_dbg_clearance_counts(self.h, out))
        return int(out[0]), int(out[1])

    # ---- continuous clearance certificate (see include/isdf.h) ----
    def certify_params(self, K_c=None, reach=None, margin=None, N0=0, max_depth=None, max_samples=None):
        p = CertifyParams()
        self._check(self.lib.isdf_certify_default_params(C.byref(p)))
        if K_c is not None:
            p.clearance.samples_per_piece = int(K_c)
        if reach is not None:
            p.clearance.reach = float(reach)
        if margin is not None:
            p.clearance.margin = float(margin)
        p.clearance.pieces_per_traj = int(N0)
        if max_depth is not None:
            p.max_depth = int(max_depth)
        if max_samples is not None:
            p.max_samples_per_traj = int(max_samples)
        return p

    def trajectory_certify(self, T, coeffs, K_c, reach, margin, N0=0, max_depth=None, max_samples=None):
        """one summary dict per trajectory (pieces b*N0 .. b*N0+N0-1; N0 = 0: a single trajectory): verdict (CERTIFIED 1, COLLIDING -1,
        UNDECIDED 0), lower_bound, min_clearance, t_min, first_hit, voxel_min, samples, undecided_intervals, depth"""
        T = _f64(T).reshape(-1)
        N = T.size
        Cc = _f64(coeffs).reshape(-1)
        assert Cc.size == 18 * N
        p = self.certify_params(K_c, reach, margin, N0, max_depth, max_samples)
        B = 1 if N0 == 0 else max(N // N0, 1)
        summ = (CertifySummary * B)()
        self._check(self.lib.isdf_trajectory_certify(self.h, N, _dp(T), _dp(Cc), C.byref(p), summ))
        return [s.as_dict() for s in summ]

    def trajectory_certify_device(self, N, d_T, d_coeffs, params, d_summary, stream=0):
        """raw device pointers (e.g. torch .data_ptr()); d_summary holds N/N0 isdf_certify_summary records (56 bytes each)"""
        self._check(self.lib.isdf_trajectory_certify_device(self.h, N, C.c_void_p(d_T), C.c_void_p(d_coeffs), C.byref(params),
                                                            C.c_void_p(d_summary), C.c_void_p(stream)))

    def dbg_certify_bound(self, T, coeffs, reach, piece, ta, tb):
        """(D_a, D_b) of the certificate's motion bound for intervals (piece, ta, tb) of the block (T, coeffs) as an (n, 2) array, and the
        body radius r it used (isdf_dbg_certify_bound, not part of include/isdf.h)"""
        T, Cc = _f64(T).reshape(-1), _f64(coeffs).reshape(-1)
        piece = np.ascontiguousarray(piece, dtype=np.int32).reshape(-1)
        ta, tb = _f64(ta).reshape(-1), _f64(tb).reshape(-1)
        n = piece.size
        out = np.zeros((n, 2))
        f = self.lib.isdf_dbg_certify_bound
        f.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                      C.POINTER(C.c_double)]
        f.restype = C.c_int
        r = C.c_double(0.0)
        self._check(f(self.h, T.size, T.ctypes.data, Cc.ctypes.data, float(reach), n, piece.ctypes.data, ta.ctypes.data, tb.ctypes.data,
                      out.ctypes.data, C.byref(r)))
        return out, r.value

    def dbg_certify_leaves(self):
        """the final leaf intervals of the last certificate call as a structured array (CERT_LEAF_DTYPE; piece = index in the call's
        block), in the order they were finished (isdf_dbg_certify_leaves, not part of include/isdf.h)"""
        f = self.lib.isdf_dbg_certify_leaves
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong)]
        f.restype = C.c_int
        n = C.c_longlong(0)
        self._check(f(self.h, None, 0, C.byref(n)))
        out = np.zeros(n.value, dtype=CERT_LEAF_DTYPE)
        if n.value:
            self._check(f(self.h, out.ctypes.data, n.value, C.byref(n)))
        return out

    # ---- front end: attitude kernels (see include/isdf.h) ----
    def frontend_build_kernels(self, max_roll=45.0, max_pitch=45.0, ang_res=9.0, front_end_safeh=0.0):
        kc = KernelConfig(max_roll, max_pitch, ang_res, front_end_safeh)
        xk, yk = C.c_int(0), C.c_int(0)
        self._check(self.lib.isdf_frontend_build_kernels(self.h, C.byref(kc), C.byref(xk), C.byref(yk)))
        self.fe_dims = (xk.value, yk.value)
        return self.fe_dims

    def frontend_kernels(self, ks):
        xk, yk = self.fe_dims
        out = np.zeros(xk * yk * ks ** 3, dtype=np.uint8)
        self._check(self.lib.isdf_frontend_get_kernels(self.h, out.ctypes.data_as(C.POINTER(C.c_uint8)), out.size))
        return out.reshape(xk * yk, ks, ks, ks)

    def frontend_feasibility(self, X, Y, Z):
        out = np.zeros((X * Y * Z, 4), dtype=np.uint32)
        self._check(self.lib.isdf_frontend_feasibility(self.h, out.ctypes.data_as(C.POINTER(C.c_uint32))))
        return out

    def frontend_feasibility_device(self, d_masks, stream=None):
        self._check(self.lib.isdf_frontend_feasibility_device(self.h, d_masks, stream))

    def frontend_check_batch(self, ind, father):
        ind = np.ascontiguousarray(ind, dtype=np.int32).reshape(-1, 3)
        father = _f64(father).reshape(-1, 2)
        n = ind.shape[0]
        child, ok = np.zeros((n, 2)), np.zeros(n, dtype=np.uint8)
        self._check(self.lib.isdf_frontend_check_batch(self.h, n, ind.ctypes.data_as(C.POINTER(C.c_int32)), _dp(father.reshape(-1)), _dp(child.reshape(-1)),
                                                       ok.ctypes.data_as(C.POINTER(C.c_uint8))))
        return child, ok.astype(bool)

    # ---- front-end path search (see include/isdf.h) ----
    def _path_cap(self, cap):
        if cap is not None:
            return int(cap)
        info = self.map_info()
        return 4 * sum(info["dims"])

    def frontend_path_batch(self, start, goals, cap=None):
        """one start, B goals -> dict(paths: list of (n_b, 3) cube centres, roll_pitch: list of (n_b, 2) degrees, offsets (B + 1),
        costs (B), found (B) bool). cap = None: a first guess, repeated once with the exact total when the paths are longer."""
        st = _f64(start).reshape(3)
        goals = _f64(goals).reshape(-1, 3)
        B = goals.shape[0]
        cap = self._path_cap(cap)
        for attempt in range(2):
            xyz, rp = np.zeros((max(cap, 1), 3)), np.zeros((max(cap, 1), 2))
            off, cost, found = np.zeros(B + 1, dtype=np.int32), np.zeros(B), np.zeros(B, dtype=np.uint8)
            r = self.lib.isdf_frontend_path_batch(self.h, _dp(st), B, _dp(goals), None, cap, _dp(xyz), _dp(rp),
                                                  off.ctypes.data_as(C.POINTER(C.c_int32)), _dp(cost), found.ctypes.data_as(C.POINTER(C.c_uint8)))
            if r == -1 and attempt == 0 and off[B] > cap:
                cap = int(off[B])
                continue
            self._check(r)
            break
        n = int(off[B])
        return dict(paths=[xyz[off[b]:off[b + 1]] for b in range(B)], roll_pitch=[rp[off[b]:off[b + 1]] for b in range(B)],
                    xyz=xyz[:n], rp=rp[:n], offsets=off, costs=cost, found=found.astype(bool))

    def frontend_path(self, start, goal, cap=None):
        """-> (path (n, 3), roll_pitch (n, 2), cost, found), through isdf_frontend_path"""
        st, gl = _f64(start).reshape(3), _f64(goal).reshape(3)
        cap = self._path_cap(cap)
        for attempt in range(2):
            xyz, rp = np.zeros((max(cap, 1), 3)), np.zeros((max(cap, 1), 2))
            n, cost, found = C.c_int32(0), C.c_double(0), C.c_uint8(0)
            r = self.lib.isdf_frontend_path(self.h, _dp(st), _dp(gl), None, cap, _dp(xyz), _dp(rp), C.byref(n), C.byref(cost), C.byref(found))
            if r == -1 and attempt == 0 and n.value > cap:
                cap = n.value
                continue
            self._check(r)
            break
        return xyz[:n.value], rp[:n.value], cost.value, bool(found.value)

    def frontend_path_raw(self, start, goal, cap):
        """isdf_frontend_path with the caller's cap: (status, n)"""
        st, gl = _f64(start).reshape(3), _f64(goal).reshape(3)
        xyz, rp = np.zeros((max(cap, 1), 3)), np.zeros((max(cap, 1), 2))
        n, cost, found = C.c_int32(-7), C.c_double(0), C.c_uint8(0)
        r = self.lib.isdf_frontend_path(self.h, _dp(st), _dp(gl), None, int(cap), _dp(xyz), _dp(rp), C.byref(n), C.byref(cost), C.byref(found))
        return r, n.value

    def frontend_path_batch_device(self, start, B, d_goals, cap, d_xyz, d_rp, d_offsets, d_costs, d_found, stream=None):
        st = _f64(start).reshape(3)
        self._check(self.lib.isdf_frontend_path_batch_device(self.h, _dp(st), B, d_goals, None, cap, d_xyz, d_rp, d_offsets, d_costs, d_found, stream))

    def frontend_path_field_device(self, start, d_g, stream=None):
        st = _f64(start).reshape(3)
        self._check(self.lib.isdf_frontend_path_field_device(self.h, _dp(st), None, d_g, stream))

    def frontend_path_info(self):
        out = FrontPathInfo()
        self._check(self.lib.isdf_frontend_path_info(self.h, C.byref(out)))
        return out.as_dict()

    def dbg_frontpath_traversable(self):
        """traversability of the last path / field call as an (X, Y, Z) bool array (isdf_dbg_frontpath_traversable, not part of include/isdf.h)"""
        X, Y, Z = self.map_info()["dims"]
        Zw = (Z + 31) // 32
        words = np.zeros(X * Y * Zw, dtype=np.uint32)
        self.lib.isdf_dbg_frontpath_traversable.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_longlong]
        self._check(self.lib.isdf_dbg_frontpath_traversable(self.h, words.ctypes.data_as(C.POINTER(C.c_uint32)), words.size))
        bits = np.unpackbits(words.view(np.uint8), bitorder="little").reshape(X, Y, Zw * 32)
        return bits[:, :, :Z].astype(bool)

    # ---- multi-GPU reduction over peer memory (see include/isdf.h) ----
    def peer_export(self, world, max_doubles):
        buf = C.create_string_buffer(64)
        self._check(self.lib.isdf_peer_export(self.h, world, max_doubles, buf))
        return bytes(buf.raw)

    def peer_connect(self, world, rank, handles, fuse=True):
        blob = b"".join(handles)
        assert len(blob) == 64 * world
        self._check(self.lib.isdf_peer_connect(self.h, world, rank, blob, int(fuse)))

    def peer_allreduce_device(self, d_vec, n, stream=None):
        self._check(self.lib.isdf_peer_allreduce_device(self.h, d_vec, n, stream))

    def peer_status(self):
        self._check(self.lib.isdf_peer_status(self.h))

    def peer_disconnect(self):
        self._check(self.lib.isdf_peer_disconnect(self.h))

    def piece_costs(self, n):
        out = np.zeros(n)
        self._check(self.lib.isdf_get_piece_costs(self.h, _dp(out), n))
        return out

    def set_points(self, pts):
        pts = _f64(pts).reshape(-1, 3)
        self._check(self.lib.isdf_set_points(self.h, _dp(pts) if pts.size else None, pts.shape[0]))
        self.n_points = pts.shape[0]

    def eval_swept(self, T, coeffs, cost=0.0, gradC=None, gradT=None):
        T = _f64(T).reshape(-1)
        N = T.size
        Cc = _f64(coeffs).reshape(-1)
        gC = np.zeros(18 * N) if gradC is None else _f64(gradC).reshape(-1)
        gT = np.zeros(N) if gradT is None else _f64(gradT).reshape(-1)
        c = C.c_double(cost)
        self._check(self.lib.isdf_eval_swept(self.h, N, _dp(T), _dp(Cc), C.byref(c), _dp(gC), _dp(gT)))
        return c.value, gC, gT

    def eval_swept_given(self, T, coeffs, tstar, sdf, grel):
        T = _f64(T).reshape(-1)
        N = T.size
        Cc = _f64(coeffs).reshape(-1)
        gC, gT, c = np.zeros(18 * N), np.zeros(N), C.c_double(0.0)
        ts, sd, gr = _f64(tstar).reshape(-1), _f64(sdf).reshape(-1), _f64(grel).reshape(-1)
        self._check(self.lib.isdf_eval_swept_given(self.h, N, _dp(T), _dp(Cc), _dp(ts), _dp(sd), _dp(gr), C.byref(c), _dp(gC), _dp(gT)))
        return c.value, gC, gT

    def swept_results(self):
        P = self.n_points
        t, s, g = np.zeros(P), np.zeros(P), np.zeros((P, 3))
        self._check(self.lib.isdf_get_swept_results(self.h, _dp(t), _dp(s), _dp(g)))
        return t, s, g

    # ---- device-resident variants: raw device pointers (e.g. torch tensor .data_ptr()), asynchronous ----
    def eval_discrete_device(self, N, d_T, d_coeffs, d_out, stream=0):
        self._check(self.lib.isdf_eval_discrete_device(self.h, N, C.c_void_p(d_T), C.c_void_p(d_coeffs), C.c_void_p(d_out), C.c_void_p(stream)))

    def eval_swept_device(self, N, d_T, d_coeffs, d_out, stream=0):
        self._check(self.lib.isdf_eval_swept_device(self.h, N, C.c_void_p(d_T), C.c_void_p(d_coeffs), C.c_void_p(d_out), C.c_void_p(stream)))

    def set_shard(self, rank, world):
        self._check(self.lib.isdf_set_shard(self.h, rank, world))

    def stats(self):
        s = Stats()
        self._check(self.lib.isdf_get_stats(self.h, C.byref(s)))
        return s

    # ---- diagnostics (isdf_dbg_*: exported by the library, not part of include/isdf.h) ----
    def dbg_schedule(self, natural_order=False, warp_slots=0):
        """natural_order: every launch as a context's first one (no work items, nothing split); warp_slots > 0: build the work items as
        if the device had that many resident warps (huge values force every non-trivial sample to be split)."""
        vp = C.c_void_p
        self.lib.isdf_dbg_schedule.argtypes = [vp, C.c_int, C.c_int]
        self._check(self.lib.isdf_dbg_schedule(self.h, int(natural_order), int(warp_slots)))

    def dbg_window_lists(self, budget=-1, arrays=False):
        """window lists of the last mesh evaluation with collision (k_discrete_prologue). budget >= 0 sets the list capacity of the
        following evaluations in codes per sample of the trajectory, i.e. budget x world per local sample of a shard (0: no lists, the
        scan kernel enumerates every window itself). Returns
        dict(runs, written, overflow, samples, capacity, requested) and, with arrays, pose (M x 8: position, quaternion w x y z, unused),
        desc (M x 2: list offset or -1, voxel count) and codes (uint32: dx | dy << 10 | dz << 20). With budget >= 0 and nothing
        evaluated yet, returns None."""
        vp, lp, dp = C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_double)
        ip, up = C.POINTER(C.c_int32), C.POINTER(C.c_uint32)
        self.lib.isdf_dbg_window_lists.argtypes = [vp, C.c_int, lp, dp, ip, up]
        self._check(self.lib.isdf_dbg_window_lists(self.h, int(budget), None, None, None, None))
        st = np.zeros(6, dtype=np.int64)
        r = self.lib.isdf_dbg_window_lists(self.h, -1, st.ctypes.data_as(lp), None, None, None)
        if r == -2 and budget >= 0:     # ISDF_ERR_STATE: no mesh evaluation with collision yet
            return None
        self._check(r)
        out = dict(runs=int(st[0]), written=int(st[1]), overflow=int(st[2]), samples=int(st[3]), capacity=int(st[4]), requested=int(st[5]))
        if arrays:
            M = out["samples"]
            pose, desc = np.zeros((M, 8)), np.zeros((M, 2), dtype=np.int32)
            codes = np.zeros(max(min(out["requested"], out["capacity"]), 1), dtype=np.uint32)
            self._check(self.lib.isdf_dbg_window_lists(self.h, -1, None, _dp(pose), desc.ctypes.data_as(ip), codes.ctypes.data_as(up)))
            out.update(pose=pose, desc=desc, codes=codes[:min(out["requested"], out["capacity"])])
        return out

    def dbg_item_stats(self):
        n, parts = C.c_int(0), C.c_int(0)
        self.lib.isdf_dbg_item_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        self._check(self.lib.isdf_dbg_item_stats(self.h, C.byref(n), C.byref(parts)))
        return n.value, parts.value

    def dbg_item_table(self):
        """the work-item table k_build_items built after the last discrete evaluation (isdf_dbg_item_table). Read it before the next
        evaluation, whose scan overwrites the work values. Returns dict(M, rank, world, max_split, warp_slots, item_count,
        builder ("none", "cached" or "uncached"), have_items: whether the last scan read a table,
        items: item_count x 3 int32 {local sample m, part (-1 = every class, else c0 | c1 << 8), split slot or -1},
        work: M uint32, the work values the builder read)"""
        vp, lp, ip, up = C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_int32), C.POINTER(C.c_uint32)
        self.lib.isdf_dbg_item_table.argtypes = [vp, lp, ip, C.c_longlong, up]
        info = np.zeros(8, dtype=np.int64)
        self._check(self.lib.isdf_dbg_item_table(self.h, info.ctypes.data_as(lp), None, 0, None))
        M, n = int(info[0]), int(info[5])
        items, work = np.zeros((max(n, 1), 3), dtype=np.int32), np.zeros(M, dtype=np.uint32)
        self._check(self.lib.isdf_dbg_item_table(self.h, info.ctypes.data_as(lp), items.ctypes.data_as(ip), n, work.ctypes.data_as(up)))
        return dict(M=M, rank=int(info[1]), world=int(info[2]), max_split=int(info[3]), warp_slots=int(info[4]), item_count=n,
                    builder=("none", "cached", "uncached")[int(info[6])], have_items=bool(info[7]), items=items[:n], work=work)

    def dbg_mesh_grid(self, arrays=True):
        """the current mesh's body-frame cell grid, copied to the host: dict(glo, gcell, ghd, gpad, sign_radius, list_reach, gdim) and,
        with arrays, cell_dist (float32) and cell_cnt (uint16; 0 = no candidate list) shaped gdim (z fastest)"""
        vp, dp = C.c_void_p, C.POINTER(C.c_double)
        ip, fp, up = C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_uint16)
        self.lib.isdf_dbg_mesh_grid.argtypes = [vp, dp, ip, fp, up]
        geom, gdim = np.zeros(8), np.zeros(3, dtype=np.int32)
        self._check(self.lib.isdf_dbg_mesh_grid(self.h, _dp(geom), gdim.ctypes.data_as(ip), None, None))
        out = dict(glo=geom[0:3].copy(), gcell=geom[3], ghd=geom[4], gpad=geom[5], sign_radius=geom[6], list_reach=geom[7], gdim=tuple(int(g) for g in gdim))
        if arrays:
            dist, cnt = np.zeros(tuple(gdim), dtype=np.float32), np.zeros(tuple(gdim), dtype=np.uint16)
            self._check(self.lib.isdf_dbg_mesh_grid(self.h, _dp(geom), gdim.ctypes.data_as(ip), dist.ctypes.data_as(fp), cnt.ctypes.data_as(up)))
            out["cell_dist"], out["cell_cnt"] = dist, cnt
        return out

    def dbg_mesh_lists(self):
        """the current mesh's candidate lists, copied to the host: dict(cell_off (shaped as dbg_mesh_grid's arrays), cand (uint32),
        cand_lb (float32), tris (ntris x 3 x 3: the leaf-order triangles cand indexes, as vertices a, a + ab, a + ac))"""
        vp, llp = C.c_void_p, C.POINTER(C.c_longlong)
        u32p, fp = C.POINTER(C.c_uint32), C.POINTER(C.c_float)
        self.lib.isdf_dbg_mesh_lists.argtypes = [vp, llp, u32p, u32p, fp, C.POINTER(C.c_double)]
        sizes = np.zeros(2, dtype=np.int64)
        self._check(self.lib.isdf_dbg_mesh_lists(self.h, sizes.ctypes.data_as(llp), None, None, None, None))
        gdim = self.dbg_mesh_grid(arrays=False)["gdim"]
        off = np.zeros(gdim, dtype=np.uint32)
        cand, lb = np.zeros(int(sizes[0]), dtype=np.uint32), np.zeros(int(sizes[0]), dtype=np.float32)
        rec = np.zeros((int(sizes[1]), 16))
        self._check(self.lib.isdf_dbg_mesh_lists(self.h, sizes.ctypes.data_as(llp), off.ctypes.data_as(u32p), cand.ctypes.data_as(u32p),
                                                 lb.ctypes.data_as(fp), _dp(rec)))
        a = rec[:, 0:3]
        tris = np.stack([a, a + rec[:, 3:6], a + rec[:, 6:9]], axis=1)
        return dict(cell_off=off, cand=cand, cand_lb=lb, tris=tris)

    def dbg_flatness(self, v, a, j, quat_grad, omg_grad, vel_grad):
        """device flatness map + adjoint as compiled into the epilogue kernel -> (quat, omg, gV, gA, gJ)"""
        vaj = np.ascontiguousarray(np.concatenate([_f64(v).reshape(-1, 3), _f64(a).reshape(-1, 3), _f64(j).reshape(-1, 3)], axis=1))
        gr = np.ascontiguousarray(np.concatenate([_f64(quat_grad).reshape(-1, 4), _f64(omg_grad).reshape(-1, 3), _f64(vel_grad).reshape(-1, 3)], axis=1))
        n = vaj.shape[0]
        out = np.zeros((n, 16))
        dp = C.POINTER(C.c_double)
        self.lib.isdf_dbg_flatness.argtypes = [C.c_void_p, C.c_int, dp, dp, dp]
        self._check(self.lib.isdf_dbg_flatness(self.h, n, _dp(vaj), _dp(gr), _dp(out)))
        return out[:, 0:4], out[:, 4:7], out[:, 7:10], out[:, 10:13], out[:, 13:16]
