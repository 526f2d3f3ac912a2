"""ctypes binding of libisdf_b200.so (include/isdf.h) used by tests/ and bench.py.

Thin by design: every method is one C-ABI call with host numpy buffers, or device pointers for the
`*_device` variants. There is NO fallback: if the shared library or a CUDA device is missing, loading /
`Evaluator()` raises.
"""
import contextlib
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
               "isdf_trajectory_certify_device", "isdf_swept_default_params", "isdf_swept_volume_sdf", "isdf_swept_volume_grid",
               "isdf_swept_volume_grid_device", "isdf_swept_volume_mesh", "isdf_dynamics_default_params", "isdf_trajectory_dynamics",
               "isdf_trajectory_dynamics_device", "isdf_gather_obstacle_points_batch", "isdf_plan_default_params", "isdf_plan_batch",
               "isdf_get_plan_info", "isdf_callback_batch_ragged", "isdf_callback_batch_ragged_device", "isdf_lbfgs_batch_ragged",
               "isdf_lbfgs_batch_ragged_device", "isdf_midend_callback_batch_ragged", "isdf_midend_batch_ragged",
               "isdf_midend_batch_ragged_device", "isdf_map_esdf", "isdf_get_esdf_f64", "isdf_esdf_query", "isdf_esdf_query_device",
               "isdf_trajectory_states", "isdf_trajectory_states_device", "isdf_pose_points", "isdf_pose_points_device",
               "isdf_frontend_path_pairs", "isdf_frontend_path_pairs_device", "isdf_frontend_path_fields_device", "isdf_plan_pairs",
               "isdf_path_waypoints_device", "isdf_plan_pairs_device", "isdf_plan_batch_device",
               "isdf_sim_default_params", "isdf_simulate", "isdf_simulate_device",
               "isdf_pose_clearance_default_params", "isdf_pose_clearance", "isdf_pose_clearance_device",
               "isdf_sense_default_params", "isdf_set_sense_cloud", "isdf_set_sense_cloud_device", "isdf_get_sense_info",
               "isdf_sense_depth", "isdf_sense_depth_device", "isdf_sense_cloud", "isdf_sense_cloud_device",
               "isdf_world_default_params", "isdf_world_cloud", "isdf_world_cloud_device",
               "isdf_map_fuse_cloud", "isdf_map_fuse_cloud_device", "isdf_plan_states", "isdf_plan_states_device",
               "isdf_trajectory_shift", "isdf_trajectory_shift_device", "isdf_brake_default_params", "isdf_trajectory_brake",
               "isdf_trajectory_brake_device", "isdf_map_observe", "isdf_map_observe_device", "isdf_map_mark_known",
               "isdf_get_map_known_u8", "isdf_set_unknown_policy", "isdf_get_unknown_policy", "isdf_gather_obstacle_points_batch_known",
               "isdf_map_frontiers", "isdf_map_frontiers_device", "isdf_frontier_default_params", "isdf_frontier_goals",
               "isdf_frontier_goals_device", "isdf_view_gain", "isdf_view_gain_device", "isdf_frontier_goals_view",
               "isdf_frontier_goals_view_device"]
WORLD_KINDS = dict(globalmap=1, perlin=2, boxes=3)   # isdf_world_kind
CERTIFIED, UNDECIDED, COLLIDING = 1, 0, -1   # isdf_certify_summary.verdict
FEASIBLE, VIOLATING = 1, -1                  # isdf_dynamics_summary.verdict (0: UNDECIDED)
DYN_QUANTITIES = ["speed", "acceleration", "body_rate", "tilt", "thrust"]   # q of isdf_dynamics_summary; mask bit 5: the thrust minimum
PLAN_CERTIFY, PLAN_DYNAMICS, PLAN_KNOWN_PREFIX, PLAN_KNOWN_ONLY = 1, 2, 8, 16     # isdf_plan_params.flags
FRONTIER_NONE, FRONTIER_GOAL, FRONTIER_FRONTIER = 0, 1, 2                        # isdf_frontier_goal.kind
PLAN_FAILED, NO_PATH, TOO_LONG, MIDEND_FAILED, OPTIMISED = -1, 0, 1, 2, 3      # isdf_plan_result.stage
ESDF_FIELDS = dict(positive=0, negative=1, signed=2)                            # isdf_esdf_field
STATE_DOUBLES = 20                                                               # ISDF_STATE_DOUBLES: pos vel acc jer quat(w,x,y,z) omg thr
SIM_INIT_DOUBLES, SIM_DOUBLES = 17, 21   # ISDF_SIM_INIT_DOUBLES: pos vel quat(w,x,y,z) omega rpm; ISDF_SIM_DOUBLES: t pos vel quat omega rpm cmd_pos
NAV_ACTIVE, NAV_ARRIVED, NAV_STOPPED, NAV_DIVERGED, NAV_TIMEOUT = 0, 1, 2, 3, 4   # Evaluator.navigate: a vehicle's status
NAV_IDLE, NAV_KEPT, NAV_REPLANNED, NAV_REPLAN_FAILED = -1, 0, 1, 2               # Evaluator.navigate: a vehicle's action in a round
NAV_NO_TRAJECTORY = -2                                                            # Evaluator.navigate: verdict of a round without one
NAV_BRAKED, NAV_HELD = 3, 4                        # Evaluator.navigate(fallback="brake"): a vehicle's action in a round
NAV_COMMITTED = 5                                  # Evaluator.navigate(unknown="occupied"): a vehicle's action in a round
NAV_COMMIT_SLACK = 0.25   # m added to the certificate margin of a commit's stop: the simulator's tracking error must not put the vehicle
                          # within the margin of unseen space where it stops, or no plan from there could be committed to again
BRAKE_NO_INPUT, BRAKE_NONE, BRAKED = -1, 0, 1      # isdf_brake_summary.status
BRAKE_MAX_PIECES = 64                              # ISDF_BRAKE_MAX_PIECES
UNKNOWN_FREE, UNKNOWN_OCCUPIED = 0, 1              # isdf_unknown_policy


class SimParams(C.Structure):
    """isdf_sim_params"""
    _fields_ = [("mass", C.c_double), ("grav", C.c_double), ("J", C.c_double * 3), ("kf", C.c_double), ("km", C.c_double),
                ("arm", C.c_double), ("motor_tau", C.c_double), ("min_rpm", C.c_double), ("max_rpm", C.c_double),
                ("ctrl_mass", C.c_double), ("ctrl_grav", C.c_double)] + \
               [(n, C.c_double * 3) for n in ["kx", "kv", "kR", "kOm", "corrections"]] + \
               [(n, C.c_double) for n in ["sim_rate", "cmd_rate", "t_end", "diverge_dist"]] + \
               [(n, C.c_int32) for n in ["log_every", "use_external_yaw", "floor", "reserved_"]]


class SimSummary(C.Structure):
    """isdf_sim_summary"""
    _fields_ = [(n, C.c_double) for n in ["max_err", "t_max_err", "rms_err", "final_err", "max_tilt", "max_omega", "t_diverged"]] + \
               [(n, C.c_int64) for n in ["accepted", "rejected"]] + \
               [(n, C.c_int32) for n in ["clamped_steps", "floor_contacts", "nan_rollbacks", "diverged"]]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


def decode_sim_summaries(raw):
    """(R, 88) uint8 rows (a numpy array or a tensor) of isdf_sim_summary records -> list of dicts"""
    b = np.ascontiguousarray(raw.cpu().numpy() if hasattr(raw, "cpu") else raw, dtype=np.uint8).reshape(-1, C.sizeof(SimSummary))
    return [SimSummary.from_buffer_copy(row.tobytes()).as_dict() for row in b]


def _cloud_records(points, stride_bytes):
    """(contiguous array, n, stride) of a host cloud: (n, k >= 3) float32, or a flat float32 / uint8 buffer of stride_bytes records"""
    pts = np.asarray(points)
    if pts.dtype == np.float32 and pts.ndim == 2:
        if pts.shape[1] < 3:
            raise ValueError("points need at least 3 columns (x, y, z)")
        pts = np.ascontiguousarray(pts)
        stride = pts.shape[1] * 4 if stride_bytes is None else int(stride_bytes)
        if stride != pts.shape[1] * 4:
            raise ValueError("stride_bytes must equal the row size of a 2-D points array")
        return pts, pts.shape[0], stride
    if pts.dtype in (np.float32, np.uint8) and pts.ndim == 1:
        if stride_bytes is None:
            raise ValueError("a flat record buffer needs stride_bytes")
        pts = np.ascontiguousarray(pts)
        stride = int(stride_bytes)
        return pts, (pts.nbytes // stride if stride > 0 else 0), stride
    raise TypeError(f"points must be float32 (n, k>=3) or a flat float32/uint8 record buffer, got {pts.dtype} {pts.shape}")


def _cloud_records_device(points, n, stride_bytes):
    """(device pointer, n, stride) of a device cloud: a contiguous float32 tensor (n, k >= 3), or a raw pointer with n and stride_bytes"""
    if hasattr(points, "data_ptr"):
        if str(points.dtype) != "torch.float32" or points.dim() != 2 or points.shape[1] < 3:
            raise TypeError(f"points must be a float32 (n, k>=3) tensor, got {points.dtype} {tuple(points.shape)}")
        if not points.is_contiguous():
            raise ValueError("points must be contiguous")
        stride = points.shape[1] * 4
        if stride_bytes is not None and int(stride_bytes) != stride:
            raise ValueError("stride_bytes must equal the row size of a points tensor")
        return points.data_ptr(), points.shape[0], stride
    if n is None or stride_bytes is None:
        raise ValueError("a raw device pointer needs n and stride_bytes")
    return int(points), n, int(stride_bytes)


def _cuda_records(records):
    """a float64 CUDA tensor of pose records as (Q, stride) with unit stride along a record"""
    if not (hasattr(records, "is_cuda") and records.is_cuda and str(records.dtype) == "torch.float64"):
        raise TypeError("records must be a float64 CUDA tensor")
    r = records.reshape(-1, records.shape[-1])
    if r.stride(1) != 1:
        r = r.contiguous()
    if r.shape[0] > 1 and r.stride(0) != r.shape[1]:
        r = r.contiguous()
    return r


def sense_params(**kw):
    """isdf_sense_params: the reference's camera (isdf_sense_default_params) with the given fields replaced; cam_to_body takes 16
    row-major values or a 4 x 4 array"""
    p = SenseParams()
    r = load_library().isdf_sense_default_params(C.byref(p))
    if r != 0:
        raise IsdfError(r, "isdf_sense_default_params")
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        if k == "cam_to_body":
            v = np.asarray(v, dtype=np.float64).reshape(16)
            for i in range(16):
                p.cam_to_body[i] = float(v[i])
        else:
            setattr(p, k, type(getattr(p, k))(v))
    return p


def sim_default_params(**kw):
    p = SimParams()
    r = load_library().isdf_sim_default_params(C.byref(p))
    if r != 0:
        raise IsdfError(r, "isdf_sim_default_params")
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        if isinstance(v, (list, tuple, np.ndarray)):
            arr = getattr(p, k)
            for i, e in enumerate(v):
                arr[i] = float(e)
        else:
            setattr(p, k, type(getattr(p, k))(v))
    return p


def sim_log_records(p):
    """n_log: the log records per rollout under params p (isdf.h: (n_ticks - 1) / log_every + 1)"""
    n_ticks = int(np.floor(p.t_end * p.cmd_rate)) + 1
    return (n_ticks - 1) // max(p.log_every, 1) + 1


def sim_init_from_log(records):
    """the simulator states (..., 17) a rollout continues from: log records (..., 21) without t and the commanded position (pos, vel, quat,
    omega, rpm are records[..., 1:18]); numpy arrays or tensors"""
    return records[..., 1:1 + SIM_INIT_DOUBLES]


def sim_init_from_trajectories(piece_off, coeffs, traj, params=None, rpm=None):
    """the initial states (R, 17) of rollouts that fly trajectories traj: each trajectory's start position, zero velocity, level attitude
    and, by default, the hover rpm sqrt(m g / (4 kf)) of params' vehicle. This departs from the reference simulator, which starts its
    motors at 0 rpm (and at the launch file's init_state); pass rpm=0 for that start."""
    p = params if params is not None else sim_default_params()
    off = np.asarray(piece_off.cpu() if hasattr(piece_off, "cpu") else piece_off).astype(np.int64)
    Cc = np.asarray(coeffs.cpu() if hasattr(coeffs, "cpu") else coeffs, dtype=np.float64).reshape(-1)
    tr = np.asarray(traj.cpu() if hasattr(traj, "cpu") else traj).astype(np.int64).reshape(-1)
    hover = np.sqrt(p.mass * p.grav / (4 * p.kf)) if rpm is None else float(rpm)
    out = np.zeros((tr.size, SIM_INIT_DOUBLES))
    for r, b in enumerate(tr):
        p0, n = off[b], off[b + 1] - off[b]
        blk = Cc[18 * p0:18 * (p0 + n)]
        out[r, 0:3] = [blk[0], blk[6 * n], blk[12 * n]]   # the constant coefficient of piece 0 per axis (6N x 3 column-major)
        out[r, 6] = 1.0
        out[r, 13:17] = hover
    return out


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


class PoseClearanceParams(C.Structure):
    """isdf_pose_clearance_params"""
    _fields_ = [("reach", C.c_double), ("margin", C.c_double), ("poses_per_group", C.c_int32), ("reserved_", C.c_int32)]


class SenseParams(C.Structure):
    """isdf_sense_params"""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("cam_to_body", C.c_double * 16), ("sensing_horizon", C.c_double)]


class WorldParams(C.Structure):
    """isdf_world_params"""
    _fields_ = [("kind", C.c_int32), ("map_id", C.c_int32), ("rand_seed", C.c_uint32), ("srand_seed", C.c_uint32),
                ("cloud_resolution", C.c_double), ("init", C.c_double * 3), ("seed", C.c_uint32), ("size", C.c_int32 * 3), ("scale", C.c_double),
                ("complexity", C.c_double), ("fill", C.c_double), ("attenuation", C.c_double), ("fractal", C.c_int32),
                ("obstacle_number", C.c_int32), ("width_min", C.c_double), ("width_max", C.c_double), ("reserved_", C.c_int32 * 2)]


def world_params(kind, **kw):
    """isdf_world_params: the reference's launch-file defaults for kind ("globalmap", "perlin", "boxes" or its isdf_world_kind value),
    with the given fields replaced (init and size take 3 values, reserved_ 2)"""
    p = WorldParams()
    k = WORLD_KINDS.get(kind, kind)
    r = load_library().isdf_world_default_params(int(k), C.byref(p))
    if r != 0:
        raise IsdfError(r, "isdf_world_default_params")
    for f, v in kw.items():
        if not hasattr(p, f):
            raise AttributeError(f)
        if f in ("init", "size", "reserved_"):
            arr = getattr(p, f)
            for i, x in enumerate(v):
                arr[i] = x
        else:
            setattr(p, f, v)
    return p


class SenseInfo(C.Structure):
    """isdf_sense_info"""
    _fields_ = [("points_used", C.c_int64), ("points_skipped", C.c_int64), ("bricks", C.c_int64)]


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


class DynamicsParams(C.Structure):
    """isdf_dynamics_params"""
    _fields_ = [(n, C.c_int32) for n in ["samples_per_piece", "pieces_per_traj", "max_depth", "max_samples_per_traj"]] + \
               [(n, C.c_double) for n in ["vmax", "amax", "omgmax", "thetamax", "thrust_min", "thrust_max",
                                          "tol_v", "tol_a", "tol_omg", "tol_theta", "tol_thrust"]] + [("reserved_", C.c_int32 * 2)]


class DynamicsSummary(C.Structure):
    """isdf_dynamics_summary (one per trajectory)"""
    _fields_ = [("upper", C.c_double * 5), ("attained", C.c_double * 5), ("t_attained", C.c_double * 5), ("thrust_lower", C.c_double),
                ("thrust_attained_min", C.c_double), ("t_thrust_attained_min", C.c_double)] + \
               [(n, C.c_int32) for n in ["verdict", "violated", "undecided", "samples", "undecided_intervals", "depth"]]

    def as_dict(self):
        return {n: (np.array(getattr(self, n)[:]) if n in ("upper", "attained", "t_attained") else getattr(self, n)) for n, _ in self._fields_}


class BrakeParams(C.Structure):
    """isdf_brake_params"""
    _fields_ = [("candidates", C.c_int32), ("pieces", C.c_int32), ("certify", CertifyParams), ("dynamics", DynamicsParams),
                ("reserved_", C.c_int32 * 2)]


class BrakeSummary(C.Structure):
    """isdf_brake_summary"""
    _fields_ = [("status", C.c_int32), ("candidate", C.c_int32), ("tau_stop", C.c_double), ("duration", C.c_double),
                ("certified", C.c_int32), ("feasible", C.c_int32), ("certify", CertifySummary), ("dynamics", DynamicsSummary)]

    def as_dict(self):
        d = {n: getattr(self, n) for n, _ in self._fields_[:6]}
        d.update(certify=self.certify.as_dict(), dynamics=self.dynamics.as_dict())
        return d


def decode_brake_summaries(raw):
    """isdf_trajectory_brake_device's raw summaries ((B, 256) uint8, on any device) -> list of B dicts (BrakeSummary.as_dict)"""
    b = np.ascontiguousarray(raw.cpu().numpy() if hasattr(raw, "cpu") else raw, dtype=np.uint8).reshape(-1, C.sizeof(BrakeSummary))
    return [BrakeSummary.from_buffer_copy(r.tobytes()).as_dict() for r in b]


class FrontPathParams(C.Structure):
    """isdf_frontpath_params"""
    _fields_ = [("unknown_weight", C.c_double), ("reserved_", C.c_int32 * 2)]


def _fpp(unknown_weight):
    """the front-end parameters of a binding: NULL (the defaults) for None, else an isdf_frontpath_params with that unknown_weight"""
    return None if unknown_weight is None else C.byref(FrontPathParams(unknown_weight=float(unknown_weight)))


class PlanParams(C.Structure):
    """isdf_plan_params"""
    _fields_ = [("parlength", C.c_double), ("half_extent", C.c_double), ("offset", C.c_double * 3), ("rho", C.c_double), ("midend", MidendParams),
                ("backend", LbfgsParams), ("flags", C.c_int32), ("reserved_", C.c_int32), ("certify", CertifyParams), ("dynamics", DynamicsParams),
                ("frontpath", FrontPathParams)]


class FrontierCluster(C.Structure):
    """isdf_frontier_cluster"""
    _fields_ = [("id", C.c_int64), ("size", C.c_int64), ("bmin", C.c_int32 * 3), ("bmax", C.c_int32 * 3), ("centroid", C.c_double * 3)]


class FrontierInfo(C.Structure):
    """isdf_frontier_info"""
    _fields_ = [("traversable_blocked", C.c_int64), ("frontier_voxels", C.c_int64), ("clusters", C.c_int64), ("reserved_", C.c_int64)] + \
               [(n, C.c_double) for n in ["traversability_ms", "frontier_ms", "cluster_ms", "field_ms", "select_ms"]]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved_"}


class FrontierParams(C.Structure):
    """isdf_frontier_params"""
    _fields_ = [("goal_weight", C.c_double), ("min_cluster_voxels", C.c_int32), ("reserved_", C.c_int32)]


class FrontierGoal(C.Structure):
    """isdf_frontier_goal"""
    _fields_ = [("kind", C.c_int32), ("gain", C.c_int32), ("voxel", C.c_int64), ("cluster", C.c_int64), ("g", C.c_double),
                ("score", C.c_double), ("point", C.c_double * 3)]


FRONTIER_GOAL_DTYPE = np.dtype([("kind", "<i4"), ("gain", "<i4"), ("voxel", "<i8"), ("cluster", "<i8"), ("g", "<f8"), ("score", "<f8"),
                                ("point", "<f8", (3,))])
FRONTIER_CLUSTER_DTYPE = np.dtype([("id", "<i8"), ("size", "<i8"), ("bmin", "<i4", (3,)), ("bmax", "<i4", (3,)), ("centroid", "<f8", (3,))])


def decode_frontier_goals(raw):
    """isdf_frontier_goal records ((B, 64) uint8 or a FRONTIER_GOAL_DTYPE array, on any device) -> a FRONTIER_GOAL_DTYPE array"""
    b = raw.cpu().numpy() if hasattr(raw, "cpu") else np.asarray(raw)
    return np.ascontiguousarray(b).view(np.uint8).reshape(-1).view(FRONTIER_GOAL_DTYPE).copy()


class PlanResult(C.Structure):
    """isdf_plan_result (one per goal)"""
    _fields_ = [(n, C.c_int32) for n in ["stage", "path_nodes", "pieces", "obstacle_points", "midend_ret", "backend_ret", "backend_iterations",
                                         "backend_evaluations"]] + [(n, C.c_double) for n in ["path_cost", "midend_f", "backend_f", "duration"]]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class PlanInfo(C.Structure):
    """isdf_plan_info"""
    _fields_ = [("groups", C.c_int32), ("backend_rounds", C.c_int32)] + \
               [(n, C.c_double) for n in ["frontend_ms", "midend_ms", "gather_ms", "backend_ms", "certify_ms", "dynamics_ms"]]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class SweptParams(C.Structure):
    """isdf_swept_params"""
    _fields_ = [("samples_per_piece", C.c_int32), ("max_depth", C.c_int32), ("max_samples_per_point", C.c_int32), ("reserved_", C.c_int32),
                ("tol", C.c_double), ("band", C.c_double)]


class SweptGrid(C.Structure):
    """isdf_swept_grid"""
    _fields_ = [("bmin", C.c_double * 3), ("res", C.c_double), ("X", C.c_int32), ("Y", C.c_int32), ("Z", C.c_int32), ("reserved_", C.c_int32)]


class SweptInfo(C.Structure):
    """isdf_swept_info"""
    _fields_ = [("nodes", C.c_int64), ("bricks", C.c_int64), ("bricks_culled", C.c_int64), ("sdf_evals", C.c_int64), ("undecided", C.c_int64),
                ("deepest", C.c_int32), ("reserved_", C.c_int32), ("prep_ms", C.c_double), ("cull_ms", C.c_double), ("refine_ms", C.c_double),
                ("mesh_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved_"}


def swept_grid_for(T, coeffs, r_body, band, res, samples_per_piece=64):
    """an isdf_swept_grid covering the trajectory's bounding box inflated by r_body + band + res, node spacing res. The box is taken over
    the piece polynomials at samples_per_piece + 1 times per piece, widened by the largest distance between consecutive samples, so the
    whole path lies inside it."""
    T = np.asarray(T, dtype=np.float64).reshape(-1)
    N = T.size
    c = np.asarray(coeffs, dtype=np.float64).reshape(3, 6 * N)
    pts = []
    for i in range(N):
        t = np.linspace(0.0, T[i], samples_per_piece + 1)
        pts.append((c[:, 6 * i:6 * i + 6] @ (t[None, :] ** np.arange(6)[:, None])).T)
    P = np.concatenate(pts)
    gap = float(np.max(np.linalg.norm(np.diff(P, axis=0), axis=1))) if len(P) > 1 else 0.0
    pad = float(r_body) + float(band) + float(res) + gap
    lo, hi = P.min(axis=0) - pad, P.max(axis=0) + pad
    n = np.maximum(np.ceil((hi - lo) / res).astype(int) + 1, 2)
    g = SweptGrid()
    g.bmin[:] = [float(x) for x in lo]
    g.res = float(res)
    g.X, g.Y, g.Z = (int(x) for x in n)
    return g


def swept_grid_nodes(g):
    """(X, Y, Z, 3) node coordinates of an isdf_swept_grid, computed as the library does: bmin[a] + (double) i * res"""
    ax = [g.bmin[a] + np.arange(n, dtype=np.float64) * g.res for a, n in enumerate((g.X, g.Y, g.Z))]
    return np.stack(np.meshgrid(*ax, indexing="ij"), axis=-1)


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


class FuseInfo(C.Structure):
    """isdf_fuse_info"""
    _fields_ = [(n, C.c_int64) for n in ["points_used", "points_outside", "points_skipped", "voxels_added"]]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class ObserveInfo(C.Structure):
    """isdf_observe_info"""
    _fields_ = [(n, C.c_int64) for n in ["poses", "voxels_tested", "voxels_added"]]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


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
    spp, sgp, sip = C.POINTER(SweptParams), C.POINTER(SweptGrid), C.POINTER(SweptInfo)
    lib.isdf_dynamics_default_params.argtypes = [vp, C.POINTER(DynamicsParams)]
    lib.isdf_trajectory_dynamics.argtypes = [vp, C.c_int, dp, dp, C.POINTER(DynamicsParams), C.POINTER(DynamicsSummary)]
    lib.isdf_trajectory_dynamics_device.argtypes = [vp, C.c_int, vp, vp, C.POINTER(DynamicsParams), vp, vp]
    lib.isdf_swept_default_params.argtypes = [spp]
    lib.isdf_swept_volume_sdf.argtypes = [vp, C.c_int, dp, dp, spp, C.c_int, dp, dp, dp, dp, C.POINTER(C.c_uint8)]
    lib.isdf_swept_volume_grid.argtypes = [vp, C.c_int, dp, dp, spp, sgp, dp, dp, dp, C.POINTER(C.c_uint8), sip]
    lib.isdf_swept_volume_grid_device.argtypes = [vp, C.c_int, vp, vp, spp, sgp, vp, vp, vp, vp, sip, vp]
    lib.isdf_swept_volume_mesh.argtypes = [vp, C.c_int, dp, dp, spp, sgp, C.c_int64, C.c_int64, dp, dp, ip, C.POINTER(C.c_int64),
                                           C.POINTER(C.c_int64), sip]
    lib.isdf_set_map_cloud.argtypes = [vp, vp, C.c_int64, C.c_int32, C.c_double, C.c_int32]
    lib.isdf_set_map_cloud_device.argtypes = [vp, vp, C.c_int64, C.c_int32, C.c_double, C.c_int32, vp]
    lib.isdf_get_map_info.argtypes = [vp, C.POINTER(MapInfo)]
    lib.isdf_map_fuse_cloud.argtypes = [vp, vp, C.c_int64, C.c_int32, C.POINTER(FuseInfo)]
    lib.isdf_map_fuse_cloud_device.argtypes = [vp, vp, C.c_int64, C.c_int32, C.POINTER(FuseInfo), vp]
    lib.isdf_trajectory_shift.argtypes = [vp, C.c_int, ip, dp, dp, dp, ip, dp, dp]
    lib.isdf_trajectory_shift_device.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.isdf_brake_default_params.argtypes = [vp, C.POINTER(BrakeParams)]
    lib.isdf_trajectory_brake.argtypes = [vp, C.c_int, ip, dp, dp, dp, C.POINTER(BrakeParams), ip, dp, dp, C.POINTER(BrakeSummary)]
    lib.isdf_trajectory_brake_device.argtypes = [vp, C.c_int, vp, vp, vp, vp, C.POINTER(BrakeParams), vp, vp, vp, vp, vp]
    lib.isdf_get_map_u8.argtypes = [vp, C.POINTER(C.c_uint8), C.c_int64]
    lib.isdf_get_map_known_u8.argtypes = [vp, C.POINTER(C.c_uint8), C.c_int64]
    lib.isdf_map_mark_known.argtypes = [vp, C.c_int64, vp]
    lib.isdf_set_unknown_policy.argtypes = [vp, C.c_int]
    lib.isdf_get_unknown_policy.argtypes = [vp, C.POINTER(C.c_int)]
    lib.isdf_get_map_f64.argtypes = [vp, dp, C.c_int64]
    lib.isdf_map_esdf.argtypes = [vp]
    lib.isdf_get_esdf_f64.argtypes = [vp, C.c_int, dp, C.c_int64]
    lib.isdf_esdf_query.argtypes = [vp, C.c_int, dp, C.c_int64, dp, dp]
    lib.isdf_esdf_query_device.argtypes = [vp, C.c_int, vp, C.c_int64, vp, vp, vp]
    fpp, u8p = C.POINTER(FrontPathParams), C.POINTER(C.c_uint8)
    lib.isdf_frontend_path.argtypes = [vp, dp, dp, fpp, C.c_int, dp, dp, ip, dp, u8p]
    lib.isdf_frontend_path_batch.argtypes = [vp, dp, C.c_int, dp, fpp, C.c_int, dp, dp, ip, dp, u8p]
    lib.isdf_frontend_path_batch_device.argtypes = [vp, dp, C.c_int, vp, fpp, C.c_int, vp, vp, vp, vp, vp, vp]
    lib.isdf_frontend_path_field_device.argtypes = [vp, dp, fpp, vp, vp]
    lib.isdf_frontend_path_info.argtypes = [vp, C.POINTER(FrontPathInfo)]
    lib.isdf_frontend_path_pairs.argtypes = [vp, C.c_int, dp, dp, fpp, C.c_int, C.c_int, dp, dp, ip, dp, u8p]
    lib.isdf_frontend_path_pairs_device.argtypes = [vp, C.c_int, vp, vp, fpp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]
    lib.isdf_frontend_path_fields_device.argtypes = [vp, C.c_int, dp, fpp, vp, vp]
    frp, fip = C.POINTER(FrontierParams), C.POINTER(FrontierInfo)
    lib.isdf_map_frontiers.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, vp, fip]
    lib.isdf_map_frontiers_device.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, vp, fip, vp]
    lib.isdf_frontier_default_params.argtypes = [frp]
    lib.isdf_frontier_goals.argtypes = [vp, C.c_int, dp, dp, frp, C.c_int, vp, fip]
    lib.isdf_frontier_goals_device.argtypes = [vp, C.c_int, vp, vp, frp, C.c_int, vp, fip, vp]
    lib.isdf_frontier_goals_view.argtypes = [vp, C.c_int, dp, dp, frp, C.c_int, vp, C.c_int64, C.c_int, vp, fip]
    lib.isdf_frontier_goals_view_device.argtypes = [vp, C.c_int, vp, vp, frp, C.c_int, vp, C.c_int64, C.c_int, vp, fip, vp]
    mpp = C.POINTER(MidendParams)
    lib.isdf_path_waypoints.argtypes = [C.c_int, ip, dp, C.c_double, C.c_double, C.c_int, dp, ip, ip]
    lib.isdf_midend_default_params.argtypes = [mpp]
    lib.isdf_midend_callback_batch.argtypes = [vp, C.c_int, C.c_int, dp, dp, C.c_int, mpp, dp, dp, dp, dp]
    lib.isdf_midend_batch.argtypes = [vp, C.c_int, C.c_int, dp, dp, C.c_int, mpp, dp, dp, dp, dp, dp, ip, ip, ip, ip]
    lib.isdf_midend_batch_device.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_int, mpp, vp, vp, vp, vp, vp, vp, vp, vp, ip, vp]
    lib.isdf_gather_obstacle_points_batch.argtypes = [vp, C.c_int, ip, dp, C.c_double, dp, C.c_int64, dp, ip, C.c_int]
    lib.isdf_gather_obstacle_points_batch_known.argtypes = [vp, C.c_int, ip, dp, C.c_double, dp, ip, C.c_int64, dp, ip, C.c_int]
    lib.isdf_plan_default_params.argtypes = [vp, C.POINTER(PlanParams)]
    lib.isdf_plan_batch.argtypes = [vp, dp, C.c_int, dp, C.POINTER(PlanParams), C.c_int, ip, dp, C.c_int, ip, dp, dp, C.POINTER(PlanResult),
                                    C.POINTER(CertifySummary), C.POINTER(DynamicsSummary)]
    lib.isdf_plan_pairs.argtypes = [vp, C.c_int, dp, dp, C.POINTER(PlanParams), C.c_int, C.c_int, ip, dp, C.c_int, ip, dp, dp,
                                    C.POINTER(PlanResult), C.POINTER(CertifySummary), C.POINTER(DynamicsSummary)]
    lib.isdf_get_plan_info.argtypes = [vp, C.POINTER(PlanInfo)]
    lib.isdf_callback_batch_ragged.argtypes = [vp, C.c_int, ip, dp, dp, C.c_int, C.c_double, dp, dp, dp]
    lib.isdf_callback_batch_ragged_device.argtypes = [vp, C.c_int, ip, vp, vp, C.c_int, C.c_double, vp, vp, vp, vp]
    lib.isdf_lbfgs_batch_ragged.argtypes = [vp, C.c_int, ip, dp, dp, C.c_int, C.c_double, C.POINTER(LbfgsParams), dp, dp, ip, ip, ip, ip]
    lib.isdf_lbfgs_batch_ragged_device.argtypes = [vp, C.c_int, ip, vp, vp, C.c_int, C.c_double, C.POINTER(LbfgsParams), vp, vp, vp, vp, vp, ip, vp]
    lib.isdf_midend_callback_batch_ragged.argtypes = [vp, C.c_int, ip, dp, dp, C.c_int, mpp, dp, dp, dp, dp]
    lib.isdf_midend_batch_ragged.argtypes = [vp, C.c_int, ip, dp, dp, C.c_int, mpp, dp, dp, dp, dp, dp, ip, ip, ip, ip]
    lib.isdf_midend_batch_ragged_device.argtypes = [vp, C.c_int, ip, vp, vp, C.c_int, mpp, vp, vp, vp, vp, vp, vp, vp, vp, ip, vp]
    lib.isdf_trajectory_states.argtypes = [vp, C.c_int, ip, dp, dp, C.c_int64, ip, dp, dp]
    lib.isdf_trajectory_states_device.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int64, vp, vp, vp, vp]
    lib.isdf_pose_points.argtypes = [vp, C.c_int64, dp, C.c_int, dp, dp]
    lib.isdf_pose_points_device.argtypes = [vp, C.c_int64, vp, C.c_int, vp, vp, vp]
    lib.isdf_path_waypoints_device.argtypes = [vp, C.c_int, vp, vp, C.c_double, C.c_double, C.c_int, vp, vp, vp, vp]
    lib.isdf_plan_pairs_device.argtypes = [vp, C.c_int, vp, vp, C.POINTER(PlanParams), C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, vp,
                                           vp, vp]
    lib.isdf_plan_states.argtypes = lib.isdf_plan_pairs.argtypes
    lib.isdf_plan_states_device.argtypes = lib.isdf_plan_pairs_device.argtypes
    lib.isdf_plan_batch_device.argtypes = [vp, dp, C.c_int, vp, C.POINTER(PlanParams), C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    pcp = C.POINTER(PoseClearanceParams)
    lib.isdf_pose_clearance_default_params.argtypes = [pcp]
    lib.isdf_pose_clearance.argtypes = [vp, C.c_int64, dp, dp, C.c_int64, pcp, dp, C.POINTER(C.c_int64), C.POINTER(ClearanceSummary)]
    lib.isdf_pose_clearance_device.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, pcp, vp, vp, vp, vp]
    sep = C.POINTER(SenseParams)
    lib.isdf_sense_default_params.argtypes = [sep]
    lib.isdf_set_sense_cloud.argtypes = [vp, vp, C.c_int64, C.c_int32]
    lib.isdf_set_sense_cloud_device.argtypes = [vp, vp, C.c_int64, C.c_int32, vp]
    lib.isdf_get_sense_info.argtypes = [vp, C.POINTER(SenseInfo)]
    lib.isdf_sense_depth.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, sep, vp]
    lib.isdf_map_observe.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, sep, C.POINTER(ObserveInfo)]
    lib.isdf_map_observe_device.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, sep, C.POINTER(ObserveInfo), vp]
    lib.isdf_view_gain.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, C.c_int, vp, vp]
    lib.isdf_view_gain_device.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, C.c_int, vp, vp, vp]
    lib.isdf_sense_depth_device.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, sep, vp, vp]
    lib.isdf_sense_cloud.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, sep, C.c_int64, vp, vp]
    lib.isdf_sense_cloud_device.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, sep, C.c_int64, vp, vp, vp]
    wpp = C.POINTER(WorldParams)
    lib.isdf_world_default_params.argtypes = [C.c_int, wpp]
    lib.isdf_world_cloud.argtypes = [vp, wpp, C.c_int64, vp, C.POINTER(C.c_int64)]
    lib.isdf_world_cloud_device.argtypes = [vp, wpp, C.c_int64, vp, C.POINTER(C.c_int64), vp]
    spp = C.POINTER(SimParams)
    lib.isdf_sim_default_params.argtypes = [spp]
    lib.isdf_simulate.argtypes = [vp, C.c_int, ip, dp, dp, C.c_int, ip, dp, dp, spp, C.c_int, dp, C.POINTER(SimSummary)]
    lib.isdf_simulate_device.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, spp, C.c_int, vp, vp, vp]
    for s in ABI_SYMBOLS:
        if s != "isdf_last_error":
            getattr(lib, s).restype = C.c_int
    if path is None:
        _lib = lib
    return lib


def _colmajor(a):
    """3x3 (or B x 3x3) row-major -> the library's column-major order"""
    return np.ascontiguousarray(np.swapaxes(np.asarray(a, dtype=np.float64), -1, -2)).reshape(-1)


class Ragged:
    """The layout of a ragged batch (include/isdf.h): problem b has N_b = pieces[b] pieces, piece_off = [0, N_0, N_0 + N_1, ...]. pack_*
    concatenates per-problem arrays into the library's layout, unpack_* splits its outputs back into per-problem arrays."""

    def __init__(self, pieces):
        self.pieces = np.asarray(pieces, dtype=np.int64).reshape(-1)
        assert self.pieces.size >= 1 and (self.pieces >= 1).all(), "every problem needs at least one piece"
        self.B = int(self.pieces.size)
        self.piece_off = np.zeros(self.B + 1, dtype=np.int32)
        self.piece_off[1:] = np.cumsum(self.pieces)
        self.P = int(self.piece_off[-1])
        b = np.arange(self.B + 1)
        self.x_off = 4 * self.piece_off.astype(np.int64) - 3 * b            # decision-vector rows [x_off[b], x_off[b+1])
        self.wp_off = self.piece_off.astype(np.int64) - b                   # waypoint rows [wp_off[b], wp_off[b+1])

    def ptr(self):
        return self.piece_off.ctypes.data_as(C.POINTER(C.c_int32))

    @staticmethod
    def _cat(parts):
        parts = [np.asarray(p, dtype=np.float64).reshape(-1) for p in parts]
        return np.ascontiguousarray(np.concatenate(parts)) if parts else np.zeros(0)

    def pack_x(self, xs):
        """B decision vectors [tau (N_b) | xi (3(N_b-1))] -> 4P - 3B rows"""
        assert len(xs) == self.B and all(np.size(x) == 4 * n - 3 for x, n in zip(xs, self.pieces))
        return self._cat(xs)

    def unpack_x(self, x):
        return [np.asarray(x[self.x_off[b]:self.x_off[b + 1]]).copy() for b in range(self.B)]

    def pack_waypoints(self, wps):
        """B arrays of (N_b - 1, 3) waypoints -> (P - B) x 3 rows, the wp_off layout of isdf_path_waypoints"""
        assert len(wps) == self.B and all(np.size(w) == 3 * (n - 1) for w, n in zip(wps, self.pieces))
        return self._cat(wps)

    def pack_T(self, Ts):
        assert len(Ts) == self.B and all(np.size(t) == n for t, n in zip(Ts, self.pieces))
        return self._cat(Ts)

    def unpack_T(self, T):
        return [np.asarray(T[self.piece_off[b]:self.piece_off[b + 1]]).copy() for b in range(self.B)]

    def pack_coeffs(self, Cs):
        """B per-problem 6N_b x 3 column-major blocks (18 N_b values each) -> one 6P x 3 column-major block"""
        assert len(Cs) == self.B and all(np.size(c) == 18 * n for c, n in zip(Cs, self.pieces))
        out = np.zeros((3, 6 * self.P))
        for b, c in enumerate(Cs):
            out[:, 6 * self.piece_off[b]:6 * self.piece_off[b + 1]] = np.asarray(c, dtype=np.float64).reshape(3, -1)
        return out.reshape(-1)

    def unpack_coeffs(self, Cc):
        """one 6P x 3 column-major block -> B per-problem 6N_b x 3 column-major blocks (18 N_b values each)"""
        c3 = np.asarray(Cc).reshape(3, 6 * self.P)
        return [c3[:, 6 * self.piece_off[b]:6 * self.piece_off[b + 1]].reshape(-1).copy() for b in range(self.B)]


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


def _cat_plans(parts):
    """the outputs of plan_*_device calls (dicts of CUDA tensors) as one call's, plans in order"""
    import torch
    if len(parts) == 1:
        return parts[0]
    out = dict(parts[0])
    for q in parts[1:]:
        for k in ("path_off", "piece_off"):
            out[k] = torch.cat([out[k], q[k][1:] + out[k][-1]])
        for k in ("path_xyz", "T", "coeffs", "results", "certify", "dynamics"):
            if out[k] is not None:
                out[k] = torch.cat([out[k], q[k]])
    return out


def _cuda_f64(t):
    """a contiguous float64 CUDA tensor (no copy when t already is one)"""
    import torch
    if not t.is_cuda:
        raise ValueError("expected a CUDA tensor")
    return t.to(torch.float64).contiguous()


def decode_plan_results(records):
    """isdf_plan_result records (B x 64 uint8, as plan_pairs_device returns them; any device) -> dict of per-field tensors of length B"""
    return {n: _field(records, PlanResult, n) for n, _ in PlanResult._fields_}


def _field(rows, struct, name):
    """field `name` of (n, sizeof(struct)) uint8 rows of ctypes struct records (a tensor on any device) -> its column as a tensor of the
    field's type: (n,), or (n, k) for an array of k"""
    import torch
    t = dict(struct._fields_)[name]
    base = t._type_ if issubclass(t, C.Array) else t
    dtype = {C.c_int32: torch.int32, C.c_int64: torch.int64, C.c_double: torch.float64}[base]
    f = getattr(struct, name)
    col = rows.reshape(-1, C.sizeof(struct))[:, f.offset:f.offset + f.size].contiguous().view(dtype)
    return col if issubclass(t, C.Array) else col.reshape(-1)


def _rows(d, off, j):
    """trajectory j's (T, coeffs) in a ragged dict d (piece_off, T, coeffs), given its piece_off read to the host as off"""
    a, e = int(off[j]), int(off[j + 1])
    return d["T"][a:e], d["coeffs"][18 * a:18 * e]


def _ragged(pieces, dev):
    """(host offsets, piece_off int32 on dev, T, coeffs) of a list of trajectories (T, coeffs) in isdf_plan_batch's ragged layout, in list
    order; without any piece, T and coeffs are one zero piece (the calls need non-NULL arrays)"""
    import torch
    offh = np.zeros(len(pieces) + 1, dtype=np.int64)
    offh[1:] = np.cumsum([t.shape[0] for t, _ in pieces])
    if offh[-1]:
        T, Cc = torch.cat([t for t, _ in pieces]), torch.cat([c for _, c in pieces])
    else:
        T, Cc = torch.zeros(1, dtype=torch.float64, device=dev), torch.zeros(18, dtype=torch.float64, device=dev)
    return offh, torch.as_tensor(offh.astype(np.int32), device=dev), T, Cc


class _Fleet:
    """Evaluator.navigate's trajectories, one per vehicle, in isdf_plan_batch's ragged layout: piece counts n and offsets offh on the host,
    piece_off, T and coeffs on the device. T and coeffs may run past piece_off[B] (as trajectory_shift_device's output does)."""

    def __init__(self, B, dev):
        import torch
        self.dev, self.n = dev, np.zeros(B, dtype=np.int64)
        none = torch.zeros(0, dtype=torch.float64, device=dev)
        self.replace({b: (none, none) for b in range(B)})

    def pieces(self, b):
        a, e = self.offh[b], self.offh[b + 1]
        return self.T[a:e], self.coeffs[18 * a:18 * e]

    def gather(self, vehicles):
        """(piece_off int32, T, coeffs) of these vehicles' trajectories, in this order"""
        return _ragged([self.pieces(b) for b in vehicles], self.dev)[1:]

    def replace(self, new):
        """vehicle b's trajectory becomes new[b] = (T, coeffs) (no pieces: none); the others keep theirs"""
        self.offh, self.piece_off, self.T, self.coeffs = _ragged([new[b] if b in new else self.pieces(b) for b in range(self.n.size)], self.dev)
        self.n = np.diff(self.offh)

    def adopt(self, d):
        """take trajectory_shift_device's output dict as the trajectories (one read of its piece_off)"""
        self.piece_off, self.T, self.coeffs = d["piece_off"], d["T"], d["coeffs"]
        self.offh = self.piece_off.cpu().numpy().astype(np.int64)
        self.n = np.diff(self.offh)


def _host_ragged(plans_or_ragged):
    """plan_batch's list of dicts, or (piece_off, T, coeffs) in isdf_plan_batch's ragged layout -> (piece_off int32, T, coeffs) host arrays"""
    if isinstance(plans_or_ragged, tuple):
        off, T, Cc = plans_or_ragged
        return np.ascontiguousarray(off, dtype=np.int32).reshape(-1), _f64(T).reshape(-1), _f64(Cc).reshape(-1)
    return Evaluator.pack_plans(plans_or_ragged)


@contextlib.contextmanager
def _timed(events, stream):
    """record the CUDA event pair events = (start, end) on stream around a block"""
    events[0].record(stream)
    yield
    events[1].record(stream)


def _rig(params):
    """one sense_params or a list of them -> a ctypes array of SenseParams (the library refuses an empty one)"""
    cams = list(params) if isinstance(params, (list, tuple)) else [params if params is not None else sense_params()]
    return (SenseParams * len(cams))(*cams)


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
        self.device = device

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
        pts, n, stride = _cloud_records(points, stride_bytes)
        self._check(self.lib.isdf_set_map_cloud(self.h, pts.ctypes.data_as(C.c_void_p) if n else None, n, stride, float(res), int(sta_threshold)))

    def set_map_cloud_device(self, points, n=None, stride_bytes=None, res=1.0, sta_threshold=1, stream=0):
        """points on the context's device: a float32 torch tensor (n, k >= 3), contiguous, or a raw device pointer with n and stride_bytes"""
        ptr, n, stride = _cloud_records_device(points, n, stride_bytes)
        self._check(self.lib.isdf_set_map_cloud_device(self.h, C.c_void_p(ptr), int(n), stride, float(res), int(sta_threshold), C.c_void_p(stream)))

    def map_fuse_cloud(self, points, stride_bytes=None):
        """adds a host cloud (as set_map_cloud takes it) to the current map in its frame (isdf_map_fuse_cloud) -> dict(points_used,
        points_outside, points_skipped, voxels_added)"""
        pts, n, stride = _cloud_records(points, stride_bytes)
        info = FuseInfo()
        self._check(self.lib.isdf_map_fuse_cloud(self.h, pts.ctypes.data_as(C.c_void_p) if n else None, n, stride, C.byref(info)))
        return info.as_dict()

    def map_fuse_cloud_device(self, points, n=None, stride_bytes=None, stream=0):
        """adds a device cloud (as set_map_cloud_device takes it; sense_cloud_device's points as they are) to the current map in its frame
        -> the isdf_fuse_info dict. Returns when the map is updated."""
        ptr, n, stride = _cloud_records_device(points, n, stride_bytes)
        info = FuseInfo()
        self._check(self.lib.isdf_map_fuse_cloud_device(self.h, C.c_void_p(ptr), int(n), stride, C.byref(info), C.c_void_p(stream)))
        return info.as_dict()

    # ---- depth sensing (isdf_sense_*): the scene cloud, depth images and sensed points at poses read in place ----
    def set_sense_cloud(self, points, stride_bytes=None):
        """the scene the camera sees: points as set_map_cloud takes them (records with a NaN or Inf coordinate are skipped)"""
        pts, n, stride = _cloud_records(points, stride_bytes)
        self._check(self.lib.isdf_set_sense_cloud(self.h, pts.ctypes.data_as(C.c_void_p) if n else None, n, stride))

    def set_sense_cloud_device(self, points, n=None, stride_bytes=None, stream=0):
        """the scene on the context's device, as set_map_cloud_device takes it"""
        ptr, n, stride = _cloud_records_device(points, n, stride_bytes)
        self._check(self.lib.isdf_set_sense_cloud_device(self.h, C.c_void_p(ptr), int(n), stride, C.c_void_p(stream)))

    def sense_info(self):
        """dict(points_used, points_skipped, bricks) of the scene cloud"""
        i = SenseInfo()
        self._check(self.lib.isdf_get_sense_info(self.h, C.byref(i)))
        return {n: getattr(i, n) for n, _ in i._fields_}

    @staticmethod
    def _pose_records(r, pos_offset, quat_offset):
        Q, stride = r.shape
        if not (0 <= pos_offset <= stride - 3 and 0 <= quat_offset <= stride - 4):
            raise ValueError("pos_offset / quat_offset outside the record")
        return Q, stride

    def sense_depth(self, records, pos_offset=0, quat_offset=3, params=None, **kw):
        """depth images (Q, H, W) int32 in mm (999999: nothing seen) at Q poses read in place from records (Q, stride) float64, as
        pose_clearance reads them (a simulate log: offsets 1 and 7; trajectory_states records: 0 and 12). params: sense_params(**kw)."""
        p = params if params is not None else sense_params(**kw)
        r = _f64(records)
        r = r.reshape(-1, r.shape[-1])
        Q, stride = self._pose_records(r, pos_offset, quat_offset)
        out = np.empty((Q, max(p.height, 0), max(p.width, 0)), dtype=np.int32)   # bad sizes are the library's to refuse
        base = r.ctypes.data
        self._check(self.lib.isdf_sense_depth(self.h, Q, C.c_void_p(base + 8 * pos_offset), C.c_void_p(base + 8 * quat_offset), stride,
                                              C.byref(p), out.ctypes.data_as(C.c_void_p)))
        return out

    def sense_depth_device(self, records, pos_offset=0, quat_offset=3, params=None, stream=None, **kw):
        """sense_depth on a float64 CUDA tensor (Q, stride) (rows may be strided views of a larger record, e.g. a simulate log reshaped to
        (R * n_log, 21)) -> (Q, H, W) int32 CUDA tensor, on torch's current stream"""
        import torch
        p = params if params is not None else sense_params(**kw)
        r = _cuda_records(records)
        Q, stride = self._pose_records(r, pos_offset, quat_offset)
        s = torch.cuda.current_stream(r.device) if stream is None else stream
        with torch.cuda.stream(s):
            out = torch.empty((Q, max(p.height, 0), max(p.width, 0)), dtype=torch.int32, device=r.device)
        base = r.data_ptr()
        self._check(self.lib.isdf_sense_depth_device(self.h, Q, C.c_void_p(base + 8 * pos_offset), C.c_void_p(base + 8 * quat_offset), stride,
                                                     C.byref(p), C.c_void_p(out.data_ptr()), C.c_void_p(s.cuda_stream)))
        return out

    def sense_cloud(self, records, pos_offset=0, quat_offset=3, params=None, cap=None, **kw):
        """the sensed points of Q poses -> (points (M, 3) float32, offsets (Q + 1) int64): pose q's in rows [offsets[q], offsets[q+1]).
        cap: rows to allocate (default 2^22); too small, the call is repeated once with the total the first call reported."""
        p = params if params is not None else sense_params(**kw)
        r = _f64(records)
        r = r.reshape(-1, r.shape[-1])
        Q, stride = self._pose_records(r, pos_offset, quat_offset)
        cap = min(Q * p.width * p.height, 1 << 22) if cap is None else int(cap)
        base = r.ctypes.data
        off = np.zeros(Q + 1, dtype=np.int64)
        for attempt in range(2):
            pts = np.empty((max(cap, 1), 3), dtype=np.float32)
            rc = self.lib.isdf_sense_cloud(self.h, Q, C.c_void_p(base + 8 * pos_offset), C.c_void_p(base + 8 * quat_offset), stride, C.byref(p),
                                           cap, pts.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p))
            if rc == 0:
                return pts[:off[Q]], off
            if attempt == 0 and off[Q] > cap:
                cap = int(off[Q])
                continue
            self._check(rc)

    def sense_cloud_device(self, records, pos_offset=0, quat_offset=3, params=None, cap=None, stream=None, **kw):
        """sense_cloud on a float64 CUDA tensor (Q, stride) -> (points (M, 3) float32 CUDA tensor, offsets (Q + 1) int64 CUDA tensor), on
        torch's current stream. points goes into set_map_cloud_device as it is. Caps as in sense_cloud."""
        import torch
        p = params if params is not None else sense_params(**kw)
        r = _cuda_records(records)
        Q, stride = self._pose_records(r, pos_offset, quat_offset)
        cap = min(Q * p.width * p.height, 1 << 22) if cap is None else int(cap)
        s = torch.cuda.current_stream(r.device) if stream is None else stream
        base = r.data_ptr()
        for attempt in range(2):
            with torch.cuda.stream(s):
                pts = torch.empty((max(cap, 1), 3), dtype=torch.float32, device=r.device)
                off = torch.zeros(Q + 1, dtype=torch.int64, device=r.device)
            rc = self.lib.isdf_sense_cloud_device(self.h, Q, C.c_void_p(base + 8 * pos_offset), C.c_void_p(base + 8 * quat_offset), stride,
                                                  C.byref(p), cap, C.c_void_p(pts.data_ptr()), C.c_void_p(off.data_ptr()),
                                                  C.c_void_p(s.cuda_stream))
            if rc == 0:
                return pts[:int(off[Q])], off
            total = int(off[Q])
            if attempt == 0 and total > cap:
                cap = total
                continue
            self._check(rc)

    # ---- known space (isdf_map_observe, isdf_map_mark_known, isdf_set_unknown_policy) ----
    def map_observe(self, records, pos_offset=0, quat_offset=3, params=None, **kw):
        """marks known the voxels the depth images at Q poses (read as sense_depth reads them) prove empty; params needs a finite
        sensing_horizon -> dict(poses, voxels_tested, voxels_added)"""
        p = params if params is not None else sense_params(**kw)
        r = _f64(records)
        r = r.reshape(-1, r.shape[-1])
        Q, stride = self._pose_records(r, pos_offset, quat_offset)
        base = r.ctypes.data
        info = ObserveInfo()
        self._check(self.lib.isdf_map_observe(self.h, Q, C.c_void_p(base + 8 * pos_offset), C.c_void_p(base + 8 * quat_offset), stride,
                                              C.byref(p), C.byref(info)))
        return info.as_dict()

    def map_observe_device(self, records, pos_offset=0, quat_offset=3, params=None, stream=None, **kw):
        """map_observe on a float64 CUDA tensor (Q, stride), read on torch's current stream (or stream); returns when the bits are set"""
        import torch
        p = params if params is not None else sense_params(**kw)
        r = _cuda_records(records)
        Q, stride = self._pose_records(r, pos_offset, quat_offset)
        s = torch.cuda.current_stream(r.device) if stream is None else stream
        base = r.data_ptr()
        info = ObserveInfo()
        self._check(self.lib.isdf_map_observe_device(self.h, Q, C.c_void_p(base + 8 * pos_offset), C.c_void_p(base + 8 * quat_offset), stride,
                                                     C.byref(p), C.byref(info), C.c_void_p(s.cuda_stream)))
        return info.as_dict()

    # ---- view gain (isdf_view_gain): the unknown voxels a rig of cameras would observe from a pose ----
    def view_gain(self, records, pos_offset=0, quat_offset=3, params=None):
        """the view gain of Q poses read in place from records (Q, stride) float64 (as sense_depth reads them) for the rig params (one
        sense_params or a list of them, each with a finite sensing_horizon) -> (Q,) int64 numpy"""
        cams = _rig(params)
        r = _f64(records)
        r = r.reshape(-1, r.shape[-1])
        Q, stride = self._pose_records(r, pos_offset, quat_offset)
        out = np.zeros(Q, dtype=np.int64)
        base = r.ctypes.data
        self._check(self.lib.isdf_view_gain(self.h, Q, C.c_void_p(base + 8 * pos_offset), C.c_void_p(base + 8 * quat_offset), stride, len(cams),
                                            C.byref(cams), out.ctypes.data_as(C.c_void_p)))
        return out

    def view_gain_device(self, records, pos_offset=0, quat_offset=3, params=None, stream=None):
        """view_gain on a float64 CUDA tensor (Q, stride), on torch's current stream (or stream) -> (Q,) int64 CUDA tensor"""
        import torch
        cams = _rig(params)
        r = _cuda_records(records)
        Q, stride = self._pose_records(r, pos_offset, quat_offset)
        s = torch.cuda.current_stream(r.device) if stream is None else stream
        with torch.cuda.stream(s):
            out = torch.empty(Q, dtype=torch.int64, device=r.device)
        base = r.data_ptr()
        self._check(self.lib.isdf_view_gain_device(self.h, Q, C.c_void_p(base + 8 * pos_offset), C.c_void_p(base + 8 * quat_offset), stride,
                                                   len(cams), C.byref(cams), C.c_void_p(out.data_ptr()), C.c_void_p(s.cuda_stream)))
        return out

    def map_mark_known(self, boxes):
        """marks known every voxel whose cube lies inside one of the closed boxes (n, 6): lo xyz, hi xyz (the caller asserts they are free)"""
        b = np.ascontiguousarray(np.asarray(boxes, dtype=np.float64).reshape(-1, 6))
        self._check(self.lib.isdf_map_mark_known(self.h, b.shape[0], b.ctypes.data_as(C.c_void_p) if b.size else None))

    def get_map_known_u8(self):
        """the known grid (X, Y, Z) uint8 in get_map_u8's layout"""
        X, Y, Z = self.map_info()["dims"]
        out = np.empty((X, Y, Z), dtype=np.uint8)
        self._check(self.lib.isdf_get_map_known_u8(self.h, out.ctypes.data_as(C.POINTER(C.c_uint8)), out.size))
        return out

    def set_unknown_policy(self, policy):
        """UNKNOWN_FREE (the default) or UNKNOWN_OCCUPIED: what the clearance family takes voxels nobody has seen to be"""
        self._check(self.lib.isdf_set_unknown_policy(self.h, int(policy)))

    def unknown_policy(self):
        v = C.c_int(-1)
        self._check(self.lib.isdf_get_unknown_policy(self.h, C.byref(v)))
        return v.value

    # ---- world generators (isdf_world_*): the reference's globalmap_gene and mockamap worlds as (n, 4) float32 clouds ----
    @staticmethod
    def world_params(kind, **overrides):
        """isdf_world_params of kind ("globalmap", "perlin", "boxes") with the reference's defaults and the given fields replaced"""
        return world_params(kind, **overrides)

    def _world_p(self, params, kind, kw):
        if params is not None:
            return params
        return world_params(kind if kind is not None else kw.pop("kind"), **kw)

    def world_cloud(self, params=None, kind=None, **kw):
        """the world's cloud -> (n, 4) float32 numpy array of (x, y, z, 1): one size query (cap 0), then the cloud"""
        p = self._world_p(params, kind, kw)
        n = C.c_int64(-1)
        rc = self.lib.isdf_world_cloud(self.h, C.byref(p), 0, None, C.byref(n))
        if n.value < 0:   # the size query answers ISDF_ERR_INVALID with *n written for a non-empty cloud; without *n it failed
            self._check(rc)
        out = np.empty((max(n.value, 1), 4), dtype=np.float32)
        self._check(self.lib.isdf_world_cloud(self.h, C.byref(p), n.value, out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return out[:n.value]

    def world_cloud_device(self, params=None, kind=None, stream=None, **kw):
        """the world's cloud -> (n, 4) float32 CUDA tensor on torch's current stream, for set_map_cloud_device(t.data_ptr(), n=n,
        stride_bytes=16) and set_sense_cloud_device as it is. The size is known after a size query (for Perlin, one run of the noise and
        selection), then the cloud is written."""
        import torch
        p = self._world_p(params, kind, kw)
        dev = torch.device("cuda", self.device)
        s = torch.cuda.current_stream(dev) if stream is None else stream
        n = C.c_int64(-1)
        rc = self.lib.isdf_world_cloud_device(self.h, C.byref(p), 0, None, C.byref(n), C.c_void_p(s.cuda_stream))
        if n.value < 0:
            self._check(rc)
        with torch.cuda.stream(s):
            out = torch.empty((max(n.value, 1), 4), dtype=torch.float32, device=dev)
        self._check(self.lib.isdf_world_cloud_device(self.h, C.byref(p), n.value, C.c_void_p(out.data_ptr()), C.byref(n),
                                                     C.c_void_p(s.cuda_stream)))
        return out[:n.value]

    def dbg_sense_chunk(self, poses):
        """render at most `poses` poses per chunk (0: automatic; isdf_dbg_sense_chunk, not part of include/isdf.h)"""
        self.lib.isdf_dbg_sense_chunk.argtypes = [C.c_void_p, C.c_int]
        self._check(self.lib.isdf_dbg_sense_chunk(self.h, int(poses)))

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

    # ---- distance field of the map (include/isdf.h: isdf_map_esdf) ----
    @staticmethod
    def _esdf_field(field):
        if field not in ESDF_FIELDS:
            raise ValueError(f"field must be one of {sorted(ESDF_FIELDS)}, got {field!r}")
        return ESDF_FIELDS[field]

    def map_esdf(self):
        """GridMap3D::generateESDF3d on the current map: builds both distance fields on the device"""
        self._check(self.lib.isdf_map_esdf(self.h))

    def get_esdf(self, field="positive"):
        """one field ("positive", "negative" or "signed") as an (X, Y, Z) float64 array"""
        f = self._esdf_field(field)
        X, Y, Z = self.map_info()["dims"]
        out = np.empty((X, Y, Z), dtype=np.float64)
        self._check(self.lib.isdf_get_esdf_f64(self.h, f, _dp(out), out.size))
        return out

    def esdf_query(self, points, field="positive", grad=True):
        """getSDFValueWithGrad (grad=True: returns (dist (n,), grad (n, 3))) or getSDFValue (grad=False: returns dist) at (n, 3) points"""
        f = self._esdf_field(field)
        p = _f64(points).reshape(-1, 3)
        n = p.shape[0]
        dist = np.empty(n)
        g = np.empty((n, 3)) if grad else None
        self._check(self.lib.isdf_esdf_query(self.h, f, _dp(p), n, _dp(dist), _dp(g)))
        return (dist, g) if grad else dist

    def esdf_query_device(self, points, field="positive", grad=True, stream=0):
        """the same on a contiguous float64 (n, 3) torch tensor on the context's device; returns tensors on that device, enqueued on
        stream (a raw cudaStream_t; 0 = the legacy default stream) and not waited for"""
        import torch
        f = self._esdf_field(field)
        if points.dtype != torch.float64 or points.dim() != 2 or points.shape[1] != 3:
            raise TypeError(f"points must be a float64 (n, 3) tensor, got {points.dtype} {tuple(points.shape)}")
        if not points.is_contiguous():
            raise ValueError("points must be contiguous")
        n = points.shape[0]
        dist = torch.empty(n, dtype=torch.float64, device=points.device)
        g = torch.empty((n, 3), dtype=torch.float64, device=points.device) if grad else None
        if n == 0:   # an empty tensor has no storage to point at
            return (dist, g) if grad else dist
        self._check(self.lib.isdf_esdf_query_device(self.h, f, C.c_void_p(points.data_ptr()), n, C.c_void_p(dist.data_ptr()),
                                                    C.c_void_p(g.data_ptr()) if grad else None, C.c_void_p(stream)))
        return (dist, g) if grad else dist

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

    def gather_obstacle_points_batch(self, waypoints, half, offset=(0.0, 0.0, 0.0), set_as_points=False, cap=None, known_rows=None):
        """isdf_gather_obstacle_points_batch: one obstacle list per plan (waypoints: list of (n_b, 3) arrays, n_b may be 0) -> list of (P_b, 3)
        arrays. cap = None: a first guess, repeated once with the reported total when the lists are longer. known_rows (B ints, or None):
        isdf_gather_obstacle_points_batch_known, plan b's first known_rows[b] rows reading the blocked grid (occupied or not known)."""
        B = len(waypoints)
        wo = np.zeros(B + 1, dtype=np.int32)
        for b, w in enumerate(waypoints):
            wo[b + 1] = wo[b] + len(w)
        wp = _f64(np.concatenate([np.asarray(w, dtype=np.float64).reshape(-1, 3) for w in waypoints])) if B and wo[B] else np.zeros((1, 3))
        off = _f64(offset).reshape(3)
        ip = C.POINTER(C.c_int32)
        cap = int(cap) if cap is not None else max(1024, 64 * int(wo[B]))
        for attempt in range(2):
            out, pt = np.zeros((max(cap, 1), 3)), np.zeros(B + 1, dtype=np.int32)
            if known_rows is None:
                r = self.lib.isdf_gather_obstacle_points_batch(self.h, B, wo.ctypes.data_as(ip), _dp(wp), float(half), _dp(off), cap, _dp(out),
                                                               pt.ctypes.data_as(ip), int(set_as_points))
            else:
                kr = np.ascontiguousarray(known_rows, dtype=np.int32).reshape(B)
                r = self.lib.isdf_gather_obstacle_points_batch_known(self.h, B, wo.ctypes.data_as(ip), _dp(wp), float(half), _dp(off),
                                                                     kr.ctypes.data_as(ip), cap, _dp(out), pt.ctypes.data_as(ip), int(set_as_points))
            if r == -1 and attempt == 0 and pt[B] > cap:
                cap = int(pt[B])
                continue
            self._check(r)
            break
        if set_as_points and pt[B]:
            self.n_points = int(pt[B])
        return [out[pt[b]:pt[b + 1]].copy() for b in range(B)]

    def callback_batch(self, head, tail, rho, X):
        """B decision vectors [tau (N0) | xi (3(N0-1))] -> (cost[B], grad[B, 4*N0-3]); head/tail 3x3 (columns p, v, a), shared (3,3)
        or per problem (B,3,3); passed to the library column-major."""
        X = _f64(X)
        B, dim = X.shape
        N0 = (dim + 3) // 4
        assert 4 * N0 - 3 == dim
        per, h, t = self._bc(head, tail)
        cost, grad = np.zeros(B), np.zeros((B, dim))
        Xf = np.ascontiguousarray(X).reshape(-1)
        self._check(self.lib.isdf_callback_batch(self.h, B, N0, _dp(h), _dp(t), per, float(rho), _dp(Xf), _dp(cost), _dp(grad.reshape(-1))))
        return cost, grad

    def callback_batch_device(self, B, N0, d_head, d_tail, per_problem_bc, rho, d_x, d_cost, d_grad, stream=None):
        self._check(self.lib.isdf_callback_batch_device(self.h, B, N0, d_head, d_tail, int(per_problem_bc), float(rho), d_x, d_cost, d_grad, stream))

    @staticmethod
    def _bc(head, tail):
        head, tail = np.asarray(head, dtype=np.float64), np.asarray(tail, dtype=np.float64)
        return int(head.ndim == 3), _colmajor(head), _colmajor(tail)

    def callback_batch_ragged(self, head, tail, rho, xs):
        """isdf_callback_batch_ragged: xs = list of B decision vectors [tau (N_b) | xi (3(N_b-1))] -> (cost[B], list of B gradients); head / tail
        as callback_batch"""
        L = Ragged([(np.size(x) + 3) // 4 for x in xs])
        per, h, t = self._bc(head, tail)
        x = L.pack_x(xs)
        cost, grad = np.zeros(L.B), np.zeros(x.size)
        self._check(self.lib.isdf_callback_batch_ragged(self.h, L.B, L.ptr(), _dp(h), _dp(t), per, float(rho), _dp(x), _dp(cost), _dp(grad)))
        return cost, L.unpack_x(grad)

    def callback_batch_ragged_device(self, piece_off, d_head, d_tail, per_problem_bc, rho, d_x, d_cost, d_grad, stream=None):
        off = np.ascontiguousarray(piece_off, dtype=np.int32)
        self._check(self.lib.isdf_callback_batch_ragged_device(self.h, off.size - 1, off.ctypes.data_as(C.POINTER(C.c_int32)), d_head, d_tail,
                                                               int(per_problem_bc), float(rho), d_x, d_cost, d_grad, stream))

    def batch_trajectories_ragged(self, pieces):
        """isdf_get_batch_trajectories after a ragged call: (list of B durations, list of B per-problem coefficient blocks, energies)"""
        L = Ragged(pieces)
        T, Cc, en = np.zeros(L.P), np.zeros(18 * L.P), np.zeros(L.B)
        self._check(self.lib.isdf_get_batch_trajectories(self.h, _dp(T), _dp(Cc), _dp(en)))
        return L.unpack_T(T), L.unpack_coeffs(Cc), en

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
        per, h, t = self._bc(head, tail)
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

    def lbfgs_batch_ragged(self, head, tail, rho, xs, params=None):
        """isdf_lbfgs_batch_ragged: xs = list of B starting points of 4 N_b - 3 values -> dict(x (list of B), f, ret, iterations, evaluations,
        rounds)"""
        L = Ragged([(np.size(x) + 3) // 4 for x in xs])
        per, h, t = self._bc(head, tail)
        x = L.pack_x(xs).copy()
        f = np.zeros(L.B)
        ret, it, evs = (np.zeros(L.B, dtype=np.int32) for _ in range(3))
        rounds = C.c_int32(0)
        ip = C.POINTER(C.c_int32)
        p = params if params is not None else self.lbfgs_params()
        self._check(self.lib.isdf_lbfgs_batch_ragged(self.h, L.B, L.ptr(), _dp(h), _dp(t), per, float(rho), C.byref(p), _dp(x), _dp(f),
                                                     ret.ctypes.data_as(ip), it.ctypes.data_as(ip), evs.ctypes.data_as(ip), C.byref(rounds)))
        return dict(x=L.unpack_x(x), f=f, ret=ret, iterations=it, evaluations=evs, rounds=rounds.value)

    def lbfgs_batch_ragged_device(self, piece_off, d_head, d_tail, per_problem_bc, rho, d_x, d_f, d_ret=None, d_iterations=None, d_evaluations=None,
                                  params=None, stream=None):
        """isdf_lbfgs_batch_ragged_device on raw device pointers; piece_off on the host; returns the rounds"""
        off = np.ascontiguousarray(piece_off, dtype=np.int32)
        p = params if params is not None else self.lbfgs_params()
        rounds = C.c_int32(0)
        self._check(self.lib.isdf_lbfgs_batch_ragged_device(self.h, off.size - 1, off.ctypes.data_as(C.POINTER(C.c_int32)), d_head, d_tail,
                                                            int(per_problem_bc), float(rho), C.byref(p), d_x, d_f, d_ret, d_iterations, d_evaluations,
                                                            C.byref(rounds), stream))
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
        wp = _f64(waypoints).reshape(-1)
        assert wp.size == 3 * B * (N0 - 1)
        return (*Evaluator._bc(head, tail), wp if wp.size else np.zeros(1))

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

    def midend_callback_batch_ragged(self, head, tail, waypoints, xs, params=None):
        """isdf_midend_callback_batch_ragged: waypoints = list of B (N_b - 1, 3) arrays, xs = list of B decision vectors -> (cost[B], list of B
        gradients)"""
        L = Ragged([len(np.asarray(w).reshape(-1, 3)) + 1 for w in waypoints])
        per, h, t = self._bc(head, tail)
        wp, x = L.pack_waypoints(waypoints), L.pack_x(xs)
        p = params if params is not None else self.midend_params()
        cost, grad = np.zeros(L.B), np.zeros(x.size)
        self._check(self.lib.isdf_midend_callback_batch_ragged(self.h, L.B, L.ptr(), _dp(h), _dp(t), per, C.byref(p), _dp(wp if wp.size else np.zeros(1)),
                                                               _dp(x), _dp(cost), _dp(grad)))
        return cost, L.unpack_x(grad)

    def midend_batch_ragged(self, head, tail, waypoints, params=None):
        """isdf_midend_batch_ragged: waypoints = list of B (N_b - 1, 3) arrays (N_b from their lengths) -> dict(x, T, coeffs (lists of B; coeffs
        per problem as its own 6N_b x 3 column-major block), f, ret, iterations, evaluations, rounds)"""
        L = Ragged([len(np.asarray(w).reshape(-1, 3)) + 1 for w in waypoints])
        per, h, t = self._bc(head, tail)
        wp = L.pack_waypoints(waypoints)
        p = params if params is not None else self.midend_params()
        x, T, Cc, f = np.zeros(4 * L.P - 3 * L.B), np.zeros(L.P), np.zeros(18 * L.P), np.zeros(L.B)
        ret, it, evs = (np.zeros(L.B, dtype=np.int32) for _ in range(3))
        rounds = C.c_int32(0)
        ip = C.POINTER(C.c_int32)
        self._check(self.lib.isdf_midend_batch_ragged(self.h, L.B, L.ptr(), _dp(h), _dp(t), per, C.byref(p), _dp(wp if wp.size else np.zeros(1)), _dp(x),
                                                      _dp(T), _dp(Cc), _dp(f), ret.ctypes.data_as(ip), it.ctypes.data_as(ip), evs.ctypes.data_as(ip),
                                                      C.byref(rounds)))
        return dict(x=L.unpack_x(x), T=L.unpack_T(T), coeffs=L.unpack_coeffs(Cc), f=f, ret=ret, iterations=it, evaluations=evs, rounds=rounds.value)

    def midend_batch_ragged_device(self, piece_off, d_head, d_tail, per_problem_bc, d_waypoints, d_x, d_T, d_coeffs, d_f, d_ret, d_iterations,
                                   d_evaluations, params=None, stream=None):
        """isdf_midend_batch_ragged_device on raw device pointers; piece_off on the host; returns the rounds"""
        off = np.ascontiguousarray(piece_off, dtype=np.int32)
        p = params if params is not None else self.midend_params()
        rounds = C.c_int32(0)
        self._check(self.lib.isdf_midend_batch_ragged_device(self.h, off.size - 1, off.ctypes.data_as(C.POINTER(C.c_int32)), d_head, d_tail,
                                                             int(per_problem_bc), C.byref(p), d_waypoints, d_x, d_T, d_coeffs, d_f, d_ret, d_iterations,
                                                             d_evaluations, C.byref(rounds), stream))
        return rounds.value

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

    # ---- planning step: generateTraj for one start and B goals (see include/isdf.h) ----
    def plan_params(self, **kw):
        """isdf_plan_default_params for this context, then overrides: parlength, half_extent, offset, rho, flags, reserved_, certify,
        dynamics, frontpath, midend (an isdf_midend_params) and backend (an isdf_lbfgs_params) by name; midend_<field> / backend_<field> set
        one field of the nested blocks (midend_init_time=200.0, backend_max_iterations=50, midend_max_rounds=1, ...); unknown_weight sets
        frontpath.unknown_weight (the front end's surcharge on unknown voxels; pair it with flags including PLAN_KNOWN_PREFIX to keep the
        back end inside the known prefix, DESIGN §3.23)"""
        p = PlanParams()
        self._check(self.lib.isdf_plan_default_params(self.h, C.byref(p)))
        lb = {n for n, _ in LbfgsParams._fields_}
        for k, v in kw.items():
            if k == "offset":
                p.offset[:] = [float(x) for x in v]
            elif k.startswith("midend_"):
                f = k[len("midend_"):]
                setattr(p.midend.lbfgs if f in lb and f != "reserved_" else p.midend, f, v)
            elif k.startswith("backend_"):
                setattr(p.backend, k[len("backend_"):], v)
            elif k == "unknown_weight":
                p.frontpath.unknown_weight = float(v)
            elif k in {n for n, _ in PlanParams._fields_}:
                setattr(p, k, v)
            else:
                raise TypeError(f"unknown isdf_plan_params field {k}")
        return p

    def plan_batch(self, start, goals, params=None, **kw):
        """isdf_plan_batch: one start, B goals -> (list of B dicts, info dict). Each dict: the isdf_plan_result fields, path (n, 3), T (N,),
        coeffs (18 N, the plan's own 6N x 3 column-major block; empty without a trajectory), certify / dynamics summary dicts (None when the
        flag is off). params: an isdf_plan_params, or None for plan_params(**kw). The caps are sized from the goals and the call repeated once
        with the reported sizes when they are too small."""
        st, gl = _f64(start).reshape(3), _f64(goals).reshape(-1, 3)
        return self._plan(lambda *args: self.lib.isdf_plan_batch(self.h, _dp(st), gl.shape[0], _dp(gl), *args), gl.shape[0], params, kw)

    def plan_pairs(self, starts, goals, params=None, max_fields=0, **kw):
        """isdf_plan_pairs: B (start, goal) pairs, start b with goal b -> what plan_batch returns, in pair order. max_fields: the fields
        of distinct start voxels held at once (0: the library's 4 GiB budget)"""
        sts, gl = _f64(starts).reshape(-1, 3), _f64(goals).reshape(-1, 3)
        if sts.shape != gl.shape:
            raise ValueError(f"starts and goals must both be (B, 3), got {sts.shape} and {gl.shape}")
        B = gl.shape[0]
        return self._plan(lambda p, *args: self.lib.isdf_plan_pairs(self.h, B, _dp(sts), _dp(gl), p, int(max_fields), *args), B, params, kw)

    def plan_states(self, starts, goals, params=None, max_fields=0, **kw):
        """isdf_plan_states: B (start state, goal) pairs, starts (B, 9) as p, v, a -> what plan_pairs returns"""
        sts, gl = _f64(starts).reshape(-1, 9), _f64(goals).reshape(-1, 3)
        if sts.shape[0] != gl.shape[0]:
            raise ValueError(f"starts must be (B, 9) and goals (B, 3), got {sts.shape} and {gl.shape}")
        B = gl.shape[0]
        return self._plan(lambda p, *args: self.lib.isdf_plan_states(self.h, B, _dp(sts), _dp(gl), p, int(max_fields), *args), B, params, kw)

    def _plan(self, call, B, params, kw):
        """call(params, cap_nodes, path_off, path_xyz, cap_pieces, piece_off, T, coeffs, results, certify, dynamics): the C call"""
        p = params if params is not None else self.plan_params(**kw)
        ip = C.POINTER(C.c_int32)
        cap_nodes, cap_pieces = self._path_cap(None) * B, 290 * B
        for attempt in range(2):
            xyz, po, T, Cc = np.zeros((max(cap_nodes, 1), 3)), np.zeros(B + 1, dtype=np.int32), np.zeros(max(cap_pieces, 1)), np.zeros(18 * max(cap_pieces, 1))
            pf = np.zeros(B + 1, dtype=np.int32)
            res, cs, ds = (PlanResult * B)(), (CertifySummary * B)(), (DynamicsSummary * B)()
            r = call(C.byref(p), cap_nodes, pf.ctypes.data_as(ip), _dp(xyz), cap_pieces, po.ctypes.data_as(ip), _dp(T), _dp(Cc), res, cs, ds)
            if r == -1 and attempt == 0 and (pf[B] > cap_nodes or po[B] > cap_pieces):
                cap_nodes, cap_pieces = max(cap_nodes, int(pf[B])), max(cap_pieces, int(po[B]))
                continue
            self._check(r)
            break
        out = []
        for b in range(B):
            d = res[b].as_dict()
            d["path"] = xyz[pf[b]:pf[b + 1]].copy()
            d["T"] = T[po[b]:po[b + 1]].copy()
            d["coeffs"] = Cc[18 * po[b]:18 * po[b + 1]].copy()
            d["certify"] = cs[b].as_dict() if p.flags & PLAN_CERTIFY else None
            d["dynamics"] = ds[b].as_dict() if p.flags & PLAN_DYNAMICS else None
            out.append(d)
        return out, self.plan_info()

    # ---- planning in device memory (include/isdf.h: isdf_plan_pairs_device, isdf_plan_batch_device) ----
    def plan_pairs_device(self, starts, goals, params=None, max_fields=0, cap_nodes=None, cap_pieces=None, stream=None, **kw):
        """isdf_plan_pairs_device: starts and goals are (B, 3) float64 CUDA tensors on this context's device -> a dict of CUDA tensors
        (see _plan_device). Runs on stream (a torch.cuda.Stream; None: torch's current stream) and returns when the outputs are written."""
        if starts.shape != goals.shape or starts.dim() != 2 or starts.shape[1] != 3:
            raise ValueError(f"starts and goals must both be (B, 3), got {tuple(starts.shape)} and {tuple(goals.shape)}")
        sts, gl = _cuda_f64(starts), _cuda_f64(goals)
        return self._plan_device(lambda p, *a: self.lib.isdf_plan_pairs_device(self.h, gl.shape[0], C.c_void_p(sts.data_ptr()), C.c_void_p(gl.data_ptr()),
                                                                                p, int(max_fields), *a),
                                 gl, params, cap_nodes, cap_pieces, stream, kw)

    def plan_states_device(self, starts, goals, params=None, max_fields=0, cap_nodes=None, cap_pieces=None, stream=None, **kw):
        """isdf_plan_states_device: starts (B, 9) start states p, v, a and goals (B, 3), float64 CUDA tensors -> what plan_pairs_device
        returns"""
        if starts.dim() != 2 or starts.shape[1] != 9 or goals.dim() != 2 or goals.shape[1] != 3 or starts.shape[0] != goals.shape[0]:
            raise ValueError(f"starts must be (B, 9) and goals (B, 3), got {tuple(starts.shape)} and {tuple(goals.shape)}")
        sts, gl = _cuda_f64(starts), _cuda_f64(goals)
        return self._plan_device(lambda p, *a: self.lib.isdf_plan_states_device(self.h, gl.shape[0], C.c_void_p(sts.data_ptr()), C.c_void_p(gl.data_ptr()),
                                                                                 p, int(max_fields), *a),
                                 gl, params, cap_nodes, cap_pieces, stream, kw)

    def plan_batch_device(self, start, goals, params=None, cap_nodes=None, cap_pieces=None, stream=None, **kw):
        """isdf_plan_batch_device: start (3 values, host), goals a (B, 3) float64 CUDA tensor -> what plan_pairs_device returns"""
        st = _f64(start).reshape(3)
        if goals.dim() != 2 or goals.shape[1] != 3:
            raise ValueError(f"goals must be (B, 3), got {tuple(goals.shape)}")
        gl = _cuda_f64(goals)
        return self._plan_device(lambda p, *a: self.lib.isdf_plan_batch_device(self.h, _dp(st), gl.shape[0], C.c_void_p(gl.data_ptr()), p, *a),
                                 gl, params, cap_nodes, cap_pieces, stream, kw)

    def _plan_device(self, call, gl, params, cap_nodes, cap_pieces, stream, kw):
        """call(params, cap_nodes, path_off, path_xyz, cap_pieces, piece_off, T, coeffs, results, certify, dynamics, stream) -> dict of
        CUDA tensors: path_off (B + 1 int32), path_xyz (path_off[B] x 3), piece_off (B + 1 int32), T (piece_off[B]), coeffs
        (18 piece_off[B]), results (B x 64 uint8 isdf_plan_result records; decode_plan_results), certify / dynamics (B summary records as
        uint8 rows, None when the flag is off). piece_off, T and coeffs go into trajectory_states_device as they are. Caps as in _plan: too
        small, the call is repeated once with the sizes the first call reported."""
        import torch
        p = params if params is not None else self.plan_params(**kw)
        B, dev = gl.shape[0], gl.device
        cap_nodes = self._path_cap(None) * B if cap_nodes is None else int(cap_nodes)
        cap_pieces = 290 * B if cap_pieces is None else int(cap_pieces)
        s = torch.cuda.current_stream(dev) if stream is None else stream
        ptr = lambda t: C.c_void_p(t.data_ptr())
        for attempt in range(2):
            with torch.cuda.stream(s):   # the outputs are allocated and filled on the stream the call runs on
                po, xyz = torch.zeros(B + 1, dtype=torch.int32, device=dev), torch.empty((max(cap_nodes, 1), 3), dtype=torch.float64, device=dev)
                pf = torch.zeros(B + 1, dtype=torch.int32, device=dev)
                T, Cc = torch.empty(max(cap_pieces, 1), dtype=torch.float64, device=dev), torch.empty(18 * max(cap_pieces, 1), dtype=torch.float64, device=dev)
                res = torch.empty((B, C.sizeof(PlanResult)), dtype=torch.uint8, device=dev)
                cs = torch.empty((B, C.sizeof(CertifySummary)), dtype=torch.uint8, device=dev)
                ds = torch.empty((B, C.sizeof(DynamicsSummary)), dtype=torch.uint8, device=dev)
                r = call(C.byref(p), cap_nodes, ptr(pf), ptr(xyz), cap_pieces, ptr(po), ptr(T), ptr(Cc), ptr(res), ptr(cs), ptr(ds), C.c_void_p(s.cuda_stream))
            if r == -1 and attempt == 0:
                need_nodes, need_pieces = int(pf[B]), int(po[B])
                if need_nodes > cap_nodes or need_pieces > cap_pieces:
                    cap_nodes, cap_pieces = max(cap_nodes, need_nodes), max(cap_pieces, need_pieces)
                    continue
            self._check(r)
            break
        nodes, pieces = int(pf[B]), int(po[B])
        return dict(path_off=pf, path_xyz=xyz[:nodes], piece_off=po, T=T[:pieces], coeffs=Cc[:18 * pieces], results=res,
                    certify=cs if p.flags & PLAN_CERTIFY else None, dynamics=ds if p.flags & PLAN_DYNAMICS else None)

    def plan_pairs_device_raw(self, B, d_starts, d_goals, params, max_fields, cap_nodes, d_path_off, d_path_xyz, cap_pieces, d_piece_off, d_T,
                              d_coeffs, d_results, d_certify, d_dynamics, stream=0):
        """isdf_plan_pairs_device on raw device pointers (0 for NULL) -> its return code (not raised). stream: a raw cudaStream_t"""
        v = C.c_void_p
        return self.lib.isdf_plan_pairs_device(self.h, int(B), v(d_starts), v(d_goals), C.byref(params), int(max_fields), int(cap_nodes), v(d_path_off),
                                               v(d_path_xyz), int(cap_pieces), v(d_piece_off), v(d_T), v(d_coeffs), v(d_results), v(d_certify),
                                               v(d_dynamics), v(stream))

    def plan_batch_device_raw(self, start, B, d_goals, params, cap_nodes, d_path_off, d_path_xyz, cap_pieces, d_piece_off, d_T, d_coeffs,
                              d_results, d_certify, d_dynamics, stream=0):
        """isdf_plan_batch_device on raw device pointers (0 for NULL) -> its return code (not raised); start: 3 host values"""
        v, st = C.c_void_p, _f64(start).reshape(3)
        return self.lib.isdf_plan_batch_device(self.h, _dp(st), int(B), v(d_goals), C.byref(params), int(cap_nodes), v(d_path_off), v(d_path_xyz),
                                               int(cap_pieces), v(d_piece_off), v(d_T), v(d_coeffs), v(d_results), v(d_certify), v(d_dynamics),
                                               v(stream))

    def path_waypoints_device(self, B, d_path_off, d_path_xyz, res, parlength, cap, d_waypoints, d_wp_off, d_pieces, stream=0):
        """isdf_path_waypoints_device on raw device pointers -> its return code (not raised: cap too small is ISDF_ERR_INVALID with wp_off
        and pieces written). stream: a raw cudaStream_t"""
        v = C.c_void_p
        return self.lib.isdf_path_waypoints_device(self.h, int(B), v(d_path_off), v(d_path_xyz), float(res), float(parlength), int(cap), v(d_waypoints),
                                                   v(d_wp_off), v(d_pieces), v(stream))

    def dbg_plan_transfers(self):
        """what the last planning call moved (isdf_dbg_plan_transfers, not part of include/isdf.h)"""
        out = (C.c_int64 * 4)()
        self.lib.isdf_dbg_plan_transfers.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        self._check(self.lib.isdf_dbg_plan_transfers(self.h, out))
        return dict(d2h_bytes=out[0], round_reads=out[1], h2d_bytes=out[2], copies=out[3])

    # ---- executing a trajectory (include/isdf.h: isdf_trajectory_states, isdf_pose_points) ----
    @staticmethod
    def pack_plans(plans):
        """isdf_plan_batch's ragged layout from plan_batch's list of dicts: (piece_off (B + 1 int32), T (P,), coeffs (18 P,)), each plan's
        own 6N x 3 column-major block at coeffs[18 piece_off[b]:]; plans without a trajectory get no pieces"""
        Ts = [_f64(d["T"]).reshape(-1) for d in plans]
        Cs = [_f64(d["coeffs"]).reshape(-1) for d in plans]
        if not Ts or any(c.size != 18 * t.size for t, c in zip(Ts, Cs)):
            raise ValueError("plans must be a non-empty list of dicts whose coeffs hold 18 values per duration in T")
        off = np.zeros(len(Ts) + 1, dtype=np.int32)
        off[1:] = np.cumsum([t.size for t in Ts])
        return off, _f64(np.concatenate(Ts)), _f64(np.concatenate(Cs))

    def trajectory_states(self, plans_or_ragged, traj, times):
        """the state of trajectory traj[q] at its local time times[q] -> (Q, 20) records: pos, vel, acc, jer, quat (w, x, y, z), omg, thr.
        plans_or_ragged: plan_batch's list of dicts, or (piece_off, T, coeffs) in isdf_plan_batch's ragged layout"""
        off, T, Cc = _host_ragged(plans_or_ragged)
        tr = np.ascontiguousarray(traj, dtype=np.int32).reshape(-1)
        tm = _f64(times).reshape(-1)
        if tr.size != tm.size:
            raise ValueError(f"traj and times must have the same length, got {tr.size} and {tm.size}")
        out = np.empty((tm.size, STATE_DOUBLES))
        ip = C.POINTER(C.c_int32)
        self._check(self.lib.isdf_trajectory_states(self.h, off.size - 1, off.ctypes.data_as(ip), _dp(T), _dp(Cc), tm.size,
                                                    tr.ctypes.data_as(ip), _dp(tm), _dp(out)))
        return out

    def trajectory_states_device(self, B, d_piece_off, d_T, d_coeffs, Q, d_traj, d_times, d_out, stream=0):
        """raw device pointers (e.g. torch .data_ptr()): piece_off B + 1 and traj Q int32, T, coeffs and times float64, out Q x 20 float64;
        enqueued on stream (a raw cudaStream_t; 0 = the legacy default stream) and not waited for"""
        self._check(self.lib.isdf_trajectory_states_device(self.h, int(B), C.c_void_p(d_piece_off), C.c_void_p(d_T), C.c_void_p(d_coeffs), int(Q),
                                                           C.c_void_p(d_traj), C.c_void_p(d_times), C.c_void_p(d_out), C.c_void_p(stream)))

    def trajectory_shift(self, plans_or_ragged, t0):
        """isdf_trajectory_shift: the rest of each trajectory from its t0[b], re-timed to start at 0 -> (piece_off (B + 1 int32), T, coeffs)
        in the ragged layout, trimmed to piece_off[B] pieces. plans_or_ragged as in trajectory_states."""
        off, T, Cc = _host_ragged(plans_or_ragged)
        B = off.size - 1
        t = _f64(t0).reshape(-1)
        if t.size != B:
            raise ValueError(f"t0 needs one time per trajectory ({B}), got {t.size}")
        P = max(int(off[-1]), 1)
        oo, oT, oC = np.zeros(B + 1, dtype=np.int32), np.zeros(P), np.zeros(18 * P)
        ip = C.POINTER(C.c_int32)
        self._check(self.lib.isdf_trajectory_shift(self.h, B, off.ctypes.data_as(ip), _dp(T), _dp(Cc), _dp(t), oo.ctypes.data_as(ip), _dp(oT), _dp(oC)))
        return oo, oT[:oo[B]].copy(), oC[:18 * oo[B]].copy()

    def trajectory_shift_device(self, piece_off, T, coeffs, t0, stream=None):
        """isdf_trajectory_shift_device on CUDA tensors (piece_off B + 1 int32, T, coeffs, t0 (B,) float64) -> dict(piece_off, T, coeffs)
        of CUDA tensors; T and coeffs have room for the input's pieces and hold piece_off[B] of them (not read here: nothing is waited
        for). Runs on stream (None: torch's current stream)."""
        import torch
        if piece_off.dtype != torch.int32 or piece_off.dim() != 1 or piece_off.numel() < 2:
            raise ValueError("piece_off must be a (B + 1) int32 CUDA tensor, B >= 1")
        B, dev = piece_off.numel() - 1, piece_off.device
        T, coeffs, t = _cuda_f64(T), _cuda_f64(coeffs), _cuda_f64(t0).reshape(-1)
        if T.numel() == 0:   # no piece at all: the call still needs non-NULL arrays
            T, coeffs = torch.zeros(1, dtype=torch.float64, device=dev), torch.zeros(18, dtype=torch.float64, device=dev)
        if t.numel() != B:
            raise ValueError(f"t0 needs one time per trajectory ({B}), got {t.numel()}")
        po = piece_off.contiguous()
        s = torch.cuda.current_stream(dev) if stream is None else stream
        with torch.cuda.stream(s):
            oo = torch.empty(B + 1, dtype=torch.int32, device=dev)
            oT, oC = torch.empty(max(T.numel(), 1), dtype=torch.float64, device=dev), torch.empty(max(coeffs.numel(), 18), dtype=torch.float64, device=dev)
        v = lambda x: C.c_void_p(x.data_ptr())
        self._check(self.lib.isdf_trajectory_shift_device(self.h, B, v(po), v(T), v(coeffs), v(t), v(oo), v(oT), v(oC), C.c_void_p(s.cuda_stream)))
        return dict(piece_off=oo, T=oT, coeffs=oC)

    def brake_params(self, **kw):
        """isdf_brake_default_params for this context, then overrides by name: candidates, pieces, certify (an isdf_certify_params),
        dynamics (an isdf_dynamics_params)"""
        p = BrakeParams()
        self._check(self.lib.isdf_brake_default_params(self.h, C.byref(p)))
        for k, v in kw.items():
            if k not in {n for n, _ in BrakeParams._fields_} or k == "reserved_":
                raise TypeError(f"unknown isdf_brake_params field {k}")
            setattr(p, k, v)
        return p

    def trajectory_brake(self, plans_or_ragged, t_stop_max, params=None):
        """isdf_trajectory_brake: a certified stop along each remaining trajectory, reaching no further than its time t_stop_max[b] ->
        (piece_off (B + 1 int32), T, coeffs) of the stops in the ragged layout (trimmed to piece_off[B] pieces), list of B summary dicts.
        plans_or_ragged as in trajectory_states."""
        off, T, Cc = _host_ragged(plans_or_ragged)
        p = params if params is not None else self.brake_params()
        B = off.size - 1
        ts = _f64(t_stop_max).reshape(-1)
        if ts.size != B:
            raise ValueError(f"t_stop_max needs one time per trajectory ({B}), got {ts.size}")
        if T.size == 0:   # no piece at all: the call still needs non-NULL arrays
            T, Cc = np.zeros(1), np.zeros(18)
        cap = max(B * int(p.pieces), 1)
        oo, oT, oC = np.zeros(B + 1, dtype=np.int32), np.zeros(cap), np.zeros(18 * cap)
        summ = (BrakeSummary * max(B, 1))()
        ip = C.POINTER(C.c_int32)
        self._check(self.lib.isdf_trajectory_brake(self.h, B, off.ctypes.data_as(ip), _dp(T), _dp(Cc), _dp(ts), C.byref(p), oo.ctypes.data_as(ip),
                                                   _dp(oT), _dp(oC), summ))
        return (oo, oT[:oo[B]].copy(), oC[:18 * oo[B]].copy()), [summ[b].as_dict() for b in range(B)]

    def trajectory_brake_device(self, piece_off, T, coeffs, t_stop_max, params=None, stream=None):
        """isdf_trajectory_brake_device on CUDA tensors (piece_off B + 1 int32, T, coeffs, t_stop_max (B,) float64) -> dict(piece_off, T,
        coeffs, summary): CUDA tensors, T and coeffs with room for B * pieces pieces and holding piece_off[B] of them, summary (B, 256) uint8
        (decode with decode_brake_summaries). Runs on stream (None: torch's current stream) and returns when the outputs are written."""
        import torch
        if piece_off.dtype != torch.int32 or piece_off.dim() != 1 or piece_off.numel() < 2:
            raise ValueError("piece_off must be a (B + 1) int32 CUDA tensor, B >= 1")
        p = params if params is not None else self.brake_params()
        B, dev = piece_off.numel() - 1, piece_off.device
        T, coeffs, ts = _cuda_f64(T), _cuda_f64(coeffs), _cuda_f64(t_stop_max).reshape(-1)
        if T.numel() == 0:
            T, coeffs = torch.zeros(1, dtype=torch.float64, device=dev), torch.zeros(18, dtype=torch.float64, device=dev)
        if ts.numel() != B:
            raise ValueError(f"t_stop_max needs one time per trajectory ({B}), got {ts.numel()}")
        po = piece_off.contiguous()
        s = torch.cuda.current_stream(dev) if stream is None else stream
        cap = max(B * int(p.pieces), 1)
        with torch.cuda.stream(s):
            oo = torch.empty(B + 1, dtype=torch.int32, device=dev)
            oT, oC = torch.empty(cap, dtype=torch.float64, device=dev), torch.empty(18 * cap, dtype=torch.float64, device=dev)
            sm = torch.empty((B, C.sizeof(BrakeSummary)), dtype=torch.uint8, device=dev)
        v = lambda x: C.c_void_p(x.data_ptr())
        self._check(self.lib.isdf_trajectory_brake_device(self.h, B, v(po), v(T), v(coeffs), v(ts), C.byref(p), v(oo), v(oT), v(oC), v(sm),
                                                          C.c_void_p(s.cuda_stream)))
        return dict(piece_off=oo, T=oT, coeffs=oC, summary=sm)

    def pose_points(self, states, body):
        """the body-frame points body (P, 3) posed at each of the (Q, 20) states -> (Q, P, 3): R(quat) b + pos (Shape::Transform)"""
        st = _f64(states).reshape(-1, STATE_DOUBLES)
        b = _f64(body).reshape(-1, 3)
        out = np.empty((st.shape[0], b.shape[0], 3))
        self._check(self.lib.isdf_pose_points(self.h, st.shape[0], _dp(st), b.shape[0], _dp(b), _dp(out)))
        return out

    def pose_points_device(self, Q, d_states, P, d_body, d_out, stream=0):
        """raw device pointers: states Q x 20, body P x 3, out Q x P x 3 float64; enqueued on stream and not waited for"""
        self._check(self.lib.isdf_pose_points_device(self.h, int(Q), C.c_void_p(d_states), int(P), C.c_void_p(d_body), C.c_void_p(d_out),
                                                     C.c_void_p(stream)))

    # ---- closed loop (include/isdf.h: isdf_simulate, isdf_simulate_device) ----
    @staticmethod
    def sim_params(**kw):
        return sim_default_params(**kw)

    def simulate(self, plans_or_ragged, traj, init, dist=None, params=None, cap_log=None):
        """fly rollouts r = 0..R-1 along trajectory traj[r] from init (R, 17) under the constant force / moment dist (R, 6) ->
        (log (R, n_log, 21), list of R summary dicts)"""
        off, T, Cc = _host_ragged(plans_or_ragged)
        p = params if params is not None else sim_default_params()
        tr = np.ascontiguousarray(traj, dtype=np.int32).reshape(-1)
        ini = _f64(init).reshape(-1, SIM_INIT_DOUBLES)
        ds = None if dist is None else _f64(dist).reshape(-1, 6)
        if ini.shape[0] != tr.size or (ds is not None and ds.shape[0] != tr.size):
            raise ValueError("traj, init and dist must have one row per rollout")
        n_log = sim_log_records(p)
        cap = n_log if cap_log is None else int(cap_log)
        log = np.empty((tr.size, max(cap, 0), SIM_DOUBLES))
        summ = (SimSummary * max(tr.size, 1))()
        ip = C.POINTER(C.c_int32)
        self._check(self.lib.isdf_simulate(self.h, off.size - 1, off.ctypes.data_as(ip), _dp(T), _dp(Cc), tr.size, tr.ctypes.data_as(ip), _dp(ini),
                                           _dp(ds), C.byref(p), cap, _dp(log), summ))
        return log, [summ[r].as_dict() for r in range(tr.size)]

    def simulate_device(self, piece_off, T, coeffs, traj, init, dist=None, params=None, log=True, stream=None):
        """isdf_simulate_device on CUDA tensors: piece_off (B + 1 int32), T, coeffs (as plan_pairs_device returns them), traj (R int32),
        init (R, 17) and dist (R, 6) float64 -> dict(log (R, n_log, 21) CUDA tensor or None, summary (R, 88) uint8 CUDA tensor; decode with
        decode_sim_summaries). Runs on stream (None: torch's current stream), not waited for."""
        import torch
        p = params if params is not None else sim_default_params()
        for name, t in (("piece_off", piece_off), ("T", T), ("coeffs", coeffs), ("traj", traj), ("init", init), ("dist", dist)):
            if t is not None and not (isinstance(t, torch.Tensor) and t.is_cuda and t.device == init.device):
                raise ValueError(f"{name} must be a CUDA tensor on init's device")
        if piece_off.dtype != torch.int32 or traj.dtype != torch.int32 or piece_off.dim() != 1 or piece_off.numel() < 2:
            raise ValueError("piece_off (B + 1, at least 2) and traj must be int32 CUDA tensors")
        dev = init.device
        tr = traj.contiguous().reshape(-1)
        ini, ds = _cuda_f64(init), (None if dist is None else _cuda_f64(dist))
        R, n_log = tr.numel(), sim_log_records(p)
        if tuple(ini.shape) != (R, SIM_INIT_DOUBLES) or (ds is not None and tuple(ds.shape) != (R, 6)):
            raise ValueError(f"init must be ({R}, {SIM_INIT_DOUBLES}) and dist ({R}, 6), got {tuple(ini.shape)} and "
                             f"{None if ds is None else tuple(ds.shape)}")
        T, coeffs, piece_off = _cuda_f64(T), _cuda_f64(coeffs), piece_off.contiguous()
        s = torch.cuda.current_stream(dev) if stream is None else stream
        with torch.cuda.stream(s):
            lg = torch.empty((R, n_log, SIM_DOUBLES), dtype=torch.float64, device=dev) if log else None
            sm = torch.empty((max(R, 1), C.sizeof(SimSummary)), dtype=torch.uint8, device=dev)
        v = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
        self._check(self.lib.isdf_simulate_device(self.h, piece_off.numel() - 1, v(piece_off), v(T), v(coeffs), R, v(tr), v(ini), v(ds), C.byref(p),
                                                  n_log if log else 0, v(lg), v(sm), C.c_void_p(s.cuda_stream)))
        return dict(log=lg, summary=sm[:R])

    def simulate_device_raw(self, B, d_piece_off, d_T, d_coeffs, R, d_traj, d_init, d_dist, params, cap_log, d_log, d_summary, stream=0):
        """isdf_simulate_device on raw device pointers (0 for NULL) -> its return code (not raised)"""
        v = C.c_void_p
        return self.lib.isdf_simulate_device(self.h, int(B), v(d_piece_off), v(d_T), v(d_coeffs), int(R), v(d_traj), v(d_init), v(d_dist),
                                             C.byref(params), int(cap_log), v(d_log), v(d_summary), v(stream))

    # ---- flying to goals through a world seen only through the depth camera (plan -> fly -> sense -> fuse -> check -> re-plan) ----
    def navigate(self, starts, goals, *, rounds, horizon, sense_every=10, tol=0.5, plan_params=None, sim_params=None, sense_params=None,
                 max_fields=0, stream=None, fallback="keep", brake_params=None, unknown="free", known_boxes=None, explore=False,
                 frontier_params=None, min_gain=None):
        """Drive B vehicles from starts (B, 3) to goals (B, 3) through the scene set by set_sense_cloud*, building their one shared map by
        fusion into the current map's frame (set it first, e.g. set_map_u8 of zeros). Needs the shape, the front-end kernels and
        plan_params with PLAN_CERTIFY (a shape the certificate supports). Each round, for the active vehicles:
          1. sense   poses: every sense_every-th record of the last flown segment and its final record (a vehicle not flown: its current
                     state); sense_cloud_device, then map_fuse_cloud_device;
          2. check   trajectory_certify_device of every remaining trajectory on the fused map (one call per distinct piece count);
          3. replan  vehicles without a CERTIFIED remaining trajectory: plan_states_device from the remaining trajectory's state at 0
                     (trajectory_states_device p, v, a; without one the start at rest) with PLAN_CERTIFY; an OPTIMISED and CERTIFIED plan
                     replaces it, else the remaining trajectory is kept and the replan counts as failed (a head outside the map fails
                     without a call). A vehicle without a trajectory stays at rest and is not flown;
          4. fly     one simulate_device call for t_end = horizon from the vehicles' simulator states;
          5. advance the state becomes the last log record (sim_init_from_log), the trajectory trajectory_shift(horizon); a vehicle whose
                     rest has no piece is ARRIVED within tol of its goal, else STOPPED; a diverged rollout is DIVERGED; vehicles still
                     active after `rounds` are TIMEOUT.
        fallback: what a vehicle whose replan failed flies. "keep": its remaining trajectory, as above. "brake": after step 3, every such
        vehicle with a remaining trajectory gets one batched trajectory_brake_device call (t_stop_max: the check's first_hit when it is
        COLLIDING, else +inf; brake_params defaults to brake_params() with plan_params' certify and dynamics); a BRAKED stop replaces the
        trajectory (action NAV_BRAKED, flown as CERTIFIED), on NONE the remaining trajectory is kept. A vehicle whose stop runs out away
        from its goal is held instead of STOPPED: active, at rest at its simulator position, not flown, sensed at its state and replanned
        every round from (position, 0, 0); a round it stays held is NAV_HELD (its replan still counts as failed). Held vehicles that never
        get a plan end as TIMEOUT.
        sense_params may be one camera or a list of cameras (a rig): every sensed pose is then rendered once per camera.
        unknown: "free" (the default) is the loop above. "occupied" needs fallback="brake" and a finite sensing_horizon on every camera; for
        the call it sets the context's unknown policy to UNKNOWN_OCCUPIED (restored on return), marks known_boxes known (map_mark_known:
        the caller asserts they are free, e.g. the space around the starts), and changes the loop so that no vehicle commits to space it
        has not seen:
          1b. observe  after fusing, map_observe_device of the same poses for every camera;
          2.  check    the certificates now read the blocked grid (occupied or not known);
          3.  replan   also the vehicles flying a commit (and, as before, the held ones); an OPTIMISED plan that is COLLIDING with
                       first_hit > 0 goes to trajectory_brake_device with t_stop_max = first_hit (one call for all such plans, in the brake
                       stage, certified with NAV_COMMIT_SLACK more margin than brake_params', then, for the plans without such a stop, a
                       second call with brake_params' margin); a BRAKED stop replaces the trajectory, flown as CERTIFIED (action NAV_COMMITTED) and marked as a commit;
                       vehicles without an accepted plan or a commit take the fallback as before, except that a vehicle still holding a
                       CERTIFIED remaining trajectory (a commit) keeps it. A commit that runs out away from the goal holds the vehicle.
        The result then also has commits (B,) numpy, and times an "observe" stage. To plan through what has been seen, pass plan_params
        with unknown_weight > 0 and PLAN_KNOWN_PREFIX in flags (plan_params(unknown_weight=W, flags=PLAN_CERTIFY | PLAN_KNOWN_PREFIX)):
        every replan then prefers routes through known voxels and keeps the back end out of unseen space along its known prefix
        (DESIGN §3.23); the loop itself is unchanged.
        explore=True (needs unknown="occupied") plans toward the frontier of what has been seen (DESIGN §3.24): in step 3, before the
        replan call, one frontier_goals_device call (frontier_params, default frontier_params()) for the replanning vehicles, from their
        replan heads to their true goals. GOAL plans to the goal and FRONTIER to the frontier point, both with plan_params' flags |
        PLAN_KNOWN_ONLY, so every node of the plan after its start is known and the certificate can accept it whole; NONE plans exactly as
        without explore. Acceptance, commits, the brake fallback and holding are unchanged; a vehicle whose frontier trajectory runs out
        away from its true goal is held (active, at rest) and replans next round from there with what it has sensed since. ARRIVED is
        judged against the true goal. The result then also has subgoal_kinds (rounds run, B): the FRONTIER_* kind each replan used, -1
        where the vehicle did not replan; and frontier_plans (B,) numpy: replans toward a frontier point.
        min_gain (an integer >= 0; needs explore=True) makes the frontier-goal call the view form (frontier_goals_device with cams =
        navigate's own rig, DESIGN §3.25): a frontier voxel is then a candidate only when the rig, level at yaw 0 at its cube centre, would
        see at least min_gain unknown voxels from there, so that a vehicle is not sent to a frontier with nothing left to show. min_gain=0
        selects exactly as the plain call (the same logs) and records the gains. The result then also has frontier_gains (rounds run, B):
        the view gain of the frontier each replan chose, -1 where no frontier was chosen.
        Vehicles share the map, so one vehicle's run depends on what the others sensed; with B = 1 it is that vehicle's alone. The world
        waits while the planner runs (no planning latency in simulated time). Within a round only per-vehicle values (stages, verdicts,
        counts, piece totals, positions of heads) cross to the host; points, pieces and logs stay on the device.
        Returns a dict: status, rounds_flown, replans, failed_replans, uncertified_rounds (B,) numpy; actions and verdicts (rounds run, B)
        (NAV_IDLE / NAV_KEPT / NAV_REPLANNED / NAV_REPLAN_FAILED; the verdict of the trajectory flown, NAV_NO_TRAJECTORY without one);
        replan_stages and replan_verdicts (rounds run, B): a replan's plan stage and certificate verdict (NAV_NO_TRAJECTORY: no plan call);
        logs: per round (vehicle indices (R,) numpy, log (R, n_log, 21) CUDA tensor); times: per round {stage: ms} from CUDA events (a
        "brake" stage with fallback="brake"); with fallback="brake" also brakes and held_rounds (B,) numpy: BRAKED stops taken and rounds
        spent held."""
        st0, gl = _f64(starts).reshape(-1, 3), _f64(goals).reshape(-1, 3)
        B = st0.shape[0]
        if gl.shape[0] != B or B < 1:
            raise ValueError(f"starts and goals must both be (B, 3), B >= 1, got {st0.shape} and {gl.shape}")
        if int(rounds) < 1 or not horizon > 0 or int(sense_every) < 1:
            raise ValueError("rounds and sense_every must be >= 1 and horizon > 0")
        if fallback not in ("keep", "brake"):
            raise ValueError(f"fallback must be 'keep' or 'brake', got {fallback!r}")
        if unknown not in ("free", "occupied"):
            raise ValueError(f"unknown must be 'free' or 'occupied', got {unknown!r}")
        if explore and unknown != "occupied":
            raise ValueError("explore=True plans through known space only: it needs unknown='occupied'")
        if min_gain is not None and (not explore or int(min_gain) < 0):
            raise ValueError("min_gain scores frontiers: it needs explore=True and must be >= 0")
        cams = list(sense_params) if isinstance(sense_params, (list, tuple)) else [sense_params if sense_params is not None else
                                                                                    globals()["sense_params"]()]
        if not cams:
            raise ValueError("sense_params: an empty camera list")
        brake, occupied = fallback == "brake", unknown == "occupied"
        if occupied and not brake:
            raise ValueError("unknown='occupied' commits to certified stops: it needs fallback='brake'")
        if occupied and not all(np.isfinite(c.sensing_horizon) for c in cams):
            raise ValueError("unknown='occupied' observes free space: every camera needs a finite sensing_horizon")
        if occupied:
            prev = self.unknown_policy()
            self.set_unknown_policy(UNKNOWN_OCCUPIED)
        try:
            if occupied and known_boxes is not None:
                self.map_mark_known(known_boxes)
            return self._navigate(st0, gl, int(rounds), float(horizon), int(sense_every), tol, plan_params, sim_params, cams, max_fields,
                                  stream, brake, brake_params, occupied, explore, frontier_params, min_gain)
        finally:
            if occupied:
                self.set_unknown_policy(prev)

    def _navigate(self, st0, gl, rounds, horizon, sense_every, tol, plan_params, sim_params, cams, max_fields, stream, brake, brake_params,
                  occupied, explore, frontier_params, min_gain=None):
        """navigate's rounds, under the unknown policy navigate set"""
        import torch
        p = plan_params if plan_params is not None else self.plan_params()
        if not p.flags & PLAN_CERTIFY:
            raise ValueError("navigate checks trajectories with the certificate: plan_params needs PLAN_CERTIFY")
        B, dev = st0.shape[0], torch.device("cuda", self.device)
        s = torch.cuda.current_stream(dev) if stream is None else stream
        sv, f64 = s.cuda_stream, dict(dtype=torch.float64, device=dev)
        bp = brake_params if brake_params is not None else self.brake_params(certify=p.certify, dynamics=p.dynamics)
        bpc = BrakeParams.from_buffer_copy(bytes(bp))   # a commit's stop
        bpc.certify.clearance.margin += NAV_COMMIT_SLACK
        sp = SimParams.from_buffer_copy(bytes(sim_params if sim_params is not None else sim_default_params()))
        sp.t_end = horizon
        hover = float(np.sqrt(sp.mass * sp.grav / (4 * sp.kf)))
        cp = CertifyParams.from_buffer_copy(bytes(p.certify))
        info = self.map_info()
        lo, hi = info["bmin"], info["bmax"]
        fpar = (frontier_params if frontier_params is not None else self.frontier_params()) if explore else None   # None: no explore
        if fpar is not None:
            pk = PlanParams.from_buffer_copy(bytes(p))
            pk.flags |= PLAN_KNOWN_ONLY

        def rest(x):   # at rest, level, at the hover rpm (as sim_init_from_trajectories)
            x[..., 3:] = 0.0
            x[..., 6] = 1.0
            x[..., 13:17] = hover

        with torch.cuda.stream(s):
            d_goals = torch.as_tensor(gl, **f64)
            init = torch.zeros((B, SIM_INIT_DOUBLES), **f64)
            init[:, 0:3] = torch.as_tensor(st0, **f64)
            rest(init)
            fleet = _Fleet(B, dev)   # the current trajectories; none yet
        status = np.full(B, NAV_ACTIVE)
        flown_rounds, replans, failed, uncert, brakes, held_rounds, commits, frontier_plans = (np.zeros(B, dtype=np.int64) for _ in range(8))
        held, braking = np.zeros(B, dtype=bool), np.zeros(B, dtype=bool)   # held at rest; flying a stop
        committed = np.zeros(B, dtype=bool)                                # flying a commit (unknown="occupied")
        subgoal = np.zeros(B, dtype=bool)                                  # flying a plan to a frontier point (explore)
        actions, subgoal_kinds, frontier_gains = np.full((rounds, B), NAV_IDLE), np.full((rounds, B), -1), np.full((rounds, B), -1)   # per round
        verdicts, replan_stages, replan_verdicts = (np.full((rounds, B), NAV_NO_TRAJECTORY) for _ in range(3))
        logs, times = [], []
        last = None   # (vehicle indices, log) of the last round flown
        stages = ("sense", "fuse") + ("observe",) * occupied + ("check", "replan") + ("brake",) * brake + ("fly", "advance")

        def sense(act):
            """the poses to sense from: every sense_every-th record of the last flown segment and its final record, else the state"""
            recs = []
            flown = set() if last is None else set(last[0].tolist())
            if last is not None:
                li, lg = last
                keep = np.isin(li, act)
                if keep.any():
                    n_log = lg.shape[1]
                    rows = sorted(set(range(0, n_log, sense_every)) | {n_log - 1})
                    sel = lg[torch.as_tensor(np.nonzero(keep)[0], device=dev)][:, rows].reshape(-1, SIM_DOUBLES)
                    recs.append(torch.cat([sel[:, 1:4], sel[:, 7:11]], 1))
            others = [b for b in act if b not in flown]
            if others:
                ini = init[torch.as_tensor(others, device=dev)]
                recs.append(torch.cat([ini[:, 0:3], ini[:, 6:10]], 1))
            return torch.cat(recs).contiguous()

        def check(act):
            """vehicle -> the certificate's verdict (and first_hit) of its remaining trajectory, one call per piece count"""
            ver, fhit = {}, {}
            have = [b for b in act if fleet.n[b] > 0]
            for N in sorted({int(fleet.n[b]) for b in have}):
                grp = [b for b in have if fleet.n[b] == N]
                _, gT, gC = fleet.gather(grp)
                gC = gC.reshape(len(grp), 3, 6 * N).permute(1, 0, 2).contiguous()
                summ = torch.empty((len(grp), C.sizeof(CertifySummary)), dtype=torch.uint8, device=dev)
                cp.clearance.pieces_per_traj = N
                self.trajectory_certify_device(len(grp) * N, gT.data_ptr(), gC.data_ptr(), cp, summ.data_ptr(), sv)
                ver.update(zip(grp, _field(summ, CertifySummary, "verdict").cpu().numpy().tolist()))
                if brake:
                    fhit.update(zip(grp, _field(summ, CertifySummary, "first_hit").cpu().numpy().tolist()))
            return ver, fhit

        def heads(need):
            """the replan heads (p, v, a) of these vehicles: the remaining trajectory's state at 0, else at rest where they are"""
            hd = torch.zeros((len(need), 9), **f64)
            moving = [i for i, b in enumerate(need) if fleet.n[b] > 0]
            if moving:
                q = torch.as_tensor([need[i] for i in moving], dtype=torch.int32, device=dev)
                out = torch.empty((len(moving), STATE_DOUBLES), **f64)
                self.trajectory_states_device(B, fleet.piece_off.data_ptr(), fleet.T.data_ptr(), fleet.coeffs.data_ptr(), len(moving), q.data_ptr(),
                                              torch.zeros(len(moving), **f64).data_ptr(), out.data_ptr(), sv)
                hd[torch.as_tensor(moving, device=dev)] = out[:, :9]
            still = [i for i, b in enumerate(need) if fleet.n[b] == 0]
            if still:   # never flown (init holds its start), or held at rest at its simulator position
                hd[torch.as_tensor(still, device=dev), :3] = init[torch.as_tensor([need[i] for i in still], device=dev), 0:3]
            return hd

        def plan(hd, gd, vs):
            """plan_states_device for vehicles vs from heads hd to goals gd -> (plans, their vehicles in plan order); with explore, GOAL and
            FRONTIER sub-goals plan known-only to the goal or the frontier point, NONE as without explore"""
            if fpar is None:
                return self.plan_states_device(hd, gd, params=p, max_fields=max_fields, stream=s), vs
            view = dict(cams=cams, min_gain=int(min_gain)) if min_gain is not None else {}
            fg, _ = self.frontier_goals_device(hd[:, :3].contiguous(), gd, params=fpar, max_fields=max_fields, stream=s, **view)
            rec = decode_frontier_goals(fg)
            kinds, gains = rec["kind"], rec["gain"]
            pts = _field(fg, FrontierGoal, "point")
            ex = [j for j in range(len(vs)) if kinds[j] != FRONTIER_NONE]
            nx = [j for j in range(len(vs)) if kinds[j] == FRONTIER_NONE]
            parts = []
            for js, to, params in ((ex, pts, pk), (nx, gd, p)):
                if js:
                    xi = torch.as_tensor(js, device=dev)
                    parts.append(self.plan_states_device(hd[xi].contiguous(), to[xi].contiguous(), params=params, max_fields=max_fields, stream=s))
            for j, b in enumerate(vs):
                skind[b] = kinds[j]
                if kinds[j] == FRONTIER_FRONTIER:
                    frontier_plans[b] += 1
                    sgain[b] = gains[j]
            return _cat_plans(parts), [vs[j] for j in ex + nx]

        def replan(act, ver):
            """replan the vehicles without a certified remaining trajectory (or flying a commit) and splice the accepted plans in ->
            (vehicles replanned, vehicle -> plan of an accepted plan, vehicle -> (plan, first_hit) to commit to a stop of, plans)"""
            need = [b for b in act if ver.get(b) != CERTIFIED or committed[b]]
            for b in ver:
                verdict[b] = ver[b]
            new, cand, pl = {}, {}, None
            if need:
                hd = heads(need)
                hp = hd[:, :3].cpu().numpy()
                inside = np.all((hp >= lo) & (hp <= hi), axis=1)   # a head outside the map fails without a call
                ok = [i for i in range(len(need)) if inside[i]]
                if ok:
                    vs = [need[i] for i in ok]
                    pl, vs = plan(hd[torch.as_tensor(ok, device=dev)].contiguous(), d_goals[torch.as_tensor(vs, device=dev)].contiguous(), vs)
                    stage = _field(pl["results"], PlanResult, "stage").cpu().numpy()
                    cv = _field(pl["certify"], CertifySummary, "verdict").cpu().numpy()
                    ph = _field(pl["certify"], CertifySummary, "first_hit").cpu().numpy() if occupied else None
                    for j, b in enumerate(vs):
                        rstage[b], rverdict[b] = stage[j], cv[j]
                        if stage[j] == OPTIMISED and cv[j] == CERTIFIED:
                            new[b] = j
                            subgoal[b] = skind[b] == FRONTIER_FRONTIER
                        elif occupied and stage[j] == OPTIMISED and cv[j] == COLLIDING and ph[j] > 0:
                            cand[b] = (j, float(ph[j]))
                for b in need:
                    replans[b] += 1
                    if b in new:
                        action[b], verdict[b] = NAV_REPLANNED, CERTIFIED
                        held[b] = braking[b] = committed[b] = False
                    else:
                        action[b] = NAV_REPLAN_FAILED
                        failed[b] += 1
                        if held[b]:
                            action[b] = NAV_HELD
                            held_rounds[b] += 1
                if new:   # the trajectories flown this round: the accepted plans, else the remaining ones
                    po = pl["piece_off"].cpu().numpy()
                    fleet.replace({b: _rows(pl, po, j) for b, j in new.items()})
            for b in act:
                if action[b] == NAV_IDLE:
                    action[b] = NAV_KEPT
            return need, new, cand, pl

        def stops(vs, ragged, t_stop_max, params):
            """one trajectory_brake_device call along vehicles vs's trajectories ragged -> vehicle -> (T, coeffs) of its BRAKED stop"""
            bk = self.trajectory_brake_device(*ragged, torch.as_tensor(t_stop_max, **f64), params=params, stream=s)
            ok = _field(bk["summary"], BrakeSummary, "status").cpu().numpy() == BRAKED
            if not ok.any():
                return {}
            ko = bk["piece_off"].cpu().numpy()
            return {b: _rows(bk, ko, j) for j, b in enumerate(vs) if ok[j]}

        def fall_back(need, new, cand, pl, ver, fhit):
            """commit to a certified stop along a new plan that collides further on; else brake along the remaining trajectory"""
            took = {}
            if cand:
                po = pl["piece_off"].cpu().numpy()
                # with the slack first; where no stop keeps it (passing close to unseen space, e.g. round a corner), the plan's margin
                for params in (bpc, bp):
                    vs = [b for b in sorted(cand) if b not in took]
                    if vs:
                        took.update(stops(vs, _ragged([_rows(pl, po, cand[b][0]) for b in vs], dev)[1:], [cand[b][1] for b in vs], params))
                for b in took:
                    if action[b] == NAV_HELD:
                        held_rounds[b] -= 1
                    action[b], verdict[b] = NAV_COMMITTED, CERTIFIED
                    commits[b] += 1
                    held[b], braking[b], committed[b] = False, True, True
                if took:
                    fleet.replace(took)
            # (a vehicle still holding a CERTIFIED remaining trajectory, a commit, keeps it)
            bv = [b for b in need if b not in new and b not in took and fleet.n[b] > 0 and ver.get(b) != CERTIFIED]
            got = stops(bv, fleet.gather(bv), [fhit[b] if ver[b] == COLLIDING else np.inf for b in bv], bp) if bv else {}
            for b in got:
                action[b], verdict[b] = NAV_BRAKED, CERTIFIED
                brakes[b] += 1
                braking[b] = True
            if got:
                fleet.replace(got)

        def advance(fly, fi, sim):
            """the state at the horizon and the rest of each trajectory; vehicles that arrive, stop, diverge or are held"""
            init[fi] = sim_init_from_log(sim["log"][:, -1])
            diverged = _field(sim["summary"], SimSummary, "diverged").cpu().numpy()
            t0 = torch.zeros(B, **f64)
            t0[fi] = horizon
            fleet.adopt(self.trajectory_shift_device(fleet.piece_off, fleet.T, fleet.coeffs, t0, stream=s))
            dist = torch.linalg.norm(init[fi, 0:3] - d_goals[fi], dim=1).cpu().numpy()
            for k, b in enumerate(fly):
                flown_rounds[b] += 1
                if verdict[b] != CERTIFIED:
                    uncert[b] += 1
                if diverged[k]:
                    status[b] = NAV_DIVERGED
                elif fleet.n[b] == 0 and (braking[b] or subgoal[b]) and dist[k] > tol:
                    # the stop (or a frontier plan) ran out: held at rest where the simulator left it
                    held[b], braking[b], committed[b], subgoal[b] = True, False, False, False
                    rest(init[b])
                elif fleet.n[b] == 0:
                    status[b] = NAV_ARRIVED if dist[k] <= tol else NAV_STOPPED
            gone = [b for b in range(B) if status[b] != NAV_ACTIVE and fleet.n[b] > 0]
            if gone:   # a vehicle that is done flies no more: its pieces go
                fleet.replace({b: (fleet.T[:0], fleet.coeffs[:0]) for b in gone})

        for r in range(rounds):
            act = np.nonzero(status == NAV_ACTIVE)[0]
            if act.size == 0:
                break
            ev = {k: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for k in stages}
            action, verdict, rstage, rverdict, skind, sgain = (actions[r], verdicts[r], replan_stages[r], replan_verdicts[r], subgoal_kinds[r],
                                                               frontier_gains[r])
            with torch.cuda.stream(s):
                with _timed(ev["sense"], s):
                    poses = sense(act)
                    seen = [self.sense_cloud_device(poses, 0, 3, params=cam, stream=s)[0] for cam in cams]
                with _timed(ev["fuse"], s):
                    for pts in seen:
                        if pts.shape[0]:
                            self.map_fuse_cloud_device(pts, stream=sv)
                if occupied:   # the free space the same images prove
                    with _timed(ev["observe"], s):
                        for cam in cams:
                            self.map_observe_device(poses, 0, 3, params=cam, stream=s)
                with _timed(ev["check"], s):
                    ver, fhit = check(act)
                with _timed(ev["replan"], s):
                    need, new, cand, pl = replan(act, ver)
                if brake:
                    with _timed(ev["brake"], s):
                        fall_back(need, new, cand, pl, ver, fhit)
                with _timed(ev["fly"], s):
                    fly = np.array([b for b in act if fleet.n[b] > 0], dtype=np.int64)
                    last = None
                    if fly.size:
                        fi = torch.as_tensor(fly, device=dev)
                        sim = self.simulate_device(fleet.piece_off, fleet.T, fleet.coeffs, fi.to(torch.int32), init[fi].contiguous(), params=sp,
                                                   stream=s)
                        last = (fly, sim["log"])
                with _timed(ev["advance"], s):
                    if fly.size:
                        advance(fly, fi, sim)
            s.synchronize()
            times.append({k: a.elapsed_time(e) for k, (a, e) in ev.items()})
            if last is not None:
                logs.append(last)
        status[status == NAV_ACTIVE] = NAV_TIMEOUT
        ran = len(times)
        out = dict(status=status, rounds_flown=flown_rounds, replans=replans, failed_replans=failed, uncertified_rounds=uncert,
                   actions=actions[:ran], verdicts=verdicts[:ran], replan_stages=replan_stages[:ran], replan_verdicts=replan_verdicts[:ran], logs=logs,
                   times=times)
        if brake:
            out.update(brakes=brakes, held_rounds=held_rounds)
        if occupied:
            out.update(commits=commits)
        if fpar is not None:
            out.update(subgoal_kinds=subgoal_kinds[:ran], frontier_plans=frontier_plans)
            if min_gain is not None:
                out.update(frontier_gains=frontier_gains[:ran])
        return out

    def plan_info(self):
        info = PlanInfo()
        self._check(self.lib.isdf_get_plan_info(self.h, C.byref(info)))
        return info.as_dict()

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
        T, Cc, N, B = self._block(T, coeffs, N0)
        p = self.clearance_params(K_c, reach, margin, N0)
        clear, vox = np.zeros(N * (int(K_c) + 1)), np.zeros(N * (int(K_c) + 1), dtype=np.int64)
        summ = (ClearanceSummary * B)()
        self._check(self.lib.isdf_trajectory_clearance(self.h, N, _dp(T), _dp(Cc), C.byref(p), _dp(clear), vox.ctypes.data_as(C.POINTER(C.c_int64)), summ))
        return clear, vox, [s.as_dict() for s in summ]

    def trajectory_clearance_device(self, N, d_T, d_coeffs, params, d_clear, d_voxel, d_summary, stream=0):
        """raw device pointers (e.g. torch .data_ptr()); d_summary holds N/N0 isdf_clearance_summary records (48 bytes each)"""
        self._check(self.lib.isdf_trajectory_clearance_device(self.h, N, C.c_void_p(d_T), C.c_void_p(d_coeffs), C.byref(params), C.c_void_p(d_clear),
                                                              C.c_void_p(d_voxel), C.c_void_p(d_summary), C.c_void_p(stream)))

    def pose_clearance_params(self, reach=None, margin=None, poses_per_group=0):
        p = PoseClearanceParams()
        self._check(self.lib.isdf_pose_clearance_default_params(C.byref(p)))
        if reach is not None:
            p.reach = float(reach)
            p.margin = float(reach) if margin is None else p.margin
        if margin is not None:
            p.margin = float(margin)
        p.poses_per_group = int(poses_per_group)
        return p

    def pose_clearance(self, records, pos_offset=0, quat_offset=3, reach=None, margin=None, poses_per_group=0):
        """clearance of the robot at Q poses read in place from records (Q, stride) float64: position at pos_offset, quaternion (w, x, y, z)
        at quat_offset -> (clear (Q,), witness voxels (Q,) int64, one summary dict per group). For isdf_simulate's log use (R * n_log, 21)
        with offsets 1 and 7; for trajectory_states' records (Q, 20) with offsets 0 and 12. Rows with a NaN pose (a log's unused records)
        report NaN and count as colliding, so pass only the rows that exist."""
        r = _f64(records)
        r = r.reshape(-1, r.shape[-1])
        Q, stride = r.shape
        if not (0 <= pos_offset <= stride - 3 and 0 <= quat_offset <= stride - 4):
            raise ValueError("pos_offset / quat_offset outside the record")
        p = self.pose_clearance_params(reach, margin, poses_per_group)
        G = 1 if poses_per_group == 0 else Q // max(int(poses_per_group), 1)
        clear, vox = np.zeros(Q), np.zeros(Q, dtype=np.int64)
        summ = (ClearanceSummary * max(G, 1))()
        base = r.ctypes.data
        self._check(self.lib.isdf_pose_clearance(self.h, Q, C.cast(base + 8 * pos_offset, C.POINTER(C.c_double)), C.cast(base + 8 * quat_offset, C.POINTER(C.c_double)), stride, C.byref(p),
                                                 _dp(clear), vox.ctypes.data_as(C.POINTER(C.c_int64)), summ))
        return clear, vox, [s.as_dict() for s in summ]

    def pose_clearance_device(self, Q, d_pos, d_quat, stride_doubles, params, d_clear, d_voxel, d_summary, stream=0):
        """raw device pointers: pose q at d_pos + q stride and d_quat + q stride (doubles); d_summary holds Q / poses_per_group records (48 bytes)"""
        v = C.c_void_p
        self._check(self.lib.isdf_pose_clearance_device(self.h, int(Q), v(d_pos), v(d_quat), int(stride_doubles), C.byref(params), v(d_clear),
                                                        v(d_voxel), v(d_summary), v(stream)))

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
        T, Cc, N, B = self._block(T, coeffs, N0)
        p = self.certify_params(K_c, reach, margin, N0, max_depth, max_samples)
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

    # ---- dynamic-limit certificate (see include/isdf.h) ----
    def dynamics_params(self, K=None, N0=0, max_depth=None, max_samples=None, **kw):
        """isdf_dynamics_default_params for this context, then the overrides: K, N0, max_depth, max_samples and any field of
        isdf_dynamics_params by name (vmax, amax, omgmax, thetamax, thrust_min, thrust_max, tol_v, tol_a, tol_omg, tol_theta, tol_thrust)"""
        p = DynamicsParams()
        self._check(self.lib.isdf_dynamics_default_params(self.h, C.byref(p)))
        if K is not None:
            p.samples_per_piece = int(K)
        p.pieces_per_traj = int(N0)
        if max_depth is not None:
            p.max_depth = int(max_depth)
        if max_samples is not None:
            p.max_samples_per_traj = int(max_samples)
        for k, v in kw.items():
            if k not in {n for n, _ in DynamicsParams._fields_} or k == "reserved_":
                raise TypeError(f"unknown isdf_dynamics_params field {k}")
            setattr(p, k, v)
        return p

    def trajectory_dynamics(self, T, coeffs, params=None, **kw):
        """one summary dict per trajectory (pieces b*N0 .. b*N0+N0-1; N0 = 0: a single trajectory): verdict (FEASIBLE 1, VIOLATING -1,
        UNDECIDED 0), upper / attained / t_attained (arrays over DYN_QUANTITIES), thrust_lower, thrust_attained_min, t_thrust_attained_min,
        violated, undecided, samples, undecided_intervals, depth. params: an isdf_dynamics_params, or None for dynamics_params(**kw)"""
        p = params if params is not None else self.dynamics_params(**kw)
        T, Cc, N, B = self._block(T, coeffs, p.pieces_per_traj)
        summ = (DynamicsSummary * B)()
        self._check(self.lib.isdf_trajectory_dynamics(self.h, N, _dp(T), _dp(Cc), C.byref(p), summ))
        return [s.as_dict() for s in summ]

    def trajectory_dynamics_device(self, N, d_T, d_coeffs, params, d_summary, stream=0):
        """raw device pointers (e.g. torch .data_ptr()); d_summary holds N/N0 isdf_dynamics_summary records (168 bytes each)"""
        self._check(self.lib.isdf_trajectory_dynamics_device(self.h, N, C.c_void_p(d_T), C.c_void_p(d_coeffs), C.byref(params),
                                                             C.c_void_p(d_summary), C.c_void_p(stream)))

    # ---- certified swept volume (see include/isdf.h) ----
    def swept_params(self, K=None, band=None, tol=None, max_depth=None, max_samples=None):
        """isdf_swept_default_params with K = this context's integral_intervs, band = 2 safety_hor, tol = occupancy_resolution / 100,
        then the given overrides"""
        p = SweptParams()
        self._check(self.lib.isdf_swept_default_params(C.byref(p)))
        p.samples_per_piece = int(self.cfg.integral_intervs if K is None else K)
        p.band = float(2.0 * self.cfg.safety_hor if band is None else band)
        p.tol = float(self.cfg.occupancy_resolution / 100.0 if tol is None else tol)
        if max_depth is not None:
            p.max_depth = int(max_depth)
        if max_samples is not None:
            p.max_samples_per_point = int(max_samples)
        return p

    @staticmethod
    def _traj(T, coeffs):
        T = _f64(T).reshape(-1)
        Cc = _f64(coeffs).reshape(-1)
        assert Cc.size == 18 * T.size
        return T, Cc

    @staticmethod
    def _block(T, coeffs, N0):
        """a block of trajectories of N0 pieces each (N0 = 0: a single trajectory) as (T, coeffs, N, B), B the number of summaries"""
        T, Cc = Evaluator._traj(T, coeffs)
        N = T.size
        return T, Cc, N, 1 if N0 <= 0 else max(N // N0, 1)

    def swept_volume_sdf(self, T, coeffs, pts, params=None):
        """(value, lower, tstar, decided) at points (n, 3): the certified swept-volume SDF of the trajectory"""
        T, Cc = self._traj(T, coeffs)
        p = params if params is not None else self.swept_params()
        P = _f64(pts).reshape(-1, 3)
        n = P.shape[0]
        v, lo, ts, dec = np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(n, dtype=np.uint8)
        self._check(self.lib.isdf_swept_volume_sdf(self.h, T.size, _dp(T), _dp(Cc), C.byref(p), n, _dp(P), _dp(v), _dp(lo), _dp(ts),
                                                   dec.ctypes.data_as(C.POINTER(C.c_uint8))))
        return v, lo, ts, dec

    def swept_volume_grid(self, T, coeffs, grid, params=None):
        """(value, lower, tstar, decided) as (X, Y, Z) arrays, and the info dict of the call"""
        T, Cc = self._traj(T, coeffs)
        p = params if params is not None else self.swept_params()
        shp = (grid.X, grid.Y, grid.Z)
        v, lo, ts, dec = np.zeros(shp), np.zeros(shp), np.zeros(shp), np.zeros(shp, dtype=np.uint8)
        info = SweptInfo()
        self._check(self.lib.isdf_swept_volume_grid(self.h, T.size, _dp(T), _dp(Cc), C.byref(p), C.byref(grid), _dp(v), _dp(lo), _dp(ts),
                                                    dec.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(info)))
        return v, lo, ts, dec, info.as_dict()

    def swept_volume_grid_device(self, N, d_T, d_coeffs, grid, params, d_value, d_lower=0, d_tstar=0, d_decided=0, stream=0, info=True):
        """raw device pointers (e.g. torch .data_ptr(); 0 = not wanted for lower / tstar / decided); returns the info dict (or None)"""
        inf = SweptInfo() if info else None
        self._check(self.lib.isdf_swept_volume_grid_device(self.h, N, C.c_void_p(d_T), C.c_void_p(d_coeffs), C.byref(params), C.byref(grid),
                                                           C.c_void_p(d_value), C.c_void_p(d_lower or None), C.c_void_p(d_tstar or None),
                                                           C.c_void_p(d_decided or None), C.byref(inf) if info else None, C.c_void_p(stream)))
        return inf.as_dict() if info else None

    def swept_volume_mesh(self, T, coeffs, grid, params=None):
        """(V (nV, 3), vtime (nV), F (nF, 3) int32, info dict): the surface {SV = 0} of the grid's field by marching tetrahedra"""
        T, Cc = self._traj(T, coeffs)
        p = params if params is not None else self.swept_params()
        nV, nF = C.c_int64(0), C.c_int64(0)
        info = SweptInfo()
        f = self.lib.isdf_swept_volume_mesh
        r = f(self.h, T.size, _dp(T), _dp(Cc), C.byref(p), C.byref(grid), 0, 0, None, None, None, C.byref(nV), C.byref(nF), C.byref(info))
        if r != 0 and not (r == -1 and (nV.value > 0 or nF.value > 0)):
            self._check(r)
        V, vt, F = np.zeros((max(nV.value, 1), 3)), np.zeros(max(nV.value, 1)), np.zeros((max(nF.value, 1), 3), dtype=np.int32)
        if r != 0:
            self._check(f(self.h, T.size, _dp(T), _dp(Cc), C.byref(p), C.byref(grid), nV.value, nF.value, _dp(V), _dp(vt),
                          F.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(nV), C.byref(nF), C.byref(info)))
        return V[:nV.value].copy(), vt[:nV.value].copy(), F[:nF.value].copy(), info.as_dict()

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

    def frontend_path_batch(self, start, goals, cap=None, unknown_weight=None):
        """one start, B goals -> dict(paths: list of (n_b, 3) cube centres, roll_pitch: list of (n_b, 2) degrees, offsets (B + 1),
        costs (B), found (B) bool). cap = None: a first guess, repeated once with the exact total when the paths are longer.
        unknown_weight (every front-end binding): None passes NULL params; a number passes isdf_frontpath_params with that surcharge on
        unknown voxels (0 is the NULL field bit for bit)."""
        st = _f64(start).reshape(3)
        goals = _f64(goals).reshape(-1, 3)
        B = goals.shape[0]
        cap = self._path_cap(cap)
        for attempt in range(2):
            xyz, rp = np.zeros((max(cap, 1), 3)), np.zeros((max(cap, 1), 2))
            off, cost, found = np.zeros(B + 1, dtype=np.int32), np.zeros(B), np.zeros(B, dtype=np.uint8)
            r = self.lib.isdf_frontend_path_batch(self.h, _dp(st), B, _dp(goals), _fpp(unknown_weight), cap, _dp(xyz), _dp(rp),
                                                  off.ctypes.data_as(C.POINTER(C.c_int32)), _dp(cost), found.ctypes.data_as(C.POINTER(C.c_uint8)))
            if r == -1 and attempt == 0 and off[B] > cap:
                cap = int(off[B])
                continue
            self._check(r)
            break
        n = int(off[B])
        return dict(paths=[xyz[off[b]:off[b + 1]] for b in range(B)], roll_pitch=[rp[off[b]:off[b + 1]] for b in range(B)],
                    xyz=xyz[:n], rp=rp[:n], offsets=off, costs=cost, found=found.astype(bool))

    def frontend_path_pairs(self, starts, goals, cap=None, max_fields=0, unknown_weight=None):
        """B (start, goal) pairs, start b with goal b -> what frontend_path_batch returns, in pair order (isdf_frontend_path_pairs).
        max_fields: the fields of distinct start voxels held at once (0: the library's 4 GiB budget)"""
        sts, goals = _f64(starts).reshape(-1, 3), _f64(goals).reshape(-1, 3)
        if sts.shape != goals.shape:
            raise ValueError(f"starts and goals must both be (B, 3), got {sts.shape} and {goals.shape}")
        B = goals.shape[0]
        cap = self._path_cap(cap)
        for attempt in range(2):
            xyz, rp = np.zeros((max(cap, 1), 3)), np.zeros((max(cap, 1), 2))
            off, cost, found = np.zeros(B + 1, dtype=np.int32), np.zeros(B), np.zeros(B, dtype=np.uint8)
            r = self.lib.isdf_frontend_path_pairs(self.h, B, _dp(sts), _dp(goals), _fpp(unknown_weight), int(max_fields), cap, _dp(xyz), _dp(rp),
                                                  off.ctypes.data_as(C.POINTER(C.c_int32)), _dp(cost), found.ctypes.data_as(C.POINTER(C.c_uint8)))
            if r == -1 and attempt == 0 and off[B] > cap:
                cap = int(off[B])
                continue
            self._check(r)
            break
        n = int(off[B])
        return dict(paths=[xyz[off[b]:off[b + 1]] for b in range(B)], roll_pitch=[rp[off[b]:off[b + 1]] for b in range(B)],
                    xyz=xyz[:n], rp=rp[:n], offsets=off, costs=cost, found=found.astype(bool))

    def frontend_path_pairs_raw(self, starts, goals, cap, max_fields=0):
        """isdf_frontend_path_pairs with the caller's cap: (status, offsets)"""
        sts, goals = _f64(starts).reshape(-1, 3), _f64(goals).reshape(-1, 3)
        B = goals.shape[0]
        xyz, rp = np.zeros((max(cap, 1), 3)), np.zeros((max(cap, 1), 2))
        off, cost, found = np.full(B + 1, -7, dtype=np.int32), np.zeros(B), np.zeros(B, dtype=np.uint8)
        r = self.lib.isdf_frontend_path_pairs(self.h, B, _dp(sts), _dp(goals), None, int(max_fields), int(cap), _dp(xyz), _dp(rp),
                                              off.ctypes.data_as(C.POINTER(C.c_int32)), _dp(cost), found.ctypes.data_as(C.POINTER(C.c_uint8)))
        return r, off

    def frontend_path(self, start, goal, cap=None, unknown_weight=None):
        """-> (path (n, 3), roll_pitch (n, 2), cost, found), through isdf_frontend_path"""
        st, gl = _f64(start).reshape(3), _f64(goal).reshape(3)
        cap = self._path_cap(cap)
        for attempt in range(2):
            xyz, rp = np.zeros((max(cap, 1), 3)), np.zeros((max(cap, 1), 2))
            n, cost, found = C.c_int32(0), C.c_double(0), C.c_uint8(0)
            r = self.lib.isdf_frontend_path(self.h, _dp(st), _dp(gl), _fpp(unknown_weight), cap, _dp(xyz), _dp(rp), C.byref(n), C.byref(cost), C.byref(found))
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

    def frontend_path_batch_device(self, start, B, d_goals, cap, d_xyz, d_rp, d_offsets, d_costs, d_found, stream=None, unknown_weight=None):
        st = _f64(start).reshape(3)
        self._check(self.lib.isdf_frontend_path_batch_device(self.h, _dp(st), B, d_goals, _fpp(unknown_weight), cap, d_xyz, d_rp, d_offsets, d_costs, d_found, stream))

    def frontend_path_field_device(self, start, d_g, stream=None, unknown_weight=None):
        st = _f64(start).reshape(3)
        self._check(self.lib.isdf_frontend_path_field_device(self.h, _dp(st), _fpp(unknown_weight), d_g, stream))

    def frontend_path_pairs_device(self, B, d_starts, d_goals, cap, d_xyz, d_rp, d_offsets, d_costs, d_found, stream=None, max_fields=0,
                                   unknown_weight=None):
        self._check(self.lib.isdf_frontend_path_pairs_device(self.h, int(B), d_starts, d_goals, _fpp(unknown_weight), int(max_fields), int(cap), d_xyz, d_rp,
                                                             d_offsets, d_costs, d_found, stream))

    def frontend_path_fields_device(self, starts, d_g, stream=None, unknown_weight=None):
        """the fields from S starts (S, 3) in one relaxation into d_g (a raw device pointer to S*X*Y*Z float64), field s at d_g + s*X*Y*Z"""
        sts = _f64(starts).reshape(-1, 3)
        self._check(self.lib.isdf_frontend_path_fields_device(self.h, sts.shape[0], _dp(sts), _fpp(unknown_weight), d_g, stream))

    # ---- frontiers of known space (see include/isdf.h, DESIGN §3.24) ----
    def map_frontiers(self):
        """-> dict(voxels (n,) int64 ascending, cluster_of (n,) int64, clusters: FRONTIER_CLUSTER_DTYPE array by ascending id, info dict)"""
        info = FrontierInfo()
        r = self.lib.isdf_map_frontiers(self.h, 0, None, None, 0, None, C.byref(info))
        if r == -1 and (info.frontier_voxels > 0 or info.clusters > 0):
            n, nc = int(info.frontier_voxels), int(info.clusters)
            vox, cid = np.zeros(max(n, 1), dtype=np.int64), np.zeros(max(n, 1), dtype=np.int64)
            tab = np.zeros(max(nc, 1), dtype=FRONTIER_CLUSTER_DTYPE)
            r = self.lib.isdf_map_frontiers(self.h, n, vox.ctypes.data, cid.ctypes.data, nc, tab.ctypes.data, C.byref(info))
            self._check(r)
            return dict(voxels=vox[:n], cluster_of=cid[:n], clusters=tab[:nc], info=info.as_dict())
        self._check(r)
        return dict(voxels=np.zeros(0, dtype=np.int64), cluster_of=np.zeros(0, dtype=np.int64), clusters=np.zeros(0, dtype=FRONTIER_CLUSTER_DTYPE),
                    info=info.as_dict())

    def map_frontiers_device(self, cap_voxels, d_voxels, d_cluster_of, cap_clusters, d_clusters, stream=None):
        """isdf_map_frontiers_device into raw device pointers (int64 x cap_voxels twice, 64-byte records x cap_clusters) -> info dict"""
        info = FrontierInfo()
        self._check(self.lib.isdf_map_frontiers_device(self.h, int(cap_voxels), d_voxels, d_cluster_of, int(cap_clusters), d_clusters,
                                                       C.byref(info), stream))
        return info.as_dict()

    def frontier_params(self, **kw):
        """isdf_frontier_default_params with any field overridden (goal_weight=, min_cluster_voxels=)"""
        p = FrontierParams()
        self._check(self.lib.isdf_frontier_default_params(C.byref(p)))
        for k, v in kw.items():
            if k not in {n for n, _ in FrontierParams._fields_}:
                raise TypeError(f"unknown frontier parameter {k!r}")
            setattr(p, k, v)
        return p

    def frontier_goals(self, starts, goals, params=None, max_fields=0, cams=None, min_gain=0):
        """B (start, goal) pairs -> (FRONTIER_GOAL_DTYPE array (B,), info dict) through isdf_frontier_goals; with a rig cams (one
        sense_params or a list), through isdf_frontier_goals_view: candidates also need a view gain >= min_gain"""
        sts, gls = _f64(starts).reshape(-1, 3), _f64(goals).reshape(-1, 3)
        if sts.shape != gls.shape:
            raise ValueError(f"starts and goals must both be (B, 3), got {sts.shape} and {gls.shape}")
        out = np.zeros(sts.shape[0], dtype=FRONTIER_GOAL_DTYPE)
        info = FrontierInfo()
        prm = None if params is None else C.byref(params)
        if cams is None:
            if min_gain:
                raise ValueError("min_gain needs a rig: pass cams")
            self._check(self.lib.isdf_frontier_goals(self.h, sts.shape[0], _dp(sts), _dp(gls), prm, int(max_fields), out.ctypes.data, C.byref(info)))
        else:
            rig = _rig(cams)
            self._check(self.lib.isdf_frontier_goals_view(self.h, sts.shape[0], _dp(sts), _dp(gls), prm, len(rig), C.byref(rig), int(min_gain),
                                                          int(max_fields), out.ctypes.data, C.byref(info)))
        return out, info.as_dict()

    def frontier_goals_device(self, d_starts, d_goals, params=None, max_fields=0, stream=None, cams=None, min_gain=0):
        """d_starts, d_goals: (B, 3) float64 CUDA tensors -> ((B, 64) uint8 CUDA tensor of isdf_frontier_goal records, info dict); cams and
        min_gain as for frontier_goals"""
        import torch
        B = int(d_starts.shape[0])
        out = torch.empty((B, C.sizeof(FrontierGoal)), dtype=torch.uint8, device=d_starts.device)
        info = FrontierInfo()
        sv = stream.cuda_stream if hasattr(stream, "cuda_stream") else stream
        prm = None if params is None else C.byref(params)
        if cams is None:
            if min_gain:
                raise ValueError("min_gain needs a rig: pass cams")
            self._check(self.lib.isdf_frontier_goals_device(self.h, B, d_starts.data_ptr(), d_goals.data_ptr(), prm, int(max_fields), out.data_ptr(),
                                                            C.byref(info), sv))
        else:
            rig = _rig(cams)
            self._check(self.lib.isdf_frontier_goals_view_device(self.h, B, d_starts.data_ptr(), d_goals.data_ptr(), prm, len(rig), C.byref(rig),
                                                                 int(min_gain), int(max_fields), out.data_ptr(), C.byref(info), sv))
        return out, info.as_dict()

    def frontend_path_info(self):
        out = FrontPathInfo()
        self._check(self.lib.isdf_frontend_path_info(self.h, C.byref(out)))
        return out.as_dict()

    def dbg_frontend_launch(self):
        """the last feasibility run's pipeline ("one_pass", "core", "tables") and (blocks, threads) of its mask-accumulation kernel
        (isdf_dbg_frontend_launch, not part of include/isdf.h); None before any run"""
        out = (C.c_int * 3)()
        self.lib.isdf_dbg_frontend_launch.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
        self._check(self.lib.isdf_dbg_frontend_launch(self.h, out))
        if out[0] < 0:
            return None
        return ("one_pass", "core", "tables")[out[0]], (out[1], out[2])

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

    def dbg_disc_k(self, k):
        """sub-boxes per cell edge of the discrete scan's filtered lists, from the next set_shape_mesh on (1: the full lists)"""
        self._check(self.lib.isdf_dbg_disc_k(self.h, int(k)))

    def dbg_disc_lists(self):
        """the discrete scan's filtered lists, copied to the host: dict(k, cell_off, cell_cnt (shaped as dbg_mesh_grid's arrays),
        cand (uint32), cand_lb (float32)); None when none were built (the scan walks the full lists)"""
        vp, llp = C.c_void_p, C.POINTER(C.c_longlong)
        u32p, u16p, fp = C.POINTER(C.c_uint32), C.POINTER(C.c_uint16), C.POINTER(C.c_float)
        self.lib.isdf_dbg_disc_lists.argtypes = [vp, llp, u32p, u16p, u32p, fp]
        sizes = np.zeros(2, dtype=np.int64)
        self._check(self.lib.isdf_dbg_disc_lists(self.h, sizes.ctypes.data_as(llp), None, None, None, None))
        if sizes[0] == 0:
            return None
        gdim = self.dbg_mesh_grid(arrays=False)["gdim"]
        off, cnt = np.zeros(gdim, dtype=np.uint32), np.zeros(gdim, dtype=np.uint16)
        cand, lb = np.zeros(int(sizes[0]), dtype=np.uint32), np.zeros(int(sizes[0]), dtype=np.float32)
        self._check(self.lib.isdf_dbg_disc_lists(self.h, sizes.ctypes.data_as(llp), off.ctypes.data_as(u32p), cnt.ctypes.data_as(u16p),
                                                 cand.ctypes.data_as(u32p), lb.ctypes.data_as(fp)))
        return dict(k=int(sizes[1]), cell_off=off, cell_cnt=cnt, cand=cand, cand_lb=lb)

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
