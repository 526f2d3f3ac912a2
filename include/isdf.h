/* isdf.h — C ABI of libisdf_b200.so: H100-native (sm_90a) collision cost/gradient evaluator for the
 * Implicit-SDF-Planner back end. Plain pointers and sizes only; no torch / Eigen / ROS types.
 *
 * Every entry point names the reference interface it replaces (paths relative to /root/reference/src):
 *   hpp   = planner_algorithm/include/planner_algorithm/back_end_optimizer.hpp
 *   swm   = swept_volume/include/swept_volume/sw_manager.hpp
 *   Shape = utils/include/utils/Shape.hpp, utils/src/Shape.cpp
 *   pcs   = map_manager/include/map_manager/PCSmap_manager.h ; grid = map_manager/src/Gridmap3D.cpp
 *   minco = utils/include/utils/minco.hpp ; lmbm = utils/include/lmbm/lmbm.h ; lbfgs = utils/include/utils/lbfgs.hpp
 *
 * Conventions
 *   - All functions return 0 on success, a negative isdf_status on failure; isdf_last_error() gives the message.
 *     On failure every output cost is set to NaN so that either optimiser driver terminates
 *     (the LMBM callback has no error channel, lmbm_call.f:125; L-BFGS aborts on NaN, lbfgs.hpp:148-197).
 *   - Matrices follow Eigen's defaults: `coeffs`/`gradC` are MatrixX3d (6N x 3) COLUMN-major:
 *     element (6*i + k, axis) at [axis*6N + 6*i + k] = t^k coefficient of piece i (hpp:434,460).
 *   - There is no CPU fallback: if no CUDA device / kernel image is usable, isdf_create fails.
 *   - Setters that replace state (maps, the robot shape, the front-end kernels, obstacle point sets) check their arguments first: a
 *     refused call leaves the previous state in place. Before a setter touches the device memory the current state lives in, it gives
 *     that state up (a new shape also gives up the front-end kernels), and it sets the new state only once it is complete: a CUDA
 *     failure leaves no map / shape / kernels / point set, and later calls that need one get ISDF_ERR_STATE.
 */
#ifndef ISDF_H
#define ISDF_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct isdf_ctx isdf_ctx;

typedef enum isdf_status {
    ISDF_OK = 0,
    ISDF_ERR_INVALID = -1,   /* bad argument */
    ISDF_ERR_STATE = -2,     /* map / shape / points not set */
    ISDF_ERR_CUDA = -3,      /* CUDA runtime or launch failure (message has the CUDA error string) */
    ISDF_ERR_UNSUPPORTED = -4
} isdf_status;

/* Subset of struct Config (utils/include/utils/config.hpp:13-203) that the hot path reads, in the units of
 * plan_manager/config/ *.yaml. Same field order as oracle/oracle_capi.cpp::orc_config. */
typedef struct isdf_config {
    double vehicle_mass, grav_acc, horiz_drag, vert_drag, paras_drag, speed_eps; /* FlatnessMap::reset, flatness.hpp:36-51 */
    double vmax, omgmax, thetamax;                                               /* hpp:678-680 */
    double weight_v, weight_p, weight_omg, weight_theta;                         /* hpp:683-687 */
    double smoothing_eps;        /* smooth_fac, hpp:689 */
    double safety_hor;           /* hpp:691 */
    double occupancy_resolution; /* bd = kernel_size * occupancy_resolution, hpp:692 */
    int32_t kernel_size;
    int32_t integral_intervs;    /* integralRes K, hpp:690: K+1 trapezoid nodes per piece */
    int32_t threads_num;         /* kept for interface parity (config.hpp:16); ignored by the GPU path */
    int32_t flags;               /* isdf_flags */
} isdf_config;

typedef enum isdf_flags {
    ISDF_WITH_DYNAMICS = 1,   /* velocity / body-rate / tilt penalties of addTimeIntPenaltyParallel (hpp:505-534) */
    ISDF_WITH_COLLISION = 2   /* grad_cost_p (hpp:766-824) wired into the sample loop as hpp:619-626 wires its SV sibling */
} isdf_flags;

/* Numeric ids shared with oracle/oracle_shapes.hpp::ShapeKind. params[] layout per kind is documented in
 * implicit-sdf-planner_b200/csrc/isdf_shapes.cuh; isdf_set_shape_named() fills the reference's hard-coded constants. */
typedef enum isdf_shape_kind {
    ISDF_SHAPE_BALL = 0, ISDF_SHAPE_POINT = 1, ISDF_SHAPE_TORUS = 2, ISDF_SHAPE_CAPPED_TORUS = 3,
    ISDF_SHAPE_CAPPED_CONE = 4, ISDF_SHAPE_ROUNDED_CONE = 5, ISDF_SHAPE_WIREFRAME_BOX = 6,
    ISDF_SHAPE_BEND_LINEAR = 7, ISDF_SHAPE_TWIST_BOX = 8, ISDF_SHAPE_BEND_BOX = 9, ISDF_SHAPE_TABLE = 10,
    ISDF_SHAPE_TREFOIL = 11, ISDF_SHAPE_SMOOTH_DIFFERENCE = 12, ISDF_SHAPE_SMOOTH_INTERSECTION = 13,
    ISDF_SHAPE_CSG = 14, ISDF_SHAPE_BOX = 15, ISDF_SHAPE_MESH = 16
} isdf_shape_kind;

/* What isdf_shape_query computes — the four BasicShape virtuals (Shape.hpp:469-472). */
typedef enum isdf_query {
    ISDF_QUERY_SDF = 0,       /* getonlySDF(pos_rel) */
    ISDF_QUERY_GRAD = 1,      /* getonlyGrad1(pos_rel) */
    ISDF_QUERY_SDF_GRAD = 2   /* getSDFwithGrad1(pos_rel, grad) */
} isdf_query;

/* attitude grid of the front end's collision kernels (config yaml: kernel_max_roll / kernel_max_pitch / kernel_ang_res, degrees;
 * front_end_safeh); kernel_size and occupancy_resolution come from isdf_config */
typedef struct isdf_kernel_config {
    double kernel_max_roll, kernel_max_pitch, kernel_ang_res, front_end_safeh;
} isdf_kernel_config;

typedef struct isdf_stats {
    int64_t kernel_launches;   /* kernels of this library launched since isdf_create */
    int64_t evals_discrete;    /* isdf_eval_discrete* calls */
    int64_t evals_swept;       /* isdf_eval_swept* calls */
    int64_t last_pairs;        /* (sample, voxel) pairs that reached the SDF in the last discrete evaluation */
    int64_t last_sdf_evals;    /* SDF evaluations in the last swept-volume evaluation */
    double last_kernel_ms;     /* device time of the last evaluation's kernels (CUDA events on the launch stream) */
} isdf_stats;

/* ---- lifetime -------------------------------------------------------------------------------------------- */
/* values of plan_manager/config/config_CappedCone.yaml; flags = DYNAMICS (the live reference callback; add ISDF_WITH_COLLISION for the discrete grad_cost_p term) */
int isdf_default_config(isdf_config *cfg);
/* replaces TrajOptimizer::setParam (hpp:667-722) + SweptVolumeManager ctor (swm:135-150). device = CUDA ordinal. */
int isdf_create(const isdf_config *cfg, int device, isdf_ctx **out);
int isdf_destroy(isdf_ctx *ctx);
const char *isdf_last_error(void);
int isdf_get_stats(isdf_ctx *ctx, isdf_stats *out);
/* Shard the evaluation: this context evaluates samples / obstacle points with index % world == rank and returns
 * partial sums (caller all-reduces 19N+1 doubles). Default rank 0 / world 1. */
int isdf_set_shard(isdf_ctx *ctx, int rank, int world);

/* ---- robot shape: replaces SweptVolumeManager::initShape (swm:255-275) and the Generalshape ctor (Shape.cpp:27-103) */
/* rotate_rowmajor / trans = Generalshape::Rotate / trans from poly_params (Shape.hpp:776-780); NULL = identity / zero */
int isdf_set_shape_analytic(isdf_ctx *ctx, int kind, const double *params, int nparams,
                            const double *rotate_rowmajor, const double *trans);
/* factory keyed by the OBJ basename like shapeConstructors (swm:74-123): "Torus", "CSG", ...; plus "Ball", "Point" */
int isdf_set_shape_named(isdf_ctx *ctx, const char *name, const double *rotate_rowmajor, const double *trans);
/* triangle mesh (V: nV x 3 row-major, F: nF x 3 row-major); poly_params = {tx,ty,tz, roll,pitch,yaw in degrees} pre-transform as
 * Shape.cpp:38-50, NULL = none. SDF = s * dist (Shape.cpp:105-151); the distance is exact, the sign factor s depends on the mode:
 *   ISDF_MESH_SIGN_AUTO    closed, consistently oriented mesh -> ISDF_MESH_SIGN_EXACT, anything else (open mesh, triangle soup) ->
 *                          ISDF_MESH_SIGN_WINDING (as igl::fast_winding_number accepts any soup);
 *   ISDF_MESH_SIGN_EXACT   s = ±1, the exact inside/outside classification (angle-weighted pseudonormals); ISDF_ERR_UNSUPPORTED if the mesh
 *                          is not closed. This is what the reference's s = 1 - 2 w rounds to; DESIGN.md "mesh sign" reports the deviation;
 *   ISDF_MESH_SIGN_WINDING s = 1 - 2 w with w the generalised winding number, NOT thresholded — the reference's form (Shape.cpp:110-111).
 *                          w is evaluated hierarchically in FP64 (first-order expansion, exact near field), i.e. closer to the true winding
 *                          number than the reference's FP32 tree, not bit-equal to it. Discrete path, isdf_shape_query and the front end
 *                          support this mode; the swept-volume entry points return ISDF_ERR_UNSUPPORTED for it.
 * isdf_set_shape_mesh = isdf_set_shape_mesh_ex(..., ISDF_MESH_SIGN_AUTO). */
typedef enum isdf_mesh_sign { ISDF_MESH_SIGN_AUTO = 0, ISDF_MESH_SIGN_EXACT = 1, ISDF_MESH_SIGN_WINDING = 2 } isdf_mesh_sign;
int isdf_set_shape_mesh(isdf_ctx *ctx, const double *V, int nV, const int32_t *F, int nF, const double *poly_params);
int isdf_set_shape_mesh_ex(isdf_ctx *ctx, const double *V, int nV, const int32_t *F, int nF, const double *poly_params, int sign_mode);
/* the BasicShape virtual surface (Shape.hpp:469-472) for n body-frame points (n x 3 row-major); sdf/grad may be NULL */
int isdf_shape_query(isdf_ctx *ctx, const double *p_rel, int n, double *sdf, double *grad, int what);

/* ---- occupancy map: replaces GridMap3D::createGridMap + the fill in PCSmap_manager.cpp:148-181 ------------ */
/* occ: X*Y*Z bytes, address ix*Y*Z + iy*Z + iz (GridMap3D.h:194-195), non-zero = occupied.
 * boundary_xyzmax is taken as bmin + size*res. */
int isdf_set_map_u8(isdf_ctx *ctx, const uint8_t *occ, int X, int Y, int Z, const double *bmin, double res);
/* the reference's own storage: one double per voxel (GridMap3D.h:215) */
int isdf_set_map_f64(isdf_ctx *ctx, const double *grid_map, int X, int Y, int Z, const double *bmin, double res);

/* PCSmapManager::rcvGlobalMapHandler (PCSmap_manager.cpp:111-181) on the device: the occupancy grid from a point cloud.
 * points: n records of stride_bytes each, with x, y, z as float32 at byte offsets 0, 4, 8 (pcl::PointXYZ: stride 16; a PointCloud2's
 * data with point_step as the stride).
 *   Bounds      per axis min starts at 999999999 and max at -999999999 (HUGE_NUMBER, PCSmap_manager.cpp:6,11-12) and is updated with
 *               strict < / > from (double) of every finite coordinate (:111-143).
 *   Dimensions  X = (int)ceil((max - min) / res) per axis in FP64 (createGridMap, Gridmap3D.cpp:25-39).
 *   Index       getGridIndex (Gridmap3D.cpp:135-175) restated exactly: ix = (int)floor(((double)x - min) / res), clamped to X - 1,
 *               including its "iy < 0 => ix = 0" branches (they cannot fire for points inside the bounds). A point on max at an exact
 *               multiple of res lands in the top layer X - 1.
 *   Occupancy   a voxel is occupied when its point count is >= sta_threshold (:151-181); sta_threshold <= 0 marks every voxel occupied,
 *               as in the reference. Every shipped config uses 1.
 *   Frame       bmin = min and bmax = max (the reference's boundary_xyzmax is the cloud's maximum, not bmin + X*res). Every index the
 *               library derives from a map is clamp(floor((clamp(c, bmin, bmax) - bmin) / res), 0, size - 1), which is the same for
 *               either bmax, so the evaluation, gather, clearance and front-end entry points behave on a cloud-built map exactly as on
 *               the same occupancy given to isdf_set_map_u8 with the same bmin and res.
 * Deviations from the reference:
 *   - records with a NaN or Inf coordinate are skipped, from the bounds and the counts, and counted in points_skipped (undefined
 *     behaviour in the reference: NaN passes isInMap and (int)floor(NaN) becomes an address);
 *   - ISDF_ERR_INVALID for n < 1 or n >= 2^32, stride_bytes < 12 or not a multiple of 4, points not 4-byte aligned, res not finite
 *     and positive, a NULL pointer, no finite point, or a degenerate extent (an axis with X < 1: every point shares that coordinate;
 *     the reference allocates a zero-size grid and writes past it);
 *   - the size limits of isdf_set_map_u8 apply with its codes (X*Y*ceil(Z/32) < 2^31, Z <= 65535, the 1023-voxel pose window), and
 *     the message names the dimensions the cloud asked for.
 * Argument checks run before any device call; refused calls and CUDA failures behave as Conventions says. The result is the same bits
 * whatever the order of the points and through either entry point. The call counts its launches in isdf_stats.kernel_launches and
 * touches no other field. sta_threshold > 1 needs 4 bytes of device scratch per voxel during the call. */
int isdf_set_map_cloud(isdf_ctx *ctx, const void *points, int64_t n, int32_t stride_bytes, double res, int32_t sta_threshold);
/* the same with the points on ctx's device. Work before the call on cuda_stream is waited for: the call synchronises cuda_stream once
 * (the grid size depends on the bounds), builds the grid on ctx's own stream and returns when the map is set, so d_points may be
 * reused at once. */
int isdf_set_map_cloud_device(isdf_ctx *ctx, const void *d_points, int64_t n, int32_t stride_bytes, double res, int32_t sta_threshold,
                              void *cuda_stream);

typedef struct isdf_map_info {
    int32_t X, Y, Z, reserved_;
    double res, bmin[3], bmax[3];         /* bmax: the cloud's maximum for cloud maps (reference boundary_xyzmax); bmin + size*res otherwise */
    int64_t occupied_voxels;              /* popcount of the grid */
    int64_t points_used, points_skipped;  /* cloud maps only (0 otherwise); skipped = records with a non-finite coordinate */
} isdf_map_info;
/* any map, however it was set; ISDF_ERR_STATE without one */
int isdf_get_map_info(isdf_ctx *ctx, isdf_map_info *out);
/* the grid as 0 / 1 in the setters' layout (address ix*Y*Z + iy*Z + iz), n = X*Y*Z elements (ISDF_ERR_INVALID otherwise). The f64
 * form fills the reference's occupancy_map->grid_map directly (after createGridMap(bmin, bmax) with isdf_get_map_info's frame). The
 * grid is expanded on the device in bounded chunks. */
int isdf_get_map_u8(isdf_ctx *ctx, uint8_t *occ, int64_t n);
int isdf_get_map_f64(isdf_ctx *ctx, double *grid_map, int64_t n);

/* PCSmapManager::getPointsInAABB (pcs:148-170) on the device map; writes up to cap centres (cap x 3), returns count in *n */
int isdf_points_in_aabb(isdf_ctx *ctx, const double *centre, double half_extent, double *out_points, int cap, int *n);

/* The obstacle list of PlannerManager::generateTraj (plan_manager.cpp:232-254): for every waypoint in order, the occupied voxels of
 * box(wp + offset, half) that are not in box(previous wp, half) (PCSmapManager::getPointsInAABBOutOfLastOne, pcs:182-216),
 * de-duplicated by voxel. waypoints: nQ x 3 row-major. Writes up to cap centres in (first-including waypoint, voxel address)
 * order and the total in *n. If set_as_points != 0 the list also becomes the swept-volume point set (== isdf_set_points). */
int isdf_gather_obstacle_points(isdf_ctx *ctx, const double *waypoints, int nQ, double half_extent, const double *offset,
                                double *out_points, int cap, int *n, int set_as_points);

/* ---- discrete collision term: addTimeIntPenaltyParallel (hpp:432-554) with grad_cost_p (hpp:766-824) wired in */
/* ACCUMULATES into *cost, gradC (6N x 3 col-major), gradT (N) exactly like the reference's reference arguments. */
int isdf_eval_discrete(isdf_ctx *ctx, int N, const double *T, const double *coeffs,
                       double *cost, double *gradC, double *gradT);
/* device-resident variant: d_T (N), d_coeffs (18N) and d_out (19N+1 = [cost | gradC 18N | gradT N], OVERWRITTEN)
 * are device pointers on ctx's device; cuda_stream is a cudaStream_t (NULL = default stream). Asynchronous. */
int isdf_eval_discrete_device(isdf_ctx *ctx, int N, const double *d_T, const double *d_coeffs, double *d_out,
                              void *cuda_stream);

/* per-piece cost terms of the last discrete evaluation (n <= N doubles). With B independent trajectories concatenated into one
 * call (pieces b*N0 .. b*N0+N0-1 belong to trajectory b — the discrete term couples nothing across pieces, so a batch of
 * random restarts is simply a longer coefficient block) the cost of trajectory b is the sum of its N0 entries. */
int isdf_get_piece_costs(isdf_ctx *ctx, double *piece_cost, int n);

/* ---- batched optimiser callback on the device (SURVEY §8f row 1: MINCO on both sides of the hot loop) -------------------- */
/* B independent problems (random restarts, BASELINE configs[4]) in one call. Restates TrajOptimizer::costFunctionLmbm
 * (back_end_optimizer.hpp:358-430) with the time-integral term as the only penalty (use the per-problem host adapter
 * host/isdf_cost_callback.hpp when the swept-volume term is wanted: obstacle point sets are per trajectory):
 *   x_b = [tau (N0) | xi (3(N0-1), waypoint-major)] -> forwardT (hpp:214-241) -> MINCO_S3NU::setParameters (minco.hpp:433-513,
 *   banded LU :99-135) -> getEnergy + partials (:530-582) -> addTimeIntPenaltyParallel over the concatenated B*N0 pieces ->
 *   propogateGrad (:584-654) -> + rho*sum(T) -> backwardGradT / backwardGradP (hpp:283-330).
 * head / tail: 3x3 column-major (columns p, v, a), one pair shared by the batch (per_problem_bc = 0) or B pairs (= 1).
 * x: B x (4*N0-3) row-major; cost: B; grad: B x (4*N0-3). On failure every cost[b] is NaN. N0 <= 290.
 * Multi-GPU: shard by problem (each rank calls this with its own problems and isdf_set_shard(ctx, 0, 1)); no collective.
 * With per-problem obstacle point sets registered for the same B (isdf_set_points_batch) the callback is the LIVE composition of the
 * reference — swept-volume term (addSaftyPenaOnSweptVolumeParallel, hpp:386-391) then time-integral term (hpp:399-405) — for every problem,
 * each stage one launch over the whole batch (grid.y = problem). */
/* problem b owns the points [offsets[b], offsets[b+1]) of pts (offsets: B+1 ints, offsets[0] = 0; what plan_manager.cpp:232-254 builds per plan);
 * t* of every point starts at 0 and persists across evaluations like lastTstar. B = 0 switches the batched swept-volume term off again.
 * Persisted trajectory duration (updateTraj, swm:287-296): a trajectory of 300 s or longer is not taken; the search then scans the
 * duration of the last trajectory shorter than 300 s (0 if there was none). The batched callback keeps one such duration per problem
 * index b; isdf_eval_swept / _device / _given keep one of their own. They never share a value. All start at 0 when the context is
 * created and live as long as it: isdf_set_points and isdf_set_points_batch leave them alone, and registering a larger B keeps the
 * durations of problems 0 .. B_old-1 and starts the new problems at 0. */
int isdf_set_points_batch(isdf_ctx *ctx, int B, const int32_t *offsets, const double *pts);
int isdf_callback_batch(isdf_ctx *ctx, int B, int N0, const double *head, const double *tail, int per_problem_bc, double rho,
                        const double *x, double *cost, double *grad);
/* device-resident variant (all pointers on ctx's device, asynchronous on cuda_stream) */
int isdf_callback_batch_device(isdf_ctx *ctx, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc,
                               double rho, const double *d_x, double *d_cost, double *d_grad, void *cuda_stream);
/* the trajectories of the last batched callback: durations (B*N0), coefficient block (6*B*N0 x 3 column-major, piece b*N0+i),
 * jerk energies (B); any may be NULL */
int isdf_get_batch_trajectories(isdf_ctx *ctx, double *T, double *coeffs, double *energy);

/* ---- device-resident lock-step L-BFGS over the batched callback (SURVEY §8f row 2) ------------------------------------------------
 * B independent instances of the reference's patched LBFGS-Lite fork (utils/include/utils/lbfgs.hpp:480-830: Lewis-Overton bracketing that
 * returns on Armijo :290-430, cautious update + two-loop recursion :742-786, the fork's direction reset :788-811, stop tests :656-690; same
 * return codes :148-197) advanced together: every round is ONE isdf_callback_batch_device evaluation of all instances' requested points plus
 * one bookkeeping kernel; iterates and histories never leave the device. Each instance's iterates, counts and return code are bit-identical
 * to the sequential driver host/isdf_lbfgs.hpp run on the same callback. The reference's own driver is single-instance (and its live LMBM
 * shim non-re-entrant, lmbm/lmbm.cpp:4-6). */
typedef struct isdf_lbfgs_params {     /* lbfgs_parameter_t (lbfgs.hpp:40-142); with_tole_ls / cast_x_range off as in the shipped configs */
    int32_t mem_size;                  /* 1..64 */
    int32_t past, max_iterations, max_linesearch;
    int32_t max_rounds;                /* 0 = until every instance has stopped; otherwise a cap on batched evaluations. An instance still
                                          running when the cap ends the call stops as under max_iterations = its iterations so far: x and f
                                          are its last accepted iterate and its value (x0 and f(x0) before the first accepted iteration),
                                          ret is LBFGSERR_MAXIMUMITERATION (-1008), iterations and evaluations are its counts so far */
    int32_t reserved_;
    double g_epsilon, delta, min_step, max_step, f_dec_coeff, cautious_factor, machine_prec;
} isdf_lbfgs_params;
int isdf_lbfgs_default_params(isdf_lbfgs_params *p);   /* config_CappedCone.yaml:99-102: mem 16, past 10, min_step 1e-32, g_epsilon 0, delta 1e-6 */
/* x: B x (4*N0-3) in/out; f: B; ret / iterations / evaluations: B (any may be NULL); rounds: batched evaluations used (may be NULL).
 * head / tail / rho / per_problem_bc as isdf_callback_batch. On failure every f[b] is NaN (d_f too, when ctx and d_f are valid). */
int isdf_lbfgs_batch(isdf_ctx *ctx, int B, int N0, const double *head, const double *tail, int per_problem_bc, double rho,
                     const isdf_lbfgs_params *params, double *x, double *f, int32_t *ret, int32_t *iterations, int32_t *evaluations, int32_t *rounds);
/* device-resident variant (all pointers on ctx's device; returns when every instance has stopped — one 4-byte read per round) */
int isdf_lbfgs_batch_device(isdf_ctx *ctx, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc, double rho,
                            const isdf_lbfgs_params *params, double *d_x, double *d_f, int32_t *d_ret, int32_t *d_iterations, int32_t *d_evaluations,
                            int32_t *rounds, void *cuda_stream);

/* ---- mid-end: warm start of the back end from front-end paths (PlannerManager::generateTraj, plan_manager.cpp:202-289) --------------
 * The reference turns an A* path into the back end's starting point in two steps: it picks waypoints from the path, then OriTraj::getOriTraj
 * (mid_end.cpp:3-94) runs an L-BFGS over a MINCO trajectory that pulls it towards them. Its solution opt_x is the x that optimize_traj_lmbm
 * starts from (back_end_optimizer.cpp:117). Here both steps run for B paths at once; a solution goes straight into isdf_lbfgs_batch.
 * Definition
 *   Waypoints      plan_manager.cpp:204-245 for each path of size S: gap = ceil(parlength / res) (parlength: traj_parlength, 3.0 in the
 *                  reference, :153; res: the map's resolution); while gap >= S - 1: parlength /= 1.5 (FP64), recompute gap; Q = path[gap],
 *                  path[2 gap], ... for indices < S - 1; N = |Q| + 1. head = [path.front(), 0, 0], tail = [path.back(), 0, 0] (3x3 column-major
 *                  as isdf_callback_batch takes them). Deviation: for S = 1 or 2 the reference never terminates (the loop divides until gap is
 *                  0, then ind += 0); here N = 1 and no waypoints. The attitude and acceleration lists built in the same loop only feed the
 *                  mid-end's addTimeIntPenalty, which is never called (mid_end.hpp:424-592), so they are not inputs.
 *   Cost           OriTraj::costFunction (mid_end.hpp:262-304) on x = [tau (N0) | xi (3(N0-1), waypoint-major)], the back end's layout:
 *                  T = forwardT(tau), MINCO -> jerk energy E and its partials; then, for waypoint i = 0..N0-2 (addPosePenalty, :201-260),
 *                  piece i + 1 evaluated at s = T_{i+1} * (1 / K), K = isdf_config.integral_intervs (integralRes, :323) — NOT the junction
 *                  where xi_i sits:
 *                    d = p(s) - Q_i, n = sqrt((d0 d0 + d1 d1) + d2 d2), c_i = (n n) n, g = (3 (n n)) (d / n),
 *                    gradC rows of piece i + 1 += w (beta0 (x) g), gradT(i + 1) += w (c_i (alpha (g . v(s)))), alpha = 1 / K;
 *                  each term only when c_i > 0 (grad_cost_dir returns cost > 0, :198), so d = 0 adds nothing.
 *                  cost = ((E + w c_1) + w c_2) + ... + rho sum(T) (every sum left to right), gradT += rho, then propogateGrad and
 *                  backwardGradT / backwardGradP exactly as the back end's callback.
 *   Quirk, kept    the T entry is multiplied by the cost c_i: the tau gradient is not the derivative of the cost.
 *   Arithmetic     IEEE operations only (no pow): glibc's pow(|d|, 3) is not correctly rounded and CUDA's differs from it, so no formula is
 *                  bit-equal to the reference on both sides. Host (host/isdf_midend.hpp) and device agree bit for bit; the difference from
 *                  the reference's pow form is about one ulp per term (DESIGN §3.10).
 *   Optimiser      getOriTraj: x starts at [backwardT(init_time) for every piece | the waypoints]; L-BFGS as isdf_lbfgs_batch with
 *                  params.lbfgs (mid_end.cpp:48-54: mem 16, past 10, min_step 1e-32, g_epsilon 0, delta 1e-6, max_iterations 100000) and
 *                  the progress callback earlyExit (mid_end.hpp:613-631): LBFGS_CANCELED (2) once k > cancel_after after a successful line
 *                  search. ret >= 0 is getOriTraj's success (plan_manager.cpp:277 runs the back end only then). The final T and coeffs are
 *                  forwardT + MINCO of the returned x, whatever ret is. f is the cost at the returned x; where the reference's
 *                  lbfgs_optimize returns from its direction-norm test without writing f (lbfgs.hpp:814-817, code -1012), f is still
 *                  the cost at x. A plan still running when params.lbfgs.max_rounds ends the call reports ret = -1008
 *                  (LBFGSERR_MAXIMUMITERATION, so not a success) with x, f, T and coeffs from its last accepted iterate.
 * Each problem's result is bit-identical to the sequential host driver on the same problem, alone or inside a batch.
 * The mid-end needs neither a map nor a shape. It has its own device buffers: it leaves isdf_get_batch_trajectories, the swept-volume
 * t* and persisted durations, the discrete work-item schedule and every isdf_stats field but kernel_launches as they were.
 * Errors: ISDF_ERR_INVALID for a NULL argument, B < 1, N0 < 1, a parameter out of range or a non-zero reserved_; ISDF_ERR_UNSUPPORTED for
 *   N0 > 290; ISDF_ERR_STATE on a sharded context (shard by problem, as isdf_callback_batch). On failure every cost[b] / f[b] is NaN. */
/* waypoint selection, host-only (needs no context or GPU). paths: B paths back to back, path b in rows [path_off[b], path_off[b+1]) of
 * path_xyz (what isdf_frontend_path_batch returns; every path at least one node). Writes the waypoints of plan b to rows
 * [wp_off[b], wp_off[b+1]) of waypoints (cap x 3) and its N to pieces[b]. ISDF_ERR_INVALID when the total exceeds cap (wp_off and pieces
 * are still written), for res or parlength not finite and positive, or for offsets that do not start at 0 and increase. */
int isdf_path_waypoints(int B, const int32_t *path_off, const double *path_xyz, double res, double parlength, int cap,
                        double *waypoints, int32_t *wp_off, int32_t *pieces);
typedef struct isdf_midend_params {
    double weight_pr;        /* weightPR (mid_end.hpp:315; yaml weight_pr 1000); >= 0 */
    double rho;              /* rho_mid_end (yaml 200); finite */
    double init_time;        /* inittime (yaml 2.5): every piece's starting duration (plan_manager.cpp:263); > 0 */
    int32_t cancel_after;    /* earlyExit: LBFGS_CANCELED once k > cancel_after (8000); 0 = never */
    int32_t reserved_;       /* must be 0 */
    isdf_lbfgs_params lbfgs; /* mid_end.cpp:48-54; the other fields keep their lbfgs.hpp defaults */
} isdf_midend_params;
int isdf_midend_default_params(isdf_midend_params *p);
/* one evaluation of the cost for B problems: waypoints B x (N0-1) x 3; x, grad B x (4*N0-3); cost B. head / tail / per_problem_bc as
 * isdf_callback_batch. */
int isdf_midend_callback_batch(isdf_ctx *ctx, int B, int N0, const double *head, const double *tail, int per_problem_bc,
                               const isdf_midend_params *p, const double *waypoints, const double *x, double *cost, double *grad);
/* getOriTraj for B problems: x (out, B x (4*N0-3)) starts at [backwardT(init_time) | waypoints] and returns the solution; f: B final costs.
 * T (B*N0) and coeffs (6*B*N0 x 3 column-major, piece b*N0+i: the layout of isdf_get_batch_trajectories) are the final trajectories.
 * Any of T / coeffs / ret / iterations / evaluations / rounds may be NULL. */
int isdf_midend_batch(isdf_ctx *ctx, int B, int N0, const double *head, const double *tail, int per_problem_bc,
                      const isdf_midend_params *p, const double *waypoints, double *x, double *T, double *coeffs,
                      double *f, int32_t *ret, int32_t *iterations, int32_t *evaluations, int32_t *rounds);
/* device-resident variant: every array on ctx's device (rounds on the host); runs on cuda_stream and returns when every instance has
 * stopped. On failure d_f is filled with NaN when ctx and d_f are valid. */
int isdf_midend_batch_device(isdf_ctx *ctx, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc,
                             const isdf_midend_params *p, const double *d_waypoints, double *d_x, double *d_T, double *d_coeffs,
                             double *d_f, int32_t *d_ret, int32_t *d_iterations, int32_t *d_evaluations, int32_t *rounds, void *cuda_stream);

/* ---- trajectory clearance check: is a trajectory collision-free over the WHOLE map, and by how much? ------------------------------
 * The reference has no working counterpart (SweptVolumeManager::isTrajCollide, swm:759-767, always returns false), and the cost terms
 * cannot stand in for it: the hinge is smoothed and positive only inside safety_hor, the swept-volume term only sees the gathered obstacle
 * list, the discrete term only the bd/2 box at its own sample spacing.
 * Definition:
 *   Samples. N pieces (T, coeffs in the layout of isdf_eval_discrete); piece i has K_c + 1 pose samples at local times j * step,
 *     step = T_i * (1 / K_c), j = 0..K_c — the discrete path's pose: position of the piece polynomial, flatness quaternion, R = quat_rot(q).
 *     Junction times are sampled twice (last sample of one piece, first of the next), as in the integral loop. The check is SAMPLED: nothing
 *     is certified between two samples T_i / K_c apart (isdf_trajectory_certify below closes those gaps).
 *   Candidates of a sample: the occupied map voxels whose centre c (getGridCubeCenter) satisfies |R^T (c - x)|_inf <= H,
 *     H = half_bd + reach, half_bd = kernel_size * occupancy_resolution / 2 (a strict > on any axis excludes, as hpp:800). Only voxels of
 *     the map count: a window reaching past the map border is cut off there (no projInMap clamping).
 *   clear(s) = min(reach, min over candidates of sdf(R^T (c - x))), sdf = getonlySDF of the shape (analytic: the closed form of
 *     isdf_shape_query(..., ISDF_QUERY_SDF); mesh: s * dist in the context's sign mode).
 *   Witness: the address ix*Y*Z + iy*Z + iz of the candidate realising the minimum when it is < reach (the smallest address among exact
 *     ties), otherwise -1.
 *   For SDFs that are true distances (exact-sign meshes, Ball) the H box loses nothing: every voxel closer than reach to a robot that fits
 *     in the bd/2 box lies inside it. For the other analytic shapes and winding-sign meshes the box is part of the definition.
 *   Trajectories: pieces b*N0 .. b*N0+N0-1 form trajectory b (N0 = 0: one trajectory of all N pieces). A sample's trajectory time is the
 *     sum of the T of the earlier pieces of its trajectory, added in ascending order, plus j * step.
 *   Summary per trajectory: min_clearance; the first sample in (piece, j) order attaining it — piece_min (index WITHIN the trajectory),
 *     sample_min (= j), t_min (trajectory time), voxel_min (its witness); first_hit = trajectory time of the first sample with
 *     clear < margin (-1 if none); colliding_samples = samples with clear < margin; collision_free = (colliding_samples == 0).
 *   A sample whose pose is not finite has clearance NaN, counts as colliding, and makes its trajectory's min_clearance NaN.
 * Results are deterministic: bit-identical run to run, through either entry point, and for a trajectory checked alone or inside a batch.
 * Errors: ISDF_ERR_INVALID for bad parameters (K_c < 1, reach <= 0 or not finite, margin > reach, N % N0 != 0) and for a window wider than
 * 1023 voxels per axis (2 H sqrt(3) / res + 4 > 1023); ISDF_ERR_STATE without a map or a shape; ISDF_ERR_UNSUPPORTED on a sharded context
 * (isdf_set_shard world > 1). On failure every summary has min_clearance NaN and collision_free 0.
 * Statistics: the call counts its launches in isdf_stats.kernel_launches and touches no other field. */
typedef struct isdf_clearance_params {
    int32_t samples_per_piece;   /* K_c >= 1 */
    int32_t pieces_per_traj;     /* N0; 0 = one trajectory of N pieces; else N % N0 == 0 */
    double reach;                /* > 0, finite: search bound and cap of every reported clearance */
    double margin;               /* a sample collides when clear < margin; margin <= reach */
} isdf_clearance_params;

typedef struct isdf_clearance_summary {
    double min_clearance, t_min, first_hit;        /* first_hit = -1 when collision-free */
    int64_t voxel_min;                             /* -1 when nothing lies within reach */
    int32_t piece_min, sample_min, colliding_samples, collision_free;
} isdf_clearance_summary;

/* K_c = integral_intervs of the default config, N0 = 0, reach = margin = safety_hor of the default config */
int isdf_clearance_default_params(isdf_clearance_params *p);
/* host buffers: sample_clearance / sample_voxel (N*(K_c+1), sample i*(K_c+1)+j) may be NULL; summary: N/N0 entries (1 for N0 = 0) */
int isdf_trajectory_clearance(isdf_ctx *ctx, int N, const double *T, const double *coeffs, const isdf_clearance_params *p,
                              double *sample_clearance, int64_t *sample_voxel, isdf_clearance_summary *summary);
/* device-resident variant: every pointer on ctx's device (none may be NULL), asynchronous on cuda_stream (NULL = default stream) */
int isdf_trajectory_clearance_device(isdf_ctx *ctx, int N, const double *d_T, const double *d_coeffs, const isdf_clearance_params *p,
                                     double *d_sample_clearance, int64_t *d_sample_voxel, isdf_clearance_summary *d_summary,
                                     void *cuda_stream);

/* ---- continuous clearance certificate: is a trajectory clear at EVERY time, not only at its samples? ---------------------------
 * The clearance check above is sampled; this call closes the gaps between the samples with a proven motion bound.
 * Definition. Inputs and parameters are the clearance check's (T, coeffs, K_c, N0, reach, margin) with 0 <= margin < reach. One verdict
 * per trajectory:
 *   CERTIFIED (1)   for every time t of the trajectory and every occupied voxel centre c of the map, the Euclidean distance from c to
 *                   the robot posed at t is at least margin;
 *   COLLIDING (-1)  some evaluated pose sample has clear < margin (or a non-finite pose);
 *   UNDECIDED (0)   neither was established within the refinement budget.
 *   Obstacles are voxel CENTRES, as in the clearance check and the cost terms. Callers who want whole voxel cubes cleared add
 *   res * sqrt(3) / 2 to margin.
 * Mechanism.
 *   The initial samples are exactly the clearance check's K_c + 1 samples per piece (bit-identical clearances). Each piece is divided
 *   into K_c intervals [ta, tb] of local time (the last one ends at T_i); intervals never cross a junction. For an interval with
 *   endpoint clearances c_a, c_b (capped at reach), D_e bounds the largest displacement of any body point over the interval from its
 *   position at endpoint e: sup_{t in [ta,tb]} sup_{p in body} |x(t) + R(t) p - x(t_e) - R(t_e) p|. Then
 *   lb = max(c_a - D_a, c_b - D_b) is a lower bound of the clearance at every t of the interval, and the interval is SAFE when
 *   lb >= margin. An interval that is not safe is split at its midpoint ta + 0.5 (tb - ta), and the midpoint gets a new clearance
 *   sample. Splitting stops when the trajectory has a colliding sample (it is COLLIDING; its remaining intervals are dropped), at
 *   max_depth, or when the trajectory's new samples would exceed max_samples_per_traj (intervals earlier in time get the samples
 *   first). Intervals left in the last two cases are undecided.
 *   Motion bound: D_e = P_e + r Q_e + eps_e.
 *     P_e   per axis, the piece polynomial re-expanded about t_e (Taylor coefficients d_1..d_5) gives sum |d_k| h^k, h = tb - ta;
 *           P_e is the Euclidean norm of the three axis bounds.
 *     Q_e   >= sup ||R(t) - R(t_e)||_2, in interval arithmetic: v and a enclosed over the interval in Taylor form;
 *           zu = a + dh_over_m (1 + cp sqrt(|v|^2 + veps)) v + g e_z, z = zu / |zu|; R(z) in the closed form of the zero-yaw attitude,
 *           rows [1 - zx^2/(1+zz), -zx zy/(1+zz), zx], [-zx zy/(1+zz), 1 - zy^2/(1+zz), zy], [-zx, -zy, zz] (quat_rot(flat_quat_only)
 *           up to rounding); Q_e = Frobenius norm of the enclosure of R(z(t)) - R(z(t_e)). Q_e = +inf (the interval must be refined)
 *           when the lower bound of |zu| or of 1 + zz is not positive.
 *     r     body radius about the body origin: 0 for Ball and Point (rotation-invariant bodies); for Box the largest corner norm of the
 *           transformed box; for a mesh the largest corner norm of its body-frame AABB.
 *     eps_e pose pad 1e-10 (1 + A_e + 2H + (r + 2H) kappa_e / delta_e), H = half_bd + reach, A_e = sum over axes and k of |c_k| |t_e|^k,
 *           kappa_e = (|a| + dh_over_m kap |v| + g) / |zu| and delta_e = 1 + zz at t_e: it covers the difference between this closed
 *           form and the pose and SDF the scan computes in round-to-nearest with FMA contraction (DESIGN §3.11).
 *     Every operation of the bound is rounded outward.
 *   Why this is sound: for a body point q(t), |c - q(t)| >= |c - q(t_e)| - D_e. Capping at reach and leaving out voxels outside the H box
 *   only lower c_e. This needs an SDF that is a true Euclidean distance outside the body, and a body inside the half_bd box (so that the
 *   H box loses no voxel within reach); the call checks both.
 * Supported shapes: Ball with 0 <= radius <= half_bd, Point, Box whose rotation is orthonormal to 1e-12 and whose corners lie in
 *   [-half_bd, half_bd]^3, exact-sign meshes (ISDF_MESH_SIGN_EXACT) whose body-frame AABB lies in [-half_bd, half_bd]^3. Everything else
 *   (other analytic shapes, winding-sign meshes, a robot wider than half_bd) is ISDF_ERR_UNSUPPORTED.
 * Summary per trajectory: verdict; lower_bound = the minimum of lb over the final leaf intervals, a proven lower bound of the continuous
 *   clearance whatever the verdict (never above reach); min_clearance, t_min (trajectory time) and voxel_min over every evaluated sample
 *   (ties: earliest time, then smallest witness address); first_hit = trajectory time of the earliest evaluated sample with
 *   clear < margin, or -1; samples (evaluated: N0 (K_c + 1) plus the new ones), undecided_intervals, depth (deepest leaf level).
 * Results are deterministic run to run, identical through both entry points, and a trajectory's result is bit-identical alone or
 * inside a batch (per-trajectory budgets, order-preserving compaction).
 * Device work per round: one scan launch over the round's new samples, one interval pass (two kernels), one 4-byte read; at most
 *   max_depth + 1 rounds. Device buffers are owned by the context and grow on demand.
 * Errors: ISDF_ERR_INVALID for the clearance check's bad parameters, margin < 0, margin >= reach, max_depth outside [0, 64],
 *   max_samples_per_traj < 0, a non-zero reserved_, sizes beyond 31-bit indexing, NULL pointers; ISDF_ERR_STATE without a map or a
 *   shape; ISDF_ERR_UNSUPPORTED for an unsupported shape and on a sharded context. On failure every summary has verdict 0 and
 *   lower_bound / min_clearance NaN.
 * The call counts its launches in isdf_stats.kernel_launches and touches no other field; it leaves the discrete schedule, the
 * swept-volume state, the mid-end buffers and the batch trajectories as they were. */
typedef struct isdf_certify_params {
    isdf_clearance_params clearance;  /* K_c, N0, reach, margin as the clearance check, with 0 <= margin < reach */
    int32_t max_depth;                /* splits per initial interval, 0..64 */
    int32_t max_samples_per_traj;     /* new samples per trajectory, >= 0 */
    int32_t reserved_[2];             /* must be 0 */
} isdf_certify_params;

typedef struct isdf_certify_summary {
    double lower_bound, min_clearance, t_min, first_hit;   /* first_hit = -1 when no evaluated sample collides */
    int64_t voxel_min;                                     /* witness of the minimum sample, -1 when nothing lies within reach */
    int32_t verdict;                                       /* 1 CERTIFIED, -1 COLLIDING, 0 UNDECIDED */
    int32_t samples, undecided_intervals, depth;
} isdf_certify_summary;

/* K_c = integral_intervs and N0 = 0 as isdf_clearance_default_params, margin = safety_hor, reach = 2 safety_hor, max_depth 16,
 * max_samples_per_traj 2048 (DESIGN §3.11) */
int isdf_certify_default_params(isdf_certify_params *p);
/* host buffers; summary: N/N0 entries (1 for N0 = 0) */
int isdf_trajectory_certify(isdf_ctx *ctx, int N, const double *T, const double *coeffs, const isdf_certify_params *p,
                            isdf_certify_summary *summary);
/* device-resident variant: d_T, d_coeffs, d_summary on ctx's device; runs on cuda_stream (NULL = default stream) and returns when the
 * summaries are written (the round loop reads 4 bytes per round) */
int isdf_trajectory_certify_device(isdf_ctx *ctx, int N, const double *d_T, const double *d_coeffs, const isdf_certify_params *p,
                                   isdf_certify_summary *d_summary, void *cuda_stream);

/* ---- certified swept volume: the region a trajectory sweeps, as a signed distance field with a proven enclosure, and its surface ----
 * Replaces SweptVolumeManager::calculateSwept / sw_calculate::calculation (a local descent per cube corner from random seeds, so an upper
 * bound that can miss a branch of the trajectory) and the standalone use of getSDFofSweptVolume (PlannerManager::geneWall).
 * Definition. One trajectory of N pieces (T, coeffs in the layout of isdf_eval_discrete); no map is needed. Trajectory time runs over
 *   [0, sum T]; piece start times are summed left to right. The pose at a time is the clearance check's (and the certificate's).
 *   SV(p) = min over t of sd(R(t)^T (p - x(t))), sd = getonlySDF of the context's shape (negative inside).
 * Supported shapes: those whose SDF is a signed Euclidean distance — Ball (radius >= 0), Point, Box whose rotation is orthonormal to
 *   1e-12, exact-sign meshes (ISDF_MESH_SIGN_EXACT). There is no half_bd condition. Everything else is ISDF_ERR_UNSUPPORTED.
 *   r_rot = the certificate's r (0 for Ball and Point); r_body = the body's bounding radius about its origin (the Ball's radius, the Box's
 *   largest corner norm, the mesh's largest body-frame AABB corner norm, 0 for Point).
 * Per point p, in level-synchronous rounds (the result depends on nothing but p):
 *   1. Initial intervals: K per piece, exactly the certificate's (local time j T_i (1/K), the last one ending at T_i), with the
 *      certificate's motion bounds D_a, D_b (r = r_rot, H = band): for these shapes sd_t(p) >= sd_e(p) - D_e on the interval.
 *   2. Sphere cull: an interval with max_e(|p - x(t_e)| - r_body - D_e) >= band (rounded down) is dropped without an SDF evaluation.
 *   3. sd at the endpoints of the kept intervals. hi = min(band, smallest value); t* = the earliest time attaining it, -1 if hi == band.
 *      Each interval has lb = max(sd_a - D_a, sd_b - D_b).
 *   4. Each round, with hi as it stood at the round's start: an interval with lb < hi - tol is split at ta + 0.5 (tb - ta) and the
 *      midpoint is evaluated; the others become leaves. Splitting stops at max_depth or when the point's new samples would exceed
 *      max_samples_per_point (earlier intervals get the samples first); intervals left then are undecided leaves.
 *   5. lower = min(hi, min leaf lb). The point is decided iff lower >= hi - tol (which covers lower >= band).
 *   Outputs: value = hi (an attained SDF value, capped at band), lower, t* (trajectory time), decided. lower <= SV(p) <= value up to the
 *   certificate's rounding pad (DESIGN §3.12). Results are bit-identical run to run, through every entry point, and for a point queried
 *   alone or as a grid node.
 * Grid: nodes (not cell centres) at bmin + (i, j, k) res, each coordinate computed as bmin[a] + (double) i * res; address i*Y*Z + j*Z + k
 *   as the map's. X, Y, Z >= 2 and X*Y*Z < 2^31.
 * Mesh: marching tetrahedra on the node values, value < 0 = inside.
 *   Cells are split into the 6 Kuhn tetrahedra {000, e_a, e_a + e_b, 111}, (a, b, c) the permutations of (x, y, z) in lexicographic
 *   order; the split is the same in every cell, so faces match and no ambiguity table is needed.
 *   Vertices lie on the 7 edge directions of a node (+x, +y, +z, +x+y, +x+z, +y+z, +x+y+z), one per crossed edge (exactly one endpoint
 *   inside), numbered in (node address, direction) order and shared by every tetrahedron that uses the edge. Position per coordinate:
 *   s = f0 / (f0 - f1), v = p0 + s (p1 - p0), each operation rounded to nearest (no contraction); vtime = t* of the endpoint with the
 *   smaller |value|, the first endpoint on ties. That endpoint may be capped at band (t* = -1), so vtime is -1 where band is smaller
 *   than the inside endpoint's |value| (possible when band < res).
 *   Triangles in (cell address, tetrahedron, local) order. Per tetrahedron (v0..v3 of the list above, E(x, y) = the vertex on edge x-y):
 *     one vertex i on its own side: (i, j, k, l) = the even permutation of (0, 1, 2, 3) starting with i — (0,1,2,3), (1,0,3,2),
 *       (2,3,0,1), (3,2,1,0) — and the triangle E(i,j), E(i,k), E(i,l) when i is inside, E(i,j), E(i,l), E(i,k) when it is outside;
 *     two inside {i < j}, two outside {k < l}, k and l swapped when (i, j, k, l) is an odd permutation: E(i,l), E(j,l), E(j,k) and
 *       E(i,l), E(j,k), E(i,k);
 *     tetrahedra of odd permutations (a, b, c) — (x,z,y), (y,x,z), (z,y,x) — swap the last two vertices of each triangle.
 *   Normals (counter-clockwise) point toward increasing value; the surface of a field whose inside stays clear of the grid border is
 *   closed and consistently oriented.
 * Errors: ISDF_ERR_INVALID for NULL pointers, N < 1, non-finite or non-positive T, non-finite coeffs or points, a parameter out of range
 *   (K < 1, tol <= 0, band <= tol, max_depth outside [0, 64], max_samples_per_point < 0, non-zero reserved_), a bad grid, or a cap too
 *   small (*nV / *nF still report the sizes needed); ISDF_ERR_STATE without a shape; ISDF_ERR_UNSUPPORTED for an unsupported shape and on
 *   a sharded context. On failure every value / lower / tstar is NaN and decided 0 (the mesh call: V and vtime NaN up to the caps).
 * State: the calls count their launches in isdf_stats.kernel_launches and touch no other field. They leave the swept-volume term's t* and
 *   persisted durations, the discrete schedule, the clearance / certificate buffers, the mid-end buffers and the batch trajectories as
 *   they were. Device buffers are owned by the context and grow on demand; a grid call holds one interval list of 64 * (max(N K, 2 M) +
 *   2 M) bytes per resident warp (M = max_samples_per_point). */
typedef struct isdf_swept_params {
    int32_t samples_per_piece;       /* K >= 1: initial intervals per piece */
    int32_t max_depth;               /* splits per initial interval, 0..64 */
    int32_t max_samples_per_point;   /* new samples per point, >= 0 */
    int32_t reserved_;               /* must be 0 */
    double tol;                      /* > 0: a point is decided when lower >= value - tol */
    double band;                     /* > tol: cap of every reported value */
} isdf_swept_params;

typedef struct isdf_swept_grid {
    double bmin[3];                  /* the node (0, 0, 0) */
    double res;                      /* > 0: node spacing */
    int32_t X, Y, Z;                 /* >= 2 each, X*Y*Z < 2^31 */
    int32_t reserved_;               /* must be 0 */
} isdf_swept_grid;

typedef struct isdf_swept_info {     /* the last grid or mesh call */
    int64_t nodes, bricks, bricks_culled;   /* bricks of 4^3 nodes; culled: no interval reaches below band (no SDF evaluation) */
    int64_t sdf_evals, undecided;           /* SDF evaluations over every node; nodes not decided */
    int32_t deepest, reserved_;             /* deepest leaf level */
    double prep_ms, cull_ms, refine_ms, mesh_ms;   /* device time per stage (CUDA events on the call's stream); mesh_ms 0 for a grid call */
} isdf_swept_info;

/* K = integral_intervs, band = 2 safety_hor, tol = occupancy_resolution / 100 of the default config, max_depth 16,
 * max_samples_per_point 512 (DESIGN §3.12) */
int isdf_swept_default_params(isdf_swept_params *p);
/* n points (n x 3, host); value (n) required, lower / tstar / decided (n each) may be NULL */
int isdf_swept_volume_sdf(isdf_ctx *ctx, int N, const double *T, const double *coeffs, const isdf_swept_params *p, int n,
                          const double *pts, double *value, double *lower, double *tstar, uint8_t *decided);
/* the field at every grid node (X*Y*Z each, host); value required, the rest and info may be NULL */
int isdf_swept_volume_grid(isdf_ctx *ctx, int N, const double *T, const double *coeffs, const isdf_swept_params *p,
                           const isdf_swept_grid *grid, double *value, double *lower, double *tstar, uint8_t *decided,
                           isdf_swept_info *info);
/* device-resident variant: d_T, d_coeffs and the outputs on ctx's device; runs on cuda_stream (NULL = default stream) and returns when
 * the field is written (the trajectory is checked on the host and the brick lists are sized with one 8-byte read) */
int isdf_swept_volume_grid_device(isdf_ctx *ctx, int N, const double *d_T, const double *d_coeffs, const isdf_swept_params *p,
                                  const isdf_swept_grid *grid, double *d_value, double *d_lower, double *d_tstar, uint8_t *d_decided,
                                  isdf_swept_info *info, void *cuda_stream);
/* the surface {SV = 0} of the grid's field: V (cap_v x 3), vtime (cap_v), F (cap_f x 3, vertex indices), sizes in *nV / *nF */
int isdf_swept_volume_mesh(isdf_ctx *ctx, int N, const double *T, const double *coeffs, const isdf_swept_params *p,
                           const isdf_swept_grid *grid, int64_t cap_v, int64_t cap_f, double *V, double *vtime, int32_t *F,
                           int64_t *nV, int64_t *nF, isdf_swept_info *info);

/* ---- multi-GPU reduction through NVLink / NVSwitch peer memory (optional; ncclAllReduce over the same 19N+1 doubles is the
 * library alternative). One process per GPU. Sequence on every rank:
 *   isdf_set_shard(ctx, rank, world); isdf_peer_export(ctx, world, max_doubles, h) -> all-gather the 64-byte handles ->
 *   isdf_peer_connect(ctx, world, rank, handles, fuse) -> barrier -> evaluations ... -> barrier -> isdf_peer_disconnect(ctx).
 * With fuse != 0 every sharded isdf_eval_discrete* / isdf_eval_swept* call ends with the exchange inside the evaluation's last
 * kernel (discrete: the same CTA that finishes the rank's vector pushes it to the peers), so `d_out` / the accumulated host
 * results are the ALL-RANK sums, added in rank order: bit-identical on every rank. All ranks must issue the same sequence of
 * evaluations. A rank that never arrives makes the others time out (~2 s) and isdf_peer_status() report it; nothing hangs. */
int isdf_peer_export(isdf_ctx *ctx, int world, int max_doubles, unsigned char *handle64);
int isdf_peer_connect(isdf_ctx *ctx, int world, int rank, const unsigned char *handles /* world x 64 */, int fuse_into_eval);
int isdf_peer_allreduce_device(isdf_ctx *ctx, double *d_vec, int n, void *cuda_stream);   /* stand-alone, in place */
int isdf_peer_status(isdf_ctx *ctx);
int isdf_peer_disconnect(isdf_ctx *ctx);

/* ---- front end: attitude-kernel collision checks (SURVEY §8f row 4) -------------------------------------------------------- */
/* BasicShape::initShape's kernel branch (Shape.hpp:405-461): one kernel_size^3 occupancy kernel of the robot per (roll, pitch)
 * attitude, voxel set when getonlySDF(pos, Rx(roll)*Ry(pitch)) <= max(front_end_safeh, occupancy_resolution/2). Returns the
 * attitude grid size (sw_manager.hpp:135-136); at most 128 attitudes, kernel_size odd and <= 29. Call again after changing
 * the shape. */
int isdf_frontend_build_kernels(isdf_ctx *ctx, const isdf_kernel_config *kc, int *xkernel_size, int *ykernel_size);
/* the kernels as booleans, [attitude i*ykernel_size+j][a*ks*ks + b*ks + c] (Shape.hpp:453), n = xk*yk*ks^3 bytes */
int isdf_frontend_get_kernels(isdf_ctx *ctx, uint8_t *out, int n);
/* kernelConv<true> (sw_manager.hpp:821-846) for EVERY voxel and EVERY attitude: masks[4*voxel .. 4*voxel+3] is a 128-bit set,
 * bit i*ykernel_size+j = 1 when attitude (i,j) is collision-free with the robot centred on that voxel (voxel = ix*Y*Z+iy*Z+iz).
 * Cells outside the map count as free, like the reference's inflated map kernel (PCSmap_manager.h:46-78). */
int isdf_frontend_feasibility(isdf_ctx *ctx, uint32_t *masks /* X*Y*Z*4, host */);
int isdf_frontend_feasibility_device(isdf_ctx *ctx, uint32_t *d_masks, void *cuda_stream);
/* checkKernelValue (sw_manager.hpp:914-941) for n queries: voxel index (n x 3), father (roll, pitch) in degrees (n x 2) ->
 * child (roll, pitch) = the first collision-free attitude in visit_kernels_by_distance's order (level pose, then BFS from the
 * father's attitude, sw_manager.hpp:852-913); ok[q] = 0 when no attitude fits (child = father). */
int isdf_frontend_check_batch(isdf_ctx *ctx, int n, const int32_t *ind, const double *father_roll_pitch,
                              double *child_roll_pitch, uint8_t *ok);

/* ---- front-end path search: replaces AstarPathSearcher::AstarPathSearch + getPath / getastarSE3Path (front_end_Astar.hpp:197-402) ----
 * Definition
 *   Traversable(v) v is in the map, not occupied, and its isdf_frontend_feasibility mask is not zero (some attitude fits; checkKernelValue's
 *                  visit_kernels_by_distance tries every attitude, swm:852-913).
 *   Source s, target t  getGridIndex (grid:135-175) of the start and of the goal; both must pass isInMap (bmin <= p <= bmax on every axis).
 *   Field g        g(s) = 0. For v != s, g(v) is the minimum, over 26-connected paths s = v0, v1, ..., vk = v whose nodes v1..vk are all
 *                  traversable, of the left-to-right FP64 sum of the edge costs sqrt((double)(di^2 + dj^2 + dk^2)); +inf where no path
 *                  exists. s itself need not be traversable. FP addition of a positive cost is monotone, so the minimum does not depend on
 *                  any processing order and a textbook FP64 Dijkstra computes the same bits. The field is exact on EVERY voxel: the
 *                  relaxation is label-correcting and runs until no value changes.
 *   Parent(v)      for v != s with g(v) < inf: among the 26 neighbours u with g(u) + w(u, v) == g(v) in FP64 (such a u is traversable or
 *                  is s), the first in the reference's offset order u = v + (i, j, k), i, j, k = -1..1, i outermost (front_end_Astar.hpp:207-211).
 *   Path to t      the parents from t back to s, reversed: node 0 is s, the last node is t; coordinates are cube centres (getGridCubeCenter).
 *                  Found iff g(t) < inf (t traversable, or t == s: a one-node path, even on an occupied voxel); the cost is g(t). No path
 *                  is not an error: found = 0, cost +inf and a one-node path (the start).
 *   Attitudes      node 0 has (roll, pitch) = (0, 0) (GridNode's defaults); node m + 1 has checkKernelValue(attitude of node m, node m + 1):
 *                  isdf_frontend_check_batch applied as a chain along the returned path.
 * Deviations from the reference, on purpose: its open set keeps the stale key of an improved open node (:324-333) and its heuristic is
 *   inflated by 1.001 (:172-187), so its cost is >= the optimum and depends on pop order; here the path is the exact shortest one. Its
 *   AstarGetSucc overwrites a neighbour's attitude on every expansion that looks at it (:227-229), so the attitude getastarSE3Path reports
 *   can come from a node that is not the path father; here the attitudes are replayed father to child along the returned path.
 * Batch: one start and B goals (candidate goals, or restarts sharing a start). The field is built once per call; every goal's result is
 *   bit-identical to a call with that goal alone, and results are bit-identical run to run and through either entry point.
 * Outputs: the B paths back to back, path b in rows [offsets[b], offsets[b+1]) of path_xyz (cap x 3) and path_roll_pitch (cap x 2,
 *   degrees; may be NULL); costs and found: B each. The single-goal call reports its length in *n.
 * Errors: ISDF_ERR_STATE without a map or without front-end kernels (isdf_frontend_build_kernels; again after a shape change);
 *   ISDF_ERR_INVALID for a NULL pointer, B < 1, a non-finite start or goal, a start or goal outside the map, non-zero reserved parameters,
 *   or cap smaller than the total path length (then *n / offsets still report the lengths needed); ISDF_ERR_UNSUPPORTED on a sharded
 *   context (isdf_set_shard world > 1).
 * State: every call rebuilds the traversability grid and the field from the current map and front-end kernels, so nothing computed for an
 *   earlier map, shape or kernel set is ever used. Device memory, allocated on first use and reused: the FP64 field (8 B per voxel, 1 GiB at
 *   512^3) and three bit grids (traversability and two frontiers, 1 bit per voxel each). The calls count their launches in
 *   isdf_stats.kernel_launches and touch no other field of isdf_stats. */
typedef struct isdf_frontpath_params {   /* NULL = defaults; the reserved fields must be zero */
    int32_t reserved_[4];
} isdf_frontpath_params;
typedef struct isdf_frontpath_info {       /* the last path or field call */
    int32_t rounds;                        /* relaxation rounds that had a non-empty frontier */
    int32_t reserved_;
    int64_t field_bytes;                   /* device bytes of the FP64 field */
    double traversability_ms, field_ms, paths_ms;   /* device time of the three stages (CUDA events on the call's stream) */
} isdf_frontpath_info;
int isdf_frontend_path(isdf_ctx *ctx, const double *start, const double *goal, const isdf_frontpath_params *params, int cap,
                       double *path_xyz, double *path_roll_pitch, int32_t *n, double *cost, uint8_t *found);
int isdf_frontend_path_batch(isdf_ctx *ctx, const double *start, int B, const double *goals, const isdf_frontpath_params *params, int cap,
                             double *path_xyz, double *path_roll_pitch, int32_t *offsets, double *costs, uint8_t *found);
/* device variant: d_goals (B x 3) and every output on ctx's device, start (3 doubles) on the host. Work queued on cuda_stream before the
 * call is waited for; the call runs on cuda_stream, synchronises it between stages and returns when the outputs are written. */
int isdf_frontend_path_batch_device(isdf_ctx *ctx, const double *start, int B, const double *d_goals, const isdf_frontpath_params *params,
                                    int cap, double *d_path_xyz, double *d_path_roll_pitch, int32_t *d_offsets, double *d_costs,
                                    uint8_t *d_found, void *cuda_stream);
/* the cost-to-come field from start (host, 3 doubles): d_g = X*Y*Z doubles on ctx's device, address ix*Y*Z + iy*Z + iz, +inf where no
 * path exists. Same errors and stream behaviour as the device variant. */
int isdf_frontend_path_field_device(isdf_ctx *ctx, const double *start, const isdf_frontpath_params *params, double *d_g, void *cuda_stream);
int isdf_frontend_path_info(isdf_ctx *ctx, isdf_frontpath_info *out);

/* ---- swept-volume term: addSaftyPenaOnSweptVolumeParallel (hpp:557-649) + getSDFofSweptVolume (swm:710-747) --- */
/* parallel_points (plan_manager.cpp:246-254): P x 3 row-major world-frame voxel centres; resets lastTstar to 0 (not the persisted
 * trajectory duration: see isdf_set_points_batch) */
int isdf_set_points(isdf_ctx *ctx, const double *pts, int P);
int isdf_eval_swept(isdf_ctx *ctx, int N, const double *T, const double *coeffs,
                    double *cost, double *gradC, double *gradT);
int isdf_eval_swept_device(isdf_ctx *ctx, int N, const double *d_T, const double *d_coeffs, double *d_out,
                           void *cuda_stream);
/* per-point results of the last swept evaluation: t* (lastTstar, hpp:59), SV-SDF value, g_rel (3 per point); any may be NULL */
int isdf_get_swept_results(isdf_ctx *ctx, double *tstar, double *sdf, double *grel);
/* tier-T1 tail parity: evaluate the chain-rule tail at caller-supplied t*, sdf*, g_rel instead of searching */
int isdf_eval_swept_given(isdf_ctx *ctx, int N, const double *T, const double *coeffs, const double *tstar,
                          const double *sdf, const double *grel, double *cost, double *gradC, double *gradT);

#ifdef __cplusplus
}
#endif
#endif /* ISDF_H */
