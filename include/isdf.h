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

/* Fusion: adds the points of a cloud to the current map, in its frame (a map sensed batch by batch, as a vehicle builds it in flight).
 *   Records     isdf_set_map_cloud's format and checks (float32 x, y, z at byte offsets 0, 4, 8; stride a multiple of 4 and >= 12;
 *               1 <= n < 2^32; 4-byte aligned); isdf_sense_cloud's output goes in with stride 12.
 *   Frame       the map already set (ISDF_ERR_STATE without one) keeps X, Y, Z, bmin, bmax and res, however it was set. An empty frame is
 *               isdf_set_map_u8 of a zero grid.
 *   Inside      a finite record is inside when bmin <= (double)c <= bmax on every axis, with isdf_get_map_info's bmin and bmax (the
 *               reference's isInMap); its voxel is isdf_set_map_cloud's index (getGridIndex). Records outside are dropped and counted in
 *               points_outside; records with a NaN or Inf coordinate are counted in points_skipped; points_used counts the inside ones.
 *   Occupancy   sta_threshold 1: a voxel hit by an inside record becomes occupied. Bits are only set, never cleared (no free-space
 *               carving); voxels_added counts the bits this call set, so the sum over calls is the growth of occupied_voxels.
 * The result is the same bits whatever the order of the points, however a cloud is split across calls, and through either form. A
 * successful call gives up the distance field (isdf_map_esdf builds it again); isdf_map_info.occupied_voxels reflects the fused grid while
 * points_used / points_skipped still describe the cloud that set the map. Refused calls leave map and field as they were; a CUDA failure
 * leaves no map. info may be NULL. The call counts its launches in isdf_stats.kernel_launches. */
typedef struct isdf_fuse_info {
    int64_t points_used, points_outside, points_skipped, voxels_added;
} isdf_fuse_info;
int isdf_map_fuse_cloud(isdf_ctx *ctx, const void *points, int64_t n, int32_t stride_bytes, isdf_fuse_info *info);
/* the same with the points on ctx's device: work before the call on cuda_stream is waited for, the grid is updated on ctx's own stream
 * and the call returns when the map is updated (one 32-byte read of the counts), so d_points may be reused at once. */
int isdf_map_fuse_cloud_device(isdf_ctx *ctx, const void *d_points, int64_t n, int32_t stride_bytes, isdf_fuse_info *info,
                               void *cuda_stream);
/* the grid as 0 / 1 in the setters' layout (address ix*Y*Z + iy*Z + iz), n = X*Y*Z elements (ISDF_ERR_INVALID otherwise). The f64
 * form fills the reference's occupancy_map->grid_map directly (after createGridMap(bmin, bmax) with isdf_get_map_info's frame). The
 * grid is expanded on the device in bounded chunks. */
int isdf_get_map_u8(isdf_ctx *ctx, uint8_t *occ, int64_t n);
int isdf_get_map_f64(isdf_ctx *ctx, double *grid_map, int64_t n);

/* ---- known space: the voxels a depth image has proven empty (DESIGN §3.22) ----------------------------------------------------------
 * The map carries a second bit grid, KNOWN, in the occupancy grid's layout. Every isdf_set_map_* call resets it to "nothing known" (its
 * memory is allocated by the first call that marks a voxel); isdf_map_fuse_cloud* leaves it as it is; bits are only ever set.
 * Voxel cube. Voxel (ix, iy, iz)'s cube is, per axis a with index i, in FP64 with nothing contracted: pad = 1e-12 (|bmin_a| + (i + 1) res),
 *   lo = (bmin_a + i res) - pad, hi = (bmin_a + (i + 1) res) + pad (closed). The pad covers the rounding of getGridIndex, so every point
 *   the cloud index puts in a voxel lies in its cube.
 * isdf_map_observe(_device): the poses, camera and scene of isdf_sense_depth (same checks; ISDF_ERR_STATE without a scene or a map), and a
 *   FINITE sensing_horizon (ISDF_ERR_INVALID otherwise, and when (ceil(2 horizon / res) + 3)^3 exceeds 2^40). Per pose the depth image is
 *   rendered exactly as isdf_sense_depth renders it; with r, t the render's FP32 camera-from-world (as doubles), fx, fy, cx, cy its FP32
 *   parameters and body the pose position, voxel v becomes known when all of these hold (FP64, nothing contracted, in this order):
 *     2. every corner k of the cube has sqrt((d0^2 + d1^2) + d2^2) <= sensing_horizon, d = corner - body;
 *        M = the largest |coordinate| of the cube; E_i = 1e-6 (((|r_i0| + |r_i1|) + |r_i2|) M + |t_i|) + 1e-30, each < 1e24;
 *        corner camera coordinates c_i = ((r_i0 X + r_i1 Y) + r_i2 Z) + t_i;
 *     1. zmin = min_k z_k > E_2 (the render's FP32 transform is within E_i of this one: its four roundings are below 2.4e-7 of the same sum);
 *     3. with qx = x_k / z_k, u_k = qx fx + cx, a = max |qx| (likewise qy, v_k, b with fy, cy), zl = zmin - E_2,
 *        dqx = (E_0 + a E_2) / zl, eu = (fx dqx + 1.2e-7 ((a + dqx) fx + |cx|)) + 1e-9 (1 + (a fx + |cx|)) (likewise ev with E_1, b, fy, cy):
 *        the rectangle x0 = floor((min u - eu) + 0.5) .. x1 = floor((max u + eu) + 0.5), y0 .. y1 likewise, lies inside the image
 *        (x0 >= 0, x1 <= W - 1, y0 >= 0, y1 <= H - 1). eu bounds the render's error in fma(x / z, fx, cx): the transform's E through the
 *        division, the division's and the fma's roundings (2^-23 relative together), and this FP64 arithmetic;
 *     4. with the image's min-mip (level l + 1 cell (i, j) = min of level l cells (2i .. 2i + 1, 2j .. 2j + 1) inside the level; level 0
 *        the image) and l the smallest level with (x1 >> l) - (x0 >> l) <= 1 and (y1 >> l) - (y0 >> l) <= 1, the minimum D of the cells
 *        (x0 >> l or x1 >> l, y0 >> l or y1 >> l) satisfies (double)D > 1000 zmax + ((1000 E_2 + 0.5) + 1.2e-7 (1000 (zmax + E_2) + 1)),
 *        zmax = max_k z_k: dist_mm = trunc(fma(z, 1000, 0.5)) of a point at most zmax + E_2 deep is below that bound.
 *   Invariant: no scene point lies in the cube of a known voxel. A point in the cube has exact camera coordinates in the corners' convex
 *   hull, so (1) puts it in front of the camera, (3) puts its rendered centre pixel in the rectangle (truncation equals floor there), and
 *   that pixel's depth is at most its dist_mm, which (4) excludes. The splat never matters, and the result is the same bits for any Q, pose
 *   order, internal chunking, and through either form. info (may be NULL): poses; voxels_tested, the (pose, voxel) pairs of the map inside
 *   each pose's index box floor((body - horizon - bmin) / res) - 1 + [0, ceil(2 horizon / res) + 3) per axis; voxels_added, the bits this
 *   call set (exact in any order). The device form reads d_pos / d_quat on cuda_stream and returns when the bits are set. A CUDA failure
 *   leaves no map.
 * isdf_map_mark_known: marks known every voxel whose unpadded closed cube [bmin + i res, bmin + (i + 1) res] (per axis, FP64) lies inside
 *   one of n closed boxes (lo[3], hi[3]: 6 doubles per box, host), so a box on voxel faces marks the voxels it holds. The caller asserts
 *   the boxes are free (the space a vehicle starts in). ISDF_ERR_INVALID for n < 0, boxes NULL with n > 0, a non-finite
 *   bound or lo > hi; ISDF_ERR_STATE without a map.
 * isdf_get_map_known_u8: the known grid in isdf_get_map_u8's layout.
 * isdf_set_unknown_policy: ISDF_UNKNOWN_FREE (the default) leaves the clearance family as it was, whatever is known;
 *   ISDF_UNKNOWN_OCCUPIED makes every call that reads candidate voxels for a clearance or a certificate (isdf_trajectory_clearance,
 *   isdf_pose_clearance, isdf_trajectory_certify, the certificate of isdf_trajectory_brake and of ISDF_PLAN_CERTIFY) read the BLOCKED grid
 *   occ | (~known within the map) instead. The front end, mid-end, back-end cost, obstacle gathers and distance field keep reading occupancy;
 *   planning that prefers known space is asked for separately (isdf_frontpath_params.unknown_weight, ISDF_PLAN_KNOWN_PREFIX, DESIGN §3.23).
 *   The blocked grid is rebuilt (one launch, and a wait on the calling stream) by the first such call after a map, fuse, observe or mark
 *   call. Voxels outside the map stay outside every candidate set. The policy is context state; it survives map changes. */
typedef enum isdf_unknown_policy { ISDF_UNKNOWN_FREE = 0, ISDF_UNKNOWN_OCCUPIED = 1 } isdf_unknown_policy;
typedef struct isdf_observe_info {
    int64_t poses, voxels_tested, voxels_added;
} isdf_observe_info;
struct isdf_sense_params;   /* defined with the depth-sensing calls below */
int isdf_map_observe(isdf_ctx *ctx, int64_t Q, const double *pos, const double *quat, int64_t stride_doubles, const struct isdf_sense_params *p,
                     isdf_observe_info *info);
int isdf_map_observe_device(isdf_ctx *ctx, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride_doubles,
                            const struct isdf_sense_params *p, isdf_observe_info *info, void *cuda_stream);
int isdf_map_mark_known(isdf_ctx *ctx, int64_t n, const double *boxes);
int isdf_get_map_known_u8(isdf_ctx *ctx, uint8_t *known, int64_t n);
int isdf_set_unknown_policy(isdf_ctx *ctx, int policy);
int isdf_get_unknown_policy(isdf_ctx *ctx, int *policy);

/* ---- distance field of the map: replaces GridMap3D::generateESDF3d (grid:361-525), getSDFValue and getSDFValueWithGrad
 * (GridMap3D.h:114-193) ------------------------------------------------------------------------------------------------------
 *   Definition  POSITIVE at a voxel is res * sqrt((double)d2), d2 the exact integer squared voxel distance to the nearest occupied voxel
 *               (0 inside obstacles); NEGATIVE is the same with free voxels as the sites (0 in free space). A field whose map has no site
 *               is res * sqrt(DBL_MAX) everywhere, as in the reference, not inf. Both are computed on the map's stored 0 / 1 occupancy
 *               and are bit-identical to the reference's grid_esdf and grid_map_buffer_neg after generateESDF3d on isdf_get_map_f64's
 *               output, for every map the call accepts.
 *   SIGNED      v = POSITIVE; if (NEGATIVE > 0.0) v += (-NEGATIVE + res). The reference's grid_map_buffer_all adds the occupancy value
 *               grid_map where this adds POSITIVE (grid:513-522); SIGNED is the signed field that sum was evidently meant to be (the
 *               Fast-Planner convention), with the reference's operation order. grid_map_buffer_all itself is not exposed (DESIGN §6).
 *   Lifetime    the field belongs to ctx: isdf_map_esdf builds it (again) for the current map; any map setter that succeeds gives it up,
 *               a refused setter leaves map and field in place, and a CUDA failure of isdf_map_esdf or of a map setter leaves no field.
 *               No other call builds or uses it. It holds 8 bytes per voxel on the device; building needs at most 8 more.
 * Every call counts its launches in isdf_stats.kernel_launches and touches no other field. */
typedef enum isdf_esdf_field {
    ISDF_ESDF_POSITIVE = 0,   /* grid_esdf: distance to the nearest occupied voxel centre, 0 inside obstacles */
    ISDF_ESDF_NEGATIVE = 1,   /* grid_map_buffer_neg: distance to the nearest free voxel centre, 0 in free space */
    ISDF_ESDF_SIGNED   = 2    /* POSITIVE, plus (-NEGATIVE + res) where NEGATIVE > 0 */
} isdf_esdf_field;
/* generateESDF3d on the current map: both fields, three launches. Errors: ISDF_ERR_INVALID for a NULL ctx; ISDF_ERR_STATE without a
 * map; ISDF_ERR_UNSUPPORTED for a map with an axis longer than 46341 voxels (the reference's fillESDF computes q * q in int, which
 * overflows there, so it has no defined field to match). */
int isdf_map_esdf(isdf_ctx *ctx);
/* one field as X*Y*Z doubles in the setters' layout (address ix*Y*Z + iy*Z + iz), expanded on the device in bounded chunks.
 * Errors: ISDF_ERR_INVALID for a NULL pointer, an unknown field or n != X*Y*Z; ISDF_ERR_STATE without a field. */
int isdf_get_esdf_f64(isdf_ctx *ctx, int field, double *out, int64_t n);
/* getSDFValueWithGrad (grad != NULL) or getSDFValue (grad == NULL) on one field at n points (pts and grad n x 3 row-major, dist n),
 * operation for operation, so bit-identical to the reference on that field, including its quirks (DESIGN §6):
 *   - the base corner is getGridIndex(pos - 0.5 res): clamped to the top index, and (0, 0, 0) when pos - 0.5 res lies outside
 *     [bmin, bmax], so points outside the map or in its first half voxel extrapolate from corner (0, 0, 0);
 *   - a corner past the top index reads 0 (getGridSDFValue(const Vector3i &)), so values fall toward 0 at the upper faces;
 *   - bmax is the map's own (isdf_get_map_info): for a cloud-built map the cloud's maximum, not bmin + X*res.
 * A point with a NaN or Inf coordinate gives NaN value and gradient (undefined behaviour in the reference). Errors: ISDF_ERR_INVALID
 * for a NULL pts / dist / ctx, n < 0 or an unknown field; ISDF_ERR_STATE without a field. */
int isdf_esdf_query(isdf_ctx *ctx, int field, const double *pts, int64_t n, double *dist, double *grad);
/* the same with d_pts, d_dist and d_grad (may be NULL) on ctx's device, enqueued on cuda_stream and not waited for: the results are
 * ready when that stream reaches them. The field must not be given up or rebuilt before then. */
int isdf_esdf_query_device(isdf_ctx *ctx, int field, const double *d_pts, int64_t n, double *d_dist, double *d_grad,
                           void *cuda_stream);

/* PCSmapManager::getPointsInAABB (pcs:148-170) on the device map; writes up to cap centres (cap x 3), returns count in *n */
int isdf_points_in_aabb(isdf_ctx *ctx, const double *centre, double half_extent, double *out_points, int cap, int *n);

/* The obstacle list of PlannerManager::generateTraj (plan_manager.cpp:232-254): for every waypoint in order, the occupied voxels of
 * box(wp + offset, half) that are not in box(previous wp, half) (PCSmapManager::getPointsInAABBOutOfLastOne, pcs:182-216),
 * de-duplicated by voxel. waypoints: nQ x 3 row-major. Writes up to cap centres in (first-including waypoint, voxel address)
 * order and the total in *n. If set_as_points != 0 the list also becomes the swept-volume point set (== isdf_set_points). */
int isdf_gather_obstacle_points(isdf_ctx *ctx, const double *waypoints, int nQ, double half_extent, const double *offset,
                                double *out_points, int cap, int *n, int set_as_points);
/* Every plan's obstacle list in one call. B plans (1 <= B <= 65535); plan b's waypoints are rows [wp_off[b], wp_off[b+1]) of waypoints
 * (x 3 row-major). A plan with no waypoints is allowed and gathers nothing.
 *   Definition  plan b's list is exactly isdf_gather_obstacle_points(ctx, its waypoints, half_extent, offset): the same points in the same
 *               (first-including waypoint, voxel address) order, with the 999 previous-waypoint sentinel for the plan's first box
 *               (plan_manager.cpp:228). A plan's boxes are de-duplicated against its own earlier boxes only.
 *   Output      the lists back to back in plan order in out_points (cap x 3); pt_off (B + 1) is their CSR, the offsets
 *               isdf_set_points_batch takes. When cap is smaller than the total the call returns ISDF_ERR_INVALID, writes no point and
 *               pt_off still reports the sizes needed. out_points may be NULL: cap is then ignored and only pt_off (and, with
 *               set_as_points, the point sets) are produced.
 *   set_as_points != 0: the lists also become the batched swept-volume point sets straight from device memory, bit-identical to
 *               isdf_set_points_batch(ctx, B, pt_off, out_points): every t* starts at 0 (plan_manager.cpp:254) and the single-problem
 *               set is given up. If no plan gathers a point, the batched term is switched off (as B = 0) and the single-problem set is
 *               given up too.
 * Device work: four launches over all plans (index boxes; per-waypoint counts, grid.y = plan; one scan of the counts; the ordered write)
 * and one read of the offsets. Errors: ISDF_ERR_INVALID for a NULL argument, B out of range, offsets that do not start at 0 or decrease,
 * cap < 0, or a total beyond 2^31 - 1; ISDF_ERR_STATE without a map. The call counts its launches in isdf_stats.kernel_launches. */
int isdf_gather_obstacle_points_batch(isdf_ctx *ctx, int B, const int32_t *wp_off, const double *waypoints, double half_extent,
                                      const double *offset, int64_t cap, double *out_points, int32_t *pt_off, int set_as_points);
/* The same with a per-plan known prefix (DESIGN §3.23). known_rows (B, host; NULL = isdf_gather_obstacle_points_batch exactly): plan b's
 *   rows j < known_rows[b] (its first known_rows[b] waypoints) take their voxels from the BLOCKED grid, occ | (~known within the map) of
 *   isdf_set_unknown_policy, instead of the occupancy grid; its other rows read occupancy as before. A value past the plan's row count
 *   covers every row. De-duplication is unchanged: a voxel belongs to the first box of its plan that includes it, each box tested on its
 *   own row's grid. Because known rows come first and an occupied voxel is blocked, testing every earlier box on the current row's grid gives
 *   the same answer, so the lists stay independent of any processing order. The blocked grid is rebuilt (one launch and a wait) when a map,
 *   fuse, observe or mark call made it stale, whatever the unknown policy. Errors: those above, and ISDF_ERR_INVALID for a negative
 *   known_rows entry. */
int isdf_gather_obstacle_points_batch_known(isdf_ctx *ctx, int B, const int32_t *wp_off, const double *waypoints, double half_extent,
                                            const double *offset, const int32_t *known_rows, int64_t cap, double *out_points,
                                            int32_t *pt_off, int set_as_points);

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
/* ---- ragged batches: problems of different piece counts in one call ----------------------------------------------------------------
 * Every *_ragged entry point below takes (B, piece_off) where its uniform sibling takes (B, N0); every other argument is the sibling's.
 * piece_off: B + 1 int32 values on the HOST (also for the _device forms: the host sizes the launches from them), piece_off[0] = 0; problem
 * b has N_b = piece_off[b+1] - piece_off[b] pieces, 1 <= N_b <= 290, and P = piece_off[B] pieces in all. Problem b's part of each array:
 *   decision vectors x, grad    rows [4 piece_off[b] - 3 b, 4 piece_off[b+1] - 3 (b+1)) = [tau (N_b) | xi (3(N_b-1))]
 *   waypoints (mid-end)         rows [piece_off[b] - b, piece_off[b+1] - (b+1)): the wp_off layout of isdf_path_waypoints, whose output
 *                               therefore feeds the ragged mid-end unchanged
 *   durations T                 T[piece_off[b] + i]
 *   coefficients                one 6P x 3 column-major block, piece piece_off[b] + i at rows 6 (piece_off[b] + i) ...
 *   per-problem scalars         index b (cost, f, ret, iterations, evaluations)
 * The uniform batch is the case piece_off[b] = b N0: with those offsets every ragged call returns what its sibling returns, bit for bit.
 * A problem's results do not depend on the batch around it: alone, in a uniform batch or in a ragged one, they are bit-identical. The
 * lock-step drivers run until the slowest instance stops, so one ragged call costs about its slowest problem where one uniform call per
 * distinct N costs the sum of each call's slowest; shared memory is sized by the largest N_b of the call.
 * The swept-volume term is on exactly when point sets are registered for the same B (isdf_set_points_batch), as for the uniform calls.
 * Errors follow the siblings': ISDF_ERR_INVALID for a NULL argument, B < 1, piece_off[0] != 0 or offsets that do not increase;
 * ISDF_ERR_UNSUPPORTED for N_b > 290 or (callback, L-BFGS) P (K+1) beyond 31 bits; ISDF_ERR_STATE on a sharded context. On failure every
 * cost[b] / f[b] is NaN, as the sibling's. */
int isdf_callback_batch_ragged(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *head, const double *tail, int per_problem_bc,
                               double rho, const double *x, double *cost, double *grad);
int isdf_callback_batch_ragged_device(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *d_head, const double *d_tail,
                                      int per_problem_bc, double rho, const double *d_x, double *d_cost, double *d_grad, void *cuda_stream);
/* the trajectories of the last batched callback (uniform or ragged): durations (P = B*N0 for a uniform call), coefficient block (6P x 3
 * column-major, piece piece_off[b]+i; b*N0+i for a uniform call), jerk energies (B); any may be NULL */
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
/* ragged forms (see "ragged batches" above): x holds 4P - 3B rows; every instance runs from the first round and stops on its own */
int isdf_lbfgs_batch_ragged(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *head, const double *tail, int per_problem_bc,
                            double rho, const isdf_lbfgs_params *params, double *x, double *f, int32_t *ret, int32_t *iterations,
                            int32_t *evaluations, int32_t *rounds);
int isdf_lbfgs_batch_ragged_device(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *d_head, const double *d_tail,
                                   int per_problem_bc, double rho, const isdf_lbfgs_params *params, double *d_x, double *d_f, int32_t *d_ret,
                                   int32_t *d_iterations, int32_t *d_evaluations, int32_t *rounds, void *cuda_stream);

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
/* the same on the device: d_path_off (B + 1), d_path_xyz, d_waypoints (cap x 3), d_wp_off (B + 1) and d_pieces (B) on ctx's device, the
 * call on cuda_stream. Every output is byte-equal to isdf_path_waypoints' on the same paths, with the same IEEE operations (one division or
 * one ceil per step, nothing contracted). One pass counts each path's waypoints, a scan gives wp_off, a second pass writes the rows below
 * cap. The host reads one 4-byte total and the call returns when the outputs are written. ISDF_ERR_INVALID when the total exceeds cap (with
 * d_wp_off and d_pieces written, and the rows below cap), for a NULL pointer (d_waypoints may be NULL when cap = 0), B < 1, cap < 0, or
 * res or parlength not finite and positive. Device data is not checked on the host: offsets that do not start at 0 or do not increase give
 * a path of fewer than three nodes (N = 1, no waypoint) wherever path_off[b+1] - path_off[b] < 3, and offsets past the nodes of d_path_xyz
 * are read as they are. Where parlength / res underflows to 0 (the host form does not terminate there) a path gets N = 1. */
int isdf_path_waypoints_device(isdf_ctx *ctx, int B, const int32_t *d_path_off, const double *d_path_xyz, double res, double parlength,
                               int cap, double *d_waypoints, int32_t *d_wp_off, int32_t *d_pieces, void *cuda_stream);
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
/* ragged form (see "ragged batches" above): waypoints P - B rows (may be NULL when P = B), x and grad 4P - 3B rows */
int isdf_midend_callback_batch_ragged(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *head, const double *tail,
                                      int per_problem_bc, const isdf_midend_params *p, const double *waypoints, const double *x,
                                      double *cost, double *grad);
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
/* ragged forms (see "ragged batches" above): waypoints P - B rows (isdf_path_waypoints' output as it stands; may be NULL when P = B),
 * x 4P - 3B rows, T P and coeffs 6P x 3 */
int isdf_midend_batch_ragged(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *head, const double *tail, int per_problem_bc,
                             const isdf_midend_params *p, const double *waypoints, double *x, double *T, double *coeffs,
                             double *f, int32_t *ret, int32_t *iterations, int32_t *evaluations, int32_t *rounds);
int isdf_midend_batch_ragged_device(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *d_head, const double *d_tail,
                                    int per_problem_bc, const isdf_midend_params *p, const double *d_waypoints, double *d_x, double *d_T,
                                    double *d_coeffs, double *d_f, int32_t *d_ret, int32_t *d_iterations, int32_t *d_evaluations,
                                    int32_t *rounds, void *cuda_stream);

/* ---- trajectory clearance check: is a trajectory collision-free over the WHOLE map, and by how much? ------------------------------
 * The reference has no working counterpart (SweptVolumeManager::isTrajCollide, swm:759-767, always returns false), and the cost terms
 * cannot stand in for it: the hinge is smoothed and positive only inside safety_hor, the swept-volume term only sees the gathered obstacle
 * list, the discrete term only the bd/2 box at its own sample spacing.
 * Definition:
 *   Samples. N pieces (T, coeffs in the layout of isdf_eval_discrete); piece i has K_c + 1 pose samples at local times j * step,
 *     step = T_i * (1 / K_c), j = 0..K_c — the discrete path's pose: position of the piece polynomial, flatness quaternion, R = quat_rot(q).
 *     Junction times are sampled twice (last sample of one piece, first of the next), as in the integral loop. The check is SAMPLED: nothing
 *     is certified between two samples T_i / K_c apart (isdf_trajectory_certify below closes those gaps).
 *   Candidates of a sample: the blocked map voxels whose centre c (getGridCubeCenter) satisfies |R^T (c - x)|_inf <= H,
 *     H = half_bd + reach, half_bd = kernel_size * occupancy_resolution / 2 (a strict > on any axis excludes, as hpp:800). Only voxels of
 *     the map count: a window reaching past the map border is cut off there (no projInMap clamping).
 *   Blocked voxels are the occupied ones under ISDF_UNKNOWN_FREE (the default) and the occupied or not known ones under
 *     ISDF_UNKNOWN_OCCUPIED (isdf_set_unknown_policy); isdf_pose_clearance, isdf_trajectory_certify, the certificate of isdf_trajectory_brake
 *     and the certificate of the planning calls (ISDF_PLAN_CERTIFY) read the same blocked voxels.
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

/* ---- clearance at caller-given poses: the clearance check's definition over Q poses instead of trajectory samples ----
 * Pose q is the position at pos + q * stride_doubles (x, y, z) and the quaternion at quat + q * stride_doubles (w, x, y, z; R = quat_rot as
 * isdf_pose_points), so records are read in place: isdf_simulate's log (pos = log + 1, quat = log + 7, stride ISDF_SIM_DOUBLES) or
 * isdf_trajectory_states' records (pos = states, quat = states + 12, stride ISDF_STATE_DOUBLES). Each pose gets what the clearance check
 * gives a sample: the same H box, reach cap, witness rule, mesh branch and bound and sign mode, with the same bits for the same pose, and
 * NaN for a non-finite pose. Poses g * poses_per_group .. + poses_per_group - 1 form group g (0: one group of all Q poses), summarised as a
 * trajectory with the pose index in place of (piece, sample): piece_min = the index within the group of the first pose attaining the
 * minimum, sample_min = 0, t_min = that index as a double, first_hit = the index of the first pose with clear < margin (-1 if none).
 * Results are bit-identical run to run, through either entry point, and for a group checked alone or inside a batch.
 * Errors: ISDF_ERR_INVALID for a NULL argument, Q < 1 or Q >= 2^31, stride_doubles < 1, reach <= 0 or not finite, margin > reach,
 * poses_per_group < 0 or not dividing Q, a non-zero reserved_ and a window wider than 1023 voxels per axis; ISDF_ERR_STATE without a map or a
 * shape; ISDF_ERR_UNSUPPORTED on a sharded context. On failure every summary has min_clearance NaN and collision_free 0. The call counts its
 * launches in isdf_stats.kernel_launches. The host form stages the poses through the device form; the device form is enqueued on
 * cuda_stream and not waited for. */
typedef struct isdf_pose_clearance_params {
    double reach, margin;      /* as isdf_clearance_params */
    int32_t poses_per_group;   /* 0 = one group of Q poses; else Q % poses_per_group == 0 */
    int32_t reserved_;
} isdf_pose_clearance_params;
/* reach = margin = safety_hor of the default config, poses_per_group 0 */
int isdf_pose_clearance_default_params(isdf_pose_clearance_params *p);
/* host buffers; clear / voxel (Q each) may be NULL; summary: Q / poses_per_group entries (1 for 0) */
int isdf_pose_clearance(isdf_ctx *ctx, int64_t Q, const double *pos, const double *quat, int64_t stride_doubles,
                        const isdf_pose_clearance_params *p, double *clear, int64_t *voxel, isdf_clearance_summary *summary);
int isdf_pose_clearance_device(isdf_ctx *ctx, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride_doubles,
                               const isdf_pose_clearance_params *p, double *d_clear, int64_t *d_voxel, isdf_clearance_summary *d_summary,
                               void *cuda_stream);

/* ---- continuous clearance certificate: is a trajectory clear at EVERY time, not only at its samples? ---------------------------
 * The clearance check above is sampled; this call closes the gaps between the samples with a proven motion bound.
 * Definition. Inputs and parameters are the clearance check's (T, coeffs, K_c, N0, reach, margin) with 0 <= margin < reach. One verdict
 * per trajectory:
 *   CERTIFIED (1)   for every time t of the trajectory and every blocked voxel centre c of the map (the clearance check's blocked voxels), the Euclidean distance from c to
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

/* ---- dynamic-limit certificate: can the vehicle fly a trajectory at EVERY time, not only at the penalty's samples? -----------------
 * The back end's dynamics term (addTimeIntPenaltyParallel, hpp:505-534) is a weighted penalty at the K + 1 samples of each piece; an
 * optimised trajectory can exceed vmax at a sample and anywhere between two. This call proves bounds over every time instead.
 * Definition. N pieces (T, coeffs in the layout of isdf_eval_discrete), pieces b*N0 .. b*N0+N0-1 form trajectory b (N0 = 0: one trajectory
 *   of all N pieces). The coefficients and durations are taken as exact; local time t runs over [0, T_i]; the flatness parameters are the
 *   context's (vehicle_mass, grav_acc, horiz_drag, vert_drag, paras_drag, speed_eps); yaw is zero, as in the back end. Quantities at t:
 *     q = 0  speed         |v(t)|
 *     q = 1  acceleration  |a(t)|
 *     q = 2  body rate     |omega(t)|, omega of FlatnessMap::optimizated_forward(v, a, j, quat, omg) (flatness.hpp:88-148)
 *     q = 3  tilt          theta(t) = acos(z_z), z = zu / |zu|, zu = a + dh/m (1 + cp sqrt(|v|^2 + veps)) v + g e_z (equal in exact
 *                          arithmetic to the back end's acos(1 - 2 (q1^2 + q2^2)), hpp:505)
 *     q = 4  thrust        f(t) = z . (mass a + dv w + mass g e_z), w = (1 + cp sqrt(|v|^2 + veps)) v, dv = vert_drag: FlatnessMap::forward
 *                          at psi = dpsi = 0 (flatness.hpp:150-207)
 *   Limits: vmax, amax, omgmax, thetamax bound q = 0..3 from above, thrust_min / thrust_max bound the thrust from both sides. +inf
 *   (-inf for thrust_min) means the quantity is reported and not checked.
 * Verdict per trajectory:
 *   FEASIBLE (1)   every checked limit holds with a proof: upper <= limit, thrust_lower >= thrust_min;
 *   VIOLATING (-1) an evaluated sample proves a limit broken (attained > limit, thrust_attained_min < thrust_min), or a sample is not finite;
 *   UNDECIDED (0)  neither was established within the refinement budget.
 * Mechanism.
 *   The initial samples are the clearance check's K + 1 per piece at local times j (T_i (1/K)) (with K = integral_intervs, exactly where
 *   the back-end penalty looks), and piece i has K intervals, the last ending at T_i; intervals never cross a junction.
 *   Interval enclosure: the piece polynomial re-expanded about the midpoint te with Taylor coefficients d_k as intervals;
 *   v in d_1 + [-1, 1] sum_{k>=2} k |d_k| h^(k-1), a and j likewise, h = sup |t - te|; every quantity is then evaluated in outward-rounded
 *   interval arithmetic (norms, the flatness map, omega, z_z, the thrust); acos is padded outward by 8 ulp (CUDA documents 2). A division
 *   by an enclosure that reaches 0 (|zu|, 1 + z_z, or sqrt(|v|^2 + veps) when speed_eps = 0 and paras_drag != 0) gives body rate
 *   [0, +inf], tilt [0, pi] and thrust [-|F|, |F|] with F = mass a + dv w + mass g e_z: such an interval must be refined.
 *   Sample: the same evaluation at h = 0 encloses the exact value at that time; its lower end is proven attained (for the thrust minimum,
 *   its upper end).
 *   Split rule: an interval is split at ta + 0.5 (tb - ta), with a new sample there, when for some quantity its upper end hi exceeds the
 *   limit while the trajectory's attained value does not (the limit is locally undecided), or hi > attained + tol (the reported maximum
 *   is not yet tight); the thrust minimum mirrors this at the lower end. tol = +inf gives pure verdict mode. A trajectory with a
 *   non-finite sample splits no further. Splitting stops at max_depth or when the trajectory's new samples would exceed
 *   max_samples_per_traj (intervals earlier in time get the samples first); a leaf whose hi exceeds a checked limit is undecided.
 * Summary per trajectory: upper[q] = the maximum of hi over the final leaves, a proven upper bound of sup_t q(t); attained[q] and
 *   t_attained[q] the largest value proven attained at an evaluated sample and its trajectory time (ties: earliest time); thrust_lower,
 *   thrust_attained_min, t_thrust_attained_min the mirror for the thrust minimum; violated / undecided: bit q (q = 0..4, bit 4 the thrust
 *   maximum) and bit 5 (the thrust minimum) of the limits proven broken / neither proven broken nor proven held; samples (N0 (K + 1) plus
 *   the new ones), undecided_intervals, depth (deepest leaf level). With a non-finite sample the bounds are NaN.
 * Results are deterministic run to run, identical through both entry points, and a trajectory's result is bit-identical alone or inside
 * a batch (every fold is a maximum with ties to the earliest time; per-trajectory budgets; order-preserving compaction).
 * Device work per round: one interval pass (two kernels) and one 4-byte read; at most max_depth + 1 rounds; no map or shape is needed.
 * Errors: ISDF_ERR_INVALID for K < 1, N < 1, N0 < 0 or not dividing N, max_depth outside [0, 64], max_samples_per_traj < 0, a tolerance
 *   that is NaN or negative, a NaN limit, thrust_min > thrust_max, a non-zero reserved_, sizes beyond 31-bit indexing, NULL pointers;
 *   ISDF_ERR_UNSUPPORTED on a sharded context. On failure every summary has verdict 0, its bounds NaN and its counts -1.
 * The call counts its launches in isdf_stats.kernel_launches and touches no other field; it leaves the discrete schedule, the clearance
 * and certificate buffers, the swept-volume state, the mid-end buffers and the batch trajectories as they were. */
typedef struct isdf_dynamics_params {
    int32_t samples_per_piece;     /* K >= 1 */
    int32_t pieces_per_traj;       /* N0; 0 = one trajectory of N pieces; else N % N0 == 0 */
    int32_t max_depth;             /* splits per initial interval, 0..64 */
    int32_t max_samples_per_traj;  /* new samples per trajectory, >= 0 */
    double vmax, amax, omgmax, thetamax, thrust_min, thrust_max;   /* +inf (thrust_min -inf): report only */
    double tol_v, tol_a, tol_omg, tol_theta, tol_thrust;           /* >= 0; +inf: verdict only */
    int32_t reserved_[2];          /* must be 0 */
} isdf_dynamics_params;

typedef struct isdf_dynamics_summary {
    double upper[5], attained[5], t_attained[5];                   /* q = speed, acceleration, body rate, tilt, thrust */
    double thrust_lower, thrust_attained_min, t_thrust_attained_min;
    int32_t verdict;                                               /* 1 FEASIBLE, -1 VIOLATING, 0 UNDECIDED */
    int32_t violated, undecided;                                   /* bit masks: q = 0..4, bit 5 the thrust minimum */
    int32_t samples, undecided_intervals, depth;
} isdf_dynamics_summary;

/* K = integral_intervs, N0 = 0, vmax / omgmax / thetamax of the context's config (of isdf_default_config for ctx NULL; thetamax 100 rad,
 * the reference's config, never binds),
 * every other limit report-only; tolerances 1e-3 m/s, 1e-3 m/s^2, 1e-3 rad/s, 1e-4 rad, 1e-3 N; max_depth 16, max_samples_per_traj 2048.
 * The tolerances and budgets are starting points, not tuned (DESIGN §3.13). */
int isdf_dynamics_default_params(isdf_ctx *ctx, isdf_dynamics_params *p);
/* host buffers; summary: N/N0 entries (1 for N0 = 0) */
int isdf_trajectory_dynamics(isdf_ctx *ctx, int N, const double *T, const double *coeffs, const isdf_dynamics_params *p,
                             isdf_dynamics_summary *summary);
/* device-resident variant: d_T, d_coeffs, d_summary on ctx's device; runs on cuda_stream (NULL = default stream) and returns when the
 * summaries are written (the round loop reads 4 bytes per round) */
int isdf_trajectory_dynamics_device(isdf_ctx *ctx, int N, const double *d_T, const double *d_coeffs, const isdf_dynamics_params *p,
                                    isdf_dynamics_summary *d_summary, void *cuda_stream);

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
 * attitude grid size (sw_manager.hpp:135-136); at most 128 attitudes. Call again after changing the shape.
 * ISDF_ERR_UNSUPPORTED, with the current kernels left as they were, when
 *   - 16 * kernel_size^3 bytes (the offset masks, staged in one CTA's shared memory) exceed the device's opt-in shared memory per
 *     block: kernel_size (odd) <= 23 on H100;
 *   - the reference's accumulating loop `for (a = -max; a <= max; a += ang_res)` (Shape.hpp:422-426) visits another number of roll
 *     or pitch angles than floor(2 * max / ang_res) + 1 (e.g. max 27, ang_res 3.6: 16 expected, 15 visited), a grid on which the
 *     reference leaves kernels unbuilt. */
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
 * father's attitude, sw_manager.hpp:852-913); ok[q] = 0 when no attitude fits (child = father). The father's grid index is
 * (int)((roll + max_roll) / ang_res), likewise for pitch; a father whose index falls outside the grid (roll < -max_roll - ang_res or
 * beyond max_roll by a step) gets the level pose when it fits, child = father + (level index - father index) * ang_res, and ok = 0
 * otherwise (no BFS: the reference's would index outside its grid). */
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
 *   Surcharge on unknown voxels (params->unknown_weight, finite and >= 0; 0, or NULL params, is the definition above bit for bit)
 *                  c = 1 + unknown_weight, once, in FP64. The edge into v costs w(u, v) = sqrt((double)n) when v is known (the map's KNOWN bit,
 *                  isdf_map_observe / isdf_map_mark_known) and sqrt((double)n) * c (one rounded product) when it is not; before any observe
 *                  or mark call nothing is known. Everything else above holds with this w: the field g, the parent rule g(u) + w(u, v) ==
 *                  g(v) (w read at v, the node the walk steps from), paths, attitudes and found; the cost is the weighted g(t). Why the
 *                  field stays exact and order-free: c >= 1 and sqrt((double)n) >= 1, so every weight is >= 1 (rounding is monotone), and FP
 *                  addition of a positive weight is monotone; so the minimum over paths of the left-to-right sums is what any label-correcting
 *                  order reaches, and a textbook FP64 Dijkstra with the same weights gives the same bits. A weight below FP64's resolution
 *                  at 1 gives c == 1, the unweighted field. A route through unseen space costs c times its length there, so a known detour
 *                  up to c times longer is preferred.
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
 *   a negative or non-finite unknown_weight, or cap smaller than the total path length (then *n / offsets still report the lengths
 *   needed); ISDF_ERR_UNSUPPORTED on a sharded context (isdf_set_shard world > 1).
 * State: every call rebuilds the traversability grid and the field from the current map and front-end kernels, so nothing computed for an
 *   earlier map, shape or kernel set is ever used. Device memory, allocated on first use and reused: the FP64 field (8 B per voxel, 1 GiB at
 *   512^3) and three bit grids (traversability and two frontiers, 1 bit per voxel each). The calls count their launches in
 *   isdf_stats.kernel_launches and touch no other field of isdf_stats. */
typedef struct isdf_frontpath_params {   /* NULL = defaults (all zero); the reserved fields must be zero. 16 bytes */
    double unknown_weight;                /* the surcharge on unknown voxels above; finite, >= 0 (ISDF_ERR_INVALID otherwise) */
    int32_t reserved_[2];
} isdf_frontpath_params;
typedef struct isdf_frontpath_info {       /* the last path, pairs or field call */
    int32_t rounds;                        /* relaxation rounds that had a non-empty frontier */
    int32_t reserved_;
    int64_t field_bytes;                   /* device bytes of the FP64 fields held at once */
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
/* ---- pairs: B (start, goal) pairs, start b with goal b (the reference's targetRcvCallBack pairs, plan_manager.cpp:434-488) ----
 * Definition: pair b's path, roll and pitch, cost and found are bit-identical to isdf_frontend_path(starts[b], goals[b]); outputs in the
 *   layout of isdf_frontend_path_batch, in pair order. Permuting the pairs permutes the outputs; max_fields never changes a bit.
 * Work: the traversability grid is built once per call. Pairs whose starts share a voxel share one field (node 0 of a path is that voxel's
 *   cube centre). The distinct start voxels' fields are relaxed together, up to max_fields at a time: each field held at once takes 8 B per
 *   voxel (1 GiB at 512^3) and 2 frontier bits per voxel; max_fields = 0 holds at most 4 GiB of fields, and at least one field. Each
 *   source's field is the exact field above whichever sources share its relaxation.
 * isdf_frontend_path_info after a pairs or fields call: rounds is the total, over the chunks of fields, of the rounds in which any source
 *   had a frontier; field_bytes the bytes of fields held at once; the stage times cover the whole call.
 * Errors: those of isdf_frontend_path_batch, and ISDF_ERR_INVALID for max_fields < 0; isdf_last_error names the index of a start or goal
 *   outside the map. */
int isdf_frontend_path_pairs(isdf_ctx *ctx, int B, const double *starts, const double *goals, const isdf_frontpath_params *params,
                             int max_fields, int cap, double *path_xyz, double *path_roll_pitch, int32_t *offsets, double *costs,
                             uint8_t *found);
/* device variant: d_starts and d_goals (B x 3 each) and every output on ctx's device; the starts and goals are read to the host to group
 * them. Stream behaviour as isdf_frontend_path_batch_device. */
int isdf_frontend_path_pairs_device(isdf_ctx *ctx, int B, const double *d_starts, const double *d_goals, const isdf_frontpath_params *params,
                                    int max_fields, int cap, double *d_path_xyz, double *d_path_roll_pitch, int32_t *d_offsets,
                                    double *d_costs, uint8_t *d_found, void *cuda_stream);
/* the fields from S starts (host, S x 3) in one relaxation: field s at d_g + s*X*Y*Z (S*X*Y*Z doubles on ctx's device), each
 * bit-identical to isdf_frontend_path_field_device(starts[s]), also when starts share a voxel. Errors: those of
 * isdf_frontend_path_field_device, and ISDF_ERR_INVALID for S < 1 or S > 65535. */
int isdf_frontend_path_fields_device(isdf_ctx *ctx, int S, const double *starts, const isdf_frontpath_params *params, double *d_g,
                                     void *cuda_stream);

/* ---- planning step: PlannerManager::generateTraj (plan_manager.cpp:202-313) for one start and B goals, end to end on the device ----
 * Definition, per goal b (each step is an existing entry point's definition):
 *   1. Front end   isdf_frontend_path_batch(start, goals, &p->frontpath). A path not found is NO_PATH: no trajectory.
 *   2. Waypoints   isdf_path_waypoints(parlength, the map's res) gives N. N > 290 (the limit of the mid-end and the callback) is TOO_LONG:
 *                  no trajectory. head = [path.front(), 0, 0], tail = [path.back(), 0, 0] (:220-223).
 *   3. Mid-end     isdf_midend_batch_ragged(per_problem_bc = 1, p->midend) over every plan that reaches it, in goal order (one call; each
 *                  plan's result equals isdf_midend_batch over the plans with its N). midend_ret < 0 is MIDEND_FAILED: its trajectory is the mid-end's final one (what recent_traj holds, :270) and
 *                  the back end does not run for it (:277).
 *   4. Gather      isdf_gather_obstacle_points_batch(half_extent, offset, set_as_points = 1) over the waypoints of the plans that passed
 *                  the mid-end, in goal order. A plan with no point gets no swept-volume term, as the reference's loop over zero points.
 *                  With ISDF_PLAN_KNOWN_PREFIX it is isdf_gather_obstacle_points_batch_known with, for plan b: k* = the index of the first
 *                  node of its path whose voxel is not known (the path length when every node is; 0 when nothing is known); waypoint row j
 *                  is path node (j + 1) g (isdf_path_waypoints' gap g), and the known rows are those with (j + 1) g < k*. So while the path is
 *                  inside what has been seen the back end treats unseen space as an obstacle, and past the first unknown node it stays
 *                  optimistic. Without the flag, nothing is known, or k* = 0, the gather is the one above.
 *   5. Durations   before the back end, problem q's persisted trajectory duration (see isdf_set_points_batch) is what
 *                  updateTraj(mid-end trajectory) (:272) leaves on a fresh context: its total duration (the left-to-right sum of T) when
 *                  shorter than 300 s, else 0. Plans are therefore independent of each other and of the order of the groups.
 *   6. Back end    isdf_lbfgs_batch_ragged(per_problem_bc = 1, p->rho, p->backend) over those plans from the mid-end x, with the
 *                  context's flags (one call, every plan active from its first round). The final T and
 *                  coeffs are forwardT + MINCO of the returned x whatever its ret (back_end_optimizer.cpp:140-163), computed without a
 *                  further evaluation. Stage OPTIMISED; backend_ret < 0 is reported and the trajectory still returned (`if (1)`, :297).
 *   7. Certificates with ISDF_PLAN_CERTIFY / ISDF_PLAN_DYNAMICS: isdf_trajectory_certify / isdf_trajectory_dynamics with p->certify /
 *                  p->dynamics and N0 = N on every returned trajectory (OPTIMISED and MIDEND_FAILED), one call per distinct N. The
 *                  certificate reads the blocked voxels of the context's unknown policy; stages 1-6 read the occupancy grid.
 * Deviation: the reference's back end is LMBM (lmbm.h, Fortran); the driver here is the project's device L-BFGS. max_iterations 10000 in
 *   the defaults is LMBM's iteration cap (lmbm.h:20-57) taken as an analogue, not an equivalent.
 * Guarantees: results are bit-identical run to run; each plan is bit-identical to the same call with that goal alone; every output is
 *   bit-identical to the composition of the public calls above on a fresh context whenever every mid-end trajectory is shorter than 300 s
 *   (the only case where step 5 differs from what the public calls can express: there, a group inherits the durations the group before
 *   it left).
 * Outputs:
 *   paths       path_off (B + 1) and path_xyz (cap_nodes x 3) in the layout of isdf_frontend_path_batch (a NO_PATH plan has its one-node
 *               path); either may be NULL (path_xyz NULL: cap_nodes is ignored).
 *   trajectories plan b's pieces are [piece_off[b], piece_off[b+1]) (0 pieces for NO_PATH and TOO_LONG): T[piece_off[b] + i], and its own
 *               6N x 3 column-major block at coeffs + 18 * piece_off[b] (cap_pieces pieces in all).
 *   results     B records: stage, path_nodes, pieces (N; 0 for NO_PATH), obstacle_points (0 for plans that did not reach the back end),
 *               midend_ret / backend_ret / backend_iterations / backend_evaluations (0 where the stage did not run), path_cost (the front
 *               end's cost, +inf for NO_PATH), midend_f / backend_f (NaN where the stage did not run), duration (total of the returned
 *               trajectory, 0 without one).
 *   certify / dynamics  B summaries each (may be NULL when the flag is off); a plan without a trajectory gets the failed-call summary of
 *               its certificate.
 *   Caps too small: after the front end and the waypoints the call returns ISDF_ERR_INVALID; path_off and piece_off give the sizes needed.
 * State the call leaves behind: both obstacle point sets given up and the batched swept-volume term off (also after a failure past the
 *   argument checks); isdf_get_batch_trajectories returns every back-end plan's final trajectory in the ragged layout (plans in goal
 *   order), and the swept-volume t* and per-problem durations are whatever the back end left; isdf_stats.kernel_launches counts every launch of the call, the other isdf_stats fields
 *   are whatever the last back-end callback left.
 * Device memory: owned by the context, grown on demand. Between stages only per-plan values and the rounds' 4-byte reads cross to the
 *   host (see the device forms below); the host form then copies its outputs back.
 * Errors: ISDF_ERR_STATE without a map, a shape or front-end kernels; ISDF_ERR_UNSUPPORTED on a sharded context and for ISDF_PLAN_CERTIFY
 *   with a shape the certificate refuses (checked before any work); ISDF_ERR_INVALID for a NULL argument, B < 1, the stages' own parameter
 *   checks, unknown flags, a non-zero reserved_ (also frontpath.reserved_), a negative or non-finite frontpath.unknown_weight,
 *   pieces_per_traj != 0 in p->certify or p->dynamics, a start or goal outside the map, or caps too small. On failure every stage is -1, midend_f / backend_f are NaN, and the summaries read as their certificates' failures. */
/* 4 is not a flag (refused as unknown).
 * ISDF_PLAN_KNOWN_ONLY (DESIGN §3.24): step 1 runs over T_b (isdf_map_frontiers: in the map, neither occupied nor unknown, and a non-zero
 *   feasibility mask on the blocked grid) instead of the traversable set; everything else in step 1 holds, so every path node but the start
 *   is in T_b, every edge steps into a known voxel and frontpath.unknown_weight, still checked, changes no bit. Step 4 is
 *   isdf_gather_obstacle_points_batch_known with every waypoint row known (known_rows = the plan's row count). It may be combined with
 *   ISDF_PLAN_KNOWN_PREFIX, which then adds nothing. The mid-end, back end and certificates are unchanged; without the flag every output
 *   keeps its bits. */
typedef enum isdf_plan_flags {
    ISDF_PLAN_CERTIFY = 1, ISDF_PLAN_DYNAMICS = 2, ISDF_PLAN_KNOWN_PREFIX = 8, ISDF_PLAN_KNOWN_ONLY = 16
} isdf_plan_flags;
typedef enum isdf_plan_stage {
    ISDF_PLAN_FAILED = -1, ISDF_PLAN_NO_PATH = 0, ISDF_PLAN_TOO_LONG = 1, ISDF_PLAN_MIDEND_FAILED = 2, ISDF_PLAN_OPTIMISED = 3
} isdf_plan_stage;
typedef struct isdf_plan_params {
    double parlength;               /* traj_parlength, 3.0 (plan_manager.cpp:153); finite, > 0 */
    double half_extent;             /* gather half extent; default kernel_size * occupancy_resolution / 3 (:135, :243); finite, >= 0 */
    double offset[3];               /* offsetAABBbox (config.hpp:146, default 0); finite */
    double rho;                     /* back-end time weight, yaml rho 20; finite */
    isdf_midend_params midend;      /* isdf_midend_default_params */
    isdf_lbfgs_params backend;      /* isdf_lbfgs_default_params with max_iterations 10000 */
    int32_t flags;                  /* isdf_plan_flags */
    int32_t reserved_;              /* must be 0 */
    isdf_certify_params certify;    /* pieces_per_traj must be 0: the call sets N0 = N per group */
    isdf_dynamics_params dynamics;  /* likewise */
    isdf_frontpath_params frontpath;   /* the front end's parameters (unknown_weight); zero in the defaults. Added at the end: the struct
                                          grew by its 16 bytes, and zero means the planning step as it was */
} isdf_plan_params;
typedef struct isdf_plan_result {
    int32_t stage;                  /* isdf_plan_stage */
    int32_t path_nodes, pieces, obstacle_points;
    int32_t midend_ret, backend_ret, backend_iterations, backend_evaluations;
    double path_cost, midend_f, backend_f, duration;
} isdf_plan_result;
typedef struct isdf_plan_info {     /* the last isdf_plan_batch or isdf_plan_pairs call */
    int32_t groups, backend_rounds;  /* distinct N that reached the mid-end; batched evaluations of the one back-end launch */
    double frontend_ms, midend_ms, gather_ms, backend_ms, certify_ms, dynamics_ms;   /* CUDA events on the call's stream */
} isdf_plan_info;
/* the values above, flags ISDF_PLAN_CERTIFY | ISDF_PLAN_DYNAMICS, isdf_certify_default_params and isdf_dynamics_default_params(ctx);
 * ctx may be NULL (isdf_default_config's values) */
int isdf_plan_default_params(isdf_ctx *ctx, isdf_plan_params *p);
int isdf_plan_batch(isdf_ctx *ctx, const double *start, int B, const double *goals, const isdf_plan_params *p,
                    int cap_nodes, int32_t *path_off, double *path_xyz,
                    int cap_pieces, int32_t *piece_off, double *T, double *coeffs,
                    isdf_plan_result *results, isdf_certify_summary *certify, isdf_dynamics_summary *dynamics);
/* B (start, goal) pairs: isdf_plan_batch's definition with starts[b] in place of start (its head is [path.front(), 0, 0] of its own path,
 * the cube centre of its start voxel) and pair order in place of goal order; the front end is isdf_frontend_path_pairs(max_fields).
 * Outputs, stages, errors, the durations rule, the state left behind and isdf_get_plan_info are isdf_plan_batch's, plus ISDF_ERR_INVALID
 * for max_fields < 0. Pair b is bit-identical to isdf_plan_batch(starts[b], 1, &goals[b]); permuting the pairs permutes the outputs;
 * max_fields never changes a bit; with every start equal, every output equals isdf_plan_batch(start, goals), which is this call with its
 * start broadcast. */
int isdf_plan_pairs(isdf_ctx *ctx, int B, const double *starts, const double *goals, const isdf_plan_params *p, int max_fields,
                    int cap_nodes, int32_t *path_off, double *path_xyz,
                    int cap_pieces, int32_t *piece_off, double *T, double *coeffs,
                    isdf_plan_result *results, isdf_certify_summary *certify, isdf_dynamics_summary *dynamics);
/* device forms: isdf_plan_pairs / isdf_plan_batch word for word (stages, durations rule, caps, errors, the poisoning of results and
 * summaries on failure, the state left behind and isdf_get_plan_info), with d_starts (B x 3) and d_goals (B x 3) and every output in
 * ctx's device memory in the host form's layout; the start of isdf_plan_batch_device is on the host (3 doubles), as in
 * isdf_frontend_path_batch_device. d_path_off and d_path_xyz may be NULL as in the host form.
 * Stream: work queued on cuda_stream before the call is waited for; the call runs on cuda_stream and returns when its outputs are written
 * (the mid-end's and back end's rounds read 4 bytes each and wait for them). With caps too small, d_path_off and d_piece_off give the sizes
 * needed and the results and summaries read as failures.
 * One pipeline: the host forms stage their outputs through the context and copy them back, so they give the same bits as the device forms.
 * Transfers: besides the starts and goals (read to the host to group them, as isdf_frontend_path_pairs_device does), only per-plan values
 * cross to the host: the path lengths and found flags, N, the mid-end return codes and the gathered point counts, plus the rounds' 4-byte
 * reads. Device-to-host bytes outside those reads are at most 80 per plan plus 64 (isdf_plan_batch_device: 56 per plan), whatever the
 * lengths of the paths and trajectories. Nothing proportional to path nodes, waypoints or pieces crosses in either direction. */
int isdf_plan_pairs_device(isdf_ctx *ctx, int B, const double *d_starts, const double *d_goals, const isdf_plan_params *p, int max_fields,
                           int cap_nodes, int32_t *d_path_off, double *d_path_xyz, int cap_pieces, int32_t *d_piece_off, double *d_T,
                           double *d_coeffs, isdf_plan_result *d_results, isdf_certify_summary *d_certify,
                           isdf_dynamics_summary *d_dynamics, void *cuda_stream);
int isdf_plan_batch_device(isdf_ctx *ctx, const double *start, int B, const double *d_goals, const isdf_plan_params *p, int cap_nodes,
                           int32_t *d_path_off, double *d_path_xyz, int cap_pieces, int32_t *d_piece_off, double *d_T, double *d_coeffs,
                           isdf_plan_result *d_results, isdf_certify_summary *d_certify, isdf_dynamics_summary *d_dynamics,
                           void *cuda_stream);
/* B (start state, goal) pairs from moving vehicles: isdf_plan_pairs with starts as B x 9 doubles (p[3], v[3], a[3]) instead of B x 3.
 * The front end starts at the voxel containing p, exactly as isdf_plan_pairs with starts[b] = p; the head of the mid-end and the back end
 * is [p, v, a] instead of [path.front(), 0, 0]; the tail is unchanged. Everything else (stages, caps, certificates, the durations rule,
 * outputs, the state left behind, isdf_get_plan_info, errors) is isdf_plan_pairs', plus ISDF_ERR_INVALID for a non-finite v or a. With
 * starts[b] = (path.front() of an isdf_plan_pairs run, 0, 0) every output is bit-identical to isdf_plan_pairs. The device form reads the
 * positions (24 bytes per pair) and one 4-byte verdict of a device-side finiteness check of v and a, so its transfers stay within
 * isdf_plan_pairs_device's bounds. */
int isdf_plan_states(isdf_ctx *ctx, int B, const double *starts, const double *goals, const isdf_plan_params *p, int max_fields,
                     int cap_nodes, int32_t *path_off, double *path_xyz,
                     int cap_pieces, int32_t *piece_off, double *T, double *coeffs,
                     isdf_plan_result *results, isdf_certify_summary *certify, isdf_dynamics_summary *dynamics);
int isdf_plan_states_device(isdf_ctx *ctx, int B, const double *d_starts, const double *d_goals, const isdf_plan_params *p, int max_fields,
                            int cap_nodes, int32_t *d_path_off, double *d_path_xyz, int cap_pieces, int32_t *d_piece_off, double *d_T,
                            double *d_coeffs, isdf_plan_result *d_results, isdf_certify_summary *d_certify,
                            isdf_dynamics_summary *d_dynamics, void *cuda_stream);
int isdf_get_plan_info(isdf_ctx *ctx, isdf_plan_info *out);

/* ---- frontiers of known space and frontier goals (DESIGN §3.24) ---------------------------------------------------------------------
 * Definition (FP64, nothing contracted; voxel index ix*Y*Z + iy*Z + iz; cube centre as getGridCubeCenter, bmin + (i + 0.5) res)
 *   T_o        the traversable set of the front end: in the map, not occupied, and a non-zero isdf_frontend_feasibility mask.
 *   T_b        the same test on the BLOCKED grid occ | (~known within the map): in the map, not blocked (so known and free), and a
 *              non-zero feasibility mask computed on the blocked grid (cells outside the map count as free, as for the feasibility call).
 *              T_b is a subset of T_o. Nothing known: T_b is empty.
 *   F          the frontier: v in T_b with some 26-neighbour u inside the map in T_o \ T_b. A place where the robot fits with every kernel
 *              cell known free, next to a place where it would fit if unseen space were free.
 *   Clusters   the 26-connected components of F. A cluster's id is its smallest voxel index; clusters are listed by ascending id. Size,
 *              index box and centroid_a = bmin_a + ((double) sum of i_a / (double) size + 0.5) * res (exact integer sums: order-free).
 * isdf_map_frontiers: the frontier voxels in ascending index (voxels, cap_voxels), each with its cluster id (cluster_of), and the cluster
 *   table (clusters, cap_clusters). info (may be NULL) gets |T_b|, |F|, the cluster count and the stage times. A cap too small is
 *   ISDF_ERR_INVALID with info holding the sizes needed (the outputs are then not written). The device form writes device buffers on
 *   cuda_stream and returns when they are written.
 * Errors: ISDF_ERR_STATE without a map or front-end kernels; ISDF_ERR_UNSUPPORTED on a sharded context; ISDF_ERR_INVALID for a NULL
 *   output with a non-zero cap, a negative cap, or caps too small. */
typedef struct isdf_frontier_cluster {   /* 64 bytes */
    int64_t id;                           /* the smallest voxel index of the cluster */
    int64_t size;                         /* voxels */
    int32_t bmin[3], bmax[3];             /* index box, inclusive */
    double centroid[3];
} isdf_frontier_cluster;
typedef struct isdf_frontier_info {       /* 72 bytes */
    int64_t traversable_blocked;          /* |T_b| */
    int64_t frontier_voxels;              /* |F| */
    int64_t clusters;
    int64_t reserved_;
    double traversability_ms, frontier_ms, cluster_ms;   /* CUDA events: the two feasibility passes, F and its list, the labelling and table */
    double field_ms, select_ms;           /* isdf_frontier_goals: the fields over T_b and the selection; 0 for isdf_map_frontiers */
} isdf_frontier_info;
int isdf_map_frontiers(isdf_ctx *ctx, int64_t cap_voxels, int64_t *voxels, int64_t *cluster_of, int64_t cap_clusters,
                       isdf_frontier_cluster *clusters, isdf_frontier_info *info);
int isdf_map_frontiers_device(isdf_ctx *ctx, int64_t cap_voxels, int64_t *d_voxels, int64_t *d_cluster_of, int64_t cap_clusters,
                              isdf_frontier_cluster *d_clusters, isdf_frontier_info *info, void *cuda_stream);
/* Frontier goals, per pair b: s and t are the start and goal voxels (path_voxel's rules: both in the map). g_b is the front end's field
 * from s over T_b, unweighted (s need not be traversable).
 *   1. g_b(t) < inf: kind GOAL, voxel t, cluster -1, g = score = g_b(t), point = the goal as given.
 *   2. else among the frontier voxels f with g_b(f) < inf in clusters of at least min_cluster_voxels voxels, the least
 *      score = g_b(f) + goal_weight * sqrt((dx*dx + dy*dy) + dz*dz), d = cube centre of f - goal; ties to the smaller voxel index:
 *      kind FRONTIER, voxel f, its cluster id, g_b(f), the score, point = f's cube centre.
 *   3. else kind NONE, voxel and cluster -1, g = score = +inf, point = the goal as given.
 * Work: pairs whose starts share a voxel share a field; the fields are relaxed together up to max_fields at a time (0: a 4 GiB budget),
 *   as isdf_frontend_path_pairs does. Guarantees: bit-identical run to run, host form to device form, under any permutation of the pairs
 *   and for any max_fields. info (may be NULL) as for isdf_map_frontiers, with field_ms and select_ms.
 * Errors: those of isdf_map_frontiers, and ISDF_ERR_INVALID for NULL arguments, B < 1, max_fields < 0, a start or goal outside the map or
 *   not finite, goal_weight not finite or <= 0, min_cluster_voxels < 1, a non-zero reserved_. NULL params: the defaults. */
typedef struct isdf_frontier_params {     /* 16 bytes */
    double goal_weight;                   /* default 1 */
    int32_t min_cluster_voxels;           /* default 1 */
    int32_t reserved_;                    /* must be 0 */
} isdf_frontier_params;
typedef enum isdf_frontier_kind { ISDF_FRONTIER_NONE = 0, ISDF_FRONTIER_GOAL = 1, ISDF_FRONTIER_FRONTIER = 2 } isdf_frontier_kind;
typedef struct isdf_frontier_goal {       /* 64 bytes */
    int32_t kind;                         /* isdf_frontier_kind */
    int32_t gain;                         /* FRONTIER from isdf_frontier_goals_view: the voxel's view gain (saturating at INT32_MAX); else 0 */
    int64_t voxel, cluster;
    double g, score;
    double point[3];
} isdf_frontier_goal;
int isdf_frontier_default_params(isdf_frontier_params *p);
int isdf_frontier_goals(isdf_ctx *ctx, int B, const double *starts, const double *goals, const isdf_frontier_params *p, int max_fields,
                        isdf_frontier_goal *out, isdf_frontier_info *info);
/* device form: d_starts, d_goals (B x 3) and d_out on ctx's device; the starts and goals are read to the host to group them. The call runs
 * on cuda_stream and returns when d_out is written. */
int isdf_frontier_goals_device(isdf_ctx *ctx, int B, const double *d_starts, const double *d_goals, const isdf_frontier_params *p,
                               int max_fields, isdf_frontier_goal *d_out, isdf_frontier_info *info, void *cuda_stream);

/* ---- view gain: the unseen space a rig of cameras would observe from a pose (DESIGN §3.25) ---------------------------------------------
 * Poses are read as isdf_sense_* and isdf_map_observe read them (pos, quat, stride_doubles; a simulate log or isdf_trajectory_states'
 * records in place). The rig is n_cams cameras, each an isdf_sense_params. Nothing is rendered, so no scene is needed; the map is. Voxel v of
 * the map counts toward gain[q] when all of these hold:
 *   (a) unknown: v is neither occupied nor known (without a known grid nothing is known);
 *   (b) in view: for at least one camera of the rig, isdf_map_observe's rules 2, 1 and 3 hold for v (every corner within that camera's
 *       horizon of the body position, in front of the camera by the transform's margin, the widened pixel rectangle inside the image), with
 *       that camera's FP32 render transform at pose q and the same arithmetic in the same order. A voxel several cameras see counts once;
 *   (c) line of sight: with s_a = floor((pos_a - bmin_a) / res) in FP64 (s may lie outside the map), d = v - s and m = max_a |d_a|, no
 *       voxel s_a + floor((2 k d_a + m) / (2 m)) (integer floor division), k = 1 .. m - 1, is occupied: a 26-connected digital line with no
 *       floating-point ties. Voxels outside the map are free, unknown voxels transparent (the optimistic gain).
 *   (b) and (a) make the gain a count of voxels isdf_map_observe of the same pose could still mark; after it, every voxel the gain still
 *   counts at that pose failed observe's rule 4 (the depth image showed something in front of it or inside it).
 * The counts are exact integers: the same bits for any Q, pose order or internal chunking, and through either form. The device form reads
 *   d_pos / d_quat and writes d_gain (Q int64) on cuda_stream, and returns when they are written.
 * Errors: ISDF_ERR_INVALID for NULL arguments, Q < 1 or Q >= 2^31, stride_doubles < 1, n_cams < 1, a camera the sensing calls refuse, an
 *   infinite horizon, and (ceil(2 h_max / res) + 3)^3 > 2^40 (h_max the rig's largest horizon); ISDF_ERR_UNSUPPORTED on a sharded context;
 *   ISDF_ERR_STATE without a map. */
int isdf_view_gain(isdf_ctx *ctx, int64_t Q, const double *pos, const double *quat, int64_t stride_doubles, int n_cams,
                   const struct isdf_sense_params *cams, int64_t *gain);
int isdf_view_gain_device(isdf_ctx *ctx, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride_doubles, int n_cams,
                          const struct isdf_sense_params *cams, int64_t *d_gain, void *cuda_stream);
/* Frontier goals that need something left to see: isdf_frontier_goals with one more candidate condition. The gain of frontier voxel f is
 *   isdf_view_gain at f's cube centre (FP64 bmin + (i + 0.5) res, the FRONTIER record's point) with quaternion (1, 0, 0, 0), the level,
 *   yaw-0 attitude a held vehicle rests in, with the rig cams (host, n_cams >= 1). A frontier voxel is a candidate when its cluster has at
 *   least min_cluster_voxels voxels AND its gain is >= min_gain (>= 0). Gains are computed once per call, only for voxels whose cluster
 *   passes the size rule. A FRONTIER record's gain field holds the chosen voxel's gain (saturating at INT32_MAX); GOAL and NONE hold 0.
 *   isdf_frontier_goals is this call without a rig and min_gain 0 (its gain fields are 0). Guarantees as isdf_frontier_goals'.
 * Errors: those of isdf_frontier_goals, the rig's of isdf_view_gain, and ISDF_ERR_INVALID for min_gain < 0. */
int isdf_frontier_goals_view(isdf_ctx *ctx, int B, const double *starts, const double *goals, const isdf_frontier_params *p, int n_cams,
                             const struct isdf_sense_params *cams, int64_t min_gain, int max_fields, isdf_frontier_goal *out,
                             isdf_frontier_info *info);
int isdf_frontier_goals_view_device(isdf_ctx *ctx, int B, const double *d_starts, const double *d_goals, const isdf_frontier_params *p,
                                    int n_cams, const struct isdf_sense_params *cams, int64_t min_gain, int max_fields,
                                    isdf_frontier_goal *d_out, isdf_frontier_info *info, void *cuda_stream);

/* ---- executing a trajectory: getStateOnTrajStamp (swm:307-341) and the playback of SweptVolumeManager::process (swm:948-988) ----
 * B trajectories in isdf_plan_batch's ragged layout: trajectory b has pieces [piece_off[b], piece_off[b+1]), durations T[piece_off[b] + i],
 * and its own 6N x 3 column-major block at coeffs + 18 * piece_off[b]. Q queries (traj[q], times[q]); out is Q records of
 * ISDF_STATE_DOUBLES = 20 doubles:
 *   pos[3] vel[3] acc[3] jer[3] quat[4] (w, x, y, z, the reference's Vector4d order) omg[3] thr
 * Each record is what process() computes at delta = times[q] (swm:961-971), bit for bit:
 *   - times[q] is local to trajectory traj[q]. The piece and its local time come from locatePieceIdx (trajectory.hpp:545-563): sequential
 *     subtraction with a strict '>', so a junction time stays in the earlier piece; a negative time stays in piece 0 and a time past the end
 *     is clamped into the last piece, both extrapolating its polynomial. NaN and infinite times go through that arithmetic as they are.
 *   - pos, vel, acc, jer are getPos / getVel / getAcc / getJer (trajectory.hpp:150-208) at that local time.
 *   - quat, omg, thr are FlatnessMap::forward(vel, acc, jer, psi = 0, dpsi = 0, thr, quat, omg) (flatness.hpp:150-228) with the context's
 *     (vehicle_mass, grav_acc, horiz_drag, vert_drag, paras_drag, speed_eps), restated operation by operation with psi and dpsi as zero
 *     operands (signs of zero included); thr = z . f_term (:203-206). Yaw is zero, as in the planner's collision model.
 * Every record depends only on its own (traj, time) and that trajectory's data, not on B, Q, the order of the queries or other trajectories.
 * A query on a trajectory without pieces (a NO_PATH or TOO_LONG plan) gets an all-NaN record.
 * Needs a context (its stream and config); no map and no shape. Q = 0 does nothing. The call counts its launch in
 * isdf_stats.kernel_launches and touches no other field. Device memory is the context's, grown on demand; the host form stages through the
 * context's pinned and device staging blocks, which every host form shares: one copy each way.
 * Errors (host form; nothing is written): ISDF_ERR_INVALID for a NULL pointer, B < 1, Q < 0 or Q records beyond 2^63 bytes,
 *   piece_off[0] != 0 or offsets that decrease, a duration that is not positive and finite, a coefficient that is not finite, or traj[q]
 *   outside [0, B). */
#define ISDF_STATE_DOUBLES 20
int isdf_trajectory_states(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *T, const double *coeffs,
                           int64_t Q, const int32_t *traj, const double *times, double *out);
/* the same with every array on ctx's device (d_piece_off too), enqueued on cuda_stream and not waited for. Device data is not checked on the
 * host: a traj[q] outside [0, B) gives an all-NaN record, offsets, durations and coefficients are taken as they are. Host and device forms
 * give identical bits. Errors: ISDF_ERR_INVALID for a NULL pointer, B < 1, Q < 0 or Q records beyond 2^63 bytes. */
int isdf_trajectory_states_device(isdf_ctx *ctx, int B, const int32_t *d_piece_off, const double *d_T, const double *d_coeffs,
                                  int64_t Q, const int32_t *d_traj, const double *d_times, double *d_out, void *cuda_stream);
/* the rest of B trajectories (isdf_plan_batch's ragged layout) from the per-trajectory times t0[b], re-timed to start at 0, written in the
 * same layout to out_piece_off (B + 1), out_T and out_coeffs, which must have room for the input's piece_off[B] pieces:
 *   - piece i and local time tau come from locatePieceIdx's rule, as in isdf_trajectory_states;
 *   - output piece 0 is piece i re-expanded about tau, d_k = sum_{j=k..5} C(j,k) c_j tau^(j-k), accumulated from 0 in ascending j
 *     as (C(j,k) c_j) tau^(j-k) with tau^m the running product of tau (FP64, nothing contracted), with duration T_i - tau; it is dropped when
 *     T_i - tau is not > 0 (t0 on a junction). Pieces after i are copied bit for bit;
 *   - a t0 outside [0, D_b) (D_b the left-to-right sum of T), not finite, or a trajectory without pieces gives 0 pieces: a result, not an error.
 * The host form checks its inputs as isdf_trajectory_states' host form does (nothing is written on a refusal); the device form checks no
 * device data and is enqueued on cuda_stream, not waited for. Both count their launches in isdf_stats.kernel_launches and give identical
 * bits. Errors: ISDF_ERR_INVALID for a NULL pointer or B < 1. */
int isdf_trajectory_shift(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *T, const double *coeffs, const double *t0,
                          int32_t *out_piece_off, double *out_T, double *out_coeffs);
int isdf_trajectory_shift_device(isdf_ctx *ctx, int B, const int32_t *d_piece_off, const double *d_T, const double *d_coeffs,
                                 const double *d_t0, int32_t *d_out_piece_off, double *d_out_T, double *d_out_coeffs, void *cuda_stream);
/* ---- braking to a certified stop along the remaining trajectory (DESIGN §3.21) -------------------------------------------------------
 * (The clearance certificate of the candidates reads the blocked voxels of the context's unknown policy, isdf_set_unknown_policy.)
 * B remaining trajectories in isdf_plan_batch's ragged layout (each starting at the vehicle's current time 0) and t_stop_max[b], the latest
 * trajectory time whose position the stop may reach (e.g. a COLLIDING certificate's first_hit). Per trajectory b, in FP64 with nothing
 * contracted, in this order:
 *   D       = T[0] + T[1] + ... (left to right, from 0.0);
 *   tau_max = t_stop_max[b] if t_stop_max[b] < D, else D; NO_INPUT (0 pieces) for a trajectory without pieces, a NaN t_stop_max[b], or
 *             a tau_max that is not finite and > 0;
 *   candidate k = 0 .. K-1: tau_k = tau_max * ((double)(k + 1) / (double)K), an M-piece MINCO S3 trajectory (isdf_midend_batch's solve,
 *             bit-identical to the host MincoS3) with
 *             head      (x, v, a) of the trajectory at time 0,
 *             tail      (x(tau_k), 0, 0),
 *             durations M equal ones, (tau_k + tau_k) / (double)M,
 *             waypoints x(tau_k * f_j), j = 1 .. M-1, f_j = 1.0 - u_j * u_j, u_j = (double)(M - j) / (double)M.
 *   Positions, velocities and accelerations are isdf_trajectory_states' (locatePieceIdx's rule, then getPos / getVel / getAcc).
 *   This is the constant-deceleration schedule: the remaining path's first tau_k of time is covered in 2 tau_k, at rest at x(tau_k).
 * All B K candidates (uniform, N0 = M) go through isdf_trajectory_certify and isdf_trajectory_dynamics in one pass each (p->certify and
 * p->dynamics with pieces_per_traj set to M; a NO_INPUT trajectory's candidates are at rest at a placeholder and never chosen). The chosen
 * candidate is the largest k that is CERTIFIED and FEASIBLE, the gentlest stop that is proven clear: status BRAKED, its M pieces written
 * at out_piece_off[b]; else status NONE and 0 pieces. out_piece_off (B + 1), out_T and out_coeffs need room for B M pieces.
 * Summary per trajectory: status, candidate (-1 without one), tau_stop and duration (the left-to-right sum of the output T; NaN without a
 * candidate), certified / feasible (how many of the K candidates passed each check; 0 for NO_INPUT), and the chosen candidate's certificate
 * summaries, bit-identical to isdf_trajectory_certify / isdf_trajectory_dynamics of the output with N0 = M (their failed-call summaries
 * without a candidate).
 * A trajectory's result is bit-identical alone or inside a batch; host and device forms give identical bits. The host form stages through
 * the context (one copy each way) and checks its inputs as isdf_trajectory_states' host form does; the device form checks no device data
 * and runs on cuda_stream; only the certificates' 4-byte round reads cross to the host, and the call returns when its outputs are written.
 * The call counts its launches in isdf_stats.kernel_launches; it leaves the discrete schedule, the swept-volume state, the mid-end buffers
 * and the batch trajectories as they were (its MINCO buffers are its own).
 * Errors: ISDF_ERR_INVALID for a NULL pointer, B < 1, K < 1, M outside [1, ISDF_BRAKE_MAX_PIECES], B K M beyond 31 bits, a non-zero
 *   pieces_per_traj in p->certify or p->dynamics or reserved_, and the certificates' own parameter errors; ISDF_ERR_STATE without a map
 *   or a shape; ISDF_ERR_UNSUPPORTED for a shape the certificate refuses and on a sharded context. On failure every summary reads status
 *   NONE, candidate -1, NaN times, counts -1 and both certificates' failed-call summaries; the outputs are otherwise left as they were. */
#define ISDF_BRAKE_MAX_PIECES 64
typedef enum isdf_brake_status { ISDF_BRAKE_NO_INPUT = -1, ISDF_BRAKE_NONE = 0, ISDF_BRAKE_BRAKED = 1 } isdf_brake_status;
typedef struct isdf_brake_params {
    int32_t candidates;             /* K >= 1, default 8 */
    int32_t pieces;                 /* M in [1, ISDF_BRAKE_MAX_PIECES], default 4 */
    isdf_certify_params certify;    /* isdf_certify_default_params; pieces_per_traj must be 0 (the call sets M) */
    isdf_dynamics_params dynamics;  /* isdf_dynamics_default_params(ctx); likewise */
    int32_t reserved_[2];           /* must be 0 */
} isdf_brake_params;
typedef struct isdf_brake_summary {
    int32_t status;                 /* isdf_brake_status */
    int32_t candidate;              /* k of the chosen candidate, -1 without one */
    double tau_stop, duration;      /* tau_k and the stop's duration; NaN without a candidate */
    int32_t certified, feasible;    /* candidates CERTIFIED / FEASIBLE */
    isdf_certify_summary certify;   /* the chosen candidate's */
    isdf_dynamics_summary dynamics;
} isdf_brake_summary;
int isdf_brake_default_params(isdf_ctx *ctx, isdf_brake_params *p);
int isdf_trajectory_brake(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *T, const double *coeffs, const double *t_stop_max,
                          const isdf_brake_params *p, int32_t *out_piece_off, double *out_T, double *out_coeffs, isdf_brake_summary *summary);
int isdf_trajectory_brake_device(isdf_ctx *ctx, int B, const int32_t *d_piece_off, const double *d_T, const double *d_coeffs,
                                 const double *d_t_stop_max, const isdf_brake_params *p, int32_t *d_out_piece_off, double *d_out_T,
                                 double *d_out_coeffs, isdf_brake_summary *d_summary, void *cuda_stream);
/* the robot's body at Q states: out[(q * P + p) * 3 + k] = (R(quat_q) body_p + pos_q)_k, R = quat_rot (Eigen's toRotationMatrix,
 * Shape.hpp:753-757), each row ((R_k0 b0 + R_k1 b1) + R_k2 b2) + pos_k rounded per operation (Shape::Transform, Shape.hpp:786-793).
 * states: Q x 20, isdf_trajectory_states records (only pos and quat are read); body: P x 3 body-frame points (mesh vertices, interior
 * points, markers: no shape needs to be set). An all-NaN record gives NaN points. Q = 0 or P = 0 does nothing.
 * Errors: ISDF_ERR_INVALID for a NULL pointer, Q < 0, P < 0, or Q * P * 3 doubles beyond 2^63 bytes. The device form is enqueued on
 * cuda_stream and not waited for; both forms count their launch in isdf_stats.kernel_launches and give identical bits. */
int isdf_pose_points(isdf_ctx *ctx, int64_t Q, const double *states, int P, const double *body, double *out);
int isdf_pose_points_device(isdf_ctx *ctx, int64_t Q, const double *d_states, int P, const double *d_body, double *d_out,
                            void *cuda_stream);

/* ---- closed loop: flying a trajectory with the reference's SO(3) controller and quadrotor model (src/uav_simulator) ----
 * R rollouts, each one vehicle tracking trajectory traj[r] of B trajectories in isdf_plan_batch's ragged layout (the d_piece_off, d_T,
 * d_coeffs that isdf_plan_pairs_device writes). Rollout r starts from init[r] (ISDF_SIM_INIT_DOUBLES = 17: pos[3] vel[3] quat[4]
 * (w, x, y, z) omega[3] rpm[4]; R(0) = quat_rot(quat) as isdf_pose_points) and feels the constant external force and moment dist[r]
 * (6 doubles: f[3] m[3]; Quadrotor::setExternalForce / setExternalMoment; dist may be NULL for zero). The caller draws any randomness.
 * Definition (one thread per rollout; nothing depends on other rollouts):
 *   Model: Quadrotor::operator() and step() (Quadrotor.cpp) on the 22-double state x v R(column-major) omega rpm. The right-hand side
 *     re-orthonormalises R as R L^-1, L the Cholesky factor of R^T R (Eigen's LLT and 3x3 cofactor inverse); thrust kf sum rpm^2;
 *     moments kf (rpm2^2 - rpm3^2) arm, kf (rpm1^2 - rpm0^2) arm, km (rpm0^2 + rpm1^2 - rpm2^2 - rpm3^2); drag 0.1 pi arm^2 |v|^2 along
 *     v/|v| (pi as the reference's 3.14159265); v' = -g e3 + thrust R e3 / m + f / m - drag v^ / m; R' = R [omega]x;
 *     omega' = J^-1 (moments - omega x J omega + m_ext); rpm' = (input - rpm) / motor_tau; NaN derivatives become 0. The last v' evaluated
 *     is the IMU's acceleration (Quadrotor::getAcc).
 *   Step (Quadrotor::step(dt), dt = 1 / sim_rate): odeint::integrate(sys, x, 0, dt, dt), i.e. integrate_adaptive with
 *     controlled_runge_kutta<runge_kutta_dopri5>: the Dormand-Prince 5(4) pair with first-same-as-last, the derivative at the start evaluated
 *     afresh each step; error max_i |err_i| / (1e-6 + 1e-6 (|x_i| + dt_try |x'_i|)) (NaN terms skipped by the max); err > 1: reject and
 *     dt_try *= max(0.9 err^(-1/3), 0.2); err < 0.5: accept and dt_try *= 0.9 max(err, 5^-5)^(-1/5); otherwise accept; a try that would pass
 *     the end is clipped to land on it. a step whose 1000th try is reached ends the rollout as diverged (odeint throws there, accepted or not), as do a
 *     try that makes no progress (t + h == t) and 100000 tries in one step (bounds odeint does not have). A NaN anywhere in the
 *     result restores the state before the step; then R is re-orthonormalised as in the right-hand side, and with the floor on, z < 0 and
 *     vz < 0 set both to 0.
 *   Attitude loop, every step (getControl, quadrotor_simulator_so3.cpp), in FP32 as written with FP64 where the reference mixes in doubles:
 *     R rebuilt from R_to_ypr(R) with yaw replaced by the command's current_yaw when use_external_yaw; Psi = (3 - tr(Rd^T R)) / 2; the
 *     commanded force projected on the body z axis, or 0 unless Psi < 1; M = -kR eR - kOm eOm + omega x J omega; w_sq mixed, negative
 *     values 0, rpm = sqrtf(w_sq). A NaN rpm keeps the last one (0 before any); setInput maps NaN to (min_rpm + max_rpm) / 2, then clamps.
 *   Position loop, every sim_rate / cmd_rate steps, at t_k = k / cmd_rate (k = 0 before the first step; the state is the one after step
 *     k sim_rate / cmd_rate): (1) odometry: position, velocity, current_yaw = tf::getYaw of Quaterniond(R) (Matrix3x3::getEulerYPR);
 *     (2) IMU: acc = the last v' (0 at k = 0, SO3Control's constructor); (3) command: while t_k < duration (the left-to-right sum of the
 *     trajectory's T) getPos, getVel, getAcc at t_k with yaw 0, yaw_dot 0; from then on the last command stays (the nodelet re-publishes
 *     its last des_* on odometry); (4) SO3Control::calculateControl (the 45-degree limit at theta = pi/2 included) -> force and
 *     Quaterniond orientation, rounded to float with kR, kOm, corrections and current_yaw as the simulator's Command struct holds them.
 *     Odometry before command within a tick is this library's choice (ROS delivers them asynchronously). The command holds until the next tick.
 *   Horizon: ticks k = 0 .. n_ticks - 1, n_ticks = floor(t_end cmd_rate) + 1; the state of the last tick is the final state.
 * Parameters (isdf_sim_default_params, from the reference's launch files and sources):
 *   vehicle (Quadrotor()): mass 0.98, grav 9.81, J diag(2.64e-3, 2.64e-3, 4.96e-3), kf 8.98132e-9, km 0.07 (3 * 0.062) kf, arm 0.26,
 *     motor_tau 1/30, rpm in [1200, 35000];
 *   controller: ctrl_mass 0.98 (simulator_example.launch "mass"), ctrl_grav 9.81 (SO3Control()); kx (5.7, 5.7, 6.2) and kv (3.4, 3.4, 4.0)
 *     (the nodelet's defaults: gains_hummingbird.yaml's pos / vel keys are never read); kR (1, 1, 1) (yaml rot x, y; launch gains/rot/z);
 *     kOm (0.07, 0.07, 0.1) (yaml ang x, y; launch gains/ang/z); corrections 0 (corrections_hummingbird.yaml); use_external_yaw 1 (the
 *     launch file's "use_external_yaw " key has a trailing space, so the nodelet's default true applies);
 *   sim_rate 1000 (rate/simulation), cmd_rate 100 (traj_server's 100 Hz timer and the simulator's rate/odom), t_end 10, log_every 1,
 *   floor 1, diverge_dist 5 m. The vehicle and gains are independent of isdf_config's flatness vehicle.
 * Outputs: log (may be NULL): R x cap_log records of ISDF_SIM_DOUBLES = 21 doubles, record j of rollout r at (r cap_log + j) 21, one per
 *   log_every ticks (tick j log_every): t, pos[3], vel[3], quat[4] (w, x, y, z; Quaterniond(R)), omega[3], rpm[4], commanded pos[3];
 *   records after the rollout ended (diverged) or past n_log = (n_ticks - 1) / log_every + 1 are NaN. summary: one per rollout, over
 *   its ticks: position error |x - des_pos| (max, its time, RMS, final), max tilt acos(R22), max |omega|, steps whose input was clamped,
 *   floor contacts, NaN rollbacks, accepted and rejected dopri5 tries, and diverged (a non-finite state or a position error above
 *   diverge_dist at a tick, which ends the rollout; t_diverged its time, NaN otherwise).
 * Guarantees: a rollout's log and summary depend only on its own inputs: the same bits run to run, alone or in any batch, through either
 *   entry point. The unit is compiled without FMA contraction, so FP64 and FP32 arithmetic rounds as the reference's g++ -O3 x86-64 build;
 *   libm's sin, cos, atan2, asin, acos and pow may differ in the last ulp from glibc's.
 * Errors: ISDF_ERR_INVALID for a NULL argument, B < 1 or R < 0; a rate not positive and finite or sim_rate / cmd_rate not a whole
 *   number; any parameter not finite, mass, J, kf, km, arm, motor_tau, ctrl_mass not positive, min_rpm < 0 or max_rpm < min_rpm, t_end < 0,
 *   log_every < 1, diverge_dist not positive, n_ticks beyond 2^31; a log with cap_log < n_log; a non-zero reserved_; and in the host form
 *   piece_off not starting at 0 or decreasing, durations not positive and finite, coefficients not finite, or traj[r] outside [0, B) or
 *   naming a trajectory without pieces. The device form checks no device data: such a rollout reads as diverged at t = NaN. On failure every
 *   summary reads diverged with NaN values (the host form writes them; the device form when the summary pointer is usable). The call counts
 *   its launches in isdf_stats.kernel_launches. The device form is enqueued on cuda_stream and not waited for. */
#define ISDF_SIM_INIT_DOUBLES 17
#define ISDF_SIM_DOUBLES 21
typedef struct isdf_sim_params {
    double mass, grav, J[3], kf, km, arm, motor_tau, min_rpm, max_rpm;   /* vehicle */
    double ctrl_mass, ctrl_grav, kx[3], kv[3], kR[3], kOm[3], corrections[3];   /* controller */
    double sim_rate, cmd_rate, t_end, diverge_dist;
    int32_t log_every, use_external_yaw, floor, reserved_;
} isdf_sim_params;
typedef struct isdf_sim_summary {
    double max_err, t_max_err, rms_err, final_err, max_tilt, max_omega, t_diverged;
    int64_t accepted, rejected;
    int32_t clamped_steps, floor_contacts, nan_rollbacks, diverged;
} isdf_sim_summary;
int isdf_sim_default_params(isdf_sim_params *p);
int isdf_simulate(isdf_ctx *ctx, int B, const int32_t *piece_off, const double *T, const double *coeffs, int R, const int32_t *traj,
                  const double *init, const double *dist, const isdf_sim_params *p, int cap_log, double *log, isdf_sim_summary *summary);
int isdf_simulate_device(isdf_ctx *ctx, int B, const int32_t *d_piece_off, const double *d_T, const double *d_coeffs, int R,
                         const int32_t *d_traj, const double *d_init, const double *d_dist, const isdf_sim_params *p, int cap_log,
                         double *d_log, isdf_sim_summary *d_summary, void *cuda_stream);

/* ---- depth sensing: the reference's depth camera (uav_simulator/local_sensing) batched over poses ---------------------------------
 * Scene. isdf_set_sense_cloud / _device take the records isdf_set_map_cloud takes (float32 x, y, z at byte offsets 0, 4, 8 of each
 *   stride_bytes record, with the same validation). Records with a NaN or Inf coordinate are skipped and counted (isdf_get_sense_info); on
 *   the GPU the reference's kernel would instead truncate such a point to pixel (0, 0) at depth 0. The context owns the cloud and gives it
 *   up before it is overwritten and on destroy. The device form reads d_points on cuda_stream and returns when the scene is built.
 * Camera (isdf_sense_params). isdf_sense_default_params gives local_sensing/params/camera.yaml: 640 x 480, fx = fy = 387.229248046875,
 *   cx = 321.04638671875, cy = 243.44969177246094; cam_to_body = cam02body of pcl_render_node.cpp:347-350 (row-major
 *   [0 0 1 0; -1 0 0 0; 0 -1 0 0; 0 0 0 1]: the camera looks along the body's x axis); sensing_horizon = +Inf, since no launch file of the
 *   reference sets one (the node then reads an unset double).
 * Poses. Pose q is the position at pos + q stride_doubles and the quaternion (w, x, y, z) at quat + q stride_doubles, R = quat_rot as
 *   isdf_pose_points, so isdf_simulate's log (pos = log + 1, quat = log + 7, stride ISDF_SIM_DOUBLES) and isdf_trajectory_states' records
 *   are read in place. In FP64, nothing contracted:
 *     cam2world[i][j] = ((B[i][0] C[0][j] + B[i][1] C[1][j]) + B[i][2] C[2][j]) + B[i][3] C[3][j], B = [R pos; 0 0 0 1], C = cam_to_body
 *     (exact with the default C, whose entries are 0 and +-1);
 *     the render's camera-from-world is the rigid inverse: r[i][j] = cam2world[j][i], t[i] = -((r[i][0] c0 + r[i][1] c1) + r[i][2] c2) with
 *     c = cam2world's translation, then every entry rounded to FP32 as the reference's Parameter holds it. The reference takes Eigen's
 *     general 4 x 4 inverse; the two may differ in the last FP64 bits before that rounding. From the rounded matrix on, this is the
 *     reference's arithmetic bit for bit.
 * Depth image (depth_render.cu:2-56), all in FP32 unless said: every pixel starts at 999999. For each scene point p:
 *     x = fma(p.z, r02, fma(p.x, r00, p.y r01)) + t0 (FMUL, FFMA, FFMA, FADD as the reference build contracts it), and likewise y,
 *     z; rejected when z <= 0;
 *     px = trunc((double)fma(x / z, fx, cx) + 0.5), py likewise with y, fy, cy (IEEE division, FP64 add, truncation toward zero that
 *     saturates and takes NaN to 0); rejected when px or py falls outside the image, even when the splat would reach in (a centre in
 *     (-1, 0) truncates to 0 and is kept);
 *     dist_mm = trunc(fma(z, 1000, 0.5)); r = trunc(0.0573 (double)fx / (double)z + 0.5) in FP64;
 *     every pixel of the (2r + 1)^2 square around (px, py) inside the image takes min(pixel, dist_mm).
 *   fx, fy, cx, cy are the FP32 roundings of the parameters here. The image is a min over integers, so it does not depend on any order.
 * Sensed points (pcl_render_node.cpp:224-258, 286-296): for u = 0 .. W - 1, then v = 0 .. H - 1 within it: depth = (float)mm / 1000.0f,
 *   0 when depth >= 500 (or NaN); a depth of 0 is skipped. In FP64 with the double parameters, nothing contracted: the camera point
 *   ((u - cx) depth / fx, (v - cy) depth / fy, depth), the world point cam2world times it (summed left to right, the translation last),
 *   dropped when sqrt((dx^2 + dy^2) + dz^2) > sensing_horizon for d = world point - pos (the body position, the node's last_pose_world);
 *   kept points are rounded to FP32 x, y, z as pcl::PointXYZ stores them.
 * Outputs. isdf_sense_depth: depth (Q x H x W int32, pixel (u, v) of pose q at (q H + v) W + u) in mm, 999999 where nothing is seen: the
 *   reference's raw buffer. isdf_sense_cloud: the kept points of pose q in rows [offsets[q], offsets[q + 1]) of points (cap x 3 float32),
 *   offsets Q + 1 int64. When the total exceeds cap the call returns ISDF_ERR_INVALID with offsets written (the sizes needed) and the rows
 *   below cap written. The device forms take device pointers, are enqueued on cuda_stream and return when the work is enqueued, except
 *   isdf_sense_cloud_device, which reads the 8-byte total to report an overflow.
 * Guarantees: pose q's image and points depend only on pose q, the camera and the scene: the same bits for any Q, order of the poses, or
 *   internal chunking, and through host and device forms. Bricks of the scene are culled per pose only where no point of them can reach
 *   the image (for clouds also where every point lies beyond the horizon plus the camera's offset from the body), so culling changes no bit.
 *   A non-finite pose gives whatever the definition gives (every point NaN: depth 0 at pixel (0, 0), no sensed point).
 * Errors: ISDF_ERR_INVALID for a NULL argument, Q < 1 or Q >= 2^31, stride_doubles < 1, width or height < 1 or width x height > 2^26, a
 *   camera parameter or cam_to_body entry not finite, fx or fy not positive, cam_to_body's last row not (0, 0, 0, 1), a NaN horizon or
 *   one <= 0, cap < 0 (points may be NULL when cap = 0); ISDF_ERR_STATE when no scene cloud is set. The calls count their launches in
 *   isdf_stats.kernel_launches. */
typedef struct isdf_sense_params {
    int32_t width, height;
    double fx, fy, cx, cy;
    double cam_to_body[16];    /* row-major 4 x 4 */
    double sensing_horizon;    /* metres; +Inf keeps every point */
} isdf_sense_params;
typedef struct isdf_sense_info {
    int64_t points_used, points_skipped, bricks;
} isdf_sense_info;
int isdf_sense_default_params(isdf_sense_params *p);
int isdf_set_sense_cloud(isdf_ctx *ctx, const void *points, int64_t n, int32_t stride_bytes);
int isdf_set_sense_cloud_device(isdf_ctx *ctx, const void *d_points, int64_t n, int32_t stride_bytes, void *cuda_stream);
int isdf_get_sense_info(isdf_ctx *ctx, isdf_sense_info *out);
int isdf_sense_depth(isdf_ctx *ctx, int64_t Q, const double *pos, const double *quat, int64_t stride_doubles, const isdf_sense_params *p,
                     int32_t *depth);
int isdf_sense_depth_device(isdf_ctx *ctx, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride_doubles,
                            const isdf_sense_params *p, int32_t *d_depth, void *cuda_stream);
int isdf_sense_cloud(isdf_ctx *ctx, int64_t Q, const double *pos, const double *quat, int64_t stride_doubles, const isdf_sense_params *p,
                     int64_t cap, float *points, int64_t *offsets);
int isdf_sense_cloud_device(isdf_ctx *ctx, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride_doubles,
                            const isdf_sense_params *p, int64_t cap, float *d_points, int64_t *d_offsets, void *cuda_stream);

/* ---- world generators: the reference's globalmap_gene maps 1-11 and mockamap's Perlin and box worlds (DESIGN §3.19) --------------
 * Output. A cloud of n records of 16 bytes: float32 x, y, z and 1.0f (what pcl::PointXYZ's constructor leaves in its fourth float), in
 *   the reference's push_back order, ready for isdf_set_map_cloud_device / isdf_set_sense_cloud_device with stride_bytes = 16. *n is
 *   always the cloud's size, so cap = 0 with points NULL is a size query; when *n > cap the call returns ISDF_ERR_INVALID with *n and the
 *   first cap records written.
 * ISDF_WORLD_GLOBALMAP: map_manager/src/globalmap_gene.cpp's mapGene(map_id), map_id 1..11, the node's first publication. Loop coordinates
 *   are the reference's FP64 accumulations (t += cloud_resolution while t < end; roads: t += res / length while t <= 1 and k from -0.5
 *   by res / width while k <= 0.5). Each point is coord + (rand() % 10) / 250.0 for x and y and / 800.0 for z, drawn in that order,
 *   added in FP64 and rounded to float32. rand() is glibc's (TYPE_3: r_i = r_{i-3} + r_{i-31} mod 2^32, output r >> 1, 310 outputs
 *   discarded after seeding, seed 0 taken as 1) started from srand(rand_seed): 1 is a process that never called srand, as the node is.
 *   Maps 4 and 11 call srand(time(NULL)) after their first two walls: srand_seed stands in for time(NULL). Map 2's trees and the cubes
 *   of maps 4 and 11 are drawn from the same stream, so their positions follow the points before them. Roads (map 9) take
 *   length = sqrt((x^2 + y^2) + z^2) and expand / sqrt(expand's squared norm) for Eigen's norm and normalize; with the shipped map 9
 *   every road has dir.y = 0, so no order of that reduction changes a bit (real Eigen's vectorised order is not pinned here).
 * ISDF_WORLD_PERLIN: mockamap's perlin3D (maps.cpp) on a BasicInfo of size[0..2] voxels, scale and seed: the permutation is libstdc++'s
 *   std::shuffle of 0..255 with std::default_random_engine(seed); tnoise(i, j, k) = sum over it = 1..fractal of (attenuation / it) *
 *   noise(dfv i complexity, dfv j complexity, dfv k complexity), dfv = 2^it, in FP64 with nothing contracted; the threshold is the
 *   tpos-th smallest value, tpos = (int)(X Y Z (1 - fill)); the points are the voxels with tnoise > threshold in (i, j, k) order (k
 *   fastest) at (i / scale - X / (2 scale), j / scale - Y / (2 scale), k / scale).
 * ISDF_WORLD_BOXES: mockamap's randomMapGenerate: obstacle_number x (x, y, w, h) drawn with std::uniform_real_distribution<double> on
 *   std::default_random_engine(seed) (libstdc++), each box's shell emitted in (r, s, t) order. The shell test is "some factor of the
 *   reference's six-factor int product is zero"; the reference's product overflows int for boxes wider than about 40 voxels, so a box
 *   whose product can reach 2^31 ((widNum - 1)^4 (heiNum - 1)^2 >= 2^31) is refused with ISDF_ERR_INVALID.
 * mockamap's node derives the sizes from its VoxelWidth and MapBound parameters (mockamap.cpp:96-111): size = floor(min(|MapBound[0]|,
 *   |MapBound[1]|)), floor(min(|MapBound[2]|, |MapBound[3]|)), floor(MapBound[5]) metres, scale = 1 / VoxelWidth, and each size times
 *   scale truncated to int. isdf_world_default_params gives globalmap_gene.launch (resolution 0.6, init 1, 1, 1, rand_seed 1, srand_seed
 *   0, map_id 4 as the launch file) and mockamap.launch (seed 511, complexity 0.03, fill 0.3, fractal 1, attenuation 0.1, widths 0.6 to
 *   1.5, 50 obstacles, 10 x 10 x 3 m at 0.1 m: size 100 x 100 x 30, scale 10).
 * The call needs a context for its stream and scratch, not a map or a shape, and counts its launches in isdf_stats.kernel_launches.
 *   isdf_world_cloud_device writes d_points (cap x 4 float32, device) on cuda_stream and returns after at most one 8-byte read (the
 *   Perlin world's count; the other kinds' sizes are known on the host). Guarantees: the same bits run to run, through either form.
 * Errors: ISDF_ERR_INVALID for a NULL pointer, cap < 0 (points may be NULL when cap = 0), an unknown kind or map_id, a non-finite or
 *   non-positive cloud_resolution or scale, non-finite init, a non-positive size, size[0] size[1] size[2] >= 2^31, fractal < 1 or
 *   2^fractal max(size) |complexity| or 2^fractal max(size) >= 2^31 (the reference's int conversions), non-finite complexity, fill or
 *   attenuation, tpos outside [0, X Y Z) (the reference throws std::out_of_range), obstacle_number < 0, width_min > width_max or a
 *   non-finite width, a box as above, a non-zero reserved_, a loop of more than 2^31 steps, and a cloud beyond 2^63 bytes. */
typedef enum isdf_world_kind { ISDF_WORLD_GLOBALMAP = 1, ISDF_WORLD_PERLIN = 2, ISDF_WORLD_BOXES = 3 } isdf_world_kind;
typedef struct isdf_world_params {
    int32_t kind, map_id;                 /* globalmap: mapGene(map_id), 1..11 */
    uint32_t rand_seed, srand_seed;       /* glibc state at the start (1: never seeded); what srand(time(NULL)) gets in maps 4 and 11 */
    double cloud_resolution, init[3];     /* globalmap_gene.launch: 0.6; init_x, init_y, init_z 1, 1, 1 */
    uint32_t seed; int32_t size[3];       /* mockamap: BasicInfo's seed and sizeX, sizeY, sizeZ (voxels) */
    double scale;                         /* 1 / VoxelWidth */
    double complexity, fill, attenuation; /* perlin3D */
    int32_t fractal, obstacle_number;     /* perlin3D; randomMapGenerate */
    double width_min, width_max;          /* randomMapGenerate */
    int32_t reserved_[2];                 /* must be 0 */
} isdf_world_params;
int isdf_world_default_params(int kind, isdf_world_params *p);
int isdf_world_cloud(isdf_ctx *ctx, const isdf_world_params *p, int64_t cap, float *points, int64_t *n);
int isdf_world_cloud_device(isdf_ctx *ctx, const isdf_world_params *p, int64_t cap, float *d_points, int64_t *n, void *cuda_stream);

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
