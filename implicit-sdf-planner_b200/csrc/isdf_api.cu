// libisdf_b200.so — C-ABI layer (include/isdf.h) over the sm_90a kernels. No CPU fallback anywhere: every entry
// point either runs CUDA kernels or fails with ISDF_ERR_CUDA / ISDF_ERR_STATE.
#include "../../include/isdf.h"
#include "isdf_types.cuh"
#include "isdf_discrete.cuh"
#include "isdf_swept.cuh"
#include "isdf_minco.cuh"
#include "isdf_frontend.cuh"
#include "isdf_frontpath.cuh"
#include "isdf_lbfgs.cuh"
#include "isdf_midend.cuh"
#include "isdf_clearance.cuh"
#include "isdf_certify.cuh"
#include "isdf_map.cuh"
#include <queue>
#include "isdf_host_mesh.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>
#include <limits>

using namespace isdf;

__global__ void k_mesh_cells(const __grid_constant__ DevMesh M, int nx, int ny, int nz, double lx, double ly, double lz, double cell,
                             float *dist, uint32_t *seed);

__global__ void k_mesh_cell_lists(const __grid_constant__ DevMesh M, long long ncell, double hd, double list_reach, uint16_t *cnt,
                                  const uint32_t *off, uint32_t *cand, float *cand_lb);
__global__ void k_mesh_cell_pack(long long ncell, const float *dist, const uint32_t *seed, const uint32_t *off, const uint16_t *cnt, uint4 *rec);

static thread_local std::string g_err;
static int fail(int code, const std::string &msg) { g_err = msg; return code; }

#define CU_TRY(expr)                                                                                  \
    do {                                                                                              \
        cudaError_t e__ = (expr);                                                                     \
        if (e__ != cudaSuccess) {                                                                     \
            return fail(ISDF_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__));          \
        }                                                                                             \
    } while (0)

// The one failure path of the entry points whose outputs include/isdf.h poisons: run body() and, when it fails, poison().
template <typename Body, typename Poison>
static int poison_on_failure(Body body, Poison poison) {
    const int r = body();
    if (r) poison();
    return r;
}
static void nan_fill(double *h, long long n) { if (h) for (long long i = 0; i < n; i++) h[i] = std::numeric_limits<double>::quiet_NaN(); }

static int minco_fits(int N0) {
    if (minco_smem_bytes(N0) > 220 * 1024) return fail(ISDF_ERR_UNSUPPORTED, "pieces per problem too large for the shared-memory banded solver (N0 <= 290)");
    return 0;
}

// The MINCO forward / adjoint workspace (isdf_minco.cuh) of one batched optimiser: B problems of N0 pieces.
struct MincoWork {
    DevBuf<double> d_T, d_C, d_lu, d_energy, d_gC, d_gT, d_out;
    int ensure(int B, int N0) {
        if (int r = minco_fits(N0)) return r;
        const size_t BN = (size_t)B * N0, smem = minco_smem_bytes(N0);
        CU_TRY(d_T.ensure(BN)); CU_TRY(d_C.ensure(18 * BN)); CU_TRY(d_lu.ensure(78 * BN)); CU_TRY(d_energy.ensure(B));
        CU_TRY(d_gC.ensure(18 * BN)); CU_TRY(d_gT.ensure(BN)); CU_TRY(d_out.ensure(19 * BN + 1));
        CU_TRY(cudaFuncSetAttribute(k_minco_forward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CU_TRY(cudaFuncSetAttribute(k_minco_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        return 0;
    }
    // the workspace's part of the arguments; the terms (swept volume, discrete output, cost and gradient) are the caller's
    MincoArgs args(int B, int N0, const double *head, const double *tail, int bc_stride, double rho, const double *x) {
        MincoArgs M = {};
        M.B = B; M.N = N0; M.x = x; M.head = head; M.tail = tail; M.bc_stride = bc_stride; M.rho = rho;
        M.T = d_T.p; M.C = d_C.p; M.lu = d_lu.p; M.energy = d_energy.p; M.gC_e = d_gC.p; M.gT_e = d_gT.p;
        return M;
    }
};

// One plain struct per subsystem; each keeps the flag that says its state is valid next to the buffers that state lives in. Every
// buffer owns its memory; ~isdf_ctx releases the rest.
struct isdf_ctx {
    int device = 0;
    isdf_config cfg;
    DevCfg dcfg;
    int rank = 0, world = 1;   // shard
    cudaStream_t stream = nullptr, aux_stream = nullptr;   // aux: work-item build, off the evaluation's critical path
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_main_done = nullptr, ev_items_done = nullptr;
    int warp_slots = 132 * 16;   // resident warps of the mesh kernel on this device (SMs x CTAs/SM x warps/CTA)
    int sm_count = 132, mesh_blocks = 4, analytic_blocks = 4;   // persistent grids: one CTA per resident slot
    size_t smem_per_sm = 228 * 1024;   // shared memory of one SM (H100: 228 KB, at most 227 KB to one CTA)
    int clr_blocks = 1;                // resident CTAs per SM of the clearance scan kernel
    isdf_stats stats = {};
    struct {
        bool have_map = false;
        DevGrid grid = {};
        DevBuf<uint32_t> d_bits;
        long long points_used = 0, points_skipped = 0;   // isdf_set_map_cloud*; 0 for dense maps
    } map;
    struct {   // the robot shape; the buffers hold a mesh's device view
        bool have_shape = false;
        DevShape shape = {};
        DevBuf<BvhNode> d_nodes; DevBuf<WideNode> d_wnodes; DevBuf<double> d_tris, d_pn, d_obb; DevBuf<float> d_cell_dist; DevBuf<uint32_t> d_cell_seed, d_cell_off, d_cand; DevBuf<float> d_cand_lb; DevBuf<uint16_t> d_cell_cnt; DevBuf<uint4> d_cell_rec; DevBuf<WnNode> d_wn;
        double list_reach = 0;  // radius (cell-centre distance) up to which cells got candidate lists (isdf_dbg_mesh_grid)
    } mesh;
    struct {   // discrete evaluation: scan / epilogue scratch and the work-item schedule
        long long order_for = -1;    // (N, rank, world) signature the work items are valid for
        bool items_pending = false;  // the aux stream is building them
        DevBuf<double> d_piece_cost;
        DevBuf<int> d_tickets;      // pieces_done counter of the epilogue kernel
        DevBuf<double> d_tot; DevBuf<unsigned> d_split_done;   // per-sample collision sums handed from the scan kernels to the epilogue
        DevBuf<int> d_items, d_item_count; DevBuf<unsigned> d_work, d_split_work; DevBuf<double> d_subsum;   // work items (longest first, heavy samples split)
        DevBuf<unsigned long long> d_counter;   // {pairs, then k_discrete_prologue's {codes requested, runs, overflowed runs, codes written}}
        DevBuf<double> d_pose; DevBuf<int2> d_wl_desc; DevBuf<uint32_t> d_wl_codes;   // mesh launches: per local sample pose and window list
        int wl_budget = WL_CODES_PER_SAMPLE;   // window-list codes per local sample (isdf_dbg_window_lists; 0: no lists)
        long long wl_samples = 0, wl_cap = 0;  // local samples and list capacity of the last launch with a prologue
        bool no_items = false;       // diagnostics: always launch in natural order, never split (isdf_dbg_schedule)
        int warp_slots_override = 0; // diagnostics: pretend the device has this many resident warps (forces splitting)
        // the last launch, for isdf_dbg_item_table: its local samples and shard, whether its scan read a work-item table, and the
        // builder it enqueued after itself (0 none, 1 k_build_items<true>, 2 k_build_items<false>) with that builder's arguments
        long long last_M = 0;
        int last_rank = 0, last_world = 1, last_max_split = 0, last_warp_slots = 0, last_builder = 0;
        bool last_have_items = false;
    } disc;
    struct {   // host entry points of the discrete and swept-volume terms: one pinned block, one copy each way
        PinnedBuf<double> h;
        DevBuf<double> d_C, d_out;
    } stage;
    struct {   // batched callback (isdf_minco.cuh); B = 0: none evaluated yet
        MincoWork minco;
        DevBuf<double> d_x, d_bc, d_cost, d_grad, d_Cpp, d_sv;
        int B = 0, N0 = 0;
    } batch;
    struct LbfgsBufs {   // device-resident lock-step L-BFGS (isdf_lbfgs.cuh)
        DevBuf<double> d_x, d_f, d_grad, d_state; DevBuf<int> d_int, d_head;
        PinnedBuf<int> h_active;
    } lbfgs;
    struct {   // mid-end (isdf_midend.cuh): buffers of its own, so that no mid-end call touches the back end's batch, swept or L-BFGS state
        MincoWork minco;
        DevBuf<double> d_x, d_bc, d_wp, d_pc, d_cost, d_grad;
        LbfgsBufs lb;
    } mid;
    SweptState sv;   // swept volume
    struct {   // front end attitude kernels (isdf_frontend.cuh)
        bool ready = false;
        DevBuf<double> d_rot; DevBuf<uint8_t> d_kernels, d_order, d_ok; DevBuf<uint32_t> d_masks, d_out;
        DevBuf<int> d_ind; DevBuf<double> d_father, d_child;
        DevBuf<uint2> d_core, d_urows, d_surv, d_chunks; DevBuf<uint4> d_tab; int nurow = 0, nchunk = 0, ntab = 0; DevBuf<unsigned> d_count; int ncore = 0;
        int xk = 0, yk = 0, ks = 0;
        double max_roll = 0, max_pitch = 0, ang_res = 0, margin = 0;
    } fe;
    struct {   // front-end path search (isdf_frontpath.cuh): rebuilt from the current map and kernels by every call, so nothing here outlives them
        DevBuf<uint32_t> d_trav, d_front, d_colliding; DevBuf<unsigned long long> d_g; DevBuf<unsigned> d_flags;
        DevBuf<int> d_tgt, d_len, d_off, d_nodes; DevBuf<double> d_xyz, d_rp, d_cost; DevBuf<uint8_t> d_found;
        PinnedBuf<unsigned> h_flag;
        cudaEvent_t ev[4] = {};
        isdf_frontpath_info info = {};
    } fp;
    struct {   // trajectory clearance check (isdf_clearance.cuh)
        DevBuf<double> d_in, d_clear; DevBuf<long long> d_vox; DevBuf<ClrSummary> d_sum; DevBuf<int> d_cursor;
        DevBuf<unsigned long long> d_counters;   // {candidate pairs, exact mesh searches} of the last check (isdf_dbg_clearance_counts)
    } clr;
    struct {   // continuous certificate (isdf_certify.cuh): samples, the two interval lists of the round loop, leaves, per-trajectory state
        DevBuf<double> d_in, d_toff, d_st, d_sc; DevBuf<int> d_sp, d_hit, d_tot, d_cursor; DevBuf<long long> d_sv;
        DevBuf<CertInterval> d_iv[2]; DevBuf<CertScratch> d_scr; DevBuf<CertLeaf> d_leaves; DevBuf<CertTraj> d_traj; DevBuf<CertSummary> d_sum;
        PinnedBuf<int> h_tot;
        long long last_leaves = 0;   // leaves of the last call (isdf_dbg_certify_leaves)
    } cert;
    struct {   // peer-memory reduction (isdf_peer.cuh)
        DevBuf<char> buf;                    // own exchange buffer (exported through CUDA IPC)
        void *open[PEER_MAX] = {};           // peers' buffers opened here (null for self / unused)
        PeerArgs args = {};                  // world == 0: not connected
        bool fused = false;                  // sharded *_device evaluations finish with the exchange
        int world_alloc = 0, cap = 0;
        DevBuf<int> d_status;
        void close_handles() { for (void *&p : open) if (p) { cudaIpcCloseMemHandle(p); p = nullptr; } }
    } peer;

    ~isdf_ctx() {
        peer.close_handles();
        peer.buf = {};
        for (cudaEvent_t e : {ev0, ev1, ev_main_done, ev_items_done}) if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : fp.ev) if (e) cudaEventDestroy(e);
        if (aux_stream) cudaStreamDestroy(aux_stream);
        if (stream) cudaStreamDestroy(stream);
    }
};

static int set_device(isdf_ctx *c) { CU_TRY(cudaSetDevice(c->device)); return 0; }
// the context's device, with the work enqueued on its stream (and, with aux, on its work-item stream) finished
static int sync_ctx(isdf_ctx *c, bool aux = false) {
    if (set_device(c)) return ISDF_ERR_CUDA;
    CU_TRY(cudaStreamSynchronize(c->stream));
    if (aux) CU_TRY(cudaStreamSynchronize(c->aux_stream));
    return 0;
}

extern "C" const char *isdf_last_error(void) { return g_err.c_str(); }

extern "C" int isdf_default_config(isdf_config *cfg) {
    if (!cfg) return fail(ISDF_ERR_INVALID, "cfg is NULL");
    // plan_manager/config/config_CappedCone.yaml
    cfg->vehicle_mass = 0.61; cfg->grav_acc = 9.8; cfg->horiz_drag = 0.10; cfg->vert_drag = 0.10; cfg->paras_drag = 0.01; cfg->speed_eps = 0.0001;
    cfg->vmax = 10; cfg->omgmax = 10; cfg->thetamax = 100.0;
    cfg->weight_v = 1000.0; cfg->weight_p = 4000.0; cfg->weight_omg = 1000.0; cfg->weight_theta = 1000.0;
    cfg->smoothing_eps = 1.0e-2; cfg->safety_hor = 0.866; cfg->occupancy_resolution = 1.0;
    cfg->kernel_size = 13; cfg->integral_intervs = 64; cfg->threads_num = 30;
    // the LIVE reference callback (hpp:358-430): collision through the swept-volume term only; grad_cost_p is dead code there, so the
    // discrete collision term is opt-in (flags |= ISDF_WITH_COLLISION) — a default BackEnd must not penalise collision twice
    cfg->flags = ISDF_WITH_DYNAMICS;
    return 0;
}

extern "C" int isdf_create(const isdf_config *cfg, int device, isdf_ctx **out) {
    if (!cfg || !out) return fail(ISDF_ERR_INVALID, "cfg/out is NULL");
    if (cfg->integral_intervs < 1 || cfg->kernel_size < 1 || !(cfg->occupancy_resolution > 0) || !(cfg->vehicle_mass > 0) ||
        !(cfg->smoothing_eps > 0))
        return fail(ISDF_ERR_INVALID, "config out of range");
    int ndev = 0;
    CU_TRY(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(ISDF_ERR_CUDA, "no such CUDA device (this library has no CPU fallback)");
    CU_TRY(cudaSetDevice(device));
    // fail loudly if the sm_90a image cannot run here
    int nb_mesh = 0, nb_analytic = 0, nb_clr = 0;
    CU_TRY(discrete_resident_blocks(&nb_mesh, &nb_analytic));
    CU_TRY(clearance_resident_blocks(&nb_clr));
    // pose-window offsets are packed 10 bits per axis (isdf_discrete.cuh); the inclusive index range of a window is at most
    // kernel_size + 2 voxels when the map resolution equals occupancy_resolution (isdf_set_map checks the resolution)
    if (cfg->kernel_size + 2 > WINDOW_AXIS_MAX) return fail(ISDF_ERR_UNSUPPORTED, "kernel_size too large (pose windows are limited to 1023 voxels per axis)");
    isdf_ctx *c = new isdf_ctx();
    c->device = device; c->cfg = *cfg;
    {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, device) == cudaSuccess && nb_mesh > 0 && nb_analytic > 0) {
            c->sm_count = prop.multiProcessorCount;
            c->smem_per_sm = prop.sharedMemPerMultiprocessor;
            c->mesh_blocks = nb_mesh; c->analytic_blocks = nb_analytic;
            c->warp_slots = prop.multiProcessorCount * nb_mesh * DISC_WARPS;
        }
        c->clr_blocks = std::max(nb_clr, 1);
    }
    DevCfg &d = c->dcfg;
    d.fp.mass = cfg->vehicle_mass; d.fp.grav = cfg->grav_acc; d.fp.dh_over_m = cfg->horiz_drag / cfg->vehicle_mass;
    d.fp.cp = cfg->paras_drag; d.fp.veps = cfg->speed_eps;
    d.vmax2 = cfg->vmax * cfg->vmax; d.omgmax2 = cfg->omgmax * cfg->omgmax; d.thetamax = cfg->thetamax;
    d.wv = cfg->weight_v; d.wp = cfg->weight_p; d.womg = cfg->weight_omg; d.wtheta = cfg->weight_theta;
    d.mu = cfg->smoothing_eps; d.safety = cfg->safety_hor;
    d.half_bd = (cfg->kernel_size * cfg->occupancy_resolution) / 2;
    d.K = cfg->integral_intervs; d.flags = cfg->flags;
    cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->aux_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_main_done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_items_done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreate(&c->ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&c->ev1);
    if (e == cudaSuccess) e = c->disc.d_counter.ensure(5);
    if (e == cudaSuccess) e = cudaMemset(c->disc.d_counter.p, 0, 5 * sizeof(unsigned long long));
    if (e != cudaSuccess) { delete c; return fail(ISDF_ERR_CUDA, std::string("isdf_create: ") + cudaGetErrorString(e)); }
    *out = c;
    return 0;
}

extern "C" int isdf_destroy(isdf_ctx *c) {
    if (!c) return 0;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    cudaStreamSynchronize(c->aux_stream);
    delete c;
    return 0;
}

extern "C" int isdf_get_stats(isdf_ctx *c, isdf_stats *out) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    *out = c->stats;
    return 0;
}

extern "C" int isdf_set_shard(isdf_ctx *c, int rank, int world) {
    if (!c || world < 1 || rank < 0 || rank >= world) return fail(ISDF_ERR_INVALID, "bad shard");
    if (world > c->cfg.integral_intervs + 1) return fail(ISDF_ERR_INVALID, "world larger than samples per piece");
    c->rank = rank; c->world = world; c->disc.order_for = -1;
    return 0;
}

// ---- shapes ---------------------------------------------------------------------------------------------------
static void shape_common(isdf_ctx *c, const double *rot, const double *trans) {
    DevShape &s = c->mesh.shape;
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int i = 0; i < 9; i++) s.rot[i] = rot ? rot[i] : I[i];
    for (int i = 0; i < 3; i++) s.trans[i] = trans ? trans[i] : 0.0;
    // CSG helper rotations: rotate(other, angle = acos(0), axis) of Shape.hpp:2021-2041 for axis = Y x X and Z x X
    const double ang = std::acos(0.0), sn = std::sin(ang), cs = std::cos(ang), mm = 1 - cs;
    auto fill = [&](double x, double y, double z, double *R) {
        R[0] = mm * x * x + cs;     R[1] = mm * x * y + z * sn; R[2] = mm * z * x - y * sn;
        R[3] = mm * x * y - z * sn; R[4] = mm * y * y + cs;     R[5] = mm * y * z + x * sn;
        R[6] = mm * z * x + y * sn; R[7] = mm * y * z - x * sn; R[8] = mm * z * z + cs;
    };
    fill(0, 0, -1, s.csg_ry);  // (0,1,0) x (1,0,0)
    fill(0, 1, 0, s.csg_rz);   // (0,0,1) x (1,0,0)
}

extern "C" int isdf_set_shape_analytic(isdf_ctx *c, int kind, const double *params, int nparams, const double *rot, const double *trans) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (kind < 0 || kind >= ISDF_SHAPE_MESH) return fail(ISDF_ERR_INVALID, "kind is not an analytic shape");
    if (nparams < 0 || nparams > 12 || (nparams > 0 && !params)) return fail(ISDF_ERR_INVALID, "bad params");
    std::memset(&c->mesh.shape, 0, sizeof(c->mesh.shape));
    c->mesh.shape.kind = kind;
    for (int i = 0; i < nparams; i++) c->mesh.shape.par[i] = params[i];
    shape_common(c, rot, trans);
    c->mesh.have_shape = true; c->fe.ready = false;
    c->disc.order_for = -1;   // work items of another shape class may carry split slots
    return 0;
}

extern "C" int isdf_set_shape_named(isdf_ctx *c, const char *name, const double *rot, const double *trans) {
    if (!c || !name) return fail(ISDF_ERR_INVALID, "NULL argument");
    struct Entry { const char *name; int kind; int n; double p[12]; };
    // constants are the reference classes' hard-coded members (Shape.hpp:609,827,863,898-900,936,1003-1005,1052,1149,1214,
    // 1239,1293,1346-1349,1520,1575,1630)
    static const Entry table[] = {
        {"Ball", ISDF_SHAPE_BALL, 1, {1.0}},
        {"Point", ISDF_SHAPE_POINT, 0, {0}},
        {"Torus", ISDF_SHAPE_TORUS, 2, {2.5, 0.3}},
        {"Torus_big", ISDF_SHAPE_TORUS, 2, {3.5, 0.3}},
        {"Cappedtorus", ISDF_SHAPE_CAPPED_TORUS, 4, {0, 0, 3.5, 0.3}},  // sc filled below: (sin 40, cos 40), radians
        {"CappedCone", ISDF_SHAPE_CAPPED_CONE, 2, {2.0, 0.8}},
        {"RoundedCone", ISDF_SHAPE_ROUNDED_CONE, 3, {1.5, 0.6, 4.5}},
        {"WireframeBox", ISDF_SHAPE_WIREFRAME_BOX, 4, {1.8, 2.5, 3.5, 0.1}},
        {"BendLinear", ISDF_SHAPE_BEND_LINEAR, 2, {2.0, 0.25}},
        {"BendLinear_big", ISDF_SHAPE_BEND_LINEAR, 2, {3.2, 0.45}},
        {"TwistBox", ISDF_SHAPE_TWIST_BOX, 4, {2.0, 2.0, 2.0, 3.14159265358979323846 / 6}},
        {"BendBox", ISDF_SHAPE_BEND_BOX, 4, {2.0, 2.0, 2.0, 0.5}},
        {"Table", ISDF_SHAPE_TABLE, 12, {0.0, 0.0, 0.0, 3.5, 1.75, 0.7, 2.8, 1.05, 0.0, 3.5, 1.75, 2.8}},
        {"Trefoil", ISDF_SHAPE_TREFOIL, 0, {0}},
        {"SmoothDifference", ISDF_SHAPE_SMOOTH_DIFFERENCE, 4, {3.0, 3.0, 0.5, 1.0}},
        {"SmoothIntersection", ISDF_SHAPE_SMOOTH_INTERSECTION, 4, {3.0, 3.0, 0.5, 1.0}},
        {"SmoothIntersection_big", ISDF_SHAPE_SMOOTH_INTERSECTION, 4, {9.0, 9.0, 1.5, 3.0}},
        {"CSG", ISDF_SHAPE_CSG, 0, {0}},
    };
    for (const Entry &e : table) {
        if (std::strcmp(e.name, name) == 0) {
            double p[12];
            for (int i = 0; i < 12; i++) p[i] = e.p[i];
            if (e.kind == ISDF_SHAPE_CAPPED_TORUS) { p[0] = std::sin(40); p[1] = std::cos(40); }
            return isdf_set_shape_analytic(c, e.kind, p, e.n, rot, trans);
        }
    }
    // the reference falls back to the mesh Generalshape for unknown names (swm:269-274); a mesh needs its geometry
    return fail(ISDF_ERR_INVALID, std::string("unknown analytic shape name '") + name + "' (use isdf_set_shape_mesh for OBJ bodies)");
}

extern "C" int isdf_set_shape_mesh(isdf_ctx *c, const double *V, int nV, const int32_t *F, int nF, const double *poly_params) {
    return isdf_set_shape_mesh_ex(c, V, nV, F, nF, poly_params, ISDF_MESH_SIGN_AUTO);
}

extern "C" int isdf_set_shape_mesh_ex(isdf_ctx *c, const double *V, int nV, const int32_t *F, int nF, const double *poly_params, int sign_mode) {
    if (!c || !V || !F) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (sign_mode < 0 || sign_mode > 2) return fail(ISDF_ERR_INVALID, "bad sign_mode");
    if (set_device(c)) return ISDF_ERR_CUDA;
    HostMesh hm; std::string err;
    // the bitmap shortcut is sized for the smallest bound the kernels use: safety_hor (discrete) — the swept path uses
    // 2*safety_hor + 0.1 >= safety_hor
    if (!build_host_mesh(V, nV, F, nF, poly_params, c->cfg.safety_hor, hm, err, sign_mode))
        return fail(err.find("not a closed") != std::string::npos ? ISDF_ERR_UNSUPPORTED : ISDF_ERR_INVALID, err);
    // the uploads may reallocate the buffers the current shape lives in: give it up (and what was built on it) first
    c->mesh.have_shape = false; c->fe.ready = false;
    c->disc.order_for = -1;
    if (!hm.wn.empty()) CU_TRY(c->mesh.d_wn.upload(hm.wn.data(), hm.wn.size(), c->stream));
    CU_TRY(c->mesh.d_nodes.upload(hm.nodes.data(), hm.nodes.size(), c->stream));
    CU_TRY(c->mesh.d_wnodes.upload(hm.wnodes.data(), hm.wnodes.size(), c->stream));
    CU_TRY(c->mesh.d_tris.upload(hm.tris.data(), hm.tris.size(), c->stream));
    CU_TRY(c->mesh.d_pn.upload(hm.pnormals.data(), hm.pnormals.size(), c->stream));
    CU_TRY(c->mesh.d_obb.upload(hm.leaf_obb.data(), hm.leaf_obb.size(), c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    std::memset(&c->mesh.shape, 0, sizeof(c->mesh.shape));
    c->mesh.shape.kind = ISDF_SHAPE_MESH;
    shape_common(c, nullptr, nullptr);
    DevMesh m = hm.view();
    m.nodes = c->mesh.d_nodes.p; m.wnodes = c->mesh.d_wnodes.p; m.tris = c->mesh.d_tris.p; m.pnormals = c->mesh.d_pn.p; m.leaf_obb = c->mesh.d_obb.p;
    m.wn = hm.wn.empty() ? nullptr : c->mesh.d_wn.p;
    // per-cell signed distance + seed triangle, computed on the device with the freshly uploaded BVH
    const size_t ncell = (size_t)m.gdim[0] * m.gdim[1] * m.gdim[2];
    CU_TRY(c->mesh.d_cell_dist.ensure(ncell));
    CU_TRY(c->mesh.d_cell_seed.ensure(ncell));
    {
        DevMesh build = m;
        build.gdim[0] = 0;            // no grid while it is being built: plain unbounded BVH queries
        build.cell_dist = nullptr; build.cell_seed = nullptr; build.cell_off = nullptr; build.cell_cnt = nullptr; build.cand = nullptr; build.cand_lb = nullptr;
        k_mesh_cells<<<(unsigned)((ncell + 127) / 128), 128, 0, c->stream>>>(build, m.gdim[0], m.gdim[1], m.gdim[2], m.glo[0], m.glo[1], m.glo[2],
                                                                           m.gcell, c->mesh.d_cell_dist.p, c->mesh.d_cell_seed.p);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaStreamSynchronize(c->stream));
    }
    m.cell_dist = c->mesh.d_cell_dist.p; m.cell_seed = c->mesh.d_cell_seed.p;
    m.cell_off = nullptr; m.cell_cnt = nullptr; m.cand = nullptr; m.cand_lb = nullptr;
    // exact candidate lists for every cell a query can land in and not be settled by the cell's distance bracket alone: the discrete
    // path queries within safety_hor of the surface, the swept-volume path within its range bound 2*safety_hor + 0.1 (swm:383) — a
    // flat pass over ~100 listed triangles answers such a query in a tenth of the time of a far-field tree search, and the sign
    // descent of the swept-volume path is a CHAIN of them
    {
        const double hd = 0.5 * std::sqrt(3.0) * m.gcell;
        const double list_reach = std::max(c->cfg.safety_hor, 2.0 * c->cfg.safety_hor + 0.1) + 2.0 * m.ghd;
        c->mesh.list_reach = list_reach;
        CU_TRY(c->mesh.d_cell_cnt.ensure(ncell)); CU_TRY(c->mesh.d_cell_off.ensure(ncell));
        const unsigned warps_grid = (unsigned)((ncell + 3) / 4);
        k_mesh_cell_lists<<<warps_grid, 128, 0, c->stream>>>(m, (long long)ncell, hd, list_reach, c->mesh.d_cell_cnt.p, nullptr, nullptr, nullptr);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        std::vector<uint16_t> cnt(ncell);
        CU_TRY(cudaMemcpyAsync(cnt.data(), c->mesh.d_cell_cnt.p, sizeof(uint16_t) * ncell, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
        std::vector<uint32_t> off(ncell);
        size_t total = 0;
        for (size_t i = 0; i < ncell; i++) { off[i] = (uint32_t)total; total += cnt[i]; }
        if (total > 0 && total < (1ull << 31)) {
            CU_TRY(c->mesh.d_cand.ensure(total)); CU_TRY(c->mesh.d_cand_lb.ensure(total));
            CU_TRY(cudaMemcpyAsync(c->mesh.d_cell_off.p, off.data(), sizeof(uint32_t) * ncell, cudaMemcpyHostToDevice, c->stream));
            k_mesh_cell_lists<<<warps_grid, 128, 0, c->stream>>>(m, (long long)ncell, hd, list_reach, c->mesh.d_cell_cnt.p, c->mesh.d_cell_off.p, c->mesh.d_cand.p, c->mesh.d_cand_lb.p);
            c->stats.kernel_launches++;
            CU_TRY(cudaGetLastError());
            CU_TRY(cudaStreamSynchronize(c->stream));
            m.cell_off = c->mesh.d_cell_off.p; m.cell_cnt = c->mesh.d_cell_cnt.p; m.cand = c->mesh.d_cand.p; m.cand_lb = c->mesh.d_cand_lb.p;
        }
        if (getenv("ISDF_VERBOSE")) {
            size_t listed = 0; for (size_t i = 0; i < ncell; i++) listed += cnt[i] != 0;
            fprintf(stderr, "[isdf] mesh cell grid %d x %d x %d (cell %.3f m), %zu cells with a candidate list, %zu candidates (%.1f MB: ids and lower bounds)\n", m.gdim[0], m.gdim[1],
                    m.gdim[2], m.gcell, listed, total, total * 8e-6);
        }
    }
    // fused 16-byte cell records for the discrete scan kernel's cull stage
    CU_TRY(c->mesh.d_cell_rec.ensure(ncell));
    k_mesh_cell_pack<<<(unsigned)((ncell + 255) / 256), 256, 0, c->stream>>>((long long)ncell, m.cell_dist, m.cell_seed, m.cell_off, m.cell_cnt, c->mesh.d_cell_rec.p);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaStreamSynchronize(c->stream));
    m.cell_rec = c->mesh.d_cell_rec.p;
    c->mesh.shape.mesh = m;
    c->mesh.have_shape = true;
    return 0;
}

__global__ void k_mesh_cell_pack(long long ncell, const float *dist, const uint32_t *seed, const uint32_t *off, const uint16_t *cnt, uint4 *rec) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ncell) return;
    rec[i] = make_uint4(__float_as_uint(dist[i]), seed[i], (off && cnt) ? off[i] : 0u, (off && cnt) ? (uint32_t)cnt[i] : 0u);
}

// signed distance + nearest triangle at every cell centre of the body-frame grid (one thread per cell)
__global__ void k_mesh_cells(const __grid_constant__ DevMesh M, int nx, int ny, int nz, double lx, double ly, double lz, double cell,
                             float *dist, uint32_t *seed) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)nx * ny * nz) return;
    const int iz = (int)(idx % nz), iy = (int)((idx / nz) % ny), ix = (int)(idx / ((size_t)nz * ny));
    const d3 p = mk3(lx + (ix + 0.5) * cell, ly + (iy + 0.5) * cell, lz + (iz + 0.5) * cell);
    d3 c = mk3(0, 0, 0); int tri, feat;
    const double d2 = mesh_closest(M, p, 1e300, c, tri, feat);
    const d3 e = p - c;
    const double *pn = M.pnormals + 21 * (size_t)tri + 3 * feat;
    double side = e.x * pn[0] + e.y * pn[1] + e.z * pn[2];
    if (side == 0.0) { const double *fn = M.pnormals + 21 * (size_t)tri; side = e.x * fn[0] + e.y * fn[1] + e.z * fn[2]; }
    dist[idx] = (float)((side < 0.0 ? -1.0 : 1.0) * sqrt(d2));
    seed[idx] = (uint32_t)tri;
}

// Candidate lists (one warp per cell). Pass 1 (cand == nullptr): count the triangles within d_c + 2 hd of the cell centre and
// store the count (0 for cells that are too far, too deep or whose list would exceed LIST_CAP). Pass 2: fill the lists, sorted by
// ascending distance from the cell centre (ties: triangle index), with each distance's lower bound in cand_lb.
constexpr int LIST_CAP = MESH_LIST_CAP;
__global__ void __launch_bounds__(128) k_mesh_cell_lists(const __grid_constant__ DevMesh M, long long ncell, double hd, double list_reach,
                                                         uint16_t *cnt, const uint32_t *off, uint32_t *cand, float *cand_lb) {
    __shared__ WideStack stk[4];
    __shared__ double s_d2[4][LIST_CAP];   // pass 2: the cell's hits in emission order, then ranked
    __shared__ int s_tri[4][LIST_CAP];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long cell = (long long)blockIdx.x * 4 + warp;
    if (cell >= ncell) return;
    const double dc = fabs((double)M.cell_dist[cell]);
    if (cand == nullptr) { if (lane == 0) cnt[cell] = 0; }
    else if (cnt[cell] == 0) return;
    if (dc > list_reach) return;
    const int nz = M.gdim[2], ny = M.gdim[1];
    const int iz = (int)(cell % nz), iy = (int)((cell / nz) % ny), ix = (int)(cell / ((long long)nz * ny));
    const d3 ctr = mk3(M.glo[0] + (ix + 0.5) * M.gcell, M.glo[1] + (iy + 0.5) * M.gcell, M.glo[2] + (iz + 0.5) * M.gcell);
    // radius: centre distance (float-rounded: add its slack) + two half diagonals, then a relative safety margin
    const double R = (dc + (M.ghd - hd) + 2.0 * hd) * (1.0 + 1e-9) + 1e-12;
    const unsigned lt_mask = (1u << lane) - 1u;
    int n = 0;
    const uint32_t base = cand ? off[cell] : 0u;
    wide_range(M, ctr, R * R, lane, &stk[warp], [&](bool hit, int t, double d2) {
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        const int slot = n + __popc(bal & lt_mask);
        if (cand && hit && slot < LIST_CAP) { s_d2[warp][slot] = d2; s_tri[warp][slot] = t; }
        n += __popc(bal);
    });
    if (cand == nullptr) {
        if (lane == 0) cnt[cell] = (n <= LIST_CAP) ? (uint16_t)n : (uint16_t)0;
        return;
    }
    // rank sort: entry i goes to the number of entries before it in (squared distance, triangle) order
    __syncwarp();
    n = min(n, LIST_CAP);
    for (int i = lane; i < n; i += 32) {
        const double di = s_d2[warp][i];
        const int ti = s_tri[warp][i];
        int rank = 0;
        for (int j = 0; j < n; j++) {
            const double dj = s_d2[warp][j];
            rank += (dj < di || (dj == di && s_tri[warp][j] < ti)) ? 1 : 0;
        }
        cand[base + rank] = (uint32_t)ti;
        // lower bound of the exact distance: relative and absolute slack for the rounding of the FP64 closest-point test, then rounded
        // down to float (monotone in di, so the bounds are non-decreasing along the list)
        cand_lb[base + rank] = __double2float_rd(fmax(sqrt(di) * (1.0 - 1e-9) - 1e-12, 0.0));
    }
}

__global__ void k_shape_query(const __grid_constant__ DevShape S, const double *p, int n, double *sdf, double *grad, int what) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const d3 q = mk3(p[3 * i], p[3 * i + 1], p[3 * i + 2]);
    d3 g = mk3(0, 0, 0);
    double s = 0;
    if (what == ISDF_QUERY_SDF) s = shape_sdf(S, q);
    else if (what == ISDF_QUERY_GRAD) g = shape_grad(S, q);
    else s = shape_sdf_grad(S, q, g);
    if (sdf && what != ISDF_QUERY_GRAD) sdf[i] = s;
    if (grad && what != ISDF_QUERY_SDF) { grad[3 * i] = g.x; grad[3 * i + 1] = g.y; grad[3 * i + 2] = g.z; }
}

extern "C" int isdf_shape_query(isdf_ctx *c, const double *p_rel, int n, double *sdf, double *grad, int what) {
    if (!c || !p_rel || n < 0) return fail(ISDF_ERR_INVALID, "bad argument");
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    if (what < 0 || what > 2) return fail(ISDF_ERR_INVALID, "bad query kind");
    if (n == 0) return 0;
    if (set_device(c)) return ISDF_ERR_CUDA;
    DevBuf<double> dp, ds, dg;
    CU_TRY(dp.upload(p_rel, (size_t)3 * n, c->stream));
    CU_TRY(ds.ensure(n)); CU_TRY(dg.ensure((size_t)3 * n));
    k_shape_query<<<(n + 127) / 128, 128, 0, c->stream>>>(c->mesh.shape, dp.p, n, ds.p, dg.p, what);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    std::vector<double> hs(n), hg((size_t)3 * n);
    CU_TRY(cudaMemcpyAsync(hs.data(), ds.p, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaMemcpyAsync(hg.data(), dg.p, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    if (sdf && what != ISDF_QUERY_GRAD) std::memcpy(sdf, hs.data(), sizeof(double) * n);
    if (grad && what != ISDF_QUERY_SDF) std::memcpy(grad, hg.data(), sizeof(double) * 3 * n);
    return 0;
}

// ---- map ------------------------------------------------------------------------------------------------------
// the limits every map must meet, whichever entry point sets it
static int map_size_check(isdf_ctx *c, long long X, long long Y, long long Z, double res) {
    if (X * Y >= (1ll << 31) / ((Z + 31) / 32)) return fail(ISDF_ERR_INVALID, "map too large");
    if (Z > 65535) return fail(ISDF_ERR_UNSUPPORTED, "Z > 65535");
    // a pose window spans 2 * half_bd / res + 2 voxels per axis of THIS map (its resolution need not equal occupancy_resolution); the scan
    // kernels pack window offsets into 10 bits per axis
    if (c && 2.0 * c->dcfg.half_bd / res + 2.0 > (double)WINDOW_AXIS_MAX)
        return fail(ISDF_ERR_UNSUPPORTED, "map resolution too fine for kernel_size * occupancy_resolution: a pose window would exceed 1023 voxels per axis");
    return 0;
}

// the map the bits in c->map.d_bits describe
static void commit_map(isdf_ctx *c, int X, int Y, int Z, const double *bmin, const double *bmax, double res, long long used, long long skipped) {
    DevGrid &g = c->map.grid;
    g.bits = c->map.d_bits.p; g.X = X; g.Y = Y; g.Z = Z; g.Zw = (Z + 31) / 32; g.res = res;
    for (int a = 0; a < 3; a++) { g.bmin[a] = bmin[a]; g.bmax[a] = bmax[a]; }
    c->map.points_used = used; c->map.points_skipped = skipped;
    c->map.have_map = true;
}

template <typename T>
static int set_map_impl(isdf_ctx *c, const T *occ, int X, int Y, int Z, const double *bmin, double res) {
    if (!c || !occ || !bmin) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (X < 1 || Y < 1 || Z < 1 || !(res > 0)) return fail(ISDF_ERR_INVALID, "bad map size");
    if (int rc = map_size_check(c, X, Y, Z, res)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    c->map.have_map = false;   // d_bits.ensure may free the current grid
    const size_t nvox = (size_t)X * Y * Z;
    DevBuf<T> d_occ;
    cudaError_t e = d_occ.upload(occ, nvox, c->stream);
    const int Zw = (Z + 31) / 32;
    const size_t nwords = (size_t)X * Y * Zw;
    if (e == cudaSuccess) e = c->map.d_bits.ensure(nwords);
    if (e == cudaSuccess) {
        const long long threads = (long long)nwords * 32;
        k_pack_bits<<<(unsigned)((threads + 255) / 256), 256, 0, c->stream>>>(NonZero<T>{d_occ.p}, c->map.d_bits.p, X * Y, Z, Zw);
        c->stats.kernel_launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) return fail(ISDF_ERR_CUDA, std::string("isdf_set_map: ") + cudaGetErrorString(e));
    const int dims[3] = {X, Y, Z};
    double bmax[3];
    for (int a = 0; a < 3; a++) bmax[a] = bmin[a] + dims[a] * res;
    commit_map(c, X, Y, Z, bmin, bmax, res, 0, 0);
    return 0;
}

extern "C" int isdf_set_map_u8(isdf_ctx *c, const uint8_t *occ, int X, int Y, int Z, const double *bmin, double res) {
    return set_map_impl<uint8_t>(c, occ, X, Y, Z, bmin, res);
}
extern "C" int isdf_set_map_f64(isdf_ctx *c, const double *grid_map, int X, int Y, int Z, const double *bmin, double res) {
    return set_map_impl<double>(c, grid_map, X, Y, Z, bmin, res);
}

// ---- map from a point cloud (PCSmapManager::rcvGlobalMapHandler, PCSmap_manager.cpp:111-181) ---------------------------
// the context is checked last, so that every other refusal can be seen without a device
static int cloud_args_check(isdf_ctx *c, const void *pts, int64_t n, int32_t stride, double res) {
    if (!pts) return fail(ISDF_ERR_INVALID, "points is NULL");
    if (n < 1 || n >= (1ll << 32)) return fail(ISDF_ERR_INVALID, "point count must be in [1, 2^32)");
    if (stride < 12 || stride % 4 != 0) return fail(ISDF_ERR_INVALID, "stride_bytes must be a multiple of 4 and at least 12 (x, y, z float32 at 0, 4, 8)");
    if ((uintptr_t)pts % 4 != 0) return fail(ISDF_ERR_INVALID, "points must be 4-byte aligned");
    if (!(res > 0) || !std::isfinite(res)) return fail(ISDF_ERR_INVALID, "res must be finite and positive");
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    return 0;
}

static int cloud_grid_blocks(isdf_ctx *c, long long n) { return (int)std::min<long long>((n + 255) / 256, (long long)c->sm_count * 8); }

// d_pts on the device and ready on stream st (which this synchronises once, for the bounds); the grid is built on c->stream
static int set_map_cloud_impl(isdf_ctx *c, const char *d_pts, long long n, int stride, double res, int thr, cudaStream_t st) {
    const int blocks = cloud_grid_blocks(c, n);
    auto cuda_fail = [&](cudaError_t e) {
        c->map.have_map = false;
        return fail(ISDF_ERR_CUDA, std::string("isdf_set_map_cloud: ") + cudaGetErrorString(e));
    };
    // 1. bounds: exact float extrema of the finite records (order-preserving uint32 min / max) and the number of skipped records
    uint32_t ext[7];
    {
        DevBuf<uint32_t> d_ext;
        cudaError_t e = d_ext.ensure(7);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_ext.p, 0xff, 3 * sizeof(uint32_t), st);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_ext.p + 3, 0, 4 * sizeof(uint32_t), st);
        if (e == cudaSuccess) {
            k_cloud_bounds<<<blocks, 256, 0, st>>>(d_pts, n, stride, d_ext.p);
            c->stats.kernel_launches++;
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(ext, d_ext.p, sizeof(ext), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return cuda_fail(e);
    }
    const long long skipped = ext[6], used = n - skipped;
    if (used == 0) return fail(ISDF_ERR_INVALID, "the cloud has no point with finite coordinates");
    // 2. the reference's frame: HUGE_NUMBER start (PCSmap_manager.cpp:6,11-12), strict updates (:111-143), createGridMap's sizes (Gridmap3D.cpp:25-39)
    double bmin[3], bmax[3], dim[3];
    for (int a = 0; a < 3; a++) {
        float lo, hi;
        const uint32_t ulo = ordered_to_float(ext[a]), uhi = ordered_to_float(ext[3 + a]);
        std::memcpy(&lo, &ulo, 4); std::memcpy(&hi, &uhi, 4);
        bmin[a] = 999999999.0; bmax[a] = -999999999.0;
        if ((double)lo < bmin[a]) bmin[a] = lo;
        if ((double)hi > bmax[a]) bmax[a] = hi;
        dim[a] = std::ceil((bmax[a] - bmin[a]) / res);
    }
    char dims_msg[160];
    std::snprintf(dims_msg, sizeof dims_msg, " (the cloud asks for %.0f x %.0f x %.0f voxels at res %g)", dim[0], dim[1], dim[2], res);
    for (int a = 0; a < 3; a++) {
        if (!(dim[a] >= 1)) return fail(ISDF_ERR_INVALID, std::string("degenerate cloud extent: an axis has fewer than one voxel") + dims_msg);
        if (dim[a] > 2147483647.0) return fail(ISDF_ERR_INVALID, std::string("map too large") + dims_msg);
    }
    const int X = (int)dim[0], Y = (int)dim[1], Z = (int)dim[2];
    if (int rc = map_size_check(c, X, Y, Z, res)) return fail(rc, g_err + dims_msg);
    // 3. occupancy (the previous map is given up from here on)
    c->map.have_map = false;
    CloudFrame F;
    for (int a = 0; a < 3; a++) F.bmin[a] = bmin[a];
    F.res = res; F.X = X; F.Y = Y; F.Z = Z; F.Zw = (Z + 31) / 32;
    const size_t nwords = (size_t)X * Y * F.Zw;
    cudaError_t e = c->map.d_bits.ensure(nwords);
    if (e != cudaSuccess) return cuda_fail(e);
    const long long pack_threads = (long long)nwords * 32;
    const unsigned pack_blocks = (unsigned)((pack_threads + 255) / 256);
    DevBuf<uint32_t> d_cnt;   // sta_threshold > 1: per-voxel counts, freed after the final synchronise
    if (thr <= 0) {
        k_pack_bits<<<pack_blocks, 256, 0, c->stream>>>(AllSet{}, c->map.d_bits.p, X * Y, Z, F.Zw);
        c->stats.kernel_launches++;
        e = cudaGetLastError();
    } else if (thr == 1) {
        e = cudaMemsetAsync(c->map.d_bits.p, 0, nwords * sizeof(uint32_t), c->stream);
        if (e == cudaSuccess) {
            k_cloud_mark<<<blocks, 256, 0, c->stream>>>(d_pts, n, stride, F, c->map.d_bits.p);
            c->stats.kernel_launches++;
            e = cudaGetLastError();
        }
    } else {
        const size_t nvox = (size_t)X * Y * Z;
        e = d_cnt.ensure(nvox);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_cnt.p, 0, nvox * sizeof(uint32_t), c->stream);
        if (e == cudaSuccess) {
            k_cloud_count<<<blocks, 256, 0, c->stream>>>(d_pts, n, stride, F, d_cnt.p);
            k_pack_bits<<<pack_blocks, 256, 0, c->stream>>>(CountAtLeast{d_cnt.p, (uint32_t)thr}, c->map.d_bits.p, X * Y, Z, F.Zw);
            c->stats.kernel_launches += 2;
            e = cudaGetLastError();
        }
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) return cuda_fail(e);
    commit_map(c, X, Y, Z, bmin, bmax, res, used, skipped);
    return 0;
}

extern "C" int isdf_set_map_cloud(isdf_ctx *c, const void *points, int64_t n, int32_t stride_bytes, double res, int32_t sta_threshold) {
    if (int rc = cloud_args_check(c, points, n, stride_bytes, res)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    DevBuf<char> d_pts;
    const size_t bytes = (size_t)n * stride_bytes;
    cudaError_t e = d_pts.ensure(bytes);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_pts.p, points, bytes, cudaMemcpyHostToDevice, c->stream);
    if (e != cudaSuccess) {
        c->map.have_map = false;
        return fail(ISDF_ERR_CUDA, std::string("isdf_set_map_cloud: ") + cudaGetErrorString(e));
    }
    return set_map_cloud_impl(c, d_pts.p, n, stride_bytes, res, sta_threshold, c->stream);
}

extern "C" int isdf_set_map_cloud_device(isdf_ctx *c, const void *d_points, int64_t n, int32_t stride_bytes, double res, int32_t sta_threshold,
                                         void *cuda_stream) {
    if (int rc = cloud_args_check(c, d_points, n, stride_bytes, res)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    return set_map_cloud_impl(c, (const char *)d_points, n, stride_bytes, res, sta_threshold, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_get_map_info(isdf_ctx *c, isdf_map_info *out) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    if (set_device(c)) return ISDF_ERR_CUDA;
    const DevGrid &g = c->map.grid;
    DevBuf<unsigned long long> d_pop;
    unsigned long long pop = 0;
    const long long nwords = (long long)g.X * g.Y * g.Zw;
    CU_TRY(d_pop.ensure(1));
    CU_TRY(cudaMemsetAsync(d_pop.p, 0, sizeof(unsigned long long), c->stream));
    k_popcount<<<cloud_grid_blocks(c, nwords), 256, 0, c->stream>>>(g.bits, nwords, d_pop.p);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(&pop, d_pop.p, sizeof(pop), cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    std::memset(out, 0, sizeof(*out));
    out->X = g.X; out->Y = g.Y; out->Z = g.Z; out->res = g.res;
    for (int a = 0; a < 3; a++) { out->bmin[a] = g.bmin[a]; out->bmax[a] = g.bmax[a]; }
    out->occupied_voxels = (int64_t)pop;
    out->points_used = c->map.points_used; out->points_skipped = c->map.points_skipped;
    return 0;
}

// the bit grid expanded to one T per voxel, a bounded number of (x, y) rows at a time through device scratch
template <typename T>
static int get_map_impl(isdf_ctx *c, T *out, int64_t n) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    const DevGrid &g = c->map.grid;
    const long long rows = (long long)g.X * g.Y;
    if (n != rows * g.Z) return fail(ISDF_ERR_INVALID, "n must be X*Y*Z of the map");
    if (set_device(c)) return ISDF_ERR_CUDA;
    const long long chunk_rows = std::max<long long>(1, (32ll << 20) / ((long long)g.Z * sizeof(T)));   // <= 32 MiB of scratch per chunk
    DevBuf<T> d_out;
    CU_TRY(d_out.ensure((size_t)std::min(rows, chunk_rows) * g.Z));
    for (long long r0 = 0; r0 < rows; r0 += chunk_rows) {
        const int nr = (int)std::min(chunk_rows, rows - r0);
        const long long cnt = (long long)nr * g.Z;
        k_unpack_bits<T><<<cloud_grid_blocks(c, cnt), 256, 0, c->stream>>>(g.bits, d_out.p, r0, nr, g.Z, g.Zw);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(out + r0 * g.Z, d_out.p, cnt * sizeof(T), cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
    }
    return 0;
}

extern "C" int isdf_get_map_u8(isdf_ctx *c, uint8_t *occ, int64_t n) { return get_map_impl<uint8_t>(c, occ, n); }
extern "C" int isdf_get_map_f64(isdf_ctx *c, double *grid_map, int64_t n) { return get_map_impl<double>(c, grid_map, n); }

// getPointsInAABB (pcs:148-170): one CTA; thread = (x, y) row of the clamped index box — popcount of the row's z-run, block-wide exclusive scan
// for the row's output offset, then every thread writes its row's voxel centres in z order: the reference's x -> y -> z output order
__global__ void __launch_bounds__(256) k_points_in_aabb(const DevGrid G, double cx, double cy, double cz, double h, double *out, int cap, int *count) {
    __shared__ int warp_tot[8];
    __shared__ int running;
    const int ix0 = grid_axis_index(cx - h, G.bmin[0], G.bmax[0], G.res, G.X), ix1 = grid_axis_index(cx + h, G.bmin[0], G.bmax[0], G.res, G.X);
    const int iy0 = grid_axis_index(cy - h, G.bmin[1], G.bmax[1], G.res, G.Y), iy1 = grid_axis_index(cy + h, G.bmin[1], G.bmax[1], G.res, G.Y);
    const int iz0 = grid_axis_index(cz - h, G.bmin[2], G.bmax[2], G.res, G.Z), iz1 = grid_axis_index(cz + h, G.bmin[2], G.bmax[2], G.res, G.Z);
    const int ny = iy1 - iy0 + 1, nrows = (ix1 - ix0 + 1) * ny;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) running = 0;
    __syncthreads();
    for (int base = 0; base < nrows; base += blockDim.x) {
        const int r = base + threadIdx.x;
        int i = 0, j = 0, cnt = 0;
        if (r < nrows) {
            i = ix0 + r / ny; j = iy0 + r % ny;
            const uint32_t *row = G.bits + ((size_t)i * G.Y + j) * G.Zw;
            for (int wz = iz0 >> 5; wz <= (iz1 >> 5); wz++) {
                uint32_t w = row[wz];
                if (wz == (iz0 >> 5)) w &= 0xffffffffu << (iz0 & 31);
                if (wz == (iz1 >> 5) && (iz1 & 31) != 31) w &= (1u << ((iz1 & 31) + 1)) - 1u;
                cnt += __popc(w);
            }
        }
        int incl = cnt;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        int off = running + incl - cnt;
        for (int w = 0; w < warp; w++) off += warp_tot[w];
        if (r < nrows && cnt > 0) {
            const uint32_t *row = G.bits + ((size_t)i * G.Y + j) * G.Zw;
            for (int k = iz0; k <= iz1; k++)
                if ((row[k >> 5] >> (k & 31)) & 1u) {
                    if (off < cap) { out[3 * off] = (i + 0.5) * G.res + G.bmin[0]; out[3 * off + 1] = (j + 0.5) * G.res + G.bmin[1]; out[3 * off + 2] = (k + 0.5) * G.res + G.bmin[2]; }
                    off++;
                }
        }
        __syncthreads();
        if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < 8; w++) t += warp_tot[w]; running += t; }
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = running;
}

extern "C" int isdf_points_in_aabb(isdf_ctx *c, const double *centre, double half_extent, double *out_points, int cap, int *n) {
    if (!c || !centre || !n || cap < 0 || (cap > 0 && !out_points)) return fail(ISDF_ERR_INVALID, "bad argument");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    if (set_device(c)) return ISDF_ERR_CUDA;
    DevBuf<double> d; DevBuf<int> dn;
    CU_TRY(d.ensure((size_t)3 * (cap > 0 ? cap : 1))); CU_TRY(dn.ensure(1));
    k_points_in_aabb<<<1, 256, 0, c->stream>>>(c->map.grid, centre[0], centre[1], centre[2], half_extent, d.p, cap, dn.p);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    int cnt = 0;
    CU_TRY(cudaMemcpyAsync(&cnt, dn.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    const int m = cnt < cap ? cnt : cap;
    if (m > 0) CU_TRY(cudaMemcpy(out_points, d.p, sizeof(double) * 3 * m, cudaMemcpyDeviceToHost));
    *n = cnt;
    return 0;
}

// ---- obstacle gather (plan_manager.cpp:232-254 / pcs:182-216) -------------------------------------------------------------
struct GatherBox { int a0[3], a1[3], l0[3], l1[3]; };
__device__ __forceinline__ bool gather_includes(const DevGrid &G, const GatherBox &b, int i, int j, int k) {
    if (i < b.a0[0] || i > b.a1[0] || j < b.a0[1] || j > b.a1[1] || k < b.a0[2] || k > b.a1[2]) return false;
    if (!(i > b.l1[0] || i < b.l0[0] || j > b.l1[1] || j < b.l0[1] || k > b.l1[2] || k < b.l0[2])) return false;
    return (G.bits[((size_t)i * G.Y + j) * G.Zw + (k >> 5)] >> (k & 31)) & 1u;
}
// Obstacle gather, one CTA per waypoint, three launches: k_gather_boxes (index boxes of every waypoint), k_gather_points<false> (how many
// voxels each waypoint emits: a voxel belongs to the FIRST waypoint whose box includes it) and, after an exclusive scan over the waypoints
// inside the kernel, k_gather_points<true> (ordered compaction inside the CTA at the waypoint's offset). Output order = the reference's:
// waypoint by waypoint, each box in x -> y -> z order.
__global__ void k_gather_boxes(const DevGrid G, const double *wps, int nQ, double h, double ox, double oy, double oz, GatherBox *boxes) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nQ) return;
    GatherBox b;
    const double c[3] = {wps[3 * q] + ox, wps[3 * q + 1] + oy, wps[3 * q + 2] + oz};
    const double l[3] = {q == 0 ? 999.0 : wps[3 * (q - 1)], q == 0 ? 999.0 : wps[3 * (q - 1) + 1], q == 0 ? 999.0 : wps[3 * (q - 1) + 2]};
    const int dims[3] = {G.X, G.Y, G.Z};
    for (int a = 0; a < 3; a++) {
        b.a0[a] = grid_axis_index(c[a] - h, G.bmin[a], G.bmax[a], G.res, dims[a]); b.a1[a] = grid_axis_index(c[a] + h, G.bmin[a], G.bmax[a], G.res, dims[a]);
        b.l0[a] = grid_axis_index(l[a] - h, G.bmin[a], G.bmax[a], G.res, dims[a]); b.l1[a] = grid_axis_index(l[a] + h, G.bmin[a], G.bmax[a], G.res, dims[a]);
    }
    boxes[q] = b;
}
template <bool WRITE>
__global__ void __launch_bounds__(256) k_gather_points(const DevGrid G, int nQ, const GatherBox *boxes, int *counts, double *out, int cap, int *count) {
    __shared__ int warp_cnt[8];
    __shared__ int running;
    const int q = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        int off = 0;
        if (WRITE) { for (int p = 0; p < q; p++) off += counts[p]; if (q == nQ - 1) *count = off + counts[q]; }
        running = off;
    }
    __syncthreads();
    const GatherBox b = boxes[q];
    const int ny = b.a1[1] - b.a0[1] + 1, nz = b.a1[2] - b.a0[2] + 1;
    const int nvox = (b.a1[0] - b.a0[0] + 1) * ny * nz;
    for (int base = 0; base < nvox; base += blockDim.x) {
        const int v = base + threadIdx.x;
        bool emit = false; int i = 0, j = 0, k = 0;
        if (v < nvox) {
            i = b.a0[0] + v / (ny * nz); j = b.a0[1] + (v / nz) % ny; k = b.a0[2] + v % nz;
            emit = gather_includes(G, b, i, j, k);
            for (int p = 0; emit && p < q; p++) if (gather_includes(G, boxes[p], i, j, k)) emit = false;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, emit);
        if (lane == 0) warp_cnt[warp] = __popc(bal);
        __syncthreads();
        if (WRITE) {
            int off = running;
            for (int w = 0; w < warp; w++) off += warp_cnt[w];
            if (emit) {
                const int pos = off + __popc(bal & ((1u << lane) - 1u));
                if (pos < cap) { out[3 * pos] = (i + 0.5) * G.res + G.bmin[0]; out[3 * pos + 1] = (j + 0.5) * G.res + G.bmin[1]; out[3 * pos + 2] = (k + 0.5) * G.res + G.bmin[2]; }
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < 8; w++) t += warp_cnt[w]; running += t; }
        __syncthreads();
    }
    if (!WRITE && threadIdx.x == 0) counts[q] = running;
}

extern "C" int isdf_gather_obstacle_points(isdf_ctx *c, const double *waypoints, int nQ, double half_extent, const double *offset,
                                           double *out_points, int cap, int *n, int set_as_points) {
    if (!c || !waypoints || nQ < 1 || !n || cap < 0 || (cap > 0 && !out_points && !set_as_points)) return fail(ISDF_ERR_INVALID, "bad argument");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    if (set_device(c)) return ISDF_ERR_CUDA;
    DevBuf<double> dw, dout; DevBuf<GatherBox> db; DevBuf<int> dn;
    const int capd = cap > 0 ? cap : 1;
    CU_TRY(dw.upload(waypoints, (size_t)3 * nQ, c->stream));
    CU_TRY(dout.ensure((size_t)3 * capd)); CU_TRY(db.ensure(nQ)); CU_TRY(dn.ensure((size_t)nQ + 1));
    const double ox = offset ? offset[0] : 0.0, oy = offset ? offset[1] : 0.0, oz = offset ? offset[2] : 0.0;
    k_gather_boxes<<<(nQ + 127) / 128, 128, 0, c->stream>>>(c->map.grid, dw.p, nQ, half_extent, ox, oy, oz, db.p);
    k_gather_points<false><<<nQ, 256, 0, c->stream>>>(c->map.grid, nQ, db.p, dn.p + 1, nullptr, 0, dn.p);
    k_gather_points<true><<<nQ, 256, 0, c->stream>>>(c->map.grid, nQ, db.p, dn.p + 1, dout.p, capd, dn.p);
    c->stats.kernel_launches += 3;
    CU_TRY(cudaGetLastError());
    int cnt = 0;
    CU_TRY(cudaMemcpyAsync(&cnt, dn.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    *n = cnt;
    const int m = cnt < cap ? cnt : cap;
    int rc = 0;
    if (m > 0 && out_points) CU_TRY(cudaMemcpy(out_points, dout.p, sizeof(double) * 3 * m, cudaMemcpyDeviceToHost));
    if (set_as_points) {
        if (cnt > cap) rc = fail(ISDF_ERR_INVALID, "cap smaller than the obstacle list");
        else {
            std::vector<double> tmp((size_t)3 * (m > 0 ? m : 1));
            if (m > 0) CU_TRY(cudaMemcpy(tmp.data(), dout.p, sizeof(double) * 3 * m, cudaMemcpyDeviceToHost));
            cudaError_t e = c->sv.set_points(tmp.data(), m, c->stream);
            if (e != cudaSuccess) rc = fail(ISDF_ERR_CUDA, cudaGetErrorString(e));
        }
    }
    return rc;
}

// ---- discrete evaluation ------------------------------------------------------------------------------------
// whether a sharded *_device evaluation finishes with the peer exchange (an unsharded call, isdf_set_shard(ctx, 0, 1), stays local)
static bool fused_exchange(const isdf_ctx *c) { return c->peer.fused && c->peer.args.world > 1 && c->world > 1; }

// what the exchange needs for an evaluation of N pieces. The caller commits the next epoch only once its exchange is enqueued: a
// local failure must not leave this rank one epoch ahead.
static int peer_fuse_check(const isdf_ctx *c, int N) {
    if (c->peer.args.world != c->world || c->peer.args.rank != c->rank) return fail(ISDF_ERR_STATE, "peer group does not match isdf_set_shard");
    if (19 * N + 1 > c->peer.args.cap) return fail(ISDF_ERR_INVALID, "peer exchange buffer too small for this N (isdf_peer_export max_doubles)");
    return 0;
}

// the exchange of d_vec (n doubles) at the next epoch, committed only once its kernel is enqueued
static int peer_allreduce_launch(isdf_ctx *c, double *d_vec, int n, cudaStream_t st) {
    PeerArgs P = c->peer.args;
    P.epoch = c->peer.args.epoch + 1;
    k_peer_allreduce<<<1, 512, 0, st>>>(P, d_vec, n);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    c->peer.args.epoch = P.epoch;
    return 0;
}

// count_out (host entry points only): where the epilogue drops the pair count, behind the result vector
static int launch_discrete(isdf_ctx *c, int N, const double *d_T, const double *d_C, double *d_out, double *count_out, cudaStream_t st) {
    const int K = c->cfg.integral_intervs;
    const long long S = (long long)N * (K + 1);
    if (S > 0x7fffffffll) return fail(ISDF_ERR_UNSUPPORTED, "N * (integral_intervs + 1) must fit in 31 bits");
    CU_TRY(c->disc.d_piece_cost.ensure(N));
    if (c->disc.d_tickets.n < 2) {   // [0] pieces_done of the epilogue, [1] work-item cursor of the persistent scan warps
        CU_TRY(c->disc.d_tickets.ensure(2));
        CU_TRY(cudaMemsetAsync(c->disc.d_tickets.p, 0, 2 * sizeof(int), st));
    }
    CU_TRY(c->disc.d_tot.ensure((size_t)S * 8));
    DiscArgs A;
    A.cfg = c->dcfg; A.grid = c->map.grid; A.shape = c->mesh.shape; A.N = N; A.T = d_T; A.C = d_C;
    A.tot = c->disc.d_tot.p; A.pieces_done = c->disc.d_tickets.p; A.item_cursor = c->disc.d_tickets.p + 1;
    A.piece_cost = c->disc.d_piece_cost.p; A.out = d_out; A.pair_counter = c->disc.d_counter.p; A.count_out = count_out;
    A.rank = c->rank; A.world = c->world;
    A.peer = PeerArgs{};
    const bool fused = fused_exchange(c);
    if (fused) {
        if (int r = peer_fuse_check(c, N)) return r;
        A.peer = c->peer.args; A.peer.epoch = c->peer.args.epoch + 1;   // committed below, once the exchange kernel is really enqueued
    }
    const long long M = (S - c->rank + c->world - 1) / c->world;
    const bool mesh = (c->mesh.shape.kind == ISDF_SHAPE_MESH);
    // mesh launches with collision: k_discrete_prologue computes every local sample's pose and lists each run's window voxels
    const bool prologue = mesh && (c->dcfg.flags & ISDF_WITH_COLLISION);
    A.pose = nullptr; A.wl_desc = nullptr; A.wl_codes = nullptr; A.wl_cap = 0; A.wl_count = c->disc.d_counter.p + 1;
    if (prologue) {
        // budget x world codes per local sample: a shard's runs are world times shorter (~54 / world samples on the bench
        // trajectory), so the same windows need world times more codes per local sample. List offsets are ints.
        const long long cap = std::min<long long>((long long)c->disc.wl_budget * M * c->world, 0x7fffffffll);
        CU_TRY(c->disc.d_pose.ensure((size_t)8 * M));
        CU_TRY(c->disc.d_wl_desc.ensure((size_t)M));
        CU_TRY(c->disc.d_wl_codes.ensure((size_t)std::max(cap, 1ll)));
        A.pose = c->disc.d_pose.p; A.wl_desc = c->disc.d_wl_desc.p; A.wl_codes = c->disc.d_wl_codes.p; A.wl_cap = (unsigned long long)cap;
        c->disc.wl_cap = cap;
    }
    c->disc.wl_samples = prologue ? M : 0;
    CU_TRY(cudaMemsetAsync(c->disc.d_counter.p, 0, 5 * sizeof(unsigned long long), st));   // pair counter, window-list counters
    if (prologue) CU_TRY(discrete_launch_prologue(A, (int)M, st));
    // longest-first order from the previous evaluation of the same problem shape (first evaluation: natural order)
    const long long sig = ((long long)N << 20) ^ ((long long)c->rank << 10) ^ c->world ^ ((long long)K << 40);
    // only mesh samples have a heavy tail worth splitting. Every sample of a launch may be split (item trace at world = 8:
    // with M/4 slots the 515 heaviest samples were split and the NEXT heaviest — unsplit, 15-25 queries, 80-110 us — set the kernel time)
    const int max_split = mesh ? (int)std::min<long long>(M, MAX_SPLIT_SLOTS) : 0;
    const size_t max_items = (size_t)M + (size_t)(ROW_CLASSES - 1) * max_split;
    CU_TRY(c->disc.d_work.ensure((size_t)S));
    if (c->disc.d_items.n < 3 * max_items + (size_t)M) { CU_TRY(c->disc.d_items.ensure(3 * max_items + (size_t)M)); c->disc.order_for = -1; }   // a regrown table holds no items yet
    CU_TRY(c->disc.d_item_count.ensure(1));
    CU_TRY(c->disc.d_subsum.ensure((size_t)std::max(max_split, 1) * ROW_CLASSES * 8));
    if (c->disc.d_split_work.n < (size_t)std::max(max_split, 1)) {
        CU_TRY(c->disc.d_split_work.ensure((size_t)std::max(max_split, 1)));
        CU_TRY(cudaMemsetAsync(c->disc.d_split_work.p, 0, sizeof(unsigned) * std::max(max_split, 1), st));
    }
    if (c->disc.d_split_done.n < (size_t)std::max(max_split, 1)) {
        CU_TRY(c->disc.d_split_done.ensure((size_t)std::max(max_split, 1)));
        CU_TRY(cudaMemsetAsync(c->disc.d_split_done.p, 0, sizeof(unsigned) * std::max(max_split, 1), st));
    }
    A.work = c->disc.d_work.p;
    // a launch with far more samples than resident warps (batched callbacks: millions) balances itself through the persistent warps'
    // dynamic item counter: sorting / splitting would only cost a long single-CTA pass over the work array
    const bool want_items = !c->disc.no_items && M <= 1024ll * ITEMS_CACHE * 4;
    const bool have_items = (c->disc.order_for == sig) && want_items;
    A.items = have_items ? c->disc.d_items.p : nullptr;
    A.item_count = c->disc.d_item_count.p; A.subsum = c->disc.d_subsum.p; A.split_work = c->disc.d_split_work.p; A.split_done = c->disc.d_split_done.p;
    // persistent grid: one CTA per resident slot (or fewer when there are fewer items than warps)
    const long long want = ((have_items ? (long long)max_items : M) + DISC_WARPS - 1) / DISC_WARPS;
    const long long resident = (long long)c->sm_count * (mesh ? c->mesh_blocks : c->analytic_blocks);
    const unsigned grid = (unsigned)std::max<long long>(1, std::min(want, resident));
    if (c->disc.items_pending) CU_TRY(cudaStreamWaitEvent(st, c->ev_items_done, 0));   // the table this launch reads (or overwrites next)
    CU_TRY(discrete_launch_scan(A, mesh, grid, st));
    CU_TRY(discrete_launch_epilogue(A, st));
    if (fused) c->peer.args.epoch = A.peer.epoch;
    const int warp_slots = c->disc.warp_slots_override > 0 ? c->disc.warp_slots_override : c->warp_slots;
    c->disc.last_M = M; c->disc.last_rank = c->rank; c->disc.last_world = c->world; c->disc.last_max_split = max_split;
    c->disc.last_warp_slots = warp_slots; c->disc.last_have_items = have_items;
    c->disc.last_builder = want_items ? (items_cached(M) ? 1 : 2) : 0;
    // build the next evaluation's work items on the aux stream: overlaps the caller's D2H / all-reduce / host work
    if (want_items) {
        CU_TRY(cudaEventRecord(c->ev_main_done, st));
        CU_TRY(cudaStreamWaitEvent(c->aux_stream, c->ev_main_done, 0));
        CU_TRY(discrete_launch_build_items(c->disc.d_work.p, c->rank, c->world, (int)M, max_split, warp_slots, c->disc.d_items.p, c->disc.d_item_count.p, c->aux_stream));
        CU_TRY(cudaEventRecord(c->ev_items_done, c->aux_stream));
        c->disc.items_pending = true;
        c->disc.order_for = sig;
        c->stats.kernel_launches++;   // work-item builder
    }
    c->stats.kernel_launches += prologue ? 3 : 2;   // (prologue,) scan kernel, epilogue
    c->stats.evals_discrete++;
    return 0;
}

static int check_eval_state(isdf_ctx *c, int N, bool need_map) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (N < 1) return fail(ISDF_ERR_INVALID, "N < 1");
    const bool coll = (c->cfg.flags & ISDF_WITH_COLLISION) != 0;
    if (coll && !c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    if (need_map && coll && !c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    return 0;
}

extern "C" int isdf_eval_discrete_device(isdf_ctx *c, int N, const double *d_T, const double *d_coeffs, double *d_out, void *cuda_stream) {
    int r = check_eval_state(c, N, true);
    if (r) return r;
    if (!d_T || !d_coeffs || !d_out) return fail(ISDF_ERR_INVALID, "NULL device pointer");
    if (set_device(c)) return ISDF_ERR_CUDA;
    return launch_discrete(c, N, d_T, d_coeffs, d_out, nullptr, (cudaStream_t)cuda_stream);
}

// The host form of the discrete and swept-volume evaluations: [coefficients 18N | durations N] go in through one pinned block and
// ONE copy, `before` runs after that copy, `launch(d_T, d_C, d_out, count_out)` between ev0 and ev1, and [cost | gradC | gradT |
// counter word] come back in ONE copy. The result is added to *cost, gradC and gradT, as the reference accumulates (hpp:539-550,
// hpp:640-645); the counter word goes to the stat `counted`. The caller poisons *cost on failure.
template <typename Before, typename Launch>
static int eval_host(isdf_ctx *c, int N, const double *T, const double *coeffs, double *cost, double *gradC, double *gradT,
                     int64_t isdf_stats::*counted, Before before, Launch launch) {
    if (set_device(c)) return ISDF_ERR_CUDA;
    const size_t nin = (size_t)19 * N, nout = (size_t)19 * N + 1;
    CU_TRY(c->stage.h.ensure(nin + nout + 1));
    CU_TRY(c->stage.d_C.ensure(nin)); CU_TRY(c->stage.d_out.ensure(nout + 1));
    std::memcpy(c->stage.h.p, coeffs, sizeof(double) * 18 * N);
    std::memcpy(c->stage.h.p + 18 * (size_t)N, T, sizeof(double) * N);
    CU_TRY(cudaMemcpyAsync(c->stage.d_C.p, c->stage.h.p, sizeof(double) * nin, cudaMemcpyHostToDevice, c->stream));
    if (int rr = before()) return rr;
    CU_TRY(cudaEventRecord(c->ev0, c->stream));
    if (int rr = launch(c->stage.d_C.p + 18 * (size_t)N, c->stage.d_C.p, c->stage.d_out.p, c->stage.d_out.p + nout)) return rr;
    CU_TRY(cudaEventRecord(c->ev1, c->stream));
    double *h_out = c->stage.h.p + nin;
    CU_TRY(cudaMemcpyAsync(h_out, c->stage.d_out.p, sizeof(double) * (nout + 1), cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    unsigned long long count = 0;
    std::memcpy(&count, h_out + nout, sizeof(count));
    if (fused_exchange(c) && isdf_peer_status(c) != ISDF_OK) return ISDF_ERR_CUDA;   // exchange timed out: the vector is NaN
    float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
    c->stats.last_kernel_ms = ms; c->stats.*counted = (int64_t)count;
    *cost += h_out[0];
    for (size_t k = 0; k < (size_t)18 * N; k++) gradC[k] += h_out[1 + k];
    for (int k = 0; k < N; k++) gradT[k] += h_out[1 + 18 * N + k];
    return 0;
}

extern "C" int isdf_eval_discrete(isdf_ctx *c, int N, const double *T, const double *coeffs, double *cost, double *gradC, double *gradT) {
    return poison_on_failure([&]() -> int {
        if (int r = check_eval_state(c, N, true)) return r;
        if (!T || !coeffs || !cost || !gradC || !gradT) return fail(ISDF_ERR_INVALID, "NULL argument");
        return eval_host(c, N, T, coeffs, cost, gradC, gradT, &isdf_stats::last_pairs, [] { return 0; },
                         [&](const double *d_T, const double *d_C, double *d_out, double *count_out) {
                             return launch_discrete(c, N, d_T, d_C, d_out, count_out, c->stream);
                         });
    }, [&] { nan_fill(cost, 1); });
}

extern "C" int isdf_get_piece_costs(isdf_ctx *c, double *piece_cost, int n) {
    if (!c || !piece_cost || n < 0) return fail(ISDF_ERR_INVALID, "bad argument");
    if ((size_t)n > c->disc.d_piece_cost.n) return fail(ISDF_ERR_STATE, "no discrete evaluation with that many pieces yet");
    if (int r = sync_ctx(c)) return r;
    CU_TRY(cudaMemcpy(piece_cost, c->disc.d_piece_cost.p, sizeof(double) * n, cudaMemcpyDeviceToHost));
    return 0;
}

// ---- batched optimiser callback on the device (MINCO -> time-integral term -> adjoint), SURVEY §8f row 1 ----------------------
static int callback_batch_launch(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int bc_stride, double rho,
                                 const double *d_x, double *d_cost, double *d_grad, cudaStream_t st) {
    const size_t BN = (size_t)B * N0;
    if (int r = minco_fits(N0)) return r;
    if (BN * (size_t)(c->cfg.integral_intervs + 1) > 0x7fffffffull) return fail(ISDF_ERR_UNSUPPORTED, "batch too large: B*N0*(K+1) must fit in 31 bits");
    if (int r = c->batch.minco.ensure(B, N0)) return r;
    MincoArgs M = c->batch.minco.args(B, N0, d_head, d_tail, bc_stride, rho, d_x);
    M.cost = d_cost; M.grad = d_grad;
    // per-problem obstacle point sets registered for exactly this batch (isdf_set_points_batch): the LIVE composition of costFunctionLmbm
    // (hpp:386-405) — swept-volume term, then time-integral term
    const bool with_swept = (c->sv.B == B);
    if (with_swept) {
        if (c->mesh.shape.kind == ISDF_SHAPE_MESH && c->mesh.shape.mesh.sign_mode == MESH_SIGN_WINDING)
            return fail(ISDF_ERR_UNSUPPORTED, "swept-volume term with a winding-sign mesh (see isdf_set_shape_mesh_ex)");
        CU_TRY(c->batch.d_Cpp.ensure(18 * BN)); CU_TRY(c->batch.d_sv.ensure((size_t)B * (19 * (size_t)N0 + 1)));
        M.Cpp = c->batch.d_Cpp.p;
    }
    const size_t smem = minco_smem_bytes(N0);
    k_minco_forward<<<B, 32, smem, st>>>(M);
    if (with_swept) {
        int launches = 0;
        cudaError_t e = c->sv.launch_batch(c->dcfg, c->mesh.shape, N0, M.T, M.Cpp, c->batch.d_sv.p, st, &launches);
        c->stats.kernel_launches += launches;
        c->stats.evals_swept++;
        if (e != cudaSuccess) return fail(e == cudaErrorInvalidValue ? ISDF_ERR_INVALID : ISDF_ERR_CUDA, std::string("batched swept: ") + cudaGetErrorString(e));
        M.sv_out = c->batch.d_sv.p;
    }
    int r = launch_discrete(c, (int)BN, M.T, M.C, c->batch.minco.d_out.p, nullptr, st);
    if (r) return r;
    M.disc_out = c->batch.minco.d_out.p; M.piece_cost = c->disc.d_piece_cost.p;
    k_minco_backward<<<B, 32, smem, st>>>(M);
    c->stats.kernel_launches += 2;
    c->batch.B = B; c->batch.N0 = N0;
    CU_TRY(cudaGetLastError());
    return 0;
}

static int callback_batch_check(isdf_ctx *c, int B, int N0) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (B < 1 || N0 < 1) return fail(ISDF_ERR_INVALID, "B < 1 or N0 < 1");
    if ((long long)B * N0 > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "B*N0 overflows");
    if (c->world != 1) return fail(ISDF_ERR_STATE, "the batched callback shards by PROBLEM: keep isdf_set_shard(ctx, 0, 1) and give each rank its own problems");
    return check_eval_state(c, B * N0, true);
}

extern "C" int isdf_callback_batch_device(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc, double rho,
                                          const double *d_x, double *d_cost, double *d_grad, void *cuda_stream) {
    int r = callback_batch_check(c, B, N0);
    if (r) return r;
    if (!d_head || !d_tail || !d_x || !d_cost || !d_grad) return fail(ISDF_ERR_INVALID, "NULL device pointer");
    if (set_device(c)) return ISDF_ERR_CUDA;
    return callback_batch_launch(c, B, N0, d_head, d_tail, per_problem_bc ? 9 : 0, rho, d_x, d_cost, d_grad, (cudaStream_t)cuda_stream);
}

// the host entry points' boundary conditions (9 doubles, or 9 per problem) in buf on c->stream: *d_head, then *d_tail
static int upload_bc(isdf_ctx *c, DevBuf<double> &buf, int B, int per_problem_bc, const double *head, const double *tail, const double **d_head,
                     const double **d_tail) {
    const size_t nbc = per_problem_bc ? (size_t)9 * B : 9;
    CU_TRY(buf.ensure(2 * nbc));
    CU_TRY(cudaMemcpyAsync(buf.p, head, sizeof(double) * nbc, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(cudaMemcpyAsync(buf.p + nbc, tail, sizeof(double) * nbc, cudaMemcpyHostToDevice, c->stream));
    *d_head = buf.p; *d_tail = buf.p + nbc;
    return 0;
}

extern "C" int isdf_callback_batch(isdf_ctx *c, int B, int N0, const double *head, const double *tail, int per_problem_bc, double rho,
                                   const double *x, double *cost, double *grad) {
    return poison_on_failure([&]() -> int {
        if (int r = callback_batch_check(c, B, N0)) return r;
        if (!head || !tail || !x || !cost || !grad) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        const size_t dim = (size_t)N0 + 3 * (size_t)(N0 - 1);
        CU_TRY(c->batch.d_x.upload(x, dim * B, c->stream));
        const double *d_head, *d_tail;
        if (int r = upload_bc(c, c->batch.d_bc, B, per_problem_bc, head, tail, &d_head, &d_tail)) return r;
        CU_TRY(c->batch.d_cost.ensure(B)); CU_TRY(c->batch.d_grad.ensure(dim * B));
        CU_TRY(cudaEventRecord(c->ev0, c->stream));
        if (int r = isdf_callback_batch_device(c, B, N0, d_head, d_tail, per_problem_bc, rho, c->batch.d_x.p, c->batch.d_cost.p, c->batch.d_grad.p,
                                               c->stream)) return r;
        CU_TRY(cudaEventRecord(c->ev1, c->stream));
        CU_TRY(cudaMemcpyAsync(cost, c->batch.d_cost.p, sizeof(double) * B, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaMemcpyAsync(grad, c->batch.d_grad.p, sizeof(double) * dim * B, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
        float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
        c->stats.last_kernel_ms = ms;
        return 0;
    }, [&] { nan_fill(cost, B); });
}

// ---- device-resident lock-step L-BFGS over the batched callback (SURVEY §8f row 2; isdf_lbfgs.cuh) ----------------------------------------
static int lbfgs_check(const isdf_lbfgs_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (p->mem_size <= 0 || p->mem_size > 64) return fail(ISDF_ERR_INVALID, "mem_size out of range (1..64)");
    if (p->past < 0 || p->g_epsilon < 0.0 || p->delta < 0.0 || p->min_step < 0.0 || p->max_step < p->min_step || !(p->f_dec_coeff > 0.0 && p->f_dec_coeff < 1.0) ||
        !(p->machine_prec > 0.0) || p->max_linesearch <= 0 || p->max_iterations < 0 || p->max_rounds < 0)
        return fail(ISDF_ERR_INVALID, "L-BFGS parameter out of range");
    return 0;
}

extern "C" int isdf_lbfgs_default_params(isdf_lbfgs_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    // lbfgs_parameter_t defaults (lbfgs.hpp:40-142) with the back end's settings (config_CappedCone.yaml:99-102: mem 16, past 10, min_step 1e-32, g_epsilon 0)
    p->mem_size = 16; p->past = 10; p->max_iterations = 0; p->max_linesearch = 64; p->max_rounds = 0;
    p->g_epsilon = 0.0; p->delta = 1.0e-6; p->min_step = 1.0e-32; p->max_step = 1.0e+20; p->f_dec_coeff = 1.0e-4; p->cautious_factor = 1.0e-6; p->machine_prec = 1.0e-16;
    return 0;
}

// The lock-step rounds of isdf_lbfgs_batch_device and isdf_midend_batch_device: every round `eval(d_x, d_f, d_grad)` evaluates the point
// every instance requested (finished instances ride along unchanged: their state is frozen), then one k_lbfgs_feed consumes the results.
// d_x: B x n (in: starting points, out: solutions); d_f: B; d_ret / d_iterations / d_evaluations: B ints (any of the three may be null).
// Synchronous with respect to the host (one 4-byte read per round decides termination), all data stays on the device.
template <typename Eval>
static int lbfgs_rounds(isdf_ctx *c, isdf_ctx::LbfgsBufs &lb, int B, int n, const isdf_lbfgs_params *prm, int cancel_after, double *d_x, double *d_f,
                        int *d_ret, int *d_iterations, int *d_evaluations, int *rounds_out, cudaStream_t st, Eval eval) {
    const int m = prm->mem_size, npf = prm->past > 1 ? prm->past : 1;
    const size_t per = (size_t)4 * n + npf + 2 * (size_t)m + 2 * (size_t)m * n + LB_NSCALAR;   // doubles of state per instance
    CU_TRY(lb.d_state.ensure(per * B)); CU_TRY(lb.d_grad.ensure((size_t)B * n)); CU_TRY(lb.d_int.ensure((size_t)B * LB_NINT + 4));
    CU_TRY(lb.h_active.ensure(1));
    CU_TRY(cudaMemsetAsync(lb.d_state.p, 0, sizeof(double) * per * B, st));
    CU_TRY(cudaMemsetAsync(lb.d_int.p, 0, sizeof(int) * ((size_t)B * LB_NINT + 4), st));   // phase = WANT_INIT
    LbfgsArgs L;
    L.B = B; L.n = n;
    L.pr.mem_size = m; L.pr.past = prm->past; L.pr.max_iterations = prm->max_iterations; L.pr.max_linesearch = prm->max_linesearch;
    L.pr.g_epsilon = prm->g_epsilon; L.pr.delta = prm->delta; L.pr.min_step = prm->min_step; L.pr.max_step = prm->max_step;
    L.pr.f_dec_coeff = prm->f_dec_coeff; L.pr.cautious_factor = prm->cautious_factor; L.pr.machine_prec = prm->machine_prec;
    L.pr.cancel_after = cancel_after;
    double *p = lb.d_state.p;
    L.x = d_x; L.f = d_f; L.grad = lb.d_grad.p;
    L.xp = p; p += (size_t)B * n; L.g = p; p += (size_t)B * n; L.gp = p; p += (size_t)B * n; L.d = p; p += (size_t)B * n;
    L.pf = p; p += (size_t)B * npf; L.alpha = p; p += (size_t)B * m; L.ys = p; p += (size_t)B * m;
    L.S = p; p += (size_t)B * m * n; L.Y = p; p += (size_t)B * m * n; L.sc = p;
    L.st = lb.d_int.p; L.active = lb.d_int.p + (size_t)B * LB_NINT;
    // olddnorm starts at 1 (lbfgs.hpp:541): scalar slot 2 of every instance
    {
        std::vector<double> init((size_t)B * LB_NSCALAR, 0.0);
        for (int b = 0; b < B; b++) init[(size_t)b * LB_NSCALAR + 2] = 1.0;
        CU_TRY(cudaMemcpyAsync(L.sc, init.data(), sizeof(double) * init.size(), cudaMemcpyHostToDevice, st));
        CU_TRY(cudaStreamSynchronize(st));
    }
    int rounds = 0;
    for (;;) {
        if (int r = eval(d_x, d_f, lb.d_grad.p)) return r;
        CU_TRY(cudaMemsetAsync(L.active, 0, sizeof(int), st));
        k_lbfgs_feed<<<(unsigned)((B + 63) / 64), 64, 0, st>>>(L);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(lb.h_active.p, L.active, sizeof(int), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
        ++rounds;
        if (*lb.h_active.p == 0) break;
        if (prm->max_rounds > 0 && rounds >= prm->max_rounds) {   // instances still running end on their last accepted iterate, ret -1008
            k_lbfgs_cap<<<(unsigned)((B + 63) / 64), 64, 0, st>>>(L);
            c->stats.kernel_launches++;
            CU_TRY(cudaGetLastError());
            break;
        }
    }
    // results: f = fx of every instance (scalar slot 0), return codes and counters
    CU_TRY(cudaMemcpy2DAsync(d_f, sizeof(double), L.sc, sizeof(double) * LB_NSCALAR, sizeof(double), B, cudaMemcpyDeviceToDevice, st));
    if (d_ret) CU_TRY(cudaMemcpy2DAsync(d_ret, sizeof(int), L.st + 1, sizeof(int) * LB_NINT, sizeof(int), B, cudaMemcpyDeviceToDevice, st));
    if (d_iterations) CU_TRY(cudaMemcpy2DAsync(d_iterations, sizeof(int), L.st + 8, sizeof(int) * LB_NINT, sizeof(int), B, cudaMemcpyDeviceToDevice, st));
    if (d_evaluations) CU_TRY(cudaMemcpy2DAsync(d_evaluations, sizeof(int), L.st + 9, sizeof(int) * LB_NINT, sizeof(int), B, cudaMemcpyDeviceToDevice, st));
    CU_TRY(cudaStreamSynchronize(st));
    if (rounds_out) *rounds_out = rounds;
    return 0;
}

static void nan_fill_device(isdf_ctx *c, double *d, int n, cudaStream_t st) {
    if (c && d && n > 0 && cudaSetDevice(c->device) == cudaSuccess) { cudaMemsetAsync(d, 0xff, sizeof(double) * n, st); cudaStreamSynchronize(st); }
}

// an L-BFGS call's results in lb to the host: x (B x n), f, and ret / iterations / evaluations from the d_head triple (each may be NULL)
static int lbfgs_copy_out(const isdf_ctx::LbfgsBufs &lb, int B, size_t n, double *x, double *f, int *ret, int *iterations, int *evaluations) {
    CU_TRY(cudaMemcpy(x, lb.d_x.p, sizeof(double) * n * B, cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemcpy(f, lb.d_f.p, sizeof(double) * B, cudaMemcpyDeviceToHost));
    if (ret) CU_TRY(cudaMemcpy(ret, lb.d_head.p, sizeof(int) * B, cudaMemcpyDeviceToHost));
    if (iterations) CU_TRY(cudaMemcpy(iterations, lb.d_head.p + B, sizeof(int) * B, cudaMemcpyDeviceToHost));
    if (evaluations) CU_TRY(cudaMemcpy(evaluations, lb.d_head.p + 2 * (size_t)B, sizeof(int) * B, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int isdf_lbfgs_batch_device(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc, double rho,
                                       const isdf_lbfgs_params *prm, double *d_x, double *d_f, int *d_ret, int *d_iterations, int *d_evaluations,
                                       int *rounds_out, void *cuda_stream) {
    cudaStream_t st = (cudaStream_t)cuda_stream;
    return poison_on_failure([&]() -> int {
        if (int r = callback_batch_check(c, B, N0)) return r;
        if (int r = lbfgs_check(prm)) return r;
        if (!d_head || !d_tail || !d_x || !d_f) return fail(ISDF_ERR_INVALID, "NULL device pointer");
        if (set_device(c)) return ISDF_ERR_CUDA;
        return lbfgs_rounds(c, c->lbfgs, B, 4 * N0 - 3, prm, 0, d_x, d_f, d_ret, d_iterations, d_evaluations, rounds_out, st,
                            [&](const double *x, double *f, double *g) {
                                return callback_batch_launch(c, B, N0, d_head, d_tail, per_problem_bc ? 9 : 0, rho, x, f, g, st);
                            });
    }, [&] { nan_fill_device(c, d_f, B, st); });
}

extern "C" int isdf_lbfgs_batch(isdf_ctx *c, int B, int N0, const double *head, const double *tail, int per_problem_bc, double rho,
                                const isdf_lbfgs_params *prm, double *x, double *f, int *ret, int *iterations, int *evaluations, int *rounds_out) {
    return poison_on_failure([&]() -> int {
        if (int r = callback_batch_check(c, B, N0)) return r;
        if (!head || !tail || !x || !f) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        isdf_ctx::LbfgsBufs &lb = c->lbfgs;
        const size_t n = (size_t)4 * N0 - 3;
        CU_TRY(lb.d_x.upload(x, n * B, c->stream));
        const double *d_head, *d_tail;
        if (int r = upload_bc(c, c->batch.d_bc, B, per_problem_bc, head, tail, &d_head, &d_tail)) return r;
        CU_TRY(lb.d_f.ensure(B)); CU_TRY(lb.d_head.ensure((size_t)3 * B));
        if (int r = isdf_lbfgs_batch_device(c, B, N0, d_head, d_tail, per_problem_bc, rho, prm, lb.d_x.p, lb.d_f.p, lb.d_head.p, lb.d_head.p + B,
                                            lb.d_head.p + 2 * (size_t)B, rounds_out, c->stream)) return r;
        return lbfgs_copy_out(lb, B, n, x, f, ret, iterations, evaluations);
    }, [&] { nan_fill(f, B); });
}

// Diagnostic (not part of include/isdf.h): the unchanged lbfgs_rounds + k_lbfgs_feed for B instances of dimension n on a HOST objective.
// Every round copies all B requested points (finished instances' included: they ride along unchanged) to the host, calls
// eval(user, B, n, x, f, g) and uploads f and g. x: B x n (in: starting points, out: solutions); f, ret, iterations, evaluations: B
// (ret / iterations / evaluations may be NULL); rounds: the rounds run (may be NULL).
typedef void (*isdf_dbg_lbfgs_eval_t)(void *user, int B, int n, const double *x, double *f, double *g);
extern "C" int isdf_dbg_lbfgs_rounds(isdf_ctx *c, int B, int n, const isdf_lbfgs_params *prm, int cancel_after, isdf_dbg_lbfgs_eval_t eval, void *user,
                                     double *x, double *f, int *ret, int *iterations, int *evaluations, int *rounds_out) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (B < 1 || n < 1 || (long long)B * n > 0x7fffffffll || cancel_after < 0) return fail(ISDF_ERR_INVALID, "B < 1, n < 1, B*n overflows or cancel_after < 0");
    if (int r = lbfgs_check(prm)) return r;
    if (!eval || !x || !f) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (set_device(c)) return ISDF_ERR_CUDA;
    const size_t bn = (size_t)B * n;
    isdf_ctx::LbfgsBufs &lb = c->lbfgs;
    CU_TRY(lb.d_x.upload(x, bn, c->stream));
    CU_TRY(lb.d_f.ensure(B)); CU_TRY(lb.d_head.ensure((size_t)3 * B));
    std::vector<double> hx(bn), hf(B), hg(bn);
    int r = lbfgs_rounds(c, lb, B, n, prm, cancel_after, lb.d_x.p, lb.d_f.p, lb.d_head.p, lb.d_head.p + B, lb.d_head.p + 2 * (size_t)B, rounds_out, c->stream,
                         [&](const double *d_x, double *d_f, double *d_g) -> int {
                             CU_TRY(cudaMemcpyAsync(hx.data(), d_x, sizeof(double) * bn, cudaMemcpyDeviceToHost, c->stream));
                             CU_TRY(cudaStreamSynchronize(c->stream));
                             eval(user, B, n, hx.data(), hf.data(), hg.data());
                             CU_TRY(cudaMemcpyAsync(d_f, hf.data(), sizeof(double) * B, cudaMemcpyHostToDevice, c->stream));
                             CU_TRY(cudaMemcpyAsync(d_g, hg.data(), sizeof(double) * bn, cudaMemcpyHostToDevice, c->stream));
                             CU_TRY(cudaStreamSynchronize(c->stream));
                             return 0;
                         });
    if (r) return r;
    return lbfgs_copy_out(lb, B, (size_t)n, x, f, ret, iterations, evaluations);
}

extern "C" int isdf_get_batch_trajectories(isdf_ctx *c, double *T, double *coeffs, double *energy) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (c->batch.B <= 0) return fail(ISDF_ERR_STATE, "no batched callback evaluated yet");
    if (int r = sync_ctx(c)) return r;
    const size_t BN = (size_t)c->batch.B * c->batch.N0;
    const MincoWork &w = c->batch.minco;
    if (T) CU_TRY(cudaMemcpy(T, w.d_T.p, sizeof(double) * BN, cudaMemcpyDeviceToHost));
    if (coeffs) CU_TRY(cudaMemcpy(coeffs, w.d_C.p, sizeof(double) * 18 * BN, cudaMemcpyDeviceToHost));
    if (energy) CU_TRY(cudaMemcpy(energy, w.d_energy.p, sizeof(double) * c->batch.B, cudaMemcpyDeviceToHost));
    return 0;
}

// ---- mid-end: waypoint selection and getOriTraj for B paths (isdf_midend.cuh) ------------------------------------------------------------
extern "C" int isdf_path_waypoints(int B, const int32_t *path_off, const double *path_xyz, double res, double parlength, int cap,
                                   double *waypoints, int32_t *wp_off, int32_t *pieces) {
    if (B < 1 || !path_off || !path_xyz || !wp_off || !pieces || cap < 0 || (cap > 0 && !waypoints)) return fail(ISDF_ERR_INVALID, "NULL argument, B < 1 or cap < 0");
    if (!(std::isfinite(res) && res > 0.0) || !(std::isfinite(parlength) && parlength > 0.0)) return fail(ISDF_ERR_INVALID, "res and parlength must be finite and positive");
    if (path_off[0] != 0) return fail(ISDF_ERR_INVALID, "path_off[0] must be 0");
    for (int b = 0; b < B; b++) if (path_off[b + 1] <= path_off[b]) return fail(ISDF_ERR_INVALID, "every path needs at least one node (path_off must increase)");
    long long total = 0;
    wp_off[0] = 0;
    for (int b = 0; b < B; b++) {
        const long long S = path_off[b + 1] - path_off[b];
        const double *path = path_xyz + 3 * (size_t)path_off[b];
        long long n = 0;
        if (S > 2) {   // plan_manager.cpp:206-213 and :235-245; S <= 2 would not terminate in the reference (include/isdf.h)
            double pl = parlength;
            double gap = std::ceil(pl / res);
            while (gap >= (double)(S - 1)) { pl /= 1.5; gap = std::ceil(pl / res); }
            const long long g = (long long)gap;
            for (long long ind = g; ind < S - 1; ind += g, n++)
                if (total + n < cap) for (int k = 0; k < 3; k++) waypoints[3 * (total + n) + k] = path[3 * ind + k];
        }
        total += n;
        if (total > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "too many waypoints");
        wp_off[b + 1] = (int32_t)total;
        pieces[b] = (int32_t)(n + 1);
    }
    if (total > cap) return fail(ISDF_ERR_INVALID, "cap smaller than the number of waypoints (wp_off reports it)");
    return 0;
}

extern "C" int isdf_midend_default_params(isdf_midend_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    // config_CappedCone.yaml: weight_pr 1000, rho_mid_end 200, inittime 2.5; earlyExit's k > 8e3 (mid_end.hpp:630)
    p->weight_pr = 1000.0; p->rho = 200.0; p->init_time = 2.5; p->cancel_after = 8000; p->reserved_ = 0;
    isdf_lbfgs_default_params(&p->lbfgs);
    p->lbfgs.max_iterations = 100000;   // mid_end.cpp:53; delta = relCostTolMidEnd 1e-6 (:54), the rest as the back end's
    return 0;
}

static int midend_check(isdf_ctx *c, int B, int N0, const isdf_midend_params *p) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (B < 1 || N0 < 1) return fail(ISDF_ERR_INVALID, "B < 1 or N0 < 1");
    if ((long long)B * (4 * (long long)N0 - 3) > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "B*(4*N0-3) overflows");
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (p->reserved_ != 0) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    if (!(std::isfinite(p->weight_pr) && p->weight_pr >= 0.0) || !std::isfinite(p->rho) || !(std::isfinite(p->init_time) && p->init_time > 0.0) ||
        p->cancel_after < 0)
        return fail(ISDF_ERR_INVALID, "mid-end parameter out of range");
    if (int r = lbfgs_check(&p->lbfgs)) return r;
    if (int r = minco_fits(N0)) return r;
    if (c->world != 1) return fail(ISDF_ERR_STATE, "the mid-end shards by PROBLEM: keep isdf_set_shard(ctx, 0, 1) and give each rank its own problems");
    return 0;
}

static int midend_buffers(isdf_ctx *c, int B, int N0) {
    if (int r = c->mid.minco.ensure(B, N0)) return r;
    CU_TRY(c->mid.d_pc.ensure((size_t)B * N0));
    return 0;
}

static MincoArgs midend_minco_args(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int bc_stride, double rho, const double *d_x) {
    MincoArgs M = c->mid.minco.args(B, N0, d_head, d_tail, bc_stride, rho, d_x);
    M.disc_out = c->mid.minco.d_out.p; M.piece_cost = c->mid.d_pc.p; M.seq_terms = 1;
    return M;
}

// one evaluation of OriTraj::costFunction for all B problems: MINCO forward -> pose term -> adjoint with the terms added one at a time
static int midend_eval_launch(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int bc_stride, const isdf_midend_params *p,
                              const double *d_wp, const double *d_x, double *d_cost, double *d_grad, cudaStream_t st) {
    const size_t BN = (size_t)B * N0, smem = minco_smem_bytes(N0);
    MincoArgs M = midend_minco_args(c, B, N0, d_head, d_tail, bc_stride, p->rho, d_x);
    M.cost = d_cost; M.grad = d_grad;
    k_minco_forward<<<B, 32, smem, st>>>(M);
    MidendArgs P;
    P.B = B; P.N = N0; P.K = c->cfg.integral_intervs; P.weight = p->weight_pr; P.T = M.T; P.C = M.C; P.wp = d_wp; P.out = c->mid.minco.d_out.p; P.piece_cost = c->mid.d_pc.p;
    k_midend_pose<<<(unsigned)((BN + 127) / 128), 128, 0, st>>>(P);
    k_minco_backward<<<B, 32, smem, st>>>(M);
    c->stats.kernel_launches += 3;
    CU_TRY(cudaGetLastError());
    return 0;
}

// the mid-end's host entry points stage their inputs in c->mid: boundary conditions (*d_head, *d_tail) and waypoints
static int midend_upload(isdf_ctx *c, int B, int N0, int per_problem_bc, const double *head, const double *tail, const double *waypoints,
                         const double **d_head, const double **d_tail, const double **d_wp) {
    const size_t nwp = (size_t)3 * B * (N0 - 1);
    if (int r = upload_bc(c, c->mid.d_bc, B, per_problem_bc, head, tail, d_head, d_tail)) return r;
    CU_TRY(c->mid.d_wp.ensure(nwp > 0 ? nwp : 1));
    if (nwp) CU_TRY(cudaMemcpyAsync(c->mid.d_wp.p, waypoints, sizeof(double) * nwp, cudaMemcpyHostToDevice, c->stream));
    *d_wp = c->mid.d_wp.p;
    return 0;
}

extern "C" int isdf_midend_callback_batch(isdf_ctx *c, int B, int N0, const double *head, const double *tail, int per_problem_bc,
                                          const isdf_midend_params *p, const double *waypoints, const double *x, double *cost, double *grad) {
    return poison_on_failure([&]() -> int {
        if (int r = midend_check(c, B, N0, p)) return r;
        if (!head || !tail || !x || !cost || !grad || (N0 > 1 && !waypoints)) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        const size_t dim = (size_t)4 * N0 - 3;
        const double *d_head, *d_tail, *d_wp;
        if (int r = midend_upload(c, B, N0, per_problem_bc, head, tail, waypoints, &d_head, &d_tail, &d_wp)) return r;
        CU_TRY(c->mid.d_x.upload(x, dim * B, c->stream));
        CU_TRY(c->mid.d_cost.ensure(B)); CU_TRY(c->mid.d_grad.ensure(dim * B));
        if (int r = midend_buffers(c, B, N0)) return r;
        if (int r = midend_eval_launch(c, B, N0, d_head, d_tail, per_problem_bc ? 9 : 0, p, d_wp, c->mid.d_x.p, c->mid.d_cost.p, c->mid.d_grad.p, c->stream)) return r;
        CU_TRY(cudaMemcpyAsync(cost, c->mid.d_cost.p, sizeof(double) * B, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaMemcpyAsync(grad, c->mid.d_grad.p, sizeof(double) * dim * B, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
        return 0;
    }, [&] { nan_fill(cost, B); });
}

static int midend_batch_run(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc, const isdf_midend_params *p,
                            const double *d_wp, double *d_x, double *d_T, double *d_coeffs, double *d_f, int *d_ret, int *d_iterations,
                            int *d_evaluations, int *rounds_out, cudaStream_t st) {
    if (set_device(c)) return ISDF_ERR_CUDA;
    const int n = 4 * N0 - 3;
    const size_t BN = (size_t)B * N0;
    if (int r = midend_buffers(c, B, N0)) return r;
    // x = [backwardT(init_time) | waypoints] (mid_end.cpp:21-36; backwardT as back_end_optimizer.hpp:243-256)
    const double T0 = p->init_time, tau0 = T0 > 1.0 ? (std::sqrt(2.0 * T0 - 1.0) - 1.0) : (1.0 - std::sqrt(2.0 / T0 - 1.0));
    k_midend_init<<<(unsigned)(((size_t)B * n + 127) / 128), 128, 0, st>>>(B, N0, tau0, d_wp, d_x);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    const int bc_stride = per_problem_bc ? 9 : 0;
    int r = lbfgs_rounds(c, c->mid.lb, B, n, &p->lbfgs, p->cancel_after, d_x, d_f, d_ret, d_iterations, d_evaluations, rounds_out, st,
                         [&](const double *x, double *f, double *g) { return midend_eval_launch(c, B, N0, d_head, d_tail, bc_stride, p, d_wp, x, f, g, st); });
    if (r) return r;
    // the final trajectories: forwardT + MINCO of the returned x (mid_end.cpp:65-71 / 79-85)
    if (d_T || d_coeffs) {
        MincoArgs M = midend_minco_args(c, B, N0, d_head, d_tail, bc_stride, p->rho, d_x);
        k_minco_forward<<<B, 32, minco_smem_bytes(N0), st>>>(M);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        if (d_T) CU_TRY(cudaMemcpyAsync(d_T, M.T, sizeof(double) * BN, cudaMemcpyDeviceToDevice, st));
        if (d_coeffs) CU_TRY(cudaMemcpyAsync(d_coeffs, M.C, sizeof(double) * 18 * BN, cudaMemcpyDeviceToDevice, st));
        CU_TRY(cudaStreamSynchronize(st));
    }
    return 0;
}

extern "C" int isdf_midend_batch_device(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc,
                                        const isdf_midend_params *p, const double *d_waypoints, double *d_x, double *d_T, double *d_coeffs,
                                        double *d_f, int32_t *d_ret, int32_t *d_iterations, int32_t *d_evaluations, int32_t *rounds, void *cuda_stream) {
    cudaStream_t st = (cudaStream_t)cuda_stream;
    return poison_on_failure([&]() -> int {
        if (int r = midend_check(c, B, N0, p)) return r;
        if (!d_head || !d_tail || !d_x || !d_f || (N0 > 1 && !d_waypoints)) return fail(ISDF_ERR_INVALID, "NULL device pointer");
        return midend_batch_run(c, B, N0, d_head, d_tail, per_problem_bc, p, d_waypoints, d_x, d_T, d_coeffs, d_f, d_ret, d_iterations, d_evaluations, rounds, st);
    }, [&] { nan_fill_device(c, d_f, B, st); });
}

extern "C" int isdf_midend_batch(isdf_ctx *c, int B, int N0, const double *head, const double *tail, int per_problem_bc,
                                 const isdf_midend_params *p, const double *waypoints, double *x, double *T, double *coeffs,
                                 double *f, int32_t *ret, int32_t *iterations, int32_t *evaluations, int32_t *rounds) {
    return poison_on_failure([&]() -> int {
        if (int r = midend_check(c, B, N0, p)) return r;
        if (!head || !tail || !x || !f || (N0 > 1 && !waypoints)) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        isdf_ctx::LbfgsBufs &lb = c->mid.lb;
        const size_t n = (size_t)4 * N0 - 3, BN = (size_t)B * N0;
        const double *d_head, *d_tail, *d_wp;
        if (int r = midend_upload(c, B, N0, per_problem_bc, head, tail, waypoints, &d_head, &d_tail, &d_wp)) return r;
        CU_TRY(lb.d_x.ensure(n * B)); CU_TRY(lb.d_f.ensure((size_t)19 * BN + B)); CU_TRY(lb.d_head.ensure((size_t)3 * B));
        double *d_f = lb.d_f.p, *d_T = d_f + B, *d_C = d_T + BN;   // [f | T | coeffs]
        int *d_i = lb.d_head.p;
        if (int r = midend_batch_run(c, B, N0, d_head, d_tail, per_problem_bc, p, d_wp, lb.d_x.p, d_T, d_C, d_f, d_i, d_i + B, d_i + 2 * (size_t)B,
                                     rounds, c->stream)) return r;
        if (T) CU_TRY(cudaMemcpy(T, d_T, sizeof(double) * BN, cudaMemcpyDeviceToHost));
        if (coeffs) CU_TRY(cudaMemcpy(coeffs, d_C, sizeof(double) * 18 * BN, cudaMemcpyDeviceToHost));
        return lbfgs_copy_out(lb, B, n, x, f, ret, iterations, evaluations);
    }, [&] { nan_fill(f, B); });
}

// ---- trajectory clearance check (isdf_clearance.cuh) -------------------------------------------------------------------------------
extern "C" int isdf_clearance_default_params(isdf_clearance_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    isdf_config d;
    isdf_default_config(&d);
    p->samples_per_piece = d.integral_intervs; p->pieces_per_traj = 0;
    p->reach = d.safety_hor; p->margin = d.safety_hor;
    return 0;
}

// number of trajectories of a call (0 when N / N0 do not define one)
static int clearance_batch(int N, const isdf_clearance_params *p) {
    if (N < 1 || !p || p->pieces_per_traj < 0) return 0;
    if (p->pieces_per_traj == 0) return 1;
    return (N % p->pieces_per_traj == 0) ? N / p->pieces_per_traj : 0;
}

// every check that needs no device work, in the order of include/isdf.h's error list
static int clearance_check(isdf_ctx *c, int N, const isdf_clearance_params *p) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (N < 1) return fail(ISDF_ERR_INVALID, "N < 1");
    if (p->samples_per_piece < 1) return fail(ISDF_ERR_INVALID, "samples_per_piece < 1");
    if (!(p->reach > 0.0) || !std::isfinite(p->reach)) return fail(ISDF_ERR_INVALID, "reach must be positive and finite");
    if (std::isnan(p->margin) || p->margin > p->reach) return fail(ISDF_ERR_INVALID, "margin must not exceed reach");
    if (clearance_batch(N, p) == 0) return fail(ISDF_ERR_INVALID, "pieces_per_traj must be 0 or divide N");
    if ((long long)N * (p->samples_per_piece + 1) > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "N * (samples_per_piece + 1) must fit in 31 bits");
    if (c->world > 1) return fail(ISDF_ERR_UNSUPPORTED, "the clearance check is not sharded: call it on a context with isdf_set_shard(ctx, 0, 1)");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    // the window of a sample spans at most 2 H sqrt(3) / res + 3 voxels per axis (rotated H box, one voxel of slack on each side); the
    // 1023-voxel limit of the pose-window offsets applies as in the discrete path
    const double H = c->dcfg.half_bd + p->reach;
    if (2.0 * H * std::sqrt(3.0) / c->map.grid.res + 4.0 > (double)WINDOW_AXIS_MAX)
        return fail(ISDF_ERR_INVALID, "reach too large for this map resolution: a sample window would exceed 1023 voxels per axis");
    return 0;
}

// a host trajectory block [coeffs 18N | T N] staged in buf on c->stream: the coefficients at buf.p, the durations at *d_T
static int stage_traj(isdf_ctx *c, DevBuf<double> &buf, int N, const double *T, const double *coeffs, const double **d_T) {
    CU_TRY(buf.ensure((size_t)19 * N));
    CU_TRY(cudaMemcpyAsync(buf.p, coeffs, sizeof(double) * 18 * N, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(cudaMemcpyAsync(buf.p + 18 * (size_t)N, T, sizeof(double) * N, cudaMemcpyHostToDevice, c->stream));
    *d_T = buf.p + 18 * (size_t)N;
    return 0;
}

// the clearance scan of the uniform samples of q over N pieces of (d_T, d_C); outputs, cursor, counters, hit flags and sample list are
// the caller's
static ClrArgs clearance_args(const isdf_ctx *c, int N, const double *d_T, const double *d_C, const isdf_clearance_params &q) {
    ClrArgs A = {};
    A.grid = c->map.grid; A.shape = c->mesh.shape; A.fp = c->dcfg.fp; A.half_bd = c->dcfg.half_bd;
    A.reach = q.reach; A.margin = q.margin;
    A.N = N; A.K = q.samples_per_piece; A.N0 = q.pieces_per_traj == 0 ? N : q.pieces_per_traj;
    A.T = d_T; A.C = d_C;
    return A;
}
static int clearance_mode(const isdf_ctx *c) {
    return c->mesh.shape.kind != ISDF_SHAPE_MESH ? 0 : (c->mesh.shape.mesh.sign_mode == MESH_SIGN_WINDING ? 2 : 1);
}
// CTAs of a scan over n samples: one warp per sample, at most every resident CTA
static unsigned clearance_grid(const isdf_ctx *c, long long n) {
    const long long want = (n + CLR_WARPS - 1) / CLR_WARPS;
    return (unsigned)std::max<long long>(1, std::min(want, (long long)c->sm_count * c->clr_blocks));
}

// on failure every summary reads "not shown to be free": min_clearance, t_min, first_hit NaN, voxel_min / piece_min / sample_min /
// colliding_samples -1, collision_free 0
static isdf_clearance_summary clearance_failed_summary() {
    isdf_clearance_summary s;
    s.min_clearance = s.t_min = s.first_hit = std::numeric_limits<double>::quiet_NaN();
    s.voxel_min = -1; s.piece_min = s.sample_min = s.colliding_samples = -1; s.collision_free = 0;
    return s;
}

// the summaries of a failed clearance check or certificate: max(B, 1) records at a host pointer, or, with dc, B records at a device pointer
// of dc's device after stream st (best effort: the pointer itself may be what was wrong)
template <typename S>
static void write_failed_summaries(S *out, int B, const S &bad, isdf_ctx *dc = nullptr, cudaStream_t st = nullptr) {
    if (!out || (dc && B < 1)) return;
    const std::vector<S> v((size_t)std::max(B, 1), bad);
    if (!dc) { std::copy(v.begin(), v.end(), out); return; }
    cudaSetDevice(dc->device);
    cudaStreamSynchronize(st);
    cudaMemcpy(out, v.data(), sizeof(S) * v.size(), cudaMemcpyHostToDevice);
    cudaGetLastError();
}

extern "C" int isdf_trajectory_clearance_device(isdf_ctx *c, int N, const double *d_T, const double *d_coeffs, const isdf_clearance_params *p,
                                                double *d_sample_clearance, int64_t *d_sample_voxel, isdf_clearance_summary *d_summary,
                                                void *cuda_stream) {
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    return poison_on_failure([&]() -> int {
        if (int r = clearance_check(c, N, p)) return r;
        if (!d_T || !d_coeffs || !d_sample_clearance || !d_sample_voxel || !d_summary) return fail(ISDF_ERR_INVALID, "NULL device pointer");
        if (set_device(c)) return ISDF_ERR_CUDA;
        ClrArgs A = clearance_args(c, N, d_T, d_coeffs, *p);   // no sample list, no hit flags: the uniform samples of the definition
        A.clear = d_sample_clearance; A.voxel = (long long *)d_sample_voxel; A.summary = (ClrSummary *)d_summary;
        CU_TRY(c->clr.d_cursor.ensure(1)); CU_TRY(c->clr.d_counters.ensure(2));
        CU_TRY(cudaMemsetAsync(c->clr.d_cursor.p, 0, sizeof(int), st));
        CU_TRY(cudaMemsetAsync(c->clr.d_counters.p, 0, 2 * sizeof(unsigned long long), st));
        A.cursor = c->clr.d_cursor.p; A.counters = c->clr.d_counters.p;
        CU_TRY(clearance_launch(A, clearance_mode(c), clearance_grid(c, (long long)N * (A.K + 1)), st));
        c->stats.kernel_launches += 2;   // scan kernel, summary kernel
        return 0;
    }, [&] { if (c) write_failed_summaries(d_summary, clearance_batch(N, p), clearance_failed_summary(), c, st); });
}

extern "C" int isdf_trajectory_clearance(isdf_ctx *c, int N, const double *T, const double *coeffs, const isdf_clearance_params *p,
                                         double *sample_clearance, int64_t *sample_voxel, isdf_clearance_summary *summary) {
    return poison_on_failure([&]() -> int {
        if (int r = clearance_check(c, N, p)) return r;
        if (!T || !coeffs || !summary) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        const int B = clearance_batch(N, p);
        const size_t S = (size_t)N * (p->samples_per_piece + 1);
        const double *d_T;
        if (int r = stage_traj(c, c->clr.d_in, N, T, coeffs, &d_T)) return r;
        CU_TRY(c->clr.d_clear.ensure(S)); CU_TRY(c->clr.d_vox.ensure(S)); CU_TRY(c->clr.d_sum.ensure((size_t)B));
        if (int r = isdf_trajectory_clearance_device(c, N, d_T, c->clr.d_in.p, p, c->clr.d_clear.p, (int64_t *)c->clr.d_vox.p,
                                                     (isdf_clearance_summary *)c->clr.d_sum.p, c->stream)) return r;
        CU_TRY(cudaMemcpyAsync(summary, c->clr.d_sum.p, sizeof(isdf_clearance_summary) * B, cudaMemcpyDeviceToHost, c->stream));
        if (sample_clearance) CU_TRY(cudaMemcpyAsync(sample_clearance, c->clr.d_clear.p, sizeof(double) * S, cudaMemcpyDeviceToHost, c->stream));
        if (sample_voxel) CU_TRY(cudaMemcpyAsync(sample_voxel, c->clr.d_vox.p, sizeof(int64_t) * S, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
        return 0;
    }, [&] { write_failed_summaries(summary, clearance_batch(N, p), clearance_failed_summary()); });
}

// ---- continuous clearance certificate (isdf_certify.cuh) --------------------------------------------------------------------------
extern "C" int isdf_certify_default_params(isdf_certify_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    std::memset(p, 0, sizeof(*p));
    isdf_clearance_default_params(&p->clearance);
    p->clearance.reach = 2.0 * p->clearance.margin;
    p->max_depth = 16; p->max_samples_per_traj = 2048;
    return 0;
}

// the shape conditions of the certificate (include/isdf.h): a true Euclidean distance outside the body and a body inside the half_bd box.
// *r: the body radius about the body origin (0 for rotation-invariant bodies), padded against the rounding of its own computation
static int certify_shape(isdf_ctx *c, double *r) {
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    const DevShape &s = c->mesh.shape;
    const double hb = c->dcfg.half_bd;
    auto inside = [&](const double p[3]) { return std::fabs(p[0]) <= hb && std::fabs(p[1]) <= hb && std::fabs(p[2]) <= hb; };
    double rr = 0.0;
    if (s.kind == ISDF_SHAPE_BALL) {
        if (!(s.par[0] >= 0.0 && s.par[0] <= hb)) return fail(ISDF_ERR_UNSUPPORTED, "certificate: the Ball's radius must lie in [0, half_bd]");
    } else if (s.kind == ISDF_SHAPE_BOX) {
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                const double d = s.rot[3 * i] * s.rot[3 * j] + s.rot[3 * i + 1] * s.rot[3 * j + 1] + s.rot[3 * i + 2] * s.rot[3 * j + 2];
                if (!(std::fabs(d - (i == j ? 1.0 : 0.0)) <= 1e-12)) return fail(ISDF_ERR_UNSUPPORTED, "certificate: the Box rotation is not orthonormal to 1e-12");
            }
        if (!(s.par[0] >= 0.0 && s.par[1] >= 0.0 && s.par[2] >= 0.0)) return fail(ISDF_ERR_UNSUPPORTED, "certificate: negative Box half extents");
        for (int k = 0; k < 8; k++) {   // body point of shape-frame corner q: Rotate q + trans (shape_pre inverted)
            const double q[3] = {(k & 1) ? s.par[0] : -s.par[0], (k & 2) ? s.par[1] : -s.par[1], (k & 4) ? s.par[2] : -s.par[2]};
            double p[3];
            for (int j = 0; j < 3; j++) p[j] = s.rot[3 * j] * q[0] + s.rot[3 * j + 1] * q[1] + s.rot[3 * j + 2] * q[2] + s.trans[j];
            if (!inside(p)) return fail(ISDF_ERR_UNSUPPORTED, "certificate: the Box reaches beyond the half_bd box");
            rr = std::max(rr, std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));
        }
    } else if (s.kind == ISDF_SHAPE_MESH) {
        if (s.mesh.sign_mode != MESH_SIGN_PSEUDONORMAL) return fail(ISDF_ERR_UNSUPPORTED, "certificate: a winding-sign mesh SDF is not a distance");
        for (int k = 0; k < 8; k++) {
            const double p[3] = {(k & 1) ? s.mesh.bhi[0] : s.mesh.blo[0], (k & 2) ? s.mesh.bhi[1] : s.mesh.blo[1], (k & 4) ? s.mesh.bhi[2] : s.mesh.blo[2]};
            if (!inside(p)) return fail(ISDF_ERR_UNSUPPORTED, "certificate: the mesh's bounding box reaches beyond the half_bd box");
            rr = std::max(rr, std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));
        }
    } else if (s.kind != ISDF_SHAPE_POINT) {
        return fail(ISDF_ERR_UNSUPPORTED, "certificate: supported shapes are Ball, Point, Box and exact-sign meshes (their SDF is a distance)");
    }
    *r = rr * (1.0 + 1e-12);
    return 0;
}

static int certify_batch(int N, const isdf_certify_params *p) { return p ? clearance_batch(N, &p->clearance) : 0; }

// every check that needs no device work; *r as certify_shape
static int certify_check(isdf_ctx *c, int N, const isdf_certify_params *p, double *r) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (p->reserved_[0] || p->reserved_[1]) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    if (p->max_depth < 0 || p->max_depth > 64) return fail(ISDF_ERR_INVALID, "max_depth must lie in [0, 64]");
    if (p->max_samples_per_traj < 0) return fail(ISDF_ERR_INVALID, "max_samples_per_traj < 0");
    const isdf_clearance_params &q = p->clearance;
    if (!(q.margin >= 0.0) || !(q.margin < q.reach)) return fail(ISDF_ERR_INVALID, "the certificate needs 0 <= margin < reach");
    if (int rr = clearance_check(c, N, &q)) return rr;
    const long long B = certify_batch(N, p), K = q.samples_per_piece;
    if ((long long)N * (2 * K + 1) + 3 * B * p->max_samples_per_traj > 0x7fffffffll)
        return fail(ISDF_ERR_INVALID, "N (2 K_c + 1) + 3 B max_samples_per_traj must fit in 31 bits");
    return certify_shape(c, r);
}

static CertArgs certify_args(isdf_ctx *c, double r, double reach, int N, const double *d_T, const double *d_C) {
    CertArgs A = {};
    A.fp = c->dcfg.fp; A.r = r; A.H = c->dcfg.half_bd + reach;
    A.N = N; A.T = d_T; A.C = d_C;
    return A;
}

static int certify_run(isdf_ctx *c, int N, const double *d_T, const double *d_C, const isdf_certify_params *p, double r, CertSummary *d_sum,
                       cudaStream_t st) {
    auto &z = c->cert;
    const isdf_clearance_params &q = p->clearance;
    const int K = q.samples_per_piece, N0 = q.pieces_per_traj == 0 ? N : q.pieces_per_traj, B = N / N0, M = p->max_samples_per_traj;
    const size_t S0 = (size_t)N * (K + 1), I0 = (size_t)N * K, Smax = S0 + (size_t)B * M, Lmax = I0 + (size_t)B * M;
    z.last_leaves = 0;
    CU_TRY(z.d_toff.ensure(N)); CU_TRY(z.d_sp.ensure(Smax)); CU_TRY(z.d_st.ensure(Smax)); CU_TRY(z.d_sc.ensure(Smax)); CU_TRY(z.d_sv.ensure(Smax));
    CU_TRY(z.d_hit.ensure(B)); CU_TRY(z.d_traj.ensure(B)); CU_TRY(z.d_tot.ensure(2)); CU_TRY(z.d_cursor.ensure(1)); CU_TRY(z.h_tot.ensure(1));
    CU_TRY(z.d_iv[0].ensure(I0)); CU_TRY(z.d_leaves.ensure(Lmax));
    CertArgs A = certify_args(c, r, q.reach, N, d_T, d_C);
    A.margin = q.margin; A.K = K; A.N0 = N0; A.B = B; A.max_depth = p->max_depth; A.max_samples = M;
    A.toff = z.d_toff.p; A.sp = z.d_sp.p; A.st = z.d_st.p; A.sc = z.d_sc.p; A.sv = z.d_sv.p; A.hit = z.d_hit.p;
    A.leaves = z.d_leaves.p; A.traj = z.d_traj.p; A.summary = d_sum; A.tot = z.d_tot.p;
    A.cur = z.d_iv[0].p;
    CU_TRY(certify_init_launch(A, st));
    c->stats.kernel_launches++;
    // the scan: round 0 is the clearance check's own uniform samples, later rounds the new midpoints
    ClrArgs S = clearance_args(c, N, d_T, d_C, q);   // no counters: a certificate leaves isdf_dbg_clearance_counts as it was
    S.clear = z.d_sc.p; S.voxel = z.d_sv.p; S.cursor = z.d_cursor.p; S.hit = z.d_hit.p;
    auto scan = [&](long long n) -> int {
        CU_TRY(cudaMemsetAsync(z.d_cursor.p, 0, sizeof(int), st));
        CU_TRY(clearance_scan_launch(S, clearance_mode(c), clearance_grid(c, n), st));
        c->stats.kernel_launches++;
        return 0;
    };
    if (int rr = scan((long long)S0)) return rr;
    long long nact = (long long)I0, S_cur = (long long)S0, L_cur = 0;
    int cur = 0;
    for (;;) {
        CU_TRY(z.d_iv[cur ^ 1].ensure((size_t)std::max(2 * nact, 1ll))); CU_TRY(z.d_scr.ensure((size_t)nact));
        A.cur = z.d_iv[cur].p; A.next = z.d_iv[cur ^ 1].p; A.scr = z.d_scr.p;
        A.S_cur = (int)S_cur; A.L_cur = (int)L_cur; A.nact = (int)nact;
        CU_TRY(certify_round_launch(A, st));
        c->stats.kernel_launches += 2;
        CU_TRY(cudaMemcpyAsync(z.h_tot.p, z.d_tot.p, sizeof(int), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
        const long long ns = *z.h_tot.p;
        L_cur += nact - ns;
        if (ns == 0) break;
        S.st = z.d_st.p + S_cur; S.sp = z.d_sp.p + S_cur; S.nlist = (int)ns; S.clear = z.d_sc.p + S_cur; S.voxel = z.d_sv.p + S_cur;
        if (int rr = scan(ns)) return rr;
        S_cur += ns; nact = 2 * ns; cur ^= 1;
    }
    CU_TRY(certify_finish_launch(A, st));
    c->stats.kernel_launches++;
    z.last_leaves = L_cur;
    return 0;
}

// on failure every summary reads verdict 0 (UNDECIDED), lower_bound / min_clearance / t_min / first_hit NaN, counts -1
static isdf_certify_summary certify_failed_summary() {
    isdf_certify_summary s;
    s.lower_bound = s.min_clearance = s.t_min = s.first_hit = std::numeric_limits<double>::quiet_NaN();
    s.voxel_min = -1; s.verdict = 0; s.samples = s.undecided_intervals = s.depth = -1;
    return s;
}

extern "C" int isdf_trajectory_certify_device(isdf_ctx *c, int N, const double *d_T, const double *d_coeffs, const isdf_certify_params *p,
                                              isdf_certify_summary *d_summary, void *cuda_stream) {
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    return poison_on_failure([&]() -> int {
        double r = 0.0;
        if (int rc = certify_check(c, N, p, &r)) return rc;
        if (!d_T || !d_coeffs || !d_summary) return fail(ISDF_ERR_INVALID, "NULL device pointer");
        if (set_device(c)) return ISDF_ERR_CUDA;
        return certify_run(c, N, d_T, d_coeffs, p, r, (CertSummary *)d_summary, st);
    }, [&] { if (c) write_failed_summaries(d_summary, certify_batch(N, p), certify_failed_summary(), c, st); });
}

extern "C" int isdf_trajectory_certify(isdf_ctx *c, int N, const double *T, const double *coeffs, const isdf_certify_params *p,
                                       isdf_certify_summary *summary) {
    return poison_on_failure([&]() -> int {
        double r = 0.0;
        if (int rc = certify_check(c, N, p, &r)) return rc;
        if (!T || !coeffs || !summary) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        const int B = certify_batch(N, p);
        const double *d_T;
        if (int rc = stage_traj(c, c->cert.d_in, N, T, coeffs, &d_T)) return rc;
        CU_TRY(c->cert.d_sum.ensure((size_t)B));
        if (int rc = isdf_trajectory_certify_device(c, N, d_T, c->cert.d_in.p, p, (isdf_certify_summary *)c->cert.d_sum.p, c->stream)) return rc;
        CU_TRY(cudaMemcpyAsync(summary, c->cert.d_sum.p, sizeof(isdf_certify_summary) * B, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
        return 0;
    }, [&] { write_failed_summaries(summary, certify_batch(N, p), certify_failed_summary()); });
}

// ---- multi-GPU: rank-ordered sum of the sharded evaluation through NVLink peer memory (isdf_peer.cuh) ------------------------------
static size_t peer_bytes(int world, int cap) { return sizeof(unsigned long long) * 2 * PEER_MAX + sizeof(double) * 2 * (size_t)world * cap; }

extern "C" int isdf_peer_export(isdf_ctx *c, int world, int max_doubles, unsigned char *handle64) {
    if (!c || !handle64 || world < 2 || world > PEER_MAX || max_doubles < 1) return fail(ISDF_ERR_INVALID, "bad argument (2 <= world <= 16)");
    if (set_device(c)) return ISDF_ERR_CUDA;
    if (c->peer.args.world) return fail(ISDF_ERR_STATE, "already connected: isdf_peer_disconnect first");
    c->peer.buf = {};
    CU_TRY(c->peer.buf.ensure(peer_bytes(world, max_doubles)));
    CU_TRY(cudaMemset(c->peer.buf.p, 0, peer_bytes(world, max_doubles)));
    CU_TRY(c->peer.d_status.ensure(1));
    CU_TRY(cudaMemset(c->peer.d_status.p, 0, sizeof(int)));
    cudaIpcMemHandle_t h;
    CU_TRY(cudaIpcGetMemHandle(&h, c->peer.buf.p));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    std::memcpy(handle64, &h, 64);
    c->peer.world_alloc = world; c->peer.cap = max_doubles;
    return 0;
}

extern "C" int isdf_peer_connect(isdf_ctx *c, int world, int rank, const unsigned char *handles, int fuse_into_eval) {
    if (!c || !handles || rank < 0 || rank >= world) return fail(ISDF_ERR_INVALID, "bad argument");
    if (!c->peer.buf.p || world != c->peer.world_alloc) return fail(ISDF_ERR_STATE, "isdf_peer_export with the same world first");
    if (c->peer.args.world != 0) return fail(ISDF_ERR_STATE, "already connected: isdf_peer_disconnect first");
    if (set_device(c)) return ISDF_ERR_CUDA;
    PeerArgs P = {};
    P.world = world; P.rank = rank; P.cap = c->peer.cap; P.epoch = 0; P.status = c->peer.d_status.p;
    for (int p = 0; p < world; p++) {
        void *base = c->peer.buf.p;
        if (p != rank) {
            cudaIpcMemHandle_t h;
            std::memcpy(&h, handles + (size_t)64 * p, 64);
            cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) {
                c->peer.close_handles();
                return fail(ISDF_ERR_CUDA, std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
            }
            c->peer.open[p] = base;
        }
        P.flags[p] = (unsigned long long *)base;
        P.slots[p] = (double *)((char *)base + sizeof(unsigned long long) * 2 * PEER_MAX);
    }
    c->peer.args = P;
    c->peer.fused = fuse_into_eval != 0;
    return 0;
}

extern "C" int isdf_peer_allreduce_device(isdf_ctx *c, double *d_vec, int n, void *cuda_stream) {
    if (!c || !d_vec || n < 1) return fail(ISDF_ERR_INVALID, "bad argument");
    if (c->peer.args.world < 2) return fail(ISDF_ERR_STATE, "not connected (isdf_peer_connect)");
    if (n > c->peer.args.cap) return fail(ISDF_ERR_INVALID, "vector longer than the exchange buffer");
    if (set_device(c)) return ISDF_ERR_CUDA;
    return peer_allreduce_launch(c, d_vec, n, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_peer_status(isdf_ctx *c) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!c->peer.d_status.p) return 0;
    if (set_device(c)) return ISDF_ERR_CUDA;
    int st = 0;
    CU_TRY(cudaMemcpy(&st, c->peer.d_status.p, sizeof(int), cudaMemcpyDeviceToHost));
    if (st) return fail(ISDF_ERR_CUDA, "peer exchange timed out: a rank did not reach the same evaluation");
    return 0;
}

extern "C" int isdf_peer_disconnect(isdf_ctx *c) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (set_device(c)) return ISDF_ERR_CUDA;
    cudaDeviceSynchronize();
    c->peer.close_handles();
    c->peer.buf = {};
    c->peer.args = PeerArgs{}; c->peer.fused = false; c->peer.world_alloc = 0; c->peer.cap = 0;
    return 0;
}

// ---- front end: attitude-kernel feasibility (isdf_frontend.cuh), SURVEY §8f row 4 ------------------------------------------------
// Eigen::AngleAxisd(rotx, UnitX) * Eigen::AngleAxisd(roty, UnitY) -> Matrix3d (Shape.hpp:431): quaternion product, toRotationMatrix
static void attitude_rotation(double rotx, double roty, double R[9]) {
    const double sa = std::sin(0.5 * rotx), sb = std::sin(0.5 * roty);
    const double aw = std::cos(0.5 * rotx), ax = sa * 1.0, ay = sa * 0.0, az = sa * 0.0;
    const double bw = std::cos(0.5 * roty), bx = sb * 0.0, by = sb * 1.0, bz = sb * 0.0;
    const double w = aw * bw - ax * bx - ay * by - az * bz;
    const double x = aw * bx + ax * bw + ay * bz - az * by;
    const double y = aw * by + ay * bw + az * bx - ax * bz;
    const double z = aw * bz + az * bw + ax * by - ay * bx;
    const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1.0 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1.0 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.0 - (txx + tyy);
}

static FrontArgs front_args(isdf_ctx *c) {
    FrontArgs A = {};
    A.grid = c->map.grid; A.shape = c->mesh.shape;
    for (int i = 0; i < 9; i++) A.rot[i] = c->mesh.shape.rot[i];
    for (int i = 0; i < 3; i++) A.trans[i] = c->mesh.shape.trans[i];
    if (c->mesh.shape.kind != ISDF_SHAPE_MESH) {   // the kernel applies ((pos - trans) * Rotate) * R_obj itself and evaluates the bare body
        const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        for (int i = 0; i < 9; i++) A.shape.rot[i] = I[i];
        for (int i = 0; i < 3; i++) A.shape.trans[i] = 0.0;
    }
    A.ks = c->fe.ks; A.xk = c->fe.xk; A.yk = c->fe.yk; A.natt = c->fe.xk * c->fe.yk;
    A.res = c->cfg.occupancy_resolution; A.margin = c->fe.margin;
    A.att_rot = c->fe.d_rot.p; A.kernels = c->fe.d_kernels.p; A.offset_masks = c->fe.d_masks.p; A.order = c->fe.d_order.p;
    A.max_roll = c->fe.max_roll; A.max_pitch = c->fe.max_pitch; A.ang_res = c->fe.ang_res;
    A.core_rows = c->fe.d_core.p; A.ncore = c->fe.ncore; A.urows = c->fe.d_urows.p; A.nurow = c->fe.nurow; A.chunks = c->fe.d_chunks.p; A.nchunk = c->fe.nchunk; A.tab = c->fe.d_tab.p; A.ntab = c->fe.ntab; A.surv = c->fe.d_surv.p; A.surv_count = c->fe.d_count.p;
    return A;
}

extern "C" int isdf_frontend_build_kernels(isdf_ctx *c, const isdf_kernel_config *kc, int *xkernel_size, int *ykernel_size) {
    if (!c || !kc) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    if (!(kc->kernel_ang_res > 0) || kc->kernel_max_roll < 0 || kc->kernel_max_pitch < 0) return fail(ISDF_ERR_INVALID, "bad attitude grid");
    const int ks = c->cfg.kernel_size;
    if (ks < 1 || (ks & 1) == 0) return fail(ISDF_ERR_INVALID, "kernel_size must be odd (Shape.hpp:258)");
    if (ks > 29) return fail(ISDF_ERR_UNSUPPORTED, "kernel_size > 29");
    const int xk = (int)std::floor(2 * kc->kernel_max_roll / kc->kernel_ang_res) + 1, yk = (int)std::floor(2 * kc->kernel_max_pitch / kc->kernel_ang_res) + 1;   // swm:135-136
    if (xk * yk > FE_MAX_ATT) return fail(ISDF_ERR_UNSUPPORTED, "more than 128 attitudes");
    if (set_device(c)) return ISDF_ERR_CUDA;
    const int natt = xk * yk, n3 = ks * ks * ks;
    std::vector<double> rot((size_t)9 * natt, 0.0);
    {
        int i = 0;
        for (double roll = -kc->kernel_max_roll; roll <= kc->kernel_max_roll && i < xk; roll += kc->kernel_ang_res, i++) {   // Shape.hpp:424-427
            int j = 0;
            for (double pitch = -kc->kernel_max_pitch; pitch <= kc->kernel_max_pitch && j < yk; pitch += kc->kernel_ang_res, j++)
                attitude_rotation(roll * M_PI / 180.0, pitch * M_PI / 180.0, &rot[(size_t)9 * (i * yk + j)]);
        }
    }
    // visiting order of visit_kernels_by_distance for every start attitude: level pose, then the BFS sequence without it
    std::vector<uint8_t> order((size_t)natt * natt, 0xff);
    const int zi = (xk - 1) / 2, zj = (yk - 1) / 2;
    for (int sx = 0; sx < xk; sx++)
        for (int sy = 0; sy < yk; sy++) {
            uint8_t *o = &order[(size_t)(sx * yk + sy) * natt];
            int n = 0;
            o[n++] = (uint8_t)(zi * yk + zj);
            std::vector<uint8_t> vis((size_t)natt, 0);
            std::queue<std::pair<int, int>> q;
            q.push({sx, sy}); vis[sx * yk + sy] = 1;
            const int dirs[4][2] = {{0, 1}, {0, -1}, {1, 0}, {-1, 0}};
            int deep = 0;
            while (!q.empty()) {
                deep++;
                const int x = q.front().first, y = q.front().second;
                q.pop();
                if (x != zi || y != zj) o[n++] = (uint8_t)(x * yk + y);
                for (auto &d : dirs) {
                    const int nx = x + d[0], ny = y + d[1];
                    if (nx < 0 || nx >= xk || ny < 0 || ny >= yk || vis[nx * yk + ny]) continue;
                    vis[nx * yk + ny] = 1;
                    q.push({nx, ny});
                }
                if (deep > 800) break;   // maxdeepth (swm:852)
            }
        }
    c->fe.ready = false;   // the current kernels and tables are overwritten from here on
    CU_TRY(c->fe.d_rot.upload(rot.data(), rot.size(), c->stream));
    CU_TRY(c->fe.d_order.upload(order.data(), order.size(), c->stream));
    CU_TRY(c->fe.d_kernels.ensure((size_t)natt * n3));
    CU_TRY(c->fe.d_masks.ensure((size_t)4 * n3));
    c->fe.xk = xk; c->fe.yk = yk; c->fe.ks = ks;
    c->fe.max_roll = kc->kernel_max_roll; c->fe.max_pitch = kc->kernel_max_pitch; c->fe.ang_res = kc->kernel_ang_res;
    c->fe.margin = std::max(kc->front_end_safeh, c->cfg.occupancy_resolution / 2);   // Shape.hpp:423
    FrontArgs A = front_args(c);
    const long long nt = (long long)natt * n3;
    k_frontend_kernels<<<(unsigned)((nt + 255) / 256), 256, 0, c->stream>>>(A);
    k_frontend_offset_masks<<<(unsigned)((n3 + 255) / 256), 256, 0, c->stream>>>(A);
    c->stats.kernel_launches += 2;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaStreamSynchronize(c->stream));
    // the kernel core (offsets every attitude occupies), row by row, densest rows first: pass 1 of the two-pass feasibility kernel
    {
        std::vector<uint32_t> om((size_t)4 * n3);
        CU_TRY(cudaMemcpy(om.data(), c->fe.d_masks.p, sizeof(uint32_t) * om.size(), cudaMemcpyDeviceToHost));
        uint32_t valid[4];
        for (int k = 0; k < 4; k++) { const int lo = 32 * k; valid[k] = natt >= lo + 32 ? 0xffffffffu : (natt > lo ? ((1u << (natt - lo)) - 1u) : 0u); }
        std::vector<uint2> rows, urows;
        for (int a = 0; a < ks; a++)
            for (int b = 0; b < ks; b++) {
                uint32_t bits = 0, ubits = 0;
                for (int cc = 0; cc < ks; cc++) {
                    const uint32_t *m = &om[(size_t)4 * ((a * ks + b) * ks + cc)];
                    if (m[0] == valid[0] && m[1] == valid[1] && m[2] == valid[2] && m[3] == valid[3]) bits |= 1u << cc;
                    if (m[0] | m[1] | m[2] | m[3]) ubits |= 1u << cc;
                }
                if (bits) rows.push_back(make_uint2((uint32_t)a | ((uint32_t)b << 8), bits));
                if (ubits) urows.push_back(make_uint2((uint32_t)a | ((uint32_t)b << 8), ubits));
            }
        c->fe.nurow = (int)urows.size();
        if (!urows.empty()) CU_TRY(c->fe.d_urows.upload(urows.data(), urows.size(), c->stream));
        // pattern tables of the union rows, in chunks of <= FE_CHUNK_BITS offsets (pass 2 of the table-driven kernels)
        std::vector<uint2> chunks; std::vector<uint4> tab;
        for (const uint2 &ur : urows) {
            const int a = (int)(ur.x & 0xffu), b = (int)(ur.x >> 8);
            const int lo = __builtin_ctz(ur.y), hi = 31 - __builtin_clz(ur.y);
            for (int c0 = lo; c0 <= hi; c0 += FE_CHUNK_BITS) {
                const int len = std::min(FE_CHUNK_BITS, hi - c0 + 1);
                if (((ur.y >> c0) & ((1u << len) - 1u)) == 0u) continue;
                chunks.push_back(make_uint2(ur.x | ((uint32_t)c0 << 16) | ((uint32_t)len << 24), (uint32_t)tab.size()));
                for (uint32_t pat = 0; pat < (1u << len); pat++) {
                    uint4 e = make_uint4(0u, 0u, 0u, 0u);
                    for (int i = 0; i < len; i++)
                        if ((pat >> i) & 1u) { const uint32_t *m = &om[(size_t)4 * ((a * ks + b) * ks + c0 + i)]; e.x |= m[0]; e.y |= m[1]; e.z |= m[2]; e.w |= m[3]; }
                    tab.push_back(e);
                }
            }
        }
        c->fe.nchunk = (int)chunks.size(); c->fe.ntab = (int)tab.size();
        if (getenv("ISDF_VERBOSE")) fprintf(stderr, "[isdf] front end: %d attitudes, kernel core %zu rows, union %zu rows, %zu chunks, %zu table entries (%.1f KB)\n", natt, rows.size(), urows.size(), chunks.size(), tab.size(), tab.size() * 16e-3);
        if (!chunks.empty()) { CU_TRY(c->fe.d_chunks.upload(chunks.data(), chunks.size(), c->stream)); CU_TRY(c->fe.d_tab.upload(tab.data(), tab.size(), c->stream)); }
        std::stable_sort(rows.begin(), rows.end(), [](const uint2 &p, const uint2 &q) { return __builtin_popcount(p.y) > __builtin_popcount(q.y); });
        c->fe.ncore = (int)rows.size();
        if (!rows.empty()) CU_TRY(c->fe.d_core.upload(rows.data(), rows.size(), c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
    }
    c->fe.ready = true;
    if (xkernel_size) *xkernel_size = xk;
    if (ykernel_size) *ykernel_size = yk;
    return 0;
}

extern "C" int isdf_frontend_get_kernels(isdf_ctx *c, uint8_t *out, int n) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->fe.ready) return fail(ISDF_ERR_STATE, "isdf_frontend_build_kernels first (and again after changing the shape)");
    const size_t want = (size_t)c->fe.xk * c->fe.yk * c->fe.ks * c->fe.ks * c->fe.ks;
    if ((size_t)n != want) return fail(ISDF_ERR_INVALID, "n must be xkernel_size * ykernel_size * kernel_size^3");
    if (set_device(c)) return ISDF_ERR_CUDA;
    CU_TRY(cudaMemcpy(out, c->fe.d_kernels.p, want, cudaMemcpyDeviceToHost));
    return 0;
}

static int frontend_state(isdf_ctx *c) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!c->fe.ready) return fail(ISDF_ERR_STATE, "isdf_frontend_build_kernels first (and again after changing the shape)");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    return 0;
}

// the feasibility pipeline into d_masks (4 words per voxel), or, with d_trav set, into the traversability bits (isdf_frontpath.cuh)
static int frontend_feasibility_run(isdf_ctx *c, uint32_t *d_masks, uint32_t *d_trav, void *cuda_stream) {
    FrontArgs A = front_args(c);
    A.out = d_masks; A.trav = d_trav;
    if (d_trav) CU_TRY(cudaMemsetAsync(d_trav, 0, sizeof(uint32_t) * (size_t)c->map.grid.X * c->map.grid.Y * c->map.grid.Zw, (cudaStream_t)cuda_stream));
    const size_t smem = sizeof(uint32_t) * 4 * (size_t)A.ks * A.ks * A.ks;
    CU_TRY(cudaFuncSetAttribute(k_frontend_feasibility, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long nrun = (long long)c->map.grid.X * c->map.grid.Y * ((c->map.grid.Z + FE_ZRUN - 1) / FE_ZRUN);
    const long long sms = c->sm_count;
    const unsigned grid = (unsigned)std::min<long long>((nrun + 255) / 256, sms * 64);
    // the input picks the pipeline: one pass when no voxel can be settled early (empty kernel core) or the runs outgrow 32-bit
    // survivor indices; two passes otherwise, table-driven when the pattern tables fit into shared memory
    if (c->fe.ncore > 0 && nrun < (1ll << 32)) {
        // two passes: the kernel core settles most voxels of a cluttered map, the mask accumulation runs on the survivors only
        CU_TRY(c->fe.d_surv.ensure((size_t)nrun));
        CU_TRY(c->fe.d_count.ensure(1));
        A.surv = c->fe.d_surv.p; A.surv_count = c->fe.d_count.p;
        CU_TRY(cudaMemsetAsync(c->fe.d_count.p, 0, sizeof(unsigned), (cudaStream_t)cuda_stream));
        const size_t tsmem = sizeof(uint4) * ((size_t)c->fe.ntab + (size_t)c->fe.nchunk);
        if (c->fe.nchunk > 0 && tsmem <= 200 * 1024) {
            // throughput form: zero-filled output, bit-parallel core pass (32 voxels per thread), table-driven accumulation on the survivors
            const long long nvox = (long long)c->map.grid.X * c->map.grid.Y * c->map.grid.Z;
            if (!d_trav) CU_TRY(cudaMemsetAsync(d_masks, 0, sizeof(uint32_t) * 4 * (size_t)nvox, (cudaStream_t)cuda_stream));
            const long long nword = (long long)c->map.grid.X * c->map.grid.Y * c->map.grid.Zw;
            CU_TRY(cudaFuncSetAttribute(k_frontend_survivors_tab, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tsmem));
            k_frontend_core_words<<<(unsigned)std::min<long long>((nword + 255) / 256, sms * 32), 256, 0, (cudaStream_t)cuda_stream>>>(A);
            // 32 warps per SM hide the row reads: two CTAs of 512 threads when two tables fit into shared memory, else one of 1024
            // (1 KB of every CTA's shared memory is reserved by the runtime)
            if (2 * (tsmem + 1024) <= c->smem_per_sm) k_frontend_survivors_tab<<<(unsigned)sms * 2, 512, tsmem, (cudaStream_t)cuda_stream>>>(A);
            else k_frontend_survivors_tab<<<(unsigned)sms, 1024, tsmem, (cudaStream_t)cuda_stream>>>(A);
        } else {
            CU_TRY(cudaFuncSetAttribute(k_frontend_survivors, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            k_frontend_core<<<grid, 256, 0, (cudaStream_t)cuda_stream>>>(A);
            k_frontend_survivors<<<(unsigned)sms * 16, 256, smem, (cudaStream_t)cuda_stream>>>(A);
        }
        c->stats.kernel_launches += 2;
    } else {
        k_frontend_feasibility<<<grid, 256, smem, (cudaStream_t)cuda_stream>>>(A);
        c->stats.kernel_launches++;
    }
    CU_TRY(cudaGetLastError());
    return 0;
}

extern "C" int isdf_frontend_feasibility_device(isdf_ctx *c, uint32_t *d_masks, void *cuda_stream) {
    int r = frontend_state(c);
    if (r) return r;
    if (!d_masks) return fail(ISDF_ERR_INVALID, "NULL device pointer");
    if (set_device(c)) return ISDF_ERR_CUDA;
    return frontend_feasibility_run(c, d_masks, nullptr, cuda_stream);
}

extern "C" int isdf_frontend_feasibility(isdf_ctx *c, uint32_t *masks) {
    int r = frontend_state(c);
    if (r) return r;
    if (!masks) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (set_device(c)) return ISDF_ERR_CUDA;
    const size_t nvox = (size_t)c->map.grid.X * c->map.grid.Y * c->map.grid.Z;
    CU_TRY(c->fe.d_out.ensure(4 * nvox));
    CU_TRY(cudaEventRecord(c->ev0, c->stream));
    r = isdf_frontend_feasibility_device(c, c->fe.d_out.p, c->stream);
    if (r) return r;
    CU_TRY(cudaEventRecord(c->ev1, c->stream));
    CU_TRY(cudaMemcpyAsync(masks, c->fe.d_out.p, sizeof(uint32_t) * 4 * nvox, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
    c->stats.last_kernel_ms = ms;
    return 0;
}

extern "C" int isdf_frontend_check_batch(isdf_ctx *c, int n, const int32_t *ind, const double *father_roll_pitch, double *child_roll_pitch, uint8_t *ok) {
    int r = frontend_state(c);
    if (r) return r;
    if (n < 0 || (n > 0 && (!ind || !father_roll_pitch || !child_roll_pitch || !ok))) return fail(ISDF_ERR_INVALID, "bad argument");
    if (n == 0) return 0;
    for (int q = 0; q < n; q++)
        if (ind[3 * q] < 0 || ind[3 * q] >= c->map.grid.X || ind[3 * q + 1] < 0 || ind[3 * q + 1] >= c->map.grid.Y || ind[3 * q + 2] < 0 || ind[3 * q + 2] >= c->map.grid.Z)
            return fail(ISDF_ERR_INVALID, "voxel index outside the map");
    if (set_device(c)) return ISDF_ERR_CUDA;
    CU_TRY(c->fe.d_ind.upload(ind, (size_t)3 * n, c->stream));
    CU_TRY(c->fe.d_father.upload(father_roll_pitch, (size_t)2 * n, c->stream));
    CU_TRY(c->fe.d_child.ensure((size_t)2 * n)); CU_TRY(c->fe.d_ok.ensure(n)); CU_TRY(c->fe.d_out.ensure((size_t)4 * n));
    FrontArgs A = front_args(c);
    A.out = c->fe.d_out.p; A.nq = n; A.q_ind = c->fe.d_ind.p; A.q_father = c->fe.d_father.p; A.q_child = c->fe.d_child.p; A.q_ok = c->fe.d_ok.p;
    const size_t smem = sizeof(uint32_t) * 4 * (size_t)A.ks * A.ks * A.ks;
    CU_TRY(cudaFuncSetAttribute(k_frontend_check, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_frontend_check<<<(unsigned)((n + 255) / 256), 256, smem, c->stream>>>(A);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(child_roll_pitch, c->fe.d_child.p, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaMemcpyAsync(ok, c->fe.d_ok.p, n, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    return 0;
}

// ---- front-end path search (isdf_frontpath.cuh) ------------------------------------------------------------------------------------
constexpr int FP_ROUNDS_PER_CHECK = 8;   // relaxation rounds launched between two reads of the frontier flag

static int path_args_check(isdf_ctx *c, const isdf_frontpath_params *prm) {
    if (int r = frontend_state(c)) return r;
    if (c->world > 1) return fail(ISDF_ERR_UNSUPPORTED, "the front-end path search is not sharded: call it on a context with isdf_set_shard(ctx, 0, 1)");
    if (prm) for (int32_t v : prm->reserved_) if (v != 0) return fail(ISDF_ERR_INVALID, "isdf_frontpath_params: reserved fields must be zero");
    return 0;
}

// isInMap (Gridmap3D.cpp) + getGridIndex (Gridmap3D.cpp:135-175) with its clamps and its "iy < 0 => ix = 0" branches (they cannot fire
// for a point inside the map)
static int path_voxel(const DevGrid &G, const double *p, int id[3], const char *what) {
    for (int a = 0; a < 3; a++)
        if (!std::isfinite(p[a])) return fail(ISDF_ERR_INVALID, std::string(what) + " is not finite");
    for (int a = 0; a < 3; a++)
        if (p[a] < G.bmin[a] || p[a] > G.bmax[a]) return fail(ISDF_ERR_INVALID, std::string(what) + " is outside the map");
    int ix = (int)std::floor((p[0] - G.bmin[0]) / G.res), iy = (int)std::floor((p[1] - G.bmin[1]) / G.res), iz = (int)std::floor((p[2] - G.bmin[2]) / G.res);
    if (ix < 0) ix = 0;
    if (ix >= G.X) ix = G.X - 1;
    if (iy < 0) ix = 0;
    if (iy >= G.Y) iy = G.Y - 1;
    if (iz < 0) ix = 0;
    if (iz >= G.Z) iz = G.Z - 1;
    id[0] = ix; id[1] = iy; id[2] = iz;
    return 0;
}

static PathArgs path_args(isdf_ctx *c, const int s[3], unsigned long long *d_g) {
    const size_t nword = (size_t)c->map.grid.X * c->map.grid.Y * c->map.grid.Zw;
    PathArgs P = {};
    P.grid = c->map.grid; P.trav = c->fp.d_trav.p; P.g = d_g;
    P.front0 = c->fp.d_front.p; P.front1 = c->fp.d_front.p + nword;
    P.flags = c->fp.d_flags.p; P.rounds = c->fp.d_flags.p + FP_FLAG_RING;
    P.sx = s[0]; P.sy = s[1]; P.sz = s[2];
    return P;
}

// traversability grid, then the field from source s into d_g (X*Y*Z bit patterns), on stream st; fills c->fp.info
static int path_field(isdf_ctx *c, const int s[3], unsigned long long *d_g, cudaStream_t st) {
    const DevGrid &G = c->map.grid;
    const size_t nword = (size_t)G.X * G.Y * G.Zw, nvox = (size_t)G.X * G.Y * G.Z;
    for (cudaEvent_t &e : c->fp.ev) if (!e) CU_TRY(cudaEventCreate(&e));
    CU_TRY(c->fp.d_trav.ensure(nword));
    CU_TRY(c->fp.d_front.ensure(2 * nword));
    CU_TRY(c->fp.d_flags.ensure(FP_FLAG_RING + 1));
    CU_TRY(c->fp.h_flag.ensure(2));
    CU_TRY(cudaEventRecord(c->fp.ev[0], st));
    if (int r = frontend_feasibility_run(c, nullptr, c->fp.d_trav.p, st)) return r;
    CU_TRY(cudaEventRecord(c->fp.ev[1], st));
    const PathArgs P = path_args(c, s, d_g);
    CU_TRY(cudaMemsetAsync(c->fp.d_front.p, 0, sizeof(uint32_t) * 2 * nword, st));
    CU_TRY(cudaMemsetAsync(c->fp.d_flags.p, 0, sizeof(unsigned) * (FP_FLAG_RING + 1), st));
    const long long sms = c->sm_count;
    k_fp_init<<<(unsigned)std::min<long long>(((long long)nvox + 255) / 256, sms * 32), 256, 0, st>>>(P);
    c->stats.kernel_launches++;
    const unsigned blocks = (unsigned)std::min<long long>(((long long)nword + 255) / 256, sms * 16);
    for (int r = 0;;) {
        for (int k = 0; k < FP_ROUNDS_PER_CHECK; k++, r++) k_fp_relax<<<blocks, 256, 0, st>>>(P, r);
        c->stats.kernel_launches += FP_ROUNDS_PER_CHECK;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(c->fp.h_flag.p, P.flags + r % FP_FLAG_RING, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
        if (!c->fp.h_flag.p[0]) break;
    }
    CU_TRY(cudaEventRecord(c->fp.ev[2], st));
    CU_TRY(cudaMemcpyAsync(c->fp.h_flag.p + 1, P.rounds, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    isdf_frontpath_info &I = c->fp.info;
    I = {};
    I.rounds = (int32_t)c->fp.h_flag.p[1];
    I.field_bytes = (int64_t)(nvox * sizeof(double));
    float ms = 0;
    cudaEventElapsedTime(&ms, c->fp.ev[0], c->fp.ev[1]); I.traversability_ms = ms;
    cudaEventElapsedTime(&ms, c->fp.ev[1], c->fp.ev[2]); I.field_ms = ms;
    return 0;
}

// field from start, then the B paths into c->fp.d_xyz / d_rp / d_cost / d_found; off (B + 1) is filled as soon as the lengths are known,
// also when they exceed cap
static int path_run(isdf_ctx *c, const double *start, int B, const double *goals, int cap, std::vector<int> &off, cudaStream_t st) {
    const DevGrid &G = c->map.grid;
    int s[3];
    if (int r = path_voxel(G, start, s, "start")) return r;
    std::vector<int> tgt((size_t)3 * B);
    for (int b = 0; b < B; b++)
        if (int r = path_voxel(G, goals + 3 * (size_t)b, &tgt[3 * (size_t)b], "a goal")) return r;
    CU_TRY(c->fp.d_g.ensure((size_t)G.X * G.Y * G.Z));
    if (int r = path_field(c, s, c->fp.d_g.p, st)) return r;
    PathArgs P = path_args(c, s, c->fp.d_g.p);
    CU_TRY(c->fp.d_tgt.upload(tgt.data(), tgt.size(), st));
    CU_TRY(c->fp.d_len.ensure(B)); CU_TRY(c->fp.d_off.ensure((size_t)B + 1));
    CU_TRY(c->fp.d_cost.ensure(B)); CU_TRY(c->fp.d_found.ensure(B));
    P.nt = B; P.tgt = c->fp.d_tgt.p; P.len = c->fp.d_len.p; P.off = c->fp.d_off.p; P.cost = c->fp.d_cost.p; P.found = c->fp.d_found.p;
    const unsigned wblocks = (unsigned)(((long long)B * 32 + 127) / 128);
    k_fp_walk<<<wblocks, 128, 0, st>>>(P, 0);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    std::vector<int> len(B);
    CU_TRY(cudaMemcpyAsync(len.data(), c->fp.d_len.p, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    off.assign((size_t)B + 1, 0);
    long long total = 0;
    for (int b = 0; b < B; b++) {
        total += len[b];
        if (total > INT32_MAX) return fail(ISDF_ERR_INVALID, "the paths hold more than 2^31 - 1 nodes");
        off[b + 1] = (int)total;
    }
    if (total > cap) return fail(ISDF_ERR_INVALID, "cap is smaller than the total path length (reported in n / offsets[B])");
    CU_TRY(c->fp.d_off.upload(off.data(), off.size(), st));
    CU_TRY(c->fp.d_nodes.ensure((size_t)3 * total)); CU_TRY(c->fp.d_colliding.ensure((size_t)4 * total));
    CU_TRY(c->fp.d_xyz.ensure((size_t)3 * total)); CU_TRY(c->fp.d_rp.ensure((size_t)2 * total));
    P.nodes = c->fp.d_nodes.p; P.xyz = c->fp.d_xyz.p; P.rp = c->fp.d_rp.p; P.colliding = c->fp.d_colliding.p;
    k_fp_walk<<<wblocks, 128, 0, st>>>(P, 1);
    FrontArgs A = front_args(c);
    A.nq = (int)total; A.q_ind = c->fp.d_nodes.p; A.out = c->fp.d_colliding.p;
    const size_t smem = sizeof(uint32_t) * 4 * (size_t)A.ks * A.ks * A.ks;
    CU_TRY(cudaFuncSetAttribute(k_fp_node_masks, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_fp_node_masks<<<(unsigned)((total + 255) / 256), 256, smem, st>>>(A);
    k_fp_attitudes<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(A, P);
    c->stats.kernel_launches += 3;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaEventRecord(c->fp.ev[3], st));
    CU_TRY(cudaStreamSynchronize(st));
    float ms = 0;
    cudaEventElapsedTime(&ms, c->fp.ev[2], c->fp.ev[3]); c->fp.info.paths_ms = ms;
    return 0;
}

extern "C" int isdf_frontend_path_batch(isdf_ctx *c, const double *start, int B, const double *goals, const isdf_frontpath_params *prm, int cap,
                                        double *path_xyz, double *path_rp, int32_t *offsets, double *costs, uint8_t *found) {
    if (!start || !goals || B < 1 || cap < 0 || (cap > 0 && !path_xyz) || !offsets || !costs || !found) return fail(ISDF_ERR_INVALID, "bad argument");
    if (int r = path_args_check(c, prm)) return r;
    if (set_device(c)) return ISDF_ERR_CUDA;
    std::vector<int> off;
    const int r = path_run(c, start, B, goals, cap, off, c->stream);
    if (!off.empty()) std::memcpy(offsets, off.data(), sizeof(int32_t) * off.size());
    if (r) return r;
    const size_t total = (size_t)off[B];
    CU_TRY(cudaMemcpyAsync(path_xyz, c->fp.d_xyz.p, sizeof(double) * 3 * total, cudaMemcpyDeviceToHost, c->stream));
    if (path_rp) CU_TRY(cudaMemcpyAsync(path_rp, c->fp.d_rp.p, sizeof(double) * 2 * total, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaMemcpyAsync(costs, c->fp.d_cost.p, sizeof(double) * B, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaMemcpyAsync(found, c->fp.d_found.p, B, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    return 0;
}

extern "C" int isdf_frontend_path(isdf_ctx *c, const double *start, const double *goal, const isdf_frontpath_params *prm, int cap,
                                  double *path_xyz, double *path_rp, int32_t *n, double *cost, uint8_t *found) {
    if (!n) return fail(ISDF_ERR_INVALID, "n is NULL");
    int32_t off[2] = {0, 0};
    const int r = isdf_frontend_path_batch(c, start, 1, goal, prm, cap, path_xyz, path_rp, off, cost, found);
    *n = off[1];
    return r;
}

extern "C" int isdf_frontend_path_batch_device(isdf_ctx *c, const double *start, int B, const double *d_goals, const isdf_frontpath_params *prm,
                                               int cap, double *d_path_xyz, double *d_path_rp, int32_t *d_offsets, double *d_costs,
                                               uint8_t *d_found, void *cuda_stream) {
    if (!start || !d_goals || B < 1 || cap < 0 || (cap > 0 && !d_path_xyz) || !d_offsets || !d_costs || !d_found) return fail(ISDF_ERR_INVALID, "bad argument");
    if (int r = path_args_check(c, prm)) return r;
    if (set_device(c)) return ISDF_ERR_CUDA;
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    std::vector<double> goals((size_t)3 * B);
    CU_TRY(cudaMemcpyAsync(goals.data(), d_goals, sizeof(double) * goals.size(), cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    std::vector<int> off;
    const int r = path_run(c, start, B, goals.data(), cap, off, st);
    if (!off.empty()) {
        CU_TRY(cudaMemcpyAsync(d_offsets, off.data(), sizeof(int32_t) * off.size(), cudaMemcpyHostToDevice, st));
        CU_TRY(cudaStreamSynchronize(st));   // off is a host temporary
    }
    if (r) return r;
    const size_t total = (size_t)off[B];
    CU_TRY(cudaMemcpyAsync(d_path_xyz, c->fp.d_xyz.p, sizeof(double) * 3 * total, cudaMemcpyDeviceToDevice, st));
    if (d_path_rp) CU_TRY(cudaMemcpyAsync(d_path_rp, c->fp.d_rp.p, sizeof(double) * 2 * total, cudaMemcpyDeviceToDevice, st));
    CU_TRY(cudaMemcpyAsync(d_costs, c->fp.d_cost.p, sizeof(double) * B, cudaMemcpyDeviceToDevice, st));
    CU_TRY(cudaMemcpyAsync(d_found, c->fp.d_found.p, B, cudaMemcpyDeviceToDevice, st));
    CU_TRY(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int isdf_frontend_path_field_device(isdf_ctx *c, const double *start, const isdf_frontpath_params *prm, double *d_g, void *cuda_stream) {
    if (!start || !d_g) return fail(ISDF_ERR_INVALID, "bad argument");
    if (int r = path_args_check(c, prm)) return r;
    if (set_device(c)) return ISDF_ERR_CUDA;
    int s[3];
    if (int r = path_voxel(c->map.grid, start, s, "start")) return r;
    return path_field(c, s, reinterpret_cast<unsigned long long *>(d_g), (cudaStream_t)cuda_stream);
}

extern "C" int isdf_frontend_path_info(isdf_ctx *c, isdf_frontpath_info *out) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    *out = c->fp.info;
    return 0;
}

// the traversability bits of the last path or field call (X*Y*ceil(Z/32) words of the map it ran on, grid.bits' layout)
extern "C" int isdf_dbg_frontpath_traversable(isdf_ctx *c, uint32_t *out, long long n) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->map.have_map || n != (long long)c->map.grid.X * c->map.grid.Y * c->map.grid.Zw || (size_t)n > c->fp.d_trav.n)
        return fail(ISDF_ERR_STATE, "no traversability grid of the current map's size");
    if (set_device(c)) return ISDF_ERR_CUDA;
    CU_TRY(cudaMemcpy(out, c->fp.d_trav.p, sizeof(uint32_t) * (size_t)n, cudaMemcpyDeviceToHost));
    return 0;
}

// ---- swept volume -------------------------------------------------------------------------------------------
extern "C" int isdf_set_points(isdf_ctx *c, const double *pts, int P) {
    if (!c || P < 0 || (P > 0 && !pts)) return fail(ISDF_ERR_INVALID, "bad argument");
    if (set_device(c)) return ISDF_ERR_CUDA;
    CU_TRY(c->sv.set_points(pts, P, c->stream));
    return 0;
}

extern "C" int isdf_set_points_batch(isdf_ctx *c, int B, const int32_t *offsets, const double *pts) {
    if (!c || B < 0 || (B > 0 && !offsets)) return fail(ISDF_ERR_INVALID, "bad argument");
    if (set_device(c)) return ISDF_ERR_CUDA;
    if (B == 0) { c->sv.B = 0; return 0; }
    if (offsets[0] != 0) return fail(ISDF_ERR_INVALID, "offsets[0] must be 0");
    for (int b = 0; b < B; b++) if (offsets[b + 1] < offsets[b]) return fail(ISDF_ERR_INVALID, "offsets must be non-decreasing");
    if (offsets[B] > 0 && !pts) return fail(ISDF_ERR_INVALID, "pts is NULL");
    if (offsets[B] == 0) return fail(ISDF_ERR_INVALID, "no points at all: use B = 0 to switch the batched swept-volume term off");
    CU_TRY(c->sv.set_points_batch(B, offsets, pts, c->stream));
    return 0;
}

// count_out as launch_discrete's
static int swept_common(isdf_ctx *c, int N, const double *d_T, const double *d_C, double *d_out, double *count_out, cudaStream_t st,
                        const double *g_t, const double *g_s, const double *g_g) {
    if (c->sv.P <= 0) return fail(ISDF_ERR_STATE, "obstacle points not set (isdf_set_points)");
    if (c->mesh.shape.kind == ISDF_SHAPE_MESH && c->mesh.shape.mesh.sign_mode == MESH_SIGN_WINDING)
        return fail(ISDF_ERR_UNSUPPORTED, "the swept-volume search prunes with distance brackets that need a true distance function: winding-sign meshes "
                                          "(open meshes / soups, ISDF_MESH_SIGN_WINDING) are supported by the discrete path and isdf_shape_query only");
    int launches = 0;
    cudaError_t e = c->sv.launch(c->dcfg, c->mesh.shape, N, d_T, d_C, d_out, count_out, c->rank, c->world, st, g_t, g_s, g_g, &launches);
    c->stats.kernel_launches += launches;
    c->stats.evals_swept++;
    if (e != cudaSuccess) return fail(e == cudaErrorInvalidValue ? ISDF_ERR_INVALID : ISDF_ERR_CUDA, std::string("swept: ") + cudaGetErrorString(e));
    if (fused_exchange(c)) {
        if (int r = peer_fuse_check(c, N)) return r;
        return peer_allreduce_launch(c, d_out, 19 * N + 1, st);
    }
    return 0;
}

extern "C" int isdf_eval_swept_device(isdf_ctx *c, int N, const double *d_T, const double *d_coeffs, double *d_out, void *cuda_stream) {
    int r = check_eval_state(c, N, false);
    if (r) return r;
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    if (!d_T || !d_coeffs || !d_out) return fail(ISDF_ERR_INVALID, "NULL device pointer");
    if (set_device(c)) return ISDF_ERR_CUDA;
    return swept_common(c, N, d_T, d_coeffs, d_out, nullptr, (cudaStream_t)cuda_stream, nullptr, nullptr, nullptr);
}

// g_t, g_s, g_g: isdf_eval_swept_given's t*, sdf and gradients (nullptr: search them). The caller poisons *cost on failure.
static int eval_swept_host(isdf_ctx *c, int N, const double *T, const double *coeffs, const double *g_t, const double *g_s, const double *g_g,
                           double *cost, double *gradC, double *gradT) {
    if (int r = check_eval_state(c, N, false)) return r;
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    if (!T || !coeffs || !cost || !gradC || !gradT) return fail(ISDF_ERR_INVALID, "NULL argument");
    DevBuf<double> dgt, dgs, dgg;
    return eval_host(c, N, T, coeffs, cost, gradC, gradT, &isdf_stats::last_sdf_evals,
                     [&]() -> int {
                         if (g_t) {
                             CU_TRY(dgt.upload(g_t, c->sv.P, c->stream)); CU_TRY(dgs.upload(g_s, c->sv.P, c->stream));
                             CU_TRY(dgg.upload(g_g, (size_t)3 * c->sv.P, c->stream));
                         }
                         return 0;
                     },
                     [&](const double *d_T, const double *d_C, double *d_out, double *count_out) {
                         return swept_common(c, N, d_T, d_C, d_out, count_out, c->stream, dgt.p, dgs.p, dgg.p);
                     });
}

extern "C" int isdf_eval_swept(isdf_ctx *c, int N, const double *T, const double *coeffs, double *cost, double *gradC, double *gradT) {
    return poison_on_failure([&] { return eval_swept_host(c, N, T, coeffs, nullptr, nullptr, nullptr, cost, gradC, gradT); },
                             [&] { nan_fill(cost, 1); });
}

extern "C" int isdf_eval_swept_given(isdf_ctx *c, int N, const double *T, const double *coeffs, const double *tstar, const double *sdf,
                          const double *grel, double *cost, double *gradC, double *gradT) {
    return poison_on_failure([&]() -> int {
        if (!tstar || !sdf || !grel) return fail(ISDF_ERR_INVALID, "NULL argument");
        return eval_swept_host(c, N, T, coeffs, tstar, sdf, grel, cost, gradC, gradT);
    }, [&] { nan_fill(cost, 1); });
}

extern "C" int isdf_get_swept_results(isdf_ctx *c, double *tstar, double *sdf, double *grel) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (c->sv.P <= 0) return fail(ISDF_ERR_STATE, "obstacle points not set");
    if (set_device(c)) return ISDF_ERR_CUDA;
    const size_t P = c->sv.P;
    if (tstar) CU_TRY(cudaMemcpy(tstar, c->sv.d_tstar.p, sizeof(double) * P, cudaMemcpyDeviceToHost));
    if (sdf) CU_TRY(cudaMemcpy(sdf, c->sv.d_sdf.p, sizeof(double) * P, cudaMemcpyDeviceToHost));
    if (grel) CU_TRY(cudaMemcpy(grel, c->sv.d_grel.p, sizeof(double) * 3 * P, cudaMemcpyDeviceToHost));
    return 0;
}


// ---- internal diagnostics (not part of include/isdf.h) ------------------------------------------------------------
// scheduling diagnostics: natural_order != 0 -> every launch in natural sample order, nothing split (the state of a context's FIRST
// evaluation); warp_slots > 0 -> build the work items as if the device had that many resident warps (huge values shrink the
// balanced share per warp and force every non-trivial sample to be split, so tests can compare split parts against the oracle on one
// GPU); 0 restores the device's own figure.
extern "C" int isdf_dbg_schedule(isdf_ctx *c, int natural_order, int warp_slots) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    c->disc.no_items = natural_order != 0; c->disc.warp_slots_override = warp_slots > 0 ? warp_slots : 0; c->disc.order_for = -1;
    return 0;
}
// window lists (k_discrete_prologue): budget >= 0 sets the list capacity of the following mesh evaluations in codes per sample of
// the trajectory, i.e. budget x world per local sample (0: no lists, every sample's window is enumerated by the scan kernel);
// budget < 0 keeps it. Of the last mesh evaluation with
// collision: stats (6 entries, optional) = {runs, codes written, overflowed runs, local samples M, code capacity, codes requested};
// pose (M x 8), desc (M x 2: list offset or -1, voxel count) and codes (min(requested, capacity) entries) are optional copies.
extern "C" int isdf_dbg_window_lists(isdf_ctx *c, int budget, long long *stats, double *pose, int *desc, uint32_t *codes) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (budget >= 0) c->disc.wl_budget = budget;
    if (!stats && !pose && !desc && !codes) return 0;
    if (c->disc.wl_samples == 0) return fail(ISDF_ERR_STATE, "no mesh evaluation with collision yet");
    if (int r = sync_ctx(c)) return r;
    unsigned long long cnt[4];
    CU_TRY(cudaMemcpy(cnt, c->disc.d_counter.p + 1, sizeof(cnt), cudaMemcpyDeviceToHost));
    const size_t M = (size_t)c->disc.wl_samples, ncodes = (size_t)std::min<unsigned long long>(cnt[0], (unsigned long long)c->disc.wl_cap);
    if (stats) {
        stats[0] = (long long)cnt[1]; stats[1] = (long long)cnt[3]; stats[2] = (long long)cnt[2];
        stats[3] = (long long)M; stats[4] = c->disc.wl_cap; stats[5] = (long long)cnt[0];
    }
    if (pose) CU_TRY(cudaMemcpy(pose, c->disc.d_pose.p, sizeof(double) * 8 * M, cudaMemcpyDeviceToHost));
    if (desc) CU_TRY(cudaMemcpy(desc, c->disc.d_wl_desc.p, sizeof(int2) * M, cudaMemcpyDeviceToHost));
    if (codes && ncodes) CU_TRY(cudaMemcpy(codes, c->disc.d_wl_codes.p, sizeof(uint32_t) * ncodes, cudaMemcpyDeviceToHost));
    return 0;
}
// number of work items / split samples of the table built by the last discrete evaluation
extern "C" int isdf_dbg_item_stats(isdf_ctx *c, int *item_count, int *split_parts) {
    if (!c || !item_count || !split_parts || !c->disc.d_item_count.p) return fail(ISDF_ERR_INVALID, "NULL argument or no discrete evaluation yet");
    if (int r = sync_ctx(c, true)) return r;
    int n = 0;
    CU_TRY(cudaMemcpy(&n, c->disc.d_item_count.p, sizeof(int), cudaMemcpyDeviceToHost));
    std::vector<int> it((size_t)3 * std::max(n, 1));
    if (n > 0) CU_TRY(cudaMemcpy(it.data(), c->disc.d_items.p, sizeof(int) * 3 * n, cudaMemcpyDeviceToHost));
    int parts = 0;
    for (int k = 0; k < n; k++) if (it[3 * k + 2] >= 0) parts++;
    *item_count = n; *split_parts = parts;
    return 0;
}
// the work-item table k_build_items built after the last discrete evaluation, with the work values it read. info (8 entries) =
// {local samples M, rank, world, max_split, warp_slots, item_count (0 when no table was built), builder (0 none, 1 cached: work values
// in registers, 2 uncached: re-read from memory), whether the last scan read a table}. items (item_count x 3: local sample, -1 or
// c0 | c1 << 8, split slot or -1; up to cap_items rows) and work (M values d_work[rank + world m]) are optional. Read it before the
// next evaluation: its scan overwrites the work values.
extern "C" int isdf_dbg_item_table(isdf_ctx *c, long long *info, int *items, long long cap_items, unsigned *work) {
    if (!c || !info) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (c->disc.last_M == 0) return fail(ISDF_ERR_STATE, "no discrete evaluation yet");
    if (int r = sync_ctx(c, true)) return r;
    int n = 0;
    if (c->disc.last_builder) CU_TRY(cudaMemcpy(&n, c->disc.d_item_count.p, sizeof(int), cudaMemcpyDeviceToHost));
    const long long M = c->disc.last_M;
    const long long v[8] = {M, c->disc.last_rank, c->disc.last_world, c->disc.last_max_split, c->disc.last_warp_slots, n, c->disc.last_builder,
                            c->disc.last_have_items ? 1 : 0};
    std::memcpy(info, v, sizeof(v));
    const long long rows = std::min<long long>(n, std::max(cap_items, 0ll));
    if (items && rows > 0) CU_TRY(cudaMemcpy(items, c->disc.d_items.p, sizeof(int) * 3 * rows, cudaMemcpyDeviceToHost));
    if (work) {
        const size_t S = (size_t)(c->disc.last_rank + c->disc.last_world * (M - 1) + 1);
        std::vector<unsigned> all(S);
        CU_TRY(cudaMemcpy(all.data(), c->disc.d_work.p, sizeof(unsigned) * S, cudaMemcpyDeviceToHost));
        for (long long m = 0; m < M; m++) work[m] = all[(size_t)(c->disc.last_rank + c->disc.last_world * m)];
    }
    return 0;
}
// the device flatness map and its adjoint as compiled into the epilogue kernel: vaj n x 9 (vel, acc, jer), grads n x 10
// (quat_grad 4, omg_grad 3, vel_grad 3) -> out n x 16 (quat 4, omg 3, total grads wrt vel, acc, jer)
extern "C" int isdf_dbg_flatness(isdf_ctx *c, int n, const double *vaj, const double *grads, double *out) {
    if (!c || n < 1 || !vaj || !grads || !out) return fail(ISDF_ERR_INVALID, "bad argument");
    if (set_device(c)) return ISDF_ERR_CUDA;
    DevBuf<double> dv, dg, dout;
    CU_TRY(dv.upload(vaj, (size_t)9 * n, c->stream));
    CU_TRY(dg.upload(grads, (size_t)10 * n, c->stream));
    CU_TRY(dout.ensure((size_t)16 * n));
    CU_TRY(discrete_launch_dbg_flatness(c->dcfg.fp, n, dv.p, dg.p, dout.p, c->stream));
    CU_TRY(cudaMemcpyAsync(out, dout.p, sizeof(double) * 16 * n, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    return 0;
}
// read-only view of the current mesh's body-frame cell grid, so tests can tell which search branch answers a query:
// geom = {glo[3], gcell, ghd, gpad, sign_radius, list_reach}, gdim[3]; cell_dist / cell_cnt (gdim[0]*gdim[1]*gdim[2] entries, z fastest)
// are optional — call with NULL first to size them. cell_cnt is 0 for every cell without a candidate list (all of them when no
// list was built).
extern "C" int isdf_dbg_mesh_grid(isdf_ctx *c, double *geom, int32_t *gdim, float *cell_dist, uint16_t *cell_cnt) {
    if (!c || !geom || !gdim) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->mesh.have_shape || c->mesh.shape.kind != ISDF_SHAPE_MESH) return fail(ISDF_ERR_STATE, "no mesh shape set");
    const DevMesh &m = c->mesh.shape.mesh;
    for (int a = 0; a < 3; a++) { geom[a] = m.glo[a]; gdim[a] = m.gdim[a]; }
    geom[3] = m.gcell; geom[4] = m.ghd; geom[5] = m.gpad; geom[6] = m.sign_radius; geom[7] = c->mesh.list_reach;
    const size_t ncell = (size_t)m.gdim[0] * m.gdim[1] * m.gdim[2];
    if (int r = sync_ctx(c)) return r;
    if (cell_dist) CU_TRY(cudaMemcpy(cell_dist, c->mesh.d_cell_dist.p, sizeof(float) * ncell, cudaMemcpyDeviceToHost));
    if (cell_cnt) {
        if (!m.cell_cnt) std::memset(cell_cnt, 0, sizeof(uint16_t) * ncell);
        else CU_TRY(cudaMemcpy(cell_cnt, m.cell_cnt, sizeof(uint16_t) * ncell, cudaMemcpyDeviceToHost));
    }
    return 0;
}
// the current mesh's candidate lists, so tests can check their order and bounds: sizes = {candidates, triangles}; cell_off (one per
// cell, as isdf_dbg_mesh_grid), cand / cand_lb (sizes[0] each) and tris (the leaf-order triangle records, 16 doubles each) are
// optional — call with NULL first to size them.
extern "C" int isdf_dbg_mesh_lists(isdf_ctx *c, long long *sizes, uint32_t *cell_off, uint32_t *cand, float *cand_lb, double *tris) {
    if (!c || !sizes) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->mesh.have_shape || c->mesh.shape.kind != ISDF_SHAPE_MESH) return fail(ISDF_ERR_STATE, "no mesh shape set");
    const DevMesh &m = c->mesh.shape.mesh;
    const size_t ncell = (size_t)m.gdim[0] * m.gdim[1] * m.gdim[2];
    if (int r = sync_ctx(c)) return r;
    size_t total = 0;
    if (m.cand) {   // the last cell's offset + count
        uint32_t off_last = 0; uint16_t cnt_last = 0;
        CU_TRY(cudaMemcpy(&off_last, m.cell_off + ncell - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost));
        CU_TRY(cudaMemcpy(&cnt_last, m.cell_cnt + ncell - 1, sizeof(uint16_t), cudaMemcpyDeviceToHost));
        total = (size_t)off_last + cnt_last;
    }
    sizes[0] = (long long)total; sizes[1] = m.ntris;
    if (cell_off && m.cand) CU_TRY(cudaMemcpy(cell_off, m.cell_off, sizeof(uint32_t) * ncell, cudaMemcpyDeviceToHost));
    if (cand && total) CU_TRY(cudaMemcpy(cand, m.cand, sizeof(uint32_t) * total, cudaMemcpyDeviceToHost));
    if (cand_lb && total) CU_TRY(cudaMemcpy(cand_lb, m.cand_lb, sizeof(float) * total, cudaMemcpyDeviceToHost));
    if (tris) CU_TRY(cudaMemcpy(tris, m.tris, sizeof(double) * TRI_STRIDE * (size_t)m.ntris, cudaMemcpyDeviceToHost));
    return 0;
}
// the swept-volume term of the last batched callback, B x (19 N0 + 1): per problem [cost | gradC 18 N0 | gradT N0], as the callback adds it
extern "C" int isdf_dbg_batch_swept_out(isdf_ctx *c, double *out, long long n) {
    if (!c || !out || n < 0 || (size_t)n > c->batch.d_sv.n) return fail(ISDF_ERR_INVALID, "bad argument or no batched swept-volume term of that size");
    if (int r = sync_ctx(c)) return r;
    CU_TRY(cudaMemcpy(out, c->batch.d_sv.p, sizeof(double) * n, cudaMemcpyDeviceToHost));
    return 0;
}
// {candidate pairs (voxel centre inside the H box), exact mesh searches} of the last clearance check
extern "C" int isdf_dbg_clearance_counts(isdf_ctx *c, unsigned long long *out) {
    if (!c || !out || !c->clr.d_counters.p) return fail(ISDF_ERR_INVALID, "NULL argument or no clearance check yet");
    if (int r = sync_ctx(c)) return r;
    CU_TRY(cudaMemcpy(out, c->clr.d_counters.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return 0;
}

// (D_a, D_b) of the certificate's motion bound for caller-given intervals (piece, ta, tb) of a trajectory block (T, coeffs: N pieces);
// out: 2n doubles; *radius (may be NULL): the body radius r the bound used. Needs a supported shape, not a map. Diagnostic; not part
// of include/isdf.h.
extern "C" int isdf_dbg_certify_bound(isdf_ctx *c, int N, const double *T, const double *coeffs, double reach, int n, const int32_t *piece,
                                      const double *ta, const double *tb, double *out, double *radius) {
    if (!c || N < 1 || n < 1 || !T || !coeffs || !piece || !ta || !tb || !out || !(reach > 0.0)) return fail(ISDF_ERR_INVALID, "bad argument");
    for (int k = 0; k < n; k++) if (piece[k] < 0 || piece[k] >= N) return fail(ISDF_ERR_INVALID, "piece out of range");
    double r = 0.0;
    if (int rr = certify_shape(c, &r)) return rr;
    if (radius) *radius = r;
    if (set_device(c)) return ISDF_ERR_CUDA;
    DevBuf<double> d;   // [coeffs 18N | T N | ta n | tb n | out 2n]
    CU_TRY(d.ensure((size_t)19 * N + 4 * (size_t)n));
    const double *dT;
    if (int rr = stage_traj(c, d, N, T, coeffs, &dT)) return rr;
    DevBuf<int> dp;
    CU_TRY(dp.upload(piece, n, c->stream));
    double *dta = d.p + 19 * (size_t)N, *dtb = dta + n, *dout = dtb + n;
    CU_TRY(cudaMemcpyAsync(dta, ta, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(cudaMemcpyAsync(dtb, tb, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
    const CertArgs A = certify_args(c, r, reach, N, dT, d.p);
    CU_TRY(certify_bound_launch(A, n, dp.p, dta, dtb, dout, c->stream));
    c->stats.kernel_launches++;
    CU_TRY(cudaMemcpyAsync(out, dout, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    return 0;
}

// the final leaf intervals of the last certificate call: records {ta, tb, c_a, c_b, D_a, D_b (double); piece (index in the call's block),
// state (1 safe, 0 undecided, -1 dropped) (int32)}, 56 bytes each, in the order they were finished; *n = their number, at most cap copied
extern "C" int isdf_dbg_certify_leaves(isdf_ctx *c, void *out, long long cap, long long *n) {
    if (!c || !n || cap < 0 || (cap > 0 && !out)) return fail(ISDF_ERR_INVALID, "bad argument");
    *n = c->cert.last_leaves;
    const long long k = std::min(cap, c->cert.last_leaves);
    if (k == 0) return 0;
    if (set_device(c)) return ISDF_ERR_CUDA;
    CU_TRY(cudaMemcpy(out, c->cert.d_leaves.p, sizeof(CertLeaf) * (size_t)k, cudaMemcpyDeviceToHost));
    return 0;
}
