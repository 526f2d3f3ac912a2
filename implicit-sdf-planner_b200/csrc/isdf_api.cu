// libisdf_b200.so — C-ABI layer (include/isdf.h) over the sm_90a kernels. No CPU fallback anywhere: every entry
// point either runs CUDA kernels or fails with ISDF_ERR_CUDA / ISDF_ERR_STATE.
#include "../../include/isdf.h"
#include "isdf_types.cuh"
#include "isdf_discrete.cuh"
#include "isdf_swept.cuh"
#include "isdf_minco.cuh"
#include "isdf_frontend.cuh"
#include "isdf_frontpath.cuh"
#include "isdf_frontier.cuh"
#include "isdf_lbfgs.cuh"
#include "isdf_midend.cuh"
#include "isdf_clearance.cuh"
#include "isdf_certify.cuh"
#include "isdf_sweptvol.cuh"
#include "isdf_dynlimits.cuh"
#include "isdf_map.cuh"
#include "isdf_esdf.cuh"
#include "isdf_states.cuh"
#include "isdf_brake.cuh"
#include "isdf_plan.cuh"
#include "isdf_sim.cuh"
#include "isdf_sense.cuh"
#include "isdf_world.cuh"
#include <cub/device/device_scan.cuh>
#include <queue>
#include "isdf_host_mesh.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <functional>
#include <string>
#include <vector>
#include <limits>
#include <unordered_map>

using namespace isdf;

__global__ void k_mesh_cells(const __grid_constant__ DevMesh M, int nx, int ny, int nz, double lx, double ly, double lz, double cell,
                             float *dist, uint32_t *seed);

__global__ void k_mesh_cell_lists(const __grid_constant__ DevMesh M, long long ncell, double hd, double list_reach, double disc_reach, uint16_t *cnt,
                                  const uint32_t *off, uint32_t *cand, float *cand_lb);
__global__ void k_mesh_cell_pack(long long ncell, const float *dist, const uint32_t *seed, const uint32_t *off, const uint16_t *cnt, uint4 *rec);
__global__ void k_mesh_disc_lists(const __grid_constant__ DevMesh M, long long ncell, int k, double margin, uint16_t *dcnt, const uint32_t *doff,
                                  uint32_t *dcand, float *dlb);

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

// an offset array off[0..B] (host): off[0] == 0, then non-decreasing (allow_empty) or increasing
static int offsets_check(const int32_t *off, int B, const char *name, bool allow_empty) {
    if (off[0] != 0) return fail(ISDF_ERR_INVALID, std::string(name) + "[0] must be 0");
    for (int b = 0; b < B; b++) {
        if (allow_empty ? off[b + 1] < off[b] : off[b + 1] <= off[b])
            return fail(ISDF_ERR_INVALID, allow_empty ? std::string(name) + " must be non-decreasing"
                                                      : std::string("every range of ") + name + " needs at least one entry (" + name + " must increase)");
    }
    return 0;
}

// The problems of a batched call and where their pieces lie. Uniform (the entry points that take B, N0): problem b owns pieces
// [b N0, b N0 + N0) and no offsets exist. Ragged (the *_ragged entry points, include/isdf.h): problem b owns pieces [piece_off[b], piece_off[b+1])
// and decision-vector rows [4 piece_off[b] - 3 b, 4 piece_off[b+1] - 3 (b+1)); both offset arrays live on the device.
struct Layout {
    int B = 0, N = 0;                                  // problems; the most pieces of one problem (sizes shared memory and grids)
    size_t P = 0, X = 0;                               // pieces; decision-vector rows
    const int *d_off = nullptr, *d_xoff = nullptr;     // B + 1 piece and B + 1 decision-vector offsets on the device (null: uniform)
};
static Layout uniform_layout(int B, int N0) {
    Layout L;
    L.B = B; L.N = N0; L.P = (size_t)B * N0; L.X = (size_t)B * (4 * (size_t)N0 - 3);
    return L;
}
// a ragged batch's offsets (host): the sizes into *L; the device offsets come from ragged_upload
static int ragged_check(int B, const int32_t *piece_off, Layout *L) {
    if (B < 1) return fail(ISDF_ERR_INVALID, "B < 1");
    if (!piece_off) return fail(ISDF_ERR_INVALID, "piece_off is NULL");
    if (int r = offsets_check(piece_off, B, "piece_off", false)) return r;
    int N = 0;
    for (int b = 0; b < B; b++) N = std::max(N, piece_off[b + 1] - piece_off[b]);
    const size_t P = (size_t)piece_off[B], X = 4 * P - 3 * (size_t)B;
    if (X > 0x7fffffffull) return fail(ISDF_ERR_INVALID, "4*P - 3*B overflows");
    L->B = B; L->N = N; L->P = P; L->X = X;
    return 0;
}
// the device offsets of a checked ragged batch, staged in buf on st: [piece offsets | decision-vector offsets]
static int ragged_upload(DevBuf<int> &buf, const int32_t *piece_off, cudaStream_t st, Layout *L) {
    const int B = L->B;
    std::vector<int> h(2 * (size_t)B + 2);
    for (int b = 0; b <= B; b++) { h[b] = piece_off[b]; h[(size_t)B + 1 + b] = 4 * piece_off[b] - 3 * b; }
    CU_TRY(buf.upload(h.data(), h.size(), st));
    CU_TRY(cudaStreamSynchronize(st));
    L->d_off = buf.p; L->d_xoff = buf.p + B + 1;
    return 0;
}

// The MINCO forward / adjoint workspace (isdf_minco.cuh) of one batched optimiser: the problems of a Layout.
struct MincoWork {
    DevBuf<double> d_T, d_C, d_lu, d_energy, d_gC, d_gT, d_out;
    int ensure(const Layout &L) {
        if (int r = minco_fits(L.N)) return r;
        const size_t BN = L.P, smem = minco_smem_bytes(L.N);
        CU_TRY(d_T.ensure(BN)); CU_TRY(d_C.ensure(18 * BN)); CU_TRY(d_lu.ensure(78 * BN)); CU_TRY(d_energy.ensure(L.B));
        CU_TRY(d_gC.ensure(18 * BN)); CU_TRY(d_gT.ensure(BN)); CU_TRY(d_out.ensure(19 * BN + 1));
        CU_TRY(cudaFuncSetAttribute(k_minco_forward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CU_TRY(cudaFuncSetAttribute(k_minco_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        return 0;
    }
    // the workspace's part of the arguments; the terms (swept volume, discrete output, cost and gradient) are the caller's
    MincoArgs args(const Layout &L, const double *head, const double *tail, int bc_stride, double rho, const double *x) {
        MincoArgs M = {};
        M.B = L.B; M.N = L.N; M.P = (int)L.P; M.poff = L.d_off; M.x = x; M.head = head; M.tail = tail; M.bc_stride = bc_stride; M.rho = rho;
        M.T = d_T.p; M.C = d_C.p; M.lu = d_lu.p; M.energy = d_energy.p; M.gC_e = d_gC.p; M.gT_e = d_gT.p;
        return M;
    }
};

// The buffers of a certificate's interval-refinement rounds (isdf_refine.cuh): piece start times, the two interval lists of the round
// loop and the round counters.
struct RefineBufs {
    DevBuf<double> d_toff; DevBuf<CertInterval> d_iv[2]; DevBuf<int> d_tot; PinnedBuf<int> h_tot;
    // room for N pieces and I0 initial intervals, and A's pointers into it
    int ensure(RefineArgs &A, int N, size_t I0) {
        CU_TRY(d_toff.ensure(N)); CU_TRY(d_tot.ensure(2)); CU_TRY(h_tot.ensure(1)); CU_TRY(d_iv[0].ensure(I0));
        A.toff = d_toff.p; A.tot = d_tot.p; A.cur = d_iv[0].p;
        return 0;
    }
};

struct GatherBox;   // the index boxes of one waypoint of the obstacle gather (defined with the gather kernels)

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
    size_t smem_optin = 227 * 1024;    // the most dynamic shared memory one CTA can opt into (cudaDevAttrMaxSharedMemoryPerBlockOptin)
    int clr_blocks = 1;                // resident CTAs per SM of the clearance scan kernel
    isdf_stats stats = {};
    struct {
        bool have_map = false;
        DevGrid grid = {};
        DevBuf<uint32_t> d_bits;
        long long points_used = 0, points_skipped = 0;   // isdf_set_map_cloud*; 0 for dense maps
    } map;
    struct {   // known space (isdf_observe.cuh): the known bits in the map's layout (allocated on first use; have = false: nothing known), the
               // blocked grid the clearance family reads under ISDF_UNKNOWN_OCCUPIED (rebuilt when a map, fuse, observe or mark call made it stale)
        bool have = false, blocked_ok = false;
        int policy = ISDF_UNKNOWN_FREE;
        DevBuf<uint32_t> d_known, d_blocked;
        DevGrid blocked = {};
    } known;
    struct {   // the map's distance field (isdf_esdf.cuh): squared voxel distances, ESDF_NONE where no site exists; given up with the map
        bool have = false;
        DevBuf<uint32_t> d_pos, d_neg;
    } esdf;
    struct {   // the robot shape; the buffers hold a mesh's device view
        bool have_shape = false;
        DevShape shape = {};
        DevBuf<BvhNode> d_nodes; DevBuf<WideNode> d_wnodes; DevBuf<double> d_tris, d_pn, d_obb; DevBuf<float> d_cell_dist; DevBuf<uint32_t> d_cell_seed, d_cell_off, d_cand; DevBuf<float> d_cand_lb; DevBuf<uint16_t> d_cell_cnt; DevBuf<uint4> d_cell_rec; DevBuf<WnNode> d_wn;
        double list_reach = 0;  // radius (cell-centre distance) up to which cells got candidate lists (isdf_dbg_mesh_grid)
        // the discrete scan's sub-box filtered lists (k_mesh_disc_lists), built when disc_k > 1; launch_discrete hands them to the scan
        int disc_k = DISC_LIST_K;   // sub-boxes per cell edge (isdf_dbg_disc_k; 1: the scan walks the full lists)
        bool disc_ready = false;
        DevBuf<uint32_t> d_disc_off, d_disc_cand; DevBuf<float> d_disc_lb; DevBuf<uint16_t> d_disc_cnt; DevBuf<uint4> d_disc_rec;
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
    struct {   // the host forms' arguments and results (Staging): one pinned block, one device block, both only grow
        PinnedBuf<char> h;
        DevBuf<char> d;
    } staging;
    struct {   // batched callback (isdf_minco.cuh); B = 0: none evaluated yet
        MincoWork minco;
        DevBuf<double> d_Cpp, d_sv;
        DevBuf<int> d_off;   // a ragged batch's offsets (ragged_upload)
        int B = 0;
        size_t P = 0;        // problems and pieces of the last evaluation
    } batch;
    struct LbfgsBufs {   // device-resident lock-step L-BFGS (isdf_lbfgs.cuh)
        DevBuf<double> d_grad, d_state; DevBuf<int> d_int;
        PinnedBuf<int> h_active;
    } lbfgs;
    struct {   // mid-end (isdf_midend.cuh): buffers of its own, so that no mid-end call touches the back end's batch, swept or L-BFGS state
        MincoWork minco;
        DevBuf<double> d_pc;
        DevBuf<int> d_off;   // a ragged batch's offsets (ragged_upload)
        LbfgsBufs lb;
    } mid;
    SweptState sv;   // swept volume
    struct {   // front end attitude kernels (isdf_frontend.cuh)
        bool ready = false;
        DevBuf<double> d_rot; DevBuf<uint8_t> d_kernels, d_order; DevBuf<uint32_t> d_masks, d_out;
        DevBuf<uint2> d_core, d_urows, d_surv, d_chunks; DevBuf<uint4> d_tab; int nurow = 0, nchunk = 0, ntab = 0; DevBuf<unsigned> d_count; int ncore = 0;
        int xk = 0, yk = 0, ks = 0;
        double max_roll = 0, max_pitch = 0, ang_res = 0, margin = 0;
        int last_launch[3] = {-1, 0, 0};   // the last feasibility run: pipeline (FE_PIPE_*), blocks and threads of its accumulation kernel
    } fe;
    struct {   // front-end path search (isdf_frontpath.cuh): rebuilt from the current map and kernels by every call, so nothing here outlives them
        DevBuf<uint32_t> d_trav, d_front, d_colliding; DevBuf<unsigned long long> d_g; DevBuf<unsigned> d_flags;
        DevBuf<int> d_src, d_tgt, d_tsrc, d_pair, d_len, d_woff, d_off, d_soff, d_scratch, d_nodes; DevBuf<double> d_xyz, d_rp, d_cost;
        DevBuf<uint8_t> d_found;
        PinnedBuf<unsigned> h_flag;
        cudaEvent_t ev[4] = {};
        isdf_frontpath_info info = {};
    } fp;
    struct {   // frontiers (isdf_frontier.cuh): T_o, F, the list, union-find and cluster table of the last frontier call
        DevBuf<uint32_t> d_to, d_f; DevBuf<int> d_cnt, d_woff, d_parent, d_root, d_slot, d_size, d_box, d_croot; DevBuf<long long> d_vox, d_cid;
        DevBuf<unsigned long long> d_ntb, d_sum, d_best; DevBuf<unsigned> d_pick; DevBuf<char> d_tmp; DevBuf<uint8_t> d_cand;
        DevBuf<double> d_vpose; DevBuf<long long> d_gain;   // frontier goals with a view rig: the poses at the frontier voxels, their gains
        DevBuf<isdf_frontier_cluster> d_table; DevBuf<int> d_pair, d_slice, d_tgt; DevBuf<double> d_goals; DevBuf<isdf_frontier_goal> d_out;
        cudaEvent_t ev[6] = {};
    } fr;
    struct {   // trajectory clearance check (isdf_clearance.cuh)
        DevBuf<int> d_cursor;
        DevBuf<unsigned long long> d_counters;   // {candidate pairs, exact mesh searches} of the last check (isdf_dbg_clearance_counts)
    } clr;
    struct {   // continuous certificate (isdf_certify.cuh): the rounds' buffers, samples, leaves, per-trajectory state
        RefineBufs ref;
        DevBuf<double> d_st, d_sc; DevBuf<int> d_sp, d_hit, d_cursor; DevBuf<long long> d_sv;
        DevBuf<CertScratch> d_scr; DevBuf<CertLeaf> d_leaves; DevBuf<CertTraj> d_traj;
        long long last_leaves = 0;   // leaves of the last call (isdf_dbg_certify_leaves)
    } cert;
    struct {   // dynamic-limit certificate (isdf_dynlimits.cuh): the rounds' buffers, samples, per-trajectory state
        RefineBufs ref;
        DevBuf<DynSample> d_smp; DevBuf<int> d_dec; DevBuf<DynTraj> d_traj;
    } dyn;
    struct {   // certified swept volume (isdf_sweptvol.cuh): per-call poses and bounds, brick lists, per-warp interval lists, field and mesh
        DevBuf<double> d_toff, d_pose, d_Dab, d_val, d_low, d_ts, d_V, d_vt;
        DevBuf<uint8_t> d_dec, d_mask; DevBuf<int32_t> d_F;
        DevBuf<long long> d_boff, d_bsum, d_voff, d_foff; DevBuf<int> d_blist, d_cursor;
        DevBuf<SvolIv> d_scratch; DevBuf<unsigned long long> d_counters;
        PinnedBuf<long long> h_n;
        int refine_blocks = 0;   // resident CTAs per SM of the refinement kernel (0: not queried yet)
        cudaEvent_t ev[5] = {};
    } svol;
    struct {   // batched obstacle gather: staged waypoints and offsets, per-row boxes, counts and offsets, the lists
        DevBuf<GatherBox> d_box; DevBuf<int> d_wpoff, d_cnt, d_ptoff; DevBuf<long long> d_offs, d_total; DevBuf<double> d_wp, d_out;
    } gat;
    struct {   // planning step (isdf_plan_pairs): the stages' buffers and the per-plan launch layouts (the host forms stage through Staging)
        DevBuf<double> d_bc, d_wp, d_mx, d_mres, d_bbc, d_bx, d_bf, d_gT, d_gC, d_dur, d_pwp; DevBuf<int> d_mi, d_bi, d_N, d_idx, d_ok, d_bplan, d_gi, d_krows;
        DevBuf<CertSummary> d_csum; DevBuf<DynSummary> d_dsum;
        DevBuf<CopySeg> d_seg; DevBuf<PlanRow> d_row;
        DevBuf<int> d_bad;   // isdf_plan_states_device's head check
        cudaEvent_t ev[2] = {};
        isdf_plan_info info = {};
        long long xfer[4] = {};   // the last planning call's transfers (isdf_dbg_plan_transfers)
    } plan;
    struct {   // isdf_trajectory_shift: per-trajectory piece counts, first piece and its local time, the scan's scratch
        DevBuf<int> d_cnt, d_first; DevBuf<double> d_tau; DevBuf<char> d_tmp;
    } shift;
    struct {   // isdf_trajectory_brake: the candidates' MINCO workspace (its own, so the mid-end's and the back end's stay as they were),
               // their heads, tails, durations and decision vectors, summaries, per-trajectory counts and picks, the scan's scratch
        MincoWork minco;
        DevBuf<double> d_head, d_tail, d_Tin, d_x; DevBuf<CertSummary> d_csum; DevBuf<DynSummary> d_dsum;
        DevBuf<int> d_cnt, d_pick; DevBuf<char> d_tmp;
    } brake;
    struct {   // waypoint selection on the device (isdf_path_waypoints_device): per-path counts and gaps, the scan's scratch
        DevBuf<int32_t> d_cnt, d_gap; DevBuf<char> d_tmp; PinnedBuf<int32_t> h_total;
    } wps;
    // the host <-> device copies made so far at the planning pipeline's copy sites (count_copy): device-to-host bytes outside the rounds'
    // reads, the rounds' 4-byte reads, host-to-device bytes, copies
    long long xfer[4] = {};
    SenseScene sense;   // depth sensing (isdf_sense.cuh): the scene cloud's bricks and the per-call scratch
    WorldScratch gen;   // world generators (isdf_world.cuh): the host program's copy, Perlin keys and selection, the host form's records
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
        for (cudaEvent_t e : fr.ev) if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : svol.ev) if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : plan.ev) if (e) cudaEventDestroy(e);
        if (aux_stream) cudaStreamDestroy(aux_stream);
        if (stream) cudaStreamDestroy(stream);
    }
};

static int set_device(isdf_ctx *c) { CU_TRY(cudaSetDevice(c->device)); return 0; }
// one copy of the planning pipeline, counted in c->xfer: host-to-device or device-to-host, a round's termination read or not. A host
// form's staged results come back as one copy (Staging::download), so XF_COPIES counts that copy once, not once per array
enum { XF_D2H_BYTES, XF_ROUND_READS, XF_H2D_BYTES, XF_COPIES };
static void count_copy(isdf_ctx *c, cudaMemcpyKind k, size_t bytes, bool round_read = false) {
    if (k == cudaMemcpyDeviceToHost) { if (round_read) c->xfer[XF_ROUND_READS]++; else c->xfer[XF_D2H_BYTES] += (long long)bytes; }
    else if (k == cudaMemcpyHostToDevice) c->xfer[XF_H2D_BYTES] += (long long)bytes;
    else return;
    c->xfer[XF_COPIES]++;
}
// the context's device, with the work enqueued on its stream (and, with aux, on its work-item stream) finished
static int sync_ctx(isdf_ctx *c, bool aux = false) {
    if (set_device(c)) return ISDF_ERR_CUDA;
    CU_TRY(cudaStreamSynchronize(c->stream));
    if (aux) CU_TRY(cudaStreamSynchronize(c->aux_stream));
    return 0;
}

// The host arrays of one host-form call, staged through c->staging: each array is a segment of the pinned and the device block, aligned
// to 256 bytes. Declare them with in / inout / out, then upload() packs the inputs and makes ONE host-to-device copy on c->stream and
// sets every declared device pointer; after the device work download() makes ONE device-to-host copy of the outputs, synchronises
// c->stream and unpacks them. An output whose host pointer is NULL gets device room that is not copied back. Device block: [inputs |
// in/out | outputs copied back | room]; the pinned block holds the inputs from its start, then the copied-back range from its start.
class Staging {
    enum Kind { IN, INOUT, OUT, ROOM };
    struct Seg {
        Kind kind;
        size_t bytes, off;
        std::function<void(char *)> set;          // the device pointer
        std::function<void(void *)> fill;         // IN, INOUT: pack into the pinned block
        std::function<void(const void *)> take;   // INOUT, OUT: unpack from the pinned block
    };
    isdf_ctx *c_;
    std::vector<Seg> segs_;
    size_t lo_ = 0, hi_ = 0;   // the copied-back range of the device block
    template <typename T> void add(Kind k, T **d, size_t n, std::function<void(void *)> fill, std::function<void(const void *)> take) {
        segs_.push_back({k, sizeof(T) * n, 0, [d](char *p) { *d = reinterpret_cast<T *>(p); }, std::move(fill), std::move(take)});
    }

public:
    template <typename T> using Same = typename std::remove_cv<T>::type;   // the host pointer's type follows the device pointer's
    explicit Staging(isdf_ctx *c) : c_(c) {}
    template <typename T> void in(const T **d, const Same<T> *h, size_t n) { in(d, n, [h, n](T *p) { std::memcpy(p, h, sizeof(T) * n); }); }
    // an input that fill(T *) writes into the pinned block
    template <typename T, typename F> void in(const T **d, size_t n, F fill) { add(IN, d, n, [fill](void *p) { fill(static_cast<T *>(p)); }, nullptr); }
    template <typename T> void inout(T **d, Same<T> *h, size_t n) {
        add(INOUT, d, n, [h, n](void *p) { std::memcpy(p, h, sizeof(T) * n); }, [h, n](const void *p) { std::memcpy(h, p, sizeof(T) * n); });
    }
    template <typename T> void out(T **d, Same<T> *h, size_t n) {
        if (h) out(d, n, [h, n](const T *p) { std::memcpy(h, p, sizeof(T) * n); });
        else add(ROOM, d, n, nullptr, nullptr);
    }
    // an output that take(const T *) reads from the pinned block, which holds it until the next staged call
    template <typename T, typename F> void out(T **d, size_t n, F take) {
        add(OUT, d, n, nullptr, [take](const void *p) { take(static_cast<const T *>(p)); });
    }
    int upload() {
        size_t off = 0, nin = 0;
        for (Kind k : {IN, INOUT, OUT, ROOM}) {
            if (k == INOUT) lo_ = off;
            for (Seg &s : segs_) if (s.kind == k) { s.off = off; off += (s.bytes + 255) & ~(size_t)255; }
            if (k == INOUT) nin = off;
            if (k == OUT) hi_ = off;
        }
        // an earlier call that failed after enqueuing its copies may still be reading or writing the pinned block
        CU_TRY(cudaStreamSynchronize(c_->stream));
        CU_TRY(c_->staging.h.ensure(std::max(nin, hi_ - lo_))); CU_TRY(c_->staging.d.ensure(off));
        char *h = c_->staging.h.p, *d = c_->staging.d.p;
        for (Seg &s : segs_) {
            s.set(d + s.off);
            if (s.fill && s.bytes) s.fill(h + s.off);
        }
        if (nin) CU_TRY(cudaMemcpyAsync(d, h, nin, cudaMemcpyHostToDevice, c_->stream));
        return 0;
    }
    int download() {
        const char *h = c_->staging.h.p;
        if (hi_ > lo_) CU_TRY(cudaMemcpyAsync(c_->staging.h.p, c_->staging.d.p + lo_, hi_ - lo_, cudaMemcpyDeviceToHost, c_->stream));
        CU_TRY(cudaStreamSynchronize(c_->stream));
        for (const Seg &s : segs_) if (s.take && s.bytes) s.take(h + (s.off - lo_));
        return 0;
    }
    size_t download_bytes() const { return hi_ - lo_; }   // what download() copies, alignment included (after upload())
};

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
            c->smem_optin = prop.sharedMemPerBlockOptin;
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
    c->mesh.have_shape = false; c->fe.ready = false; c->mesh.disc_ready = false;
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
    // descent of the swept-volume path is a CHAIN of them. Cells wholly within the discrete reach take lists up to
    // MESH_LIST_CAP_DISCRETE long (read by the discrete scan only, see mesh_list_cnt), every other cell up to MESH_LIST_CAP.
    {
        const double hd = 0.5 * std::sqrt(3.0) * m.gcell;
        const double list_reach = std::max(c->cfg.safety_hor, 2.0 * c->cfg.safety_hor + 0.1) + 2.0 * m.ghd;
        c->mesh.list_reach = list_reach;
        const unsigned warps_grid = (unsigned)((ncell + 3) / 4);
        // one kind of candidate list: launch(off, cand, lb) counts into cnt (off null), the counts' prefix sums become off, and, when the
        // lists hold 1 to 2^31 - 1 candidates in all, launch fills cand and lb; *total: the candidates, h_cnt: the counts
        auto build_lists = [&](auto launch, DevBuf<uint16_t> &cnt, DevBuf<uint32_t> &off, DevBuf<uint32_t> &cand, DevBuf<float> &lb,
                               std::vector<uint16_t> &h_cnt, size_t *total) -> int {
            CU_TRY(cnt.ensure(ncell)); CU_TRY(off.ensure(ncell));
            launch(nullptr, nullptr, nullptr);
            c->stats.kernel_launches++;
            CU_TRY(cudaGetLastError());
            h_cnt.resize(ncell);
            CU_TRY(cudaMemcpyAsync(h_cnt.data(), cnt.p, sizeof(uint16_t) * ncell, cudaMemcpyDeviceToHost, c->stream));
            CU_TRY(cudaStreamSynchronize(c->stream));
            std::vector<uint32_t> h_off(ncell);
            *total = 0;
            for (size_t i = 0; i < ncell; i++) { h_off[i] = (uint32_t)*total; *total += h_cnt[i]; }
            if (*total == 0 || *total >= (1ull << 31)) return 0;
            CU_TRY(cand.ensure(*total)); CU_TRY(lb.ensure(*total));
            CU_TRY(cudaMemcpyAsync(off.p, h_off.data(), sizeof(uint32_t) * ncell, cudaMemcpyHostToDevice, c->stream));
            launch(off.p, cand.p, lb.p);
            c->stats.kernel_launches++;
            CU_TRY(cudaGetLastError());
            CU_TRY(cudaStreamSynchronize(c->stream));
            return 0;
        };
        std::vector<uint16_t> cnt;
        size_t total = 0;
        if (int r = build_lists([&](const uint32_t *off, uint32_t *cand, float *lb) {
                k_mesh_cell_lists<<<warps_grid, 128, 0, c->stream>>>(m, (long long)ncell, hd, list_reach, c->cfg.safety_hor, c->mesh.d_cell_cnt.p, off, cand, lb);
            }, c->mesh.d_cell_cnt, c->mesh.d_cell_off, c->mesh.d_cand, c->mesh.d_cand_lb, cnt, &total)) return r;
        if (total > 0 && total < (1ull << 31)) {
            m.cell_off = c->mesh.d_cell_off.p; m.cell_cnt = c->mesh.d_cell_cnt.p; m.cand = c->mesh.d_cand.p; m.cand_lb = c->mesh.d_cand_lb.p;
            if (c->mesh.disc_k > 1) {
                // the discrete scan's sub-box filtered lists, counted, then written into their own arrays. margin covers the scan
                // finding p's cell with floor() in a unit with FMA contraction: p may lie outside its cell by a few ulps of its coordinate
                double scale = 1.0;
                for (int a = 0; a < 3; a++) scale = std::max(scale, std::max(std::fabs(m.glo[a]), std::fabs(m.glo[a] + m.gdim[a] * m.gcell)));
                const double margin = 1e-9 * scale + 1e-12;
                // the filtered lists are subsequences of the full ones and keep each one's first entry: 0 < dtotal <= total
                std::vector<uint16_t> dcnt;
                size_t dtotal = 0;
                if (int r = build_lists([&](const uint32_t *off, uint32_t *cand, float *lb) {
                        k_mesh_disc_lists<<<warps_grid, 128, 0, c->stream>>>(m, (long long)ncell, c->mesh.disc_k, margin, c->mesh.d_disc_cnt.p, off, cand, lb);
                    }, c->mesh.d_disc_cnt, c->mesh.d_disc_off, c->mesh.d_disc_cand, c->mesh.d_disc_lb, dcnt, &dtotal)) return r;
                CU_TRY(c->mesh.d_disc_rec.ensure(ncell));
                k_mesh_cell_pack<<<(unsigned)((ncell + 255) / 256), 256, 0, c->stream>>>((long long)ncell, m.cell_dist, m.cell_seed, c->mesh.d_disc_off.p,
                                                                                         c->mesh.d_disc_cnt.p, c->mesh.d_disc_rec.p);
                c->stats.kernel_launches++;
                CU_TRY(cudaGetLastError());
                CU_TRY(cudaStreamSynchronize(c->stream));
                c->mesh.disc_ready = true;
                if (getenv("ISDF_VERBOSE"))
                    fprintf(stderr, "[isdf] discrete-scan lists (%d^3 sub-boxes per cell): %zu candidates (%.1f MB)\n", c->mesh.disc_k, dtotal, dtotal * 8e-6);
            }
        }
        if (getenv("ISDF_VERBOSE")) {
            size_t listed = 0, nlong = 0, long_total = 0;
            for (size_t i = 0; i < ncell; i++) {
                listed += cnt[i] != 0;
                if (cnt[i] > MESH_LIST_CAP) { nlong++; long_total += cnt[i]; }
            }
            fprintf(stderr, "[isdf] mesh cell grid %d x %d x %d (cell %.3f m), %zu cells with a candidate list, %zu candidates (%.1f MB: ids and lower bounds); "
                    "of these %zu lists longer than %d, %zu candidates (%.1f MB)\n", m.gdim[0], m.gdim[1], m.gdim[2], m.gcell, listed, total, total * 8e-6,
                    nlong, MESH_LIST_CAP, long_total, long_total * 8e-6);
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
// store the count (0 for cells that are too far, too deep or whose list would exceed the cell's cap). Pass 2: fill the lists, sorted
// by ascending distance from the cell centre (ties: triangle index), with each distance's lower bound in cand_lb.
// The cap is MESH_LIST_CAP_DISCRETE for a cell the discrete scan answers everywhere (d_c + ghd < disc_reach = safety_hor: the same
// float bound as its cull, so every voxel that lands in the cell is searched, never culled) and MESH_LIST_CAP for every other cell.
// A cell that the hinge boundary sdf = safety_hor crosses keeps the short cap: only part of its volume is ever answered, so a long
// list buys less there for its set-up time and memory.
constexpr int LIST_CAP = MESH_LIST_CAP_DISCRETE;   // the longer of the two caps sizes the shared arrays
__global__ void __launch_bounds__(128) k_mesh_cell_lists(const __grid_constant__ DevMesh M, long long ncell, double hd, double list_reach,
                                                         double disc_reach, uint16_t *cnt, const uint32_t *off, uint32_t *cand, float *cand_lb) {
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
        const int cap = ((double)M.cell_dist[cell] + M.ghd < disc_reach) ? MESH_LIST_CAP_DISCRETE : MESH_LIST_CAP;
        if (lane == 0) cnt[cell] = (n <= cap) ? (uint16_t)n : (uint16_t)0;
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

// The discrete scan's lists (one warp per cell): the rule of k_mesh_cell_lists applied on k^3 sub-boxes of the cell. A sub-box with
// centre y and half diagonal delta (half edge gcell / 2k + margin) keeps triangle T of the cell's list when d(y, T) <= dmin(y) + 2 delta,
// dmin(y) the smallest distance from y over the list. For p in that sub-box and T* nearest to p, d(y, T*) <= d(p, T*) + delta <=
// d(p, T_y) + delta <= dmin(y) + 2 delta: every triangle nearest to some point of the sub-box is kept, exact ties included, and the
// 1e-9 relative + 1e-12 slack covers the FP64 rounding of both distances. The kept triangles are written in list order with their
// cand_lb, and the first entry (nearest to the centre, the scan's upper-bound seed) is always kept. Pass 1 (dcand == nullptr) stores
// the counts; lists of at most DISC_FILTER_MIN candidates are copied whole (they take one pass either way).
__global__ void __launch_bounds__(128) k_mesh_disc_lists(const __grid_constant__ DevMesh M, long long ncell, int k, double margin, uint16_t *dcnt,
                                                         const uint32_t *doff, uint32_t *dcand, float *dlb) {
    constexpr int CH = MESH_LIST_CAP_DISCRETE / 32;   // list candidates per lane
    const int lane = threadIdx.x & 31;
    const long long cell = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (cell >= ncell) return;
    const int n = (int)M.cell_cnt[cell];
    const uint32_t off = M.cell_off[cell];
    uint32_t keep = 0;   // bit j: candidate j * 32 + lane
    if (n <= DISC_FILTER_MIN) {
        if (lane < n) keep = 1u;
    } else {
        const int nz = M.gdim[2], ny = M.gdim[1];
        const int iz = (int)(cell % nz), iy = (int)((cell / nz) % ny), ix = (int)(cell / ((long long)nz * ny));
        const d3 ctr = mk3(M.glo[0] + (ix + 0.5) * M.gcell, M.glo[1] + (iy + 0.5) * M.gcell, M.glo[2] + (iz + 0.5) * M.gcell);
        const double two_delta = 2.0 * sqrt(3.0) * (0.5 * M.gcell / k + margin);
        int ids[CH];
#pragma unroll
        for (int j = 0; j < CH; j++) ids[j] = (j * 32 + lane < n) ? (int)M.cand[off + j * 32 + lane] : -1;
#pragma unroll 1
        for (int s = 0; s < k * k * k; s++) {
            const int sx = s / (k * k), sy = (s / k) % k, sz = s % k;
            const d3 y = mk3(ctr.x + ((sx + 0.5) / k - 0.5) * M.gcell, ctr.y + ((sy + 0.5) / k - 0.5) * M.gcell, ctr.z + ((sz + 0.5) / k - 0.5) * M.gcell);
            double d[CH];
            double mn = 1e300;
#pragma unroll
            for (int j = 0; j < CH; j++) {
                d[j] = 1e300;
                if (j * 32 < n && ids[j] >= 0) {
                    int f;
                    const d3 q = tri_closest_rec(y, M.tris + TRI_STRIDE * (size_t)ids[j], f);
                    const d3 e = y - q;
                    d[j] = sqrt(dot3(e, e));
                    mn = fmin(mn, d[j]);
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            const double lim = (mn + two_delta) * (1.0 + 1e-9) + 1e-12;
#pragma unroll
            for (int j = 0; j < CH; j++)
                if (d[j] <= lim) keep |= 1u << j;
        }
        if (lane == 0) keep |= 1u;
    }
    if (dcand == nullptr) {
        int total = __popc(keep);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
        if (lane == 0) dcnt[cell] = (uint16_t)total;
        return;
    }
    const unsigned lt_mask = (1u << lane) - 1u;
    uint32_t pos = doff[cell];
    for (int j = 0; j * 32 < n; j++) {
        const bool kept = (keep >> j) & 1u;
        const unsigned bal = __ballot_sync(0xffffffffu, kept);
        if (kept) {
            const uint32_t o = pos + __popc(bal & lt_mask);
            dcand[o] = M.cand[off + j * 32 + lane];
            dlb[o] = M.cand_lb[off + j * 32 + lane];
        }
        pos += __popc(bal);
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
    Staging S(c);
    const double *dp;
    double *ds, *dg;
    S.in(&dp, p_rel, (size_t)3 * n);
    S.out(&ds, what != ISDF_QUERY_GRAD ? sdf : nullptr, n); S.out(&dg, what != ISDF_QUERY_SDF ? grad : nullptr, (size_t)3 * n);
    if (int r = S.upload()) return r;
    k_shape_query<<<(n + 127) / 128, 128, 0, c->stream>>>(c->mesh.shape, dp, n, ds, dg, what);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    return S.download();
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

// gives up the map and the distance field built on it (its memory too: it is 8 bytes per voxel)
static void drop_map(isdf_ctx *c) {
    c->map.have_map = false;
    c->known.have = c->known.blocked_ok = false;
    c->esdf.have = false;
    c->esdf.d_pos = {}; c->esdf.d_neg = {};
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
    drop_map(c);   // d_bits.ensure may free the current grid
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
        drop_map(c);
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
    drop_map(c);
    CloudFrame F;
    for (int a = 0; a < 3; a++) { F.bmin[a] = bmin[a]; F.bmax[a] = bmax[a]; }
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
            k_cloud_mark<<<blocks, 256, 0, c->stream>>>(d_pts, n, stride, F, c->map.d_bits.p, nullptr);
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
        drop_map(c);
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

// ---- fusing a cloud into the current map, in its frame (k_cloud_mark with the frame's bounds) ---------------------------------------
// every check that needs no device work: the cloud's (res is the map's) and a map to fuse into
static int fuse_args_check(isdf_ctx *c, const void *pts, int64_t n, int32_t stride) {
    if (int rc = cloud_args_check(c, pts, n, stride, 1.0)) return rc;
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set: fusion adds to the current map's frame (an empty frame is isdf_set_map_u8 of zeros)");
    return 0;
}

// d_pts on the device and ready on stream st; the bits are updated on c->stream. The distance field no longer describes the map afterwards.
static int fuse_cloud_impl(isdf_ctx *c, const char *d_pts, long long n, int stride, isdf_fuse_info *info, cudaStream_t st) {
    const DevGrid &g = c->map.grid;
    CloudFrame F;
    for (int a = 0; a < 3; a++) { F.bmin[a] = g.bmin[a]; F.bmax[a] = g.bmax[a]; }
    F.res = g.res; F.X = g.X; F.Y = g.Y; F.Z = g.Z; F.Zw = g.Zw;
    unsigned long long cnt[4] = {};
    DevBuf<unsigned long long> d_cnt;
    cudaError_t e = d_cnt.ensure(4);
    if (e == cudaSuccess && st != c->stream) e = cudaStreamSynchronize(st);   // the points are ready on st
    if (e == cudaSuccess) e = cudaMemsetAsync(d_cnt.p, 0, sizeof(cnt), c->stream);
    if (e == cudaSuccess) {
        k_cloud_mark<<<cloud_grid_blocks(c, n), 256, 0, c->stream>>>(d_pts, n, stride, F, c->map.d_bits.p, d_cnt.p);
        c->stats.kernel_launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(cnt, d_cnt.p, sizeof(cnt), cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) {
        drop_map(c);
        return fail(ISDF_ERR_CUDA, std::string("isdf_map_fuse_cloud: ") + cudaGetErrorString(e));
    }
    c->esdf.have = false;   // the field described the map before this call
    c->esdf.d_pos = {}; c->esdf.d_neg = {};
    c->known.blocked_ok = false;
    if (info) {
        info->points_used = (int64_t)cnt[FUSE_USED]; info->points_outside = (int64_t)cnt[FUSE_OUTSIDE];
        info->points_skipped = (int64_t)cnt[FUSE_SKIPPED]; info->voxels_added = (int64_t)cnt[FUSE_ADDED];
    }
    return 0;
}

extern "C" int isdf_map_fuse_cloud(isdf_ctx *c, const void *points, int64_t n, int32_t stride_bytes, isdf_fuse_info *info) {
    if (int rc = fuse_args_check(c, points, n, stride_bytes)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    DevBuf<char> d_pts;
    const size_t bytes = (size_t)n * stride_bytes;
    cudaError_t e = d_pts.ensure(bytes);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_pts.p, points, bytes, cudaMemcpyHostToDevice, c->stream);
    if (e != cudaSuccess) return fail(ISDF_ERR_CUDA, std::string("isdf_map_fuse_cloud: ") + cudaGetErrorString(e));
    return fuse_cloud_impl(c, d_pts.p, n, stride_bytes, info, c->stream);
}

extern "C" int isdf_map_fuse_cloud_device(isdf_ctx *c, const void *d_points, int64_t n, int32_t stride_bytes, isdf_fuse_info *info,
                                          void *cuda_stream) {
    if (int rc = fuse_args_check(c, d_points, n, stride_bytes)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    return fuse_cloud_impl(c, (const char *)d_points, n, stride_bytes, info, (cudaStream_t)cuda_stream);
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
// (known: the known bits, all 0 when nothing is known)
template <typename T>
static int get_map_impl(isdf_ctx *c, T *out, int64_t n, bool known = false) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    DevGrid g = c->map.grid;
    const long long rows = (long long)g.X * g.Y;
    if (n != rows * g.Z) return fail(ISDF_ERR_INVALID, "n must be X*Y*Z of the map");
    if (known && !c->known.have) { std::memset(out, 0, sizeof(T) * (size_t)n); return 0; }
    if (known) g.bits = c->known.d_known.p;
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
extern "C" int isdf_get_map_known_u8(isdf_ctx *c, uint8_t *known, int64_t n) { return get_map_impl<uint8_t>(c, known, n, true); }

// ---- known space (isdf_observe.cuh, compiled in isdf_sense_tu.cu) ----
// the known bits, allocated and cleared on st the first time after a map was set
static int known_bits(isdf_ctx *c, cudaStream_t st) {
    if (c->known.have) return 0;
    const DevGrid &g = c->map.grid;
    const size_t nwords = (size_t)g.X * g.Y * g.Zw;
    CU_TRY(c->known.d_known.ensure(nwords));
    CU_TRY(cudaMemsetAsync(c->known.d_known.p, 0, nwords * sizeof(uint32_t), st));
    c->known.have = true;
    return 0;
}

extern "C" int isdf_set_unknown_policy(isdf_ctx *c, int policy) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (policy != ISDF_UNKNOWN_FREE && policy != ISDF_UNKNOWN_OCCUPIED) return fail(ISDF_ERR_INVALID, "unknown policy (ISDF_UNKNOWN_FREE or ISDF_UNKNOWN_OCCUPIED)");
    c->known.policy = policy;
    return 0;
}
extern "C" int isdf_get_unknown_policy(isdf_ctx *c, int *policy) {
    if (!c || !policy) return fail(ISDF_ERR_INVALID, "NULL argument");
    *policy = c->known.policy;
    return 0;
}

extern "C" int isdf_map_mark_known(isdf_ctx *c, int64_t n, const double *boxes) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (n < 0 || (n > 0 && !boxes)) return fail(ISDF_ERR_INVALID, "n < 0, or boxes NULL with n > 0");
    for (int64_t b = 0; b < n; b++)
        for (int a = 0; a < 3; a++) {
            const double lo = boxes[6 * b + a], hi = boxes[6 * b + 3 + a];
            if (!std::isfinite(lo) || !std::isfinite(hi) || !(lo <= hi)) return fail(ISDF_ERR_INVALID, "box " + std::to_string(b) + ": lo and hi must be finite with lo <= hi");
        }
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    if (set_device(c)) return ISDF_ERR_CUDA;
    if (int r = known_bits(c, c->stream)) return r;
    int launches = 0;
    cudaError_t e = cudaSuccess;
    for (int64_t b = 0; b < n && e == cudaSuccess; b++) e = known_mark_box(c->map.grid, c->known.d_known.p, boxes + 6 * b, boxes + 6 * b + 3, c->stream, &launches);
    c->stats.kernel_launches += launches;
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    c->known.blocked_ok = false;
    if (e != cudaSuccess) {
        drop_map(c);
        return fail(ISDF_ERR_CUDA, std::string("isdf_map_mark_known: ") + cudaGetErrorString(e));
    }
    return 0;
}

// ---- distance field of the map (GridMap3D::generateESDF3d, getSDFValue, getSDFValueWithGrad; isdf_esdf.cuh) --------------------
extern "C" int isdf_map_esdf(isdf_ctx *c) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    const DevGrid &g = c->map.grid;
    if (g.X > ESDF_AXIS_MAX || g.Y > ESDF_AXIS_MAX || g.Z > ESDF_AXIS_MAX)
        return fail(ISDF_ERR_UNSUPPORTED, "an axis longer than 46341 voxels: the reference's fillESDF computes q * q in int, which overflows "
                                          "there, so its distance field is undefined");
    if (set_device(c)) return ISDF_ERR_CUDA;
    c->esdf.have = false;   // rebuilt in place: the old field is gone from here on
    auto cuda_fail = [&](cudaError_t e) {
        c->esdf.have = false;
        c->esdf.d_pos = {}; c->esdf.d_neg = {};
        return fail(ISDF_ERR_CUDA, std::string("isdf_map_esdf: ") + cudaGetErrorString(e));
    };
    const long long X = g.X, Y = g.Y, Z = g.Z, nvox = X * Y * Z;
    cudaError_t e = c->esdf.d_pos.ensure((size_t)nvox);
    if (e == cudaSuccess) e = c->esdf.d_neg.ensure((size_t)nvox);
    if (e != cudaSuccess) return cuda_fail(e);
    uint32_t *pos = c->esdf.d_pos.p, *neg = c->esdf.d_neg.p;
    // pass z: one warp per row
    const long long rows = X * Y;
    k_esdf_z<<<(unsigned)std::min<long long>((rows * 32 + 255) / 256, (long long)c->sm_count * 16), 256, 0, c->stream>>>(g.bits, rows, g.Z, g.Zw, pos, neg);
    c->stats.kernel_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_fail(e);
    // passes y and x: at most one thread per line of a field, and one stack of m entries per thread, so the stack never exceeds
    // 8 bytes per voxel (DESIGN §3.15)
    int per_sm = 0;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_esdf_line, 256, 0)) != cudaSuccess) return cuda_fail(e);
    const long long resident = (long long)std::max(per_sm, 1) * c->sm_count * 256;
    EsdfLines P[2];
    P[0] = {{pos, neg}, X * Z, Y * Z, Z, (int)Y, (int)Z};   // pass y: lines (x, z)
    P[1] = {{pos, neg}, Y * Z, Z, Y * Z, (int)X, (int)Z};   // pass x: lines (y, z)
    long long G[2], stack = 0;
    for (int k = 0; k < 2; k++) {
        G[k] = std::min(P[k].nlines, resident);
        stack = std::max(stack, G[k] * P[k].m);
    }
    DevBuf<uint2> d_stack;
    if ((e = d_stack.ensure((size_t)stack)) != cudaSuccess) return cuda_fail(e);
    for (int k = 0; k < 2; k++) {
        k_esdf_line<<<(unsigned)((G[k] + 255) / 256), 256, 0, c->stream>>>(P[k], G[k], d_stack.p);
        c->stats.kernel_launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) return cuda_fail(e);
    }
    if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess) return cuda_fail(e);
    c->esdf.have = true;
    return 0;
}

static int esdf_field_check(int field) {
    if (field != ESDF_POSITIVE && field != ESDF_NEGATIVE && field != ESDF_SIGNED) return fail(ISDF_ERR_INVALID, "unknown ESDF field");
    return 0;
}

extern "C" int isdf_get_esdf_f64(isdf_ctx *c, int field, double *out, int64_t n) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (int rc = esdf_field_check(field)) return rc;
    if (!c->esdf.have) return fail(ISDF_ERR_STATE, "no ESDF: build it with isdf_map_esdf after setting the map");
    const DevGrid &g = c->map.grid;
    const long long total = (long long)g.X * g.Y * g.Z;
    if (n != total) return fail(ISDF_ERR_INVALID, "n must be X*Y*Z of the map");
    if (set_device(c)) return ISDF_ERR_CUDA;
    const long long chunk = 4ll << 20;   // 32 MiB of doubles per chunk
    DevBuf<double> d_out;
    CU_TRY(d_out.ensure((size_t)std::min(total, chunk)));
    for (long long i0 = 0; i0 < total; i0 += chunk) {
        const long long cnt = std::min(chunk, total - i0);
        k_esdf_expand<<<cloud_grid_blocks(c, cnt), 256, 0, c->stream>>>(c->esdf.d_pos.p, c->esdf.d_neg.p, field, g.res, i0, cnt, d_out.p);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(out + i0, d_out.p, cnt * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
    }
    return 0;
}

static int esdf_query_check(isdf_ctx *c, int field, const double *pts, int64_t n, const double *dist) {
    if (!c || !pts || !dist) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (n < 0) return fail(ISDF_ERR_INVALID, "n < 0");
    if (int rc = esdf_field_check(field)) return rc;
    if (!c->esdf.have) return fail(ISDF_ERR_STATE, "no ESDF: build it with isdf_map_esdf after setting the map");
    return 0;
}

static void esdf_query_launch(isdf_ctx *c, int field, const double *d_pts, long long n, double *d_dist, double *d_grad, cudaStream_t st) {
    const DevGrid &g = c->map.grid;
    EsdfView V;
    V.pos = c->esdf.d_pos.p; V.neg = c->esdf.d_neg.p; V.X = g.X; V.Y = g.Y; V.Z = g.Z; V.res = g.res;
    for (int a = 0; a < 3; a++) { V.bmin[a] = g.bmin[a]; V.bmax[a] = g.bmax[a]; }
    k_esdf_query<<<(unsigned)std::min<long long>((n + 255) / 256, (long long)c->sm_count * 16), 256, 0, st>>>(V, field, d_pts, n, d_dist, d_grad);
    c->stats.kernel_launches++;
}

extern "C" int isdf_esdf_query(isdf_ctx *c, int field, const double *pts, int64_t n, double *dist, double *grad) {
    if (int rc = esdf_query_check(c, field, pts, n, dist)) return rc;
    if (n == 0) return 0;
    if (set_device(c)) return ISDF_ERR_CUDA;
    Staging S(c);
    const double *d_pts;
    double *d_dist, *d_grad = nullptr;   // no gradient room: the kernel computes no gradients
    S.in(&d_pts, pts, (size_t)n * 3);
    S.out(&d_dist, dist, (size_t)n);
    if (grad) S.out(&d_grad, grad, (size_t)n * 3);
    if (int r = S.upload()) return r;
    esdf_query_launch(c, field, d_pts, n, d_dist, d_grad, c->stream);
    CU_TRY(cudaGetLastError());
    return S.download();
}

extern "C" int isdf_esdf_query_device(isdf_ctx *c, int field, const double *d_pts, int64_t n, double *d_dist, double *d_grad, void *cuda_stream) {
    if (int rc = esdf_query_check(c, field, d_pts, n, d_dist)) return rc;
    if (n == 0) return 0;
    if (set_device(c)) return ISDF_ERR_CUDA;
    esdf_query_launch(c, field, d_pts, n, d_dist, d_grad, (cudaStream_t)cuda_stream);
    CU_TRY(cudaGetLastError());
    return 0;
}

// ---- executing a trajectory (isdf_states.cuh): states at (trajectory, local time) queries, and the body posed at states ----
static int swept_traj_check(int N, const double *T, const double *coeffs);

static const long long STATES_MAX_Q = std::numeric_limits<int64_t>::max() / (8 * STATE_DOUBLES);   // Q records of 160 bytes stay addressable

static int states_args_check(isdf_ctx *c, int B, const void *piece_off, const void *T, const void *coeffs, int64_t Q, const void *traj,
                             const void *times, const void *out) {
    if (!c || !piece_off || !T || !coeffs || !traj || !times || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (B < 1) return fail(ISDF_ERR_INVALID, "B < 1");
    if (Q < 0 || Q > STATES_MAX_Q) return fail(ISDF_ERR_INVALID, "Q < 0 or Q * 160 bytes beyond int64");
    return 0;
}

static void states_launch(isdf_ctx *c, int B, const int *d_off, const double *d_T, const double *d_C, long long Q, const int *d_traj,
                          const double *d_times, double *d_out, cudaStream_t st) {
    const FlatParams &g = c->dcfg.fp;
    const FlatForwardParams fp = {g.mass, g.grav, g.dh_over_m, c->cfg.vert_drag, g.cp, g.veps};
    const long long blocks = std::min<long long>((Q + STATES_THREADS - 1) / STATES_THREADS, 0x7fffffffll);
    k_traj_states<<<(unsigned)blocks, STATES_THREADS, 0, st>>>(d_off, d_T, d_C, B, Q, d_traj, d_times, fp, d_out);
    c->stats.kernel_launches++;
}

extern "C" int isdf_trajectory_states(isdf_ctx *c, int B, const int32_t *piece_off, const double *T, const double *coeffs, int64_t Q,
                                      const int32_t *traj, const double *times, double *out) {
    if (int rc = states_args_check(c, B, piece_off, T, coeffs, Q, traj, times, out)) return rc;
    if (int rc = offsets_check(piece_off, B, "piece_off", true)) return rc;
    const int P = piece_off[B];
    if (int rc = swept_traj_check(P, T, coeffs)) return rc;
    for (long long q = 0; q < Q; q++) if (traj[q] < 0 || traj[q] >= B) return fail(ISDF_ERR_INVALID, "traj[q] outside [0, B)");
    if (Q == 0) return 0;
    if (set_device(c)) return ISDF_ERR_CUDA;
    Staging S(c);
    const double *d_C, *d_T, *d_times;
    const int *d_off, *d_traj;
    double *d_out;
    S.in(&d_C, coeffs, 18 * (size_t)P); S.in(&d_T, T, (size_t)P); S.in(&d_times, times, (size_t)Q);
    S.in(&d_off, piece_off, (size_t)B + 1); S.in(&d_traj, traj, (size_t)Q);
    S.out(&d_out, out, (size_t)STATE_DOUBLES * Q);
    if (int rc = S.upload()) return rc;
    states_launch(c, B, d_off, d_T, d_C, Q, d_traj, d_times, d_out, c->stream);
    CU_TRY(cudaGetLastError());
    return S.download();
}

extern "C" int isdf_trajectory_states_device(isdf_ctx *c, int B, const int32_t *d_piece_off, const double *d_T, const double *d_coeffs, int64_t Q,
                                             const int32_t *d_traj, const double *d_times, double *d_out, void *cuda_stream) {
    if (int rc = states_args_check(c, B, d_piece_off, d_T, d_coeffs, Q, d_traj, d_times, d_out)) return rc;
    if (Q == 0) return 0;
    if (set_device(c)) return ISDF_ERR_CUDA;
    states_launch(c, B, d_piece_off, d_T, d_coeffs, Q, d_traj, d_times, d_out, (cudaStream_t)cuda_stream);
    CU_TRY(cudaGetLastError());
    return 0;
}

// the rest of B trajectories from t0 (isdf_states.cuh) on stream st: locate and count, scan the counts into out_off, write the pieces
static int shift_launch(isdf_ctx *c, int B, const int *d_off, const double *d_T, const double *d_C, const double *d_t0, int *d_out_off,
                        double *d_out_T, double *d_out_C, cudaStream_t st) {
    auto &z = c->shift;
    CU_TRY(z.d_cnt.ensure(B)); CU_TRY(z.d_first.ensure(B)); CU_TRY(z.d_tau.ensure(B));
    size_t tmp = 0;
    CU_TRY(cub::DeviceScan::InclusiveSum(nullptr, tmp, z.d_cnt.p, d_out_off + 1, B, st));
    CU_TRY(z.d_tmp.ensure(std::max<size_t>(tmp, 1)));
    k_shift_locate<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(B, d_off, d_T, d_t0, z.d_cnt.p, z.d_first.p, z.d_tau.p, d_out_off);
    CU_TRY(cub::DeviceScan::InclusiveSum(z.d_tmp.p, tmp, z.d_cnt.p, d_out_off + 1, B, st));
    k_shift_write<<<(unsigned)(((long long)B * 32 + 127) / 128), 128, 0, st>>>(B, d_off, d_T, d_C, z.d_cnt.p, z.d_first.p, z.d_tau.p, d_out_off,
                                                                               d_out_T, d_out_C);
    c->stats.kernel_launches += 3;
    CU_TRY(cudaGetLastError());
    return 0;
}

extern "C" int isdf_trajectory_shift(isdf_ctx *c, int B, const int32_t *piece_off, const double *T, const double *coeffs, const double *t0,
                                     int32_t *out_piece_off, double *out_T, double *out_coeffs) {
    if (!c || !piece_off || !T || !coeffs || !t0 || !out_piece_off || !out_T || !out_coeffs) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (B < 1) return fail(ISDF_ERR_INVALID, "B < 1");
    if (int rc = offsets_check(piece_off, B, "piece_off", true)) return rc;
    const int P = piece_off[B];
    if (int rc = swept_traj_check(P, T, coeffs)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    Staging S(c);
    const double *d_C, *d_T, *d_t0;
    const int *d_off;
    int *d_out_off;
    double *d_out_T, *d_out_C;
    S.in(&d_C, coeffs, 18 * (size_t)P); S.in(&d_T, T, (size_t)P); S.in(&d_t0, t0, (size_t)B); S.in(&d_off, piece_off, (size_t)B + 1);
    S.out(&d_out_off, out_piece_off, (size_t)B + 1); S.out(&d_out_T, out_T, (size_t)P); S.out(&d_out_C, out_coeffs, 18 * (size_t)P);
    if (int rc = S.upload()) return rc;
    if (int rc = shift_launch(c, B, d_off, d_T, d_C, d_t0, d_out_off, d_out_T, d_out_C, c->stream)) return rc;
    return S.download();
}

extern "C" int isdf_trajectory_shift_device(isdf_ctx *c, int B, const int32_t *d_piece_off, const double *d_T, const double *d_coeffs,
                                            const double *d_t0, int32_t *d_out_piece_off, double *d_out_T, double *d_out_coeffs, void *cuda_stream) {
    if (!c || !d_piece_off || !d_T || !d_coeffs || !d_t0 || !d_out_piece_off || !d_out_T || !d_out_coeffs) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (B < 1) return fail(ISDF_ERR_INVALID, "B < 1");
    if (set_device(c)) return ISDF_ERR_CUDA;
    return shift_launch(c, B, d_piece_off, d_T, d_coeffs, d_t0, d_out_piece_off, d_out_T, d_out_coeffs, (cudaStream_t)cuda_stream);
}

static int pose_args_check(isdf_ctx *c, int64_t Q, const void *states, int P, const void *body, const void *out) {
    if (!c || !states || !body || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (Q < 0 || Q > STATES_MAX_Q) return fail(ISDF_ERR_INVALID, "Q < 0 or Q * 160 bytes beyond int64");
    if (P < 0) return fail(ISDF_ERR_INVALID, "P < 0");
    if (P > 0 && Q > std::numeric_limits<int64_t>::max() / (8 * 3 * (int64_t)P)) return fail(ISDF_ERR_INVALID, "Q * P * 3 doubles beyond int64");
    return 0;
}

static void pose_launch(isdf_ctx *c, long long Q, const double *d_states, int P, const double *d_body, double *d_out, cudaStream_t st) {
    const long long L = 3ll * P;
    const int S = (int)std::max(1ll, std::min<long long>((POSE_TARGET + L - 1) / L, POSE_MAX_STATES));
    const long long blocks = std::min<long long>((Q + S - 1) / S, 0x7fffffffll);
    k_pose_points<<<(unsigned)blocks, POSE_THREADS, 0, st>>>(Q, d_states, P, d_body, S, d_out);
    c->stats.kernel_launches++;
}

extern "C" int isdf_pose_points(isdf_ctx *c, int64_t Q, const double *states, int P, const double *body, double *out) {
    if (int rc = pose_args_check(c, Q, states, P, body, out)) return rc;
    if (Q == 0 || P == 0) return 0;
    if (set_device(c)) return ISDF_ERR_CUDA;
    Staging S(c);
    const double *d_states, *d_body;
    double *d_out;
    S.in(&d_states, states, (size_t)STATE_DOUBLES * Q); S.in(&d_body, body, 3 * (size_t)P);
    S.out(&d_out, out, 3 * (size_t)P * (size_t)Q);
    if (int rc = S.upload()) return rc;
    pose_launch(c, Q, d_states, P, d_body, d_out, c->stream);
    CU_TRY(cudaGetLastError());
    return S.download();
}

extern "C" int isdf_pose_points_device(isdf_ctx *c, int64_t Q, const double *d_states, int P, const double *d_body, double *d_out, void *cuda_stream) {
    if (int rc = pose_args_check(c, Q, d_states, P, d_body, d_out)) return rc;
    if (Q == 0 || P == 0) return 0;
    if (set_device(c)) return ISDF_ERR_CUDA;
    pose_launch(c, Q, d_states, P, d_body, d_out, (cudaStream_t)cuda_stream);
    CU_TRY(cudaGetLastError());
    return 0;
}

// ---- closed loop (isdf_sim.cuh, compiled in isdf_sim_tu.cu) ----
extern "C" int isdf_sim_default_params(isdf_sim_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    std::memset(p, 0, sizeof(*p));
    p->mass = 0.98; p->grav = 9.81; p->J[0] = 2.64e-3; p->J[1] = 2.64e-3; p->J[2] = 4.96e-3;   // Quadrotor::Quadrotor()
    p->kf = 8.98132e-9; p->km = 0.07 * (3 * 0.062) * p->kf; p->arm = 0.26; p->motor_tau = 1.0 / 30; p->min_rpm = 1200; p->max_rpm = 35000;
    p->ctrl_mass = 0.98; p->ctrl_grav = 9.81;                                                  // simulator_example.launch "mass"; SO3Control()
    const double kx[3] = {5.7, 5.7, 6.2}, kv[3] = {3.4, 3.4, 4.0}, kR[3] = {1.0, 1.0, 1.0}, kOm[3] = {0.07, 0.07, 0.1};
    for (int i = 0; i < 3; i++) { p->kx[i] = kx[i]; p->kv[i] = kv[i]; p->kR[i] = kR[i]; p->kOm[i] = kOm[i]; p->corrections[i] = 0.0; }
    p->sim_rate = 1000; p->cmd_rate = 100; p->t_end = 10; p->diverge_dist = 5;
    p->log_every = 1; p->use_external_yaw = 1; p->floor = 1;
    return 0;
}

// validated parameters -> ticks, steps per tick and log records per rollout
static int sim_params_check(const isdf_sim_params *p, int *n_ticks, int *m, int *n_log) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    const double *d = &p->mass;
    for (size_t i = 0; i < offsetof(isdf_sim_params, log_every) / sizeof(double); i++)
        if (!std::isfinite(d[i])) return fail(ISDF_ERR_INVALID, "a simulation parameter is not finite");
    if (!(p->mass > 0 && p->J[0] > 0 && p->J[1] > 0 && p->J[2] > 0 && p->kf > 0 && p->km > 0 && p->arm > 0 && p->motor_tau > 0 && p->ctrl_mass > 0))
        return fail(ISDF_ERR_INVALID, "mass, J, kf, km, arm, motor_tau and ctrl_mass must be positive");
    if (!(p->min_rpm >= 0 && p->max_rpm >= p->min_rpm)) return fail(ISDF_ERR_INVALID, "rpm limits must satisfy 0 <= min_rpm <= max_rpm");
    if (!(p->sim_rate > 0 && p->cmd_rate > 0)) return fail(ISDF_ERR_INVALID, "sim_rate and cmd_rate must be positive");
    const double ratio = p->sim_rate / p->cmd_rate;
    if (std::fmod(p->sim_rate, p->cmd_rate) != 0 || ratio < 1 || ratio > 1e6) return fail(ISDF_ERR_INVALID, "sim_rate must be a whole multiple of cmd_rate");
    if (!(p->t_end >= 0) || p->t_end * p->cmd_rate >= 2147483646.0) return fail(ISDF_ERR_INVALID, "t_end must be >= 0 with fewer than 2^31 ticks");
    if (p->log_every < 1) return fail(ISDF_ERR_INVALID, "log_every must be >= 1");
    if (!(p->diverge_dist > 0)) return fail(ISDF_ERR_INVALID, "diverge_dist must be positive");
    if (p->reserved_ != 0) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    *m = (int)ratio;
    *n_ticks = (int)std::floor(p->t_end * p->cmd_rate) + 1;
    *n_log = (*n_ticks - 1) / p->log_every + 1;
    return 0;
}

static int sim_args_check(isdf_ctx *c, int B, const void *off, const void *T, const void *C, int R, const void *traj, const void *init,
                          const isdf_sim_params *p, int cap_log, const void *log, const void *summary, int *n_ticks, int *m) {
    if (!c || !off || !T || !C || !traj || !init || !summary) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (B < 1) return fail(ISDF_ERR_INVALID, "B < 1");
    if (R < 0) return fail(ISDF_ERR_INVALID, "R < 0");
    int n_log = 0;
    if (int rc = sim_params_check(p, n_ticks, m, &n_log)) return rc;
    if (log && cap_log < n_log) return fail(ISDF_ERR_INVALID, "cap_log is smaller than the log records per rollout");
    if (log && (long long)R * cap_log > (1ll << 40)) return fail(ISDF_ERR_INVALID, "log too large");
    return 0;
}

static int sim_launch(isdf_ctx *c, int B, const int *d_off, const double *d_T, const double *d_C, int R, const int *d_traj, const double *d_init,
                      const double *d_dist, const isdf_sim_params *p, int n_ticks, int m, int cap_log, double *d_log, isdf_sim_summary *d_sum,
                      cudaStream_t st) {
    SimArgs A;
    A.p = *p; A.B = B; A.R = R; A.n_ticks = n_ticks; A.m = m; A.cap_log = cap_log;
    A.off = d_off; A.traj = d_traj; A.T = d_T; A.C = d_C; A.init = d_init; A.dist = d_dist; A.log = d_log; A.summary = d_sum;
    CU_TRY(simulate_launch(A, st));
    c->stats.kernel_launches++;
    return 0;
}

static void sim_poison_host(isdf_sim_summary *s, int R) {
    if (!s || R < 1) return;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    for (int r = 0; r < R; r++) {
        s[r].max_err = s[r].t_max_err = s[r].rms_err = s[r].final_err = s[r].max_tilt = s[r].max_omega = s[r].t_diverged = nan;
        s[r].accepted = s[r].rejected = -1;
        s[r].clamped_steps = s[r].floor_contacts = s[r].nan_rollbacks = -1;
        s[r].diverged = 1;
    }
}

extern "C" int isdf_simulate(isdf_ctx *c, int B, const int32_t *piece_off, const double *T, const double *coeffs, int R, const int32_t *traj,
                             const double *init, const double *dist, const isdf_sim_params *p, int cap_log, double *log, isdf_sim_summary *summary) {
    return poison_on_failure([&]() -> int {
        int n_ticks = 0, m = 0;
        if (int rc = sim_args_check(c, B, piece_off, T, coeffs, R, traj, init, p, cap_log, log, summary, &n_ticks, &m)) return rc;
        if (int rc = offsets_check(piece_off, B, "piece_off", true)) return rc;
        const int P = piece_off[B];
        if (P > 0) if (int rc = swept_traj_check(P, T, coeffs)) return rc;
        for (int r = 0; r < R; r++)
            if (traj[r] < 0 || traj[r] >= B || piece_off[traj[r] + 1] == piece_off[traj[r]])
                return fail(ISDF_ERR_INVALID, "traj[r] outside [0, B) or naming a trajectory without pieces");
        if (R == 0) return 0;
        if (set_device(c)) return ISDF_ERR_CUDA;
        Staging S(c);
        const double *d_C, *d_T, *d_init, *d_dist = nullptr;
        const int *d_off, *d_traj;
        double *d_log = nullptr;
        isdf_sim_summary *d_sum;
        S.in(&d_C, coeffs, 18 * (size_t)P); S.in(&d_T, T, (size_t)P); S.in(&d_init, init, (size_t)ISDF_SIM_INIT_DOUBLES * R);
        if (dist) S.in(&d_dist, dist, (size_t)6 * R);
        S.in(&d_off, piece_off, (size_t)B + 1); S.in(&d_traj, traj, (size_t)R);
        S.out(&d_sum, summary, (size_t)R);
        if (log) S.out(&d_log, log, (size_t)R * cap_log * ISDF_SIM_DOUBLES);
        if (int rc = S.upload()) return rc;
        if (int rc = sim_launch(c, B, d_off, d_T, d_C, R, d_traj, d_init, d_dist, p, n_ticks, m, cap_log, d_log, d_sum, c->stream)) return rc;
        return S.download();
    }, [&]() { sim_poison_host(summary, R); });
}

extern "C" int isdf_simulate_device(isdf_ctx *c, int B, const int32_t *d_piece_off, const double *d_T, const double *d_coeffs, int R,
                                    const int32_t *d_traj, const double *d_init, const double *d_dist, const isdf_sim_params *p, int cap_log,
                                    double *d_log, isdf_sim_summary *d_summary, void *cuda_stream) {
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    return poison_on_failure([&]() -> int {
        int n_ticks = 0, m = 0;
        if (int rc = sim_args_check(c, B, d_piece_off, d_T, d_coeffs, R, d_traj, d_init, p, cap_log, d_log, d_summary, &n_ticks, &m)) return rc;
        if (R == 0) return 0;
        if (set_device(c)) return ISDF_ERR_CUDA;
        return sim_launch(c, B, d_piece_off, d_T, d_coeffs, R, d_traj, d_init, d_dist, p, n_ticks, m, cap_log, d_log, d_summary, st);
    }, [&]() {
        if (c && d_summary && R > 0 && set_device(c) == 0 && sim_poison_launch(d_summary, R, st) == cudaSuccess) c->stats.kernel_launches++;
    });
}

// ---- depth sensing (isdf_sense.cuh, compiled in isdf_sense_tu.cu) ----
extern "C" int isdf_sense_default_params(isdf_sense_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    std::memset(p, 0, sizeof(*p));
    p->width = 640; p->height = 480;                                   // local_sensing/params/camera.yaml
    p->fx = 387.229248046875; p->fy = 387.229248046875; p->cx = 321.04638671875; p->cy = 243.44969177246094;
    const double cam02body[16] = {0, 0, 1, 0, -1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 0, 1};   // pcl_render_node.cpp:347-350
    std::memcpy(p->cam_to_body, cam02body, sizeof cam02body);
    p->sensing_horizon = std::numeric_limits<double>::infinity();
    return 0;
}

static int sense_cloud_set(isdf_ctx *c, const void *pts, int64_t n, int32_t stride, bool device, cudaStream_t st) {
    if (int rc = cloud_args_check(c, pts, n, stride, 1.0)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    c->sense.release();
    DevBuf<char> d_pts;
    const char *d = (const char *)pts;
    int launches = 0;
    cudaError_t e = cudaSuccess;
    if (!device) {
        e = d_pts.ensure((size_t)n * stride);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_pts.p, pts, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream);
        d = d_pts.p; st = c->stream;
    }
    if (e == cudaSuccess) e = sense_set_cloud(c->sense, d, n, stride, st, &launches);
    c->stats.kernel_launches += launches;
    if (e != cudaSuccess) {
        c->sense.release();
        return fail(ISDF_ERR_CUDA, std::string("isdf_set_sense_cloud: ") + cudaGetErrorString(e));
    }
    return 0;
}
extern "C" int isdf_set_sense_cloud(isdf_ctx *c, const void *points, int64_t n, int32_t stride_bytes) {
    return sense_cloud_set(c, points, n, stride_bytes, false, nullptr);
}
extern "C" int isdf_set_sense_cloud_device(isdf_ctx *c, const void *d_points, int64_t n, int32_t stride_bytes, void *cuda_stream) {
    return sense_cloud_set(c, d_points, n, stride_bytes, true, (cudaStream_t)cuda_stream);
}
extern "C" int isdf_get_sense_info(isdf_ctx *c, isdf_sense_info *out) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->sense.have) return fail(ISDF_ERR_STATE, "no scene cloud: set one with isdf_set_sense_cloud");
    out->points_used = c->sense.n; out->points_skipped = c->sense.skipped; out->bricks = c->sense.nb;
    return 0;
}

static int sense_cam_check(const isdf_sense_params *p);
// the checks every sensing call shares; the context (and its scene) last
static int sense_args_check(isdf_ctx *c, int64_t Q, const void *pos, const void *quat, int64_t stride, const isdf_sense_params *p,
                            const void *out) {
    if (!pos || !quat || !p || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (Q < 1 || Q >= (1ll << 31)) return fail(ISDF_ERR_INVALID, "Q must be in [1, 2^31)");
    if (stride < 1) return fail(ISDF_ERR_INVALID, "stride_doubles < 1");
    if (int rc = sense_cam_check(p)) return rc;
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!c->sense.have) return fail(ISDF_ERR_STATE, "no scene cloud: set one with isdf_set_sense_cloud");
    return 0;
}

// the checks of one camera
static int sense_cam_check(const isdf_sense_params *p) {
    if (p->width < 1 || p->height < 1 || (long long)p->width * p->height > (1ll << 26))
        return fail(ISDF_ERR_INVALID, "width and height must be >= 1 with width x height <= 2^26");
    if (!std::isfinite(p->fx) || !std::isfinite(p->fy) || !std::isfinite(p->cx) || !std::isfinite(p->cy))
        return fail(ISDF_ERR_INVALID, "a camera parameter is not finite");
    if (!(p->fx > 0 && p->fy > 0)) return fail(ISDF_ERR_INVALID, "fx and fy must be positive");
    for (int i = 0; i < 16; i++) if (!std::isfinite(p->cam_to_body[i])) return fail(ISDF_ERR_INVALID, "a cam_to_body entry is not finite");
    if (p->cam_to_body[12] != 0 || p->cam_to_body[13] != 0 || p->cam_to_body[14] != 0 || p->cam_to_body[15] != 1)
        return fail(ISDF_ERR_INVALID, "cam_to_body's last row must be (0, 0, 0, 1)");
    if (!(p->sensing_horizon > 0)) return fail(ISDF_ERR_INVALID, "sensing_horizon must be positive (+Inf keeps every point)");
    return 0;
}

// Q poses read at a stride of `stride` doubles, staged as (x, y, z, w, qx, qy, qz) records 7 doubles apart at *d
static void stage_poses(Staging &S, int64_t Q, const double *pos, const double *quat, int64_t stride, const double **d) {
    S.in(d, 7 * (size_t)Q, [=](double *h) {
        for (int64_t q = 0; q < Q; q++) {
            std::memcpy(h + 7 * q, pos + q * stride, 3 * sizeof(double));
            std::memcpy(h + 7 * q + 3, quat + q * stride, 4 * sizeof(double));
        }
    });
}

static int sense_depth_impl(isdf_ctx *c, int64_t Q, const double *pos, const double *quat, int64_t stride, const isdf_sense_params *p,
                            int32_t *depth, bool device, cudaStream_t st) {
    if (int rc = sense_args_check(c, Q, pos, quat, stride, p, depth)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    SenseCall C{Q, pos, quat, stride, *p};
    Staging S(c);
    if (!device) {
        const double *d_pose;
        stage_poses(S, Q, pos, quat, stride, &d_pose);
        if (int rc = S.upload()) return rc;
        C.pos = d_pose; C.quat = d_pose + 3; C.stride = 7;
        st = c->stream;
    }
    int launches = 0;
    const cudaError_t e = sense_depth_run(c->sense, C, depth, device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st, &launches);
    c->stats.kernel_launches += launches;
    if (e != cudaSuccess) return fail(ISDF_ERR_CUDA, std::string("isdf_sense_depth: ") + cudaGetErrorString(e));
    if (!device) CU_TRY(cudaStreamSynchronize(st));
    return 0;
}
extern "C" int isdf_sense_depth(isdf_ctx *c, int64_t Q, const double *pos, const double *quat, int64_t stride_doubles,
                                const isdf_sense_params *p, int32_t *depth) {
    return sense_depth_impl(c, Q, pos, quat, stride_doubles, p, depth, false, nullptr);
}
extern "C" int isdf_sense_depth_device(isdf_ctx *c, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride_doubles,
                                       const isdf_sense_params *p, int32_t *d_depth, void *cuda_stream) {
    return sense_depth_impl(c, Q, d_pos, d_quat, stride_doubles, p, d_depth, true, (cudaStream_t)cuda_stream);
}

static int sense_cloud_impl(isdf_ctx *c, int64_t Q, const double *pos, const double *quat, int64_t stride, const isdf_sense_params *p,
                            int64_t cap, float *points, int64_t *offsets, bool device, cudaStream_t st) {
    if (int rc = sense_args_check(c, Q, pos, quat, stride, p, offsets)) return rc;
    if (cap < 0 || (cap > 0 && !points)) return fail(ISDF_ERR_INVALID, "cap < 0, or points NULL with cap > 0");
    if (set_device(c)) return ISDF_ERR_CUDA;
    SenseCall C{Q, pos, quat, stride, *p};
    float *d_points = points;
    int64_t *d_off = offsets;
    Staging S(c);
    if (!device) {   // the results' room; their sizes are known after the call, so they come back by themselves below
        const double *d_pose;
        stage_poses(S, Q, pos, quat, stride, &d_pose);
        S.out(&d_off, nullptr, (size_t)Q + 1); S.out(&d_points, nullptr, 3 * (size_t)cap);
        if (int rc = S.upload()) return rc;
        C.pos = d_pose; C.quat = d_pose + 3; C.stride = 7;
        st = c->stream;
    }
    int launches = 0;
    const cudaError_t e = sense_cloud_run(c->sense, C, d_points, cap, d_off, st, &launches);
    c->stats.kernel_launches += launches;
    if (e != cudaSuccess) return fail(ISDF_ERR_CUDA, std::string("isdf_sense_cloud: ") + cudaGetErrorString(e));
    int64_t total = 0;
    CU_TRY(cudaMemcpyAsync(&total, d_off + Q, sizeof total, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    if (!device) {
        CU_TRY(cudaMemcpyAsync(offsets, d_off, sizeof(int64_t) * (Q + 1), cudaMemcpyDeviceToHost, st));
        if (std::min(total, cap) > 0) CU_TRY(cudaMemcpyAsync(points, d_points, 3 * sizeof(float) * std::min(total, cap), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
    }
    if (total > cap) return fail(ISDF_ERR_INVALID, "cap smaller than the sensed points (offsets report the sizes)");
    return 0;
}
extern "C" int isdf_sense_cloud(isdf_ctx *c, int64_t Q, const double *pos, const double *quat, int64_t stride_doubles,
                                const isdf_sense_params *p, int64_t cap, float *points, int64_t *offsets) {
    return sense_cloud_impl(c, Q, pos, quat, stride_doubles, p, cap, points, offsets, false, nullptr);
}
extern "C" int isdf_sense_cloud_device(isdf_ctx *c, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride_doubles,
                                       const isdf_sense_params *p, int64_t cap, float *d_points, int64_t *d_offsets, void *cuda_stream) {
    return sense_cloud_impl(c, Q, d_pos, d_quat, stride_doubles, p, cap, d_points, d_offsets, true, (cudaStream_t)cuda_stream);
}
// ---- known space from depth images (isdf_observe.cuh) ----
static int observe_impl(isdf_ctx *c, int64_t Q, const double *pos, const double *quat, int64_t stride, const isdf_sense_params *p,
                        isdf_observe_info *info, bool device, cudaStream_t st) {
    if (int rc = sense_args_check(c, Q, pos, quat, stride, p, pos)) return rc;
    if (!std::isfinite(p->sensing_horizon)) return fail(ISDF_ERR_INVALID, "isdf_map_observe needs a finite sensing_horizon");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    const double D = std::ceil(2.0 * p->sensing_horizon / c->map.grid.res) + 3.0;
    if (!(D * D * D <= (double)(1ll << 40))) return fail(ISDF_ERR_INVALID, "sensing_horizon / res too large: a pose's horizon box exceeds 2^40 voxels");
    if (set_device(c)) return ISDF_ERR_CUDA;
    SenseCall C{Q, pos, quat, stride, *p};
    Staging S(c);
    if (!device) {
        const double *d_pose;
        stage_poses(S, Q, pos, quat, stride, &d_pose);
        if (int rc = S.upload()) return rc;
        C.pos = d_pose; C.quat = d_pose + 3; C.stride = 7;
        st = c->stream;
    }
    if (int r = known_bits(c, st)) return r;
    int launches = 0;
    unsigned long long cnt[2] = {0, 0};
    const cudaError_t e = sense_observe_run(c->sense, C, c->map.grid, c->known.d_known.p, cnt, st, &launches);
    c->stats.kernel_launches += launches;
    c->known.blocked_ok = false;
    if (e != cudaSuccess) {
        drop_map(c);
        return fail(ISDF_ERR_CUDA, std::string("isdf_map_observe: ") + cudaGetErrorString(e));
    }
    if (info) { info->poses = Q; info->voxels_tested = (int64_t)cnt[0]; info->voxels_added = (int64_t)cnt[1]; }
    return 0;
}
extern "C" int isdf_map_observe(isdf_ctx *c, int64_t Q, const double *pos, const double *quat, int64_t stride_doubles, const isdf_sense_params *p,
                                isdf_observe_info *info) {
    return observe_impl(c, Q, pos, quat, stride_doubles, p, info, false, nullptr);
}
extern "C" int isdf_map_observe_device(isdf_ctx *c, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride_doubles,
                                       const isdf_sense_params *p, isdf_observe_info *info, void *cuda_stream) {
    return observe_impl(c, Q, d_pos, d_quat, stride_doubles, p, info, true, (cudaStream_t)cuda_stream);
}

// ---- view gain (isdf_view.cuh) ----
// the checks of a view-gain rig, and the map it needs: every camera as the sensing calls check one, a finite horizon, and a horizon box of
// at most 2^40 voxels
static int view_rig_check(isdf_ctx *c, int n_cams, const isdf_sense_params *cams) {
    if (n_cams < 1 || !cams) return fail(ISDF_ERR_INVALID, "a view gain needs n_cams >= 1 cameras");
    double hmax = 0.0;
    for (int k = 0; k < n_cams; k++) {
        if (int rc = sense_cam_check(cams + k)) return rc;
        if (!std::isfinite(cams[k].sensing_horizon)) return fail(ISDF_ERR_INVALID, "a view gain needs a finite sensing_horizon on every camera");
        hmax = std::max(hmax, cams[k].sensing_horizon);
    }
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (c->world > 1) return fail(ISDF_ERR_UNSUPPORTED, "the view gain is not sharded: call it on a context with isdf_set_shard(ctx, 0, 1)");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    const double D = std::ceil(2.0 * hmax / c->map.grid.res) + 3.0;
    if (!(D * D * D <= (double)(1ll << 40))) return fail(ISDF_ERR_INVALID, "sensing_horizon / res too large: a pose's horizon box exceeds 2^40 voxels");
    return 0;
}

static int view_gain_impl(isdf_ctx *c, int64_t Q, const double *pos, const double *quat, int64_t stride, int n_cams, const isdf_sense_params *cams,
                          int64_t *gain, bool device, cudaStream_t st) {
    if (!pos || !quat || !gain) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (Q < 1 || Q >= (1ll << 31)) return fail(ISDF_ERR_INVALID, "Q must be in [1, 2^31)");
    if (stride < 1) return fail(ISDF_ERR_INVALID, "stride_doubles < 1");
    if (int rc = view_rig_check(c, n_cams, cams)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    int64_t *d_gain = gain;
    Staging S(c);
    if (!device) {
        const double *d_pose;
        stage_poses(S, Q, pos, quat, stride, &d_pose);
        S.out(&d_gain, gain, (size_t)Q);
        if (int rc = S.upload()) return rc;
        pos = d_pose; quat = d_pose + 3; stride = 7;
        st = c->stream;
    }
    int launches = 0;
    const cudaError_t e = view_gain_run(c->sense, Q, pos, quat, stride, n_cams, cams, c->map.grid, c->known.have ? c->known.d_known.p : nullptr,
                                        nullptr, d_gain, st, &launches);
    c->stats.kernel_launches += launches;
    if (e != cudaSuccess) return fail(ISDF_ERR_CUDA, std::string("isdf_view_gain: ") + cudaGetErrorString(e));
    if (!device) return S.download();
    CU_TRY(cudaStreamSynchronize(st));
    return 0;
}
extern "C" int isdf_view_gain(isdf_ctx *c, int64_t Q, const double *pos, const double *quat, int64_t stride_doubles, int n_cams,
                              const isdf_sense_params *cams, int64_t *gain) {
    return view_gain_impl(c, Q, pos, quat, stride_doubles, n_cams, cams, gain, false, nullptr);
}
extern "C" int isdf_view_gain_device(isdf_ctx *c, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride_doubles, int n_cams,
                                     const isdf_sense_params *cams, int64_t *d_gain, void *cuda_stream) {
    return view_gain_impl(c, Q, d_pos, d_quat, stride_doubles, n_cams, cams, d_gain, true, (cudaStream_t)cuda_stream);
}

// the blocked grid occ | ~known, rebuilt on st (and waited for, so that a later call on another stream reads it whole) when stale
static int blocked_grid_ready(isdf_ctx *c, cudaStream_t st) {
    if (c->known.blocked_ok || !c->map.have_map) return 0;
    const DevGrid &g = c->map.grid;
    CU_TRY(c->known.d_blocked.ensure((size_t)g.X * g.Y * g.Zw));
    int launches = 0;
    const cudaError_t e = blocked_build(g, c->known.have ? c->known.d_known.p : nullptr, c->known.d_blocked.p, st, &launches);
    c->stats.kernel_launches += launches;
    CU_TRY(e);
    CU_TRY(cudaStreamSynchronize(st));
    c->known.blocked = g;
    c->known.blocked.bits = c->known.d_blocked.p;
    c->known.blocked_ok = true;
    return 0;
}

// the grid the clearance family reads: the occupancy grid, or under ISDF_UNKNOWN_OCCUPIED the blocked grid (blocked_grid_ready)
static int clearance_grid_ready(isdf_ctx *c, cudaStream_t st) {
    if (c->known.policy != ISDF_UNKNOWN_OCCUPIED) return 0;
    return blocked_grid_ready(c, st);
}

// ---- world generators (isdf_world.cuh, compiled in isdf_world_tu.cu) ----
extern "C" int isdf_world_default_params(int kind, isdf_world_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (kind != ISDF_WORLD_GLOBALMAP && kind != ISDF_WORLD_PERLIN && kind != ISDF_WORLD_BOXES) return fail(ISDF_ERR_INVALID, "unknown world kind");
    std::memset(p, 0, sizeof(*p));
    p->kind = kind;
    p->map_id = 4; p->rand_seed = 1; p->srand_seed = 0;                               // globalmap_gene.launch
    p->cloud_resolution = 0.6; p->init[0] = p->init[1] = p->init[2] = 1.0;
    p->seed = 511; p->size[0] = 100; p->size[1] = 100; p->size[2] = 30; p->scale = 10;   // mockamap.launch: 10 x 10 x 3 m at 0.1 m
    p->complexity = 0.03; p->fill = 0.3; p->fractal = 1; p->attenuation = 0.1;
    p->obstacle_number = 50; p->width_min = 0.6; p->width_max = 1.5;
    return 0;
}

static int world_impl(isdf_ctx *c, const isdf_world_params *p, int64_t cap, float *points, int64_t *n, bool device, cudaStream_t st) {
    if (!p || !n) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (cap < 0 || (cap > 0 && !points)) return fail(ISDF_ERR_INVALID, "cap < 0, or points NULL with cap > 0");
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    WorldPlan P;
    std::string msg;
    if (int rc = world_plan(*p, P, &msg)) return fail(rc, "isdf_world_cloud: " + msg);
    if (set_device(c)) return ISDF_ERR_CUDA;
    float *d_points = points;
    long long room = cap;
    if (!device) {   // the records' device room: the cloud's size, or for Perlin the voxel count that bounds it
        room = std::min<long long>(cap, P.n);
        CU_TRY(c->gen.d_out.ensure(4 * (size_t)std::max(room, 1ll)));
        d_points = c->gen.d_out.p; st = c->stream;
    }
    int launches = 0;
    long long total = 0;
    const cudaError_t e = world_emit(c->gen, P, room, d_points, &total, st, &launches);
    c->stats.kernel_launches += launches;
    if (e != cudaSuccess) return fail(ISDF_ERR_CUDA, std::string("isdf_world_cloud: ") + cudaGetErrorString(e));
    *n = total;
    if (!device) {
        if (std::min(total, room) > 0)
            CU_TRY(cudaMemcpyAsync(points, d_points, 4 * sizeof(float) * std::min(total, room), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
    }
    if (total > cap) return fail(ISDF_ERR_INVALID, "cap smaller than the cloud (*n reports its size)");
    return 0;
}
extern "C" int isdf_world_cloud(isdf_ctx *c, const isdf_world_params *p, int64_t cap, float *points, int64_t *n) {
    return world_impl(c, p, cap, points, n, false, nullptr);
}
extern "C" int isdf_world_cloud_device(isdf_ctx *c, const isdf_world_params *p, int64_t cap, float *d_points, int64_t *n, void *cuda_stream) {
    return world_impl(c, p, cap, d_points, n, true, (cudaStream_t)cuda_stream);
}
// diagnostics (not in include/isdf.h): render at most `poses` poses per chunk (0: the automatic chunking)
extern "C" int isdf_dbg_sense_chunk(isdf_ctx *c, int poses) {
    if (!c || poses < 0) return fail(ISDF_ERR_INVALID, "bad argument");
    c->sense.chunk_override = poses;
    return 0;
}

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
// ---- every plan's obstacle list in one call (isdf_gather_obstacle_points_batch) -----------------------------------------------------
// B plans, plan b owning the waypoint rows [wp_off[b], wp_off[b+1]). Four launches over all plans: k_gather_boxes_batch (the index boxes of
// every row, the 999 sentinel at each plan's first row), k_gather_points_batch<false> (grid (waypoint, plan): how many voxels each row
// emits), k_gather_scan (the exclusive scan of the row counts) and k_gather_points_batch<true> (the ordered compaction at each row's
// offset). The rows of all plans are scanned in one pass: plans lie back to back, so a row's offset is its plan's offset plus the counts of
// the plan's earlier rows, and a plan's offset is the offset of its first row. Output order = the reference's: plan by plan, waypoint by
// waypoint, each box in x -> y -> z order; a voxel belongs to the FIRST waypoint of its plan whose box includes it.
constexpr int GATHER_LIST_CAP = 1024;   // earlier boxes of a plan kept per CTA; with more, every earlier box of the plan is tested

// the plan b with wp_off[b] <= q < wp_off[b+1] (empty plans skipped): the smallest b with wp_off[b+1] > q
__device__ __forceinline__ int gather_plan_of(const int *wp_off, int B, int q) {
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (wp_off[mid + 1] > q) hi = mid; else lo = mid + 1;
    }
    return lo;
}

__global__ void k_gather_boxes_batch(const DevGrid G, const int *wp_off, int B, const double *wps, int R, double h, double ox, double oy, double oz,
                                     GatherBox *boxes) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= R) return;
    const bool first = wp_off[gather_plan_of(wp_off, B, q)] == q;
    GatherBox b;
    const double c[3] = {wps[3 * q] + ox, wps[3 * q + 1] + oy, wps[3 * q + 2] + oz};
    const double l[3] = {first ? 999.0 : wps[3 * (q - 1)], first ? 999.0 : wps[3 * (q - 1) + 1], first ? 999.0 : wps[3 * (q - 1) + 2]};
    const int dims[3] = {G.X, G.Y, G.Z};
    for (int a = 0; a < 3; a++) {
        b.a0[a] = grid_axis_index(c[a] - h, G.bmin[a], G.bmax[a], G.res, dims[a]); b.a1[a] = grid_axis_index(c[a] + h, G.bmin[a], G.bmax[a], G.res, dims[a]);
        b.l0[a] = grid_axis_index(l[a] - h, G.bmin[a], G.bmax[a], G.res, dims[a]); b.l1[a] = grid_axis_index(l[a] + h, G.bmin[a], G.bmax[a], G.res, dims[a]);
    }
    boxes[q] = b;
}

// CTA (j, b): row wp_off[b] + j. An earlier box of the plan can claim a voxel of this box only if their include boxes (a0..a1) intersect;
// those are listed once per CTA and the voxel loop tests only them. Count pass: counts[row]; write pass: the voxels at offs[row] (< cap).
// known_rows (may be NULL): plan b's rows j < known_rows[b] read the blocked grid's words instead of the occupancy grid's. The earlier boxes
// are tested on the row's own grid: a known row's earlier rows are known, and an occupied voxel is blocked, so an occupancy row's voxel is
// set in every earlier row's grid alike.
template <bool WRITE>
__global__ void __launch_bounds__(256) k_gather_points_batch(DevGrid G, const int *wp_off, const GatherBox *boxes, int *counts,
                                                            const long long *offs, double *out, long long cap, const uint32_t *blocked,
                                                            const int *known_rows) {
    __shared__ int warp_cnt[8];
    __shared__ int nlist;
    __shared__ long long running;
    __shared__ int list[GATHER_LIST_CAP];
    const int q0 = wp_off[blockIdx.y], j = blockIdx.x;
    if (j >= wp_off[blockIdx.y + 1] - q0) return;   // the plan has fewer rows (uniform over the CTA)
    if (known_rows && j < known_rows[blockIdx.y]) G.bits = blocked;
    const int q = q0 + j;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const GatherBox b = boxes[q];
    if (threadIdx.x == 0) { running = WRITE ? offs[q] : 0; nlist = 0; }
    __syncthreads();
    for (int base = 0; base < j; base += blockDim.x) {
        const int p = base + threadIdx.x;
        bool hit = false;
        if (p < j) {
            const GatherBox &o = boxes[q0 + p];
            hit = o.a0[0] <= b.a1[0] && o.a1[0] >= b.a0[0] && o.a0[1] <= b.a1[1] && o.a1[1] >= b.a0[1] && o.a0[2] <= b.a1[2] && o.a1[2] >= b.a0[2];
        }
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) warp_cnt[warp] = __popc(bal);
        __syncthreads();
        int off = nlist;
        for (int w = 0; w < warp; w++) off += warp_cnt[w];
        if (hit) {
            const int pos = off + __popc(bal & ((1u << lane) - 1u));
            if (pos < GATHER_LIST_CAP) list[pos] = q0 + p;
        }
        __syncthreads();
        if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < 8; w++) t += warp_cnt[w]; nlist += t; }
        __syncthreads();
    }
    const int nl = nlist;
    const int ny = b.a1[1] - b.a0[1] + 1, nz = b.a1[2] - b.a0[2] + 1;
    const int nvox = (b.a1[0] - b.a0[0] + 1) * ny * nz;
    for (int base = 0; base < nvox; base += blockDim.x) {
        const int v = base + threadIdx.x;
        bool emit = false; int i = 0, jj = 0, k = 0;
        if (v < nvox) {
            i = b.a0[0] + v / (ny * nz); jj = b.a0[1] + (v / nz) % ny; k = b.a0[2] + v % nz;
            emit = gather_includes(G, b, i, jj, k);
            if (nl <= GATHER_LIST_CAP) { for (int t = 0; emit && t < nl; t++) if (gather_includes(G, boxes[list[t]], i, jj, k)) emit = false; }
            else { for (int p = q0; emit && p < q; p++) if (gather_includes(G, boxes[p], i, jj, k)) emit = false; }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, emit);
        if (lane == 0) warp_cnt[warp] = __popc(bal);
        __syncthreads();
        if (WRITE && emit) {
            long long pos = running + __popc(bal & ((1u << lane) - 1u));
            for (int w = 0; w < warp; w++) pos += warp_cnt[w];
            if (pos < cap) { out[3 * pos] = (i + 0.5) * G.res + G.bmin[0]; out[3 * pos + 1] = (jj + 0.5) * G.res + G.bmin[1]; out[3 * pos + 2] = (k + 0.5) * G.res + G.bmin[2]; }
        }
        __syncthreads();
        if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < 8; w++) t += warp_cnt[w]; running += t; }
        __syncthreads();
    }
    if (!WRITE && threadIdx.x == 0) counts[q] = (int)running;
}

// one CTA: offs[r] = sum of counts[0 .. r-1] over the R rows (in chunks of 1024, each a warp-shuffle scan plus a scan of the warp totals),
// pt_off[b] = the offset of plan b's first row (the total for plans at the end), *total = the sum of every count
__global__ void __launch_bounds__(1024) k_gather_scan(const int *counts, int R, const int *wp_off, int B, long long *offs, int *pt_off, long long *total) {
    __shared__ long long warp_sum[32];
    __shared__ long long running;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) running = 0;
    __syncthreads();
    for (int base = 0; base < R; base += 1024) {
        const int r = base + threadIdx.x;
        const long long v = r < R ? counts[r] : 0;
        long long incl = v;
        for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            long long s = warp_sum[lane];
            for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += t; }
            warp_sum[lane] = s;
        }
        __syncthreads();
        const long long excl = running + (warp ? warp_sum[warp - 1] : 0) + incl - v;
        if (r < R) offs[r] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) running = excl + v;
        __syncthreads();
    }
    for (int b = threadIdx.x; b <= B; b += blockDim.x) {
        const long long o = wp_off[b] < R ? offs[wp_off[b]] : running;
        pt_off[b] = (int)(o < 0x7fffffffll ? o : 0x7fffffffll);
    }
    if (threadIdx.x == 0) *total = running;
}

// the batched gather on stream st from staged inputs: d_wp (R x 3 rows), d_wp_off (its B + 1 offsets; h_wp_off the same on the host),
// d_known_rows (B, may be NULL: every row reads the occupancy grid). Counts and scans, reads the plans' offsets into pt_off (B + 1, also
// when the lists exceed cap) and the total into *total; then, when the total fits cap, writes every list to c->gat.d_out.
static int gather_batch_run(isdf_ctx *c, int B, const int *h_wp_off, const int *d_wp_off, const double *d_wp, double half, const double *offset,
                            const int *d_known_rows, long long cap, std::vector<int> &pt_off, long long *total, cudaStream_t st) {
    auto &g = c->gat;
    if (d_known_rows) if (int r = blocked_grid_ready(c, st)) return r;
    const uint32_t *blocked = d_known_rows ? c->known.d_blocked.p : nullptr;
    const int R = h_wp_off[B];
    int maxQ = 0;
    for (int b = 0; b < B; b++) maxQ = std::max(maxQ, h_wp_off[b + 1] - h_wp_off[b]);
    const size_t Rd = (size_t)std::max(R, 1);
    CU_TRY(g.d_box.ensure(Rd)); CU_TRY(g.d_cnt.ensure(Rd)); CU_TRY(g.d_offs.ensure(Rd)); CU_TRY(g.d_ptoff.ensure((size_t)B + 1)); CU_TRY(g.d_total.ensure(1));
    const double ox = offset ? offset[0] : 0.0, oy = offset ? offset[1] : 0.0, oz = offset ? offset[2] : 0.0;
    if (R > 0) {
        k_gather_boxes_batch<<<(R + 127) / 128, 128, 0, st>>>(c->map.grid, d_wp_off, B, d_wp, R, half, ox, oy, oz, g.d_box.p);
        k_gather_points_batch<false><<<dim3(maxQ, B), 256, 0, st>>>(c->map.grid, d_wp_off, g.d_box.p, g.d_cnt.p, nullptr, nullptr, 0, blocked, d_known_rows);
        c->stats.kernel_launches += 2;
    }
    k_gather_scan<<<1, 1024, 0, st>>>(g.d_cnt.p, R, d_wp_off, B, g.d_offs.p, g.d_ptoff.p, g.d_total.p);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    pt_off.assign((size_t)B + 1, 0);
    CU_TRY(cudaMemcpyAsync(pt_off.data(), g.d_ptoff.p, sizeof(int) * ((size_t)B + 1), cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaMemcpyAsync(total, g.d_total.p, sizeof(long long), cudaMemcpyDeviceToHost, st));
    count_copy(c, cudaMemcpyDeviceToHost, sizeof(int) * ((size_t)B + 1)); count_copy(c, cudaMemcpyDeviceToHost, sizeof(long long));
    CU_TRY(cudaStreamSynchronize(st));
    if (*total > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "the obstacle lists hold more than 2^31 - 1 points");
    if (*total > cap) return fail(ISDF_ERR_INVALID, "cap smaller than the obstacle lists (pt_off reports their sizes)");
    if (*total == 0) return 0;
    CU_TRY(g.d_out.ensure((size_t)3 * *total));
    k_gather_points_batch<true><<<dim3(maxQ, B), 256, 0, st>>>(c->map.grid, d_wp_off, g.d_box.p, nullptr, g.d_offs.p, g.d_out.p, *total, blocked,
                                                          d_known_rows);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}

// the lists in c->gat.d_out become the batched swept-volume point sets (isdf_set_points_batch from device memory); no point at all gives
// up both sets and switches the batched term off
static int gather_set_points(isdf_ctx *c, int B, const std::vector<int> &pt_off, long long total, cudaStream_t st) {
    if (total == 0) CU_TRY(c->sv.set_points(nullptr, 0, st));
    else {
        CU_TRY(c->sv.set_points_batch(B, pt_off.data(), c->gat.d_out.p, st, cudaMemcpyDeviceToDevice));
        count_copy(c, cudaMemcpyHostToDevice, sizeof(int) * ((size_t)B + 1));   // the offsets
    }
    return 0;
}

// one plan's list: the batched gather with B = 1, whose write pass always runs, so that *n is the whole list's size
extern "C" int isdf_gather_obstacle_points(isdf_ctx *c, const double *waypoints, int nQ, double half_extent, const double *offset,
                                           double *out_points, int cap, int *n, int set_as_points) {
    if (!c || !waypoints || nQ < 1 || !n || cap < 0 || (cap > 0 && !out_points && !set_as_points)) return fail(ISDF_ERR_INVALID, "bad argument");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    if (set_device(c)) return ISDF_ERR_CUDA;
    auto &g = c->gat;
    const int wp_off[2] = {0, nQ};
    Staging S(c);
    const int *d_wpoff;
    const double *d_wp;
    S.in(&d_wpoff, wp_off, 2); S.in(&d_wp, waypoints, (size_t)3 * nQ);
    if (int r = S.upload()) return r;
    std::vector<int> off;
    long long total = 0;
    if (int r = gather_batch_run(c, 1, wp_off, d_wpoff, d_wp, half_extent, offset, nullptr, 0x7fffffffll, off, &total, c->stream)) return r;
    *n = (int)total;
    const long long m = std::min<long long>(total, cap);
    if (m > 0 && out_points) {   // the write pass runs on the context's non-blocking stream
        CU_TRY(cudaMemcpyAsync(out_points, g.d_out.p, sizeof(double) * 3 * m, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
    }
    if (!set_as_points) return 0;
    if (total > cap) return fail(ISDF_ERR_INVALID, "cap smaller than the obstacle list");
    CU_TRY(c->sv.set_points(g.d_out.p, (int)m, c->stream, cudaMemcpyDeviceToDevice));
    return 0;
}

extern "C" int isdf_gather_obstacle_points_batch_known(isdf_ctx *c, int B, const int32_t *wp_off, const double *waypoints, double half_extent,
                                                       const double *offset, const int32_t *known_rows, int64_t cap, double *out_points,
                                                       int32_t *pt_off, int set_as_points) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (B < 1 || B > 65535) return fail(ISDF_ERR_INVALID, "B must lie in [1, 65535]");
    if (!wp_off || !pt_off || cap < 0) return fail(ISDF_ERR_INVALID, "NULL argument or cap < 0");
    if (int r = offsets_check(wp_off, B, "wp_off", true)) return r;
    if (wp_off[B] > 0 && !waypoints) return fail(ISDF_ERR_INVALID, "waypoints is NULL");
    if (known_rows)
        for (int b = 0; b < B; b++)
            if (known_rows[b] < 0) return fail(ISDF_ERR_INVALID, "known_rows[" + std::to_string(b) + "] < 0");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    if (set_device(c)) return ISDF_ERR_CUDA;
    auto &g = c->gat;
    Staging S(c);
    const int *d_wpoff, *d_krows = nullptr;
    const double *d_wp;
    S.in(&d_wpoff, wp_off, (size_t)B + 1); S.in(&d_wp, waypoints, (size_t)3 * wp_off[B]);
    if (known_rows) S.in(&d_krows, known_rows, (size_t)B);
    if (int r = S.upload()) return r;
    std::vector<int> off;
    long long total = 0;
    const int r = gather_batch_run(c, B, wp_off, d_wpoff, d_wp, half_extent, offset, d_krows, out_points ? cap : 0x7fffffffll, off, &total,
                                   c->stream);
    if (!off.empty()) std::memcpy(pt_off, off.data(), sizeof(int32_t) * off.size());
    if (r) return r;
    if (out_points && total > 0) {   // the write pass runs on the context's non-blocking stream
        CU_TRY(cudaMemcpyAsync(out_points, g.d_out.p, sizeof(double) * 3 * total, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
    }
    if (set_as_points) return gather_set_points(c, B, off, total, c->stream);
    return 0;
}

extern "C" int isdf_gather_obstacle_points_batch(isdf_ctx *c, int B, const int32_t *wp_off, const double *waypoints, double half_extent,
                                                 const double *offset, int64_t cap, double *out_points, int32_t *pt_off, int set_as_points) {
    return isdf_gather_obstacle_points_batch_known(c, B, wp_off, waypoints, half_extent, offset, nullptr, cap, out_points, pt_off, set_as_points);
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
    if (c->mesh.shape.kind == ISDF_SHAPE_MESH && c->mesh.disc_ready) {   // the scan walks the sub-box filtered lists (DevMesh's two contracts)
        DevMesh &dm = A.shape.mesh;
        dm.cell_off = c->mesh.d_disc_off.p; dm.cell_cnt = c->mesh.d_disc_cnt.p; dm.cand = c->mesh.d_disc_cand.p; dm.cand_lb = c->mesh.d_disc_lb.p;
        dm.cell_rec = c->mesh.d_disc_rec.p;
    }
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

// The host form of the discrete and swept-volume evaluations: [coefficients 18N | durations N] and the inputs S already holds go in
// with ONE copy, `launch(d_T, d_C, d_out, count_out)` runs between ev0 and ev1, and [cost | gradC | gradT | counter word] come back
// in ONE copy. The result is added to *cost, gradC and gradT, as the reference accumulates (hpp:539-550, hpp:640-645); the counter
// word goes to the stat `counted`. The caller poisons *cost on failure.
template <typename Launch>
static int eval_host(isdf_ctx *c, Staging &S, int N, const double *T, const double *coeffs, double *cost, double *gradC, double *gradT,
                     int64_t isdf_stats::*counted, Launch launch) {
    if (set_device(c)) return ISDF_ERR_CUDA;
    const size_t nout = (size_t)19 * N + 1;
    const double *d_C, *d_T, *h_out = nullptr;
    double *d_out, *d_count;
    unsigned long long count = 0;
    S.in(&d_C, coeffs, 18 * (size_t)N); S.in(&d_T, T, (size_t)N);
    S.out(&d_out, nout, [&](const double *h) { h_out = h; });
    S.out(&d_count, 1, [&](const double *h) { std::memcpy(&count, h, sizeof(count)); });
    if (int rr = S.upload()) return rr;
    CU_TRY(cudaEventRecord(c->ev0, c->stream));
    if (int rr = launch(d_T, d_C, d_out, d_count)) return rr;
    CU_TRY(cudaEventRecord(c->ev1, c->stream));
    if (int rr = S.download()) return rr;
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
        Staging S(c);
        return eval_host(c, S, N, T, coeffs, cost, gradC, gradT, &isdf_stats::last_pairs,
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
static int callback_batch_launch(isdf_ctx *c, const Layout &L, const double *d_head, const double *d_tail, int bc_stride, double rho,
                                 const double *d_x, double *d_cost, double *d_grad, cudaStream_t st) {
    const int B = L.B;
    const size_t BN = L.P;
    if (int r = minco_fits(L.N)) return r;
    if (BN * (size_t)(c->cfg.integral_intervs + 1) > 0x7fffffffull) return fail(ISDF_ERR_UNSUPPORTED, "batch too large: B*N0*(K+1) must fit in 31 bits");
    if (int r = c->batch.minco.ensure(L)) return r;
    MincoArgs M = c->batch.minco.args(L, d_head, d_tail, bc_stride, rho, d_x);
    M.cost = d_cost; M.grad = d_grad;
    // per-problem obstacle point sets registered for exactly this batch (isdf_set_points_batch): the LIVE composition of costFunctionLmbm
    // (hpp:386-405) — swept-volume term, then time-integral term
    const bool with_swept = (c->sv.B == B);
    if (with_swept) {
        if (c->mesh.shape.kind == ISDF_SHAPE_MESH && c->mesh.shape.mesh.sign_mode == MESH_SIGN_WINDING)
            return fail(ISDF_ERR_UNSUPPORTED, "swept-volume term with a winding-sign mesh (see isdf_set_shape_mesh_ex)");
        CU_TRY(c->batch.d_Cpp.ensure(18 * BN)); CU_TRY(c->batch.d_sv.ensure(19 * BN + B));
        M.Cpp = c->batch.d_Cpp.p;
    }
    const size_t smem = minco_smem_bytes(L.N);
    k_minco_forward<<<B, 32, smem, st>>>(M);
    if (with_swept) {
        int launches = 0;
        cudaError_t e = c->sv.launch_batch(c->dcfg, c->mesh.shape, L.N, L.d_off, BN, M.T, M.Cpp, c->batch.d_sv.p, st, &launches);
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
    c->batch.B = B; c->batch.P = BN;
    CU_TRY(cudaGetLastError());
    return 0;
}

// the batched callback's checks, in order: the batch (ragged: the *_ragged entry points' piece_off; else B problems of N0 pieces) and
// its sizes into *L, the sharding, the evaluation state
static int callback_batch_check(isdf_ctx *c, bool ragged, int B, int N0, const int32_t *piece_off, Layout *L) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (ragged) {
        if (int r = ragged_check(B, piece_off, L)) return r;
    } else {
        if (B < 1 || N0 < 1) return fail(ISDF_ERR_INVALID, "B < 1 or N0 < 1");
        if ((long long)B * N0 > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "B*N0 overflows");
        *L = uniform_layout(B, N0);
    }
    if (c->world != 1) return fail(ISDF_ERR_STATE, "the batched callback shards by PROBLEM: keep isdf_set_shard(ctx, 0, 1) and give each rank its own problems");
    return check_eval_state(c, (int)L->P, true);
}

// the device form of the batched callback on st; a ragged batch's offsets are uploaded first, a uniform batch has none
static int callback_device(isdf_ctx *c, bool ragged, int B, int N0, const int32_t *piece_off, const double *d_head, const double *d_tail,
                           int per_problem_bc, double rho, const double *d_x, double *d_cost, double *d_grad, cudaStream_t st) {
    Layout L;
    if (int r = callback_batch_check(c, ragged, B, N0, piece_off, &L)) return r;
    if (!d_head || !d_tail || !d_x || !d_cost || !d_grad) return fail(ISDF_ERR_INVALID, "NULL device pointer");
    if (set_device(c)) return ISDF_ERR_CUDA;
    if (ragged) if (int r = ragged_upload(c->batch.d_off, piece_off, st, &L)) return r;
    return callback_batch_launch(c, L, d_head, d_tail, per_problem_bc ? 9 : 0, rho, d_x, d_cost, d_grad, st);
}

extern "C" int isdf_callback_batch_device(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc, double rho,
                                          const double *d_x, double *d_cost, double *d_grad, void *cuda_stream) {
    return callback_device(c, false, B, N0, nullptr, d_head, d_tail, per_problem_bc, rho, d_x, d_cost, d_grad, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_callback_batch_ragged_device(isdf_ctx *c, int B, const int32_t *piece_off, const double *d_head, const double *d_tail,
                                                 int per_problem_bc, double rho, const double *d_x, double *d_cost, double *d_grad, void *cuda_stream) {
    return callback_device(c, true, B, 0, piece_off, d_head, d_tail, per_problem_bc, rho, d_x, d_cost, d_grad, (cudaStream_t)cuda_stream);
}

// a checked batch's host inputs shared by the batched host entry points, staged in S: a ragged batch's offsets into *L (as ragged_upload
// lays them out), the boundary conditions (9 doubles, or 9 per problem) at *d_head and *d_tail
static void stage_batch(Staging &S, bool ragged, const int32_t *piece_off, int per_problem_bc, const double *head, const double *tail, Layout *L,
                        const double **d_head, const double **d_tail) {
    const int B = L->B;
    if (ragged) {
        S.in(&L->d_off, piece_off, (size_t)B + 1);
        S.in(&L->d_xoff, (size_t)B + 1, [=](int *h) { for (int b = 0; b <= B; b++) h[b] = 4 * piece_off[b] - 3 * b; });
    }
    const size_t nbc = per_problem_bc ? (size_t)9 * B : 9;
    S.in(d_head, head, nbc); S.in(d_tail, tail, nbc);
}

// the host form of the batched callback: inputs staged, the batch launched on c->stream between ev0 and ev1, results copied back
static int callback_host(isdf_ctx *c, bool ragged, int B, int N0, const int32_t *piece_off, const double *head, const double *tail, int per_problem_bc,
                         double rho, const double *x, double *cost, double *grad) {
    return poison_on_failure([&]() -> int {
        Layout L;
        if (int r = callback_batch_check(c, ragged, B, N0, piece_off, &L)) return r;
        if (!head || !tail || !x || !cost || !grad) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        Staging S(c);
        const double *d_head, *d_tail, *d_x;
        double *d_cost, *d_grad;
        stage_batch(S, ragged, piece_off, per_problem_bc, head, tail, &L, &d_head, &d_tail);
        S.in(&d_x, x, L.X); S.out(&d_cost, cost, (size_t)B); S.out(&d_grad, grad, L.X);
        if (int r = S.upload()) return r;
        CU_TRY(cudaEventRecord(c->ev0, c->stream));
        if (int r = callback_batch_launch(c, L, d_head, d_tail, per_problem_bc ? 9 : 0, rho, d_x, d_cost, d_grad, c->stream)) return r;
        CU_TRY(cudaEventRecord(c->ev1, c->stream));
        if (int r = S.download()) return r;
        float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
        c->stats.last_kernel_ms = ms;
        return 0;
    }, [&] { nan_fill(cost, B); });
}

extern "C" int isdf_callback_batch(isdf_ctx *c, int B, int N0, const double *head, const double *tail, int per_problem_bc, double rho,
                                   const double *x, double *cost, double *grad) {
    return callback_host(c, false, B, N0, nullptr, head, tail, per_problem_bc, rho, x, cost, grad);
}

extern "C" int isdf_callback_batch_ragged(isdf_ctx *c, int B, const int32_t *piece_off, const double *head, const double *tail, int per_problem_bc,
                                          double rho, const double *x, double *cost, double *grad) {
    return callback_host(c, true, B, 0, piece_off, head, tail, per_problem_bc, rho, x, cost, grad);
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
// d_xoff (device, B + 1; may be null): instance b has rows [d_xoff[b], d_xoff[b+1]) of X in all, as a ragged batch's decision vectors; null:
// every instance has n rows, X = B n. Synchronous with respect to the host (one 4-byte read per round decides termination), all data stays
// on the device.
template <typename Eval>
static int lbfgs_rounds(isdf_ctx *c, isdf_ctx::LbfgsBufs &lb, int B, int n, const int *d_xoff, size_t X, const isdf_lbfgs_params *prm, int cancel_after,
                        double *d_x, double *d_f, int *d_ret, int *d_iterations, int *d_evaluations, int *rounds_out, cudaStream_t st, Eval eval) {
    const int m = prm->mem_size, npf = prm->past > 1 ? prm->past : 1;
    const size_t total = 4 * X + (size_t)B * (npf + 2 * (size_t)m + LB_NSCALAR) + 2 * (size_t)m * X;   // doubles of state
    CU_TRY(lb.d_state.ensure(total)); CU_TRY(lb.d_grad.ensure(X)); CU_TRY(lb.d_int.ensure((size_t)B * LB_NINT + 4));
    CU_TRY(lb.h_active.ensure(1));
    CU_TRY(cudaMemsetAsync(lb.d_state.p, 0, sizeof(double) * total, st));
    CU_TRY(cudaMemsetAsync(lb.d_int.p, 0, sizeof(int) * ((size_t)B * LB_NINT + 4), st));   // phase = WANT_INIT
    LbfgsArgs L;
    L.B = B; L.n = n; L.xoff = d_xoff;
    L.pr.mem_size = m; L.pr.past = prm->past; L.pr.max_iterations = prm->max_iterations; L.pr.max_linesearch = prm->max_linesearch;
    L.pr.g_epsilon = prm->g_epsilon; L.pr.delta = prm->delta; L.pr.min_step = prm->min_step; L.pr.max_step = prm->max_step;
    L.pr.f_dec_coeff = prm->f_dec_coeff; L.pr.cautious_factor = prm->cautious_factor; L.pr.machine_prec = prm->machine_prec;
    L.pr.cancel_after = cancel_after;
    double *p = lb.d_state.p;
    L.x = d_x; L.f = d_f; L.grad = lb.d_grad.p;
    L.xp = p; p += X; L.g = p; p += X; L.gp = p; p += X; L.d = p; p += X;
    L.pf = p; p += (size_t)B * npf; L.alpha = p; p += (size_t)B * m; L.ys = p; p += (size_t)B * m;
    L.S = p; p += (size_t)m * X; L.Y = p; p += (size_t)m * X; L.sc = p;
    L.st = lb.d_int.p; L.active = lb.d_int.p + (size_t)B * LB_NINT;
    // olddnorm starts at 1 (lbfgs.hpp:541): scalar slot 2 of every instance
    {
        std::vector<double> init((size_t)B * LB_NSCALAR, 0.0);
        for (int b = 0; b < B; b++) init[(size_t)b * LB_NSCALAR + 2] = 1.0;
        CU_TRY(cudaMemcpyAsync(L.sc, init.data(), sizeof(double) * init.size(), cudaMemcpyHostToDevice, st));
        count_copy(c, cudaMemcpyHostToDevice, sizeof(double) * init.size());
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
        count_copy(c, cudaMemcpyDeviceToHost, sizeof(int), true);
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

// the lock-step L-BFGS over the batched callback of a checked batch on st
static int lbfgs_batch_run(isdf_ctx *c, const Layout &L, const double *d_head, const double *d_tail, int per_problem_bc, double rho,
                           const isdf_lbfgs_params *prm, double *d_x, double *d_f, int *d_ret, int *d_iterations, int *d_evaluations, int *rounds_out,
                           cudaStream_t st) {
    return lbfgs_rounds(c, c->lbfgs, L.B, 4 * L.N - 3, L.d_xoff, L.X, prm, 0, d_x, d_f, d_ret, d_iterations, d_evaluations, rounds_out, st,
                        [&](const double *x, double *f, double *g) {
                            return callback_batch_launch(c, L, d_head, d_tail, per_problem_bc ? 9 : 0, rho, x, f, g, st);
                        });
}

// the device form of the lock-step L-BFGS over the batched callback on st; a ragged batch's offsets are uploaded first
static int lbfgs_device(isdf_ctx *c, bool ragged, int B, int N0, const int32_t *piece_off, const double *d_head, const double *d_tail, int per_problem_bc,
                        double rho, const isdf_lbfgs_params *prm, double *d_x, double *d_f, int *d_ret, int *d_iterations, int *d_evaluations,
                        int *rounds_out, cudaStream_t st) {
    return poison_on_failure([&]() -> int {
        Layout L;
        if (int r = callback_batch_check(c, ragged, B, N0, piece_off, &L)) return r;
        if (int r = lbfgs_check(prm)) return r;
        if (!d_head || !d_tail || !d_x || !d_f) return fail(ISDF_ERR_INVALID, "NULL device pointer");
        if (set_device(c)) return ISDF_ERR_CUDA;
        if (ragged) if (int r = ragged_upload(c->batch.d_off, piece_off, st, &L)) return r;
        return lbfgs_batch_run(c, L, d_head, d_tail, per_problem_bc, rho, prm, d_x, d_f, d_ret, d_iterations, d_evaluations, rounds_out, st);
    }, [&] { nan_fill_device(c, d_f, B, st); });
}

extern "C" int isdf_lbfgs_batch_device(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc, double rho,
                                       const isdf_lbfgs_params *prm, double *d_x, double *d_f, int *d_ret, int *d_iterations, int *d_evaluations,
                                       int *rounds_out, void *cuda_stream) {
    return lbfgs_device(c, false, B, N0, nullptr, d_head, d_tail, per_problem_bc, rho, prm, d_x, d_f, d_ret, d_iterations, d_evaluations, rounds_out,
                        (cudaStream_t)cuda_stream);
}

extern "C" int isdf_lbfgs_batch_ragged_device(isdf_ctx *c, int B, const int32_t *piece_off, const double *d_head, const double *d_tail,
                                              int per_problem_bc, double rho, const isdf_lbfgs_params *prm, double *d_x, double *d_f, int *d_ret,
                                              int *d_iterations, int *d_evaluations, int *rounds_out, void *cuda_stream) {
    return lbfgs_device(c, true, B, 0, piece_off, d_head, d_tail, per_problem_bc, rho, prm, d_x, d_f, d_ret, d_iterations, d_evaluations, rounds_out,
                        (cudaStream_t)cuda_stream);
}

// the host form of the L-BFGS: inputs staged, the rounds on c->stream, results copied back
static int lbfgs_host(isdf_ctx *c, bool ragged, int B, int N0, const int32_t *piece_off, const double *head, const double *tail, int per_problem_bc,
                      double rho, const isdf_lbfgs_params *prm, double *x, double *f, int *ret, int *iterations, int *evaluations, int *rounds_out) {
    return poison_on_failure([&]() -> int {
        Layout L;
        if (int r = callback_batch_check(c, ragged, B, N0, piece_off, &L)) return r;
        if (!head || !tail || !x || !f) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (int r = lbfgs_check(prm)) return r;
        if (set_device(c)) return ISDF_ERR_CUDA;
        Staging S(c);
        const double *d_head, *d_tail;
        double *d_x, *d_f;
        int *d_ret, *d_it, *d_ev;
        stage_batch(S, ragged, piece_off, per_problem_bc, head, tail, &L, &d_head, &d_tail);
        S.inout(&d_x, x, L.X); S.out(&d_f, f, (size_t)B);
        S.out(&d_ret, ret, (size_t)B); S.out(&d_it, iterations, (size_t)B); S.out(&d_ev, evaluations, (size_t)B);
        if (int r = S.upload()) return r;
        if (int r = lbfgs_batch_run(c, L, d_head, d_tail, per_problem_bc, rho, prm, d_x, d_f, d_ret, d_it, d_ev, rounds_out, c->stream)) return r;
        return S.download();
    }, [&] { nan_fill(f, B); });
}

extern "C" int isdf_lbfgs_batch(isdf_ctx *c, int B, int N0, const double *head, const double *tail, int per_problem_bc, double rho,
                                const isdf_lbfgs_params *prm, double *x, double *f, int *ret, int *iterations, int *evaluations, int *rounds_out) {
    return lbfgs_host(c, false, B, N0, nullptr, head, tail, per_problem_bc, rho, prm, x, f, ret, iterations, evaluations, rounds_out);
}

extern "C" int isdf_lbfgs_batch_ragged(isdf_ctx *c, int B, const int32_t *piece_off, const double *head, const double *tail, int per_problem_bc,
                                       double rho, const isdf_lbfgs_params *prm, double *x, double *f, int *ret, int *iterations, int *evaluations,
                                       int *rounds_out) {
    return lbfgs_host(c, true, B, 0, piece_off, head, tail, per_problem_bc, rho, prm, x, f, ret, iterations, evaluations, rounds_out);
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
    Staging S(c);
    double *d_xs, *d_fs;
    int *d_ret, *d_it, *d_ev;
    S.inout(&d_xs, x, bn); S.out(&d_fs, f, (size_t)B);
    S.out(&d_ret, ret, (size_t)B); S.out(&d_it, iterations, (size_t)B); S.out(&d_ev, evaluations, (size_t)B);
    if (int r = S.upload()) return r;
    std::vector<double> hx(bn), hf(B), hg(bn);   // the rounds' points and the objective's results
    int r = lbfgs_rounds(c, c->lbfgs, B, n, nullptr, bn, prm, cancel_after, d_xs, d_fs, d_ret, d_it, d_ev, rounds_out, c->stream,
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
    return S.download();
}

extern "C" int isdf_get_batch_trajectories(isdf_ctx *c, double *T, double *coeffs, double *energy) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (c->batch.B <= 0) return fail(ISDF_ERR_STATE, "no batched callback evaluated yet");
    if (int r = sync_ctx(c)) return r;
    const size_t BN = c->batch.P;
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
    if (int r = offsets_check(path_off, B, "path_off", false)) return r;
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

// isdf_path_waypoints on the device (isdf_plan.cuh), on stream st: counts and pieces, wp_off by a scan, then the rows below cap. *total
// (may be null: nothing is read) gets wp_off[B], one 4-byte read.
static int waypoints_run(isdf_ctx *c, int B, const int32_t *d_path_off, const double *d_xyz, double res, double parlength, long long cap,
                         double *d_wp, int32_t *d_wp_off, int32_t *d_pieces, int *total, cudaStream_t st) {
    auto &z = c->wps;
    CU_TRY(z.d_cnt.ensure(B)); CU_TRY(z.d_gap.ensure(B));
    size_t tmp = 0;
    CU_TRY(cub::DeviceScan::InclusiveSum(nullptr, tmp, z.d_cnt.p, d_wp_off + 1, B, st));
    CU_TRY(z.d_tmp.ensure(std::max<size_t>(tmp, 1)));
    k_wp_count<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(B, d_path_off, res, parlength, z.d_cnt.p, z.d_gap.p, d_pieces, d_wp_off);
    CU_TRY(cub::DeviceScan::InclusiveSum(z.d_tmp.p, tmp, z.d_cnt.p, d_wp_off + 1, B, st));
    if (cap > 0) k_wp_write<<<(unsigned)(((long long)B * 32 + 127) / 128), 128, 0, st>>>(B, d_path_off, d_xyz, z.d_gap.p, d_wp_off, cap, d_wp);
    c->stats.kernel_launches += cap > 0 ? 3 : 2;
    CU_TRY(cudaGetLastError());
    if (total) {
        CU_TRY(z.h_total.ensure(1));
        CU_TRY(cudaMemcpyAsync(z.h_total.p, d_wp_off + B, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        count_copy(c, cudaMemcpyDeviceToHost, sizeof(int32_t));
        CU_TRY(cudaStreamSynchronize(st));
        *total = *z.h_total.p;
    }
    return 0;
}

extern "C" int isdf_path_waypoints_device(isdf_ctx *c, int B, const int32_t *d_path_off, const double *d_path_xyz, double res, double parlength,
                                          int cap, double *d_waypoints, int32_t *d_wp_off, int32_t *d_pieces, void *cuda_stream) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (B < 1 || !d_path_off || !d_path_xyz || !d_wp_off || !d_pieces || cap < 0 || (cap > 0 && !d_waypoints))
        return fail(ISDF_ERR_INVALID, "NULL argument, B < 1 or cap < 0");
    if (!(std::isfinite(res) && res > 0.0) || !(std::isfinite(parlength) && parlength > 0.0)) return fail(ISDF_ERR_INVALID, "res and parlength must be finite and positive");
    if (set_device(c)) return ISDF_ERR_CUDA;
    int total = 0;
    if (int r = waypoints_run(c, B, d_path_off, d_path_xyz, res, parlength, cap, d_waypoints, d_wp_off, d_pieces, &total, (cudaStream_t)cuda_stream)) return r;
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

// the mid-end parameters' checks, in the order of midend_check
static int midend_params_check(const isdf_midend_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (p->reserved_ != 0) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    if (!(std::isfinite(p->weight_pr) && p->weight_pr >= 0.0) || !std::isfinite(p->rho) || !(std::isfinite(p->init_time) && p->init_time > 0.0) ||
        p->cancel_after < 0)
        return fail(ISDF_ERR_INVALID, "mid-end parameter out of range");
    return lbfgs_check(&p->lbfgs);
}

// the mid-end's checks, in order: the batch (ragged: the *_ragged entry points' piece_off; else B problems of N0 pieces) and its sizes
// into *L, the parameters, the shared-memory solver, the sharding
static int midend_check(isdf_ctx *c, bool ragged, int B, int N0, const int32_t *piece_off, const isdf_midend_params *p, Layout *L) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (ragged) {
        if (int r = ragged_check(B, piece_off, L)) return r;
    } else {
        if (B < 1 || N0 < 1) return fail(ISDF_ERR_INVALID, "B < 1 or N0 < 1");
        if ((long long)B * (4 * (long long)N0 - 3) > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "B*(4*N0-3) overflows");
        *L = uniform_layout(B, N0);
    }
    if (int r = midend_params_check(p)) return r;
    if (int r = minco_fits(L->N)) return r;
    if (c->world != 1) return fail(ISDF_ERR_STATE, "the mid-end shards by PROBLEM: keep isdf_set_shard(ctx, 0, 1) and give each rank its own problems");
    return 0;
}

static int midend_buffers(isdf_ctx *c, const Layout &L) {
    if (int r = c->mid.minco.ensure(L)) return r;
    CU_TRY(c->mid.d_pc.ensure(L.P));
    return 0;
}

static MincoArgs midend_minco_args(isdf_ctx *c, const Layout &L, const double *d_head, const double *d_tail, int bc_stride, double rho, const double *d_x) {
    MincoArgs M = c->mid.minco.args(L, d_head, d_tail, bc_stride, rho, d_x);
    M.disc_out = c->mid.minco.d_out.p; M.piece_cost = c->mid.d_pc.p; M.seq_terms = 1;
    return M;
}

// one evaluation of OriTraj::costFunction for all B problems: MINCO forward -> pose term -> adjoint with the terms added one at a time
static int midend_eval_launch(isdf_ctx *c, const Layout &L, const double *d_head, const double *d_tail, int bc_stride, const isdf_midend_params *p,
                              const double *d_wp, const double *d_x, double *d_cost, double *d_grad, cudaStream_t st) {
    const int B = L.B;
    const size_t BN = L.P, smem = minco_smem_bytes(L.N);
    MincoArgs M = midend_minco_args(c, L, d_head, d_tail, bc_stride, p->rho, d_x);
    M.cost = d_cost; M.grad = d_grad;
    k_minco_forward<<<B, 32, smem, st>>>(M);
    MidendArgs P;
    P.B = B; P.N = L.N; P.P = (int)BN; P.poff = L.d_off; P.K = c->cfg.integral_intervs; P.weight = p->weight_pr; P.T = M.T; P.C = M.C; P.wp = d_wp; P.out = c->mid.minco.d_out.p; P.piece_cost = c->mid.d_pc.p;
    k_midend_pose<<<(unsigned)((BN + 127) / 128), 128, 0, st>>>(P);
    k_minco_backward<<<B, 32, smem, st>>>(M);
    c->stats.kernel_launches += 3;
    CU_TRY(cudaGetLastError());
    return 0;
}

// the host form of one mid-end evaluation: inputs staged (the waypoints, 3 per inner piece, after the batch's), results copied back
static int midend_callback_host(isdf_ctx *c, bool ragged, int B, int N0, const int32_t *piece_off, const double *head, const double *tail,
                                int per_problem_bc, const isdf_midend_params *p, const double *waypoints, const double *x, double *cost, double *grad) {
    return poison_on_failure([&]() -> int {
        Layout L;
        if (int r = midend_check(c, ragged, B, N0, piece_off, p, &L)) return r;
        if (!head || !tail || !x || !cost || !grad || (L.P > (size_t)B && !waypoints)) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        Staging S(c);
        const double *d_head, *d_tail, *d_wp, *d_x;
        double *d_cost, *d_grad;
        stage_batch(S, ragged, piece_off, per_problem_bc, head, tail, &L, &d_head, &d_tail);
        S.in(&d_wp, waypoints, 3 * (L.P - B)); S.in(&d_x, x, L.X);
        S.out(&d_cost, cost, (size_t)B); S.out(&d_grad, grad, L.X);
        if (int r = S.upload()) return r;
        if (int r = midend_buffers(c, L)) return r;
        if (int r = midend_eval_launch(c, L, d_head, d_tail, per_problem_bc ? 9 : 0, p, d_wp, d_x, d_cost, d_grad, c->stream)) return r;
        return S.download();
    }, [&] { nan_fill(cost, B); });
}

extern "C" int isdf_midend_callback_batch(isdf_ctx *c, int B, int N0, const double *head, const double *tail, int per_problem_bc,
                                          const isdf_midend_params *p, const double *waypoints, const double *x, double *cost, double *grad) {
    return midend_callback_host(c, false, B, N0, nullptr, head, tail, per_problem_bc, p, waypoints, x, cost, grad);
}

extern "C" int isdf_midend_callback_batch_ragged(isdf_ctx *c, int B, const int32_t *piece_off, const double *head, const double *tail,
                                                 int per_problem_bc, const isdf_midend_params *p, const double *waypoints, const double *x,
                                                 double *cost, double *grad) {
    return midend_callback_host(c, true, B, 0, piece_off, head, tail, per_problem_bc, p, waypoints, x, cost, grad);
}

static int midend_batch_run(isdf_ctx *c, const Layout &L, const double *d_head, const double *d_tail, int per_problem_bc, const isdf_midend_params *p,
                            const double *d_wp, double *d_x, double *d_T, double *d_coeffs, double *d_f, int *d_ret, int *d_iterations,
                            int *d_evaluations, int *rounds_out, cudaStream_t st) {
    if (set_device(c)) return ISDF_ERR_CUDA;
    const int B = L.B, n = 4 * L.N - 3;
    const size_t BN = L.P;
    if (int r = midend_buffers(c, L)) return r;
    // x = [backwardT(init_time) | waypoints] (mid_end.cpp:21-36; backwardT as back_end_optimizer.hpp:243-256)
    const double T0 = p->init_time, tau0 = T0 > 1.0 ? (std::sqrt(2.0 * T0 - 1.0) - 1.0) : (1.0 - std::sqrt(2.0 / T0 - 1.0));
    k_midend_init<<<(unsigned)((L.X + 127) / 128), 128, 0, st>>>(B, L.N, L.d_off, L.d_xoff, (long long)L.X, tau0, d_wp, d_x);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    const int bc_stride = per_problem_bc ? 9 : 0;
    int r = lbfgs_rounds(c, c->mid.lb, B, n, L.d_xoff, L.X, &p->lbfgs, p->cancel_after, d_x, d_f, d_ret, d_iterations, d_evaluations, rounds_out, st,
                         [&](const double *x, double *f, double *g) { return midend_eval_launch(c, L, d_head, d_tail, bc_stride, p, d_wp, x, f, g, st); });
    if (r) return r;
    // the final trajectories: forwardT + MINCO of the returned x (mid_end.cpp:65-71 / 79-85)
    if (d_T || d_coeffs) {
        MincoArgs M = midend_minco_args(c, L, d_head, d_tail, bc_stride, p->rho, d_x);
        k_minco_forward<<<B, 32, minco_smem_bytes(L.N), st>>>(M);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        if (d_T) CU_TRY(cudaMemcpyAsync(d_T, M.T, sizeof(double) * BN, cudaMemcpyDeviceToDevice, st));
        if (d_coeffs) CU_TRY(cudaMemcpyAsync(d_coeffs, M.C, sizeof(double) * 18 * BN, cudaMemcpyDeviceToDevice, st));
        CU_TRY(cudaStreamSynchronize(st));
    }
    return 0;
}

// the device form of getOriTraj on st; a ragged batch's offsets are uploaded first
static int midend_device(isdf_ctx *c, bool ragged, int B, int N0, const int32_t *piece_off, const double *d_head, const double *d_tail, int per_problem_bc,
                         const isdf_midend_params *p, const double *d_waypoints, double *d_x, double *d_T, double *d_coeffs, double *d_f, int32_t *d_ret,
                         int32_t *d_iterations, int32_t *d_evaluations, int32_t *rounds, cudaStream_t st) {
    return poison_on_failure([&]() -> int {
        Layout L;
        if (int r = midend_check(c, ragged, B, N0, piece_off, p, &L)) return r;
        if (!d_head || !d_tail || !d_x || !d_f || (L.P > (size_t)B && !d_waypoints)) return fail(ISDF_ERR_INVALID, "NULL device pointer");
        if (set_device(c)) return ISDF_ERR_CUDA;
        if (ragged) if (int r = ragged_upload(c->mid.d_off, piece_off, st, &L)) return r;
        return midend_batch_run(c, L, d_head, d_tail, per_problem_bc, p, d_waypoints, d_x, d_T, d_coeffs, d_f, d_ret, d_iterations, d_evaluations, rounds, st);
    }, [&] { nan_fill_device(c, d_f, B, st); });
}

extern "C" int isdf_midend_batch_device(isdf_ctx *c, int B, int N0, const double *d_head, const double *d_tail, int per_problem_bc,
                                        const isdf_midend_params *p, const double *d_waypoints, double *d_x, double *d_T, double *d_coeffs,
                                        double *d_f, int32_t *d_ret, int32_t *d_iterations, int32_t *d_evaluations, int32_t *rounds, void *cuda_stream) {
    return midend_device(c, false, B, N0, nullptr, d_head, d_tail, per_problem_bc, p, d_waypoints, d_x, d_T, d_coeffs, d_f, d_ret, d_iterations,
                         d_evaluations, rounds, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_midend_batch_ragged_device(isdf_ctx *c, int B, const int32_t *piece_off, const double *d_head, const double *d_tail,
                                               int per_problem_bc, const isdf_midend_params *p, const double *d_waypoints, double *d_x, double *d_T,
                                               double *d_coeffs, double *d_f, int32_t *d_ret, int32_t *d_iterations, int32_t *d_evaluations,
                                               int32_t *rounds, void *cuda_stream) {
    return midend_device(c, true, B, 0, piece_off, d_head, d_tail, per_problem_bc, p, d_waypoints, d_x, d_T, d_coeffs, d_f, d_ret, d_iterations,
                         d_evaluations, rounds, (cudaStream_t)cuda_stream);
}

// the host form of getOriTraj: inputs staged, results copied back; the final trajectories are computed also when T and coeffs are NULL
static int midend_host(isdf_ctx *c, bool ragged, int B, int N0, const int32_t *piece_off, const double *head, const double *tail, int per_problem_bc,
                       const isdf_midend_params *p, const double *waypoints, double *x, double *T, double *coeffs, double *f, int32_t *ret,
                       int32_t *iterations, int32_t *evaluations, int32_t *rounds) {
    return poison_on_failure([&]() -> int {
        Layout L;
        if (int r = midend_check(c, ragged, B, N0, piece_off, p, &L)) return r;
        if (!head || !tail || !x || !f || (L.P > (size_t)B && !waypoints)) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        Staging S(c);
        const double *d_head, *d_tail, *d_wp;
        double *d_x, *d_f, *d_T, *d_C;
        int *d_ret, *d_it, *d_ev;
        stage_batch(S, ragged, piece_off, per_problem_bc, head, tail, &L, &d_head, &d_tail);
        S.in(&d_wp, waypoints, 3 * (L.P - B));
        S.out(&d_x, x, L.X); S.out(&d_T, T, L.P); S.out(&d_C, coeffs, 18 * L.P); S.out(&d_f, f, (size_t)B);   // x starts on the device
        S.out(&d_ret, ret, (size_t)B); S.out(&d_it, iterations, (size_t)B); S.out(&d_ev, evaluations, (size_t)B);
        if (int r = S.upload()) return r;
        if (int r = midend_batch_run(c, L, d_head, d_tail, per_problem_bc, p, d_wp, d_x, d_T, d_C, d_f, d_ret, d_it, d_ev, rounds, c->stream)) return r;
        return S.download();
    }, [&] { nan_fill(f, B); });
}

extern "C" int isdf_midend_batch(isdf_ctx *c, int B, int N0, const double *head, const double *tail, int per_problem_bc,
                                 const isdf_midend_params *p, const double *waypoints, double *x, double *T, double *coeffs,
                                 double *f, int32_t *ret, int32_t *iterations, int32_t *evaluations, int32_t *rounds) {
    return midend_host(c, false, B, N0, nullptr, head, tail, per_problem_bc, p, waypoints, x, T, coeffs, f, ret, iterations, evaluations, rounds);
}

extern "C" int isdf_midend_batch_ragged(isdf_ctx *c, int B, const int32_t *piece_off, const double *head, const double *tail, int per_problem_bc,
                                        const isdf_midend_params *p, const double *waypoints, double *x, double *T, double *coeffs,
                                        double *f, int32_t *ret, int32_t *iterations, int32_t *evaluations, int32_t *rounds) {
    return midend_host(c, true, B, 0, piece_off, head, tail, per_problem_bc, p, waypoints, x, T, coeffs, f, ret, iterations, evaluations, rounds);
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

// number of groups (trajectories, pose groups) of N pieces or poses with N0 per group, N0 = 0 for one group (0 when N / N0 define none)
static int traj_batch(int64_t N, int64_t N0) {
    if (N < 1 || N0 < 0) return 0;
    if (N0 == 0) return 1;
    return (N % N0 == 0) ? (int)(N / N0) : 0;
}

// a clearance scan's reach and margin
static int reach_margin_check(double reach, double margin) {
    if (!(reach > 0.0) || !std::isfinite(reach)) return fail(ISDF_ERR_INVALID, "reach must be positive and finite");
    if (std::isnan(margin) || margin > reach) return fail(ISDF_ERR_INVALID, "margin must not exceed reach");
    return 0;
}

// a clearance scan's scene: an unsharded context, the map and the shape set, and the window of every `what` ("sample", "pose") within
// the 1023-voxel limit
static int clearance_scene_check(const isdf_ctx *c, double reach, const char *what) {
    if (c->world > 1) return fail(ISDF_ERR_UNSUPPORTED, "the clearance check is not sharded: call it on a context with isdf_set_shard(ctx, 0, 1)");
    if (!c->map.have_map) return fail(ISDF_ERR_STATE, "map not set");
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    // the window spans at most 2 H sqrt(3) / res + 3 voxels per axis (rotated H box, one voxel of slack on each side); the 1023-voxel
    // limit of the pose-window offsets applies as in the discrete path
    const double H = c->dcfg.half_bd + reach;
    if (2.0 * H * std::sqrt(3.0) / c->map.grid.res + 4.0 > (double)WINDOW_AXIS_MAX)
        return fail(ISDF_ERR_INVALID, std::string("reach too large for this map resolution: a ") + what + " window would exceed 1023 voxels per axis");
    return 0;
}

// every check that needs no device work, in the order of include/isdf.h's error list
static int clearance_check(isdf_ctx *c, int N, const isdf_clearance_params *p) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (N < 1) return fail(ISDF_ERR_INVALID, "N < 1");
    if (p->samples_per_piece < 1) return fail(ISDF_ERR_INVALID, "samples_per_piece < 1");
    if (int r = reach_margin_check(p->reach, p->margin)) return r;
    if (traj_batch(N, p->pieces_per_traj) == 0) return fail(ISDF_ERR_INVALID, "pieces_per_traj must be 0 or divide N");
    if ((long long)N * (p->samples_per_piece + 1) > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "N * (samples_per_piece + 1) must fit in 31 bits");
    return clearance_scene_check(c, p->reach, "sample");
}

// the clearance scan of N sources in groups of N0 (0: one group) with reach and margin: the K + 1 uniform samples of each piece of
// (d_T, d_C), or, with K = 0, poses the caller sets; outputs, cursor, counters, hit flags and sample list are the caller's
// (clearance_grid_ready has run on the call's stream)
static ClrArgs clearance_args(const isdf_ctx *c, int N, int K, int N0, double reach, double margin, const double *d_T = nullptr,
                              const double *d_C = nullptr) {
    ClrArgs A = {};
    A.grid = c->known.policy == ISDF_UNKNOWN_OCCUPIED ? c->known.blocked : c->map.grid; A.shape = c->mesh.shape; A.fp = c->dcfg.fp; A.half_bd = c->dcfg.half_bd;
    A.reach = reach; A.margin = margin;
    A.N = N; A.K = K; A.N0 = N0 == 0 ? N : N0;
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

// one clearance check on st: the cursor and counters reset, then the scan and summary kernels over n samples
static int clearance_scan(isdf_ctx *c, ClrArgs &A, long long n, cudaStream_t st) {
    CU_TRY(c->clr.d_cursor.ensure(1)); CU_TRY(c->clr.d_counters.ensure(2));
    CU_TRY(cudaMemsetAsync(c->clr.d_cursor.p, 0, sizeof(int), st));
    CU_TRY(cudaMemsetAsync(c->clr.d_counters.p, 0, 2 * sizeof(unsigned long long), st));
    A.cursor = c->clr.d_cursor.p; A.counters = c->clr.d_counters.p;
    CU_TRY(clearance_launch(A, clearance_mode(c), clearance_grid(c, n), st));
    c->stats.kernel_launches += 2;   // scan kernel, summary kernel
    return 0;
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
        if (int r = clearance_grid_ready(c, st)) return r;
        // no sample list, no hit flags: the uniform samples of the definition
        ClrArgs A = clearance_args(c, N, p->samples_per_piece, p->pieces_per_traj, p->reach, p->margin, d_T, d_coeffs);
        A.clear = d_sample_clearance; A.voxel = (long long *)d_sample_voxel; A.summary = (ClrSummary *)d_summary;
        return clearance_scan(c, A, (long long)N * (A.K + 1), st);
    }, [&] { if (c) write_failed_summaries(d_summary, p ? traj_batch(N, p->pieces_per_traj) : 0, clearance_failed_summary(), c, st); });
}

extern "C" int isdf_trajectory_clearance(isdf_ctx *c, int N, const double *T, const double *coeffs, const isdf_clearance_params *p,
                                         double *sample_clearance, int64_t *sample_voxel, isdf_clearance_summary *summary) {
    return poison_on_failure([&]() -> int {
        if (int r = clearance_check(c, N, p)) return r;
        if (!T || !coeffs || !summary) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        const size_t S = (size_t)N * (p->samples_per_piece + 1);
        Staging St(c);
        const double *d_C, *d_T;
        double *d_clear;
        int64_t *d_vox;
        isdf_clearance_summary *d_sum;
        St.in(&d_C, coeffs, 18 * (size_t)N); St.in(&d_T, T, (size_t)N);
        St.out(&d_sum, summary, (size_t)traj_batch(N, p->pieces_per_traj)); St.out(&d_clear, sample_clearance, S); St.out(&d_vox, sample_voxel, S);
        if (int r = St.upload()) return r;
        if (int r = isdf_trajectory_clearance_device(c, N, d_T, d_C, p, d_clear, d_vox, d_sum, c->stream)) return r;
        return St.download();
    }, [&] { write_failed_summaries(summary, p ? traj_batch(N, p->pieces_per_traj) : 0, clearance_failed_summary()); });
}

// ---- clearance at caller-given poses (the pose source of k_clearance_scan) ----
extern "C" int isdf_pose_clearance_default_params(isdf_pose_clearance_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    isdf_config d;
    isdf_default_config(&d);
    p->reach = d.safety_hor; p->margin = d.safety_hor; p->poses_per_group = 0; p->reserved_ = 0;
    return 0;
}

static int pose_clearance_check(isdf_ctx *c, int64_t Q, const void *pos, const void *quat, int64_t stride, const isdf_pose_clearance_params *p) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!p || !pos || !quat) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (Q < 1 || Q > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "Q must be in [1, 2^31)");
    if (stride < 1) return fail(ISDF_ERR_INVALID, "stride_doubles < 1");
    if (int r = reach_margin_check(p->reach, p->margin)) return r;
    if (traj_batch(Q, p->poses_per_group) == 0) return fail(ISDF_ERR_INVALID, "poses_per_group must be 0 or divide Q");
    if (p->reserved_ != 0) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    return clearance_scene_check(c, p->reach, "pose");
}

extern "C" int isdf_pose_clearance_device(isdf_ctx *c, int64_t Q, const double *d_pos, const double *d_quat, int64_t stride,
                                          const isdf_pose_clearance_params *p, double *d_clear, int64_t *d_voxel, isdf_clearance_summary *d_summary,
                                          void *cuda_stream) {
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    return poison_on_failure([&]() -> int {
        if (int r = pose_clearance_check(c, Q, d_pos, d_quat, stride, p)) return r;
        if (!d_clear || !d_voxel || !d_summary) return fail(ISDF_ERR_INVALID, "NULL device pointer");
        if (set_device(c)) return ISDF_ERR_CUDA;
        if (int r = clearance_grid_ready(c, st)) return r;
        ClrArgs A = clearance_args(c, (int)Q, 0, p->poses_per_group, p->reach, p->margin);   // one "sample" per pose
        A.ppos = d_pos; A.pquat = d_quat; A.pstride = stride;
        A.clear = d_clear; A.voxel = (long long *)d_voxel; A.summary = (ClrSummary *)d_summary;
        return clearance_scan(c, A, Q, st);
    }, [&] { if (c) write_failed_summaries(d_summary, p ? traj_batch(Q, p->poses_per_group) : 0, clearance_failed_summary(), c, st); });
}

extern "C" int isdf_pose_clearance(isdf_ctx *c, int64_t Q, const double *pos, const double *quat, int64_t stride, const isdf_pose_clearance_params *p,
                                   double *clear, int64_t *voxel, isdf_clearance_summary *summary) {
    return poison_on_failure([&]() -> int {
        if (int r = pose_clearance_check(c, Q, pos, quat, stride, p)) return r;
        if (!summary) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        Staging S(c);
        const double *d_pose;
        double *d_clear;
        int64_t *d_vox;
        isdf_clearance_summary *d_sum;
        stage_poses(S, Q, pos, quat, stride, &d_pose);
        S.out(&d_sum, summary, (size_t)traj_batch(Q, p->poses_per_group)); S.out(&d_clear, clear, (size_t)Q); S.out(&d_vox, voxel, (size_t)Q);
        if (int r = S.upload()) return r;
        if (int r = isdf_pose_clearance_device(c, Q, d_pose, d_pose + 3, 7, p, d_clear, d_vox, d_sum, c->stream)) return r;
        return S.download();
    }, [&] { write_failed_summaries(summary, p ? traj_batch(Q, p->poses_per_group) : 0, clearance_failed_summary()); });
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

// the shapes whose SDF is a signed Euclidean distance (include/isdf.h): Ball, Point, Box with an orthonormal rotation, exact-sign meshes.
// `who` prefixes the messages. *r_rot: the radius about the body origin that rotation moves (0 for rotation-invariant bodies);
// *r_body: the body's bounding radius about its origin; both padded against the rounding of their own computation. pts / npts: the
// points whose norms give them (Box corners, mesh AABB corners), for the caller's own conditions on the body's extent.
static int distance_shape(isdf_ctx *c, const char *who, double *r_rot, double *r_body, double pts[8][3], int *npts) {
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    const DevShape &s = c->mesh.shape;
    const std::string w(who);
    double rr = 0.0, rb = 0.0;
    *npts = 0;
    if (s.kind == ISDF_SHAPE_BALL) {
        rb = std::max(s.par[0], 0.0);
    } else if (s.kind == ISDF_SHAPE_BOX) {
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                const double d = s.rot[3 * i] * s.rot[3 * j] + s.rot[3 * i + 1] * s.rot[3 * j + 1] + s.rot[3 * i + 2] * s.rot[3 * j + 2];
                if (!(std::fabs(d - (i == j ? 1.0 : 0.0)) <= 1e-12)) return fail(ISDF_ERR_UNSUPPORTED, w + ": the Box rotation is not orthonormal to 1e-12");
            }
        if (!(s.par[0] >= 0.0 && s.par[1] >= 0.0 && s.par[2] >= 0.0)) return fail(ISDF_ERR_UNSUPPORTED, w + ": negative Box half extents");
        for (int k = 0; k < 8; k++) {   // body point of shape-frame corner q: Rotate q + trans (shape_pre inverted)
            const double q[3] = {(k & 1) ? s.par[0] : -s.par[0], (k & 2) ? s.par[1] : -s.par[1], (k & 4) ? s.par[2] : -s.par[2]};
            for (int j = 0; j < 3; j++) pts[k][j] = s.rot[3 * j] * q[0] + s.rot[3 * j + 1] * q[1] + s.rot[3 * j + 2] * q[2] + s.trans[j];
        }
        *npts = 8;
    } else if (s.kind == ISDF_SHAPE_MESH) {
        if (s.mesh.sign_mode != MESH_SIGN_PSEUDONORMAL) return fail(ISDF_ERR_UNSUPPORTED, w + ": a winding-sign mesh SDF is not a distance");
        for (int k = 0; k < 8; k++) {
            pts[k][0] = (k & 1) ? s.mesh.bhi[0] : s.mesh.blo[0]; pts[k][1] = (k & 2) ? s.mesh.bhi[1] : s.mesh.blo[1]; pts[k][2] = (k & 4) ? s.mesh.bhi[2] : s.mesh.blo[2];
        }
        *npts = 8;
    } else if (s.kind != ISDF_SHAPE_POINT) {
        return fail(ISDF_ERR_UNSUPPORTED, w + ": supported shapes are Ball, Point, Box and exact-sign meshes (their SDF is a distance)");
    }
    for (int k = 0; k < *npts; k++) rr = std::max(rr, std::sqrt(pts[k][0] * pts[k][0] + pts[k][1] * pts[k][1] + pts[k][2] * pts[k][2]));
    if (*npts) rb = rr;
    *r_rot = rr * (1.0 + 1e-12);
    *r_body = rb * (1.0 + 1e-12);
    return 0;
}

// the shape conditions of the certificate (include/isdf.h): a true Euclidean distance outside the body and a body inside the half_bd box.
// *r: the body radius about the body origin (0 for rotation-invariant bodies), padded against the rounding of its own computation
static int certify_shape(isdf_ctx *c, double *r) {
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    const DevShape &s = c->mesh.shape;
    const double hb = c->dcfg.half_bd;
    if (s.kind == ISDF_SHAPE_BALL && !(s.par[0] >= 0.0 && s.par[0] <= hb)) return fail(ISDF_ERR_UNSUPPORTED, "certificate: the Ball's radius must lie in [0, half_bd]");
    double pts[8][3], rb = 0.0;
    int npts = 0;
    if (int rc = distance_shape(c, "certificate", r, &rb, pts, &npts)) return rc;
    for (int k = 0; k < npts; k++)
        if (!(std::fabs(pts[k][0]) <= hb && std::fabs(pts[k][1]) <= hb && std::fabs(pts[k][2]) <= hb))
            return fail(ISDF_ERR_UNSUPPORTED, s.kind == ISDF_SHAPE_BOX ? "certificate: the Box reaches beyond the half_bd box"
                                                                     : "certificate: the mesh's bounding box reaches beyond the half_bd box");
    return 0;
}

static int certify_batch(int N, const isdf_certify_params *p) { return p ? traj_batch(N, p->clearance.pieces_per_traj) : 0; }

// the refinement's parameters, each checked where its certificate's error list puts it; the size check needs valid N, K and B
static int refine_param_check(int max_depth, int max_samples) {
    if (max_depth < 0 || max_depth > 64) return fail(ISDF_ERR_INVALID, "max_depth must lie in [0, 64]");
    if (max_samples < 0) return fail(ISDF_ERR_INVALID, "max_samples_per_traj < 0");
    return 0;
}
static int refine_size_check(long long N, long long K, long long B, int max_samples) {
    return N * (2 * K + 1) + 3 * B * max_samples > 0x7fffffffll ? fail(ISDF_ERR_INVALID, "N (2 K + 1) + 3 B max_samples_per_traj must fit in 31 bits") : 0;
}

// every check that needs no device work; *r as certify_shape
static int certify_check(isdf_ctx *c, int N, const isdf_certify_params *p, double *r) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (p->reserved_[0] || p->reserved_[1]) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    if (int rr = refine_param_check(p->max_depth, p->max_samples_per_traj)) return rr;
    const isdf_clearance_params &q = p->clearance;
    if (!(q.margin >= 0.0) || !(q.margin < q.reach)) return fail(ISDF_ERR_INVALID, "the certificate needs 0 <= margin < reach");
    if (int rr = clearance_check(c, N, &q)) return rr;
    if (int rr = refine_size_check(N, q.samples_per_piece, certify_batch(N, p), p->max_samples_per_traj)) return rr;
    return certify_shape(c, r);
}

static CertArgs certify_args(isdf_ctx *c, double r, double reach, int N, const double *d_T, const double *d_C) {
    CertArgs A = {};
    A.fp = c->dcfg.fp; A.r = r; A.H = c->dcfg.half_bd + reach;
    A.N = N; A.T = d_T; A.C = d_C;
    return A;
}

// the rounds of a certificate after its init kernel, from the I0 initial intervals in z.d_iv[0] and the S0 initial samples: per round,
// launch() runs decide + emit over the A.nact intervals A.cur with one record per interval in scr (A.*a_scr), one 4-byte read gives
// the round's splits ns, and after(nact, ns) sees them with the new samples at A.S_cur. Stops when no interval splits.
template <class Args, class Scr, class After>
static int refine_rounds(isdf_ctx *c, RefineBufs &z, Args &A, long long S0, long long I0, DevBuf<Scr> &scr, Scr *Args::*a_scr,
                         cudaError_t (*launch)(const Args &, cudaStream_t), After after, cudaStream_t st) {
    long long nact = I0, S_cur = S0;
    int cur = 0;
    for (;;) {
        CU_TRY(z.d_iv[cur ^ 1].ensure((size_t)std::max(2 * nact, 1ll))); CU_TRY(scr.ensure((size_t)nact));
        A.cur = z.d_iv[cur].p; A.next = z.d_iv[cur ^ 1].p; A.*a_scr = scr.p;
        A.S_cur = (int)S_cur; A.nact = (int)nact;
        CU_TRY(launch(A, st));
        c->stats.kernel_launches += 2;
        CU_TRY(cudaMemcpyAsync(z.h_tot.p, z.d_tot.p, sizeof(int), cudaMemcpyDeviceToHost, st));
        count_copy(c, cudaMemcpyDeviceToHost, sizeof(int), true);
        CU_TRY(cudaStreamSynchronize(st));
        const long long ns = *z.h_tot.p;
        if (int rr = after(nact, ns)) return rr;
        if (ns == 0) return 0;
        S_cur += ns; nact = 2 * ns; cur ^= 1;
    }
}

static int certify_run(isdf_ctx *c, int N, const double *d_T, const double *d_C, const isdf_certify_params *p, double r, CertSummary *d_sum,
                       cudaStream_t st) {
    auto &z = c->cert;
    const isdf_clearance_params &q = p->clearance;
    const int K = q.samples_per_piece, N0 = q.pieces_per_traj == 0 ? N : q.pieces_per_traj, B = N / N0, M = p->max_samples_per_traj;
    const size_t S0 = (size_t)N * (K + 1), I0 = (size_t)N * K, Smax = S0 + (size_t)B * M, Lmax = I0 + (size_t)B * M;
    z.last_leaves = 0;
    CertArgs A = certify_args(c, r, q.reach, N, d_T, d_C);
    if (int rr = z.ref.ensure(A, N, I0)) return rr;
    CU_TRY(z.d_sp.ensure(Smax)); CU_TRY(z.d_st.ensure(Smax)); CU_TRY(z.d_sc.ensure(Smax)); CU_TRY(z.d_sv.ensure(Smax));
    CU_TRY(z.d_hit.ensure(B)); CU_TRY(z.d_traj.ensure(B)); CU_TRY(z.d_cursor.ensure(1)); CU_TRY(z.d_leaves.ensure(Lmax));
    A.margin = q.margin; A.K = K; A.N0 = N0; A.B = B; A.max_depth = p->max_depth; A.max_samples = M;
    A.sp = z.d_sp.p; A.st = z.d_st.p; A.sc = z.d_sc.p; A.sv = z.d_sv.p; A.hit = z.d_hit.p;
    A.leaves = z.d_leaves.p; A.traj = z.d_traj.p; A.summary = d_sum;
    CU_TRY(certify_init_launch(A, st));
    c->stats.kernel_launches++;
    // the scan: round 0 is the clearance check's own uniform samples, later rounds the new midpoints
    if (int rr = clearance_grid_ready(c, st)) return rr;
    ClrArgs S = clearance_args(c, N, K, q.pieces_per_traj, q.reach, q.margin, d_T, d_C);   // no counters: a certificate leaves isdf_dbg_clearance_counts as it was
    S.clear = z.d_sc.p; S.voxel = z.d_sv.p; S.cursor = z.d_cursor.p; S.hit = z.d_hit.p;
    auto scan = [&](long long n) -> int {
        CU_TRY(cudaMemsetAsync(z.d_cursor.p, 0, sizeof(int), st));
        CU_TRY(clearance_scan_launch(S, clearance_mode(c), clearance_grid(c, n), st));
        c->stats.kernel_launches++;
        return 0;
    };
    if (int rr = scan((long long)S0)) return rr;
    auto after = [&](long long nact, long long ns) -> int {   // the leaf cursor, and the scan of the new midpoints
        A.L_cur += (int)(nact - ns);
        if (ns == 0) return 0;
        S.st = z.d_st.p + A.S_cur; S.sp = z.d_sp.p + A.S_cur; S.nlist = (int)ns; S.clear = z.d_sc.p + A.S_cur; S.voxel = z.d_sv.p + A.S_cur;
        return scan(ns);
    };
    if (int rr = refine_rounds(c, z.ref, A, (long long)S0, (long long)I0, z.d_scr, &CertArgs::scr, certify_round_launch, after, st)) return rr;
    CU_TRY(certify_finish_launch(A, st));
    c->stats.kernel_launches++;
    z.last_leaves = A.L_cur;
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

// the host form of a certificate over its device form: check(), the trajectory block in and B summaries out through the staging; on
// failure max(B, 1) summaries read `bad`
template <class S, class P, class Check>
static int certificate_host(isdf_ctx *c, int N, const double *T, const double *coeffs, const P *p, S *summary, int B, const S &bad, Check check,
                            int (*device)(isdf_ctx *, int, const double *, const double *, const P *, S *, void *)) {
    return poison_on_failure([&]() -> int {
        if (int rc = check()) return rc;
        if (!T || !coeffs || !summary) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (set_device(c)) return ISDF_ERR_CUDA;
        Staging St(c);
        const double *d_C, *d_T;
        S *d_sum;
        St.in(&d_C, coeffs, 18 * (size_t)N); St.in(&d_T, T, (size_t)N); St.out(&d_sum, summary, (size_t)B);
        if (int rc = St.upload()) return rc;
        if (int rc = device(c, N, d_T, d_C, p, d_sum, c->stream)) return rc;
        return St.download();
    }, [&] { write_failed_summaries(summary, B, bad); });
}

extern "C" int isdf_trajectory_certify(isdf_ctx *c, int N, const double *T, const double *coeffs, const isdf_certify_params *p,
                                       isdf_certify_summary *summary) {
    double r = 0.0;
    return certificate_host(c, N, T, coeffs, p, summary, certify_batch(N, p), certify_failed_summary(), [&] { return certify_check(c, N, p, &r); },
                            isdf_trajectory_certify_device);
}

// ---- dynamic-limit certificate (isdf_dynlimits.cuh) -------------------------------------------------------------------------------
extern "C" int isdf_dynamics_default_params(isdf_ctx *c, isdf_dynamics_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    isdf_config d;
    isdf_default_config(&d);
    const isdf_config &g = c ? c->cfg : d;
    std::memset(p, 0, sizeof(*p));
    const double inf = std::numeric_limits<double>::infinity();
    p->samples_per_piece = g.integral_intervs; p->pieces_per_traj = 0;
    p->max_depth = 16; p->max_samples_per_traj = 2048;
    p->vmax = g.vmax; p->amax = inf; p->omgmax = g.omgmax; p->thetamax = g.thetamax; p->thrust_min = -inf; p->thrust_max = inf;
    p->tol_v = 1e-3; p->tol_a = 1e-3; p->tol_omg = 1e-3; p->tol_theta = 1e-4; p->tol_thrust = 1e-3;
    return 0;
}

static_assert(sizeof(isdf_dynamics_summary) == sizeof(DynSummary) && offsetof(isdf_dynamics_summary, thrust_lower) == offsetof(DynSummary, thrust_lower) &&
              offsetof(isdf_dynamics_summary, verdict) == offsetof(DynSummary, verdict) && offsetof(isdf_dynamics_summary, depth) == offsetof(DynSummary, depth),
              "isdf_dynamics_summary layout");

static int dynamics_batch(int N, const isdf_dynamics_params *p) { return p ? traj_batch(N, p->pieces_per_traj) : 0; }

// every check that needs no device work, in the order of include/isdf.h's error list
static int dynamics_check(isdf_ctx *c, int N, const isdf_dynamics_params *p) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (N < 1) return fail(ISDF_ERR_INVALID, "N < 1");
    if (p->samples_per_piece < 1) return fail(ISDF_ERR_INVALID, "samples_per_piece < 1");
    if (dynamics_batch(N, p) == 0) return fail(ISDF_ERR_INVALID, "pieces_per_traj must be 0 or divide N");
    if (int rr = refine_param_check(p->max_depth, p->max_samples_per_traj)) return rr;
    for (double t : {p->tol_v, p->tol_a, p->tol_omg, p->tol_theta, p->tol_thrust})
        if (!(t >= 0.0)) return fail(ISDF_ERR_INVALID, "tolerances must be >= 0 (+inf: verdict only)");
    for (double l : {p->vmax, p->amax, p->omgmax, p->thetamax, p->thrust_min, p->thrust_max})
        if (std::isnan(l)) return fail(ISDF_ERR_INVALID, "a limit is NaN");
    if (p->thrust_min > p->thrust_max) return fail(ISDF_ERR_INVALID, "thrust_min > thrust_max");
    if (p->reserved_[0] || p->reserved_[1]) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    if (int rr = refine_size_check(N, p->samples_per_piece, dynamics_batch(N, p), p->max_samples_per_traj)) return rr;
    if (c->world > 1) return fail(ISDF_ERR_UNSUPPORTED, "the dynamic-limit certificate is not sharded: call it on a context with isdf_set_shard(ctx, 0, 1)");
    return 0;
}

static int dynamics_run(isdf_ctx *c, int N, const double *d_T, const double *d_C, const isdf_dynamics_params *p, DynSummary *d_sum,
                        cudaStream_t st) {
    auto &z = c->dyn;
    const int K = p->samples_per_piece, N0 = p->pieces_per_traj == 0 ? N : p->pieces_per_traj, B = N / N0, M = p->max_samples_per_traj;
    const size_t S0 = (size_t)N * (K + 1), I0 = (size_t)N * K, Smax = S0 + (size_t)B * M;
    DynArgs A = {};
    if (int rr = z.ref.ensure(A, N, I0)) return rr;
    CU_TRY(z.d_smp.ensure(Smax)); CU_TRY(z.d_traj.ensure(B));
    A.fp = c->dcfg.fp; A.mass = c->cfg.vehicle_mass; A.dv = c->cfg.vert_drag;
    const double lim[DYN_CH] = {p->vmax, p->amax, p->omgmax, p->thetamax, p->thrust_max, -p->thrust_min};
    const double tol[DYN_CH] = {p->tol_v, p->tol_a, p->tol_omg, p->tol_theta, p->tol_thrust, p->tol_thrust};
    for (int q = 0; q < DYN_CH; q++) { A.lim[q] = lim[q]; A.tol[q] = tol[q]; }
    A.N = N; A.K = K; A.N0 = N0; A.B = B; A.max_depth = p->max_depth; A.max_samples = M;
    A.T = d_T; A.C = d_C; A.smp = z.d_smp.p; A.traj = z.d_traj.p; A.summary = d_sum;
    CU_TRY(dyn_init_launch(A, st));
    c->stats.kernel_launches++;
    auto no_after = [](long long, long long) { return 0; };   // nothing between rounds: the midpoints are evaluated by k_dyn_emit
    if (int rr = refine_rounds(c, z.ref, A, (long long)S0, (long long)I0, z.d_dec, &DynArgs::dec, dyn_round_launch, no_after, st)) return rr;
    CU_TRY(dyn_finish_launch(A, st));
    c->stats.kernel_launches++;
    return 0;
}

// on failure every summary reads verdict 0 (UNDECIDED), every bound and time NaN, masks 0, counts -1
static isdf_dynamics_summary dynamics_failed_summary() {
    isdf_dynamics_summary s;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    for (int q = 0; q < 5; q++) s.upper[q] = s.attained[q] = s.t_attained[q] = nan;
    s.thrust_lower = s.thrust_attained_min = s.t_thrust_attained_min = nan;
    s.verdict = 0; s.violated = s.undecided = 0; s.samples = s.undecided_intervals = s.depth = -1;
    return s;
}

extern "C" int isdf_trajectory_dynamics_device(isdf_ctx *c, int N, const double *d_T, const double *d_coeffs, const isdf_dynamics_params *p,
                                               isdf_dynamics_summary *d_summary, void *cuda_stream) {
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    return poison_on_failure([&]() -> int {
        if (int rc = dynamics_check(c, N, p)) return rc;
        if (!d_T || !d_coeffs || !d_summary) return fail(ISDF_ERR_INVALID, "NULL device pointer");
        if (set_device(c)) return ISDF_ERR_CUDA;
        return dynamics_run(c, N, d_T, d_coeffs, p, (DynSummary *)d_summary, st);
    }, [&] { if (c) write_failed_summaries(d_summary, dynamics_batch(N, p), dynamics_failed_summary(), c, st); });
}

extern "C" int isdf_trajectory_dynamics(isdf_ctx *c, int N, const double *T, const double *coeffs, const isdf_dynamics_params *p,
                                        isdf_dynamics_summary *summary) {
    return certificate_host(c, N, T, coeffs, p, summary, dynamics_batch(N, p), dynamics_failed_summary(), [&] { return dynamics_check(c, N, p); },
                            isdf_trajectory_dynamics_device);
}

// a public struct as the device struct of the same layout
template <typename D, typename S>
static D same_layout(const S &s) {
    static_assert(sizeof(D) == sizeof(S), "layouts differ");
    D d;
    std::memcpy(&d, &s, sizeof(D));
    return d;
}

// ---- braking to a certified stop (isdf_brake.cuh) ----------------------------------------------------------------------------------
static_assert(sizeof(isdf_brake_summary) == sizeof(BrakeSummary) && offsetof(isdf_brake_summary, certify) == offsetof(BrakeSummary, cert) &&
              offsetof(isdf_brake_summary, dynamics) == offsetof(BrakeSummary, dyn) && offsetof(isdf_brake_summary, certified) == offsetof(BrakeSummary, certified),
              "isdf_brake_summary layout");

extern "C" int isdf_brake_default_params(isdf_ctx *c, isdf_brake_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    std::memset(p, 0, sizeof(*p));
    p->candidates = 8; p->pieces = 4;
    isdf_certify_default_params(&p->certify);
    isdf_dynamics_default_params(c, &p->dynamics);
    return 0;
}

// every check that needs no device work, in the order of include/isdf.h's error list; *pc / *pd: the certificates' parameters with N0 = M,
// *r as certify_shape
static int brake_check(isdf_ctx *c, int B, const isdf_brake_params *p, isdf_certify_params *pc, isdf_dynamics_params *pd, double *r) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (B < 1) return fail(ISDF_ERR_INVALID, "B < 1");
    if (p->candidates < 1) return fail(ISDF_ERR_INVALID, "candidates < 1");
    if (p->pieces < 1 || p->pieces > ISDF_BRAKE_MAX_PIECES) return fail(ISDF_ERR_INVALID, "pieces must lie in [1, ISDF_BRAKE_MAX_PIECES]");
    if (p->reserved_[0] || p->reserved_[1]) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    if (p->certify.clearance.pieces_per_traj != 0) return fail(ISDF_ERR_INVALID, "certify.clearance.pieces_per_traj must be 0 (the call sets M)");
    if (p->dynamics.pieces_per_traj != 0) return fail(ISDF_ERR_INVALID, "dynamics.pieces_per_traj must be 0 (the call sets M)");
    const long long n = (long long)B * p->candidates * p->pieces;
    if (n > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "B * candidates * pieces must fit in 31 bits");
    *pc = p->certify; pc->clearance.pieces_per_traj = p->pieces;
    *pd = p->dynamics; pd->pieces_per_traj = p->pieces;
    if (int rc = certify_check(c, (int)n, pc, r)) return rc;
    return dynamics_check(c, (int)n, pd);
}

// the brake on st (include/isdf.h): setup, MINCO, both certificates over the B K candidates, select, scan, write
static int brake_run(isdf_ctx *c, int B, const int *d_off, const double *d_T, const double *d_C, const double *d_ts, const isdf_brake_params *p,
                     const isdf_certify_params &pc, const isdf_dynamics_params &pd, double r, int *d_out_off, double *d_out_T, double *d_out_C,
                     BrakeSummary *d_sum, cudaStream_t st) {
    auto &z = c->brake;
    const int K = p->candidates, M = p->pieces, Q = B * K, n = Q * M;
    const Layout L = uniform_layout(Q, M);
    if (int rc = z.minco.ensure(L)) return rc;
    CU_TRY(z.d_head.ensure(9 * (size_t)Q)); CU_TRY(z.d_tail.ensure(9 * (size_t)Q)); CU_TRY(z.d_Tin.ensure((size_t)n)); CU_TRY(z.d_x.ensure(L.X));
    CU_TRY(z.d_csum.ensure(Q)); CU_TRY(z.d_dsum.ensure(Q)); CU_TRY(z.d_cnt.ensure(B)); CU_TRY(z.d_pick.ensure(B));
    size_t tmp = 0;
    CU_TRY(cub::DeviceScan::InclusiveSum(nullptr, tmp, z.d_cnt.p, d_out_off + 1, B, st));
    CU_TRY(z.d_tmp.ensure(std::max<size_t>(tmp, 1)));
    const double *bm = c->map.grid.bmin;
    k_brake_setup<<<(unsigned)((Q + 127) / 128), 128, 0, st>>>(B, K, M, d_off, d_T, d_C, d_ts, bm[0], bm[1], bm[2], z.d_head.p, z.d_tail.p, z.d_Tin.p, z.d_x.p);
    MincoArgs A = z.minco.args(L, z.d_head.p, z.d_tail.p, 9, 0.0, z.d_x.p);
    A.T_in = z.d_Tin.p;
    k_minco_forward<<<Q, 32, minco_smem_bytes(M), st>>>(A);
    c->stats.kernel_launches += 2;
    CU_TRY(cudaGetLastError());
    if (int rc = certify_run(c, n, A.T, A.C, &pc, r, z.d_csum.p, st)) return rc;
    if (int rc = dynamics_run(c, n, A.T, A.C, &pd, z.d_dsum.p, st)) return rc;
    const CertSummary cbad = same_layout<CertSummary>(certify_failed_summary());
    const DynSummary dbad = same_layout<DynSummary>(dynamics_failed_summary());
    k_brake_select<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(B, K, M, d_off, d_T, d_ts, A.T, z.d_csum.p, z.d_dsum.p, cbad, dbad, d_sum, z.d_cnt.p,
                                                                z.d_pick.p, d_out_off);
    CU_TRY(cub::DeviceScan::InclusiveSum(z.d_tmp.p, tmp, z.d_cnt.p, d_out_off + 1, B, st));
    k_brake_write<<<(unsigned)(((long long)B * 32 + 127) / 128), 128, 0, st>>>(B, K, M, z.d_pick.p, A.T, A.C, d_out_off, d_out_T, d_out_C);
    c->stats.kernel_launches += 3;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaStreamSynchronize(st));
    return 0;
}

// on failure every summary reads status NONE, candidate -1, NaN times, counts -1 and the certificates' failed-call summaries
static isdf_brake_summary brake_failed_summary() {
    isdf_brake_summary s;
    s.status = ISDF_BRAKE_NONE; s.candidate = -1;
    s.tau_stop = s.duration = std::numeric_limits<double>::quiet_NaN();
    s.certified = s.feasible = -1;
    s.certify = certify_failed_summary(); s.dynamics = dynamics_failed_summary();
    return s;
}

extern "C" int isdf_trajectory_brake(isdf_ctx *c, int B, const int32_t *piece_off, const double *T, const double *coeffs, const double *t_stop_max,
                                     const isdf_brake_params *p, int32_t *out_piece_off, double *out_T, double *out_coeffs, isdf_brake_summary *summary) {
    return poison_on_failure([&]() -> int {
        isdf_certify_params pc; isdf_dynamics_params pd; double r = 0.0;
        if (!c || !piece_off || !T || !coeffs || !t_stop_max || !out_piece_off || !out_T || !out_coeffs || !summary) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (int rc = brake_check(c, B, p, &pc, &pd, &r)) return rc;
        if (int rc = offsets_check(piece_off, B, "piece_off", true)) return rc;
        const int P = piece_off[B];
        if (int rc = swept_traj_check(P, T, coeffs)) return rc;
        if (set_device(c)) return ISDF_ERR_CUDA;
        const size_t cap = (size_t)B * p->pieces;
        Staging S(c);
        const double *d_C, *d_T, *d_ts;
        const int *d_off;
        int *d_out_off;
        double *d_out_T, *d_out_C;
        isdf_brake_summary *d_sum;
        S.in(&d_C, coeffs, 18 * (size_t)P); S.in(&d_T, T, (size_t)P); S.in(&d_ts, t_stop_max, (size_t)B); S.in(&d_off, piece_off, (size_t)B + 1);
        S.out(&d_sum, summary, (size_t)B); S.out(&d_out_off, out_piece_off, (size_t)B + 1);
        S.out(&d_out_T, out_T, cap); S.out(&d_out_C, out_coeffs, 18 * cap);
        if (int rc = S.upload()) return rc;
        if (int rc = brake_run(c, B, d_off, d_T, d_C, d_ts, p, pc, pd, r, d_out_off, d_out_T, d_out_C, (BrakeSummary *)d_sum, c->stream)) return rc;
        return S.download();
    }, [&] { if (B >= 1) write_failed_summaries(summary, B, brake_failed_summary()); });
}

extern "C" int isdf_trajectory_brake_device(isdf_ctx *c, int B, const int32_t *d_piece_off, const double *d_T, const double *d_coeffs,
                                            const double *d_t_stop_max, const isdf_brake_params *p, int32_t *d_out_piece_off, double *d_out_T,
                                            double *d_out_coeffs, isdf_brake_summary *d_summary, void *cuda_stream) {
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    return poison_on_failure([&]() -> int {
        isdf_certify_params pc; isdf_dynamics_params pd; double r = 0.0;
        if (!c || !d_piece_off || !d_T || !d_coeffs || !d_t_stop_max || !d_out_piece_off || !d_out_T || !d_out_coeffs || !d_summary)
            return fail(ISDF_ERR_INVALID, "NULL argument");
        if (int rc = brake_check(c, B, p, &pc, &pd, &r)) return rc;
        if (set_device(c)) return ISDF_ERR_CUDA;
        return brake_run(c, B, d_piece_off, d_T, d_coeffs, d_t_stop_max, p, pc, pd, r, d_out_piece_off, d_out_T, d_out_coeffs, (BrakeSummary *)d_summary, st);
    }, [&] { if (c && B >= 1) write_failed_summaries(d_summary, B, brake_failed_summary(), c, st); });
}

// ---- certified swept volume (isdf_sweptvol.cuh) ------------------------------------------------------------------------------------
extern "C" int isdf_swept_default_params(isdf_swept_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    std::memset(p, 0, sizeof(*p));
    isdf_config d;
    isdf_default_config(&d);
    p->samples_per_piece = d.integral_intervs;
    p->max_depth = 16; p->max_samples_per_point = 512;
    p->tol = d.occupancy_resolution / 100.0;
    p->band = 2.0 * d.safety_hor;
    return 0;
}

// every check that needs no device work and no trajectory, in the order of include/isdf.h's error list; *r_rot / *r_body as distance_shape
static int swept_check(isdf_ctx *c, int N, const isdf_swept_params *p, double *r_rot, double *r_body) {
    if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    if (N < 1) return fail(ISDF_ERR_INVALID, "N < 1");
    if (p->reserved_) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    if (p->samples_per_piece < 1) return fail(ISDF_ERR_INVALID, "samples_per_piece < 1");
    if (!(p->tol > 0.0) || !std::isfinite(p->tol)) return fail(ISDF_ERR_INVALID, "tol must be positive and finite");
    if (!(p->band > p->tol) || !std::isfinite(p->band)) return fail(ISDF_ERR_INVALID, "band must be finite and larger than tol");
    if (p->max_depth < 0 || p->max_depth > 64) return fail(ISDF_ERR_INVALID, "max_depth must lie in [0, 64]");
    if (p->max_samples_per_point < 0) return fail(ISDF_ERR_INVALID, "max_samples_per_point < 0");
    if ((long long)N * (p->samples_per_piece + 1) > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "N * (samples_per_piece + 1) must fit in 31 bits");
    if (c->world > 1) return fail(ISDF_ERR_UNSUPPORTED, "the swept volume is not sharded: call it on a context with isdf_set_shard(ctx, 0, 1)");
    double pts[8][3];
    int npts = 0;
    if (int rc = distance_shape(c, "swept volume", r_rot, r_body, pts, &npts)) return rc;
    if (c->mesh.shape.kind == ISDF_SHAPE_BALL && !(c->mesh.shape.par[0] >= 0.0))
        return fail(ISDF_ERR_UNSUPPORTED, "swept volume: the Ball's radius must not be negative");
    return 0;
}

static long long swept_nodes(const isdf_swept_grid *g) { return g ? (long long)g->X * g->Y * g->Z : 0; }

static int swept_grid_check(const isdf_swept_grid *g) {
    if (!g) return fail(ISDF_ERR_INVALID, "grid is NULL");
    if (g->reserved_) return fail(ISDF_ERR_INVALID, "grid reserved_ must be 0");
    if (!(g->res > 0.0) || !std::isfinite(g->res)) return fail(ISDF_ERR_INVALID, "grid res must be positive and finite");
    if (g->X < 2 || g->Y < 2 || g->Z < 2) return fail(ISDF_ERR_INVALID, "grid sizes must be >= 2");
    if (swept_nodes(g) >= 0x80000000ll) return fail(ISDF_ERR_INVALID, "X * Y * Z must be < 2^31");
    const int n[3] = {g->X, g->Y, g->Z};
    for (int a = 0; a < 3; a++)
        if (!std::isfinite(g->bmin[a]) || !std::isfinite(g->bmin[a] + (double)(n[a] - 1) * g->res)) return fail(ISDF_ERR_INVALID, "grid coordinates must be finite");
    return 0;
}

// the trajectory (host copies): durations finite and positive, coefficients finite
static int swept_traj_check(int N, const double *T, const double *coeffs) {
    for (int i = 0; i < N; i++) if (!(T[i] > 0.0) || !std::isfinite(T[i])) return fail(ISDF_ERR_INVALID, "every T must be positive and finite");
    for (long long i = 0; i < 18ll * N; i++) if (!std::isfinite(coeffs[i])) return fail(ISDF_ERR_INVALID, "coeffs must be finite");
    return 0;
}
// the same checks on a device trajectory (one copy of 19 N doubles to the host)
static int swept_traj_check_device(isdf_ctx *c, int N, const double *d_T, const double *d_coeffs, cudaStream_t st) {
    std::vector<double> h((size_t)19 * N);
    CU_TRY(cudaMemcpyAsync(h.data(), d_coeffs, sizeof(double) * 18 * N, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaMemcpyAsync(h.data() + 18 * (size_t)N, d_T, sizeof(double) * N, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    (void)c;
    return swept_traj_check(N, h.data() + 18 * (size_t)N, h.data());
}

// the field at the nodes of g (or at npts points d_pts when g is null) into device arrays; info (may be null) gets the counters and times
static int swept_run(isdf_ctx *c, int N, const double *d_T, const double *d_C, const isdf_swept_params *p, double r_rot, double r_body,
                     const isdf_swept_grid *g, int npts, const double *d_pts, double *d_val, double *d_low, double *d_ts, uint8_t *d_dec,
                     isdf_swept_info *info, cudaStream_t st) {
    auto &z = c->svol;
    const int K = p->samples_per_piece, M = p->max_samples_per_point;
    const long long NK = (long long)N * K, S = (long long)N * (K + 1);
    CU_TRY(z.d_toff.ensure(N)); CU_TRY(z.d_pose.ensure((size_t)(12 * S))); CU_TRY(z.d_Dab.ensure((size_t)(2 * NK)));
    CU_TRY(z.d_cursor.ensure(1)); CU_TRY(z.d_counters.ensure(4)); CU_TRY(z.h_n.ensure(1));
    if (info) for (cudaEvent_t &e : z.ev) if (!e) CU_TRY(cudaEventCreate(&e));
    SvolArgs A = {};
    A.shape = c->mesh.shape; A.fp = c->dcfg.fp; A.r_rot = r_rot; A.r_body = r_body; A.band = p->band; A.tol = p->tol;
    A.N = N; A.K = K; A.max_depth = p->max_depth; A.max_samples = M; A.T = d_T; A.C = d_C;
    A.toff = z.d_toff.p; A.pose = z.d_pose.p; A.Dab = z.d_Dab.p;
    A.value = d_val; A.lower = d_low; A.tstar = d_ts; A.decided = d_dec;
    A.cursor = z.d_cursor.p; A.counters = z.d_counters.p;
    if (info) CU_TRY(cudaEventRecord(z.ev[0], st));
    CU_TRY(cudaMemsetAsync(z.d_counters.p, 0, 4 * sizeof(unsigned long long), st));
    CU_TRY(sv_prep_launch(A, st));
    c->stats.kernel_launches++;
    if (info) CU_TRY(cudaEventRecord(z.ev[1], st));
    long long nitems = npts, nbricks = 0;
    if (g) {
        for (int a = 0; a < 3; a++) A.bmin[a] = g->bmin[a];
        A.res = g->res; A.X = g->X; A.Y = g->Y; A.Z = g->Z;
        A.BX = (g->X + SV_BRICK - 1) / SV_BRICK; A.BY = (g->Y + SV_BRICK - 1) / SV_BRICK; A.BZ = (g->Z + SV_BRICK - 1) / SV_BRICK;
        nbricks = (long long)A.BX * A.BY * A.BZ;
        CU_TRY(z.d_boff.ensure((size_t)nbricks + 1)); CU_TRY(z.d_bsum.ensure((size_t)(nbricks + SV_SCAN_THREADS) / SV_SCAN_THREADS + 1));
        A.boff = z.d_boff.p;
        CU_TRY(sv_bricks_launch(A, (int)nbricks, false, st));
        CU_TRY(sv_scan_launch(z.d_boff.p, nbricks, z.d_bsum.p, st));
        c->stats.kernel_launches += 4;   // count pass, three scan kernels
        CU_TRY(cudaMemcpyAsync(z.h_n.p, z.d_boff.p + nbricks, sizeof(long long), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
        CU_TRY(z.d_blist.ensure((size_t)std::max(*z.h_n.p, 1ll)));
        A.blist = z.d_blist.p;
        CU_TRY(sv_bricks_launch(A, (int)nbricks, true, st));
        c->stats.kernel_launches++;
        nitems = nbricks;
    } else {
        A.pts = d_pts; A.npts = npts;
    }
    if (info) CU_TRY(cudaEventRecord(z.ev[2], st));
    if (nitems > 0) {
        if (!z.refine_blocks) { CU_TRY(sv_refine_resident_blocks(&z.refine_blocks)); z.refine_blocks = std::max(z.refine_blocks, 1); }
        // each resident warp owns two interval lists: round 0's kept intervals (at most N K) and children (at most 2 M) per round
        A.split_at = std::max(NK, 2ll * M);
        A.scap = A.split_at + 2ll * M;
        const long long want = (nitems + SV_WARPS - 1) / SV_WARPS;
        const unsigned grid = (unsigned)std::max<long long>(1, std::min(want, (long long)c->sm_count * std::min(z.refine_blocks, 2)));
        A.nwarps = (int)grid * SV_WARPS;
        CU_TRY(z.d_scratch.ensure((size_t)(A.nwarps * A.scap)));
        A.scratch = z.d_scratch.p;
        CU_TRY(cudaMemsetAsync(z.d_cursor.p, 0, sizeof(int), st));
        CU_TRY(sv_refine_launch(A, c->mesh.shape.kind == ISDF_SHAPE_MESH ? 1 : 0, (int)nitems, grid, st));
        c->stats.kernel_launches++;
    }
    if (info) {
        CU_TRY(cudaEventRecord(z.ev[3], st));
        unsigned long long cnt[4];
        CU_TRY(cudaMemcpyAsync(cnt, z.d_counters.p, sizeof(cnt), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
        std::memset(info, 0, sizeof(*info));
        info->nodes = g ? swept_nodes(g) : npts;
        info->bricks = nbricks; info->bricks_culled = g ? (long long)cnt[3] : 0;
        info->sdf_evals = (long long)cnt[0]; info->undecided = (long long)cnt[1]; info->deepest = (int)cnt[2];
        float ms = 0.f;
        CU_TRY(cudaEventElapsedTime(&ms, z.ev[0], z.ev[1])); info->prep_ms = ms;
        CU_TRY(cudaEventElapsedTime(&ms, z.ev[1], z.ev[2])); info->cull_ms = ms;
        CU_TRY(cudaEventElapsedTime(&ms, z.ev[2], z.ev[3])); info->refine_ms = ms;
    }
    return 0;
}

static void swept_poison_host(long long n, double *value, double *lower, double *tstar, uint8_t *decided) {
    nan_fill(value, n); nan_fill(lower, n); nan_fill(tstar, n);
    if (decided && n > 0) std::memset(decided, 0, (size_t)n);
}

extern "C" int isdf_swept_volume_sdf(isdf_ctx *c, int N, const double *T, const double *coeffs, const isdf_swept_params *p, int n,
                                     const double *pts, double *value, double *lower, double *tstar, uint8_t *decided) {
    return poison_on_failure([&]() -> int {
        double r_rot = 0.0, r_body = 0.0;
        if (int rc = swept_check(c, N, p, &r_rot, &r_body)) return rc;
        if (!T || !coeffs || !value || (n > 0 && !pts)) return fail(ISDF_ERR_INVALID, "NULL argument");
        if (n < 0) return fail(ISDF_ERR_INVALID, "n < 0");
        if (int rc = swept_traj_check(N, T, coeffs)) return rc;
        for (long long i = 0; i < 3ll * n; i++) if (!std::isfinite(pts[i])) return fail(ISDF_ERR_INVALID, "points must be finite");
        if (n == 0) return 0;
        if (set_device(c)) return ISDF_ERR_CUDA;
        Staging S(c);
        const double *d_C, *d_T, *d_pts;
        double *d_val, *d_low, *d_ts;
        uint8_t *d_dec;
        S.in(&d_C, coeffs, 18 * (size_t)N); S.in(&d_T, T, (size_t)N); S.in(&d_pts, pts, (size_t)3 * n);
        S.out(&d_val, value, (size_t)n); S.out(&d_low, lower, (size_t)n); S.out(&d_ts, tstar, (size_t)n); S.out(&d_dec, decided, (size_t)n);
        if (int rc = S.upload()) return rc;
        if (int rc = swept_run(c, N, d_T, d_C, p, r_rot, r_body, nullptr, n, d_pts, d_val, d_low, d_ts, d_dec, nullptr, c->stream)) return rc;
        return S.download();
    }, [&] { swept_poison_host(std::max(n, 0), value, lower, tstar, decided); });
}

extern "C" int isdf_swept_volume_grid_device(isdf_ctx *c, int N, const double *d_T, const double *d_coeffs, const isdf_swept_params *p,
                                             const isdf_swept_grid *g, double *d_value, double *d_lower, double *d_tstar, uint8_t *d_decided,
                                             isdf_swept_info *info, void *cuda_stream) {
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    return poison_on_failure([&]() -> int {
        double r_rot = 0.0, r_body = 0.0;
        if (int rc = swept_check(c, N, p, &r_rot, &r_body)) return rc;
        if (int rc = swept_grid_check(g)) return rc;
        if (!d_T || !d_coeffs || !d_value) return fail(ISDF_ERR_INVALID, "NULL device pointer");
        if (set_device(c)) return ISDF_ERR_CUDA;
        if (int rc = swept_traj_check_device(c, N, d_T, d_coeffs, st)) return rc;
        return swept_run(c, N, d_T, d_coeffs, p, r_rot, r_body, g, 0, nullptr, d_value, d_lower, d_tstar, d_decided, info, st);
    }, [&] {
        const long long n = swept_nodes(g) > 0 && swept_nodes(g) < 0x80000000ll ? swept_nodes(g) : 0;
        nan_fill_device(c, d_value, (int)n, st); nan_fill_device(c, d_lower, (int)n, st); nan_fill_device(c, d_tstar, (int)n, st);
        if (c && d_decided && n > 0 && cudaSetDevice(c->device) == cudaSuccess) { cudaMemsetAsync(d_decided, 0, (size_t)n, st); cudaStreamSynchronize(st); }
    });
}

// the field of g in the context's buffers (the host grid and mesh entries)
static int swept_grid_ctx(isdf_ctx *c, int N, const double *T, const double *coeffs, const isdf_swept_params *p, const isdf_swept_grid *g,
                          isdf_swept_info *info) {
    double r_rot = 0.0, r_body = 0.0;
    if (int rc = swept_check(c, N, p, &r_rot, &r_body)) return rc;
    if (int rc = swept_grid_check(g)) return rc;
    if (!T || !coeffs) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (int rc = swept_traj_check(N, T, coeffs)) return rc;
    if (set_device(c)) return ISDF_ERR_CUDA;
    auto &z = c->svol;
    const size_t n = (size_t)swept_nodes(g);
    Staging S(c);
    const double *d_C, *d_T;
    S.in(&d_C, coeffs, 18 * (size_t)N); S.in(&d_T, T, (size_t)N);
    if (int rc = S.upload()) return rc;
    CU_TRY(z.d_val.ensure(n)); CU_TRY(z.d_low.ensure(n)); CU_TRY(z.d_ts.ensure(n)); CU_TRY(z.d_dec.ensure(n));
    return swept_run(c, N, d_T, d_C, p, r_rot, r_body, g, 0, nullptr, z.d_val.p, z.d_low.p, z.d_ts.p, z.d_dec.p, info, c->stream);
}

extern "C" int isdf_swept_volume_grid(isdf_ctx *c, int N, const double *T, const double *coeffs, const isdf_swept_params *p,
                                      const isdf_swept_grid *g, double *value, double *lower, double *tstar, uint8_t *decided,
                                      isdf_swept_info *info) {
    return poison_on_failure([&]() -> int {
        if (c && !value) return fail(ISDF_ERR_INVALID, "value is NULL");
        if (int rc = swept_grid_ctx(c, N, T, coeffs, p, g, info)) return rc;
        if (!value) return fail(ISDF_ERR_INVALID, "value is NULL");
        auto &z = c->svol;
        const size_t n = (size_t)swept_nodes(g);
        CU_TRY(cudaMemcpyAsync(value, z.d_val.p, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
        if (lower) CU_TRY(cudaMemcpyAsync(lower, z.d_low.p, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
        if (tstar) CU_TRY(cudaMemcpyAsync(tstar, z.d_ts.p, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
        if (decided) CU_TRY(cudaMemcpyAsync(decided, z.d_dec.p, n, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(cudaStreamSynchronize(c->stream));
        return 0;
    }, [&] {
        const long long n = swept_nodes(g) > 0 && swept_nodes(g) < 0x80000000ll ? swept_nodes(g) : 0;
        swept_poison_host(n, value, lower, tstar, decided);
    });
}

extern "C" int isdf_swept_volume_mesh(isdf_ctx *c, int N, const double *T, const double *coeffs, const isdf_swept_params *p,
                                      const isdf_swept_grid *g, int64_t cap_v, int64_t cap_f, double *V, double *vtime, int32_t *F,
                                      int64_t *nV, int64_t *nF, isdf_swept_info *info) {
    return poison_on_failure([&]() -> int {
        if (c && (!nV || !nF)) return fail(ISDF_ERR_INVALID, "nV / nF is NULL");
        if (c && (cap_v < 0 || cap_f < 0)) return fail(ISDF_ERR_INVALID, "cap_v / cap_f < 0");
        if (c && ((cap_v > 0 && (!V || !vtime)) || (cap_f > 0 && !F))) return fail(ISDF_ERR_INVALID, "NULL output with a positive cap");
        if (int rc = swept_grid_ctx(c, N, T, coeffs, p, g, info)) return rc;
        if (!nV || !nF) return fail(ISDF_ERR_INVALID, "nV / nF is NULL");
        auto &z = c->svol;
        const cudaStream_t st = c->stream;
        const long long n = swept_nodes(g);
        if (info) CU_TRY(cudaEventRecord(z.ev[3], st));
        CU_TRY(z.d_mask.ensure((size_t)n)); CU_TRY(z.d_voff.ensure((size_t)n + 1)); CU_TRY(z.d_foff.ensure((size_t)n + 1));
        CU_TRY(z.d_bsum.ensure((size_t)(n + SV_SCAN_THREADS) / SV_SCAN_THREADS + 1)); CU_TRY(z.h_n.ensure(2));
        SvolMeshArgs Mg = {};
        for (int a = 0; a < 3; a++) Mg.bmin[a] = g->bmin[a];
        Mg.res = g->res; Mg.X = g->X; Mg.Y = g->Y; Mg.Z = g->Z;
        Mg.value = z.d_val.p; Mg.tstar = z.d_ts.p; Mg.emask = z.d_mask.p; Mg.voff = z.d_voff.p; Mg.foff = z.d_foff.p;
        CU_TRY(sv_mesh_count_launch(Mg, st));
        CU_TRY(sv_scan_launch(z.d_voff.p, n, z.d_bsum.p, st));
        CU_TRY(sv_scan_launch(z.d_foff.p, n, z.d_bsum.p, st));
        c->stats.kernel_launches += 7;   // count, two three-kernel scans
        CU_TRY(cudaMemcpyAsync(z.h_n.p, z.d_voff.p + n, sizeof(long long), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaMemcpyAsync(z.h_n.p + 1, z.d_foff.p + n, sizeof(long long), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
        *nV = z.h_n.p[0]; *nF = z.h_n.p[1];
        if (*nV > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "more than 2^31 - 1 vertices: use a coarser grid");
        if (*nV > cap_v || *nF > cap_f) return fail(ISDF_ERR_INVALID, "cap_v / cap_f smaller than the mesh (*nV / *nF hold the sizes needed)");
        CU_TRY(z.d_V.ensure((size_t)std::max<long long>(3 * *nV, 1))); CU_TRY(z.d_vt.ensure((size_t)std::max<long long>(*nV, 1)));
        CU_TRY(z.d_F.ensure((size_t)std::max<long long>(3 * *nF, 1)));
        Mg.V = z.d_V.p; Mg.vtime = z.d_vt.p; Mg.F = z.d_F.p;
        CU_TRY(sv_mesh_emit_launch(Mg, st));
        c->stats.kernel_launches++;
        if (info) {
            CU_TRY(cudaEventRecord(z.ev[4], st));
            CU_TRY(cudaEventSynchronize(z.ev[4]));
            float ms = 0.f;
            CU_TRY(cudaEventElapsedTime(&ms, z.ev[3], z.ev[4])); info->mesh_ms = ms;
        }
        if (*nV) {
            CU_TRY(cudaMemcpyAsync(V, z.d_V.p, sizeof(double) * 3 * *nV, cudaMemcpyDeviceToHost, st));
            CU_TRY(cudaMemcpyAsync(vtime, z.d_vt.p, sizeof(double) * *nV, cudaMemcpyDeviceToHost, st));
        }
        if (*nF) CU_TRY(cudaMemcpyAsync(F, z.d_F.p, sizeof(int32_t) * 3 * *nF, cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
        return 0;
    }, [&] { if (cap_v > 0) { nan_fill(V, 3 * cap_v); nan_fill(vtime, cap_v); } });
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
    if (!(kc->kernel_ang_res > 0) || !(kc->kernel_max_roll >= 0) || !(kc->kernel_max_pitch >= 0) || !std::isfinite(kc->kernel_ang_res) ||
        !std::isfinite(kc->kernel_max_roll) || !std::isfinite(kc->kernel_max_pitch))
        return fail(ISDF_ERR_INVALID, "bad attitude grid");
    const int ks = c->cfg.kernel_size;
    if (ks < 1 || (ks & 1) == 0) return fail(ISDF_ERR_INVALID, "kernel_size must be odd (Shape.hpp:258)");
    // every front-end kernel but k_frontend_kernels stages the ks^3 offset masks (16 B each) in one CTA's shared memory
    if (16.0 * ks * ks * ks > (double)c->smem_optin)
        return fail(ISDF_ERR_UNSUPPORTED, "kernel_size too large: its offset masks (16 * kernel_size^3 B) exceed one CTA's shared memory");
    const double xkd = std::floor(2 * kc->kernel_max_roll / kc->kernel_ang_res) + 1, ykd = std::floor(2 * kc->kernel_max_pitch / kc->kernel_ang_res) + 1;   // swm:135-136
    if (!(xkd * ykd <= FE_MAX_ATT)) return fail(ISDF_ERR_UNSUPPORTED, "more than 128 attitudes");
    const int xk = (int)xkd, yk = (int)ykd;
    // the reference builds its kernels in accumulating loops (Shape.hpp:422-426); where rounding makes them visit another number of angles
    // than xk / yk, it leaves kernels unbuilt or writes past them, so such a grid has no defined answer
    auto loop_angles = [](double max_angle, double step) { int n = 0; for (double a = -max_angle; a <= max_angle; a += step) n++; return n; };
    if (loop_angles(kc->kernel_max_roll, kc->kernel_ang_res) != xk || loop_angles(kc->kernel_max_pitch, kc->kernel_ang_res) != yk)
        return fail(ISDF_ERR_UNSUPPORTED, "attitude grid: the accumulating angle loop does not visit floor(2 max / step) + 1 angles");
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

// the feasibility pipelines, as isdf_dbg_frontend_launch reports them
enum { FE_PIPE_ONE_PASS = 0, FE_PIPE_CORE = 1, FE_PIPE_TABLES = 2 };

// the feasibility pipeline into d_masks (4 words per voxel), or, with d_trav set, into the traversability bits (isdf_frontpath.cuh);
// bits (may be NULL: the map's occupancy): the grid it reads in place of the occupancy grid, in its layout (the blocked grid for T_b)
static int frontend_feasibility_run(isdf_ctx *c, uint32_t *d_masks, uint32_t *d_trav, void *cuda_stream, const uint32_t *bits = nullptr) {
    FrontArgs A = front_args(c);
    A.out = d_masks; A.trav = d_trav;
    if (bits) A.grid.bits = bits;
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
            const bool two = 2 * (tsmem + 1024) <= c->smem_per_sm;
            const unsigned blocks = two ? (unsigned)sms * 2 : (unsigned)sms, threads = two ? 512 : 1024;
            k_frontend_survivors_tab<<<blocks, threads, tsmem, (cudaStream_t)cuda_stream>>>(A);
            c->fe.last_launch[0] = FE_PIPE_TABLES; c->fe.last_launch[1] = (int)blocks; c->fe.last_launch[2] = (int)threads;
        } else {
            CU_TRY(cudaFuncSetAttribute(k_frontend_survivors, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            k_frontend_core<<<grid, 256, 0, (cudaStream_t)cuda_stream>>>(A);
            k_frontend_survivors<<<(unsigned)sms * 16, 256, smem, (cudaStream_t)cuda_stream>>>(A);
            c->fe.last_launch[0] = FE_PIPE_CORE; c->fe.last_launch[1] = (int)sms * 16; c->fe.last_launch[2] = 256;
        }
        c->stats.kernel_launches += 2;
    } else {
        k_frontend_feasibility<<<grid, 256, smem, (cudaStream_t)cuda_stream>>>(A);
        c->fe.last_launch[0] = FE_PIPE_ONE_PASS; c->fe.last_launch[1] = (int)grid; c->fe.last_launch[2] = 256;
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
    Staging S(c);
    FrontArgs A = front_args(c);
    S.in(&A.q_ind, ind, (size_t)3 * n); S.in(&A.q_father, father_roll_pitch, (size_t)2 * n);
    S.out(&A.q_child, child_roll_pitch, (size_t)2 * n); S.out(&A.q_ok, ok, (size_t)n);
    if (int rr = S.upload()) return rr;
    CU_TRY(c->fe.d_out.ensure((size_t)4 * n));
    A.out = c->fe.d_out.p; A.nq = n;
    const size_t smem = sizeof(uint32_t) * 4 * (size_t)A.ks * A.ks * A.ks;
    CU_TRY(cudaFuncSetAttribute(k_frontend_check, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_frontend_check<<<(unsigned)((n + 255) / 256), 256, smem, c->stream>>>(A);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    return S.download();
}

// ---- front-end path search (isdf_frontpath.cuh) ------------------------------------------------------------------------------------
constexpr int FP_ROUNDS_PER_CHECK = 8;   // relaxation rounds launched between two reads of the frontier flag

// the parameters' own checks; *cw = 1 + unknown_weight (1 for NULL params), the edge factor of a voxel that is not known
static int frontpath_params_check(const isdf_frontpath_params *prm, double *cw) {
    *cw = 1.0;
    if (!prm) return 0;
    for (int32_t v : prm->reserved_) if (v != 0) return fail(ISDF_ERR_INVALID, "isdf_frontpath_params: reserved fields must be zero");
    if (!(std::isfinite(prm->unknown_weight) && prm->unknown_weight >= 0.0))
        return fail(ISDF_ERR_INVALID, "isdf_frontpath_params: unknown_weight must be finite and >= 0");
    *cw = 1.0 + prm->unknown_weight;
    return 0;
}

static int path_args_check(isdf_ctx *c, const isdf_frontpath_params *prm, double *cw) {
    if (int r = frontend_state(c)) return r;
    if (c->world > 1) return fail(ISDF_ERR_UNSUPPORTED, "the front-end path search is not sharded: call it on a context with isdf_set_shard(ctx, 0, 1)");
    return frontpath_params_check(prm, cw);
}

// isInMap (Gridmap3D.cpp) + getGridIndex (Gridmap3D.cpp:135-175) with its clamps and its "iy < 0 => ix = 0" branches (they cannot fire
// for a point inside the map)
static int path_voxel(const DevGrid &G, const double *p, int id[3], const std::string &what) {
    for (int a = 0; a < 3; a++)
        if (!std::isfinite(p[a])) return fail(ISDF_ERR_INVALID, what + " is not finite");
    for (int a = 0; a < 3; a++)
        if (p[a] < G.bmin[a] || p[a] > G.bmax[a]) return fail(ISDF_ERR_INVALID, what + " is outside the map");
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

static PathArgs path_args(isdf_ctx *c, unsigned long long *d_g) {
    PathArgs P = {};
    P.grid = c->map.grid; P.trav = c->fp.d_trav.p; P.g = d_g;
    P.front = c->fp.d_front.p; P.src = c->fp.d_src.p;
    return P;
}

// the surcharge with edge factor cw; cw == 1 (weight 0, or a weight below FP64's resolution at 1, where w * cw == w) selects the
// unweighted kernels
static FpSurcharge path_surcharge(const isdf_ctx *c, double cw) { return {c->known.have ? c->known.d_known.p : nullptr, cw}; }

// the traversability grid of the current map and kernels on stream st, between events 0 and 1; clears c->fp.info. known_only: T_b,
// the traversability of the blocked grid (isdf_map_frontiers), in place of T_o
static int path_trav(isdf_ctx *c, cudaStream_t st, bool known_only = false) {
    const DevGrid &G = c->map.grid;
    for (cudaEvent_t &e : c->fp.ev) if (!e) CU_TRY(cudaEventCreate(&e));
    CU_TRY(c->fp.d_trav.ensure((size_t)G.X * G.Y * G.Zw));
    CU_TRY(c->fp.h_flag.ensure(2));
    if (known_only) if (int r = blocked_grid_ready(c, st)) return r;
    c->fp.info = {};
    CU_TRY(cudaEventRecord(c->fp.ev[0], st));
    if (int r = frontend_feasibility_run(c, nullptr, c->fp.d_trav.p, st, known_only ? c->known.d_blocked.p : nullptr)) return r;
    CU_TRY(cudaEventRecord(c->fp.ev[1], st));
    return 0;
}

// one relaxation from the n source voxels src (host, 3 each) into d_g (field s at d_g + s*X*Y*Z) on stream st, after path_trav, with
// the unknown-voxel edge factor cw; adds its device time and its rounds to c->fp.info
static int path_fields(isdf_ctx *c, int n, const int *src, double cw, unsigned long long *d_g, cudaStream_t st) {
    const DevGrid &G = c->map.grid;
    const size_t nword = (size_t)G.X * G.Y * G.Zw, nvox = (size_t)G.X * G.Y * G.Z, nflag = (size_t)(n + 1) * FP_FLAG_RING + 1;
    CU_TRY(c->fp.d_front.ensure(2 * (size_t)n * nword));
    CU_TRY(c->fp.d_flags.ensure(nflag));
    CU_TRY(c->fp.d_src.upload(src, (size_t)3 * n, st));
    count_copy(c, cudaMemcpyHostToDevice, sizeof(int) * 3 * (size_t)n);
    PathArgs P = path_args(c, d_g);
    const FpSurcharge U = path_surcharge(c, cw);
    P.flags = c->fp.d_flags.p; P.rounds = P.flags + (size_t)(n + 1) * FP_FLAG_RING;
    P.any = n == 1 ? P.flags : P.flags + (size_t)n * FP_FLAG_RING;
    P.front1 = P.front + nword;
    CU_TRY(cudaEventRecord(c->fp.ev[2], st));
    CU_TRY(cudaMemsetAsync(c->fp.d_front.p, 0, sizeof(uint32_t) * 2 * (size_t)n * nword, st));
    CU_TRY(cudaMemsetAsync(c->fp.d_flags.p, 0, sizeof(unsigned) * nflag, st));
    const long long sms = c->sm_count;
    k_fp_init<<<dim3((unsigned)std::min<long long>(((long long)nvox + 255) / 256, sms * 32), (unsigned)n), 256, 0, st>>>(P);
    c->stats.kernel_launches++;
    const dim3 blocks((unsigned)std::min<long long>(((long long)nword + 255) / 256, sms * 16), (unsigned)n);
    for (int r = 0;;) {
        for (int k = 0; k < FP_ROUNDS_PER_CHECK; k++, r++) {
            if (cw == 1.0) {
                if (n == 1) k_fp_relax<false><<<blocks, 256, 0, st>>>(P, r, U);
                else k_fp_relax_multi<false><<<blocks, 256, 0, st>>>(P, r, U);
            } else {
                if (n == 1) k_fp_relax<true><<<blocks, 256, 0, st>>>(P, r, U);
                else k_fp_relax_multi<true><<<blocks, 256, 0, st>>>(P, r, U);
            }
        }
        c->stats.kernel_launches += FP_ROUNDS_PER_CHECK;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(c->fp.h_flag.p, P.any + r % FP_FLAG_RING, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        count_copy(c, cudaMemcpyDeviceToHost, sizeof(unsigned), true);
        CU_TRY(cudaStreamSynchronize(st));
        if (!c->fp.h_flag.p[0]) break;
    }
    CU_TRY(cudaEventRecord(c->fp.ev[3], st));
    CU_TRY(cudaMemcpyAsync(c->fp.h_flag.p + 1, P.rounds, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    count_copy(c, cudaMemcpyDeviceToHost, sizeof(unsigned), true);
    CU_TRY(cudaStreamSynchronize(st));
    float ms = 0;
    cudaEventElapsedTime(&ms, c->fp.ev[2], c->fp.ev[3]);
    c->fp.info.field_ms += ms;
    c->fp.info.rounds += (int32_t)c->fp.h_flag.p[1];
    return 0;
}

// the stage times of a call that ran path_trav, then its fields, then (up to event 2) its paths; field_bytes: the fields held at once
static void path_info(isdf_ctx *c, size_t field_bytes, bool paths) {
    isdf_frontpath_info &I = c->fp.info;
    I.field_bytes = (int64_t)field_bytes;
    float ms = 0;
    cudaEventElapsedTime(&ms, c->fp.ev[0], c->fp.ev[1]); I.traversability_ms = ms;
    if (paths) { cudaEventElapsedTime(&ms, c->fp.ev[1], c->fp.ev[2]); I.paths_ms = ms - I.field_ms; }
}

// the paths of B (start, goal) pairs into c->fp.d_xyz / d_rp / d_cost / d_found in pair order. starts: B x 3, or one start for every
// goal (sstride 0). Pairs whose starts share a voxel share a field: node 0 of a path is its start voxel's cube centre, so their paths are
// the same. The distinct start voxels' fields are built in chunks of at most max_fields (0: FP_FIELD_BUDGET bytes, at least one field),
// and each chunk's paths are walked into scratch before its fields are reused. off (B + 1) is filled as soon as every length is known,
// also when they exceed cap. cw: the unknown-voxel edge factor of the fields and the walk (frontpath_params_check). known_only: over
// T_b instead of T_o (ISDF_PLAN_KNOWN_ONLY).
static int path_run(isdf_ctx *c, int B, const double *starts, int sstride, const double *goals, double cw, int max_fields, int cap,
                    std::vector<int> &off, cudaStream_t st, bool known_only = false) {
    const DevGrid &G = c->map.grid;
    const size_t nvox = (size_t)G.X * G.Y * G.Z;
    std::vector<int> tgt((size_t)3 * B), ps(B), src;   // ps[b]: pair b's source; src: 3 per distinct start voxel, in order of first use
    std::unordered_map<long long, int> seen;
    for (int b = 0; b < B; b++) {
        int s[3];
        if (int r = path_voxel(G, starts + (size_t)sstride * b, s, sstride ? "starts[" + std::to_string(b) + "]" : std::string("start"))) return r;
        if (int r = path_voxel(G, goals + 3 * (size_t)b, &tgt[3 * (size_t)b], "goals[" + std::to_string(b) + "]")) return r;
        const auto ins = seen.emplace(((long long)s[0] * G.Y + s[1]) * G.Z + s[2], (int)(src.size() / 3));
        if (ins.second) src.insert(src.end(), s, s + 3);
        ps[b] = ins.first->second;
    }
    const int S = (int)(src.size() / 3);
    const long long want = max_fields > 0 ? max_fields : std::max<long long>(1, FP_FIELD_BUDGET / (long long)(sizeof(double) * nvox));
    const int F = (int)std::min<long long>(std::min<long long>(want, S), 65535);   // fields per chunk (grid.y of the relaxation)
    // walk order: the pairs grouped by source, in pair order within a source; pair b is walked at wpos[b]
    std::vector<int> wstart((size_t)S + 1, 0), walk(B), wpos(B);
    for (int b = 0; b < B; b++) wstart[ps[b] + 1]++;
    for (int s = 0; s < S; s++) wstart[s + 1] += wstart[s];
    std::vector<int> wtgt((size_t)3 * B), wsrc((size_t)4 * B);
    {
        std::vector<int> next(wstart.begin(), wstart.end() - 1);
        for (int b = 0; b < B; b++) {
            const int w = next[ps[b]]++;
            wpos[b] = w; walk[w] = b;
            for (int k = 0; k < 3; k++) { wtgt[3 * (size_t)w + k] = tgt[3 * (size_t)b + k]; wsrc[4 * (size_t)w + k] = src[3 * (size_t)ps[b] + k]; }
            wsrc[4 * (size_t)w + 3] = ps[b] % F;   // the field's slice in its chunk
        }
    }
    if (int r = path_trav(c, st, known_only)) return r;
    CU_TRY(c->fp.d_g.ensure((size_t)F * nvox));
    CU_TRY(c->fp.d_tgt.upload(wtgt.data(), wtgt.size(), st)); CU_TRY(c->fp.d_tsrc.upload(wsrc.data(), wsrc.size(), st));
    CU_TRY(c->fp.d_pair.upload(walk.data(), walk.size(), st));
    count_copy(c, cudaMemcpyHostToDevice, sizeof(int) * (wtgt.size() + wsrc.size() + walk.size())); c->xfer[XF_COPIES] += 2;
    CU_TRY(c->fp.d_len.ensure(B)); CU_TRY(c->fp.d_woff.ensure((size_t)B + 1)); CU_TRY(c->fp.d_cost.ensure(B)); CU_TRY(c->fp.d_found.ensure(B));
    std::vector<int> len(B), woff((size_t)B + 1, 0);   // walk order; woff: first node in scratch
    for (int s0 = 0; s0 < S; s0 += F) {
        const int n = std::min(F, S - s0), w0 = wstart[s0], w1 = wstart[s0 + n], nt = w1 - w0;
        if (int r = path_fields(c, n, &src[3 * (size_t)s0], cw, c->fp.d_g.p, st)) return r;
        PathArgs P = path_args(c, c->fp.d_g.p);
        const auto walk_kernel = cw == 1.0 ? k_fp_walk<false> : k_fp_walk<true>;
        const FpSurcharge U = path_surcharge(c, cw);
        P.nt = nt; P.tgt = c->fp.d_tgt.p + 3 * (size_t)w0; P.tsrc = c->fp.d_tsrc.p + 4 * (size_t)w0; P.pair = c->fp.d_pair.p + w0;
        P.len = c->fp.d_len.p + w0; P.cost = c->fp.d_cost.p; P.found = c->fp.d_found.p;
        const unsigned wblocks = (unsigned)(((long long)nt * 32 + 127) / 128);
        walk_kernel<<<wblocks, 128, 0, st>>>(P, 0, U);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(len.data() + w0, P.len, sizeof(int) * nt, cudaMemcpyDeviceToHost, st));
        count_copy(c, cudaMemcpyDeviceToHost, sizeof(int) * nt);
        CU_TRY(cudaStreamSynchronize(st));
        for (int w = w0; w < w1; w++) {
            if ((long long)woff[w] + len[w] > INT32_MAX) return fail(ISDF_ERR_INVALID, "the paths hold more than 2^31 - 1 nodes");
            woff[w + 1] = woff[w] + len[w];
        }
        if ((size_t)3 * woff[w1] > c->fp.d_scratch.n) {   // grow the scratch, keeping the earlier chunks' paths
            DevBuf<int> grown;
            CU_TRY(grown.ensure(std::max((size_t)3 * woff[w1], 2 * c->fp.d_scratch.n)));
            if (woff[w0]) CU_TRY(cudaMemcpyAsync(grown.p, c->fp.d_scratch.p, sizeof(int) * 3 * (size_t)woff[w0], cudaMemcpyDeviceToDevice, st));
            CU_TRY(cudaStreamSynchronize(st));   // the old buffer is freed when grown goes out of scope
            std::swap(c->fp.d_scratch, grown);
        }
        CU_TRY(cudaMemcpyAsync(c->fp.d_woff.p + w0, woff.data() + w0, sizeof(int) * ((size_t)nt + 1), cudaMemcpyHostToDevice, st));
        count_copy(c, cudaMemcpyHostToDevice, sizeof(int) * ((size_t)nt + 1));
        P.off = c->fp.d_woff.p + w0; P.scratch = c->fp.d_scratch.p;
        walk_kernel<<<wblocks, 128, 0, st>>>(P, 1, U);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
    }
    path_info(c, (size_t)F * nvox * sizeof(double), false);
    // pair order
    off.assign((size_t)B + 1, 0);
    std::vector<int> soff(B);
    for (int b = 0; b < B; b++) { off[b + 1] = off[b] + len[wpos[b]]; soff[b] = woff[wpos[b]]; }
    const int total = off[B];
    if (total > cap) return fail(ISDF_ERR_INVALID, "cap is smaller than the total path length (reported in n / offsets[B])");
    CU_TRY(c->fp.d_off.upload(off.data(), off.size(), st)); CU_TRY(c->fp.d_soff.upload(soff.data(), soff.size(), st));
    count_copy(c, cudaMemcpyHostToDevice, sizeof(int) * (off.size() + soff.size())); c->xfer[XF_COPIES]++;
    CU_TRY(c->fp.d_nodes.ensure((size_t)3 * total)); CU_TRY(c->fp.d_colliding.ensure((size_t)4 * total));
    CU_TRY(c->fp.d_xyz.ensure((size_t)3 * total)); CU_TRY(c->fp.d_rp.ensure((size_t)2 * total));
    PathArgs P = path_args(c, c->fp.d_g.p);
    P.nt = B; P.off = c->fp.d_off.p; P.soff = c->fp.d_soff.p; P.scratch = c->fp.d_scratch.p;
    P.nodes = c->fp.d_nodes.p; P.xyz = c->fp.d_xyz.p; P.rp = c->fp.d_rp.p; P.colliding = c->fp.d_colliding.p;
    k_fp_place<<<(unsigned)(((long long)B * 32 + 127) / 128), 128, 0, st>>>(P);
    FrontArgs A = front_args(c);
    A.nq = total; A.q_ind = c->fp.d_nodes.p; A.out = c->fp.d_colliding.p;
    const size_t smem = sizeof(uint32_t) * 4 * (size_t)A.ks * A.ks * A.ks;
    CU_TRY(cudaFuncSetAttribute(k_fp_node_masks, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_fp_node_masks<<<(unsigned)(((long long)total + 255) / 256), 256, smem, st>>>(A);
    k_fp_attitudes<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(A, P);
    c->stats.kernel_launches += 3;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaEventRecord(c->fp.ev[2], st));
    CU_TRY(cudaStreamSynchronize(st));
    path_info(c, (size_t)F * nvox * sizeof(double), true);
    return 0;
}

// a device-form call's goals (B x 3) and, with sstride 3 or 9, its starts' positions, read to the host on st for path_run's grouping; goals
// and starts then point at hg and hs (sstride 3). Start states (sstride 9, isdf_plan_states_device): only the positions cross, and v and a
// are checked on the device, one 4-byte verdict.
static int read_endpoints(isdf_ctx *c, int B, const double *&starts, int &sstride, const double *&goals, std::vector<double> &hs,
                          std::vector<double> &hg, cudaStream_t st) {
    hg.resize((size_t)3 * B);
    CU_TRY(cudaMemcpyAsync(hg.data(), goals, sizeof(double) * hg.size(), cudaMemcpyDeviceToHost, st));
    count_copy(c, cudaMemcpyDeviceToHost, sizeof(double) * hg.size());
    int bad = 0x7fffffff;
    if (sstride == 9) {
        CU_TRY(c->plan.d_bad.ensure(1));
        CU_TRY(cudaMemcpyAsync(c->plan.d_bad.p, &bad, sizeof(int), cudaMemcpyHostToDevice, st));
        count_copy(c, cudaMemcpyHostToDevice, sizeof(int));
        k_plan_heads_check<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(B, starts, c->plan.d_bad.p);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(&bad, c->plan.d_bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
        count_copy(c, cudaMemcpyDeviceToHost, sizeof(int));
    }
    if (sstride) {
        hs.resize((size_t)3 * B);
        CU_TRY(cudaMemcpy2DAsync(hs.data(), 3 * sizeof(double), starts, sstride * sizeof(double), 3 * sizeof(double), B, cudaMemcpyDeviceToHost, st));
        count_copy(c, cudaMemcpyDeviceToHost, sizeof(double) * hs.size());
        starts = hs.data();
        sstride = 3;
    }
    CU_TRY(cudaStreamSynchronize(st));
    goals = hg.data();
    if (bad != 0x7fffffff) return fail(ISDF_ERR_INVALID, "starts[" + std::to_string(bad) + "]: velocity or acceleration is not finite");
    return 0;
}

// the path calls (starts: sstride 0 for one start, on the host in every form). dev: goals, starts (sstride 3) and every output in device
// memory, the call on cuda_stream; else host memory, the call on ctx's stream
static int path_entry(isdf_ctx *c, bool dev, int B, const double *starts, int sstride, const double *goals, const isdf_frontpath_params *prm,
                      int max_fields, int cap, double *path_xyz, double *path_rp, int32_t *offsets, double *costs, uint8_t *found,
                      void *cuda_stream) {
    if (!starts || !goals || B < 1 || max_fields < 0 || cap < 0 || (cap > 0 && !path_xyz) || !offsets || !costs || !found)
        return fail(ISDF_ERR_INVALID, "bad argument");
    double cw = 1.0;
    if (int r = path_args_check(c, prm, &cw)) return r;
    if (set_device(c)) return ISDF_ERR_CUDA;
    const cudaStream_t st = dev ? (cudaStream_t)cuda_stream : c->stream;
    std::vector<double> hs, hg;
    if (dev) if (int r = read_endpoints(c, B, starts, sstride, goals, hs, hg, st)) return r;
    std::vector<int> off;
    const int r = path_run(c, B, starts, sstride, goals, cw, max_fields, cap, off, st);
    if (!off.empty() && !dev) std::memcpy(offsets, off.data(), sizeof(int32_t) * off.size());
    if (!off.empty() && dev) {
        CU_TRY(cudaMemcpyAsync(offsets, off.data(), sizeof(int32_t) * off.size(), cudaMemcpyHostToDevice, st));
        CU_TRY(cudaStreamSynchronize(st));   // off is a host temporary
    }
    if (r) return r;
    const cudaMemcpyKind k = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    const size_t total = (size_t)off[B];
    CU_TRY(cudaMemcpyAsync(path_xyz, c->fp.d_xyz.p, sizeof(double) * 3 * total, k, st));
    if (path_rp) CU_TRY(cudaMemcpyAsync(path_rp, c->fp.d_rp.p, sizeof(double) * 2 * total, k, st));
    CU_TRY(cudaMemcpyAsync(costs, c->fp.d_cost.p, sizeof(double) * B, k, st));
    CU_TRY(cudaMemcpyAsync(found, c->fp.d_found.p, B, k, st));
    CU_TRY(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int isdf_frontend_path_batch(isdf_ctx *c, const double *start, int B, const double *goals, const isdf_frontpath_params *prm, int cap,
                                        double *path_xyz, double *path_rp, int32_t *offsets, double *costs, uint8_t *found) {
    return path_entry(c, false, B, start, 0, goals, prm, 0, cap, path_xyz, path_rp, offsets, costs, found, nullptr);
}

extern "C" int isdf_frontend_path_pairs(isdf_ctx *c, int B, const double *starts, const double *goals, const isdf_frontpath_params *prm,
                                        int max_fields, int cap, double *path_xyz, double *path_rp, int32_t *offsets, double *costs, uint8_t *found) {
    return path_entry(c, false, B, starts, 3, goals, prm, max_fields, cap, path_xyz, path_rp, offsets, costs, found, nullptr);
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
    return path_entry(c, true, B, start, 0, d_goals, prm, 0, cap, d_path_xyz, d_path_rp, d_offsets, d_costs, d_found, cuda_stream);
}

extern "C" int isdf_frontend_path_pairs_device(isdf_ctx *c, int B, const double *d_starts, const double *d_goals, const isdf_frontpath_params *prm,
                                               int max_fields, int cap, double *d_path_xyz, double *d_path_rp, int32_t *d_offsets,
                                               double *d_costs, uint8_t *d_found, void *cuda_stream) {
    return path_entry(c, true, B, d_starts, 3, d_goals, prm, max_fields, cap, d_path_xyz, d_path_rp, d_offsets, d_costs, d_found, cuda_stream);
}

// the fields of the S source voxels src (host, 3 each) in one relaxation into d_g
static int path_fields_run(isdf_ctx *c, int S, const int *src, double cw, double *d_g, cudaStream_t st) {
    if (int r = path_trav(c, st)) return r;
    if (int r = path_fields(c, S, src, cw, reinterpret_cast<unsigned long long *>(d_g), st)) return r;
    path_info(c, (size_t)S * c->map.grid.X * c->map.grid.Y * c->map.grid.Z * sizeof(double), false);
    return 0;
}

extern "C" int isdf_frontend_path_field_device(isdf_ctx *c, const double *start, const isdf_frontpath_params *prm, double *d_g, void *cuda_stream) {
    if (!start || !d_g) return fail(ISDF_ERR_INVALID, "bad argument");
    double cw = 1.0;
    if (int r = path_args_check(c, prm, &cw)) return r;
    if (set_device(c)) return ISDF_ERR_CUDA;
    int s[3];
    if (int r = path_voxel(c->map.grid, start, s, "start")) return r;
    return path_fields_run(c, 1, s, cw, d_g, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_frontend_path_fields_device(isdf_ctx *c, int S, const double *starts, const isdf_frontpath_params *prm, double *d_g,
                                                void *cuda_stream) {
    if (!starts || !d_g || S < 1) return fail(ISDF_ERR_INVALID, "bad argument");
    if (S > 65535) return fail(ISDF_ERR_INVALID, "S must be at most 65535");
    double cw = 1.0;
    if (int r = path_args_check(c, prm, &cw)) return r;
    if (set_device(c)) return ISDF_ERR_CUDA;
    std::vector<int> src((size_t)3 * S);
    for (int s = 0; s < S; s++)
        if (int r = path_voxel(c->map.grid, starts + 3 * (size_t)s, &src[3 * (size_t)s], "starts[" + std::to_string(s) + "]")) return r;
    return path_fields_run(c, S, src.data(), cw, d_g, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_frontend_path_info(isdf_ctx *c, isdf_frontpath_info *out) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    *out = c->fp.info;
    return 0;
}

// ---- frontiers of known space and frontier goals (isdf_frontier.cuh) ------------------------------------------------------------------
static int frontier_state(isdf_ctx *c) {
    if (int r = frontend_state(c)) return r;
    if (c->world > 1) return fail(ISDF_ERR_UNSUPPORTED, "the frontier calls are not sharded: call them on a context with isdf_set_shard(ctx, 0, 1)");
    return 0;
}

template <typename T>
static int fr_scan(isdf_ctx *c, const T *in, T *out, long long n, cudaStream_t st) {
    size_t bytes = 0;
    CU_TRY(cub::DeviceScan::InclusiveSum(nullptr, bytes, in, out, n, st));
    CU_TRY(c->fr.d_tmp.ensure(std::max<size_t>(bytes, 1)));
    CU_TRY(cub::DeviceScan::InclusiveSum(c->fr.d_tmp.p, bytes, in, out, n, st));
    return 0;
}

// T_o into c->fr.d_to, T_b into c->fp.d_trav (so that path_fields relaxes over T_b), F, its list, labels and cluster table into c->fr on
// st; counts and the first three stage times into *I. Leaves c->fp.info cleared (path_trav).
static int frontier_run(isdf_ctx *c, isdf_frontier_info *I, cudaStream_t st) {
    auto &z = c->fr;
    const DevGrid &G = c->map.grid;
    const long long nword = (long long)G.X * G.Y * G.Zw;
    for (cudaEvent_t &e : z.ev) if (!e) CU_TRY(cudaEventCreate(&e));
    *I = {};
    CU_TRY(z.d_to.ensure((size_t)nword)); CU_TRY(z.d_f.ensure((size_t)nword)); CU_TRY(z.d_cnt.ensure((size_t)nword));
    CU_TRY(z.d_woff.ensure((size_t)nword + 1)); CU_TRY(z.d_ntb.ensure(1));
    if (int r = blocked_grid_ready(c, st)) return r;
    CU_TRY(cudaEventRecord(z.ev[0], st));
    if (int r = frontend_feasibility_run(c, nullptr, z.d_to.p, st)) return r;
    if (int r = path_trav(c, st, true)) return r;
    CU_TRY(cudaEventRecord(z.ev[1], st));
    FrArgs A = {};
    A.grid = G; A.to = z.d_to.p; A.tb = c->fp.d_trav.p; A.f = z.d_f.p; A.cnt = z.d_cnt.p; A.woff = z.d_woff.p; A.ntb = z.d_ntb.p;
    const long long sms = c->sm_count;
    CU_TRY(cudaMemsetAsync(z.d_ntb.p, 0, sizeof(unsigned long long), st));
    CU_TRY(cudaMemsetAsync(z.d_woff.p, 0, sizeof(int), st));
    k_fr_frontier<<<(unsigned)std::min<long long>((nword + 255) / 256, sms * 32), 256, 0, st>>>(A);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    if (int r = fr_scan(c, z.d_cnt.p, z.d_woff.p + 1, nword, st)) return r;
    int n = 0;
    unsigned long long ntb = 0;
    CU_TRY(cudaMemcpyAsync(&n, z.d_woff.p + nword, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaMemcpyAsync(&ntb, z.d_ntb.p, sizeof(ntb), cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    A.n = n;
    CU_TRY(z.d_vox.ensure(std::max(n, 1))); CU_TRY(z.d_parent.ensure(std::max(n, 1))); CU_TRY(z.d_root.ensure((size_t)n + 1));
    CU_TRY(z.d_slot.ensure((size_t)n + 1)); CU_TRY(z.d_cid.ensure(std::max(n, 1)));
    A.vox = z.d_vox.p; A.parent = z.d_parent.p; A.root = z.d_root.p; A.cid = z.d_cid.p;
    const unsigned lb = (unsigned)std::max<long long>(1, std::min<long long>(((long long)n + 255) / 256, sms * 32));
    if (n) {
        k_fr_list<<<(unsigned)std::min<long long>((nword + 255) / 256, sms * 32), 256, 0, st>>>(A);
        c->stats.kernel_launches++;
    }
    CU_TRY(cudaEventRecord(z.ev[2], st));
    int nc = 0;
    if (n) {
        k_fr_hook<<<lb, 256, 0, st>>>(A);
        k_fr_flatten<<<lb, 256, 0, st>>>(A);
        c->stats.kernel_launches += 2;
        CU_TRY(cudaGetLastError());
        if (int r = fr_scan(c, z.d_root.p, z.d_slot.p + 1, n, st)) return r;
        CU_TRY(cudaMemsetAsync(z.d_slot.p, 0, sizeof(int), st));
        CU_TRY(cudaMemcpyAsync(&nc, z.d_slot.p + n, sizeof(int), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
    }
    // slot[r] = the roots before position r: root r's cluster slot, in ascending cluster id; slot[n] = the clusters
    CU_TRY(z.d_size.ensure(std::max(nc, 1))); CU_TRY(z.d_box.ensure(6 * (size_t)std::max(nc, 1))); CU_TRY(z.d_croot.ensure(std::max(nc, 1)));
    CU_TRY(z.d_sum.ensure(3 * (size_t)std::max(nc, 1))); CU_TRY(z.d_table.ensure(std::max(nc, 1)));
    A.slot = z.d_slot.p; A.nc = nc; A.size = z.d_size.p; A.box = z.d_box.p; A.croot = z.d_croot.p; A.sum = z.d_sum.p; A.table = z.d_table.p;
    if (nc) {
        k_fr_table_init<<<(unsigned)((nc + 127) / 128), 128, 0, st>>>(A);
        k_fr_accum<<<lb, 256, 0, st>>>(A);
        k_fr_table<<<(unsigned)((nc + 127) / 128), 128, 0, st>>>(A);
        c->stats.kernel_launches += 3;
        CU_TRY(cudaGetLastError());
    }
    CU_TRY(cudaEventRecord(z.ev[3], st));
    CU_TRY(cudaStreamSynchronize(st));
    float ms = 0;
    cudaEventElapsedTime(&ms, z.ev[0], z.ev[1]); I->traversability_ms = ms;
    cudaEventElapsedTime(&ms, z.ev[1], z.ev[2]); I->frontier_ms = ms;
    cudaEventElapsedTime(&ms, z.ev[2], z.ev[3]); I->cluster_ms = ms;
    I->traversable_blocked = (int64_t)ntb; I->frontier_voxels = n; I->clusters = nc;
    return 0;
}

static int frontiers_entry(isdf_ctx *c, bool dev, int64_t cap_voxels, int64_t *voxels, int64_t *cluster_of, int64_t cap_clusters,
                           isdf_frontier_cluster *clusters, isdf_frontier_info *info, cudaStream_t st) {
    if (int r = frontier_state(c)) return r;
    if (cap_voxels < 0 || cap_clusters < 0 || (cap_voxels > 0 && (!voxels || !cluster_of)) || (cap_clusters > 0 && !clusters))
        return fail(ISDF_ERR_INVALID, "a negative cap, or a NULL output with a non-zero cap");
    if (set_device(c)) return ISDF_ERR_CUDA;
    if (!dev) st = c->stream;
    isdf_frontier_info I;
    const int r = frontier_run(c, &I, st);
    if (info) *info = I;
    if (r) return r;
    if (I.frontier_voxels > cap_voxels || I.clusters > cap_clusters)
        return fail(ISDF_ERR_INVALID, "cap_voxels or cap_clusters too small (info reports the sizes needed)");
    const cudaMemcpyKind k = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (I.frontier_voxels) {
        CU_TRY(cudaMemcpyAsync(voxels, c->fr.d_vox.p, sizeof(int64_t) * I.frontier_voxels, k, st));
        CU_TRY(cudaMemcpyAsync(cluster_of, c->fr.d_cid.p, sizeof(int64_t) * I.frontier_voxels, k, st));
        CU_TRY(cudaMemcpyAsync(clusters, c->fr.d_table.p, sizeof(isdf_frontier_cluster) * I.clusters, k, st));
    }
    CU_TRY(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int isdf_map_frontiers(isdf_ctx *c, int64_t cap_voxels, int64_t *voxels, int64_t *cluster_of, int64_t cap_clusters,
                                  isdf_frontier_cluster *clusters, isdf_frontier_info *info) {
    return frontiers_entry(c, false, cap_voxels, voxels, cluster_of, cap_clusters, clusters, info, nullptr);
}

extern "C" int isdf_map_frontiers_device(isdf_ctx *c, int64_t cap_voxels, int64_t *d_voxels, int64_t *d_cluster_of, int64_t cap_clusters,
                                         isdf_frontier_cluster *d_clusters, isdf_frontier_info *info, void *cuda_stream) {
    return frontiers_entry(c, true, cap_voxels, d_voxels, d_cluster_of, cap_clusters, d_clusters, info, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_frontier_default_params(isdf_frontier_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    std::memset(p, 0, sizeof(*p));
    p->goal_weight = 1.0;
    p->min_cluster_voxels = 1;
    return 0;
}

// the frontier goals of B pairs (starts and goals on the host, B x 3) into out (B records, device) on st
// ncam cameras at cams (host; 0: no rig, every gain 0): a candidate also needs a view gain of at least min_gain
static int frontier_goals_run(isdf_ctx *c, int B, const double *starts, const double *goals, const isdf_frontier_params *p, int ncam,
                              const isdf_sense_params *cams, long long min_gain, int max_fields, isdf_frontier_goal *out, isdf_frontier_info *I,
                              cudaStream_t st) {
    const DevGrid &G = c->map.grid;
    const size_t nvox = (size_t)G.X * G.Y * G.Z;
    auto &z = c->fr;
    std::vector<int> tgt((size_t)3 * B), ps(B), src;   // as path_run: ps[b] is pair b's source, src the distinct start voxels
    std::unordered_map<long long, int> seen;
    for (int b = 0; b < B; b++) {
        int s[3];
        if (int r = path_voxel(G, starts + 3 * (size_t)b, s, "starts[" + std::to_string(b) + "]")) return r;
        if (int r = path_voxel(G, goals + 3 * (size_t)b, &tgt[3 * (size_t)b], "goals[" + std::to_string(b) + "]")) return r;
        const auto ins = seen.emplace(((long long)s[0] * G.Y + s[1]) * G.Z + s[2], (int)(src.size() / 3));
        if (ins.second) src.insert(src.end(), s, s + 3);
        ps[b] = ins.first->second;
    }
    if (int r = frontier_run(c, I, st)) return r;
    const int S = (int)(src.size() / 3), n = (int)I->frontier_voxels;
    const long long want = max_fields > 0 ? max_fields : std::max<long long>(1, FP_FIELD_BUDGET / (long long)(sizeof(double) * nvox));
    const int F = (int)std::min<long long>(std::min<long long>(want, S), 65535);
    // walk order: the pairs grouped by source
    std::vector<int> wstart((size_t)S + 1, 0), wpair(B), wslice(B);
    for (int b = 0; b < B; b++) wstart[ps[b] + 1]++;
    for (int s = 0; s < S; s++) wstart[s + 1] += wstart[s];
    {
        std::vector<int> next(wstart.begin(), wstart.end() - 1);
        for (int b = 0; b < B; b++) { const int w = next[ps[b]]++; wpair[w] = b; wslice[w] = ps[b] % F; }
    }
    CU_TRY(z.d_pair.upload(wpair.data(), wpair.size(), st)); CU_TRY(z.d_slice.upload(wslice.data(), wslice.size(), st));
    CU_TRY(z.d_tgt.upload(tgt.data(), tgt.size(), st)); CU_TRY(z.d_goals.upload(goals, (size_t)3 * B, st));
    CU_TRY(z.d_best.ensure(B)); CU_TRY(z.d_pick.ensure(B)); CU_TRY(z.d_cand.ensure(std::max(n, 1)));
    CU_TRY(cudaMemsetAsync(z.d_best.p, 0xff, sizeof(unsigned long long) * B, st));   // above every score's bits, +inf's included
    CU_TRY(cudaMemsetAsync(z.d_pick.p, 0xff, sizeof(unsigned) * B, st));
    if (n) {
        k_fg_cand<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, z.d_parent.p, z.d_slot.p, z.d_size.p, p->min_cluster_voxels, z.d_cand.p);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
    }
    if (n && ncam) {   // the gains of the voxels the size rule kept (the others count 0 and stay out)
        CU_TRY(z.d_vpose.ensure(7 * (size_t)n)); CU_TRY(z.d_gain.ensure(n));
        k_fg_view_poses<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(G, n, z.d_vox.p, z.d_vpose.p);
        int launches = 1;
        const cudaError_t e = view_gain_run(c->sense, n, z.d_vpose.p, z.d_vpose.p + 3, 7, ncam, cams, G, c->known.have ? c->known.d_known.p : nullptr,
                                            z.d_cand.p, reinterpret_cast<int64_t *>(z.d_gain.p), st, &launches);
        k_fg_gain_cand<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, z.d_gain.p, min_gain, z.d_cand.p);
        c->stats.kernel_launches += launches + 1;
        CU_TRY(e);
        CU_TRY(cudaGetLastError());
    }
    CU_TRY(c->fp.d_g.ensure((size_t)F * nvox));
    FgArgs A = {};
    A.grid = G; A.g = c->fp.d_g.p; A.vox = z.d_vox.p; A.cand = z.d_cand.p; A.n = n; A.goal_weight = p->goal_weight;
    A.goals = z.d_goals.p; A.tgt = z.d_tgt.p; A.best = z.d_best.p; A.pick = z.d_pick.p; A.table = z.d_table.p; A.cid = z.d_cid.p; A.out = out;
    A.gain = ncam ? z.d_gain.p : nullptr;
    const long long sms = c->sm_count;
    for (int s0 = 0; s0 < S; s0 += F) {
        const int m = std::min(F, S - s0), w0 = wstart[s0], w1 = wstart[s0 + m];
        if (int r = path_fields(c, m, &src[3 * (size_t)s0], 1.0, c->fp.d_g.p, st)) return r;
        CU_TRY(cudaEventRecord(z.ev[4], st));
        A.nt = w1 - w0; A.pair = z.d_pair.p + w0; A.slice = z.d_slice.p + w0;
        if (n) {
            const dim3 grid((unsigned)std::max<long long>(1, std::min<long long>(((long long)n + 255) / 256, sms * 8)), (unsigned)std::min(A.nt, 65535));
            // a pair without a candidate keeps best = ~0, which no score equals: k_fg_select<true> picks nothing for it
            k_fg_select<false><<<grid, 256, 0, st>>>(A);
            k_fg_select<true><<<grid, 256, 0, st>>>(A);
            c->stats.kernel_launches += 2;
        }
        k_fg_record<<<(unsigned)((A.nt + 127) / 128), 128, 0, st>>>(A);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaEventRecord(z.ev[5], st));
        CU_TRY(cudaStreamSynchronize(st));
        float ms = 0;
        cudaEventElapsedTime(&ms, z.ev[4], z.ev[5]);
        I->select_ms += ms;
    }
    I->field_ms = c->fp.info.field_ms;
    return 0;
}

// ncam < 0: isdf_frontier_goals (no rig, min_gain 0); else the view form's rig
static int frontier_goals_entry(isdf_ctx *c, bool dev, int B, const double *starts, const double *goals, const isdf_frontier_params *prm,
                                int ncam, const isdf_sense_params *cams, long long min_gain, int max_fields, isdf_frontier_goal *out,
                                isdf_frontier_info *info, cudaStream_t st) {
    if (int r = frontier_state(c)) return r;
    if (!starts || !goals || !out || B < 1) return fail(ISDF_ERR_INVALID, "NULL argument or B < 1");
    if (max_fields < 0) return fail(ISDF_ERR_INVALID, "max_fields < 0");
    if (ncam >= 0) {
        if (int r = view_rig_check(c, ncam, cams)) return r;
        if (min_gain < 0) return fail(ISDF_ERR_INVALID, "min_gain < 0");
    }
    isdf_frontier_params p;
    isdf_frontier_default_params(&p);
    if (prm) p = *prm;
    if (p.reserved_ != 0) return fail(ISDF_ERR_INVALID, "isdf_frontier_params: reserved_ must be 0");
    if (!(std::isfinite(p.goal_weight) && p.goal_weight > 0.0)) return fail(ISDF_ERR_INVALID, "isdf_frontier_params: goal_weight must be finite and > 0");
    if (p.min_cluster_voxels < 1) return fail(ISDF_ERR_INVALID, "isdf_frontier_params: min_cluster_voxels must be >= 1");
    if (set_device(c)) return ISDF_ERR_CUDA;
    if (!dev) st = c->stream;
    std::vector<double> hs, hg;
    if (dev) {
        int sstride = 3;
        if (int r = read_endpoints(c, B, starts, sstride, goals, hs, hg, st)) return r;
    }
    CU_TRY(c->fr.d_out.ensure(B));
    isdf_frontier_info I = {};
    const int r = frontier_goals_run(c, B, starts, goals, &p, std::max(ncam, 0), cams, min_gain, max_fields, dev ? out : c->fr.d_out.p, &I, st);
    if (info) *info = I;
    if (r) return r;
    if (!dev) CU_TRY(cudaMemcpyAsync(out, c->fr.d_out.p, sizeof(isdf_frontier_goal) * B, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int isdf_frontier_goals(isdf_ctx *c, int B, const double *starts, const double *goals, const isdf_frontier_params *p, int max_fields,
                                   isdf_frontier_goal *out, isdf_frontier_info *info) {
    return frontier_goals_entry(c, false, B, starts, goals, p, -1, nullptr, 0, max_fields, out, info, nullptr);
}

extern "C" int isdf_frontier_goals_device(isdf_ctx *c, int B, const double *d_starts, const double *d_goals, const isdf_frontier_params *p,
                                          int max_fields, isdf_frontier_goal *d_out, isdf_frontier_info *info, void *cuda_stream) {
    return frontier_goals_entry(c, true, B, d_starts, d_goals, p, -1, nullptr, 0, max_fields, d_out, info, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_frontier_goals_view(isdf_ctx *c, int B, const double *starts, const double *goals, const isdf_frontier_params *p, int n_cams,
                                        const isdf_sense_params *cams, int64_t min_gain, int max_fields, isdf_frontier_goal *out,
                                        isdf_frontier_info *info) {
    return frontier_goals_entry(c, false, B, starts, goals, p, n_cams, cams, min_gain, max_fields, out, info, nullptr);
}

extern "C" int isdf_frontier_goals_view_device(isdf_ctx *c, int B, const double *d_starts, const double *d_goals, const isdf_frontier_params *p,
                                               int n_cams, const isdf_sense_params *cams, int64_t min_gain, int max_fields,
                                               isdf_frontier_goal *d_out, isdf_frontier_info *info, void *cuda_stream) {
    return frontier_goals_entry(c, true, B, d_starts, d_goals, p, n_cams, cams, min_gain, max_fields, d_out, info, (cudaStream_t)cuda_stream);
}

// ---- planning step: PlannerManager::generateTraj for B (start, goal) pairs (include/isdf.h) --------------------------------------------
// The stages are the existing entry points' internals on device buffers: path_run, isdf_path_waypoints, one ragged midend_batch_run, the
// batched gather with set_as_points, one ragged lbfgs_rounds over callback_batch_launch, one ragged k_minco_forward for the final
// trajectories, then certify_run and dynamics_run with N0 = N per group of plans with the same N.
extern "C" int isdf_plan_default_params(isdf_ctx *c, isdf_plan_params *p) {
    if (!p) return fail(ISDF_ERR_INVALID, "params is NULL");
    std::memset(p, 0, sizeof(*p));
    isdf_config d;
    isdf_default_config(&d);
    const isdf_config &g = c ? c->cfg : d;
    p->parlength = 3.0;                                             // traj_parlength (plan_manager.cpp:153)
    p->half_extent = g.kernel_size * g.occupancy_resolution / 3.0;  // (:135, :243)
    p->rho = 20.0;
    isdf_midend_default_params(&p->midend);
    isdf_lbfgs_default_params(&p->backend);
    p->backend.max_iterations = 10000;                              // LMBM's cap (lmbm.h:20-57), taken as an analogue
    p->flags = ISDF_PLAN_CERTIFY | ISDF_PLAN_DYNAMICS;
    isdf_certify_default_params(&p->certify);
    isdf_dynamics_default_params(c, &p->dynamics);
    return 0;
}

extern "C" int isdf_get_plan_info(isdf_ctx *c, isdf_plan_info *out) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    *out = c->plan.info;
    return 0;
}

// every check that needs no device work; *r_cert: the certificate's body radius (ISDF_PLAN_CERTIFY)
static int plan_check(isdf_ctx *c, const isdf_plan_params *p, double *r_cert) {
    if (int r = frontend_state(c)) return r;
    if (!c->mesh.have_shape) return fail(ISDF_ERR_STATE, "shape not set");
    if (c->world > 1) return fail(ISDF_ERR_UNSUPPORTED, "the planning step is not sharded: call it on a context with isdf_set_shard(ctx, 0, 1)");
    if (p->reserved_ != 0) return fail(ISDF_ERR_INVALID, "reserved_ must be 0");
    if (p->flags & ~(ISDF_PLAN_CERTIFY | ISDF_PLAN_DYNAMICS | ISDF_PLAN_KNOWN_PREFIX | ISDF_PLAN_KNOWN_ONLY)) return fail(ISDF_ERR_INVALID, "unknown flags");
    double cw;
    if (int r = frontpath_params_check(&p->frontpath, &cw)) return r;
    if (!(std::isfinite(p->parlength) && p->parlength > 0.0)) return fail(ISDF_ERR_INVALID, "parlength must be finite and positive");
    if (!(std::isfinite(p->half_extent) && p->half_extent >= 0.0)) return fail(ISDF_ERR_INVALID, "half_extent must be finite and >= 0");
    for (double v : {p->offset[0], p->offset[1], p->offset[2], p->rho}) if (!std::isfinite(v)) return fail(ISDF_ERR_INVALID, "offset and rho must be finite");
    if (Layout L; int r = midend_check(c, false, 1, 1, nullptr, &p->midend, &L)) return r;
    if (int r = lbfgs_check(&p->backend)) return r;
    if (p->flags & ISDF_PLAN_CERTIFY) {
        if (p->certify.clearance.pieces_per_traj != 0) return fail(ISDF_ERR_INVALID, "certify.clearance.pieces_per_traj must be 0 (the call sets N0 = N)");
        if (int r = certify_check(c, 1, &p->certify, r_cert)) return r;
    }
    if (p->flags & ISDF_PLAN_DYNAMICS) {
        if (p->dynamics.pieces_per_traj != 0) return fail(ISDF_ERR_INVALID, "dynamics.pieces_per_traj must be 0 (the call sets N0 = N)");
        if (int r = dynamics_check(c, 1, &p->dynamics)) return r;
    }
    return 0;
}

// The outputs of the planning pipeline, in device memory in include/isdf.h's layout: the caller's (the device forms) or Staging's (the
// host forms). path_xyz is NULL in the host forms, which read the paths' nodes from c->fp.d_xyz.
struct PlanOut {
    int32_t *path_off = nullptr, *piece_off = nullptr;
    double *path_xyz = nullptr, *T = nullptr, *coeffs = nullptr;
    PlanResult *res = nullptr; CertSummary *cert = nullptr; DynSummary *dyn = nullptr;
    bool want_xyz = false;   // the paths' nodes are an output
    bool sized = false;      // path_off (when wanted) and piece_off hold the sizes
    int nodes = 0, pieces = 0;
};
static_assert(sizeof(isdf_plan_result) == sizeof(PlanResult) && offsetof(isdf_plan_result, path_cost) == offsetof(PlanResult, path_cost) &&
              offsetof(isdf_plan_result, duration) == offsetof(PlanResult, duration), "isdf_plan_result layout");
static_assert(sizeof(isdf_certify_summary) == sizeof(CertSummary) && offsetof(isdf_certify_summary, voxel_min) == offsetof(CertSummary, voxel_min) &&
              offsetof(isdf_certify_summary, depth) == offsetof(CertSummary, depth), "isdf_certify_summary layout");

// a host array of the pipeline's launch layouts to the device on st
template <typename T>
static int plan_upload(isdf_ctx *c, DevBuf<T> &buf, const std::vector<T> &h, cudaStream_t st) {
    CU_TRY(buf.ensure(std::max<size_t>(h.size(), 1)));
    if (h.empty()) return 0;
    CU_TRY(cudaMemcpyAsync(buf.p, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice, st));
    count_copy(c, cudaMemcpyHostToDevice, sizeof(T) * h.size());
    return 0;
}

// one copy stage: every segment in one launch
static int copy_segments(isdf_ctx *c, const std::vector<CopySeg> &seg, cudaStream_t st) {
    if (seg.empty()) return 0;
    if (int r = plan_upload(c, c->plan.d_seg, seg, st)) return r;
    k_copy_segments<<<(unsigned)seg.size(), 128, 0, st>>>(c->plan.d_seg.p);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}

template <typename S>
static int plan_fill(isdf_ctx *c, int n, const S &v, S *out, cudaStream_t st) {
    k_plan_fill<S><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n, v, out);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}

// The pipeline on stream st. Per plan, only the path lengths and found flags, N, the mid-end return codes and the gathered point counts
// cross to the host, besides the rounds' 4-byte reads; everything sized by nodes, waypoints or pieces stays on the device.
// d_heads (may be NULL): the plans' head states p, v, a (9 per plan, on the device) in place of [path.front(), 0, 0].
static int plan_run(isdf_ctx *c, int B, const double *starts, int sstride, const double *d_heads, const double *goals, int max_fields,
                    const isdf_plan_params *p, double r_cert, int cap_nodes, int cap_pieces, PlanOut &o, cudaStream_t st) {
    auto &z = c->plan;
    isdf_plan_info &info = z.info;
    info = {};
    for (cudaEvent_t &e : z.ev) if (!e) CU_TRY(cudaEventCreate(&e));
    // the device time of one stage's work on st, added to acc
    auto timed = [&](double &acc, auto body) -> int {
        CU_TRY(cudaEventRecord(z.ev[0], st));
        if (int r = body()) return r;
        CU_TRY(cudaEventRecord(z.ev[1], st));
        CU_TRY(cudaEventSynchronize(z.ev[1]));
        float ms = 0;
        CU_TRY(cudaEventElapsedTime(&ms, z.ev[0], z.ev[1]));
        acc += ms;
        return 0;
    };
    // 1. front end
    std::vector<int> off;
    const double cw = 1.0 + p->frontpath.unknown_weight;   // checked by plan_check
    const bool known_only = p->flags & ISDF_PLAN_KNOWN_ONLY;
    if (int r = timed(info.frontend_ms, [&] { return path_run(c, B, starts, sstride, goals, cw, max_fields, 0x7fffffff, off, st, known_only); }))
        return r;
    const int nodes = off[B];
    const int32_t *d_off = c->fp.d_off.p;
    const double *d_xyz = c->fp.d_xyz.p;
    // 2. waypoints: N and the rows of every path at wp_off (z.d_N = [N | wp_off])
    CU_TRY(z.d_pwp.ensure((size_t)3 * std::max(nodes, 1))); CU_TRY(z.d_N.ensure((size_t)2 * B + 1));
    if (int r = waypoints_run(c, B, d_off, d_xyz, c->map.grid.res, p->parlength, nodes, z.d_pwp.p, z.d_N.p + B, z.d_N.p, nullptr, st)) return r;
    std::vector<uint8_t> found(B);
    std::vector<int> N(B);
    CU_TRY(cudaMemcpyAsync(found.data(), c->fp.d_found.p, B, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaMemcpyAsync(N.data(), z.d_N.p, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    count_copy(c, cudaMemcpyDeviceToHost, B); count_copy(c, cudaMemcpyDeviceToHost, sizeof(int) * B);
    CU_TRY(cudaStreamSynchronize(st));
    // stages known before the mid-end, sizes
    std::vector<int> poff((size_t)B + 1, 0), wpo((size_t)B + 1, 0);   // piece offsets; wp_off as the device holds it
    std::vector<PlanRow> row(B);
    for (int b = 0; b < B; b++) {
        const bool traj = found[b] && minco_smem_bytes(N[b]) <= 220 * 1024;   // N <= 290 (minco_fits)
        const long long t = (long long)poff[b] + (traj ? N[b] : 0);
        if (t > 0x7fffffffll) return fail(ISDF_ERR_INVALID, "the trajectories hold more than 2^31 - 1 pieces");
        poff[b + 1] = (int)t;
        wpo[b + 1] = wpo[b] + N[b] - 1;
        // OPTIMISED: pending until the mid-end
        row[b] = {!found[b] ? ISDF_PLAN_NO_PATH : (traj ? ISDF_PLAN_OPTIMISED : ISDF_PLAN_TOO_LONG), off[b + 1] - off[b], found[b] ? N[b] : 0, 0, -1, -1};
    }
    if (o.path_off) CU_TRY(cudaMemcpyAsync(o.path_off, d_off, sizeof(int32_t) * ((size_t)B + 1), cudaMemcpyDeviceToDevice, st));
    CU_TRY(cudaMemcpyAsync(o.piece_off, poff.data(), sizeof(int32_t) * poff.size(), cudaMemcpyHostToDevice, st));
    count_copy(c, cudaMemcpyHostToDevice, sizeof(int32_t) * poff.size());
    o.sized = true; o.nodes = nodes; o.pieces = poff[B];
    if ((o.want_xyz && nodes > cap_nodes) || poff[B] > cap_pieces)
        return fail(ISDF_ERR_INVALID, "cap_nodes or cap_pieces too small (path_off / piece_off report the sizes needed)");
    if (o.path_xyz && nodes) CU_TRY(cudaMemcpyAsync(o.path_xyz, d_xyz, sizeof(double) * 3 * (size_t)nodes, cudaMemcpyDeviceToDevice, st));
    // 3-6. one ragged mid-end over every plan that reaches it, one gather and one ragged back end over the plans that pass it, in pair order
    std::vector<int> idx;   // the plans that reach the mid-end
    for (int b = 0; b < B; b++) if (row[b].stage == ISDF_PLAN_OPTIMISED) idx.push_back(b);
    std::vector<int> Ns;
    for (const int b : idx) Ns.push_back(N[b]);
    std::sort(Ns.begin(), Ns.end());
    Ns.erase(std::unique(Ns.begin(), Ns.end()), Ns.end());
    info.groups = (int)Ns.size();
    const int Bg = (int)idx.size();
    const double *d_mf = nullptr, *d_bf = nullptr;
    const int *d_mi = nullptr, *d_bi = nullptr;
    int Bp = 0;
    if (Bg > 0) {
        // plan idx[q] owns mid-end pieces [moff[q], moff[q+1]) and waypoint rows [moff[q] - q, moff[q+1] - q - 1); z.d_bc = [heads | tails]
        std::vector<int> moff((size_t)Bg + 1, 0);
        for (int q = 0; q < Bg; q++) moff[q + 1] = moff[q] + N[idx[q]];
        const size_t MP = (size_t)moff[Bg];
        Layout ML;
        if (int r = midend_check(c, true, Bg, 0, moff.data(), &p->midend, &ML)) return r;
        if (int r = ragged_upload(c->mid.d_off, moff.data(), st, &ML)) return r;
        count_copy(c, cudaMemcpyHostToDevice, sizeof(int) * (2 * (size_t)Bg + 2));
        if (int r = plan_upload(c, z.d_idx, idx, st)) return r;
        CU_TRY(z.d_bc.ensure((size_t)18 * Bg)); CU_TRY(z.d_wp.ensure(3 * std::max<size_t>(MP - Bg, 1)));
        k_plan_bc<<<(unsigned)((Bg + 127) / 128), 128, 0, st>>>(Bg, z.d_idx.p, d_off, d_xyz, d_heads, z.d_bc.p);
        c->stats.kernel_launches++;
        CU_TRY(cudaGetLastError());
        std::vector<CopySeg> seg;
        for (int q = 0; q < Bg; q++) {
            const int b = idx[q];
            if (N[b] > 1) seg.push_back({z.d_pwp.p + 3 * (size_t)wpo[b], z.d_wp.p + 3 * ((size_t)moff[q] - q), 3 * (long long)(N[b] - 1)});
        }
        if (int r = copy_segments(c, seg, st)) return r;
        CU_TRY(z.d_mx.ensure(ML.X)); CU_TRY(z.d_mres.ensure(19 * MP + Bg)); CU_TRY(z.d_mi.ensure((size_t)3 * Bg));
        double *mf = z.d_mres.p, *d_mT = mf + Bg, *d_mC = d_mT + MP;   // [f | T | coeffs]
        int mrounds = 0;
        if (int r = timed(info.midend_ms, [&] {
                return midend_batch_run(c, ML, z.d_bc.p, z.d_bc.p + 9 * (size_t)Bg, 1, &p->midend, z.d_wp.p, z.d_mx.p, d_mT, d_mC, mf, z.d_mi.p,
                                        z.d_mi.p + Bg, z.d_mi.p + 2 * (size_t)Bg, &mrounds, st);
            })) return r;
        d_mf = mf; d_mi = z.d_mi.p;
        std::vector<int> mi(Bg);
        CU_TRY(cudaMemcpyAsync(mi.data(), z.d_mi.p, sizeof(int) * Bg, cudaMemcpyDeviceToHost, st));
        count_copy(c, cudaMemcpyDeviceToHost, sizeof(int) * Bg);
        CU_TRY(cudaStreamSynchronize(st));
        std::vector<int> ok, pos(Bg, -1);   // the plans that passed the mid-end (plan_manager.cpp:277) and their back-end instance
        for (int q = 0; q < Bg; q++) {
            row[idx[q]].q = q;
            if (mi[q] >= 0) { pos[q] = (int)ok.size(); ok.push_back(q); }
            else row[idx[q]].stage = ISDF_PLAN_MIDEND_FAILED;
        }
        Bp = (int)ok.size();
        std::vector<int> boff((size_t)Bp + 1, 0);   // back-end instance k owns pieces [boff[k], boff[k+1])
        for (int k = 0; k < Bp; k++) boff[k + 1] = boff[k] + N[idx[ok[k]]];
        const size_t BP = (size_t)boff[Bp];
        if (Bp > 0) {
            // 4. the passed plans' obstacle lists become the batched point sets
            std::vector<int> gwo((size_t)Bp + 1, 0);
            CU_TRY(c->gat.d_wp.ensure(3 * std::max<size_t>(BP - Bp, 1)));
            seg.clear();
            for (int k = 0; k < Bp; k++) {
                const int q = ok[k], W = N[idx[q]] - 1;
                gwo[k + 1] = gwo[k] + W;
                if (W) seg.push_back({z.d_wp.p + 3 * ((size_t)moff[q] - q), c->gat.d_wp.p + 3 * (size_t)gwo[k], 3 * (long long)W});
            }
            if (int r = copy_segments(c, seg, st)) return r;
            if (int r = plan_upload(c, c->gat.d_wpoff, gwo, st)) return r;
            std::vector<int> bplan(Bp);   // back-end instance k's plan
            for (int k = 0; k < Bp; k++) bplan[k] = idx[ok[k]];
            if (int r = plan_upload(c, z.d_bplan, bplan, st)) return r;
            const int *d_krows = nullptr;   // ISDF_PLAN_KNOWN_PREFIX: each instance's rows inside its path's known prefix
            if (known_only) {   // every row: the path is known but for its start
                std::vector<int> kr(Bp);
                for (int k = 0; k < Bp; k++) kr[k] = gwo[k + 1] - gwo[k];
                if (int r = plan_upload(c, z.d_krows, kr, st)) return r;
                d_krows = z.d_krows.p;
            } else if (p->flags & ISDF_PLAN_KNOWN_PREFIX) {
                CU_TRY(z.d_krows.ensure(Bp));
                k_plan_known_rows<<<(unsigned)((Bp + 127) / 128), 128, 0, st>>>(Bp, z.d_bplan.p, d_off, c->fp.d_nodes.p,
                                                                                c->known.have ? c->known.d_known.p : nullptr, c->map.grid,
                                                                                c->wps.d_gap.p, z.d_N.p, z.d_krows.p);
                c->stats.kernel_launches++;
                CU_TRY(cudaGetLastError());
                d_krows = z.d_krows.p;
            }
            std::vector<int> pto;
            long long tot = 0;
            if (int r = timed(info.gather_ms, [&] {
                    if (int rr = gather_batch_run(c, Bp, gwo.data(), c->gat.d_wpoff.p, c->gat.d_wp.p, p->half_extent, p->offset, d_krows, 0x7fffffffll,
                                                  pto, &tot, st)) return rr;
                    return gather_set_points(c, Bp, pto, tot, st);
                })) return r;
            for (int k = 0; k < Bp; k++) { row[idx[ok[k]]].points = pto[k + 1] - pto[k]; row[idx[ok[k]]].k = k; }
            // 5. persisted durations: what updateTraj(mid-end trajectory) leaves on a fresh context (swm:287-296)
            if (int r = plan_upload(c, z.d_ok, ok, st)) return r;
            CU_TRY(z.d_dur.ensure(Bp));
            k_plan_durations<<<(unsigned)((Bp + 127) / 128), 128, 0, st>>>(Bp, z.d_ok.p, ML.d_off, d_mT, z.d_dur.p);
            c->stats.kernel_launches++;
            CU_TRY(cudaGetLastError());
            CU_TRY(c->sv.set_durations(Bp, z.d_dur.p, st, cudaMemcpyDeviceToDevice));
            // 6. back end from the mid-end x
            Layout BL;
            if (int r = callback_batch_check(c, true, Bp, 0, boff.data(), &BL)) return r;
            if (int r = ragged_upload(c->batch.d_off, boff.data(), st, &BL)) return r;
            count_copy(c, cudaMemcpyHostToDevice, sizeof(int) * (2 * (size_t)Bp + 2));
            CU_TRY(z.d_bbc.ensure((size_t)18 * Bp));
            k_plan_bc<<<(unsigned)((Bp + 127) / 128), 128, 0, st>>>(Bp, z.d_bplan.p, d_off, d_xyz, d_heads, z.d_bbc.p);
            c->stats.kernel_launches++;
            CU_TRY(cudaGetLastError());
            const double *d_bh = z.d_bbc.p, *d_bt = z.d_bbc.p + 9 * (size_t)Bp;
            CU_TRY(z.d_bx.ensure(BL.X)); CU_TRY(z.d_bf.ensure(Bp)); CU_TRY(z.d_bi.ensure((size_t)3 * Bp));
            seg.clear();
            for (int k = 0; k < Bp; k++) {
                const int q = ok[k];
                seg.push_back({z.d_mx.p + 4 * (size_t)moff[q] - 3 * (size_t)q, z.d_bx.p + 4 * (size_t)boff[k] - 3 * (size_t)k, 4 * (long long)N[idx[q]] - 3});
            }
            if (int r = copy_segments(c, seg, st)) return r;
            int brounds = 0;
            if (int r = timed(info.backend_ms, [&]() -> int {
                    if (int rr = lbfgs_rounds(c, c->lbfgs, Bp, 4 * BL.N - 3, BL.d_xoff, BL.X, &p->backend, 0, z.d_bx.p, z.d_bf.p, z.d_bi.p, z.d_bi.p + Bp,
                                              z.d_bi.p + 2 * (size_t)Bp, &brounds, st, [&](const double *x, double *f, double *g) {
                                                  return callback_batch_launch(c, BL, d_bh, d_bt, 9, p->rho, x, f, g, st);
                                              })) return rr;
                    // the final trajectories: forwardT + MINCO of the returned x (back_end_optimizer.cpp:140-163), into the batch trajectories
                    MincoArgs M = c->batch.minco.args(BL, d_bh, d_bt, 9, p->rho, z.d_bx.p);
                    k_minco_forward<<<Bp, 32, minco_smem_bytes(BL.N), st>>>(M);
                    c->stats.kernel_launches++;
                    CU_TRY(cudaGetLastError());
                    c->batch.B = Bp; c->batch.P = BP;
                    return 0;
                })) return r;
            info.backend_rounds = brounds;
            d_bf = z.d_bf.p; d_bi = z.d_bi.p;
        }
        // the returned trajectories, plan b's at piece_off[b]: the back end's, or the mid-end's for MIDEND_FAILED
        seg.clear();
        for (int q = 0; q < Bg; q++) {
            const bool be = pos[q] >= 0;
            const int Nq = N[idx[q]];
            const size_t po = (size_t)poff[idx[q]], p0 = be ? (size_t)boff[pos[q]] : (size_t)moff[q], rows = 6 * (be ? BP : MP);
            const double *sT = be ? c->batch.minco.d_T.p : d_mT, *sC = be ? c->batch.minco.d_C.p : d_mC;
            seg.push_back({sT + p0, o.T + po, Nq});
            for (int a = 0; a < 3; a++) seg.push_back({sC + a * rows + 6 * p0, o.coeffs + 18 * po + 6 * (size_t)a * Nq, 6 * (long long)Nq});
        }
        if (int r = copy_segments(c, seg, st)) return r;
    }
    // the result records
    if (int r = plan_upload(c, z.d_row, row, st)) return r;
    k_plan_results<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(B, z.d_row.p, c->fp.d_cost.p, d_mf, d_mi, d_bf, d_bi, Bp, o.piece_off, o.T, o.res);
    c->stats.kernel_launches++;
    CU_TRY(cudaGetLastError());
    // 7. certificates on every returned trajectory, per group of plans with the same N, ascending; a plan without one reads as a failed call
    if (o.cert) if (int r = plan_fill(c, B, same_layout<CertSummary>(certify_failed_summary()), o.cert, st)) return r;
    if (o.dyn) if (int r = plan_fill(c, B, same_layout<DynSummary>(dynamics_failed_summary()), o.dyn, st)) return r;
    if (p->flags & (ISDF_PLAN_CERTIFY | ISDF_PLAN_DYNAMICS)) {
        for (const int Ng : Ns) {
            std::vector<int> gi;   // the group's plans, in pair order
            for (const int b : idx) if (N[b] == Ng) gi.push_back(b);
            const int Bn = (int)gi.size();
            const size_t BN = (size_t)Bn * Ng;
            // the group's trajectories as one block (piece q*N + i of a 6BN x 3 column-major block)
            CU_TRY(z.d_gT.ensure(BN)); CU_TRY(z.d_gC.ensure(18 * BN));
            std::vector<CopySeg> seg;
            for (int q = 0; q < Bn; q++) {
                const size_t po = (size_t)poff[gi[q]];
                seg.push_back({o.T + po, z.d_gT.p + (size_t)q * Ng, Ng});
                for (int a = 0; a < 3; a++) seg.push_back({o.coeffs + 18 * po + 6 * (size_t)a * Ng, z.d_gC.p + 6 * ((size_t)a * BN + (size_t)q * Ng), 6 * (long long)Ng});
            }
            if (int r = copy_segments(c, seg, st)) return r;
            if (int r = plan_upload(c, z.d_gi, gi, st)) return r;
            if (p->flags & ISDF_PLAN_CERTIFY) {
                isdf_certify_params pc = p->certify;
                pc.clearance.pieces_per_traj = Ng;
                double rr = r_cert;
                if (int r = certify_check(c, (int)BN, &pc, &rr)) return r;
                CU_TRY(z.d_csum.ensure(Bn));
                if (int r = timed(info.certify_ms, [&] { return certify_run(c, (int)BN, z.d_gT.p, z.d_gC.p, &pc, rr, z.d_csum.p, st); })) return r;
                k_plan_scatter<CertSummary><<<(unsigned)((Bn + 127) / 128), 128, 0, st>>>(Bn, z.d_gi.p, z.d_csum.p, o.cert);
                c->stats.kernel_launches++;
                CU_TRY(cudaGetLastError());
            }
            if (p->flags & ISDF_PLAN_DYNAMICS) {
                isdf_dynamics_params pd = p->dynamics;
                pd.pieces_per_traj = Ng;
                if (int r = dynamics_check(c, (int)BN, &pd)) return r;
                CU_TRY(z.d_dsum.ensure(Bn));
                if (int r = timed(info.dynamics_ms, [&] { return dynamics_run(c, (int)BN, z.d_gT.p, z.d_gC.p, &pd, z.d_dsum.p, st); })) return r;
                k_plan_scatter<DynSummary><<<(unsigned)((Bn + 127) / 128), 128, 0, st>>>(Bn, z.d_gi.p, z.d_dsum.p, o.dyn);
                c->stats.kernel_launches++;
                CU_TRY(cudaGetLastError());
            }
        }
    }
    CU_TRY(cudaStreamSynchronize(st));
    return 0;
}

// the planning calls (starts: sstride 0 for one start, on the host in every form; sstride 9 for start states p, v, a). dev: goals, starts
// (sstride 3 or 9) and every output in device memory, the call on st; else host memory, the outputs staged through Staging on ctx's stream
// (st). One pipeline, plan_run, for both.
static int plan_entry(isdf_ctx *c, bool dev, int B, const double *starts, int sstride, const double *goals, const isdf_plan_params *p, int max_fields,
                      int cap_nodes, int32_t *path_off, double *path_xyz, int cap_pieces, int32_t *piece_off, double *T, double *coeffs,
                      isdf_plan_result *results, isdf_certify_summary *certify, isdf_dynamics_summary *dynamics, cudaStream_t st) {
    bool started = false;
    const int rc = poison_on_failure([&]() -> int {
        if (!c) return fail(ISDF_ERR_INVALID, "ctx is NULL");
        if (!starts || !goals || B < 1 || !p || !piece_off || !results || cap_pieces < 0 || (cap_pieces > 0 && (!T || !coeffs)) ||
            (path_xyz && (!path_off || cap_nodes < 0)))
            return fail(ISDF_ERR_INVALID, "NULL argument, B < 1 or a cap < 0");
        if (max_fields < 0) return fail(ISDF_ERR_INVALID, "max_fields < 0");
        if (((p->flags & ISDF_PLAN_CERTIFY) && !certify) || ((p->flags & ISDF_PLAN_DYNAMICS) && !dynamics))
            return fail(ISDF_ERR_INVALID, "a summary array of a requested certificate is NULL");
        if (sstride == 9 && !dev)
            for (int b = 0; b < B; b++)
                for (int k = 3; k < 9; k++)
                    if (!std::isfinite(starts[9 * (size_t)b + k]))
                        return fail(ISDF_ERR_INVALID, "starts[" + std::to_string(b) + "]: velocity or acceleration is not finite");
        double r_cert = 0.0;
        if (int r = plan_check(c, p, &r_cert)) return r;
        if (set_device(c)) return ISDF_ERR_CUDA;
        started = true;
        std::fill(c->xfer, c->xfer + 4, 0ll);
        PlanOut o;
        o.want_xyz = path_xyz != nullptr;
        auto *res = reinterpret_cast<PlanResult *>(results);
        auto *cert = reinterpret_cast<CertSummary *>(certify);
        auto *dyn = reinterpret_cast<DynSummary *>(dynamics);
        std::vector<double> hs, hg;
        Staging S(c);
        const double *d_heads = sstride == 9 && dev ? starts : nullptr;
        if (dev) {
            if (int r = read_endpoints(c, B, starts, sstride, goals, hs, hg, st)) return r;
            o.path_off = path_off; o.path_xyz = path_xyz; o.piece_off = piece_off; o.T = T; o.coeffs = coeffs; o.res = res; o.cert = cert; o.dyn = dyn;
        } else {   // cert and dyn only when asked for: each is one more fill launch. T and coeffs: room for cap_pieces, read back below
            S.out(&o.piece_off, piece_off, (size_t)B + 1); S.out(&o.res, res, (size_t)B);
            if (path_off) S.out(&o.path_off, path_off, (size_t)B + 1);
            if (cert) S.out(&o.cert, cert, (size_t)B);
            if (dyn) S.out(&o.dyn, dyn, (size_t)B);
            S.out(&o.T, nullptr, (size_t)cap_pieces); S.out(&o.coeffs, nullptr, 18 * (size_t)cap_pieces);
            if (sstride == 9) S.in(&d_heads, starts, 9 * (size_t)B);
            if (int r = S.upload()) return r;
        }
        int r = plan_run(c, B, starts, sstride, d_heads, goals, max_fields, p, r_cert, cap_nodes, cap_pieces, o, st);
        if (dev || !o.sized) return r;   // a host form that failed before the sizes leaves path_off and piece_off as they were
        // the paths' nodes and the used prefix of T and coeffs after a success, then the staged outputs, whose offsets report the sizes also
        // after a failure (the results and summaries are poisoned then)
        auto get = [&](void *dst, const void *src, size_t bytes) -> int {
            if (!bytes) return 0;
            CU_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
            count_copy(c, cudaMemcpyDeviceToHost, bytes);
            return 0;
        };
        if (!r && path_xyz) r = get(path_xyz, c->fp.d_xyz.p, sizeof(double) * 3 * (size_t)o.nodes);
        if (!r) r = get(T, o.T, sizeof(double) * (size_t)o.pieces);
        if (!r) r = get(coeffs, o.coeffs, sizeof(double) * 18 * (size_t)o.pieces);
        const int rb = S.download();
        count_copy(c, cudaMemcpyDeviceToHost, S.download_bytes());
        return r ? r : rb;
    }, [&] {
        if (B < 1) return;
        isdf_plan_result bad = {};
        bad.stage = ISDF_PLAN_FAILED;
        bad.path_cost = bad.midend_f = bad.backend_f = bad.duration = std::numeric_limits<double>::quiet_NaN();
        isdf_ctx *dc = dev ? c : nullptr;   // device outputs: written after st, best effort
        if (dev && !c) return;
        if (results) write_failed_summaries(results, B, bad, dc, st);
        if (certify) write_failed_summaries(certify, B, certify_failed_summary(), dc, st);
        if (dynamics) write_failed_summaries(dynamics, B, dynamics_failed_summary(), dc, st);
    });
    if (started) {
        c->sv.set_points(nullptr, 0, st);   // both point sets given up, the batched swept-volume term off
        std::copy(c->xfer, c->xfer + 4, c->plan.xfer);
    }
    return rc;
}

extern "C" int isdf_plan_batch(isdf_ctx *c, const double *start, int B, const double *goals, const isdf_plan_params *p, int cap_nodes,
                               int32_t *path_off, double *path_xyz, int cap_pieces, int32_t *piece_off, double *T, double *coeffs,
                               isdf_plan_result *results, isdf_certify_summary *certify, isdf_dynamics_summary *dynamics) {
    return plan_entry(c, false, B, start, 0, goals, p, 0, cap_nodes, path_off, path_xyz, cap_pieces, piece_off, T, coeffs, results, certify,
                      dynamics, c ? c->stream : nullptr);
}

extern "C" int isdf_plan_pairs(isdf_ctx *c, int B, const double *starts, const double *goals, const isdf_plan_params *p, int max_fields,
                               int cap_nodes, int32_t *path_off, double *path_xyz, int cap_pieces, int32_t *piece_off, double *T, double *coeffs,
                               isdf_plan_result *results, isdf_certify_summary *certify, isdf_dynamics_summary *dynamics) {
    return plan_entry(c, false, B, starts, 3, goals, p, max_fields, cap_nodes, path_off, path_xyz, cap_pieces, piece_off, T, coeffs, results, certify,
                      dynamics, c ? c->stream : nullptr);
}

extern "C" int isdf_plan_batch_device(isdf_ctx *c, const double *start, int B, const double *d_goals, const isdf_plan_params *p, int cap_nodes,
                                      int32_t *d_path_off, double *d_path_xyz, int cap_pieces, int32_t *d_piece_off, double *d_T, double *d_coeffs,
                                      isdf_plan_result *d_results, isdf_certify_summary *d_certify, isdf_dynamics_summary *d_dynamics,
                                      void *cuda_stream) {
    return plan_entry(c, true, B, start, 0, d_goals, p, 0, cap_nodes, d_path_off, d_path_xyz, cap_pieces, d_piece_off, d_T, d_coeffs, d_results,
                      d_certify, d_dynamics, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_plan_pairs_device(isdf_ctx *c, int B, const double *d_starts, const double *d_goals, const isdf_plan_params *p, int max_fields,
                                      int cap_nodes, int32_t *d_path_off, double *d_path_xyz, int cap_pieces, int32_t *d_piece_off, double *d_T,
                                      double *d_coeffs, isdf_plan_result *d_results, isdf_certify_summary *d_certify,
                                      isdf_dynamics_summary *d_dynamics, void *cuda_stream) {
    return plan_entry(c, true, B, d_starts, 3, d_goals, p, max_fields, cap_nodes, d_path_off, d_path_xyz, cap_pieces, d_piece_off, d_T, d_coeffs,
                      d_results, d_certify, d_dynamics, (cudaStream_t)cuda_stream);
}

extern "C" int isdf_plan_states(isdf_ctx *c, int B, const double *starts, const double *goals, const isdf_plan_params *p, int max_fields,
                                int cap_nodes, int32_t *path_off, double *path_xyz, int cap_pieces, int32_t *piece_off, double *T, double *coeffs,
                                isdf_plan_result *results, isdf_certify_summary *certify, isdf_dynamics_summary *dynamics) {
    return plan_entry(c, false, B, starts, 9, goals, p, max_fields, cap_nodes, path_off, path_xyz, cap_pieces, piece_off, T, coeffs, results, certify,
                      dynamics, c ? c->stream : nullptr);
}

extern "C" int isdf_plan_states_device(isdf_ctx *c, int B, const double *d_starts, const double *d_goals, const isdf_plan_params *p, int max_fields,
                                       int cap_nodes, int32_t *d_path_off, double *d_path_xyz, int cap_pieces, int32_t *d_piece_off, double *d_T,
                                       double *d_coeffs, isdf_plan_result *d_results, isdf_certify_summary *d_certify,
                                       isdf_dynamics_summary *d_dynamics, void *cuda_stream) {
    return plan_entry(c, true, B, d_starts, 9, d_goals, p, max_fields, cap_nodes, d_path_off, d_path_xyz, cap_pieces, d_piece_off, d_T, d_coeffs,
                      d_results, d_certify, d_dynamics, (cudaStream_t)cuda_stream);
}

// what the last planning call moved between host and device, counted at the pipeline's copy sites: out = {device-to-host bytes outside
// the rounds' 4-byte reads, the rounds' reads, host-to-device bytes, copies (reads included)}
extern "C" int isdf_dbg_plan_transfers(isdf_ctx *c, int64_t *out) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    for (int k = 0; k < 4; k++) out[k] = c->plan.xfer[k];
    return 0;
}

// the traversability bits of the last path or field call (X*Y*ceil(Z/32) words of the map it ran on, grid.bits' layout)
// the feasibility pipeline the last front-end feasibility run (masks or traversability) chose: out = {pipeline: 0 one pass, 1 kernel core +
// offset-mask survivors, 2 kernel core words + table survivors; blocks; threads} of its mask-accumulation kernel; pipeline -1 before any run
extern "C" int isdf_dbg_frontend_launch(isdf_ctx *c, int *out) {
    if (!c || !out) return fail(ISDF_ERR_INVALID, "NULL argument");
    for (int k = 0; k < 3; k++) out[k] = c->fe.last_launch[k];
    return 0;
}
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
    if (int r = offsets_check(offsets, B, "offsets", true)) return r;
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
    Staging S(c);
    const double *dgt = nullptr, *dgs = nullptr, *dgg = nullptr;
    if (g_t) { S.in(&dgt, g_t, (size_t)c->sv.P); S.in(&dgs, g_s, (size_t)c->sv.P); S.in(&dgg, g_g, (size_t)3 * c->sv.P); }
    return eval_host(c, S, N, T, coeffs, cost, gradC, gradT, &isdf_stats::last_sdf_evals,
                     [&](const double *d_T, const double *d_C, double *d_out, double *count_out) {
                         return swept_common(c, N, d_T, d_C, d_out, count_out, c->stream, dgt, dgs, dgg);
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
    Staging S(c);
    const double *dv, *dg;
    double *dout;
    S.in(&dv, vaj, (size_t)9 * n); S.in(&dg, grads, (size_t)10 * n); S.out(&dout, out, (size_t)16 * n);
    if (int r = S.upload()) return r;
    CU_TRY(discrete_launch_dbg_flatness(c->dcfg.fp, n, dv, dg, dout, c->stream));
    return S.download();
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
// sub-boxes per cell edge of the discrete scan's filtered lists, from the next isdf_set_shape_mesh on (1: the scan walks the full lists)
extern "C" int isdf_dbg_disc_k(isdf_ctx *c, int k) {
    if (!c || k < 1 || k > 8) return fail(ISDF_ERR_INVALID, "NULL context or k outside 1..8");
    c->mesh.disc_k = k;
    return 0;
}
// the discrete scan's filtered lists, so tests can hold them to the full ones: sizes = {candidates (0: not built, the scan walks the
// full lists), k}; cell_off / cell_cnt (one per cell, as isdf_dbg_mesh_grid) and cand / cand_lb (sizes[0] each) are optional
extern "C" int isdf_dbg_disc_lists(isdf_ctx *c, long long *sizes, uint32_t *cell_off, uint16_t *cell_cnt, uint32_t *cand, float *cand_lb) {
    if (!c || !sizes) return fail(ISDF_ERR_INVALID, "NULL argument");
    if (!c->mesh.have_shape || c->mesh.shape.kind != ISDF_SHAPE_MESH) return fail(ISDF_ERR_STATE, "no mesh shape set");
    const DevMesh &m = c->mesh.shape.mesh;
    const size_t ncell = (size_t)m.gdim[0] * m.gdim[1] * m.gdim[2];
    if (int r = sync_ctx(c)) return r;
    size_t total = 0;
    if (c->mesh.disc_ready) {
        uint32_t off_last = 0; uint16_t cnt_last = 0;
        CU_TRY(cudaMemcpy(&off_last, c->mesh.d_disc_off.p + ncell - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost));
        CU_TRY(cudaMemcpy(&cnt_last, c->mesh.d_disc_cnt.p + ncell - 1, sizeof(uint16_t), cudaMemcpyDeviceToHost));
        total = (size_t)off_last + cnt_last;
    }
    sizes[0] = (long long)total; sizes[1] = c->mesh.disc_k;
    if (!c->mesh.disc_ready) return 0;
    if (cell_off) CU_TRY(cudaMemcpy(cell_off, c->mesh.d_disc_off.p, sizeof(uint32_t) * ncell, cudaMemcpyDeviceToHost));
    if (cell_cnt) CU_TRY(cudaMemcpy(cell_cnt, c->mesh.d_disc_cnt.p, sizeof(uint16_t) * ncell, cudaMemcpyDeviceToHost));
    if (cand && total) CU_TRY(cudaMemcpy(cand, c->mesh.d_disc_cand.p, sizeof(uint32_t) * total, cudaMemcpyDeviceToHost));
    if (cand_lb && total) CU_TRY(cudaMemcpy(cand_lb, c->mesh.d_disc_lb.p, sizeof(float) * total, cudaMemcpyDeviceToHost));
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
    Staging S(c);
    const double *dC, *dT, *dta, *dtb;
    const int *dp;
    double *dout;
    S.in(&dC, coeffs, 18 * (size_t)N); S.in(&dT, T, (size_t)N); S.in(&dp, piece, (size_t)n); S.in(&dta, ta, (size_t)n); S.in(&dtb, tb, (size_t)n);
    S.out(&dout, out, 2 * (size_t)n);
    if (int rr = S.upload()) return rr;
    const CertArgs A = certify_args(c, r, reach, N, dT, dC);
    CU_TRY(certify_bound_launch(A, n, dp, dta, dtb, dout, c->stream));
    c->stats.kernel_launches++;
    return S.download();
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
