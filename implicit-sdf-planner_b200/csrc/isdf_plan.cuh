// The planning step's glue on the device (isdf_plan_pairs / isdf_plan_batch and their _device forms, include/isdf.h): waypoint selection,
// the mid-end's and back end's boundary conditions, ragged copies between the stages' buffers, the persisted durations and the result
// records. Everything that is proportional to path nodes, waypoints or pieces stays on the device; the host only lays out the launches.
//
// Waypoints (isdf_path_waypoints, plan_manager.cpp:206-213 and :235-245): k_wp_count runs the `pl /= 1.5` loop per path, one thread per
// path, with the host form's operations (one IEEE division or one ceil per step; the unit is compiled with -fmad=false, and nothing here
// could contract anyway). A path of S > 2 nodes takes the nodes g, 2g, ... < S - 1, which are (S - 2) / g of them. A scan of the counts gives
// wp_off, and k_wp_write copies the rows, one warp per path, leaving out rows at or past cap as the host form does.
#pragma once
#include "isdf_types.cuh"

namespace isdf {

__global__ void k_wp_count(int B, const int32_t *off, double res, double parlength, int32_t *cnt, int32_t *gap, int32_t *pieces, int32_t *wp_off) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b == 0) wp_off[0] = 0;
    if (b >= B) return;
    const long long S = (long long)off[b + 1] - off[b];
    long long n = 0, g = 0;
    if (S > 2) {
        double pl = parlength;
        double gp = ceil(pl / res);
        while (gp >= (double)(S - 1)) { pl /= 1.5; gp = ceil(pl / res); }
        g = (long long)gp;
        n = g > 0 ? (S - 2) / g : 0;   // g = 0 only when parlength / res underflows, where the host form does not terminate
    }
    cnt[b] = (int32_t)n; gap[b] = (int32_t)g; pieces[b] = (int32_t)(n + 1);
}

__global__ void k_wp_write(int B, const int32_t *off, const double *xyz, const int32_t *gap, const int32_t *wp_off, long long cap, double *wp) {
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= B) return;
    const long long o = wp_off[w], n = (long long)wp_off[w + 1] - o, g = gap[w], base = off[w];
    for (long long i = lane; i < 3 * n; i += 32) {
        const long long k = i / 3, row = o + k;
        if (row < cap) wp[3 * row + (i - 3 * k)] = xyz[3 * (base + (k + 1) * g) + (i - 3 * k)];
    }
}

// plan plan[i]'s boundary conditions: head = [path.front(), 0, 0] at bc + 9 i, tail = [path.back(), 0, 0] at bc + 9 (n + i) (3x3
// column-major, column 0 the position; plan_manager.cpp:220-223). heads (may be NULL): plan b's head is the state p, v, a at heads + 9 b
// (isdf_plan_states), which is the same column-major order.
__global__ void k_plan_bc(int n, const int *plan, const int32_t *path_off, const double *xyz, const double *heads, double *bc) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int b = plan[i];
    const double *f = xyz + 3 * (size_t)path_off[b], *l = xyz + 3 * ((size_t)path_off[b + 1] - 1);
    double *h = bc + 9 * (size_t)i, *t = bc + 9 * ((size_t)n + i);
    for (int k = 0; k < 9; k++) { h[k] = heads ? heads[9 * (size_t)b + k] : (k < 3 ? f[k] : 0.0); t[k] = k < 3 ? l[k] : 0.0; }
}

// ISDF_PLAN_KNOWN_PREFIX: the rows of back-end instance i (plan plan[i]) that lie inside its path's known prefix. k* = the first path node
// whose voxel is not known (the path length when every node is; 0 when nothing is known: known NULL); waypoint row j is path node
// (j + 1) gap (k_wp_write), so the known rows are the j < pieces - 1 with (j + 1) gap < k*.
__global__ void k_plan_known_rows(int n, const int *plan, const int32_t *path_off, const int *nodes, const uint32_t *known, const DevGrid G,
                                  const int32_t *gap, const int32_t *pieces, int *rows) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int b = plan[i];
    long long ks = 0;
    if (known)
        for (long long m = path_off[b]; m < path_off[b + 1]; m++, ks++) {
            const int *v = nodes + 3 * m;
            if (!((known[((size_t)v[0] * G.Y + v[1]) * G.Zw + (v[2] >> 5)] >> (v[2] & 31)) & 1u)) break;
        }
    int r = 0;
    while (r < pieces[b] - 1 && (long long)(r + 1) * gap[b] < ks) r++;
    rows[i] = r;
}

// isdf_plan_states_device's check of the heads' v and a: *bad = the least b whose v or a has a non-finite entry (left as set when none)
__global__ void k_plan_heads_check(int B, const double *heads, int *bad) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    bool ok = true;
    for (int k = 3; k < 9; k++) ok = ok && isfinite(heads[9 * (size_t)b + k]);
    if (!ok) atomicMin(bad, b);
}

// one ragged copy: n doubles from src to dst
struct CopySeg {
    const double *src;
    double *dst;
    long long n;
};
// every segment of a copy stage in one launch: one CTA per segment
__global__ void k_copy_segments(const CopySeg *seg) {
    const CopySeg s = seg[blockIdx.x];
    for (long long i = threadIdx.x; i < s.n; i += blockDim.x) s.dst[i] = s.src[i];
}

// the persisted duration of back-end problem k (mid-end instance q[k]): the left-to-right sum of its mid-end T when shorter than 300 s,
// else 0 (what updateTraj leaves on a fresh context, swm:287-296)
__global__ void k_plan_durations(int n, const int *q, const int *moff, const double *T, double *dur) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    double td = 0.0;
    for (int i = moff[q[k]]; i < moff[q[k] + 1]; i++) td += T[i];
    dur[k] = td < 3 * 1e2 ? td : 0.0;
}

// layout of isdf_plan_result
struct PlanResult {
    int32_t stage, path_nodes, pieces, obstacle_points, midend_ret, backend_ret, backend_iterations, backend_evaluations;
    double path_cost, midend_f, backend_f, duration;
};
static_assert(sizeof(PlanResult) == 64, "isdf_plan_result layout");

// what the host knows of plan b: stage, path nodes, pieces, obstacle points, its mid-end instance q and back-end instance k (-1: none)
struct PlanRow {
    int stage, nodes, pieces, points, q, k;
};

// plan b's record from its row, the front end's cost, the mid-end's and back end's outputs (nb back-end instances: ret, iterations and
// evaluations nb apart) and its returned trajectory at T + piece_off[b] (duration: its left-to-right sum)
__global__ void k_plan_results(int B, const PlanRow *row, const double *path_cost, const double *mf, const int *mi, const double *bf, const int *bi,
                               int nb, const int32_t *piece_off, const double *T, PlanResult *out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const PlanRow r = row[b];
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    PlanResult o;
    o.stage = r.stage; o.path_nodes = r.nodes; o.pieces = r.pieces; o.obstacle_points = r.points;
    o.midend_ret = r.q >= 0 ? mi[r.q] : 0;
    o.backend_ret = r.k >= 0 ? bi[r.k] : 0;
    o.backend_iterations = r.k >= 0 ? bi[nb + r.k] : 0;
    o.backend_evaluations = r.k >= 0 ? bi[2 * (size_t)nb + r.k] : 0;
    o.path_cost = path_cost[b];
    o.midend_f = r.q >= 0 ? mf[r.q] : nan;
    o.backend_f = r.k >= 0 ? bf[r.k] : nan;
    double td = 0.0;
    if (r.q >= 0) for (int i = 0; i < r.pieces; i++) td += T[piece_off[b] + i];
    o.duration = td;
    out[b] = o;
}

template <typename S>
__global__ void k_plan_fill(int n, const S v, S *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = v;
}

// out[at[i]] = in[i]
template <typename S>
__global__ void k_plan_scatter(int n, const int *at, const S *in, S *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[at[i]] = in[i];
}

}  // namespace isdf
