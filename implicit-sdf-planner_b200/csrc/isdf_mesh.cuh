// Device-side triangle-mesh signed distance: the Generalshape mesh path (Shape.cpp:105-151), which the reference
// evaluates with libigl's AABB tree (exact closest point) and fast winding number (sign).
//
// Device layout: a binary BVH whose nodes carry BOTH children's boxes (one 112-byte fetch decides the descent),
// leaves of <= 4 triangles stored in leaf order as (a, b-a, c-a), 7 pseudonormals per triangle (face, 3 edges,
// 3 vertices) for the sign, and a coarse body-frame inside/outside bitmap that resolves the sign of points that
// have no triangle within the query bound. The whole structure for a 4000-triangle robot is < 2 MB: L2-resident.
//
// Sign: for a closed, consistently oriented mesh the generalised winding number is exactly 0 outside / 1 inside,
// so s = 1 - 2w = ±1 (Shape.cpp:111). The device gets the same ±1 from the angle-weighted pseudonormal at the
// closest feature (Baerentzen & Aanaes 2005) — no O(#triangles) solid-angle sum per query.
#pragma once
#include "isdf_math.cuh"

namespace isdf {

struct BvhNode {       // 112 bytes
    double lbox[6];    // left child lo(3), hi(3)
    double rbox[6];    // right child
    int left, right;   // >= 0: node index; < 0: leaf, ~code with code = first_tri*4 + (count-1)
    int pad0, pad1;
};

// 32-ary node for WARP-COOPERATIVE queries: lane i owns child i (SoA boxes => one coalesced 256-byte load per plane).
// Built by collapsing five levels of the same binary tree, so leaves (<= 4 triangles) and triangle order are shared.
constexpr int WIDE_EMPTY = 0x7fffffff;
struct WideNode {           // 1664 bytes
    double lo[3][32];
    double hi[3][32];
    int child[32];          // >= 0: WideNode index; < 0: leaf, ~code with code = first_tri*8 + (count-1); WIDE_EMPTY: unused slot
};

// Node of the winding-number tree (same binary tree / triangle order as the BVH): first-order Barnes-Hut expansion of the solid angle the
// node's triangles subtend (Barill et al. 2018, the scheme behind igl::fast_winding_number): vector area N = sum a_t n_t about the
// area-weighted centroid c, first-moment tensor M = sum a_t (x_t - c) (x) n_t, and the squared radius of the node about c.
struct WnNode {
    double c[3], N[3], M[9], r2;
    int left, right;        // node indices; left < 0: leaf
    int first, count;       // triangle range (leaf order)
};
enum { MESH_SIGN_PSEUDONORMAL = 0, MESH_SIGN_WINDING = 1 };

// Candidate-list caps. A cell the discrete scan can query (centre inside the mesh, or |d_c| - ghd < safety_hor) keeps its list up
// to MESH_LIST_CAP_DISCRETE candidates, every other cell up to MESH_LIST_CAP. Only the discrete scan reads a list longer than
// MESH_LIST_CAP: every other search takes such a cell as unlisted (mesh_list_cnt) and answers it from the tree, so its results
// and tie-breaking do not depend on the longer lists.
constexpr int MESH_LIST_CAP = 160;
constexpr int MESH_LIST_CAP_DISCRETE = 512;
__host__ __device__ inline int mesh_list_cnt(int cnt) { return cnt <= MESH_LIST_CAP ? cnt : 0; }
// The discrete scan walks sub-box filtered copies of the lists (k_mesh_disc_lists): DISC_LIST_K^3 sub-boxes per cell, lists of at most
// DISC_FILTER_MIN candidates (one pass) copied unfiltered.
constexpr int DISC_LIST_K = 4;
constexpr int DISC_FILTER_MIN = 32;

struct DevMesh {
    const BvhNode *nodes;   // nodes[0] is the root (a single-leaf mesh still gets one node with right = left)
    const WideNode *wnodes; // wnodes[0] is the root of the 32-ary tree
    const double *tris;     // TRI_STRIDE doubles per triangle in leaf order: a, ab, ac, Gram entries, reciprocal denominators
    const double *pnormals; // 21 doubles per triangle: face, edge ab, edge bc, edge ca, vertex a, b, c
    // oriented box of every 32-ary-tree leaf, 15 doubles at index first_tri: centre, three unit axes (leaf normal first), half
    // extents. A leaf is a handful of adjacent triangles, i.e. a nearly flat patch: the oriented box is ~1 mm thick where the
    // axis-aligned one is centimetres, and 1-2 m away from the mesh (the swept-volume range test) that difference decides
    // whether a search opens ten leaves or a quarter of the mesh. May be null (no extra pruning).
    const double *leaf_obb;
    // body-frame cell grid over the mesh AABB padded by gpad (filled on the device at isdf_set_shape_mesh time):
    const float *cell_dist;     // signed distance of the cell CENTRE to the mesh
    const uint32_t *cell_seed;  // triangle (leaf order) nearest to the cell centre: a tight initial bound for queries in the cell
    // exact candidate lists: for a cell with centre c and centre distance d_c, EVERY triangle that can be the closest one for
    // some point of the cell lies within d_c + 2*half_diag of c. Cells near the surface store that set (cell_cnt > 0) and a
    // query in such a cell is a flat, traversal-free loop over it; cell_cnt == 0 means "search the tree" (far or deep cells, or
    // more candidates than the cell's cap: MESH_LIST_CAP_DISCRETE where the discrete scan can query, MESH_LIST_CAP elsewhere)
    const uint32_t *cell_off;   // offset into cand
    const uint16_t *cell_cnt;   // number of candidates (0 = no list)
    const uint32_t *cand;       // triangle indices (leaf order), each list sorted by ascending distance from the cell centre (ties: index)
    // parallel to cand: a float lower bound of dist(cell centre, triangle), non-decreasing along each list. A query point p at
    // distance r from the centre is at least cand_lb[k] - r from triangle cand[k] (1-Lipschitz), so once that exceeds the best
    // distance found so far the triangle — and, the list being sorted, every later one — cannot be the closest
    const float *cand_lb;
    // the same four per-cell values fused into one 16-byte record {float bits of cell_dist, cell_seed, cell_off, cell_cnt}: the
    // discrete scan kernel's cull stage fetches it with ONE 128-bit load and hands offset / count / seed to the search, instead
    // of three dependent loads per query (packed by k_mesh_cell_pack at isdf_set_shape_mesh time; may be null)
    const uint4 *cell_rec;
    // Two list contracts. The view every search uses holds in cell_off / cell_cnt / cand / cand_lb / cell_rec the full lists above.
    // The discrete scan's copy of this view (launch_discrete) holds in the same five fields the sub-box filtered lists
    // (k_mesh_disc_lists): each an ordered subsequence of the cell's full list, with the same first entry and the same cand_lb values,
    // that keeps every triangle that can be nearest (exactly tied ones included) to some point the scan assigns to the cell. The
    // scan's pass returns the earliest exact minimum in list order, so both lists give it the same triangle, point and feature.
    double inv_gcell;           // 1 / gcell
    int ntris;
    int gdim[3];
    double glo[3];
    double gcell;           // cell edge
    double ghd;             // half cell diagonal plus float-rounding slack: sdf(p) >= cell_dist - ghd for every p in the cell
    double gpad;            // padding of the grid around the AABB: a point outside the grid is at least gpad away
    double sign_radius;     // a point with no triangle within this distance shares its cell centre's sign (0 = unusable)
    double blo[3], bhi[3];  // mesh AABB
    // sign source. PSEUDONORMAL: s = ±1 from the angle-weighted pseudonormal of the closest feature — exact inside/outside for closed,
    // consistently oriented meshes. WINDING: s = 1 - 2 w with the generalised winding number w evaluated hierarchically and NOT thresholded —
    // the reference's form (Shape.cpp:110-111), the only meaningful one for open meshes and triangle soups.
    int sign_mode;
    const WnNode *wn;       // winding-number tree (root 0); null when sign_mode == PSEUDONORMAL
    double wn_beta2;        // a node is expanded in the far field when |q - c|^2 > wn_beta2 * r2
};

// Triangle record, TRI_STRIDE doubles (128 B = four 32-byte sectors, 32-byte aligned), in leaf order:
//   [0..2] a   [3..5] ab = b-a   [6..8] ac = c-a   [9] ab.ab  [10] ab.ac  [11] ac.ac
//   [12] 1/ab.ab  [13] 1/ac.ac  [14] 1/|bc|^2  [15] 1/(ab.ab ac.ac - (ab.ac)^2)      (0 where the denominator is 0)
// The Gram entries turn four of the six dot products of the closest-point test into subtractions, and every quotient of the
// test has a per-triangle constant denominator (d1-d3 = ab.ab, d2-d6 = ac.ac, (d4-d3)+(d5-d6) = |bc|^2, va+vb+vc = Gram
// determinant), so the division-free form tri_closest_rec_fast needs no FP64 division at all.
constexpr int TRI_STRIDE = 16;

ISDF_HD double box_dist2(const double *b, d3 p) {
    const double ex = fmax(fmax(b[0] - p.x, p.x - b[3]), 0.0);
    const double ey = fmax(fmax(b[1] - p.y, p.y - b[4]), 0.0);
    const double ez = fmax(fmax(b[2] - p.z, p.z - b[5]), 0.0);
    return ex * ex + ey * ey + ez * ez;
}

// Closest point on triangle (a, a+ab, a+ac) by Voronoi-region classification (Ericson's regions and priorities);
// feat: 0 face, 1 ab, 2 bc, 3 ca, 4 a, 5 b, 6 c. Written branch-free: every region's barycentric candidate is computed
// from independent dot products / divisions and the winner is picked by predicated selects in reverse priority order,
// so the FP64 dependency chain is ~15 operations + one division instead of ~100 — the search kernels are bound by
// exactly this latency.
ISDF_HD d3 tri_closest(d3 p, d3 a, d3 ab, d3 ac, int &feat) {
    const d3 ap = p - a;
    const d3 bp = ap - ab, cp = ap - ac;
    const double d1 = dot3(ab, ap), d2 = dot3(ac, ap);
    const double d3_ = dot3(ab, bp), d4 = dot3(ac, bp);
    const double d5 = dot3(ab, cp), d6 = dot3(ac, cp);
    const double vc = d1 * d4 - d3_ * d2, vb = d5 * d2 - d1 * d6, va = d3_ * d6 - d5 * d4;
    const double e43 = d4 - d3_, e56 = d5 - d6;
    const double tab = d1 / (d1 - d3_), tac = d2 / (d2 - d6), tbc = e43 / (e43 + e56), den = 1.0 / (va + vb + vc);
    double s = vb * den, t = vc * den;
    int f = 0;
    if (va <= 0.0 && e43 >= 0.0 && e56 >= 0.0) { s = 1.0 - tbc; t = tbc; f = 2; }
    if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) { s = 0.0; t = tac; f = 3; }
    if (d6 >= 0.0 && d5 <= d6) { s = 0.0; t = 1.0; f = 6; }
    if (vc <= 0.0 && d1 >= 0.0 && d3_ <= 0.0) { s = tab; t = 0.0; f = 1; }
    if (d3_ >= 0.0 && d4 <= d3_) { s = 1.0; t = 0.0; f = 5; }
    if (d1 <= 0.0 && d2 <= 0.0) { s = 0.0; t = 0.0; f = 4; }
    feat = f;
    return mk3(a.x + (s * ab.x + t * ac.x), a.y + (s * ab.y + t * ac.y), a.z + (s * ab.z + t * ac.z));
}

// Same classification on a TRI_STRIDE record with the precomputed Gram entries / reciprocals: ~45 FP64 operations, no division.
// Differs from tri_closest by rounding only (1e-16 relative); used where no sequential decision replays the oracle bit for bit
// (the discrete path; ISDF_FAST_TRI), tri_closest stays in the swept-volume search.
ISDF_HD d3 tri_closest_rec_fast(d3 p, const double *T, int &feat) {
#ifdef __CUDA_ARCH__
    const double2 *T2 = reinterpret_cast<const double2 *>(T);
    const double2 r0 = __ldg(T2), r1 = __ldg(T2 + 1), r2 = __ldg(T2 + 2), r3 = __ldg(T2 + 3), r4 = __ldg(T2 + 4), r5 = __ldg(T2 + 5),
                  r6 = __ldg(T2 + 6), r7 = __ldg(T2 + 7);
    const d3 a = mk3(r0.x, r0.y, r1.x), ab = mk3(r1.y, r2.x, r2.y), ac = mk3(r3.x, r3.y, r4.x);
    const double abab = r4.y, abac = r5.x, acac = r5.y, i_ab = r6.x, i_ac = r6.y, i_bc = r7.x, i_det = r7.y;
#else
    const d3 a = mk3(T[0], T[1], T[2]), ab = mk3(T[3], T[4], T[5]), ac = mk3(T[6], T[7], T[8]);
    const double abab = T[9], abac = T[10], acac = T[11], i_ab = T[12], i_ac = T[13], i_bc = T[14], i_det = T[15];
#endif
    const d3 ap = p - a;
    const double d1 = dot3(ab, ap), d2 = dot3(ac, ap);
    const double d3_ = d1 - abab, d4 = d2 - abac, d5 = d1 - abac, d6 = d2 - acac;
    const double vc = d1 * d4 - d3_ * d2, vb = d5 * d2 - d1 * d6, va = d3_ * d6 - d5 * d4;
    const double e43 = d4 - d3_, e56 = d5 - d6;
    const double tab = d1 * i_ab, tac = d2 * i_ac, tbc = e43 * i_bc;
    double s = vb * i_det, t = vc * i_det;
    int f = 0;
    if (va <= 0.0 && e43 >= 0.0 && e56 >= 0.0) { s = 1.0 - tbc; t = tbc; f = 2; }
    if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) { s = 0.0; t = tac; f = 3; }
    if (d6 >= 0.0 && d5 <= d6) { s = 0.0; t = 1.0; f = 6; }
    if (vc <= 0.0 && d1 >= 0.0 && d3_ <= 0.0) { s = tab; t = 0.0; f = 1; }
    if (d3_ >= 0.0 && d4 <= d3_) { s = 1.0; t = 0.0; f = 5; }
    if (d1 <= 0.0 && d2 <= 0.0) { s = 0.0; t = 0.0; f = 4; }
    feat = f;
    return mk3(a.x + (s * ab.x + t * ac.x), a.y + (s * ab.y + t * ac.y), a.z + (s * ab.z + t * ac.z));
}

// closest point of triangle record T (TRI_STRIDE doubles) to p
ISDF_HD d3 tri_closest_rec(d3 p, const double *T, int &feat) {
#ifdef ISDF_FAST_TRI
    return tri_closest_rec_fast(p, T, feat);
#else
    return tri_closest(p, mk3(T[0], T[1], T[2]), mk3(T[3], T[4], T[5]), mk3(T[6], T[7], T[8]), feat);
#endif
}

// Exact nearest triangle within sqrt(bound2). Returns squared distance (bound2 if none found; tri = -1).
// "while-while" traversal: every lane first descends through internal nodes until it holds a leaf, then all lanes of the
// warp test their leaves together — the long triangle test is not serialised against other lanes' box tests.
__host__ __device__ inline double mesh_closest(const DevMesh &M, d3 p, double bound2, d3 &cbest, int &tri, int &feat) {
    constexpr int DONE = 0x7fffffff;
    double best = bound2;
    tri = -1; feat = 0;
    int stack[40];
    double stack_d2[40];
    int sp = 0;
    int cur = 0;   // node index (>= 0), leaf code (< 0) or DONE
    for (;;) {
        while (cur >= 0 && cur != DONE) {
            const BvhNode *nd = M.nodes + cur;
            const double dl = box_dist2(nd->lbox, p), dr = box_dist2(nd->rbox, p);
            const int l = nd->left, r = nd->right;
            const bool hl = dl < best, hr = (dr < best) && (r != l);
            if (hl && hr) {
                if (dl <= dr) { stack[sp] = r; stack_d2[sp++] = dr; cur = l; } else { stack[sp] = l; stack_d2[sp++] = dl; cur = r; }
            } else if (hl) cur = l;
            else if (hr) cur = r;
            else {
                cur = DONE;
                while (sp > 0) { --sp; if (stack_d2[sp] < best) { cur = stack[sp]; break; } }
            }
        }
        if (cur == DONE) return best;
        {
            const int code = ~cur;
            const int first = code >> 2, cnt = (code & 3) + 1;
            for (int t = first; t < first + cnt; t++) {
                const double *T = M.tris + TRI_STRIDE * (size_t)t;
                int f;
                const d3 q = tri_closest_rec(p, T, f);
                const d3 e = p - q;
                const double dd = dot3(e, e);
                if (dd < best) { best = dd; cbest = q; tri = t; feat = f; }
            }
        }
        cur = DONE;
        while (sp > 0) { --sp; if (stack_d2[sp] < best) { cur = stack[sp]; break; } }
    }
}

ISDF_HD int mesh_cell_index(const DevMesh &M, d3 p) {
    const int ix = (int)floor((p.x - M.glo[0]) / M.gcell), iy = (int)floor((p.y - M.glo[1]) / M.gcell), iz = (int)floor((p.z - M.glo[2]) / M.gcell);
    if (ix < 0 || iy < 0 || iz < 0 || ix >= M.gdim[0] || iy >= M.gdim[1] || iz >= M.gdim[2]) return -1;
    return (ix * M.gdim[1] + iy) * M.gdim[2] + iz;
}
// true when sdf(q) >= reach for EVERY q in p's cell (SDF is 1-Lipschitz), i.e. a hinge / range test with that reach is
// exactly inactive. `cell` returns the cell index (-1 outside the grid).
ISDF_HD bool mesh_far(const DevMesh &M, d3 p, double reach, int &cell) {
    cell = (M.gdim[0] > 0) ? mesh_cell_index(M, p) : -1;
    if (cell < 0) return (M.gdim[0] > 0) && (reach <= M.gpad);
    return (double)M.cell_dist[cell] - M.ghd >= reach;
}
ISDF_HD bool mesh_cell_inside(const DevMesh &M, int cell) { return cell >= 0 && M.cell_dist[cell] < 0.0f; }

// signed solid angle of triangle record T seen from q (van Oosterom & Strackee 1983), positive for an outward triangle seen from inside
ISDF_HD double tri_solid_angle(d3 q, const double *T) {
    const d3 A = mk3(T[0] - q.x, T[1] - q.y, T[2] - q.z), B = mk3(A.x + T[3], A.y + T[4], A.z + T[5]), C = mk3(A.x + T[6], A.y + T[7], A.z + T[8]);
    const double la = len3(A), lb = len3(B), lc = len3(C);
    const double num = dot3(A, cross3(B, C));
    const double den = la * lb * lc + dot3(A, B) * lc + dot3(B, C) * la + dot3(C, A) * lb;
    return 2.0 * atan2(num, den);
}

// Generalised winding number of the mesh at q: Barnes-Hut traversal of the WnNode tree — far nodes contribute their first-order expansion
// (dipole + first-moment term), near leaves the exact solid angles of their triangles. One query per thread.
__host__ __device__ inline double mesh_winding(const DevMesh &M, d3 q) {
    double om = 0.0;
    int stack[64];
    int sp = 0;
    stack[sp++] = 0;
    while (sp > 0) {
        const WnNode &nd = M.wn[stack[--sp]];
        const d3 r = mk3(nd.c[0] - q.x, nd.c[1] - q.y, nd.c[2] - q.z);
        const double d2 = dot3(r, r);
        if (d2 > M.wn_beta2 * nd.r2 && d2 > 0.0) {
            const double inv = 1.0 / sqrt(d2), inv3 = inv * inv * inv;
            const double Nr = nd.N[0] * r.x + nd.N[1] * r.y + nd.N[2] * r.z;
            const double tr = nd.M[0] + nd.M[4] + nd.M[8];
            const double rMr = r.x * (nd.M[0] * r.x + nd.M[1] * r.y + nd.M[2] * r.z) + r.y * (nd.M[3] * r.x + nd.M[4] * r.y + nd.M[5] * r.z) +
                               r.z * (nd.M[6] * r.x + nd.M[7] * r.y + nd.M[8] * r.z);
            om += (Nr + tr) * inv3 - 3.0 * rMr * inv3 * inv * inv;
        } else if (nd.left < 0) {
            for (int t = nd.first; t < nd.first + nd.count; t++) om += tri_solid_angle(q, M.tris + TRI_STRIDE * (size_t)t);
        } else if (sp + 2 <= 64) {
            stack[sp++] = nd.left; stack[sp++] = nd.right;
        }
    }
    return om / (4.0 * 3.14159265358979323846);
}

// sign factor of the SDF at p given the vector e = p - closest point and the closest feature
__host__ __device__ inline double mesh_sign(const DevMesh &M, d3 p, d3 e, int tri, int feat) {
    if (M.sign_mode == MESH_SIGN_WINDING) return 1.0 - 2.0 * mesh_winding(M, p);   // Shape.cpp:110-111: not thresholded
    const double *pn = M.pnormals + 21 * (size_t)tri + 3 * feat;
    double side = e.x * pn[0] + e.y * pn[1] + e.z * pn[2];
    if (side == 0.0) {  // on the surface or numerically tangent: fall back to the face normal
        const double *fn = M.pnormals + 21 * (size_t)tri;
        side = e.x * fn[0] + e.y * fn[1] + e.z * fn[2];
    }
    return (side < 0.0) ? -1.0 : 1.0;
}

// getSDFwithGrad1 for the mesh shape (Shape.cpp:139-151): sdf = s * dist, grad = normalise(s * (p - c)).
// `reach` prunes the search: the caller only needs the value when sdf < reach (pass 1e300 for "always").
// If nothing lies within reach the point is either farther out than reach (returns +reach, grad untouched => the
// hinge is inactive) or deep inside (full search).
__host__ __device__ inline double mesh_sdf_grad(const DevMesh &M, d3 p, double reach, d3 &g) {
    d3 c = mk3(0, 0, 0);
    int tri = -1, feat = 0, cell;
    // winding sign: s = 1 - 2 w is not ±1, so no distance bound can decide the hinge — every query is answered exactly
    const bool bounded = (reach < 1e150) && (M.sign_radius > 0.0) && (reach >= M.sign_radius) && (M.sign_mode == MESH_SIGN_PSEUDONORMAL);
    const bool far = mesh_far(M, p, reach, cell);
    if (bounded && far) return reach;                                  // exact: every point of this cell is >= reach away
    if (cell >= 0 && M.cell_cnt && mesh_list_cnt(M.cell_cnt[cell]) != 0) {
        // flat loop over the cell's exact candidate list: no traversal, no stack, identical code on every lane
        const uint32_t off = M.cell_off[cell];
        const int cnt = (int)M.cell_cnt[cell];
        double bd = 1e300;
        for (int k = 0; k < cnt; k++) {
            const int t = (int)M.cand[off + k];
            const double *T = M.tris + TRI_STRIDE * (size_t)t;
            int f;
            const d3 q = tri_closest_rec(p, T, f);
            const d3 e = p - q;
            const double dd = dot3(e, e);
            if (dd < bd) { bd = dd; c = q; tri = t; feat = f; }
        }
        const d3 e = p - c;
        const double s = mesh_sign(M, p, e, tri, feat);
        g = unit3(s * e);
        return s * sqrt(bd);
    }
    // seed: the triangle nearest to the cell centre gives a tight starting bound
    double seed_d2 = 1e300;
    if (cell >= 0) {
        const int st = (int)M.cell_seed[cell];
        const double *T = M.tris + TRI_STRIDE * (size_t)st;
        const d3 q = tri_closest_rec(p, T, feat);
        const d3 e = p - q;
        seed_d2 = dot3(e, e); c = q; tri = st;
    }
    double d2;
    if (bounded) {
        const double r2 = reach * reach;
        if (seed_d2 < r2) {
            d3 c2; int t2, f2;
            d2 = mesh_closest(M, p, seed_d2, c2, t2, f2);
            if (t2 >= 0) { c = c2; tri = t2; feat = f2; } else d2 = seed_d2;
        } else {
            tri = -1;
            d2 = mesh_closest(M, p, r2, c, tri, feat);
            if (tri < 0) {
                if (!mesh_cell_inside(M, cell)) return reach;          // outside and at least `reach` away
                d2 = mesh_closest(M, p, 1e300, c, tri, feat);          // deep inside: rare
            }
        }
    } else if (tri >= 0) {
        d3 c2; int t2, f2;
        d2 = mesh_closest(M, p, seed_d2, c2, t2, f2);
        if (t2 >= 0) { c = c2; tri = t2; feat = f2; } else d2 = seed_d2;
    } else {
        d2 = mesh_closest(M, p, 1e300, c, tri, feat);
    }
    const d3 e = p - c;
    const double s = mesh_sign(M, p, e, tri, feat);
    g = unit3(s * e);
    return s * sqrt(d2);
}

// ---- warp-cooperative exact nearest triangle --------------------------------------------------------------------------
// Every lane passes the SAME query point; lane i tests child i of the current 32-ary node, leaf triangles are tested
// 32 at a time (8 leaves x 4 slots), the winner is found with a butterfly arg-min. All lanes return identical results.
// `stk` is a per-warp shared-memory scratch of WIDE_STACK (node, d2) pairs.
constexpr int WIDE_STACK = 96;
// the stacked bounds are floats ROUNDED DOWN: still lower bounds, so pruning stays exact (a node is at worst opened needlessly)
struct WideStack {
    int node[WIDE_STACK]; float d2[WIDE_STACK]; int leaf[32]; float leaf_d2[32];
};

__device__ __forceinline__ double wide_closest(const DevMesh &M, d3 p, double bound2, int seed, d3 &cbest, int &tri, int &feat,
                                               int lane, WideStack *stk) {
    double best = bound2;
    tri = -1; feat = 0;
    const unsigned lt_mask = (1u << lane) - 1u;
    if (seed >= 0) {   // every lane evaluates the seed triangle (uniform): a tight bound before the first node is opened
        const double *T = M.tris + TRI_STRIDE * (size_t)seed;
        int f;
        const d3 q = tri_closest_rec(p, T, f);
        const d3 e = p - q;
        const double dd = dot3(e, e);
        if (dd < best) { best = dd; cbest = q; tri = seed; feat = f; }
    }
    int sp = 0;
    int cur = 0; double cur_d2 = 0.0;
    for (;;) {
        if (cur_d2 < best) {
            const WideNode *nd = M.wnodes + cur;
            const int ch = nd->child[lane];
            const double ex = fmax(fmax(nd->lo[0][lane] - p.x, p.x - nd->hi[0][lane]), 0.0);
            const double ey = fmax(fmax(nd->lo[1][lane] - p.y, p.y - nd->hi[1][lane]), 0.0);
            const double ez = fmax(fmax(nd->lo[2][lane] - p.z, p.z - nd->hi[2][lane]), 0.0);
            double d2 = ex * ex + ey * ey + ez * ez;
            bool alive = (ch != WIDE_EMPTY) && (d2 < best);
            if (alive && ch < 0 && M.leaf_obb) {   // second, tighter lower bound for leaves: distance to the oriented box
                const double *o = M.leaf_obb + 15 * (size_t)((~ch) >> 3);
                const d3 r = mk3(p.x - o[0], p.y - o[1], p.z - o[2]);
                const double e0 = fmax(fabs(r.x * o[3] + r.y * o[4] + r.z * o[5]) - o[12], 0.0);
                const double e1 = fmax(fabs(r.x * o[6] + r.y * o[7] + r.z * o[8]) - o[13], 0.0);
                const double e2 = fmax(fabs(r.x * o[9] + r.y * o[10] + r.z * o[11]) - o[14], 0.0);
                d2 = fmax(d2, e0 * e0 + e1 * e1 + e2 * e2);
                alive = d2 < best;
            }
            // ---- leaves: compacted into a shared list, then 8 per pass x 4 triangle slots ------------------------------
            const bool is_leaf = alive && ch < 0;
            const unsigned leafmask = __ballot_sync(0xffffffffu, is_leaf);
            const int nleaf = __popc(leafmask);
            if (is_leaf) { const int r = __popc(leafmask & lt_mask); stk->leaf[r] = ch; stk->leaf_d2[r] = __double2float_rd(d2); }
            __syncwarp();
            for (int base = 0; base < nleaf; base += 8) {
                const int idx = base + (lane >> 2), slot = lane & 3;
                double dd = 1e300; d3 q = mk3(0, 0, 0); int f = 0, t = -1;
                if (idx < nleaf && (double)stk->leaf_d2[idx] < best) {
                    const int code = ~stk->leaf[idx];
                    const int first = code >> 3, cnt = (code & 7) + 1;
                    for (int k = slot; k < cnt; k += 4) {   // leaves of up to 8 triangles: slots take triangle k and k+4
                        const double *T = M.tris + TRI_STRIDE * (size_t)(first + k);
                        int ff;
                        const d3 qq = tri_closest_rec(p, T, ff);
                        const d3 e = p - qq;
                        const double d = dot3(e, e);
                        if (d < dd) { dd = d; q = qq; f = ff; t = first + k; }
                    }
                }
                // arg-min: 32-bit order-preserving key (float rounded down) + one REDUX; exact tie-break among equal keys
                const bool cand = dd < best;
                const unsigned key = cand ? __float_as_uint(__double2float_rd(dd)) : 0xffffffffu;
                const unsigned kmin = __reduce_min_sync(0xffffffffu, key);
                if (kmin != 0xffffffffu) {
                    unsigned tied = __ballot_sync(0xffffffffu, cand && key == kmin);
                    int win = __ffs(tied) - 1;
                    double wd = __shfl_sync(0xffffffffu, dd, win);
                    tied &= tied - 1;
                    while (tied) {   // rare: several lanes within one float ulp
                        const int o = __ffs(tied) - 1;
                        tied &= tied - 1;
                        const double od = __shfl_sync(0xffffffffu, dd, o);
                        if (od < wd) { wd = od; win = o; }
                    }
                    best = wd;
                    cbest = mk3(__shfl_sync(0xffffffffu, q.x, win), __shfl_sync(0xffffffffu, q.y, win), __shfl_sync(0xffffffffu, q.z, win));
                    tri = __shfl_sync(0xffffffffu, t, win);
                    feat = __shfl_sync(0xffffffffu, f, win);
                }
            }
            // ---- internal children: push farthest first so the nearest is popped next ---------------------------------
            unsigned imask = __ballot_sync(0xffffffffu, alive && ch >= 0 && ch != WIDE_EMPTY && d2 < best);
            while (imask) {
                const unsigned key = ((imask >> lane) & 1u) ? ((__float_as_uint((float)d2) & ~31u) | (unsigned)lane) : 0u;
                const unsigned kmax = __reduce_max_sync(0xffffffffu, key);
                const int sl = (int)(kmax & 31u);
                const int snode = __shfl_sync(0xffffffffu, ch, sl);
                const double sd2 = __shfl_sync(0xffffffffu, d2, sl);
                if (lane == 0 && sp < WIDE_STACK) { stk->node[sp] = snode; stk->d2[sp] = __double2float_rd(sd2); }
                sp = min(sp + 1, WIDE_STACK);
                imask &= ~(1u << sl);
            }
            __syncwarp();
        }
        if (sp == 0) return best;
        --sp;
        cur = stk->node[sp]; cur_d2 = (double)stk->d2[sp];
        __syncwarp();
    }
}

// Warp-cooperative range query on the 32-ary tree: calls emit(valid, tri, d2) for every triangle whose exact distance to c is
// <= sqrt(R2) (d2: its squared distance), 32 triangles per call (lanes without one pass valid = false). Used to build the per-cell
// candidate lists.
template <class Emit>
__device__ __forceinline__ void wide_range(const DevMesh &M, d3 c, double R2, int lane, WideStack *stk, Emit &&emit) {
    const unsigned lt_mask = (1u << lane) - 1u;
    int sp = 0, cur = 0;
    for (;;) {
        const WideNode *nd = M.wnodes + cur;
        const int ch = nd->child[lane];
        const double ex = fmax(fmax(nd->lo[0][lane] - c.x, c.x - nd->hi[0][lane]), 0.0);
        const double ey = fmax(fmax(nd->lo[1][lane] - c.y, c.y - nd->hi[1][lane]), 0.0);
        const double ez = fmax(fmax(nd->lo[2][lane] - c.z, c.z - nd->hi[2][lane]), 0.0);
        const bool alive = (ch != WIDE_EMPTY) && (ex * ex + ey * ey + ez * ez <= R2);
        const bool is_leaf = alive && ch < 0;
        const unsigned leafmask = __ballot_sync(0xffffffffu, is_leaf);
        const int nleaf = __popc(leafmask);
        if (is_leaf) stk->leaf[__popc(leafmask & lt_mask)] = ch;
        __syncwarp();
        for (int base = 0; base < nleaf; base += 4) {      // 4 leaves x 8 triangle slots
            const int idx = base + (lane >> 3), slot = lane & 7;
            bool hit = false; int t = -1;
            double d2 = 0.0;
            if (idx < nleaf) {
                const int code = ~stk->leaf[idx];
                const int first = code >> 3, cnt = (code & 7) + 1;
                if (slot < cnt) {
                    t = first + slot;
                    const double *T = M.tris + TRI_STRIDE * (size_t)t;
                    int ff;
                    const d3 q = tri_closest_rec(c, T, ff);
                    const d3 e = c - q;
                    d2 = dot3(e, e);
                    hit = d2 <= R2;
                }
            }
            emit(hit, t, d2);
        }
        unsigned imask = __ballot_sync(0xffffffffu, alive && ch >= 0);
        while (imask) {
            const int sl = __ffs(imask) - 1;
            imask &= imask - 1;
            const int snode = __shfl_sync(0xffffffffu, ch, sl);
            if (lane == 0 && sp < WIDE_STACK) stk->node[sp] = snode;
            sp = min(sp + 1, WIDE_STACK);
        }
        __syncwarp();
        if (sp == 0) return;
        cur = stk->node[--sp];
        __syncwarp();
    }
}

// arg-min step shared by the cooperative searches: every lane offers (dd, q, t, f); if the warp's smallest dd beats `best` the
// winner's values are broadcast. 32-bit order-preserving key (float rounded down) + one REDUX; exact tie-break among equal keys.
__device__ __forceinline__ void warp_argmin_update(double dd, d3 q, int t, int f, double &best, d3 &cbest, int &tri, int &feat) {
    const bool candd = dd < best;
    const unsigned key = candd ? __float_as_uint(__double2float_rd(dd)) : 0xffffffffu;
    const unsigned kmin = __reduce_min_sync(0xffffffffu, key);
    if (kmin != 0xffffffffu) {
        unsigned tied = __ballot_sync(0xffffffffu, candd && key == kmin);
        int win = __ffs(tied) - 1;
        double wd = __shfl_sync(0xffffffffu, dd, win);
        tied &= tied - 1;
        while (tied) {   // rare: several lanes within one float ulp
            const int o = __ffs(tied) - 1;
            tied &= tied - 1;
            const double od = __shfl_sync(0xffffffffu, dd, o);
            if (od < wd) { wd = od; win = o; }
        }
        best = wd;
        cbest = mk3(__shfl_sync(0xffffffffu, q.x, win), __shfl_sync(0xffffffffu, q.y, win), __shfl_sync(0xffffffffu, q.z, win));
        tri = __shfl_sync(0xffffffffu, t, win);
        feat = __shfl_sync(0xffffffffu, f, win);
    }
}

// Warp-cooperative nearest triangle from a cell's candidate list: lanes test 32 candidates per pass, REDUX arg-min.
// (Two candidates per lane and pass — a second independent chain — was measured slower.)
//
// The pass is pruned with the lists' lower bounds (DevMesh::cand_lb). p lies within r_up of the centre of the cell whose list this
// is, so candidate k is at least cand_lb[k] - r_up away from p. A lane whose bound already exceeds the best distance found so far
// skips its candidate (no 128-byte record load, no test), and since each list is sorted by that bound the warp stops as soon as the
// first candidate of the next pass is ruled out. The bounds carry slack for rounding and the test is strict, so a candidate exactly
// tied with the best is still tested and the arg-min's tie rule decides as it would without pruning.
__device__ __forceinline__ bool list_lb_prunes(float lb, double r_up, double best) {
    const double g = (double)lb - r_up;
    return g > 0.0 && g * g > best;
}
// upper bound of |p - c| for the centre c of cell (ix, iy, iz): the lists were built in a translation unit without FMA contraction
// and the scan kernels contract, so the two may round c differently by an ulp
__device__ __forceinline__ double list_centre_dist_up(const DevMesh &M, d3 p, double ix, double iy, double iz) {
    const d3 e = mk3(p.x - (M.glo[0] + (ix + 0.5) * M.gcell), p.y - (M.glo[1] + (iy + 0.5) * M.gcell), p.z - (M.glo[2] + (iz + 0.5) * M.gcell));
    return sqrt(dot3(e, e)) * (1.0 + 1e-9) + 1e-12;
}
// first_id / first_lb: this lane's candidate of the FIRST pass and its bound (cand[off + lane], cand_lb[off + lane]; -1 beyond the
// list) — the caller may have loaded them long before (software pipelining across queries); those of every following pass are
// requested one pass ahead. r_up: list_centre_dist_up of p and the list's cell. bound2 seeds the best squared distance: when no
// candidate is closer, tri = -1 (and the returned value is not a distance).
__device__ __forceinline__ double list_closest_pre(const DevMesh &M, d3 p, uint32_t off, int cnt, int first_id, float first_lb, double r_up,
                                                   double bound2, d3 &cbest, int &tri, int &feat, int lane) {
    // the list's first candidate is the triangle nearest to the cell centre, so p's closest triangle lies within that distance plus
    // r_up: an upper bound (the slack undoes the bound's round-down) that prunes the first pass too. No candidate is returned unless
    // it is below bound2, and the closest one always is below this bound, so starting from the smaller of the two changes no answer.
    const double ub = (double)__shfl_sync(0xffffffffu, first_lb, 0) * (1.0 + 1e-6) + 1e-9 + r_up;
    double best = fmin(bound2, ub * ub);
    tri = -1; feat = 0;
    int t = first_id;
    float lb = first_lb;
    for (int base = 0; base < cnt; base += 32) {
        const int nb = base + 32 + lane;
        int t_next = -1;
        float lb_next = 0.0f;
        if (nb < cnt) { t_next = (int)__ldg(M.cand + off + nb); lb_next = __ldg(M.cand_lb + off + nb); }   // next pass, in flight during this one
        const bool test = t >= 0 && !list_lb_prunes(lb, r_up, best);
        double dd = 1e300; d3 q = mk3(0, 0, 0); int f = 0;
        if (test) {
            const double *T = M.tris + TRI_STRIDE * (size_t)t;
            q = tri_closest_rec(p, T, f);
            const d3 e = p - q;
            dd = dot3(e, e);
        }
        warp_argmin_update(dd, q, t, f, best, cbest, tri, feat);
        if (base + 32 < cnt && list_lb_prunes(__shfl_sync(0xffffffffu, lb_next, 0), r_up, best)) break;
        t = t_next; lb = lb_next;
    }
    return best;
}
__device__ __forceinline__ double list_closest(const DevMesh &M, d3 p, int cell, d3 &cbest, int &tri, int &feat, int lane) {
    const uint32_t off = M.cell_off[cell];
    const int cnt = (int)M.cell_cnt[cell];
    const int nz = M.gdim[2], ny = M.gdim[1];
    const int iz = cell % nz, iy = (cell / nz) % ny, ix = cell / (nz * ny);
    const bool has = lane < cnt;
    return list_closest_pre(M, p, off, cnt, has ? (int)__ldg(M.cand + off + lane) : -1, has ? __ldg(M.cand_lb + off + lane) : 0.0f,
                            list_centre_dist_up(M, p, ix, iy, iz), 1e300, cbest, tri, feat, lane);
}

// Latency-oriented list pass for callers that run ONE query at a time on an otherwise idle SM (the swept-volume path's descent and
// fine-scan chains): all of this lane's candidate ids are requested at once, the 128-byte records of every pass after the first are
// prefetched into L1 while the first pass computes — one DRAM/L2 round trip for the whole list instead of one per pass. Same
// arithmetic, same pass order and tie-breaking as list_closest_pre.
constexpr int MESH_LIST_PASSES = MESH_LIST_CAP / 32;
__device__ __forceinline__ double list_closest_lat(const DevMesh &M, d3 p, uint32_t off, int cnt, d3 &cbest, int &tri, int &feat, int lane) {
    int ids[MESH_LIST_PASSES];
#pragma unroll
    for (int k = 0; k < MESH_LIST_PASSES; k++) { const int i = k * 32 + lane; ids[k] = (i < cnt) ? (int)__ldg(M.cand + off + i) : -1; }
#ifdef __CUDA_ARCH__
#pragma unroll
    for (int k = 1; k < MESH_LIST_PASSES; k++)
        if (ids[k] >= 0) asm volatile("prefetch.global.L1 [%0];" ::"l"(M.tris + TRI_STRIDE * (size_t)ids[k]));
#endif
    double best = 1e300;
    tri = -1; feat = 0;
#pragma unroll
    for (int k = 0; k < MESH_LIST_PASSES; k++) {
        if (k * 32 >= cnt) break;
        const int t = ids[k];
        double dd = 1e300; d3 q = mk3(0, 0, 0); int f = 0;
        if (t >= 0) {
            const double *T = M.tris + TRI_STRIDE * (size_t)t;
            q = tri_closest_rec(p, T, f);
            const d3 e = p - q;
            dd = dot3(e, e);
        }
        warp_argmin_update(dd, q, t, f, best, cbest, tri, feat);
    }
    return best;
}

// Search half of getSDFwithGrad1 for the mesh shape, warp-cooperative: closest triangle of p (cell = p's cell index, or -1
// outside the grid; the caller has already ruled out "far"). Returns false when nothing lies within `reach` and p is outside
// (sdf >= reach: the caller's hinge / range test is inactive); otherwise (d2, c, tri, feat), identical on every lane.
__device__ __forceinline__ bool mesh_search_warp(const DevMesh &M, d3 p, double reach, int lane, WideStack *stk, int cell,
                                                 double &d2, d3 &c, int &tri, int &feat) {
    const bool bounded = (reach < 1e150) && (M.sign_radius > 0.0) && (reach >= M.sign_radius);
    const int seed = (cell >= 0) ? (int)M.cell_seed[cell] : -1;
    if (cell >= 0 && M.cell_cnt && mesh_list_cnt(M.cell_cnt[cell]) != 0) {
        d2 = list_closest(M, p, cell, c, tri, feat, lane);       // exact: the list holds every possible closest triangle
    } else if (bounded) {
        d2 = wide_closest(M, p, reach * reach, seed, c, tri, feat, lane, stk);
        if (tri < 0) {
            if (!mesh_cell_inside(M, cell)) return false;
            d2 = wide_closest(M, p, 1e300, seed, c, tri, feat, lane, stk);
        }
    } else {
        d2 = wide_closest(M, p, 1e300, seed, c, tri, feat, lane, stk);
    }
    return true;
}

// The same search with the cell's record already fetched (DevMesh::cell_rec): cnt / off = candidate list (cnt 0: none), seed =
// nearest triangle of the cell centre (-1 outside the grid), inside = the cell centre is inside the mesh. first_id / first_lb: the
// list's first pass as list_closest_pre takes it. With an exact sign (pseudonormal, reach >= sign_radius) both searches start from
// the bound reach^2: nothing closer means sdf >= reach when the cell centre is outside (false), and a second, unbounded search when
// it is inside. deep: the caller has shown d_c + ghd <= -reach for the cell, so every point of it is at least reach inside (the
// ghd slack covers the float rounding of d_c with room to spare for the FP64 distances) and the bounded search would find nothing:
// the unbounded one runs straight away, with the same result.
__device__ __forceinline__ bool mesh_search_rec(const DevMesh &M, d3 p, double reach, int lane, WideStack *stk, int cnt, uint32_t off,
                                                int first_id, float first_lb, int seed, bool inside, bool deep, double &d2, d3 &c, int &tri,
                                                int &feat) {
    const bool bounded = (reach < 1e150) && (M.sign_radius > 0.0) && (reach >= M.sign_radius) && (M.sign_mode == MESH_SIGN_PSEUDONORMAL);
    double bound2 = (bounded && !deep) ? reach * reach : 1e300;
    if (cnt != 0) {
        // the list's cell is p's cell, found exactly as the callers' cull stages find it
        const double r_up = list_centre_dist_up(M, p, floor((p.x - M.glo[0]) * M.inv_gcell), floor((p.y - M.glo[1]) * M.inv_gcell),
                                                floor((p.z - M.glo[2]) * M.inv_gcell));
        for (;;) {   // one inlined copy of the list pass: first within `reach`, then (deep inside only) unbounded
            d2 = list_closest_pre(M, p, off, cnt, first_id, first_lb, r_up, bound2, c, tri, feat, lane);
            if (tri >= 0 || bound2 >= 1e299) return true;
            if (!inside) return false;
            bound2 = 1e300;
        }
    }
    for (;;) {   // one inlined copy of the tree search, the same way (a separate loop: merged with the list pass, it spills)
        d2 = wide_closest(M, p, bound2, seed, c, tri, feat, lane, stk);
        if (tri >= 0 || bound2 >= 1e299) return true;
        if (!inside) return false;
        bound2 = 1e300;
    }
}

// Sign + gradient half (Shape.cpp:139-151): e = p - closest point; sdf = s * dist, grad = normalise(s * e), s = ±1 from the
// angle-weighted pseudonormal of the closest feature.
__device__ __forceinline__ double mesh_finish(const DevMesh &M, d3 p, d3 e, double d2, int tri, int feat, d3 &g) {
    const double s = mesh_sign(M, p, e, tri, feat);
    g = unit3(s * e);
    return s * sqrt(d2);
}
// compile-time choice of the sign source: the closed-mesh instantiation of a kernel carries no winding-number code at all (the discrete
// scan kernel is sensitive to its code size)
template <bool WINDING>
__device__ __forceinline__ double mesh_finish_t(const DevMesh &M, d3 p, d3 e, double d2, int tri, int feat, d3 &g) {
    double s;
    if (WINDING) s = 1.0 - 2.0 * mesh_winding(M, p);
    else {
        const double *pn = M.pnormals + 21 * (size_t)tri + 3 * feat;
        double side = e.x * pn[0] + e.y * pn[1] + e.z * pn[2];
        if (side == 0.0) { const double *fn = M.pnormals + 21 * (size_t)tri; side = e.x * fn[0] + e.y * fn[1] + e.z * fn[2]; }
        s = (side < 0.0) ? -1.0 : 1.0;
    }
    g = unit3(s * e);
    return s * sqrt(d2);
}

// Warp-cooperative getSDFwithGrad1 for the mesh shape — same contract as mesh_sdf_grad, all lanes get the same answer.
// known_cell: cell index already looked up by the caller (and known not to be "far"), or -2 to look it up here.
__device__ __forceinline__ double mesh_sdf_grad_warp(const DevMesh &M, d3 p, double reach, d3 &g, int lane, WideStack *stk, int known_cell = -2) {
    d3 c = mk3(0, 0, 0);
    int tri, feat, cell = known_cell;
    double d2;
    if (known_cell == -2) {
        const bool bounded = (reach < 1e150) && (M.sign_radius > 0.0) && (reach >= M.sign_radius);
        const bool far = mesh_far(M, p, reach, cell);
        if (bounded && far) return reach;
    }
    if (!mesh_search_warp(M, p, reach, lane, stk, cell, d2, c, tri, feat)) return reach;
    return mesh_finish(M, p, p - c, d2, tri, feat, g);
}

// The same query for latency-bound callers: the cell's fused 16-byte record (one load instead of three dependent ones) and the
// latency-oriented list pass. Identical results (same search, same order).
__device__ __forceinline__ double mesh_sdf_grad_warp_lat(const DevMesh &M, d3 p, double reach, d3 &g, int lane, WideStack *stk) {
    if (!M.cell_rec || M.gdim[0] <= 0) return mesh_sdf_grad_warp(M, p, reach, g, lane, stk);
    const int cell = mesh_cell_index(M, p);
    const bool bounded = (reach < 1e150) && (M.sign_radius > 0.0) && (reach >= M.sign_radius);
    d3 c = mk3(0, 0, 0);
    int tri, feat;
    double d2;
    if (cell < 0) {
        if (bounded && reach <= M.gpad) return reach;
        if (!mesh_search_warp(M, p, reach, lane, stk, cell, d2, c, tri, feat)) return reach;
    } else {
        const uint4 rec = __ldg(M.cell_rec + cell);
        const float dc = __uint_as_float(rec.x);
        if (bounded && (double)dc - M.ghd >= reach) return reach;
        const int cnt = (int)rec.w;
        if (cnt != 0 && cnt <= MESH_LIST_CAP) d2 = list_closest_lat(M, p, rec.z, cnt, c, tri, feat, lane);
        else if (!mesh_search_warp(M, p, reach, lane, stk, cell, d2, c, tri, feat)) return reach;
    }
    return mesh_finish(M, p, p - c, d2, tri, feat, g);
}

}  // namespace isdf
