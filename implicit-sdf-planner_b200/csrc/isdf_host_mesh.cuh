// Host-side, one-off construction of the device mesh structure at isdf_set_shape_mesh time:
// the counterpart of the Generalshape constructor (Shape.cpp:27-103: read mesh, pre-transform by poly_params,
// tree.init(V,F), fast_winding_number precompute). Produces the BVH, leaf-ordered triangles, pseudonormals and the
// inside/outside bitmap described in isdf_mesh.cuh.
#pragma once
#include "isdf_mesh.cuh"
#include <vector>
#include <map>
#include <array>
#include <string>
#include <algorithm>
#include <numeric>
#include <cmath>

namespace isdf {

struct HostMesh {
    std::vector<BvhNode> nodes;
    std::vector<WideNode> wnodes;
    std::vector<double> tris, pnormals, leaf_obb;
    std::vector<WnNode> wn;
    int sign_mode = MESH_SIGN_PSEUDONORMAL;
    bool closed = true;
    double wn_beta2 = 256.0;   // beta = 16: measured max |w_tree - w_exact| ~1e-4 on a 3800-triangle mesh (tests/host_mesh_check.cu); the reference's FP32 order-2 tree at beta = 2 is at 1e-4..1e-3
    int ntris = 0;
    int gdim[3] = {0, 0, 0};
    double glo[3] = {0, 0, 0}, gcell = 0, ghd = 0, gpad = 0, sign_radius = 0;
    double blo[3] = {0, 0, 0}, bhi[3] = {0, 0, 0};
    DevMesh view() const {  // host pointers; same code path as the device for the bitmap construction
        DevMesh m;
        m.nodes = nodes.data(); m.wnodes = wnodes.data(); m.tris = tris.data(); m.pnormals = pnormals.data(); m.leaf_obb = leaf_obb.empty() ? nullptr : leaf_obb.data(); m.cell_dist = nullptr; m.cell_seed = nullptr; m.cell_off = nullptr; m.cell_cnt = nullptr; m.cand = nullptr; m.cand_lb = nullptr; m.cell_rec = nullptr;
        m.sign_mode = sign_mode; m.wn = wn.empty() ? nullptr : wn.data(); m.wn_beta2 = wn_beta2;
        m.ntris = ntris;
        for (int a = 0; a < 3; a++) { m.gdim[a] = gdim[a]; m.glo[a] = glo[a]; m.blo[a] = blo[a]; m.bhi[a] = bhi[a]; }
        m.gcell = gcell; m.inv_gcell = gcell > 0 ? 1.0 / gcell : 0.0; m.ghd = ghd; m.gpad = gpad; m.sign_radius = sign_radius;
        return m;
    }
};

namespace detail {
struct BuildNode { double lo[3], hi[3]; int left = -1, right = -1, first = 0, count = 0; };
constexpr int LEAF_MAX = 4;

inline int build_rec(std::vector<BuildNode> &bn, std::vector<int> &order, int b, int e, const std::vector<std::array<double, 9>> &tv,
                     const std::vector<std::array<double, 3>> &cen) {
    BuildNode nd;
    double clo[3], chi[3];
    for (int a = 0; a < 3; a++) { nd.lo[a] = clo[a] = 1e300; nd.hi[a] = chi[a] = -1e300; }
    for (int i = b; i < e; i++) {
        const auto &t = tv[order[i]];
        for (int k = 0; k < 3; k++)
            for (int a = 0; a < 3; a++) { nd.lo[a] = std::min(nd.lo[a], t[3 * k + a]); nd.hi[a] = std::max(nd.hi[a], t[3 * k + a]); }
        for (int a = 0; a < 3; a++) { clo[a] = std::min(clo[a], cen[order[i]][a]); chi[a] = std::max(chi[a], cen[order[i]][a]); }
    }
    nd.first = b; nd.count = e - b;
    const int me = (int)bn.size();
    bn.push_back(nd);
    if (e - b <= LEAF_MAX) return me;
    int ax = 0;
    if (chi[1] - clo[1] > chi[ax] - clo[ax]) ax = 1;
    if (chi[2] - clo[2] > chi[ax] - clo[ax]) ax = 2;
    const int mid = (b + e) / 2;
    std::nth_element(order.begin() + b, order.begin() + mid, order.begin() + e, [&](int x, int y) { return cen[x][ax] < cen[y][ax]; });
    const int l = build_rec(bn, order, b, mid, tv, cen);
    const int r = build_rec(bn, order, mid, e, tv, cen);
    bn[me].left = l; bn[me].right = r;
    return me;
}
}  // namespace detail

// V: nV x 3, F: nF x 3 (row-major). poly_params {tx,ty,tz, roll,pitch,yaw [deg]} or nullptr (Shape.cpp:38-50).
// sign_reach: smallest query bound the kernels will use with the bitmap shortcut (safety_hor).
// want_sign: 0 = automatic (closed, consistently oriented mesh -> exact ±1 from pseudonormals; anything else -> winding number),
//            1 = exact ±1 required (fails for open meshes / soups), 2 = winding number s = 1 - 2 w (the reference's form) even when closed.
inline bool build_host_mesh(const double *Vin, int nV, const int32_t *F, int nF, const double *poly_params, double sign_reach,
                            HostMesh &out, std::string &err, int want_sign = 0) {
    if (nV < 3 || nF < 1) { err = "mesh needs at least 3 vertices and 1 face"; return false; }
    for (int i = 0; i < 3 * nF; i++) if (F[i] < 0 || F[i] >= nV) { err = "face index out of range"; return false; }
    std::vector<std::array<double, 3>> V(nV);
    for (int i = 0; i < nV; i++) V[i] = {Vin[3 * i], Vin[3 * i + 1], Vin[3 * i + 2]};
    if (poly_params) {  // V <- Rz(yaw) Ry(pitch) Rx(roll) V + t
        const double PI = 3.14159265358979323846;
        const double r = poly_params[3] * PI / 180.0, p = poly_params[4] * PI / 180.0, y = poly_params[5] * PI / 180.0;
        const double cr = std::cos(r), sr = std::sin(r), cp = std::cos(p), sp = std::sin(p), cy = std::cos(y), sy = std::sin(y);
        for (auto &v : V) {
            const double x1 = v[0], y1 = cr * v[1] - sr * v[2], z1 = sr * v[1] + cr * v[2];           // Rx
            const double x2 = cp * x1 + sp * z1, y2 = y1, z2 = -sp * x1 + cp * z1;                    // Ry
            const double x3 = cy * x2 - sy * y2, y3 = sy * x2 + cy * y2, z3 = z2;                     // Rz
            v = {x3 + poly_params[0], y3 + poly_params[1], z3 + poly_params[2]};
        }
    }
    // weld vertices that coincide exactly so adjacency survives unindexed input
    std::map<std::array<double, 3>, int> weld;
    std::vector<int> canon(nV);
    for (int i = 0; i < nV; i++) { auto it = weld.find(V[i]); if (it == weld.end()) { weld[V[i]] = i; canon[i] = i; } else canon[i] = it->second; }

    std::vector<std::array<double, 9>> tv(nF);
    std::vector<std::array<double, 3>> cen(nF), fn(nF);
    std::vector<std::array<int, 3>> fi(nF);
    for (int t = 0; t < nF; t++) {
        for (int k = 0; k < 3; k++) { fi[t][k] = canon[F[3 * t + k]]; for (int a = 0; a < 3; a++) tv[t][3 * k + a] = V[F[3 * t + k]][a]; }
        for (int a = 0; a < 3; a++) cen[t][a] = (tv[t][a] + tv[t][3 + a] + tv[t][6 + a]) / 3.0;
        const d3 A = mk3(tv[t][0], tv[t][1], tv[t][2]), B = mk3(tv[t][3], tv[t][4], tv[t][5]), C = mk3(tv[t][6], tv[t][7], tv[t][8]);
        const d3 n = unit3(cross3(B - A, C - A));
        fn[t] = {n.x, n.y, n.z};
    }
    // pseudonormals: edges = sum of adjacent unit face normals, vertices = incident-angle-weighted sum
    std::map<std::pair<int, int>, std::array<double, 3>> en;
    std::vector<std::array<double, 3>> vn(nV, {0, 0, 0});
    for (int t = 0; t < nF; t++) {
        for (int k = 0; k < 3; k++) {
            const int u = fi[t][k], v = fi[t][(k + 1) % 3];
            auto &e = en[{std::min(u, v), std::max(u, v)}];
            for (int a = 0; a < 3; a++) e[a] += fn[t][a];
            const d3 P0 = mk3(tv[t][3 * k], tv[t][3 * k + 1], tv[t][3 * k + 2]);
            const d3 P1 = mk3(tv[t][3 * ((k + 1) % 3)], tv[t][3 * ((k + 1) % 3) + 1], tv[t][3 * ((k + 1) % 3) + 2]);
            const d3 P2 = mk3(tv[t][3 * ((k + 2) % 3)], tv[t][3 * ((k + 2) % 3) + 1], tv[t][3 * ((k + 2) % 3) + 2]);
            const d3 e1 = unit3(P1 - P0), e2 = unit3(P2 - P0);
            const double ang = std::acos(std::max(-1.0, std::min(1.0, dot3(e1, e2))));
            for (int a = 0; a < 3; a++) vn[u][a] += ang * fn[t][a];
        }
    }
    // The ±1 sign from pseudonormals is the generalised winding number's 0/1 only for a CLOSED, consistently oriented surface:
    // every undirected edge must be used exactly twice, once in each direction.
    {
        std::map<std::pair<int, int>, int> directed;
        for (int t = 0; t < nF; t++)
            for (int k = 0; k < 3; k++) directed[{fi[t][k], fi[t][(k + 1) % 3]}]++;
        for (const auto &e : directed) {
            const auto rev = directed.find({e.first.second, e.first.first});
            if (e.first.first == e.first.second || e.second != 1 || rev == directed.end() || rev->second != 1) { out.closed = false; break; }
        }
        if (!out.closed && want_sign == 1) {
            err = "mesh is not a closed, consistently oriented 2-manifold (open, duplicated or flipped edge): the exact ±1 sign needs one — "
                  "use the automatic or the winding-number sign mode";
            return false;
        }
        out.sign_mode = (want_sign == 2 || !out.closed) ? MESH_SIGN_WINDING : MESH_SIGN_PSEUDONORMAL;
    }
    // BVH
    std::vector<int> order(nF);
    std::iota(order.begin(), order.end(), 0);
    std::vector<detail::BuildNode> bn;
    bn.reserve(2 * nF);
    detail::build_rec(bn, order, 0, nF, tv, cen);
    // leaf-ordered triangle + pseudonormal arrays
    out.ntris = nF;
    out.tris.assign((size_t)TRI_STRIDE * nF, 0.0); out.pnormals.resize((size_t)21 * nF);
    for (int pos = 0; pos < nF; pos++) {
        const int t = order[pos];
        double *T = &out.tris[(size_t)TRI_STRIDE * pos];
        for (int a = 0; a < 3; a++) { T[a] = tv[t][a]; T[3 + a] = tv[t][3 + a] - tv[t][a]; T[6 + a] = tv[t][6 + a] - tv[t][a]; }
        {   // Gram entries and the reciprocal denominators of the division-free closest-point test (isdf_mesh.cuh, TRI_STRIDE)
            const double abab = T[3] * T[3] + T[4] * T[4] + T[5] * T[5], abac = T[3] * T[6] + T[4] * T[7] + T[5] * T[8],
                         acac = T[6] * T[6] + T[7] * T[7] + T[8] * T[8];
            const double bcbc = (abab - abac) + (acac - abac), det = abab * acac - abac * abac;
            T[9] = abab; T[10] = abac; T[11] = acac;
            T[12] = abab > 0.0 ? 1.0 / abab : 0.0; T[13] = acac > 0.0 ? 1.0 / acac : 0.0; T[14] = bcbc > 0.0 ? 1.0 / bcbc : 0.0;
            T[15] = det > 0.0 ? 1.0 / det : 0.0;
        }
        double *Pn = &out.pnormals[(size_t)21 * pos];
        for (int a = 0; a < 3; a++) Pn[a] = fn[t][a];
        for (int k = 0; k < 3; k++) {  // edges ab, bc, ca
            const int u = fi[t][k], v = fi[t][(k + 1) % 3];
            const auto &e = en[{std::min(u, v), std::max(u, v)}];
            for (int a = 0; a < 3; a++) Pn[3 + 3 * k + a] = e[a];
        }
        for (int k = 0; k < 3; k++) for (int a = 0; a < 3; a++) Pn[12 + 3 * k + a] = vn[fi[t][k]][a];
    }
    // winding-number tree over the same nodes: vector area, first-moment tensor and radius about the area-weighted centroid
    if (out.sign_mode == MESH_SIGN_WINDING) {
        out.wn.resize(bn.size());
        for (size_t i = 0; i < bn.size(); i++) {
            WnNode &w = out.wn[i];
            const auto &b = bn[i];
            w.left = b.left; w.right = b.right; w.first = b.first; w.count = b.count;
            double asum = 0, c[3] = {0, 0, 0};
            for (int t = b.first; t < b.first + b.count; t++) {
                const double *T = &out.tris[(size_t)TRI_STRIDE * t];
                const double nx = T[4] * T[8] - T[5] * T[7], ny = T[5] * T[6] - T[3] * T[8], nz = T[3] * T[7] - T[4] * T[6];   // ab x ac = 2 a_t n_t
                const double ar = 0.5 * std::sqrt(nx * nx + ny * ny + nz * nz);
                for (int a = 0; a < 3; a++) c[a] += ar * (T[a] + (T[3 + a] + T[6 + a]) / 3.0);
                asum += ar;
            }
            for (int a = 0; a < 3; a++) w.c[a] = asum > 0 ? c[a] / asum : 0.5 * (b.lo[a] + b.hi[a]);
            for (int a = 0; a < 3; a++) w.N[a] = 0;
            for (int a = 0; a < 9; a++) w.M[a] = 0;
            w.r2 = 0;
            for (int t = b.first; t < b.first + b.count; t++) {
                const double *T = &out.tris[(size_t)TRI_STRIDE * t];
                const double an[3] = {0.5 * (T[4] * T[8] - T[5] * T[7]), 0.5 * (T[5] * T[6] - T[3] * T[8]), 0.5 * (T[3] * T[7] - T[4] * T[6])};   // a_t n_t
                double dct[3];
                for (int a = 0; a < 3; a++) { dct[a] = T[a] + (T[3 + a] + T[6 + a]) / 3.0 - w.c[a]; w.N[a] += an[a]; }
                for (int a = 0; a < 3; a++) for (int q = 0; q < 3; q++) w.M[3 * a + q] += dct[a] * an[q];
                for (int k = 0; k < 3; k++) {
                    double d2 = 0;
                    for (int a = 0; a < 3; a++) { const double v = T[a] + (k == 1 ? T[3 + a] : 0.0) + (k == 2 ? T[6 + a] : 0.0) - w.c[a]; d2 += v * v; }
                    w.r2 = std::max(w.r2, d2);
                }
            }
        }
    }
    // fat nodes: every internal node carries both children's boxes
    auto code_of = [&](int bi, const std::vector<int> &fat_index) -> int {
        const auto &b = bn[bi];
        if (b.left < 0) return ~(b.first * 4 + (b.count - 1));
        return fat_index[bi];
    };
    std::vector<int> fat_index(bn.size(), -1);
    int nfat = 0;
    for (size_t i = 0; i < bn.size(); i++) if (bn[i].left >= 0) fat_index[i] = nfat++;
    if (nfat == 0) {  // whole mesh is one leaf
        out.nodes.resize(1);
        BvhNode &n = out.nodes[0];
        for (int a = 0; a < 3; a++) { n.lbox[a] = n.rbox[a] = bn[0].lo[a]; n.lbox[3 + a] = n.rbox[3 + a] = bn[0].hi[a]; }
        n.left = n.right = code_of(0, fat_index); n.pad0 = n.pad1 = 0;
    } else {
        out.nodes.resize(nfat);
        for (size_t i = 0; i < bn.size(); i++) {
            if (bn[i].left < 0) continue;
            BvhNode &n = out.nodes[fat_index[i]];
            const auto &L = bn[bn[i].left], &R = bn[bn[i].right];
            for (int a = 0; a < 3; a++) { n.lbox[a] = L.lo[a]; n.lbox[3 + a] = L.hi[a]; n.rbox[a] = R.lo[a]; n.rbox[3 + a] = R.hi[a]; }
            n.left = code_of(bn[i].left, fat_index); n.right = code_of(bn[i].right, fat_index); n.pad0 = n.pad1 = 0;
        }
    }
    // 32-ary nodes: collapse five binary levels per wide level (same leaves, same triangle order)
    {
        out.wnodes.clear();
        struct Job { int bin; int wide; int depth; };
        std::vector<Job> jobs;
        out.wnodes.emplace_back();
        jobs.push_back({0, 0, 1});
        int max_depth = 1;
        for (size_t j = 0; j < jobs.size(); j++) {
            const Job job = jobs[j];
            max_depth = std::max(max_depth, job.depth);
            std::vector<int> frontier{job.bin};
            if (bn[job.bin].left >= 0) {
                for (int lvl = 0; lvl < 5; lvl++) {
                    std::vector<int> nxt;
                    for (int f : frontier) {
                        if (bn[f].left >= 0) { nxt.push_back(bn[f].left); nxt.push_back(bn[f].right); }
                        else nxt.push_back(f);
                    }
                    frontier.swap(nxt);
                }
            }
            WideNode w;
            for (int k = 0; k < 32; k++) {
                for (int a = 0; a < 3; a++) { w.lo[a][k] = 1e300; w.hi[a][k] = -1e300; }
                w.child[k] = WIDE_EMPTY;
            }
            for (size_t k = 0; k < frontier.size(); k++) {
                const auto &b = bn[frontier[k]];
                for (int a = 0; a < 3; a++) { w.lo[a][k] = b.lo[a]; w.hi[a][k] = b.hi[a]; }
                if (b.left < 0) w.child[k] = ~(b.first * 8 + (b.count - 1));
                else {
                    w.child[k] = (int)out.wnodes.size();
                    out.wnodes.emplace_back();
                    jobs.push_back({frontier[k], w.child[k], job.depth + 1});
                }
            }
            out.wnodes[job.wide] = w;
        }
        // oriented boxes of the leaves (see DevMesh::leaf_obb): axis 0 = area-weighted mean normal of the leaf's triangles,
        // axis 1 = its longest edge projected into the plane, axis 2 = their cross product; extents from the vertices,
        // padded so that rounding can never put a vertex outside the box
        out.leaf_obb.assign((size_t)15 * nF, 0.0);
        for (const auto &b : bn) {
            if (b.left >= 0) continue;
            double n[3] = {0, 0, 0}, le[3] = {0, 0, 0}, le2 = -1.0;
            std::vector<std::array<double, 3>> pts;
            for (int t = b.first; t < b.first + b.count; t++) {
                const double *T = &out.tris[(size_t)TRI_STRIDE * t];
                const double A[3] = {T[0], T[1], T[2]}, B[3] = {T[0] + T[3], T[1] + T[4], T[2] + T[5]}, Cc[3] = {T[0] + T[6], T[1] + T[7], T[2] + T[8]};
                pts.push_back({A[0], A[1], A[2]}); pts.push_back({B[0], B[1], B[2]}); pts.push_back({Cc[0], Cc[1], Cc[2]});
                n[0] += T[4] * T[8] - T[5] * T[7]; n[1] += T[5] * T[6] - T[3] * T[8]; n[2] += T[3] * T[7] - T[4] * T[6];
                const double *E[3][2] = {{A, B}, {B, Cc}, {Cc, A}};
                for (auto &e : E) {
                    const double d[3] = {e[1][0] - e[0][0], e[1][1] - e[0][1], e[1][2] - e[0][2]};
                    const double l2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
                    if (l2 > le2) { le2 = l2; le[0] = d[0]; le[1] = d[1]; le[2] = d[2]; }
                }
            }
            double ax[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
            const double nl = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
            if (nl > 1e-300 && le2 > 0) {
                for (int a = 0; a < 3; a++) n[a] /= nl;
                const double dp = le[0] * n[0] + le[1] * n[1] + le[2] * n[2];
                double u[3] = {le[0] - dp * n[0], le[1] - dp * n[1], le[2] - dp * n[2]};
                const double ul = std::sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
                if (ul > 1e-9 * std::sqrt(le2)) {
                    for (int a = 0; a < 3; a++) u[a] /= ul;
                    const double w[3] = {n[1] * u[2] - n[2] * u[1], n[2] * u[0] - n[0] * u[2], n[0] * u[1] - n[1] * u[0]};
                    for (int a = 0; a < 3; a++) { ax[0][a] = n[a]; ax[1][a] = u[a]; ax[2][a] = w[a]; }
                }
            }
            double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300}, scale = 0;
            for (const auto &q : pts)
                for (int k = 0; k < 3; k++) {
                    const double pr = q[0] * ax[k][0] + q[1] * ax[k][1] + q[2] * ax[k][2];
                    lo[k] = std::min(lo[k], pr); hi[k] = std::max(hi[k], pr);
                    scale = std::max(scale, std::fabs(pr));
                }
            double *o = &out.leaf_obb[(size_t)15 * b.first];
            for (int a = 0; a < 3; a++) {
                o[a] = 0.0;
                for (int k = 0; k < 3; k++) o[a] += 0.5 * (lo[k] + hi[k]) * ax[k][a];
            }
            for (int k = 0; k < 3; k++) {
                for (int a = 0; a < 3; a++) o[3 + 3 * k + a] = ax[k][a];
                o[12 + k] = 0.5 * (hi[k] - lo[k]) + 1e-9 * (1.0 + scale);
            }
        }
        if (max_depth > 3) { err = "mesh too large for the 3-level 32-ary tree (more than ~130k triangles)"; return false; }
    }
    for (int a = 0; a < 3; a++) { out.blo[a] = bn[0].lo[a]; out.bhi[a] = bn[0].hi[a]; }
    // cell grid geometry (the per-cell distance / seed arrays are filled by k_mesh_cells on the device):
    // AABB padded by `pad`, cell edge 0.1 (body-frame metres) or coarser so that no axis exceeds 160 cells.
    {
        const double pad = 2.0 * sign_reach + 0.1;   // covers the discrete reach (safety_hor) and the swept one (2*safety_hor+0.1)
        double ext = 0;
        for (int a = 0; a < 3; a++) ext = std::max(ext, out.bhi[a] - out.blo[a] + 2 * pad);
        const double cell = std::max(0.1, ext / 160.0);
        out.gcell = cell; out.gpad = pad;
        for (int a = 0; a < 3; a++) {
            out.glo[a] = out.blo[a] - pad;
            out.gdim[a] = (int)std::ceil((out.bhi[a] - out.blo[a] + 2 * pad) / cell) + 1;
        }
        const double hd = 0.5 * std::sqrt(3.0) * cell;
        out.ghd = hd * (1.0 + 1e-6) + 1e-5 * std::max(1.0, ext);   // + float rounding of cell_dist
        out.sign_radius = (2.0 * hd < 0.9 * sign_reach) ? sign_reach : 0.0;
    }
    return true;
}

}  // namespace isdf
