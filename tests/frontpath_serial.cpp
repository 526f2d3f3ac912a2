// TEST INFRASTRUCTURE ONLY: CPU restatements that isdf_frontend_path is held against (tests/frontpath_oracle.py).
//   fp_dijkstra   a textbook FP64 binary-heap Dijkstra over the 26-connected voxel graph of a traversability array: the exact
//                 shortest-path field of include/isdf.h (left-to-right FP64 sums of sqrt((double)(di^2 + dj^2 + dk^2)))
//   fp_path       the parent rule of include/isdf.h on a field: first neighbour in the reference's offset order with g(u) + w == g(v)
//   fp_ref_astar  the reference's search (AstarPathSearcher::AstarPathSearch / getastarSE3Path, front_end_Astar.hpp:160-402), restated
//                 with its quirks, for comparison only: a std::multimap open set keyed on f (FIFO among equal keys), stale keys of
//                 improved open nodes, the 1.001-inflated octile heuristic, closed nodes reopened when improved, a start node that is
//                 not the grid's node, and checkKernelValue's attitude written into every neighbour an expansion looks at.
#include <cmath>
#include <cstdint>
#include <functional>
#include <map>
#include <queue>
#include <utility>
#include <vector>

namespace {
struct Dims {
    int X, Y, Z;
    long long addr(int x, int y, int z) const { return ((long long)x * Y + y) * Z + z; }
    bool in(int x, int y, int z) const { return x >= 0 && x < X && y >= 0 && y < Y && z >= 0 && z < Z; }
};
}  // namespace

extern "C" {
// g: X*Y*Z doubles, +inf where unreachable. The source is expanded whether it is traversable or not. Returns the settled count.
int64_t fp_dijkstra(const uint8_t *trav, int X, int Y, int Z, const int32_t *src, double *g) {
    const Dims D{X, Y, Z};
    const long long n = (long long)X * Y * Z;
    for (long long v = 0; v < n; v++) g[v] = INFINITY;
    std::vector<uint8_t> done((size_t)n, 0);
    typedef std::pair<double, long long> Item;
    std::priority_queue<Item, std::vector<Item>, std::greater<Item>> heap;
    const long long s = D.addr(src[0], src[1], src[2]);
    g[s] = 0.0;
    heap.push(Item(0.0, s));
    int64_t settled = 0;
    while (!heap.empty()) {
        const Item it = heap.top();
        heap.pop();
        const long long u = it.second;
        if (done[u] || it.first != g[u]) continue;
        done[u] = 1;
        settled++;
        const int ux = (int)(u / ((long long)Y * Z)), uy = (int)((u / Z) % Y), uz = (int)(u % Z);
        for (int i = -1; i <= 1; i++)
            for (int j = -1; j <= 1; j++)
                for (int k = -1; k <= 1; k++) {
                    const int x = ux + i, y = uy + j, z = uz + k;
                    if ((i == 0 && j == 0 && k == 0) || !D.in(x, y, z)) continue;
                    const long long v = D.addr(x, y, z);
                    if (!trav[v] || done[v]) continue;
                    const double cand = g[u] + std::sqrt((double)(i * i + j * j + k * k));
                    if (cand < g[v]) { g[v] = cand; heap.push(Item(cand, v)); }
                }
    }
    return settled;
}

// path from src to t (start first) by the parent rule; returns the node count (1: the start alone when g(t) = inf) and writes up to
// cap nodes (3 ints each)
int64_t fp_path(const double *g, int X, int Y, int Z, const int32_t *src, const int32_t *t, int32_t *out, int64_t cap) {
    const Dims D{X, Y, Z};
    std::vector<int> rev;
    int x = t[0], y = t[1], z = t[2];
    if (!std::isfinite(g[D.addr(x, y, z)])) { x = src[0]; y = src[1]; z = src[2]; }
    rev.insert(rev.end(), {x, y, z});
    while (!(x == src[0] && y == src[1] && z == src[2])) {
        const double gv = g[D.addr(x, y, z)];
        bool ok = false;
        for (int i = -1; i <= 1 && !ok; i++)
            for (int j = -1; j <= 1 && !ok; j++)
                for (int k = -1; k <= 1 && !ok; k++) {
                    const int ux = x + i, uy = y + j, uz = z + k;
                    if ((i == 0 && j == 0 && k == 0) || !D.in(ux, uy, uz)) continue;
                    const double gu = g[D.addr(ux, uy, uz)];
                    if (std::isfinite(gu) && gu + std::sqrt((double)(i * i + j * j + k * k)) == gv) { x = ux; y = uy; z = uz; ok = true; }
                }
        if (!ok) return -1;   // not a field of this definition
        rev.insert(rev.end(), {x, y, z});
    }
    const int64_t len = (int64_t)rev.size() / 3;
    for (int64_t m = 0; m < len && m < cap; m++)
        for (int a = 0; a < 3; a++) out[3 * m + a] = rev[3 * (len - 1 - m) + a];
    return len;
}

// The reference's A*. occ: X*Y*Z bytes; masks: 4 words per voxel, the free attitudes (isdf_frontend_feasibility). Attitudes follow
// checkKernelValue (level pose first, then a BFS from the father's attitude; maxdeepth 800). Returns 1 when the goal is popped, 0 when the
// open set empties; *cost = the goal's gScore, the path (start first) and its attitudes as getastarSE3Path reports them, up to cap nodes;
// *n = the path's node count; *expanded = nodes popped.
int fp_ref_astar(const uint8_t *occ, const uint32_t *masks, int X, int Y, int Z, const int32_t *src, const int32_t *goal, int xk, int yk,
                 double max_roll, double max_pitch, double ang_res, double *cost, int32_t *path, double *rp, int64_t cap, int64_t *n,
                 int64_t *expanded) {
    const Dims D{X, Y, Z};
    const long long nv = (long long)X * Y * Z;
    struct Node { double g = 0, f = 0, roll = 0, pitch = 0; int id = 0; long long father = -1; };
    std::vector<Node> N((size_t)nv + 1);   // N[nv]: the start node, a GridNode of its own (:261)
    const long long START = nv;
    auto fits = [&](long long v, int att) { return (masks[4 * v + (att >> 5)] >> (att & 31)) & 1u; };
    // checkKernelValue (swm:914-941) + visit_kernels_by_distance (swm:852-913)
    auto check = [&](double fr, double fp, double &cr, double &cp, long long v) {
        const int fi = (int)((fr + max_roll) / ang_res), fj = (int)((fp + max_pitch) / ang_res);
        const int zi = (xk - 1) / 2, zj = (yk - 1) / 2;
        int ri = -1, rj = -1;
        if (fits(v, zi * yk + zj)) { ri = zi; rj = zj; }
        else if (fi >= 0 && fi < xk && fj >= 0 && fj < yk) {
            std::vector<char> vis((size_t)xk * yk, 0);
            std::queue<std::pair<int, int>> q;
            q.push({fi, fj}); vis[fi * yk + fj] = 1;
            const int dirs[4][2] = {{0, 1}, {0, -1}, {1, 0}, {-1, 0}};
            int deep = 0;
            while (!q.empty()) {
                deep++;
                const int x = q.front().first, y = q.front().second;
                q.pop();
                if ((x != zi || y != zj) && fits(v, x * yk + y)) { ri = x; rj = y; break; }
                for (auto &d : dirs) {
                    const int nx = x + d[0], ny = y + d[1];
                    if (nx < 0 || nx >= xk || ny < 0 || ny >= yk || vis[nx * yk + ny]) continue;
                    vis[nx * yk + ny] = 1;
                    q.push({nx, ny});
                }
                if (deep > 800) break;
            }
        }
        if (ri < 0) return false;
        cr = fr + (ri - fi) * ang_res; cp = fp + (rj - fj) * ang_res;
        return true;
    };
    auto heu = [&](long long a) {   // getHeu (:171-187)
        const int ax = (int)(a / ((long long)Y * Z)), ay = (int)((a / Z) % Y), az = (int)(a % Z);
        const int dx = std::abs(ax - goal[0]), dy = std::abs(ay - goal[1]), dz = std::abs(az - goal[2]);
        const int dmin = std::min(dx, std::min(dy, dz)), dmax = std::max(dx, std::max(dy, dz)), dmid = dx + dy + dz - dmin - dmax;
        const double h = std::sqrt(3) * dmin + std::sqrt(2) * (dmid - dmin) + (dmax - dmid);
        return h * (1 + 1.0 / 1000);
    };
    auto index_of = [&](long long a, int id[3]) {
        if (a == START) { id[0] = src[0]; id[1] = src[1]; id[2] = src[2]; return; }
        id[0] = (int)(a / ((long long)Y * Z)); id[1] = (int)((a / Z) % Y); id[2] = (int)(a % Z);
    };
    const long long s_grid = D.addr(src[0], src[1], src[2]), gaddr = D.addr(goal[0], goal[1], goal[2]);
    std::multimap<double, long long> open;
    N[START].g = 0; N[START].f = heu(s_grid); N[START].id = 1;
    open.insert(std::make_pair(N[START].f, START));
    N[s_grid].id = 1; N[s_grid].g = 0; N[s_grid].f = N[START].f;   // :278-280 (the grid's start node is marked open, never inserted)
    long long term = -1;
    *expanded = 0;
    while (!open.empty()) {
        auto it = open.begin();
        const long long cur = it->second;
        open.erase(it);
        N[cur].id = -1;
        (*expanded)++;
        int ci[3];
        index_of(cur, ci);
        if (D.addr(ci[0], ci[1], ci[2]) == gaddr) { term = cur; break; }
        for (int i = -1; i <= 1; i++)   // AstarGetSucc (:197-236): all 27 offsets, (0, 0, 0) included
            for (int j = -1; j <= 1; j++)
                for (int k = -1; k <= 1; k++) {
                    const int x = ci[0] + i, y = ci[1] + j, z = ci[2] + k;
                    if (!D.in(x, y, z)) continue;
                    const long long v = D.addr(x, y, z);
                    if (occ[v]) continue;
                    double cr, cp;
                    if (!check(N[cur].roll, N[cur].pitch, cr, cp, v)) continue;
                    N[v].roll = cr; N[v].pitch = cp;
                    const double ec = std::sqrt((double)(i * i + j * j + k * k));
                    const double tg = ec + N[cur].g;
                    if (N[v].id == 0) {
                        N[v].father = cur; N[v].g = tg; N[v].f = tg + heu(v); N[v].id = 1;
                        open.insert(std::make_pair(N[v].f, v));
                    } else if (N[v].id == 1) {
                        if (tg < N[v].g) { N[v].father = cur; N[v].g = tg; N[v].f = tg + heu(v); }   // the open key stays stale
                    } else if (tg < N[v].g) {
                        N[v].father = cur; N[v].g = tg; N[v].f = tg + heu(v); N[v].id = 1;
                        open.insert(std::make_pair(N[v].f, v));
                    }
                }
    }
    if (term < 0) { *n = 0; *cost = INFINITY; return 0; }
    *cost = N[term].g;
    std::vector<long long> rev;
    for (long long p = term; p >= 0; p = N[p].father) rev.push_back(p);
    *n = (int64_t)rev.size();
    for (int64_t m = 0; m < *n && m < cap; m++) {
        const long long p = rev[(size_t)(*n - 1 - m)];
        index_of(p, path + 3 * m);
        rp[2 * m] = N[p].roll; rp[2 * m + 1] = N[p].pitch;
    }
    return 1;
}
}
