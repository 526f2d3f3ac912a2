// TEST INFRASTRUCTURE ONLY: the front end's surcharge on unknown voxels (include/isdf.h, isdf_frontpath_params.unknown_weight) restated
// serially (tests/known_plan_oracle.py).
//   kp_dijkstra  a textbook FP64 binary-heap Dijkstra over the 26-connected voxel graph of a traversability array, with the edge into v
//                costing sqrt((double)n) when known[v] and sqrt((double)n) * cw when not (cw = 1 + unknown_weight; known NULL: nothing known)
//   kp_path      the parent rule on such a field: the first neighbour u in the reference's offset order with g(u) + w(u, v) == g(v), w read
//                at v
#include <cmath>
#include <cstdint>
#include <functional>
#include <queue>
#include <utility>
#include <vector>

namespace {
struct Dims {
    int X, Y, Z;
    long long addr(int x, int y, int z) const { return ((long long)x * Y + y) * Z + z; }
    bool in(int x, int y, int z) const { return x >= 0 && x < X && y >= 0 && y < Y && z >= 0 && z < Z; }
};
double weight(const uint8_t *known, long long v, int n, double cw) {
    const double e = std::sqrt((double)n);
    return (known && known[v]) ? e : e * cw;
}
}  // namespace

extern "C" {
// g: X*Y*Z doubles, +inf where unreachable. The source is expanded whether it is traversable or not. Returns the settled count.
int64_t kp_dijkstra(const uint8_t *trav, const uint8_t *known, int X, int Y, int Z, const int32_t *src, double cw, double *g) {
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
                    const double cand = g[u] + weight(known, v, i * i + j * j + k * k, cw);
                    if (cand < g[v]) { g[v] = cand; heap.push(Item(cand, v)); }
                }
    }
    return settled;
}

// path from src to t (start first) by the parent rule; returns the node count (1: the start alone when g(t) = inf; -1: a voxel without a
// parent) and writes up to cap nodes (3 ints each)
int64_t kp_path(const double *g, const uint8_t *known, int X, int Y, int Z, const int32_t *src, const int32_t *t, double cw, int32_t *out,
                int64_t cap) {
    const Dims D{X, Y, Z};
    std::vector<int> rev;
    int x = t[0], y = t[1], z = t[2];
    if (!std::isfinite(g[D.addr(x, y, z)])) { x = src[0]; y = src[1]; z = src[2]; }
    rev.insert(rev.end(), {x, y, z});
    while (!(x == src[0] && y == src[1] && z == src[2])) {
        const long long v = D.addr(x, y, z);
        const double gv = g[v];
        bool ok = false;
        for (int i = -1; i <= 1 && !ok; i++)
            for (int j = -1; j <= 1 && !ok; j++)
                for (int k = -1; k <= 1 && !ok; k++) {
                    const int ux = x + i, uy = y + j, uz = z + k;
                    if ((i == 0 && j == 0 && k == 0) || !D.in(ux, uy, uz)) continue;
                    const double gu = g[D.addr(ux, uy, uz)];
                    if (std::isfinite(gu) && gu + weight(known, v, i * i + j * j + k * k, cw) == gv) { x = ux; y = uy; z = uz; ok = true; }
                }
        if (!ok) return -1;
        rev.insert(rev.end(), {x, y, z});
    }
    const int64_t len = (int64_t)rev.size() / 3;
    for (int64_t m = 0; m < len && m < cap; m++)
        for (int a = 0; a < 3; a++) out[3 * m + a] = rev[3 * (len - 1 - m) + a];
    return len;
}
}
