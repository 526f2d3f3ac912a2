// TEST INFRASTRUCTURE ONLY: the serial CPU voxelisation of a point cloud, in the loop structure of the reference's
// PCSmapManager::rcvGlobalMapHandler (PCSmap_manager.cpp:111-181) on the oracle's grid (orc::Grid: createGridMap, getGridIndex).
// It is the CPU arm of bench_map.py and a second restatement beside the numpy one in tests/cloud_oracle.py. Same deviations as
// isdf_set_map_cloud: records with a non-finite coordinate are skipped (undefined behaviour in the reference).
#include "../oracle/oracle_planner.hpp"
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

extern "C" {
// pass 1 (dims_only != 0): dims[3], bmin[3], bmax[3], *skipped. pass 2: also occ (dims[0]*dims[1]*dims[2] bytes, 0 / 1).
// Returns 0, or -1 for no finite point or a degenerate extent.
int cloud_map_serial(const void *points, int64_t n, int32_t stride, double res, int32_t sta_threshold, int dims_only, int32_t *dims,
                     double *bmin, double *bmax, int64_t *skipped, uint8_t *occ) {
    const char *base = (const char *)points;
    auto rec = [&](int64_t i, float c[3]) {
        std::memcpy(c, base + i * stride, 3 * sizeof(float));
        return std::isfinite(c[0]) && std::isfinite(c[1]) && std::isfinite(c[2]);
    };
    orc::V3 mn(999999999, 999999999, 999999999), mx(-999999999, -999999999, -999999999);   // HUGE_NUMBER (PCSmap_manager.cpp:6,11-12)
    int64_t skip = 0;
    float c[3];
    for (int64_t i = 0; i < n; i++) {   // :111-143
        if (!rec(i, c)) { skip++; continue; }
        for (int a = 0; a < 3; a++) {
            if (c[a] > mx[a]) mx[a] = c[a];
            if (c[a] < mn[a]) mn[a] = c[a];
        }
    }
    if (skip == n) return -1;
    orc::Grid g;
    g.create(mn, mx, res);   // createGridMap
    for (int a = 0; a < 3; a++) { bmin[a] = mn[a]; bmax[a] = mx[a]; }
    dims[0] = g.X; dims[1] = g.Y; dims[2] = g.Z;
    *skipped = skip;
    if (g.X < 1 || g.Y < 1 || g.Z < 1) return -1;
    if (dims_only) return 0;
    const size_t nvox = (size_t)g.X * g.Y * g.Z;
    std::vector<uint32_t> cnt(nvox, 0);
    for (int64_t i = 0; i < n; i++) {   // :145-150
        if (!rec(i, c)) continue;
        int id[3];
        g.grid_index(orc::V3(c[0], c[1], c[2]), id);
        cnt[(size_t)id[0] * g.Y * g.Z + (size_t)id[1] * g.Z + id[2]]++;
    }
    for (size_t v = 0; v < nvox; v++) occ[v] = (int64_t)cnt[v] >= sta_threshold ? 1 : 0;   // :151-181
    return 0;
}
}
