// ORACLE — TEST INFRASTRUCTURE ONLY.
// C wrapper around the reference's own distance field, compiled UNMODIFIED from where it lies:
//   /root/reference/src/map_manager/src/Gridmap3D.cpp + include/map_manager/GridMap3D.h
//     createGridMap :25-39, generateESDF3d :361-525 with fillESDF :527-560, getGridSDFValue(const Vector3i &) :562-569,
//     getSDFValue / getSDFValueWithGrad GridMap3D.h:114-193
// against oracle/_shim_dyn/Eigen/Eigen and the ROS stand-ins beside it (esdf.mk builds it into oracle/_ref/libref_esdf.so). The map is
// created with an explicit bmax, so cloud-framed maps (bmax != bmin + X*res) are covered.
#include "map_manager/GridMap3D.h"
#include <cstdint>
#include <cstddef>

static GridMap3D *make(const uint8_t *occ, int X, int Y, int Z, const double *bmin, const double *bmax, double res) {
    GridMap3D *g = new GridMap3D();
    g->grid_resolution = res;
    g->debug_output = false;
    g->createGridMap(Vector3d(bmin[0], bmin[1], bmin[2]), Vector3d(bmax[0], bmax[1], bmax[2]));
    if (g->X_size != X || g->Y_size != Y || g->Z_size != Z) { g->releaseMemory(); delete g; return nullptr; }
    const size_t n = (size_t)X * Y * Z;
    for (size_t i = 0; i < n; i++) g->grid_map[i] = occ[i] ? 1.0 : 0.0;
    g->generateESDF3d();
    return g;
}

// generateESDF3d allocates grid_esdf and its two buffers; releaseMemory frees neither
static void destroy(GridMap3D *g) {
    delete[] g->grid_esdf; delete[] g->grid_esdf_buffer1; delete[] g->grid_esdf_buffer2;
    g->releaseMemory();
    delete g;
}

extern "C" {
// grid_esdf, grid_map_buffer_neg and grid_map_buffer_all after generateESDF3d (X*Y*Z doubles each); -1 if createGridMap's sizes differ
int ref_grid_esdf(const uint8_t *occ, int X, int Y, int Z, const double *bmin, const double *bmax, double res, double *pos, double *neg, double *all) {
    GridMap3D *g = make(occ, X, Y, Z, bmin, bmax, res);
    if (!g) return -1;
    const size_t n = (size_t)X * Y * Z;
    for (size_t i = 0; i < n; i++) { pos[i] = g->grid_esdf[i]; neg[i] = g->grid_map_buffer_neg[i]; all[i] = g->grid_map_buffer_all[i]; }
    destroy(g);
    return 0;
}

// getSDFValueWithGrad (grad != NULL) or getSDFValue at n points on field 0 (grid_esdf), 1 (grid_map_buffer_neg) or 2 (the signed field
// pos + (-neg + res) where neg > 0). For 1 and 2 grid_esdf points at that field while the queries run, so the trilinear arithmetic is the
// reference's own; only the signed field's combine is restated here.
int ref_grid_sdf_query(const uint8_t *occ, int X, int Y, int Z, const double *bmin, const double *bmax, double res, int field, int n,
                       const double *pts, double *dist, double *grad) {
    GridMap3D *g = make(occ, X, Y, Z, bmin, bmax, res);
    if (!g) return -1;
    double *own = g->grid_esdf, *sgn = nullptr;
    if (field == 1) g->grid_esdf = g->grid_map_buffer_neg;
    if (field == 2) {
        const size_t nv = (size_t)X * Y * Z;
        sgn = new double[nv];
        for (size_t i = 0; i < nv; i++) {
            sgn[i] = own[i];
            if (g->grid_map_buffer_neg[i] > 0.0) sgn[i] += (-g->grid_map_buffer_neg[i] + res);
        }
        g->grid_esdf = sgn;
    }
    for (int q = 0; q < n; q++) {
        const Vector3d p(pts[3 * q], pts[3 * q + 1], pts[3 * q + 2]);
        if (grad) {
            Vector3d gr;
            dist[q] = g->getSDFValueWithGrad(p, gr);
            for (int k = 0; k < 3; k++) grad[3 * q + k] = gr(k);
        } else {
            dist[q] = g->getSDFValue(p);
        }
    }
    g->grid_esdf = own;
    delete[] sgn;
    destroy(g);
    return 0;
}
}
