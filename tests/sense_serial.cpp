// TEST INFRASTRUCTURE: a serial CPU restatement of depth sensing (include/isdf.h, isdf_sense_*), without culling, bricks or chunks.
// Built by tests/sense_oracle.py with -ffp-contract=off: every FP32 and FP64 operation rounds on its own except where std::fmaf restates
// the reference CUDA build's contraction (FFMA). Float-to-int conversions are the GPU's: truncation toward zero, saturating, NaN to 0.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <climits>

namespace {

int f2i(double x) {   // cvt.rzi.s32: NaN -> 0, saturating
    if (std::isnan(x)) return 0;
    if (x >= 2147483647.0) return INT_MAX;
    if (x <= -2147483648.0) return INT_MIN;
    return (int)std::trunc(x);
}

// Eigen's toRotationMatrix as quat_rot writes it
void quat_rot(const double *q, double R[9]) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1.0 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1.0 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.0 - (txx + tyy);
}

}  // namespace

extern "C" {

// cam2world (16, row-major) and the render's camera-from-world as double[16] (the FP32 roundings of the rigid inverse, widened back)
void sense_pose(const double *pos, const double *quat, const double *C, double *c2w, double *cw) {
    double R[9];
    quat_rot(quat, R);
    const double B[3][4] = {{R[0], R[1], R[2], pos[0]}, {R[3], R[4], R[5], pos[1]}, {R[6], R[7], R[8], pos[2]}};
    for (int r = 0; r < 3; r++)
        for (int j = 0; j < 4; j++) c2w[4 * r + j] = ((B[r][0] * C[j] + B[r][1] * C[4 + j]) + B[r][2] * C[8 + j]) + B[r][3] * C[12 + j];
    c2w[12] = 0; c2w[13] = 0; c2w[14] = 0; c2w[15] = 1;
    const double c0 = c2w[3], c1 = c2w[7], c2 = c2w[11];
    for (int r = 0; r < 3; r++) {
        const double a0 = c2w[r], a1 = c2w[4 + r], a2 = c2w[8 + r];
        cw[4 * r] = (float)a0; cw[4 * r + 1] = (float)a1; cw[4 * r + 2] = (float)a2;
        cw[4 * r + 3] = (float)(-((a0 * c0 + a1 * c1) + a2 * c2));
    }
    cw[12] = 0; cw[13] = 0; cw[14] = 0; cw[15] = 1;
}

// DepthRender::render_pose from its double[16] input: img (H x W) in mm; returns the records skipped as non-finite
long long sense_render(const float *rec, long long n, int stride_floats, const double *T, int W, int H, double fxd, double fyd, double cxd,
                       double cyd, int32_t *img) {
    float r[9], t[3];
    for (int i = 0; i < 3; i++) { t[i] = (float)T[4 * i + 3]; for (int j = 0; j < 3; j++) r[3 * i + j] = (float)T[4 * i + j]; }
    const float fx = (float)fxd, fy = (float)fyd, cx = (float)cxd, cy = (float)cyd;
    for (long long i = 0; i < (long long)W * H; i++) img[i] = 999999;
    long long skipped = 0;
    for (long long i = 0; i < n; i++) {
        const float *p = rec + i * stride_floats;
        if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) { skipped++; continue; }
        float c[3];
        for (int k = 0; k < 3; k++) c[k] = std::fmaf(p[2], r[3 * k + 2], std::fmaf(p[0], r[3 * k], p[1] * r[3 * k + 1])) + t[k];
        if (c[2] <= 0.0f) continue;
        const int u = f2i((double)std::fmaf(c[0] / c[2], fx, cx) + 0.5);
        const int v = f2i((double)std::fmaf(c[1] / c[2], fy, cy) + 0.5);
        if (u < 0 || u >= W || v < 0 || v >= H) continue;
        const int dmm = f2i((double)std::fmaf(c[2], 1000.0f, 0.5f));
        const long long rad = f2i(0.0573 * (double)fx / (double)c[2] + 0.5);
        for (long long y = std::max<long long>(v - rad, 0); y <= std::min<long long>(v + rad, H - 1); y++)
            for (long long x = std::max<long long>(u - rad, 0); x <= std::min<long long>(u + rad, W - 1); x++)
                if (img[y * W + x] > dmm) img[y * W + x] = dmm;
    }
    return skipped;
}

// render_pcl_world of one pose's image: up to W H points (3 floats each) in the node's order; returns their number
long long sense_backproject(const int32_t *img, int W, int H, double fx, double fy, double cx, double cy, const double *c2w,
                            const double *body, double horizon, float *out) {
    long long m = 0;
    for (int u = 0; u < W; u++)
        for (int v = 0; v < H; v++) {
            float depth = (float)img[(long long)v * W + u] / 1000.0f;
            depth = depth < 500.0f ? depth : 0;
            if (depth == 0.0) continue;
            const double pc[3] = {(u - cx) * depth / fx, (v - cy) * depth / fy, (double)depth};
            double w[3];
            for (int i = 0; i < 3; i++) w[i] = ((c2w[4 * i] * pc[0] + c2w[4 * i + 1] * pc[1]) + c2w[4 * i + 2] * pc[2]) + c2w[4 * i + 3];
            const double d0 = w[0] - body[0], d1 = w[1] - body[1], d2 = w[2] - body[2];
            if (std::sqrt((d0 * d0 + d1 * d1) + d2 * d2) > horizon) continue;
            out[3 * m] = (float)w[0]; out[3 * m + 1] = (float)w[1]; out[3 * m + 2] = (float)w[2];
            m++;
        }
    return m;
}

}  // extern "C"
