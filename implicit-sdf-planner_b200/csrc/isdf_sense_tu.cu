// Translation unit of depth sensing (isdf_sense.cuh): the scene's bricks, the per-pose cull, the splat and the sensed-point compaction.
// Compiled with -fmad=false, so the FP64 pose and back-projection arithmetic rounds operation by operation as the reference's g++ build;
// the render's FP32 arithmetic is spelled with intrinsics, so its contraction is the reference CUDA build's whatever the unit's setting.
#include "isdf_sense.cuh"
#include "isdf_observe.cuh"
#include "isdf_view.cuh"
#include "isdf_math.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <vector>
#include <cmath>

namespace isdf {
namespace {

__device__ __forceinline__ uint32_t ord_of(float f) { const uint32_t u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float float_of(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }
__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }
__device__ __forceinline__ uint32_t spread10(uint32_t v) {
    v &= 0x3ffu;
    v = (v | (v << 16)) & 0x030000ffu; v = (v | (v << 8)) & 0x0300f00fu; v = (v | (v << 4)) & 0x030c30c3u; v = (v | (v << 2)) & 0x09249249u;
    return v;
}

// ext[0..2] ordered min, ext[3..5] ordered max of the finite records, ext[6] records skipped
__global__ void __launch_bounds__(256) k_sense_bounds(const char *rec, long long n, int stride, uint32_t *ext) {
    uint32_t lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0, 0, 0}, bad = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float *p = reinterpret_cast<const float *>(rec + i * stride);
        const float c[3] = {p[0], p[1], p[2]};
        if (!finite3(c[0], c[1], c[2])) { bad++; continue; }
        for (int a = 0; a < 3; a++) { const uint32_t o = ord_of(c[a]); lo[a] = min(lo[a], o); hi[a] = max(hi[a], o); }
    }
    for (int a = 0; a < 3; a++) { atomicMin(ext + a, lo[a]); atomicMax(ext + 3 + a, hi[a]); }
    if (bad) atomicAdd(ext + 6, bad);
}

// Morton key over the cloud's box (10 bits per axis); non-finite records sort last
__global__ void __launch_bounds__(256) k_sense_keys(const char *rec, long long n, int stride, const uint32_t *ext, uint32_t *key, uint32_t *idx) {
    float lo[3], sc[3];
    for (int a = 0; a < 3; a++) {
        lo[a] = float_of(ext[a]);
        const float w = float_of(ext[3 + a]) - lo[a];
        sc[a] = w > 0.0f ? 1023.0f / w : 0.0f;
    }
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float *p = reinterpret_cast<const float *>(rec + i * stride);
        uint32_t k = 0xffffffffu;
        if (finite3(p[0], p[1], p[2])) {
            k = 0;
            for (int a = 0; a < 3; a++) k |= spread10((uint32_t)min(1023.0f, fmaxf(0.0f, (p[a] - lo[a]) * sc[a]))) << a;
        }
        key[i] = k; idx[i] = (uint32_t)i;
    }
}

__global__ void __launch_bounds__(256) k_sense_gather(const char *rec, long long m, int stride, const uint32_t *idx, float *pts) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) {
        const float *p = reinterpret_cast<const float *>(rec + (long long)idx[i] * stride);
        pts[3 * i] = p[0]; pts[3 * i + 1] = p[1]; pts[3 * i + 2] = p[2];
    }
}

// one warp per brick: the FP32 box of its points
__global__ void __launch_bounds__(256) k_sense_bricks(const float *pts, long long m, long long nb, float *box) {
    const long long b = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (b >= nb) return;
    const long long i0 = b * SENSE_BRICK, i1 = min(m, i0 + SENSE_BRICK);
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (long long i = i0 + lane; i < i1; i += 32)
        for (int a = 0; a < 3; a++) { lo[a] = fminf(lo[a], pts[3 * i + a]); hi[a] = fmaxf(hi[a], pts[3 * i + a]); }
    for (int o = 16; o; o >>= 1)
        for (int a = 0; a < 3; a++) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    if (lane == 0) for (int a = 0; a < 3; a++) { box[6 * b + a] = lo[a]; box[6 * b + 3 + a] = hi[a]; }
}

// the pose of record q0 + i (include/isdf.h: cam2world in FP64, then the rigid inverse rounded to FP32)
__global__ void k_sense_poses(const SenseCall C, long long q0, int P, SensePose *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const long long q = q0 + i;
    const double *ps = C.pos + q * C.stride, *qs = C.quat + q * C.stride;
    quat4 qq; qq.w = qs[0]; qq.x = qs[1]; qq.y = qs[2]; qq.z = qs[3];
    const rot3 R = quat_rot(qq);
    const double B[3][4] = {{R.r0.x, R.r0.y, R.r0.z, ps[0]}, {R.r1.x, R.r1.y, R.r1.z, ps[1]}, {R.r2.x, R.r2.y, R.r2.z, ps[2]}};
    const double *Cb = C.p.cam_to_body;
    SensePose o;
    for (int r = 0; r < 3; r++)
        for (int j = 0; j < 4; j++)
            o.c2w[4 * r + j] = ((B[r][0] * Cb[j] + B[r][1] * Cb[4 + j]) + B[r][2] * Cb[8 + j]) + B[r][3] * Cb[12 + j];
    const double c0 = o.c2w[3], c1 = o.c2w[7], c2 = o.c2w[11];
    for (int r = 0; r < 3; r++) {
        const double a0 = o.c2w[r], a1 = o.c2w[4 + r], a2 = o.c2w[8 + r];   // column r of the rotation = row r of its transpose
        o.r[3 * r] = (float)a0; o.r[3 * r + 1] = (float)a1; o.r[3 * r + 2] = (float)a2;
        o.t[r] = (float)(-((a0 * c0 + a1 * c1) + a2 * c2));
    }
    for (int k = 0; k < 3; k++) o.body[k] = ps[k];
    const double d0 = c0 - ps[0], d1 = c1 - ps[1], d2 = c2 - ps[2];
    o.cull_off = sqrt((d0 * d0 + d1 * d1) + d2 * d2);
    out[i] = o;
}

// The cull. For a linear f(p) = a.p + b of the world point, its extremes over a box are exact in real numbers and tiny-error in FP64; the
// kernel's FP32 transform differs from the real transform by at most E_i = 1e-6 (sum_k |r_ik| M + |t_i|), M the box's largest |coordinate|
// (four roundings of 2^-24 each are below 5e-7). A brick is dropped when, with these margins, (1) z <= 0 over the whole box, or (2) the
// projected centre lies a whole pixel (plus a relative 1e-5) outside the image on one side over the whole box, or (3) for clouds, every z
// exceeds (horizon + camera offset)(1 + 1e-6) + 2 mm. Boxes or poses beyond 1e30 are never dropped (their FP32 transform may overflow).
__device__ bool sense_keep(const SensePose &P, const float *bx, const isdf_sense_params &cam, bool horizon) {
    double c[3], h[3], M = 0;
    for (int a = 0; a < 3; a++) {
        const double lo = bx[a], hi = bx[3 + a];
        c[a] = 0.5 * (lo + hi); h[a] = 0.5 * (hi - lo);
        M = fmax(M, fmax(fabs(lo), fabs(hi)));
    }
    double cen[3], ext[3], E[3];
    for (int i = 0; i < 3; i++) {
        const double r0 = P.r[3 * i], r1 = P.r[3 * i + 1], r2 = P.r[3 * i + 2];
        cen[i] = r0 * c[0] + r1 * c[1] + r2 * c[2] + (double)P.t[i];
        ext[i] = fabs(r0) * h[0] + fabs(r1) * h[1] + fabs(r2) * h[2];
        E[i] = 1e-6 * ((fabs(r0) + fabs(r1) + fabs(r2)) * M + fabs((double)P.t[i])) + 1e-30;
        if (!(E[i] < 1e24)) return true;   // also NaN poses
    }
    // the linear functions below share the box; their extremes come from the camera-frame centre and the per-axis half extents
    auto maxlin = [&](double ax, double az, double b) {   // max over the box of ax x + az z + b, plus its FP32 margin
        double v = b, e = 0;
        for (int k = 0; k < 3; k++) {
            const double a = ax * P.r[k] + az * P.r[6 + k];
            v += a * c[k]; e += fabs(a) * h[k];
        }
        return v + ax * P.t[0] + az * P.t[2] + e + fabs(ax) * E[0] + fabs(az) * E[2];
    };
    if (cen[2] + ext[2] + E[2] <= 0) return false;
    const double fx = cam.fx, fy = cam.fy, cx = cam.cx, cy = cam.cy, W = cam.width, H = cam.height;
    const double wx = 1.0 + 1e-5 * (fabs(cx) + W), wy = 1.0 + 1e-5 * (fabs(cy) + H);
    const double ax_lo = (-1.5 - wx - cx) / fx, ax_hi = (W - 0.5 + wx - cx) / fx;
    const double ay_lo = (-1.5 - wy - cy) / fy, ay_hi = (H - 0.5 + wy - cy) / fy;
    if (maxlin(1.0, -ax_lo, 0.0) <= 0) return false;   // x / z < ax_lo everywhere
    if (maxlin(-1.0, ax_hi, 0.0) <= 0) return false;   // x / z > ax_hi everywhere
    // the same for y (row 1 of the transform)
    auto maxlin_y = [&](double ay, double az) {
        double v = 0, e = 0;
        for (int k = 0; k < 3; k++) {
            const double a = ay * P.r[3 + k] + az * P.r[6 + k];
            v += a * c[k]; e += fabs(a) * h[k];
        }
        return v + ay * P.t[1] + az * P.t[2] + e + fabs(ay) * E[1] + fabs(az) * E[2];
    };
    if (maxlin_y(1.0, -ay_lo) <= 0) return false;
    if (maxlin_y(-1.0, ay_hi) <= 0) return false;
    if (horizon && isfinite(cam.sensing_horizon)) {
        const double zmin = cen[2] - ext[2] - E[2];
        if (zmin > (cam.sensing_horizon + P.cull_off) * (1.0 + 1e-6) + 2e-3) return false;
    }
    return true;
}

__global__ void __launch_bounds__(256) k_sense_cull(const SensePose *poses, int P, const float *box, long long nb, isdf_sense_params cam,
                                                    bool horizon, uint2 *work, unsigned long long *nwork) {
    const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (tid >= (long long)P * nb) return;
    const int p = (int)(tid / nb);
    const long long b = tid - (long long)p * nb;
    const bool keep = sense_keep(poses[p], box + 6 * b, cam, horizon);
    // warp-aggregated append
    const unsigned m = __ballot_sync(__activemask(), keep);
    if (!keep) return;
    const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(nwork, (unsigned long long)__popc(m));
    base = __shfl_sync(m, base, leader);
    work[base + __popc(m & ((1u << lane) - 1u))] = make_uint2((unsigned)p, (unsigned)b);
}

__global__ void __launch_bounds__(256) k_sense_fill(int32_t *img, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) img[i] = SENSE_INIT;
}

__device__ __forceinline__ void sense_min(int32_t *px, int v) { if (*px > v) atomicMin(px, v); }   // pixels only decrease: a stale read is safe

// one warp per (pose, brick) item, one lane per point (depth_render.cu:2-43 with the splat clipped to the image first)
__global__ void __launch_bounds__(256) k_sense_splat(const SensePose *poses, const float *pts, long long m, const uint2 *work,
                                                     const unsigned long long *nwork, int W, int H, float fx, float fy, float cx, float cy,
                                                     int32_t *img) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    const long long nw = (long long)*nwork;
    const double fxd = fx;
    for (long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; w < nw; w += warps) {
        const uint2 it = work[w];
        const SensePose &P = poses[it.x];
        float r[9], t[3];
        for (int k = 0; k < 9; k++) r[k] = P.r[k];
        for (int k = 0; k < 3; k++) t[k] = P.t[k];
        int32_t *im = img + (long long)it.x * W * H;
        const long long i0 = (long long)it.y * SENSE_BRICK, i1 = min(m, i0 + SENSE_BRICK);
        for (long long i = i0 + lane; i - lane < i1; i += 32) {
            int x0 = 0, x1 = -1, y0 = 0, y1 = -1, dmm = 0;
            if (i < i1) {
                const float px = pts[3 * i], py = pts[3 * i + 1], pz = pts[3 * i + 2];
                // the reference build's contraction of x r0 + y r1 + z r2 + t: FMUL y r1, FFMA x r0, FFMA z r2, FADD t
                const float X = __fadd_rn(__fmaf_rn(pz, r[2], __fmaf_rn(px, r[0], __fmul_rn(py, r[1]))), t[0]);
                const float Y = __fadd_rn(__fmaf_rn(pz, r[5], __fmaf_rn(px, r[3], __fmul_rn(py, r[4]))), t[1]);
                const float Z = __fadd_rn(__fmaf_rn(pz, r[8], __fmaf_rn(px, r[6], __fmul_rn(py, r[7]))), t[2]);
                if (!(Z <= 0.0f)) {
                    const int u = __double2int_rz(__dadd_rn((double)__fmaf_rn(__fdiv_rn(X, Z), fx, cx), 0.5));
                    const int v = __double2int_rz(__dadd_rn((double)__fmaf_rn(__fdiv_rn(Y, Z), fy, cy), 0.5));
                    if (u >= 0 && u < W && v >= 0 && v < H) {
                        dmm = __float2int_rz(__fmaf_rn(Z, 1000.0f, 0.5f));
                        const int rad = min(__double2int_rz(__dadd_rn(__ddiv_rn(__dmul_rn(0.0573, fxd), (double)Z), 0.5)), W + H);
                        x0 = max(u - rad, 0); x1 = min(u + rad, W - 1); y0 = max(v - rad, 0); y1 = min(v + rad, H - 1);
                    }
                }
            }
            const int cells = (x1 - x0 + 1) * (y1 - y0 + 1);
            if (cells > 0 && cells <= SENSE_SMALL) {
                for (int y = y0; y <= y1; y++)
                    for (int x = x0; x <= x1; x++) sense_min(im + (long long)y * W + x, dmm);
            }
            // large splats: the whole warp takes them one by one
            unsigned big = __ballot_sync(0xffffffffu, cells > SENSE_SMALL);
            while (big) {
                const int src = __ffs(big) - 1;
                big &= big - 1;
                const int bx0 = __shfl_sync(0xffffffffu, x0, src), bx1 = __shfl_sync(0xffffffffu, x1, src);
                const int by0 = __shfl_sync(0xffffffffu, y0, src), by1 = __shfl_sync(0xffffffffu, y1, src);
                const int bd = __shfl_sync(0xffffffffu, dmm, src);
                const int bw = bx1 - bx0 + 1, bc = bw * (by1 - by0 + 1);
                for (int k = lane; k < bc; k += 32) {
                    const int yy = by0 + k / bw, xx = bx0 + k % bw;
                    sense_min(im + (long long)yy * W + xx, bd);
                }
            }
        }
    }
}

// pixel k of pose p in the node's order (u = k / H, v = k % H): its world point, or false when it is skipped or beyond the horizon
__device__ __forceinline__ bool sense_point(const SensePose &P, const int32_t *im, long long k, const isdf_sense_params &cam, double w[3]) {
    const int u = (int)(k / cam.height), v = (int)(k - (long long)u * cam.height);
    float depth = __fdiv_rn((float)im[(long long)v * cam.width + u], 1000.0f);
    depth = depth < 500.0f ? depth : 0.0f;
    if (depth == 0.0f) return false;
    const double d = depth;
    const double pc0 = __ddiv_rn(__dmul_rn(__dsub_rn((double)u, cam.cx), d), cam.fx);
    const double pc1 = __ddiv_rn(__dmul_rn(__dsub_rn((double)v, cam.cy), d), cam.fy);
    for (int i = 0; i < 3; i++) {
        const double *m = P.c2w + 4 * i;
        w[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], pc0), __dmul_rn(m[1], pc1)), __dmul_rn(m[2], d)), m[3]);
    }
    const double e0 = __dsub_rn(w[0], P.body[0]), e1 = __dsub_rn(w[1], P.body[1]), e2 = __dsub_rn(w[2], P.body[2]);
    return !(__dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(e0, e0), __dmul_rn(e1, e1)), __dmul_rn(e2, e2))) > cam.sensing_horizon);
}

__global__ void __launch_bounds__(256) k_sense_flags(const SensePose *poses, int P, const int32_t *img, isdf_sense_params cam, int32_t *flag) {
    const long long WH = (long long)cam.width * cam.height, n = (long long)P * WH;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x) {
        if (i == n) { flag[i] = 0; continue; }
        const int p = (int)(i / WH);
        double w[3];
        flag[i] = sense_point(poses[p], img + p * WH, i - p * WH, cam, w) ? 1 : 0;
    }
}

// pos: the exclusive scan of the flags; base: the points of the chunks before this one
__global__ void __launch_bounds__(256) k_sense_write(const SensePose *poses, int P, long long q0, const int32_t *img, isdf_sense_params cam,
                                                     const int32_t *flag, const int32_t *pos, const long long *base, float *out, long long cap,
                                                     int64_t *off) {
    const long long WH = (long long)cam.width * cam.height, n = (long long)P * WH, b0 = *base;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(i / WH);
        const long long k = i - p * WH;
        if (k == 0) off[q0 + p] = b0 + pos[i];
        if (!flag[i]) continue;
        const long long j = b0 + pos[i];
        if (j >= cap) continue;
        double w[3];
        sense_point(poses[p], img + p * WH, k, cam, w);
        out[3 * j] = (float)w[0]; out[3 * j + 1] = (float)w[1]; out[3 * j + 2] = (float)w[2];
    }
}

__global__ void k_sense_advance(long long *base, const int32_t *pos_end, int64_t *off_end) {
    *base += *pos_end;
    if (off_end) *off_end = *base;
}

int grid_for(long long n) { return (int)std::max<long long>(1, std::min<long long>((n + 255) / 256, 132ll * 16)); }

// poses per chunk: the images and the work list of one chunk stay within their caps
int chunk_poses(const SenseScene &S, const SenseCall &C) {
    const long long WH = (long long)C.p.width * C.p.height;
    long long P = std::min<long long>(C.Q, std::max<long long>(1, SENSE_PIX_CAP / WH));
    P = std::min<long long>(P, std::max<long long>(1, SENSE_WORK_CAP / std::max<long long>(1, S.nb)));
    if (S.chunk_override > 0) P = std::min<long long>({C.Q, (long long)S.chunk_override, std::max<long long>(1, (1ll << 28) / WH)});
    return (int)P;
}

cudaError_t ensure_scratch(SenseScene &S, const SenseCall &C, int P) {
    const long long WH = (long long)C.p.width * C.p.height;
    cudaError_t e;
    if ((e = S.d_pose.ensure(P)) != cudaSuccess) return e;
    if ((e = S.d_work.ensure((size_t)P * S.nb)) != cudaSuccess) return e;
    if ((e = S.d_nwork.ensure(1)) != cudaSuccess) return e;
    return S.d_img.ensure((size_t)P * WH);
}

// render the P poses from q0 into S.d_img
cudaError_t render_chunk(SenseScene &S, const SenseCall &C, long long q0, int P, bool horizon, cudaStream_t st, int *launches) {
    const long long WH = (long long)C.p.width * C.p.height;
    k_sense_poses<<<(P + 127) / 128, 128, 0, st>>>(C, q0, P, S.d_pose.p);
    cudaError_t e = cudaMemsetAsync(S.d_nwork.p, 0, sizeof(unsigned long long), st);
    if (e != cudaSuccess) return e;
    k_sense_fill<<<grid_for((long long)P * WH), 256, 0, st>>>(S.d_img.p, (long long)P * WH);
    *launches += 2;
    if (S.nb == 0) return cudaGetLastError();   // a cloud of non-finite records only: nothing is seen
    const long long pairs = (long long)P * S.nb;
    k_sense_cull<<<(unsigned)((pairs + 255) / 256), 256, 0, st>>>(S.d_pose.p, P, S.d_box.p, S.nb, C.p, horizon, S.d_work.p, S.d_nwork.p);
    k_sense_splat<<<132 * 8, 256, 0, st>>>(S.d_pose.p, S.d_pts.p, S.n, S.d_work.p, S.d_nwork.p, C.p.width, C.p.height, (float)C.p.fx,
                                           (float)C.p.fy, (float)C.p.cx, (float)C.p.cy, S.d_img.p);
    *launches += 2;
    return cudaGetLastError();
}

}  // namespace

cudaError_t sense_set_cloud(SenseScene &S, const char *d_rec, long long n, int stride, cudaStream_t st, int *launches) {
    DevBuf<uint32_t> d_ext, d_key[2], d_idx[2]; DevBuf<char> d_tmp;
    cudaError_t e;
    if ((e = d_ext.ensure(7)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(d_ext.p, 0xff, 3 * sizeof(uint32_t), st)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(d_ext.p + 3, 0, 4 * sizeof(uint32_t), st)) != cudaSuccess) return e;
    k_sense_bounds<<<grid_for(n), 256, 0, st>>>(d_rec, n, stride, d_ext.p);
    uint32_t ext[7];
    if ((e = cudaMemcpyAsync(ext, d_ext.p, sizeof ext, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
    const long long m = n - ext[6];
    S.skipped = ext[6];
    for (int k = 0; k < 2; k++) {
        if ((e = d_key[k].ensure(n)) != cudaSuccess) return e;
        if ((e = d_idx[k].ensure(n)) != cudaSuccess) return e;
    }
    k_sense_keys<<<grid_for(n), 256, 0, st>>>(d_rec, n, stride, d_ext.p, d_key[0].p, d_idx[0].p);
    cub::DoubleBuffer<uint32_t> keys(d_key[0].p, d_key[1].p), vals(d_idx[0].p, d_idx[1].p);
    size_t tmp = 0;
    if ((e = cub::DeviceRadixSort::SortPairs(nullptr, tmp, keys, vals, n, 0, 32, st)) != cudaSuccess) return e;
    if ((e = d_tmp.ensure(tmp)) != cudaSuccess) return e;
    if ((e = cub::DeviceRadixSort::SortPairs(d_tmp.p, tmp, keys, vals, n, 0, 32, st)) != cudaSuccess) return e;
    S.n = m; S.nb = (m + SENSE_BRICK - 1) / SENSE_BRICK;
    if (m > 0) {
        if ((e = S.d_pts.ensure(3 * (size_t)m)) != cudaSuccess) return e;
        if ((e = S.d_box.ensure(6 * (size_t)S.nb)) != cudaSuccess) return e;
        k_sense_gather<<<grid_for(m), 256, 0, st>>>(d_rec, m, stride, vals.Current(), S.d_pts.p);
        k_sense_bricks<<<(unsigned)((S.nb * 32 + 255) / 256), 256, 0, st>>>(S.d_pts.p, m, S.nb, S.d_box.p);
    }
    *launches += m > 0 ? 4 : 2;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;   // the temporaries go out of scope here
    S.have = true;
    return cudaSuccess;
}

cudaError_t sense_depth_run(SenseScene &S, const SenseCall &C, int32_t *out, cudaMemcpyKind kind, cudaStream_t st, int *launches) {
    const long long WH = (long long)C.p.width * C.p.height;
    const int P = chunk_poses(S, C);
    cudaError_t e = ensure_scratch(S, C, P);
    if (e != cudaSuccess) return e;
    for (long long q0 = 0; q0 < C.Q; q0 += P) {
        const int np = (int)std::min<long long>(P, C.Q - q0);
        if ((e = render_chunk(S, C, q0, np, false, st, launches)) != cudaSuccess) return e;
        if ((e = cudaMemcpyAsync(out + q0 * WH, S.d_img.p, sizeof(int32_t) * np * WH, kind, st)) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t sense_cloud_run(SenseScene &S, const SenseCall &C, float *d_points, long long cap, int64_t *d_off, cudaStream_t st, int *launches) {
    const long long WH = (long long)C.p.width * C.p.height;
    const int P = chunk_poses(S, C);
    cudaError_t e = ensure_scratch(S, C, P);
    if (e != cudaSuccess) return e;
    const size_t nf = (size_t)P * WH + 1;
    if ((e = S.d_flag.ensure(2 * nf)) != cudaSuccess) return e;
    if ((e = S.d_base.ensure(1)) != cudaSuccess) return e;
    size_t tmp = 0;
    if ((e = cub::DeviceScan::ExclusiveSum(nullptr, tmp, S.d_flag.p, S.d_flag.p + nf, (int)nf, st)) != cudaSuccess) return e;
    if ((e = S.d_tmp.ensure(tmp)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(S.d_base.p, 0, sizeof(long long), st)) != cudaSuccess) return e;
    for (long long q0 = 0; q0 < C.Q; q0 += P) {
        const int np = (int)std::min<long long>(P, C.Q - q0);
        if ((e = render_chunk(S, C, q0, np, true, st, launches)) != cudaSuccess) return e;
        const long long n = (long long)np * WH;
        int32_t *flag = S.d_flag.p, *pos = S.d_flag.p + nf;
        k_sense_flags<<<grid_for(n + 1), 256, 0, st>>>(S.d_pose.p, np, S.d_img.p, C.p, flag);
        if ((e = cub::DeviceScan::ExclusiveSum(S.d_tmp.p, tmp, flag, pos, (int)(n + 1), st)) != cudaSuccess) return e;
        k_sense_write<<<grid_for(n), 256, 0, st>>>(S.d_pose.p, np, q0, S.d_img.p, C.p, flag, pos, S.d_base.p, d_points, cap, d_off);
        k_sense_advance<<<1, 1, 0, st>>>(S.d_base.p, pos + n, q0 + np == C.Q ? d_off + C.Q : nullptr);
        *launches += 4;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t sense_observe_run(SenseScene &S, const SenseCall &C, const DevGrid &G, uint32_t *known, unsigned long long cnt[2], cudaStream_t st,
                              int *launches) {
    const int P = chunk_poses(S, C);
    cudaError_t e = ensure_scratch(S, C, P);
    if (e != cudaSuccess) return e;
    ObsArgs A = {};
    A.w[0] = C.p.width; A.h[0] = C.p.height;
    long long per_image = 0;   // mip cells of one image, levels >= 1
    for (A.nlev = 1; A.w[A.nlev - 1] > 1 || A.h[A.nlev - 1] > 1; A.nlev++) {
        A.w[A.nlev] = (A.w[A.nlev - 1] + 1) / 2; A.h[A.nlev] = (A.h[A.nlev - 1] + 1) / 2;
        per_image += (long long)A.w[A.nlev] * A.h[A.nlev];
    }
    if ((e = S.d_mip.ensure((size_t)std::max(1ll, (long long)P * per_image))) != cudaSuccess) return e;
    if ((e = S.d_obs_cnt.ensure(2)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(S.d_obs_cnt.p, 0, 2 * sizeof(unsigned long long), st)) != cudaSuccess) return e;
    for (int a = 0; a < 3; a++) A.bmin[a] = G.bmin[a];
    A.res = G.res; A.X = G.X; A.Y = G.Y; A.Z = G.Z; A.Zw = G.Zw;
    A.D = (int)std::ceil(2.0 * C.p.sensing_horizon / G.res) + 3;
    A.horizon = C.p.sensing_horizon;
    A.fx = (float)C.p.fx; A.fy = (float)C.p.fy; A.cx = (float)C.p.cx; A.cy = (float)C.p.cy;
    A.known = known; A.cnt = S.d_obs_cnt.p; A.poses = S.d_pose.p; A.img = S.d_img.p; A.mip = S.d_mip.p;
    for (long long q0 = 0; q0 < C.Q; q0 += P) {
        const int np = (int)std::min<long long>(P, C.Q - q0);
        if ((e = render_chunk(S, C, q0, np, false, st, launches)) != cudaSuccess) return e;
        long long off = 0;
        for (int l = 1; l < A.nlev; l++) {
            A.off[l] = off;
            const int32_t *src = l == 1 ? S.d_img.p : S.d_mip.p + A.off[l - 1];
            k_obs_mip<<<grid_for((long long)np * A.w[l] * A.h[l]), 256, 0, st>>>(src, A.w[l - 1], A.h[l - 1], S.d_mip.p + off, A.w[l], A.h[l], np);
            off += (long long)np * A.w[l] * A.h[l];
        }
        A.P = np;
        const long long n = (long long)np * A.D * A.D * A.D;
        k_obs_voxels<<<(unsigned)std::min<long long>((n + 255) / 256, 132ll * 32), 256, 0, st>>>(A);
        *launches += A.nlev;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    if ((e = cudaMemcpyAsync(cnt, S.d_obs_cnt.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
    return cudaStreamSynchronize(st);
}

cudaError_t view_gain_run(SenseScene &S, long long Q, const double *pos, const double *quat, long long stride, int ncam,
                          const isdf_sense_params *cams, const DevGrid &G, const uint32_t *known, const uint8_t *d_want, int64_t *d_gain,
                          cudaStream_t st, int *launches) {
    // poses per chunk: one grid row each (gridDim.y <= 65535), and at most 2^18 (camera, pose) transforms
    const int P = (int)std::min<long long>({Q, 65535ll, std::max(1ll, (1ll << 18) / ncam)});
    cudaError_t e;
    if ((e = S.d_view_pose.ensure((size_t)P * ncam)) != cudaSuccess) return e;
    std::vector<ViewCam> hc(ncam);
    ViewArgs A = {};
    A.hmax = 0.0;
    for (int c = 0; c < ncam; c++) {
        hc[c] = {cams[c].sensing_horizon, (double)(float)cams[c].fx, (double)(float)cams[c].fy, (double)(float)cams[c].cx,
                 (double)(float)cams[c].cy, cams[c].width, cams[c].height};
        A.hmax = std::max(A.hmax, cams[c].sensing_horizon);
    }
    if ((e = S.d_view_cam.upload(hc.data(), hc.size(), st)) != cudaSuccess) return e;
    for (int a = 0; a < 3; a++) A.bmin[a] = G.bmin[a];
    A.res = G.res; A.X = G.X; A.Y = G.Y; A.Z = G.Z; A.Zw = G.Zw;
    A.D = (int)std::ceil(2.0 * A.hmax / G.res) + 3;
    A.occ = G.bits; A.known = known; A.cams = S.d_view_cam.p; A.ncam = ncam; A.poses = S.d_view_pose.p;
    if ((e = cudaMemsetAsync(d_gain, 0, sizeof(int64_t) * Q, st)) != cudaSuccess) return e;
    const long long D3 = (long long)A.D * A.D * A.D;
    for (long long q0 = 0; q0 < Q; q0 += P) {
        const int np = (int)std::min<long long>(P, Q - q0);
        for (int c = 0; c < ncam; c++) {
            const SenseCall C{Q, pos, quat, stride, cams[c]};
            k_sense_poses<<<(np + 127) / 128, 128, 0, st>>>(C, q0, np, S.d_view_pose.p + (size_t)c * np);
        }
        A.P = np; A.want = d_want ? d_want + q0 : nullptr; A.gain = reinterpret_cast<unsigned long long *>(d_gain + q0);
        // CTAs per pose: enough to cover the box once, fewer when many poses already fill the device
        const long long bx = std::max(1ll, std::min((D3 + 255) / 256, (132ll * 32 + np - 1) / np));
        k_view_gain<<<dim3((unsigned)bx, (unsigned)np), 256, 0, st>>>(A);
        *launches += ncam + 1;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t known_mark_box(const DevGrid &G, uint32_t *known, const double lo[3], const double hi[3], cudaStream_t st, int *launches) {
    const int dims[3] = {G.X, G.Y, G.Z};
    int i0[3], n[3];
    for (int a = 0; a < 3; a++) {   // a loose index range (one voxel of slack each side); the kernel tests each cube exactly
        const double f0 = std::floor((lo[a] - G.bmin[a]) / G.res) - 1.0, f1 = std::floor((hi[a] - G.bmin[a]) / G.res) + 1.0;
        const double c0 = std::max(0.0, f0), c1 = std::min((double)dims[a] - 1.0, f1);
        if (!(c0 <= c1)) return cudaSuccess;   // the box misses the map
        i0[a] = (int)c0; n[a] = (int)(c1 - c0) + 1;
    }
    const long long cnt = (long long)n[0] * n[1] * n[2];
    k_known_boxes<<<grid_for(cnt), 256, 0, st>>>(G, known, lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], i0[0], i0[1], i0[2], n[0], n[1], n[2]);
    (*launches)++;
    return cudaGetLastError();
}

cudaError_t blocked_build(const DevGrid &G, const uint32_t *known, uint32_t *out, cudaStream_t st, int *launches) {
    const long long nwords = (long long)G.X * G.Y * G.Zw;
    k_blocked<<<grid_for(nwords), 256, 0, st>>>(G.bits, known, out, nwords, G.Z, G.Zw);
    (*launches)++;
    return cudaGetLastError();
}

}  // namespace isdf
