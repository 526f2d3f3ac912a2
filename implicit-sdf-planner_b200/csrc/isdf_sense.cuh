// Depth sensing from poses (include/isdf.h, DESIGN §3.18): the reference's depth camera (local_sensing: DepthRender::render_pose and
// pcl_render_node.cpp's render_pcl_world), batched over poses.
//   k_sense_bounds / k_sense_keys / k_sense_gather / k_sense_bricks : the scene cloud binned once per context: the finite records sorted by
//                     a 30-bit Morton code over the cloud's box and cut into bricks of SENSE_BRICK consecutive points, each with its FP32 box
//   k_sense_poses   : per pose, cam2world in FP64 and the render's camera-from-world in FP32 (the reference's Parameter)
//   k_sense_cull    : one thread per (pose, brick): a brick no point of which can reach the image (or, for clouds, lie within the horizon)
//                     is dropped; the survivors go to a work list
//   k_sense_splat   : one warp per work item, one lane per point; splats of more than SENSE_SMALL clipped pixels are done by the whole warp
//   k_sense_flags / k_sense_write : the sensed points, one thread per pixel in the node's order (u outer, v inner), compacted by a scan
// Compiled only into isdf_sense_tu.cu with -fmad=false; the FP32 render arithmetic is written with explicit intrinsics as well, so that it
// has the reference build's contraction (FMUL y, FFMA x, FFMA z, FADD t; FFMA for the projection and for dist_mm) whatever the unit's
// setting.
#pragma once
#include "../../include/isdf.h"
#include "isdf_types.cuh"

namespace isdf {

constexpr int SENSE_BRICK = 128;        // points per brick (the last brick of the cloud may hold fewer)
constexpr int SENSE_SMALL = 16;         // a splat of at most this many clipped pixels stays with its lane
constexpr int SENSE_INIT = 999999;      // depth_initial's value: nothing seen
constexpr long long SENSE_PIX_CAP = 1ll << 25;    // image pixels of one chunk of poses (128 MB of int32)
constexpr long long SENSE_WORK_CAP = 1ll << 24;   // (pose, brick) pairs of one chunk

// one pose: the render's camera-from-world (FP32, as Parameter holds it), cam2world's top three rows and the body position (FP64)
struct SensePose {
    float r[9], t[3];
    double c2w[12], body[3];
    double cull_off;   // |camera position - body position|: the horizon cull's offset
};

// one camera of a view-gain rig (isdf_view.cuh): its horizon, the render's FP32 intrinsics (as doubles) and its image size
struct ViewCam { double horizon, fx, fy, cx, cy; int w, h; };

// the scene cloud of a context: sorted finite points, brick boxes; set once by sense_set_cloud
struct SenseScene {
    bool have = false;
    long long n = 0, skipped = 0, nb = 0;
    DevBuf<float> d_pts;    // 3 n floats, brick-contiguous
    DevBuf<float> d_box;    // 6 nb floats: lo xyz, hi xyz
    // per-call scratch: poses, work list, images, flags and their scan
    DevBuf<SensePose> d_pose; DevBuf<uint2> d_work; DevBuf<unsigned long long> d_nwork; DevBuf<int32_t> d_img, d_flag;
    DevBuf<long long> d_base; DevBuf<char> d_tmp;
    DevBuf<int32_t> d_mip; DevBuf<unsigned long long> d_obs_cnt;   // isdf_map_observe: the chunk's min-mips, its counts
    DevBuf<SensePose> d_view_pose; DevBuf<ViewCam> d_view_cam;     // isdf_view_gain: the chunk's (camera, pose) transforms, the rig
    int chunk_override = 0;   // poses per chunk (isdf_dbg_sense_chunk; 0: automatic)
    // give up the cloud and the scratch sized for it
    void release() {
        have = false; n = skipped = nb = 0;
        d_pts = {}; d_box = {}; d_work = {}; d_img = {}; d_flag = {}; d_tmp = {}; d_mip = {};
    }
};

// the pose records of a call: Q poses at pos + q stride and quat + q stride (device pointers)
struct SenseCall {
    long long Q;
    const double *pos, *quat;
    long long stride;
    isdf_sense_params p;
};

// ---- host interface of the sensing translation unit (isdf_sense_tu.cu); each returns a CUDA error or cudaSuccess ----
// d_rec: n records of stride bytes on the device, ready on st (synchronised once). On success the scene holds the finite ones and counts
// the others in S.skipped; the caller has released the previous cloud.
cudaError_t sense_set_cloud(SenseScene &S, const char *d_rec, long long n, int stride, cudaStream_t st, int *launches);
// depth images Q x H x W into out (device or host memory, by kind), on st
cudaError_t sense_depth_run(SenseScene &S, const SenseCall &C, int32_t *out, cudaMemcpyKind kind, cudaStream_t st, int *launches);
// sensed points: d_points (cap x 3 floats, device, may be NULL when cap = 0) and d_off (Q + 1 int64, device), on st
cudaError_t sense_cloud_run(SenseScene &S, const SenseCall &C, float *d_points, long long cap, int64_t *d_off, cudaStream_t st, int *launches);

// ---- known space (isdf_observe.cuh, compiled in the same unit) ----
// marks known, in the grid G's layout at known, the voxels the images of the call's poses prove empty; cnt[0..1] = {voxels tested, voxels
// added} (host), on st, which this synchronises
cudaError_t sense_observe_run(SenseScene &S, const SenseCall &C, const DevGrid &G, uint32_t *known, unsigned long long cnt[2], cudaStream_t st,
                              int *launches);
// marks known the voxels whose padded cube lies inside the closed box lo, hi (host), on st
cudaError_t known_mark_box(const DevGrid &G, uint32_t *known, const double lo[3], const double hi[3], cudaStream_t st, int *launches);
// view gain: d_gain[q] (device, Q) = the unknown voxels of G (known NULL: nothing known) the ncam cameras would see from pose q of the records
// at pos / quat (device, stride doubles apart), on st; poses with d_want[q] == 0 (d_want may be NULL: every pose wanted) are skipped and count 0
cudaError_t view_gain_run(SenseScene &S, long long Q, const double *pos, const double *quat, long long stride, int ncam,
                          const isdf_sense_params *cams, const DevGrid &G, const uint32_t *known, const uint8_t *d_want, int64_t *d_gain,
                          cudaStream_t st, int *launches);
// out = G.bits | (~known & valid bits), known NULL meaning nothing known, on st
cudaError_t blocked_build(const DevGrid &G, const uint32_t *known, uint32_t *out, cudaStream_t st, int *launches);

}  // namespace isdf
