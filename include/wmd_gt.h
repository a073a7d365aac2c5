/*
 * wmd_gt.h - KITTI's ground-truth depths of libwmd.so on the device: the velodyne projection of
 * KITTI/kitti_utils.py:generate_depth_map (which KITTI/export_gt_depth.py runs to make splits/<split>/gt_depths.npz),
 * bit for bit, batched over frames.
 *
 * Same conventions as wmd.h (device pointers unless the name says host, caller-owned buffers, asynchronous on `stream`,
 * no host sync, no allocation, wmd_status return codes).  A header of its own: it prepares evaluation data rather than
 * running a network.  The Python binding is _lib.GT_SIGNATURES; oracle/kitti_gt.py restates the contract in numpy.
 *
 * Per frame n: the scan is points[offsets[n] .. offsets[n+1]) of (total, 4) float32 points (x forward, y left, z up,
 * reflectance) in file order; P (3, 4) fp64 is np.dot(np.dot(P_rect_0{cam}, R_cam2rect), velo2cam); (H, W) comes
 * from S_rect_02 (for either camera).  In fp64:
 *   1. a point is kept only if x >= 0 (a NaN x is dropped, -0.0 kept);
 *   2. q_r = fma(P[r][3], 1, fma(P[r][2], z, fma(P[r][1], y, P[r][0] x))), x, y, z widened from fp32 (the reflectance
 *      plays no part: the reference replaces it by 1) - np.dot(P, velo.T)'s operation order;
 *   3. u' = rint(q0 / q2) - 1, v' = rint(q1 / q2) - 1 (IEEE division, rint half to even as np.round); kept if
 *      0 <= u' < W and 0 <= v' < H (a non-finite coordinate fails; q2 <= 0 inside the image is kept);
 *   4. the point's depth is x if vel_depth, else q2;
 *   5. each pixel takes the depth of the LAST kept point on it (numpy's fancy-index assignment);
 *   6. every kept point has a group g = v' (W - 1) + u' - 1 (the reference's sub2ind, so (y, W-1) and (y+1, 0) share
 *      a group, and with W = 1 every point is in group -1); where a group holds more than one point, the pixel of its
 *      FIRST point takes the least depth of the whole group; of equal zeros that is the later point's (numpy's min
 *      of such a group), so the sign of a zero minimum is the later point's;
 *   7. depth < 0 becomes 0 (-0.0 stays -0.0).
 * Pixels no kept point reaches are +0.0, as is the padding past each frame's (H, W) in the (N, Hmax, Wmax) output.
 * Only integer atomics (max of the last point, min of the first, a count, min of an order-preserving key of the
 * depth), so the bits depend only on the inputs, never on timing, the batch or the device's SM count.
 */
#ifndef WMD_GT_H
#define WMD_GT_H

#include "wmd.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Host-only: workspace bytes of wmd_velo_depth_f64 (20 per pixel of (N, Hmax, Wmax)); 0 for a shape it refuses:
 * N < 0, Hmax or Wmax < 1, Hmax x Wmax or total_points above 2^30, or a workspace size_t cannot hold. */
size_t wmd_velo_depth_ws_bytes(int32_t N, int32_t Hmax, int32_t Wmax, long long total_points);
/* points (total, 4) fp32, 16-byte aligned; offsets (N + 1) int32, offsets[0] = 0 and nondecreasing; P (N, 3, 4) fp64;
 * sizes_host (N, 2) int32 (H, W) per frame, in HOST memory (checked here, then passed to the kernels by value);
 * depth (N, Hmax, Wmax) fp64.  WMD_ERR_ARG for a null or misaligned pointer; WMD_ERR_SHAPE for the shapes
 * wmd_velo_depth_ws_bytes refuses or a frame with H or W below 1 or above Hmax or Wmax; WMD_ERR_WORKSPACE for a short
 * workspace; all before any CUDA call.  N = 0 does nothing. */
int wmd_velo_depth_f64(const float* points, const int32_t* offsets, const double* P, const int32_t* sizes_host,
                       int32_t N, int32_t Hmax, int32_t Wmax, int32_t vel_depth, void* ws, size_t ws_bytes,
                       double* depth, wmd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* WMD_GT_H */
