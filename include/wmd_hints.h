/*
 * wmd_hints.h - KITTI's depth hints of libwmd.so on the device: OpenCV's StereoSGBM matcher, bit for bit, and the
 * fusion of the twelve matchers' depths by reprojection error (KITTI/precompute_depth_hints.py).
 *
 * Same conventions as wmd.h (device pointers unless the name says host, caller-owned buffers, asynchronous on `stream`,
 * no host sync, no allocation, wmd_status return codes).  A header of its own: it prepares training data rather than
 * running a network.  The Python binding is _lib.HINTS_SIGNATURES.
 *
 * Matcher: cv2.StereoSGBM_create(minDisparity=0, numDisparities, blockSize, P1=36, P2=288, preFilterCap=63,
 * uniquenessRatio=10, speckleWindowSize=100, speckleRange=16, disp12MaxDiff=0, mode=MODE_SGBM).compute(left, right)
 * on uint8 (H, W, 3) views, int16 disparity x16 out, (0 - 1) x16 = -16 where invalid.  oracle/sgbm.py restates every
 * stage: the clipped x-Sobel and raw planes, Birchfield-Tomasi costs summed over the six planes (raw ones >> 2), the
 * box sum of half-width blockSize / 2 (blockSize 2 and 3 are the same matcher) clamped to columns [D, W - 1] and rows
 * [0, H - 1], five aggregation paths (left-to-right, top-left, top, top-right, right-to-left), the first minimum with
 * the uniqueness check, the sub-pixel parabola with C's truncating division, the left-right check (bound 1, the right
 * view's winner being the least cost, ties to the larger column), the 3x3 median (edges replicated), and
 * filterSpeckles (4-connected components whose neighbours differ by at most 256; components of at most 100 pixels
 * become invalid).  Columns [0, D) are invalid.  With these parameters no path cost or sum reaches int16 saturation
 * (a path cost is at most 9 x 567 + 288 and S at most five of them), so the sums are exact in any order.
 * reverse[n] != 0 matches frame n as the script's right view: both views mirrored around the matcher, the map
 * mirrored back (by indexing; nothing is copied).
 * Fusion (per pixel, over the twelve maps in the script's order: blockSize 1, 2, 3, each numDisparities 64 .. 160):
 *   disp = map / 16 (fp32), depth = fp32(fp32(K[0][0] 0.1f) / fp32(disp + 1e-7f)) * (disp > 0) in fp32 (-0.0 where
 *   the quotient is negative); the lookup view (uint8 / 255 in fp32) warped by depth and scored against the base view
 *   exactly as wmd_loss_kitti.h's warp(D) and reproj (fp64, rounded to fp32 per pixel); best = torch.argmin over the
 *   twelve (the first NaN, else the first minimum); depth_out = that map's depth.
 * Bits depend only on the inputs and the shapes, never on timing, the batch or the device's SM count.
 */
#ifndef WMD_HINTS_H
#define WMD_HINTS_H

#include "wmd.h"

#ifdef __cplusplus
extern "C" {
#endif

#define WMD_HINTS_MATCHERS 12

/* Host-only: workspace bytes of wmd_sgbm_u8; 0 for a configuration or shape it refuses. */
size_t wmd_sgbm_ws_bytes(int32_t N, int32_t H, int32_t W, int32_t num_disparities, int32_t block_size);
/* left, right (N, H, W, 3) uint8; reverse (N) uint8 or NULL (every frame a left view); disp (N, H, W) int16.
 * WMD_ERR_ARG for a null pointer; WMD_ERR_SHAPE for num_disparities outside {64, 96, 128, 160}, block_size outside
 * {1, 2, 3}, a width OpenCV refuses (W - num_disparities <= block_size / 2), H < 1, H or W above 32767, or a batch whose
 * pixels or workspace cannot be addressed; WMD_ERR_WORKSPACE for a short workspace; all before any CUDA call.  N = 0
 * does nothing. */
int wmd_sgbm_u8(const uint8_t* left, const uint8_t* right, const uint8_t* reverse, int32_t N, int32_t H, int32_t W,
                int32_t num_disparities, int32_t block_size, void* ws, size_t ws_bytes, int16_t* disp,
                wmd_stream_t stream);

/* Host-only: workspace bytes of wmd_depth_hints_f32; 0 for a shape it refuses. */
size_t wmd_depth_hints_ws_bytes(int32_t N, int32_t H, int32_t W);
/* base, lookup (N, H, W, 3) uint8; disp (WMD_HINTS_MATCHERS, N, H, W) int16 in the script's matcher order; K, inv_K, T
 * (N, 4, 4) fp32 (T the stereo transform, T[0][3] = -0.1 for a left view, +0.1 for a right one); depth (N, 1, H, W)
 * fp32; index (N, 1, H, W) int32 or NULL.  The same argument checks as wmd_sgbm_u8 (H and W of at least 2). */
int wmd_depth_hints_f32(const uint8_t* base, const uint8_t* lookup, const int16_t* disp, const float* K,
                        const float* inv_K, const float* T, int32_t N, int32_t H, int32_t W, void* ws, size_t ws_bytes,
                        float* depth, int32_t* index, wmd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* WMD_HINTS_H */
