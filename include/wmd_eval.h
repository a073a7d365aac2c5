/*
 * wmd_eval.h - depth evaluation entry points of libwmd.so: KITTI (KITTI/evaluate_depth.py) and NYUv2
 * (NYUv2/utils.py: add_results, evaluate, compute_errors_nyu) on the device.
 *
 * Same conventions as wmd.h (device pointers, caller-owned buffers, asynchronous on `stream`, no host sync, wmd_status
 * return codes).  Kept apart from wmd.h: these kernels score decoder output, they are not part of the decoder path
 * whose every launch tests/launch_check.py checks.  The Python binding is _lib.EVAL_SIGNATURES.
 */
#ifndef WMD_EVAL_H
#define WMD_EVAL_H

#include "wmd.h"

#ifdef __cplusplus
extern "C" {
#endif
/* ---------------------------------------------------------------- KITTI depth evaluation (KITTI/evaluate_depth.py)
 * A ground-truth split is gt (N, Hmax, Wmax) fp32, zero padded, with hw (N, 2) int32 each frame's own (H, W).
 *
 * Valid pixels (evaluate_depth.py:283-293), mask (N, Hmax, Wmax) bytes; nothing outside a frame's own H x W is valid:
 *   WMD_EVAL_EIGEN:        1e-3 < gt < 80 compared in float32 (numpy 2 compares a float32 array with a Python float in
 *                          float32), inside the crop [int32(0.40810811 H), int32(0.99189189 H)) x [int32(0.03594771 W),
 *                          int32(0.96405229 W)) with the products in float64
 *   WMD_EVAL_GT_POSITIVE:  gt > 0 (every other split)
 * wmd_compact_mask on the mask gives the pixel list and per-frame offsets; wmd_eval_gather_f32 then gathers
 * out[i] = src[pixels[i]] for i < min(*count, max_rows) (the valid ground truth, once per split). */
enum { WMD_EVAL_EIGEN = 0, WMD_EVAL_GT_POSITIVE = 1 };
int wmd_eval_gt_mask(const float* gt, const int32_t* hw, uint8_t* mask, int N, int Hmax, int Wmax, int split,
                     wmd_stream_t stream);
int wmd_eval_gather_f32(const float* src, const int32_t* pixels, const int32_t* count, int max_rows, float* out,
                        wmd_stream_t stream);
/* evaluate_depth.py:276-307 for frames f = frame0 .. frame0 + n - 1 of a split, one CTA per frame.  disp (n, h, w) fp32
 * (disp_f64 = 0) or fp64 is frame f's predicted disparity, h <= H and w <= W of every frame.  At each valid pixel
 * (pixels / offsets of the split, gt the gathered valid values) it is sampled by cv2.resize's INTER_LINEAR rule in fp64
 * (per axis f = (d + 0.5) src / dst - 0.5, s = floor(f), weight f - s; s < 0: s = 0, weight 0; s >= src - 1: s = src - 1,
 * weight 0; horizontal pass - the last column one tap - then vertical), and depth = (1 / disp) * scale_factor.  With
 * median_scaling, ratio = median(gt) / median(depth) (np.median: exact, by radix select; the ground truth's two middle
 * values average in float32; NaN for a NaN or no value) and depth *= ratio, else ratio = 1.  depth is clamped to
 * [1e-3, 80] by comparisons (NaN stays NaN) and compute_errors (:50-68) is summed in fp64 in a fixed order:
 *   errors (n, 7) = abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3;  ratio (n);  count (n) valid pixels.
 * gt_log (per valid pixel, nullable): log(gt) as the caller rounds it (the reference takes numpy's float32 log of the
 * float32 ground truth); NULL = fp64 log.  depth: fp64 workspace of offsets[frame0 + n] values.  Bits do not depend
 * on n, frame0 or timing. */
int wmd_eval_frames(const void* disp, int disp_f64, int n, int h, int w, int frame0, const int32_t* hw,
                    const int32_t* pixels, const int32_t* offsets, const float* gt, const float* gt_log, int Hmax,
                    int Wmax, double scale_factor, int median_scaling, double* depth, double* errors, double* ratio,
                    int32_t* count, wmd_stream_t stream);
/* compute_errors (evaluate_depth.py:50-68) of n fp64 pairs, the same sums in one CTA -> errors[7] */
int wmd_eval_errors_f64(const double* gt, const double* pred, int n, double* errors, wmd_stream_t stream);
/* batch_post_process_disparity (evaluate_depth.py:71-79): l_disp, r_disp (N, h, w), both fp32 (in_f64 = 0) or fp64
 * -> out fp64, with linspace(0, 1, w) as numpy forms it and m_disp = 0.5 (l + r) in the inputs' precision. */
int wmd_post_process_disparity(const void* l_disp, const void* r_disp, int in_f64, double* out, int N, int h, int w,
                               wmd_stream_t stream);

/* ---------------------------------------------------------------- NYUv2 depth evaluation (NYUv2/utils.py)
 * evaluate() / add_results() (:183-335) for n frames.  disp (n, h, w) fp32 is the decoder's ("disp", 0).  Per frame,
 * in fp64 from the fp32 values:
 *   1. p = disp / 100, or with use_disparity DepthNorm(disp, 1000) / 10000 as torch evaluates it:
 *      (reciprocal(disp) * 1000) / 10000;
 *   WMD_EVAL_NYU_EIGEN (any h x w):
 *   2. bilinear, align_corners=True, to (224, 304);  3. ReplicationPad2d(8) to (240, 320);
 *   4. bilinear, align_corners=True, to (480, 640) (scale_factor 2 plays no part: the scale is (in - 1) / (out - 1));
 *   5. clamp to [0.4, 10];  6. crop rows 20..459, columns 24..615 -> (440, 592);
 *   WMD_EVAL_NYU_224 (h = w = 224): steps 1 and 5 only -> (224, 224).
 * Each resize is torch's formula and order, h0 * (w0 * x00 + w1 * x01) + h1 * (w0 * x10 + w1 * x11), with
 * src = scale * d, lambda = src - (int)src, w0 = 1 - lambda and the second tap at i0 + (i0 < in - 1), all with
 * explicit _rn operations.  Taps with zero weight are still read and multiplied, as torch does, so a NaN or +-Inf
 * disparity spreads NaN to outputs that give it zero weight; the clamp compares, so NaN stays NaN.
 * gt, gt_log10: (n, 440, 592) or (n, 224, 224) fp32, the ground truth as the metrics see it (the Eigen crop, or the
 * border-cropped 224 x 224 resize) and its float32 log10 (the reference takes torch.log10 of the float32 values).
 * compute_errors_nyu (:85-98) with y = gt, x = the prediction, summed per frame in fp64 in a fixed order (a fixed grid
 * of CTAs per frame, a fixed tree in each, the slabs added in order; no atomics):
 *   sums (n, 7) = sum |y - x| / y, sum (y - x)^2, sum |log10 y - log10 x| (log10 x in fp64), the counts of
 *   max(y / x, x / y) < 1.25, 1.25^2, 1.25^3 (NaN-propagating max), and the pixel count.
 * No pixel is masked.  depth_out (nullable): the fp64 prediction map, the reference's `predictions`.  ws: at least
 * wmd_eval_nyu_ws_bytes(n, mode) bytes (0 for a bad mode or n < 0).  Bits do not depend on n or timing. */
enum { WMD_EVAL_NYU_EIGEN = 0, WMD_EVAL_NYU_224 = 1, WMD_EVAL_NYU_CROP_H = 440, WMD_EVAL_NYU_CROP_W = 592 };
size_t wmd_eval_nyu_ws_bytes(int n, int mode);
int wmd_eval_nyu_frames(const float* disp, int n, int h, int w, int mode, int use_disparity, const float* gt,
                        const float* gt_log10, double* depth_out, void* ws, size_t ws_bytes, double* sums,
                        wmd_stream_t stream);
/* compute_errors_nyu (:85-98) of n fp64 pairs, log10 y in fp64 too: the same sums, pooled over a fixed grid of CTAs
 * of 4096 pixels each and added in CTA order -> errors[6] = rel, rms, log_10, a1, a2, a3.  ws: at least
 * wmd_eval_nyu_errors_ws_bytes(n) bytes. */
size_t wmd_eval_nyu_errors_ws_bytes(long long n);
int wmd_eval_nyu_errors_f64(const double* pred, const double* gt, long long n, void* ws, size_t ws_bytes,
                            double* errors, wmd_stream_t stream);

/* ---------------------------------------------------------------- NYUv2 depth boundary error (NYUv2/utils.py:122-169)
 * compute_depth_boundary_error for n frames of any h x w (h, w >= 1, n h w < 2^31).  pred (n, h, w) is fp32
 * (pred_f64 = 0) or fp64, which is rounded to fp32 first (the reference's pred.astype('f')).  Per frame:
 *   1. p = pred with zeros as NaN, p = (p - nanmin p) / fl(nanmax p - nanmin p), both operations in fp32;
 *   2. scikit-image 0.16.2's canny(p, sigma sqrt(2)) with thresholds `low`, `high`:
 *      sm = the 13-tap gaussian `taps` (w0 .. w6, scipy's weights) in scipy's order, mode constant 0, along axis 0 and
 *      then axis 1, each pass accumulated in fp64 as t = x w0, t += (x[-j] + x[+j]) wj for j = 6 .. 1 and stored in
 *      fp32; smoothed = sm / (bleed + DBL_EPSILON) in fp64, `bleed` (h, w) fp64 the same gaussian of ones (scipy's);
 *      isobel, jsobel = ndi.sobel(smoothed, 0 / 1) (reflect): d = 0 s + (s[+1] - s[-1]) along the axis, then
 *      2 d + (d[-1] + d[+1]) along the other; magnitude = glibc's non-FMA hypot kernel; local maxima of the interior
 *      pixels with magnitude > 0 by skimage's four octants in its order (a later octant's assignment stands), each
 *      side c2 w + c1 (1 - w) <= m; low / high = local maxima with magnitude >= low / high; edges_est = the
 *      8-connected components of low that hold a high pixel (union-find: the result is a set, timing-independent);
 *   3. d_est = the exact Euclidean distance of each pixel to the nearest edges_est pixel (scipy's
 *      distance_transform_edt(1 - edges_est)), sqrt of the integer squared distance; with no edge pixel at all,
 *      scipy's sqrt((y + 1)^2 + x^2);
 *   4. with edges_gt (n, h, w) fp32, d_gt (n, h, w) fp64 its distance map (wmd_eval_edt of edges_gt == 1) and
 *      gt_sums (n, 2) fp64 = (np.sum(edges_gt), np.nansum(edges_gt)) as numpy's float32 sums: near = edges_est &
 *      (d_gt < 10);  scores (n, 2) = NaN, NaN if gt_sums[0] == 0;  10, 10 if near is empty;  else
 *      acc = sum_near d_gt / |near|,  comp = (sum_est min(d_gt, 10) + nansum min(d_est edges_gt, 10)) /
 *      (|edges_est| + gt_sums[1]), each sum in fp64 over a fixed grid of CTAs and a fixed tree, without atomics.
 * edges_est (n, h, w) bytes 0 / 1, d_est (n, h, w) fp64.  ws: at least wmd_eval_edges_ws_bytes(n, h, w) bytes (0 for
 * a bad shape).  Bits do not depend on n or timing. */
size_t wmd_eval_edges_ws_bytes(int n, int h, int w);
int wmd_eval_edges_frames(const void* pred, int pred_f64, int n, int h, int w, const double* taps,
                          const double* bleed, double low, double high, const float* edges_gt, const double* d_gt,
                          const double* gt_sums, uint8_t* edges_est, double* d_est, double* scores, void* ws,
                          size_t ws_bytes, wmd_stream_t stream);
/* the exact Euclidean distance transform of n (h, w) feature masks (bytes, non-zero = feature): dist (n, h, w) fp64
 * as in step 3 above.  ws: at least wmd_eval_edt_ws_bytes(n, h, w) bytes. */
size_t wmd_eval_edt_ws_bytes(int n, int h, int w);
int wmd_eval_edt(const uint8_t* features, int n, int h, int w, double* dist, void* ws, size_t ws_bytes,
                 wmd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* WMD_EVAL_H */
