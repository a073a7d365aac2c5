/*
 * wmd_eval.h - KITTI depth evaluation entry points of libwmd.so (KITTI/evaluate_depth.py on the device).
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

#ifdef __cplusplus
}
#endif
#endif /* WMD_EVAL_H */
