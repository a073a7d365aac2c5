/*
 * wmd_loss_kitti.h - KITTI's stereo depth-hints training loss of libwmd.so, forward and backward, on the device.
 *
 * Same conventions as wmd.h and wmd_loss.h (device pointers unless the name says host, caller-owned buffers,
 * asynchronous on `stream`, no host sync, wmd_status return codes).  A header of its own, beside wmd_loss.h: it scores
 * decoder output with a different set of inputs (images, intrinsics, the stereo transform and the depth hints).  The
 * Python binding is _lib.KITTI_LOSS_SIGNATURES.
 *
 * The objective is KITTI/trainer.py's generate_images_pred + compute_losses_hints with --use_depth_hints --frame_ids 0
 * --use_stereo: the stereo pair is the only source frame, automasking and SSIM are on, v1_multiscale and
 * avg_reprojection are off.  oracle/kitti_loss.py restates it in numpy, expression for expression.
 * Inputs (fp32): target = color(0, 0) and source = color("s", 0) (N, 3, H, W); K, inv_K, stereo_T (N, 4, 4);
 * depth_hint, depth_hint_mask, and per loss scale s the noise (N, 1, H, W); disp and color(0, s) (N, 1|3, H >> s, W >> s).
 * H and W are multiples of 8.  Evaluation, every step in fp64 from the fp32 inputs unless marked fp32:
 *   warp(D): P = K stereo_T (each element summed over k = 0..3 in order); a = P[:3, :3] inv_K[:3, :3] (x, y, 1);
 *     q = D a + P[:, 3]; u = q0 / (q2 + 1e-7); ix = (((u / (W - 1) - 0.5) 2 + 1) W - 1) / 2 (iy alike); then torch's
 *     grid_sampler_2d bilinear sample with border padding (clamp to [0, W - 1], taps past the edge read 0), rounded
 *     to fp32 (the warped colour, an output).  A NaN coordinate gives NaN.
 *   reproj(p, t) per pixel: SSIM over reflection-padded 3x3 windows (row sums, then the three rows, / 9; C1 = 0.01^2,
 *     C2 = 0.03^2; clamp((1 - n / d) / 2, 0, 1), a NaN kept), 0.85 mean_c SSIM + 0.15 mean_c |t - p|, rounded to fp32.
 *   once: chint = warp(depth_hint) (color_depth_hint); id = reproj(source, target); hl = fp32(reproj(chint, target) +
 *     fp32(1000 fp32(1 - depth_hint_mask))).
 *   per loss scale: up = torch's align_corners=False bilinear upsample of disp (src = max((d + 0.5) in / out - 0.5, 0);
 *     exact at these factors); D = 1 / (1 / max_depth + (1 / min_depth - 1 / max_depth) up); r = reproj(warp(D),
 *     target); ids = fp32(id + fp32(noise 1e-5f)); k = argmin(r, ids, hl): the first NaN, else the first minimum
 *     (torch.argmin); rm = k != 1, hm = k == 2; identity_selection = 1 - rm, depth_hint_pixels = hm (fp32 maps);
 *     reproj_loss = fp32(sum r rm / (sum rm + 1e-7)); depth_hint_loss = fp32(sum log(|D - hint| + 1) mask hm /
 *     (sum hm + 1e-7)); smooth = get_smooth_loss(disp / (mean + 1e-7), color(0, s)) (gamma 2) in fp64;
 *     loss/s = fp32(reproj_loss + depth_hint_loss + disparity_smoothness smooth / 2^s).
 *   loss = fp32(sum over loss scales ascending of loss/s / n_scales).
 *   Sums: fp64, per CTA of WMD_LOSS_PIXELS_PER_CTA pixels a fixed per-thread order and tree, the partials in CTA order.
 * terms (1 + 3 n_loss fp32): loss, then per loss scale reproj_loss, depth_hint_loss, loss/s.
 * Backward: grads[i] = d(sum_k grad_terms[k] terms[k]) / d disp_i, in gather form: the SSIM coefficients of every
 * centre (the clamp passes on [0, 1] inclusive, NaN gives 0), a gather over the reflected windows that read each warped
 * pixel, sign(p - t) with sign(0) = 0, the sample's derivative in its coordinates (0 where the clamp is active or the
 * coordinate lies on the border, as torch's clip_coordinates_set_grad), the projection's closed-form derivative in D,
 * the hint term, d D / d up, then per low-resolution pixel its upsample footprint plus the smoothness gradient with the
 * per-frame mean's term.  All fp64, rounded once.  The masks and every input but disp are constants.
 * Bits depend only on the inputs and the shapes, never on timing or the device's SM count.
 */
#ifndef WMD_LOSS_KITTI_H
#define WMD_LOSS_KITTI_H

#include "wmd_loss.h"

#ifdef __cplusplus
extern "C" {
#endif

/* KITTI depth-hints loss: one call's inputs; the loss scales ascending, at most 4 */
typedef struct wmd_loss_kitti_desc {
  int32_t N, H, W;
  const float *target, *source;           /* (N, 3, H, W) */
  const float *K, *inv_K, *stereo_T;      /* (N, 4, 4) */
  const float *depth_hint, *depth_hint_mask;  /* (N, 1, H, W) */
  int32_t n_scales;                       /* len(scales): the total's divisor, n_loss .. 4 */
  int32_t n_loss;                         /* 1 .. 4 */
  int32_t scale[4];                       /* 0 .. 3, ascending */
  const float* disp[4];                   /* (N, 1, H >> s, W >> s) */
  const float* color[4];                  /* (N, 3, H >> s, W >> s): color(0, s) */
  const float* noise[4];                  /* (N, 1, H, W) */
  double min_depth, max_depth, disparity_smoothness;
} wmd_loss_kitti_desc;

/* Host-only: bytes of the forward's state (partials, counts, means, static maps), which the backward reads; 0 for a bad
 * descriptor. */
size_t wmd_loss_kitti_ws_bytes(const wmd_loss_kitti_desc* d);
/* Host-only: bytes of the backward's scratch; 0 for a bad descriptor. */
size_t wmd_loss_kitti_bwd_ws_bytes(const wmd_loss_kitti_desc* d);
/* color_depth_hint (N, 3, H, W); warped (n_loss, N, 3, H, W); idsel, hpix (n_loss, N, 1, H, W); terms (1 + 3 n_loss).
 * WMD_ERR_ARG for a null pointer or a depth range outside 0 < min_depth < max_depth, WMD_ERR_SHAPE for sizes outside
 * the contract, WMD_ERR_WORKSPACE for a short workspace, all before any CUDA call.  With N = 0 only d, ws and terms are
 * read. */
int wmd_loss_kitti_fwd(const wmd_loss_kitti_desc* d, float* color_depth_hint, float* warped, float* idsel, float* hpix,
                       void* ws, size_t ws_bytes, float* terms, wmd_stream_t stream);
/* The forward's warped, idsel, hpix and state fwd_ws; grad_terms (1 + 3 n_loss) fp32 on the device; grads: HOST array
 * of n_loss device pointers, grads[i] (N, 1, H >> s_i, W >> s_i).  The same argument checks as the forward. */
int wmd_loss_kitti_bwd(const wmd_loss_kitti_desc* d, const float* warped, const float* idsel, const float* hpix,
                       const void* fwd_ws, const float* grad_terms, void* ws, size_t ws_bytes, float* const* grads,
                       wmd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* WMD_LOSS_KITTI_H */
