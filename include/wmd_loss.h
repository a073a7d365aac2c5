/*
 * wmd_loss.h - training-loss entry points of libwmd.so: NYUv2's supervised objective (NYUv2/train.py:279-327), forward
 * and backward, on the device.
 *
 * Same conventions as wmd.h (device pointers unless the name says host, caller-owned buffers, asynchronous on
 * `stream`, no host sync, wmd_status return codes).  Kept apart from wmd.h: these kernels score decoder output, they
 * are not part of the decoder path whose every launch tests/launch_check.py checks.  The Python binding is
 * _lib.LOSS_SIGNATURES.
 *
 * One call scores up to WMD_LOSS_MAX_TERMS predictions against one target t (N, 1, H, W) fp32.  Term k is pred_k
 * (N, 1, h, w) fp32 with h << log2_factor == H, w << log2_factor == W, 0 <= log2_factor <= 3, upsampled to (H, W) by
 * torch's bilinear, align_corners=True rule, per axis (in -> out, destination index d):
 *   r = fp32(in - 1) / fp32(out - 1) in fp32, or 0 when out == 1;  src = fp32(r d);  i0 = min(int(src), in - 1);
 *   i1 = i0 + (i0 < in - 1);  l1 = fp32(src - i0) clamped to [0, 1];  l0 = 1 - l1 EXACTLY, in fp64 (torch rounds it to
 *   fp32);
 * sample = l0y (l0x a + l1x b) + l1y (l0x c + l1x d) in fp64 from the fp32 taps (a, b on row i0y; c, d on row i1y;
 * columns i0x, i1x), every tap read and multiplied, zero weights included, so a NaN spreads where it spreads in torch.
 * Factor 1 is the identity (sample = pred: no neighbour is read), as torch's interpolate is at equal sizes.  The
 * weights are multiples of 2^-27 at these factors, so l0 + l1 == 1 and the map of a constant is that constant.
 *
 * Forward:  means[k] = fp32( sum |sample - t| / (N H W) ), the sum in fp64 in a fixed order (a fixed grid of CTAs of
 *           WMD_LOSS_PIXELS_PER_CTA target pixels, a fixed tree in each, the CTA partials added in CTA order; no
 *           atomics).  N = 0 gives NaN.  signs (nullable): (n_terms, N, H, W) int8 sgn(sample - t) of the fp64
 *           difference, 0 on an exact tie and on NaN, kept for the backward.
 * Backward: grads[k] (N, 1, h, w) fp32 = fp32( (g_k / (N H W)) S ), g_k = grad_means[k] read on the device, and
 *           S = sum over the target pixels (Y, X) that read pixel (y, x) of signs[k] wy(Y) wx(X), the weight of the
 *           tap (l0 at i0, l1 at i1, both when i0 == i1).  Gather form, one thread per low-resolution pixel: the
 *           footprint comes from the forward rule evaluated over a candidate range, and S = sum over Y ascending of
 *           wy(Y) (sum over X ascending of signs wx(X)), the inner sums exact, the outer one in fp64.  No atomics.
 * Bits depend only on the inputs and the shapes, never on timing or the device's SM count.
 */
#ifndef WMD_LOSS_H
#define WMD_LOSS_H

#include "wmd.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { WMD_LOSS_MAX_TERMS = 4, WMD_LOSS_PIXELS_PER_CTA = 2048 };

/* one prediction scored against the call's target */
typedef struct wmd_loss_term {
  const float* pred;    /* (N, 1, h, w) */
  int32_t h, w;
  int32_t log2_factor;  /* 0 .. 3: H = h << log2_factor, W = w << log2_factor */
} wmd_loss_term;

/* Host-only: workspace bytes of wmd_loss_nyu_fwd (the fp64 CTA partials); 0 for a bad shape. */
size_t wmd_loss_nyu_ws_bytes(int N, int H, int W, int n_terms);
/* terms: HOST array of n_terms (1 .. WMD_LOSS_MAX_TERMS) descriptors.  Returns WMD_ERR_ARG for a null pointer,
 * WMD_ERR_SHAPE for sizes that do not fit the contract above (or N H W >= 2^31), WMD_ERR_WORKSPACE for a short
 * workspace, all before any CUDA call.  With N = 0, target, pred and ws may be null. */
int wmd_loss_nyu_fwd(const float* target, int N, int H, int W, const wmd_loss_term* terms, int n_terms, int8_t* signs,
                     void* ws, size_t ws_bytes, float* means, wmd_stream_t stream);
/* signs: the forward's (n_terms, N, H, W); grad_means (n_terms) fp32; grads: HOST array of n_terms device pointers,
 * grads[k] (N, 1, h, w).  The same argument checks as the forward. */
int wmd_loss_nyu_bwd(const int8_t* signs, int N, int H, int W, const wmd_loss_term* terms, int n_terms,
                     const float* grad_means, float* const* grads, wmd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* WMD_LOSS_H */
