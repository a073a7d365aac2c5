/*
 * wmd_inputs.h - KITTI's training inputs of libwmd.so on the device: the flip, Pillow's LANCZOS pyramid, torchvision's
 * ColorJitter and ToTensor of KITTI/datasets/mono_dataset.py, bit for bit, over a batch of decoded views of mixed sizes.
 *
 * Same conventions as wmd.h (device pointers, caller-owned buffers, asynchronous on `stream`, no host sync, no
 * allocation, wmd_status return codes).  A header of its own: it prepares training data rather than running a network.
 * The Python binding is _lib.INPUTS_SIGNATURES.
 *
 * Per view (oracle/kitti_inputs.py restates every step):
 *   Stage j = 0 .. n_scales - 1 resamples stage j - 1's output (stage 0: the source view, mirrored when flip is set)
 *   to (out_h[j], out_w[j]) with Pillow's 8-bit two-pass resample: horizontal first, then vertical, uint8 between;
 *   each output value is clip((1 << 21 + sum_t tab[t] * in[first + t]) >> 22, 0, 255).  The tables are Pillow's
 *   22-bit fixed-point LANCZOS coefficients, which the caller computes on the host (they need libm's sin); a row of a
 *   table is (first tap, taps, k coefficients), k the table's row stride less two.  The kernels are integer-only.
 *   Each stage's image is then written twice as (3, out_h, out_w) fp32 uint8 / 255 (correctly rounded): plain to
 *   color[j] and, after the view's jitter, to color_aug[j].  The jitter applies order[0..3] in turn:
 *     0 brightness  Image.blend(black, img, factor[0])
 *     1 contrast    Image.blend(int(mean(L) + 0.5), img, factor[1]), the mean over this stage's image as it is at
 *                   that point of the order (an exact integer sum, divided in double)
 *     2 saturation  Image.blend(L(img), img, factor[2])
 *     3 hue         Pillow's RGB -> HSV, hue byte + hue_shift modulo 256, HSV -> RGB
 *   with blend(a, b, alpha) = clip(trunc(a + alpha (b - a)), 0, 255) in fp32 without contraction, and
 *   L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16.  order[0] < 0: no jitter, color_aug[j] = color[j].
 * Bits depend only on the inputs, never on the batch, timing or the device's SM count.
 */
#ifndef WMD_INPUTS_H
#define WMD_INPUTS_H

#include "wmd.h"

#ifdef __cplusplus
extern "C" {
#endif

#define WMD_INPUTS_MAX_SCALES 4

/* One source view of stage 0 (device memory, 40 bytes). */
typedef struct wmd_inputs_view {
  const int32_t* xtab; /* (out_w[0], 2 + xk): the horizontal table for w -> out_w[0] */
  const int32_t* ytab; /* (out_h[0], 2 + yk): the vertical table for h -> out_h[0] */
  int32_t h, w;        /* the decoded extent, within the padded (src_h, src_w) */
  int32_t xk, yk;
  int32_t flip;        /* != 0: FLIP_LEFT_RIGHT before the resample */
  int32_t pad;
} wmd_inputs_view;

/* One view's colour jitter (device memory, 32 bytes). */
typedef struct wmd_inputs_jitter {
  int32_t order[4];  /* op at each position: 0 brightness, 1 contrast, 2 saturation, 3 hue; order[0] < 0: none */
  float factor[3];   /* fp32 blend factors of brightness, contrast, saturation */
  int32_t hue_shift; /* 0 .. 255, added to the HSV hue byte */
} wmd_inputs_jitter;

typedef struct wmd_inputs_desc {
  int32_t N;                   /* views */
  int32_t src_h, src_w;        /* src is (N, src_h, src_w, 3) uint8, each view at its top-left */
  int32_t n_scales;            /* 1 .. WMD_INPUTS_MAX_SCALES stages */
  int32_t out_h[WMD_INPUTS_MAX_SCALES], out_w[WMD_INPUTS_MAX_SCALES];
  const uint8_t* src;
  const wmd_inputs_view* views;                         /* (N): stage 0's per-view sizes, flips and tables */
  const int32_t* xtab[WMD_INPUTS_MAX_SCALES];           /* stage j >= 1: out_w[j - 1] -> out_w[j], (out_w[j], 2 + xk[j]) */
  const int32_t* ytab[WMD_INPUTS_MAX_SCALES];           /* stage j >= 1: out_h[j - 1] -> out_h[j], (out_h[j], 2 + yk[j]) */
  int32_t xk[WMD_INPUTS_MAX_SCALES], yk[WMD_INPUTS_MAX_SCALES];
  const wmd_inputs_jitter* jitter;                      /* (N) */
  float* color[WMD_INPUTS_MAX_SCALES];                  /* (N, 3, out_h[j], out_w[j]) */
  float* color_aug[WMD_INPUTS_MAX_SCALES];
} wmd_inputs_desc;

/* Host-only: workspace bytes of wmd_inputs_u8; 0 for a descriptor it refuses. */
size_t wmd_inputs_ws_bytes(const wmd_inputs_desc* d);
/* WMD_ERR_ARG for a null descriptor or a null pointer the shape needs, or k < 1; WMD_ERR_SHAPE for N outside
 * [0, 65535], n_scales outside [1, 4], an extent outside [1, 32767], or a stage of more than 2^31 values; WMD_ERR_WORKSPACE
 * for a short workspace; all before any CUDA call.  N = 0 does nothing.  Per-view sizes in `views` are device data the
 * caller keeps within the padded extent; reads are clamped to the view regardless. */
int wmd_inputs_u8(const wmd_inputs_desc* d, void* ws, size_t ws_bytes, wmd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* WMD_INPUTS_H */
