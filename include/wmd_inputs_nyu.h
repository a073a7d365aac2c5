/*
 * wmd_inputs_nyu.h - NYUv2's training inputs of libwmd.so on the device: the flip, channel swap, gamma, crop, Pillow
 * resize and ToTensor of NYUv2/data.py's getDefaultTrainTransform / getNoTransform, bit for bit, over a batch.
 *
 * Same conventions as wmd.h (device pointers, caller-owned buffers, asynchronous on `stream`, no host sync, no
 * allocation, wmd_status return codes).  The Python binding is _lib.NYU_INPUTS_SIGNATURES.
 *
 * Per item (oracle/nyu_inputs.py restates every step), from a decoded (480, 640, 3) RGB image and (480, 640) L depth:
 *   1. flip != 0 mirrors the image and the depth over the full 640 columns;
 *   2. output channel c of the image is input channel perm[c];
 *   3. every image byte v becomes lut[v] (torchvision's adjust_gamma, Pillow's point; the caller builds the 256-entry
 *      table on the host with libm's pow, an identity table when there is no gamma);
 *   4. both are cropped to columns 16 .. 623 and rows 16 .. 463 (608 x 448);
 *   5. both are resized with Pillow's 8-bit two-pass resample: horizontal first, uint8 between the passes; each value
 *      is clip((1 << 21 + sum_t tab[t] * in[first + t]) >> 22, 0, 255).  A table row is (first, taps, k coefficients),
 *      k the table's row stride less two, with `first` in uncropped, flipped coordinates (the crop offset is in the
 *      table).  Pillow's BICUBIC tables are the 22-bit rounded normalised weights; NEAREST is a one-tap table whose
 *      coefficient is 1 << 22.  Reads are clamped to the crop window, whatever the table says;
 *   6. ToTensor: image[c] = u / 255 in fp32 (correctly rounded); depth = clamp((u / 255) * 1000, 10, 1000) in fp32,
 *      each operation rounded on its own (no contraction).
 * Two launches per call: the horizontal pass of the image and the depth together (flip, swap and LUT applied to each
 * source byte), then the vertical pass with the fp32 epilogue.  Integer-only up to the epilogue, so the bits depend
 * only on the item and its draws, never on the batch, timing or the device's SM count.
 */
#ifndef WMD_INPUTS_NYU_H
#define WMD_INPUTS_NYU_H

#include "wmd.h"

#ifdef __cplusplus
extern "C" {
#endif

#define WMD_NYU_SRC_H 480
#define WMD_NYU_SRC_W 640
#define WMD_NYU_CROP 16

/* One item's draws (device memory, 16 bytes). */
typedef struct wmd_nyu_inputs_item {
  int32_t flip;    /* != 0: FLIP_LEFT_RIGHT of the image and the depth */
  int32_t perm[3]; /* output channel c is input channel perm[c], each in 0 .. 2 */
} wmd_nyu_inputs_item;

typedef struct wmd_nyu_inputs_desc {
  int32_t N;                     /* items */
  int32_t image_h, image_w;      /* the image's output extent */
  int32_t depth_h, depth_w;      /* the depth's output extent */
  int32_t image_xk, image_yk;    /* coefficients per row of the image's tables */
  int32_t depth_xk, depth_yk;    /* coefficients per row of the depth's tables */
  const uint8_t* image_src;      /* (N, 480, 640, 3) RGB */
  const uint8_t* depth_src;      /* (N, 480, 640) L */
  const wmd_nyu_inputs_item* items; /* (N) */
  const uint8_t* lut;            /* (N, 256) */
  const int32_t* image_xtab;     /* (image_w, 2 + image_xk): 608 -> image_w, first offset by 16 */
  const int32_t* image_ytab;     /* (image_h, 2 + image_yk): 448 -> image_h, first offset by 16 */
  const int32_t* depth_xtab;     /* (depth_w, 2 + depth_xk) */
  const int32_t* depth_ytab;     /* (depth_h, 2 + depth_yk) */
  float* image;                  /* (N, 3, image_h, image_w) */
  float* depth;                  /* (N, 1, depth_h, depth_w) */
} wmd_nyu_inputs_desc;

/* Host-only: workspace bytes of wmd_nyu_inputs_u8; 0 for a descriptor it refuses on shape. */
size_t wmd_nyu_inputs_ws_bytes(const wmd_nyu_inputs_desc* d);
/* WMD_ERR_ARG for a null descriptor or a null pointer, or k < 1; WMD_ERR_SHAPE for N outside [0, 65535], an output
 * extent outside [1, 32767], or a buffer of more than 2^31 values; WMD_ERR_WORKSPACE for a short workspace; all before
 * any CUDA call.  N = 0 does nothing. */
int wmd_nyu_inputs_u8(const wmd_nyu_inputs_desc* d, void* ws, size_t ws_bytes, wmd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* WMD_INPUTS_NYU_H */
