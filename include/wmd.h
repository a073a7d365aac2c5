/*
 * wmd.h - C ABI of libwmd.so: the H100 (sm_90a) wavelet-monodepth decoder hot path.
 *
 * The reference (nianticlabs/wavelet-monodepth) has no native/FFI layer: its
 * boundary for this path is a Python nn.Module / function API built on ATen ops
 * and the un-vendored pytorch_wavelets package.  Every entry point below names
 * the reference interface it replaces (paths relative to the reference tree).
 * The Python mirror of that API lives in wavelet_monodepth_b200/ and reaches
 * these symbols through ctypes with tensor.data_ptr() (INTEGRATION.md).
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is DEVICE memory unless the
 *    name says host; all tensors are contiguous fp32 / int32 / uint8;
 *  - the caller owns every buffer; nothing is allocated, freed or retained;
 *  - every call is asynchronous on `stream` (a cudaStream_t), re-entrant, and
 *    never synchronises the device; data-dependent counts stay on the device;
 *  - return value: WMD_OK (0) or a negative wmd_status; never throws / exits.
 *
 * Sparse feature layout ("rows"): active pixels of all samples are enumerated
 * in (n, y, x) row-major order - the reference's order (KITTI/layers.py:377-378,
 * 387) extended over the batch - and a feature tensor is a row-major matrix
 * [rows][ld] (pixel-major, channels contiguous), not the reference's
 * channel-major (C, M) vector (layers.py:358).  wmd_nchw_to_rows_f32 /
 * wmd_rows_to_nchw_f32 (with N=1, HW=M) convert at the functional-API boundary.
 */
#ifndef WMD_H
#define WMD_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WMD_VERSION 100 /* major*100 + minor */

typedef void* wmd_stream_t; /* cudaStream_t */

typedef enum wmd_status {
  WMD_OK = 0,
  WMD_ERR_ARG = -1,         /* null pointer / bad enum */
  WMD_ERR_SHAPE = -2,       /* unsupported size (odd extent, misaligned leading dim ...) */
  WMD_ERR_CUDA = -3,        /* a CUDA call failed; see wmd_last_cuda_error() */
  WMD_ERR_WORKSPACE = -4,   /* workspace too small */
  WMD_ERR_UNSUPPORTED = -5
} wmd_status;

enum { WMD_PAD_ZERO = 0, WMD_PAD_REFLECT = 1, WMD_PAD_REPLICATE = 2 };
enum { WMD_ACT_NONE = 0, WMD_ACT_ELU = 1, WMD_ACT_LRELU = 2, WMD_ACT_SIGMOID = 3 };

int wmd_version(void);
const char* wmd_status_string(int status);
/* last cudaError_t recorded by a failing call on this host thread (0 if none) */
int wmd_last_cuda_error(void);
/* number of kernels this library has launched on this host thread since load (bench.py's gpu_launches) */
long long wmd_launch_count(void);

/* ---------------------------------------------------------------- Haar transforms
 * Replaces pytorch_wavelets.DWTInverse.forward((yl,[yh])) for wave='haar', one level
 * (call sites KITTI/networks/decoders/depth_decoder.py:164,372,416;
 * NYUv2/networks/decoders/densedepth_decoder.py:129,137,145,309,357,404) and the
 * reference's closed form my_iwt_once (depth_decoder.py:225-239).
 *   ll (N,C,H,W), hf (N,C,3,H,W) [LH,HL,HH] -> out (N,C,2H,2W)
 *   out[2i+a,2j+b] = 1/2 (ll + (-1)^a lh + (-1)^b hl + (-1)^(a+b) hh), evaluated in
 *   the dependency's separable order (two 1/sqrt2 passes) so results are bit-equal to it.
 * Fused consumer (optional, disp may be NULL):
 *   disp  (N,C,2H,2W) = out * disp_scale, clamped to [0,1] if clamp01   (depth_decoder.py:166)
 * The clamp propagates NaN as torch.clamp does: a NaN reconstruction gives a NaN disparity, not 0.
 */
int wmd_idwt_haar_f32(const float* ll, const float* hf, float* out, float* disp, float disp_scale, int clamp01,
                      int N, int C, int H, int W, wmd_stream_t stream);

/* Fused IDWT + disparity epilogue + bilinear resize: full (N,C,full_h,full_w) = bilinear(disp) with
 * disp = [clamp01](idwt(ll,hf) * disp_scale), PyTorch F.interpolate(mode="bilinear") index arithmetic for either
 * align_corners setting.  Replaces the consumers of ("disp", s): KITTI/trainer.py:338-339 (align_corners=False),
 * NYUv2/utils.py:223-227, NYUv2/train.py:305-306 (align_corners=True).  The intermediate disp plane is not read
 * back from HBM.  Upsampling only, by about 1.6x per axis or more: with sy, sx = source / destination size per axis (the
 * disp plane is 2H x 2W), a 32 x 128 output tile's source patch must fit 2048 floats, (floor(32 sy) + 4) (floor(128 sx)
 * + 4) <= 2048; smaller factors (equal sizes, 1.5x) return WMD_ERR_UNSUPPORTED.  The clamp propagates NaN as
 * torch.clamp does, so a NaN disparity spreads into the outputs that read it. */
int wmd_idwt_bilinear_f32(const float* ll, const float* hf, float* full, float disp_scale, int clamp01, int full_h,
                          int full_w, int align_corners, int N, int C, int H, int W, wmd_stream_t stream);

/* Replaces one level of pytorch_wavelets.DWTForward.forward (NYUv2/train.py:258,289); also the
 * adjoint used for the IDWT's backward (KITTI/trainer.py:208-212 trains through inverse_wt).
 *   x (N,C,H,W), H and W even -> ll (N,C,H/2,W/2), hf (N,C,3,H/2,W/2) */
int wmd_dwt_haar_f32(const float* x, float* ll, float* hf, int N, int C, int H, int W, wmd_stream_t stream);

/* ---------------------------------------------------------------- threshold + masks
 * thresh[n] = (max(x_n) - min(x_n)) * ratio over per_sample contiguous floats of sample n.
 * Replaces `thresh = (yl.max() - yl.min()) * thresh_ratio` (depth_decoder.py:308;
 * densedepth_decoder.py:316,363), per sample instead of the reference's batch-1.
 * minmax (2N floats: min,max) is optional.  N <= 16384.  ws: wmd_range_ws_bytes() bytes whose first
 * 64 KiB (per-sample ticket counters) must be zero before the FIRST use only: the kernel leaves them
 * zeroed, for any later N, so one scratch buffer can be shared by all calls on a stream. */
size_t wmd_range_ws_bytes(int N, long long per_sample);
int wmd_range_thresh_f32(const float* x, int N, long long per_sample, float ratio, float* thresh, float* minmax,
                         void* ws, size_t ws_bytes, wmd_stream_t stream);

/* The six per-level pixel sets (depth_decoder.py:305-319, densedepth_decoder.py:316-322):
 *   S0 = max_band |yh| > thresh[n]  (strict; thresh == NULL -> all ones, the reference's level-4 case :305-306)
 *   S1 = dilate3(S0)  S2 = dilate5(S0)                  low resolution  (N,H,W)
 *   S5 = up2(S0)  S4 = dilate3(S5)  S3 = dilate5(S5)    high resolution (N,2H,2W)
 * yh is (N,3,H,W).  Any output pointer may be NULL.  Masks are 0/1 bytes. */
int wmd_level_masks(const float* yh, const float* thresh, uint8_t* s0, uint8_t* s1, uint8_t* s2, uint8_t* s3,
                    uint8_t* s4, uint8_t* s5, int N, int H, int W, wmd_stream_t stream);

/* Replaces mask2idxmap + mask2yx (KITTI/layers.py:371-389) for a whole batch, without the
 * reference's host sync (layers.py:385):
 *   idxmap  (N,H,W) int32 : running row index over the batch, -1 where inactive   [nullable]
 *   pixels  (<= N*H*W) int32 : linear pixel index (n*H + y)*W + x of each active pixel [nullable]
 *   offsets (N+1) int32 : offsets[n] = rows before sample n, offsets[N] = total rows */
size_t wmd_compact_ws_bytes(int N, int H, int W);
int wmd_compact_mask(const uint8_t* mask, int32_t* idxmap, int32_t* pixels, int32_t* offsets, int N, int H, int W,
                     void* ws, size_t ws_bytes, wmd_stream_t stream);

/* out[p] = gate[p] ? (idxmap ? idxmap[p] : p) : -1   for p < count.
 * The fused form of sparse_select (layers.py:337-362): re-indexing onto a subset is a map rewrite. */
int wmd_gate_map(const uint8_t* gate, const int32_t* idxmap, int32_t* out, long long count, wmd_stream_t stream);

/* ---------------------------------------------------------------- layout helpers
 * (N,C,HW) <-> (N,HW,ld) batched transposes (ld >= C; pad columns are zero-filled on the way in).
 * Used for NCHW encoder features -> pixel-major rows, and for the reference's channel-major
 * wire format (layers.py:358) at the functional API. */
int wmd_nchw_to_rows_f32(const float* src, float* dst, int N, int C, long long HW, int ld, wmd_stream_t stream);
int wmd_rows_to_nchw_f32(const float* src, float* dst, int N, int C, long long HW, int ld, wmd_stream_t stream);
/* Same move, but only for the pixels marked in gate (N, HW) bytes: rows of unmarked pixels are left untouched and
 * their source is not read (whole 32-pixel groups without a mark cost no traffic).  The sparse levels read a skip map
 * only under the level's upsample mask (sparse_upsample: skip[mask], KITTI/layers.py:500; the conv's gate argument
 * below), so the decoder passes that mask here and the transpose scales with the mask density. */
int wmd_nchw_to_rows_gated_f32(const float* src, float* dst, const uint8_t* gate, int N, int C, long long HW, int ld,
                               wmd_stream_t stream);
/* rows at an active-pixel list <-> dense NCHW (x[mask] selection, depth_decoder.py:347; make_result, layers.py:365-368) */
int wmd_gather_rows_nchw_f32(const float* src_nchw, float* rows, int ld, int C, const int32_t* pixels,
                             const int32_t* count, int max_rows, int N, int H, int W, wmd_stream_t stream);
int wmd_scatter_rows_nchw_f32(const float* rows, int ld, int C, const int32_t* pixels, const int32_t* count,
                              int max_rows, float* dst_nchw, int N, int H, int W, wmd_stream_t stream);
/* conv weight (Cout,Cin,kh,kw) -> packed [kh*kw][Cin][ldw] (ldw >= Cout, multiple of 4, pad zero) */
int wmd_pack_conv_weight_f32(const float* w, float* packed, int Cout, int Cin, int taps, int ldw, wmd_stream_t stream);

/* ---------------------------------------------------------------- fused 1x1 head stages
 * z = Wz . lrelu(W1 . x + b1): the 1x1 stages of a level's + / - coefficient heads (Conv1x1 + LeakyReLU(0.1),
 * depth_decoder.py:111-120) chained with the per-row tap products of their 3x3 stages (the 9 x 6 values
 * wmd_head_gather_f32 sums per pixel).  x rows (M, c), W1 (n1, c), Wz (nz <= 56, n1); z rows (M, ldz >= 56), columns
 * nz..55 are written as zeros.  The intermediate (M, n1) never reaches memory.  Both GEMMs run tf32x3: |z - exact| <=
 * 4e-6 S + F, F the tf32x3 floor of the first stage carried through |Wz| plus that of the second (tests/head_ref.py);
 * a pre-activation that is non-finite in the contract may be NaN, so a non-finite x makes its own row non-finite.  Supported (c, n1): (32, 64), (64, 128);
 * other shapes return WMD_ERR_UNSUPPORTED (the caller then runs the two stages as wmd_conv_rows launches). */
int wmd_head_mlp_supported(int c, int n1);
size_t wmd_head_mlp_weight_floats(int c, int n1);
int wmd_pack_head_mlp_f32(const float* w1, const float* wz, const float* b1, int c, int n1, int nz, float* packed,
                          wmd_stream_t stream);
int wmd_head_mlp_f32(const float* x, int ldx, int c, const float* packed, int n1, float slope, const int32_t* count,
                     int max_rows, float* z, int ldz, wmd_stream_t stream);

/* ---------------------------------------------------------------- gather-GEMM convolution
 * Replaces sparse_conv3x3 / sparse_conv1x1 / sparse_upsample / sparse_select (KITTI/layers.py:337-508,
 * NYUv2/networks/layers.py:82-223) and, with pixels == NULL, the dense Conv3x3/ConvBlock/Conv1x1 layers
 * (KITTI/layers.py:120-173) of the decoder.  For each output row m (pixel p = pixels[m], or m itself):
 *   y[m, :] = act( bias + sum_{tap, c} in(p + tap)[c] * w[tap][c][:] )
 * where in(q) is the channel concatenation of
 *   source 0: x0[ row0(q), 0:c0 ]  with row0(q) = map0[n, qy>>shift0, qx>>shift0]  (map0 NULL: that pixel's
 *             linear index; taps==1 && map0==NULL: row m itself), zero if row0 < 0        [sparse_select/upsample]
 *   source 1: x1[ (n*H+qy)*W+qx, 0:c1 ]  (dense pixel-major skip map at output resolution)  [skip concat, :500]
 * and in(q) = 0 entirely if gate != NULL and gate[q] == 0, or q is out of the image under WMD_PAD_ZERO.
 * q is mapped into the image by pad_mode exactly as padding the index map does (layers.py:444).
 */
typedef struct wmd_conv_desc {
  int32_t N, H, W;          /* output grid */
  const float* x0;          /* source 0 rows [*][ld0] */
  int32_t c0, ld0;
  const int32_t* map0;      /* (N, H>>shift0, W>>shift0) or NULL */
  int32_t shift0;           /* 0 or 1 */
  const float* x1;          /* source 1 rows [N*H*W][ld1] or NULL */
  int32_t c1, ld1;
  const uint8_t* gate;      /* (N,H,W) or NULL */
  const float* w;           /* packed [taps][c0+c1][ldw] */
  const float* bias;        /* [cout] or NULL */
  int32_t cout, ldw, taps;  /* taps: 1 or 9 */
  int32_t pad_mode;         /* WMD_PAD_* */
  const int32_t* pixels;    /* active output list or NULL (= every pixel) */
  const int32_t* count;     /* device row count (with pixels) */
  int32_t max_rows;         /* capacity of y / upper bound of *count */
  float* y;                 /* rows [max_rows][ldy] */
  int32_t ldy;
  int32_t act;              /* WMD_ACT_* */
  float act_param;          /* LeakyReLU slope */
  const int32_t* map1;      /* (N,H,W): row of pixel q in x1, -1 = none; NULL = x1 is dense (row q).  With a map, x1 holds
                               only the rows of the listed pixels (sparse_upsample's skip[mask], KITTI/layers.py:500, kept
                               compact: wmd_gather_rows_list_f32) */
  int32_t precision;        /* tensor-core engine only.  0 = WMD_PREC_TF32X3: operands split into tf32 hi + lo.  1 = WMD_PREC_F16X3:
                               operands split into two fp16 pieces of x * 2^k - half the MMA instructions and twice their
                               rate; needs amax0 (and amax1 when c1 > 0) and weights packed by wmd_pack_conv_weight_tc16_f32.
                               k puts max(amax0, amax1) into [2^13, 2^14) (one k for both sources and every frame; the weights
                               get their own from max |w|), so no finite operand overflows.  The pair carries tf32x3's 22
                               mantissa bits only for operands within 2^-11 of their maximum: below that the low piece is an
                               fp16 subnormal, whose absolute error is 2^-25 of a scaled unit.  See the bound below.  The
                               Python KITTI decoders use F16X3 by default; launches without source maxima use TF32X3 */
  const float* amax0;       /* device scalars: max |x0|, max |x1| over the finite values of the rows the launch can read
                               (upper bounds are fine) */
  const float* amax1;
  float* amax_out;          /* device scalar, or NULL: atomically raised to max |y| over the finite y of the rows written
                               (zero it before the first producer; both precisions, every scheduling mode).  Every maximum
                               libwmd produces skips NaN and +-Inf, so one non-finite value leaves the scales of the rest */
  int32_t rows0;            /* rows allocated in x0, 0 = unknown.  Only used by the tensor-core engine's 1x1 form (taps == 1,
                               map0 == NULL: output row m reads x0 row m): with rows0 > 0 rows past rows0 read zeros */
} wmd_conv_desc;

int wmd_conv_rows_f32(const wmd_conv_desc* d, wmd_stream_t stream);

/* Tensor-core engine for the same contract: wgmma tf32 with a 3xTF32 split (hi*hi + lo*hi + hi*lo,
 * fp32 accumulation), so results stay fp32-faithful: |y - exact| <= 1.7e-5 S + F, S = |bias| + sum |x w| of the element's
 * terms (measured worst, same-sign operands, H100; f16x3: 8.6e-6 S for operands within 2^-11 of their maxima, the SIMT
 * kernel: 6.5e-6 S + F at K = 18432).  F is an absolute floor for the bottom of the fp32 range (tests/conv_ref.py
 * derives it): tf32x3 F = 2^-126 (sum |w| over the nonzero x + sum |x| over the nonzero w + 6 K') + 16 x 2^-149, which
 * holds even where subnormal pieces, products and sums are flushed; the fp32 FMA engine F = 2^-149 (K' + 8).  Both are
 * below 2^-22 S wherever operands and products are normal.  f16x3 in general: |y - exact| <= 2.5e-5 S + F, with the absolute floor
 *   F = 2^-25 (sum |w| over the nonzero x / s_x + sum |x| over the nonzero w / s_w) + 2^-50 K' / (s_x s_w) + 2^-149
 * (s_x, s_w the two scales, K' the number of terms with both factors nonzero): each operand's split is off by at most
 * 2^-22 of itself or 2^-25 / s, whichever is larger (tests/conv_ref.py derives it).  Non-finite inputs: an output is
 * non-finite exactly where the fp64 contract's is (the rows whose taps read a NaN or +-Inf), except on the tensor-core
 * engines: their split's remainder of an Inf is Inf - Inf, so the activation is applied to a pre-activation that may be
 * NaN wherever the contract's pre-activation is non-finite, and an output may be NaN where the contract's is +-Inf or
 * where ELU(-Inf) = -1 or sigmoid(+-Inf) is finite.  The SIMT engine follows the contract exactly.  Other rows are
 * unaffected.  The weight packs split to nearest, except that a finite |w| >= (2 - 2^-11) 2^127, which would round up
 * to Inf, takes the truncated high piece.
 * d->w must point to weights packed by wmd_pack_conv_weight_tc_f32 for the same (cout, c0, c1, taps); d->ldw is ignored.
 *   wmd_conv_tc_tile_n(cout)                 N-tile of the kernel for this cout (128 / 64 / 32; the CTA tile is 128 rows x N)
 *   wmd_conv_tc_weight_floats(...)           size of the packed weight buffer, in floats
 *   wmd_pack_conv_weight_tc_f32(w, packed..) (Cout, c0+c1, kh, kw) -> per (n-tile, 32-channel chunk) fp32
 *                                            shared-memory images [tf32 hi | tf32 lo] of N x 32, K-major, 128-byte swizzled
 * Accumulation runs in epochs of K = 1024 in the wgmma accumulators, each added into fp32 registers with
 * round-to-nearest adds, because the tensor core's own fp32 accumulation does not round to nearest (a one-signed bias of
 * ~1.6e-8 * K of S in tf32x3, ~8.5e-9 * K in f16x3, measured on H100: it stays that of one epoch, not of the whole K).
 * Dense 3x3 launches (no pixels, map0, map1 or gate; splits 0 or 1) whose per-tile source windows fit 288 rows (output
 * width W <= 79 with a full-resolution source; W <= 192 when the only source is x0 with shift0 = 1) run in a second
 * kernel, conv_rows_tc_kernel_window, that loads each source's window of rows once per 32-channel chunk instead of once
 * per tap; the results are bit-identical to the gather kernel's. */
enum { WMD_PREC_TF32X3 = 0, WMD_PREC_F16X3 = 1 };
int wmd_conv_tc_tile_n(int cout);
/* Weights for precision = WMD_PREC_F16X3: 128-byte header (float 0: 1 / s_w, float 1: max |w|, int 2: e_w = log2 s_w) +
 * per (n-tile, 32-channel chunk) one N x 128 B image whose rows hold [fp16(w s_w): 32 channels | fp16(w s_w - that): 32
 * channels], s_w = 2^e_w the power of two that puts max |w| over the finite w into [2^13, 2^14), e_w <= 127 (computed
 * on the device, no host sync).  `packed` needs wmd_conv_tc16_weight_bytes() bytes. */
size_t wmd_conv_tc16_weight_bytes(int cout, int c0, int c1, int taps);
int wmd_pack_conv_weight_tc16_f32(const float* w, void* packed, int Cout, int c0, int c1, int taps, wmd_stream_t stream);
/* max |x| of `count` floats, atomically raised into *amax (device scalar, zero it first): for sources that no libwmd
 * kernel produced (channels_last feature maps used in place).  The layout moves below take an optional `amax` too. */
int wmd_amax_f32(const float* x, long long count, float* amax, wmd_stream_t stream);
/* max |x| over the rows r of x (rows x cols, contiguous) with mask[r] != 0: a channels_last map used in place whose
 * consumer reads only the masked pixels */
int wmd_amax_rows_masked_f32(const float* x, long long rows, int cols, const uint8_t* mask, float* amax, wmd_stream_t stream);
int wmd_nchw_to_rows_amax_f32(const float* src, float* dst, int N, int C, long long HW, int ld, float* amax, wmd_stream_t stream);
/* plain move (every row) whose maximum covers only the pixels `mask` (N, HW) marks: the rows its consumer reads */
int wmd_nchw_to_rows_masked_amax_f32(const float* src, float* dst, const uint8_t* mask, int N, int C, long long HW, int ld,
                                     float* amax, wmd_stream_t stream);
/* gated move: the maximum covers exactly the marked pixels (the rows written), as the list gather's covers the listed
 * rows - the three moves of one map under one mask report the same maximum */
int wmd_nchw_to_rows_gated_amax_f32(const float* src, float* dst, const uint8_t* gate, int N, int C, long long HW, int ld,
                                    float* amax, wmd_stream_t stream);
int wmd_gather_rows_list_amax_f32(const float* src_nchw, float* rows, int ld, int C, const int32_t* pixels,
                                  const int32_t* count, int max_rows, int N, int H, int W, float* amax, wmd_stream_t stream);
size_t wmd_conv_tc_weight_floats(int cout, int c0, int c1, int taps);
int wmd_pack_conv_weight_tc_f32(const float* w, float* packed, int Cout, int c0, int c1, int taps, wmd_stream_t stream);
int wmd_conv_rows_tc_f32(const wmd_conv_desc* d, wmd_stream_t stream);
/* Same, with the reduction split `splits` ways across CTAs (split-K): layers with few output tiles then fill all
 * SMs.  Partial sums go to `ws` (wmd_conv_tc_splitk_ws_bytes) and are summed in a fixed order, biased and
 * activated by a second small kernel, so results stay deterministic.  splits = 1 is wmd_conv_rows_tc_f32.
 * splits = 0 selects BALANCED scheduling (data-parallel + stream-K): full rounds of tiles run whole; the (tile,
 * 32-channel chunk) units of the remainder tiles are dealt to the CTAs in equal contiguous ranges computed on the
 * device from the actual row count, so sparse layers whose tile count is data dependent still finish on all SMs
 * together; only remainder tiles cut by a range boundary (<= 8 segments) go through the workspace: the LAST segment of
 * a tile to arrive (per-tile arrival counter) sums all of them in slab order - bias first - inside the same kernel, so
 * there is no second pass and the bits do not depend on the arrival order.  Its workspace size does not depend on the
 * layer (4 KiB of counters + SMs x 8 x 128 x 128 floats).  The first 4 KiB of `ws` (any splits) must be ZERO before the
 * first launch that uses the buffer; every launch leaves them zero. */
size_t wmd_conv_tc_splitk_ws_bytes(int max_rows, int ldy, int splits);
/* The tensor-core engine runs one persistent CTA per SM, and such a CTA holds most of the SM's shared memory: no other kernel -
 * an NCCL collective of the previous step in particular - can run beside it.  wmd_conv_tc_set_reserved_sms(n) makes the
 * persistent grid n CTAs smaller so that n SMs stay free (multi-GPU serving: the all-gather of step k then really runs
 * under the convolutions of step k + 1).  0 by default; n < 0 only queries.  Returns the previous setting.  Process-wide;
 * set it before capturing CUDA graphs. */
int wmd_conv_tc_set_reserved_sms(int n);
int wmd_conv_rows_tc_splitk_f32(const wmd_conv_desc* d, int splits, void* ws, size_t ws_bytes, wmd_stream_t stream);

/* ---------------------------------------------------------------- coefficient heads (few output channels)
 * The 3x3 stage of the wavelet heads (depth_decoder.py:104-120,126-136,242-290; NYU wave convs
 * densedepth_decoder.py:104-115) on pixel-major rows `t`, scattered to a dense NCHW tensor:
 *   a = conv3x3(t[:, off_a:off_a+c]; wa, ba)   b = conv3x3(t[:, off_b:off_b+c]; wb, bb)   (off_b < 0: single head)
 *   out[n, :, y, x] = scale * (act(a) - act(b))     or   scale * act(a)
 * out must be zero-filled by the caller when pixels != NULL (the reference's make_result, layers.py:473-478).
 */
typedef struct wmd_head_desc {
  int32_t N, H, W;
  const float* t;
  int32_t ld, c, off_a, off_b;
  const int32_t* map;       /* (N,H,W) row of each pixel, -1 inactive; NULL = linear pixel index */
  const float* wa; const float* ba;   /* packed [9][c][cout], bias [cout] */
  const float* wb; const float* bb;
  int32_t cout;             /* 1..4 */
  int32_t pad_mode, act;
  float scale;
  const int32_t* pixels; const int32_t* count; int32_t max_rows;
  float* out;               /* (N,cout,H,W) */
} wmd_head_desc;

int wmd_head_conv3x3_f32(const wmd_head_desc* d, wmd_stream_t stream);

/* Factored form of the same stage (what the decoders use for the +/- heads): the per-tap products
 * z[row, tap*groups + g] = t[row, :] . w_g[:, tap] are computed once per active input row by wmd_conv_rows_*_f32
 * (taps = 1, cout = 9*groups); this entry point gathers and sums the nine taps per output pixel,
 *   s_g = bias[g] + sum_tap z[map(p + tap), tap*groups + g],
 * and scatters  out[n, j, y, x] = scale * (act(s_j) - act(s_{cout+j}))  (dual, groups = 2*cout)  or  scale * act(s_j)
 * (groups = cout) into the dense NCHW tensor (zero-filled by the caller when pixels != NULL).  groups in {1,2,3,4,6,8}.
 * z has no alignment requirement (any column offset, any ldz); 8-byte aligned z with an even ldz reads float2 pairs,
 * with the same sums. */
int wmd_head_gather_f32(const float* z, int ldz, int groups, const int32_t* map, const float* bias, float scale, int act,
                        int dual, int pad_mode, const int32_t* pixels, const int32_t* count, int max_rows, float* out,
                        int cout, int N, int H, int W, wmd_stream_t stream);

/* ---------------------------------------------------------------- fused tail of a decoder level
 * One kernel for:  factored 3x3 stage of the +/- coefficient heads (get_coefficients / get_sparse_coefficients,
 * depth_decoder.py:126-136,242-290: yh = 2^(i-1) (sigmoid(.) - sigmoid(.)), zero outside the wavelet mask)
 *                  -> pytorch_wavelets.DWTInverse (depth_decoder.py:164,372,416)
 *                  -> disp = clamp(yl / 2^(i-1), 0, 1) (depth_decoder.py:166)
 *                  -> the consumer's epilogue of ("disp", 0): disp_to_depth (KITTI/layers.py:16-25) or depth / 100
 *                     + clamp (NYUv2/utils.py:219,229)
 *                  -> thresh = (max - min)(yl) * ratio of the NEXT level's masks (depth_decoder.py:308), per sample.
 * z: rows of tap products from wmd_head_mlp_f32 / the tap-product GEMM, 54 floats [tap][+LH,+HL,+HH,-LH,-HL,-HH] from
 * z[0] (pass z + col0 for a column offset), row of pixel q = map[q] (map == NULL: q), pixels with mask == 0 (mask != NULL)
 * get zero coefficients.  yh (N,3,H,W) is written once (an output of the decoder) and not read back; out / disp are
 * (N,1,2H,2W).  ll / mask rows of a tile are staged by TMA bulk copies when W % 16 == 0.  Results are bit-identical to
 * wmd_head_gather_f32 + wmd_idwt_haar_f32 + wmd_range_thresh_f32.  thresh == NULL skips the range reduction (then ws may
 * be NULL); otherwise ws needs wmd_head_idwt_ws_bytes() bytes whose first 64 KiB are zero before the first use (the kernel
 * leaves them zeroed, like wmd_range_thresh_f32). */
enum { WMD_EPI_NONE = 0, WMD_EPI_DISP_TO_DEPTH = 1, WMD_EPI_DIV_CLAMP = 2 };
typedef struct wmd_head_idwt_desc {
  int32_t N, H, W;           /* coefficient grid of the level */
  const float* z;            /* tap-product rows [*][ldz] */
  int32_t ldz;
  const int32_t* map;        /* (N,H,W) row of a pixel in z, -1 = none; NULL = linear index */
  const uint8_t* mask;       /* (N,H,W) wavelet mask (S5) or NULL = every pixel */
  const float* bias;         /* [6]: + head's 3 biases then - head's, or NULL */
  float scale;               /* 2^(i-1) */
  int32_t pad_mode;          /* WMD_PAD_* of the heads' 3x3 stage */
  const float* ll;           /* (N,1,H,W) */
  float* yh;                 /* (N,3,H,W) */
  float* out;                /* (N,1,2H,2W) reconstruction */
  float* disp;               /* (N,1,2H,2W) = [clamp01](out * disp_scale), or NULL */
  float disp_scale;
  int32_t clamp01;
  int32_t epi_mode;          /* WMD_EPI_*: DISP_TO_DEPTH: epi_out0 = epi_a + epi_b * disp, epi_out1 = 1 / epi_out0 (nullable);
                                DIV_CLAMP: epi_out0 = out / epi_a, clamped to [epi_lo, epi_hi] if epi_b != 0.
                                The disparity clamp and DIV_CLAMP propagate NaN as torch.clamp does */
  float epi_a, epi_b, epi_lo, epi_hi;
  float* epi_out0;
  float* epi_out1;
  float* thresh;             /* (N) (max - min)(out_n) * thresh_ratio, or NULL */
  float thresh_ratio;
} wmd_head_idwt_desc;
/* The plain IDWT with the same consumer epilogue (NYU decoders: the last level's reconstruction IS ("disp", 0)). */
int wmd_idwt_haar_epi_f32(const float* ll, const float* hf, float* out, float* disp, float disp_scale, int clamp01,
                          int epi_mode, float epi_a, float epi_b, float epi_lo, float epi_hi, float* epi_out0,
                          float* epi_out1, int N, int C, int H, int W, wmd_stream_t stream);
/* rows[m][0..C) = src[n, :, y, x] for the m-th pixel of a list (pixels[m] = (n*H + y)*W + x, m < *count), columns C..ld-1
 * zero: the layout move of a skip map restricted to EXACTLY the active pixels (the reference's skip[mask],
 * KITTI/layers.py:500) - 128 list entries x 32 channels per tile, coalesced on both sides for clustered lists.  `src` may
 * be pinned HOST memory (read in place over PCIe: only the listed pixels cross the bus).  ld % 4 == 0. */
int wmd_gather_rows_list_f32(const float* src_nchw, float* rows, int ld, int C, const int32_t* pixels, const int32_t* count,
                             int max_rows, int N, int H, int W, wmd_stream_t stream);
size_t wmd_head_idwt_ws_bytes(int N, int H, int W);
int wmd_head_idwt_f32(const wmd_head_idwt_desc* d, void* ws, size_t ws_bytes, wmd_stream_t stream);

/* ---------------------------------------------------------------- full-resolution tail of the baseline decoder
 * ("disp", 0) of monodepth2's DepthDecoder (KITTI/networks/decoders/depth_decoder.py:55-67 at i = 0) in one launch:
 *   u    = ELU(b1 + conv3x3(up2(x); W1))        upconv(0,1): nearest x2, ZERO padding, 16 -> 16 channels
 *   disp = sigmoid(b2 + conv3x3(u; W2))         dispconv(0): REFLECT padding (KITTI/layers.py:149), 16 -> cout
 * x: rows (N*H*W, ld) at half resolution H x W (upconv(0,0)'s output as wmd_conv_rows_f32 writes it: ld >= 16,
 * ld % 4 == 0, 16-byte aligned); disp: (N, cout, 2H, 2W) NCHW, cout = 1..4; nothing else is written.  u never reaches
 * memory.  The 16 -> 16 stage runs on tensor cores with the 3xTF32 split (fp32-faithful, fp32 accumulation), the
 * dispconv in fp32 FMAs: |disp - exact| <= 3e-8 S + F plus the ELU / sigmoid's own absolute error, F the tf32x3 floor
 * carried through |W2| plus the FMA floor (tests/disp_tail_ref.py).  A non-finite x gives NaN over its up2, 3x3, 3x3
 * footprint (sigmoid of a NaN pre-activation, where the contract's may be sigmoid(-Inf) = 0).  N = 0 launches nothing.
 * The weights are packed once by wmd_pack_disp_tail16_f32: w1 (16,16,3,3), b1 (16) or NULL, w2 (cout,16,3,3), b2 (cout)
 * or NULL -> packed, WMD_DISP_TAIL16_PACKED_FLOATS floats, 16-byte aligned. */
enum { WMD_DISP_TAIL16_PACKED_FLOATS = 5332 };
int wmd_pack_disp_tail16_f32(const float* w1, const float* b1, const float* w2, const float* b2, int cout, float* packed,
                             wmd_stream_t stream);
int wmd_disp_tail16_f32(const float* x, int ld, const float* packed, int cout, float* disp, int N, int H, int W,
                        wmd_stream_t stream);

/* ---------------------------------------------------------------- convolution backward (training)
 * The backward of one dense wmd_conv_desc layer (pixels, gate and map1 NULL) y = act(bias + A W), A the gathered rows:
 *
 * Activation backward: dz[r, o] = dy[r, o] * act'(y[r, o]) from the saved post-activation output y (ELU: y > 0 ? 1 : y + 1;
 * LeakyReLU: y > 0 ? 1 : act_param; sigmoid: y (1 - y); none: 1), for rows r < rows and o < cout.  db (nullable) = sum over
 * rows of dz, summed in fp64 in a fixed order (per-block partials, then block order) and rounded to fp32 once, so the bits
 * do not depend on timing.
 * amax_dz (nullable) is raised to max |dz|: the fp16-pair operand form of the data-gradient launch needs it.  ws (with db):
 * wmd_act_bwd_ws_bytes() bytes whose first 4 KiB are zero before the first use; the kernel leaves them zero.  The same
 * buffer may serve wmd_conv_wgrad_f32 launches on the same stream. */
size_t wmd_act_bwd_ws_bytes(int rows, int cout);
int wmd_act_bwd_f32(const float* y, int ldy, const float* dy, int lddy, int rows, int cout, int act, float act_param,
                    float* dz, int lddz, float* db, float* amax_dz, void* ws, size_t ws_bytes, wmd_stream_t stream);
/* Weight gradient: dw[o][c][ky][kx] = sum_p A(p)[tap][c] dz[p][o] (torch's (Cout, Cin, kh, kw) layout, tap = 3 ky + kx),
 * A gathered exactly as the forward gathers it from the desc's sources, map0 / shift0, pad mode and taps; d->w, bias, y
 * and act are not read.  Tensor cores (mma.sync tf32) with the operands split into tf32 hi + lo (3 MMAs per product)
 * and each 32-pixel chunk's MMA sum added into fp32 sums with round-to-nearest adds.  taps = 1 needs shift0 = 0.  Layers with few output tiles split the
 * pixel reduction across CTAs; the last CTA of a tile to arrive sums the partial slabs in slab order, so results are
 * deterministic (no float atomics).  |dw - exact| <= 2.5e-6 S + F with the tf32x3 floor of A against dz plus 2^-149 per
 * chunk add (tests/conv_grad_ref.py, wgrad_floor).  ws: wmd_conv_wgrad_ws_bytes(d) bytes (0: none needed) whose first 4 KiB (per-tile
 * arrival counters) are zero before the first use; the kernel leaves them zero. */
size_t wmd_conv_wgrad_ws_bytes(const wmd_conv_desc* d);
int wmd_conv_wgrad_f32(const wmd_conv_desc* d, const float* dz, int lddz, float* dw, void* ws, size_t ws_bytes,
                       wmd_stream_t stream);
/* Fold of the data gradient.  g: rows (N (H+2) (W+2), ldg) of the gradient of the padded input, i.e. the forward contract
 * run over the grid extended by one pixel on each side with the flipped, transposed weight, zero padding and a map0 that
 * reads dz (-1 on the ring).  Each ring value is added into the pixel the pad mode maps it to (pad_coord; zero padding
 * drops it).  Channels [0, c0) go to dx0 rows: per pixel, or with shift0 = 1 summed over the 2x2 children into the
 * (N, H/2, W/2) low-resolution rows (the nearest x2 upsample's adjoint); columns c0..lddx0-1 are written as zeros.
 * Channels [c0, c0 + c1) go to dx1_nchw (N, c1, H, W).  Fixed summation order. */
int wmd_conv_dgrad_fold_f32(const float* g, int ldg, int N, int H, int W, int pad_mode, int c0, int shift0, float* dx0,
                            int lddx0, int c1, float* dx1_nchw, wmd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* WMD_H */
