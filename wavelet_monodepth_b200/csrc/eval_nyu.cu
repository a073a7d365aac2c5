// NYUv2 depth evaluation (NYUv2/utils.py: add_results, evaluate, compute_errors_nyu): the reference's prediction chain
// (scale, align_corners bilinear resize, replication pad, resize, clamp, Eigen crop) in fp64 with explicit _rn
// intrinsics, so nvcc's FMA contraction cannot change a rounding, then the metrics' per-frame sums in a fixed order.
//
// Eigen mode runs three launches per batch: the (224, 304) intermediate of each frame into the workspace (0.55 MB per
// frame, L2-resident at the batch sizes an evaluation uses); one CTA per (frame, band of output rows) for the rest of
// the chain and that band's sums; a last launch that adds each frame's band slabs in band order.  224 mode skips the
// first.  No atomics anywhere, so the bits depend only on each frame's own inputs.
#include <math.h>
#include "common.cuh"
#include "wmd_eval.h"

namespace wmd {

constexpr int kNyuThreads = 256;
constexpr int kNyuBandRows = 8;
constexpr int kNyuMidH = 224, kNyuMidW = 304;          // utils.py:223: (240 - 16, 320 - 16)
constexpr int kNyuPad = 8;                             // ReplicationPad2d(16 // 2)
constexpr int kNyuFullH = 480, kNyuFullW = 640;        // scale_factor 2 of the padded (240, 320)
constexpr int kNyuCropY = 20, kNyuCropX = 24;          // EIGEN_CROP = [20, 459, 24, 615]
constexpr int kNyuErrChunk = kNyuThreads * 16;         // pixels per CTA of wmd_eval_nyu_errors_f64

__host__ __device__ constexpr int nyu_out_h(int mode) { return mode == WMD_EVAL_NYU_224 ? 224 : WMD_EVAL_NYU_CROP_H; }
__host__ __device__ constexpr int nyu_out_w(int mode) { return mode == WMD_EVAL_NYU_224 ? 224 : WMD_EVAL_NYU_CROP_W; }
__host__ __device__ constexpr int nyu_bands(int mode) { return (nyu_out_h(mode) + kNyuBandRows - 1) / kNyuBandRows; }

// ------------------------------------------------------------------------------------ the prediction chain
// utils.py:216-219: disp / 100, or DepthNorm(disp, 1000) / 10000, where torch evaluates 1000 / t as reciprocal(t) * 1000
__device__ __forceinline__ double nyu_scale(float d, int use_disparity) {
  const double v = static_cast<double>(d);
  return use_disparity ? __ddiv_rn(__dmul_rn(__drcp_rn(v), 1000.0), 10000.0) : __ddiv_rn(v, 100.0);
}

// torch's align_corners=True taps of one axis: src = scale * d, i0 = (int)src, lambda = src - i0, i1 = i0 + (i0 < in-1)
struct AcTap {
  int i0, i1;
  double w0, w1;
};
__device__ __forceinline__ AcTap ac_tap(int d, int in, double scale) {
  const double src = __dmul_rn(scale, static_cast<double>(d));
  AcTap t;
  t.i0 = min(static_cast<int>(src), in - 1);
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  t.w1 = __dadd_rn(src, -static_cast<double>(t.i0));
  t.w0 = __dadd_rn(1.0, -t.w1);
  return t;
}
__device__ __forceinline__ double ac_scale(int in, int out) {
  return out > 1 ? __ddiv_rn(static_cast<double>(in - 1), static_cast<double>(out - 1)) : 0.0;
}

// h0 * (w0 * x00 + w1 * x01) + h1 * (w0 * x10 + w1 * x11): every tap read and multiplied, zero weights included
__device__ __forceinline__ double bilerp(const AcTap& ty, const AcTap& tx, double x00, double x01, double x10,
                                         double x11) {
  const double r0 = __dadd_rn(__dmul_rn(tx.w0, x00), __dmul_rn(tx.w1, x01));
  const double r1 = __dadd_rn(__dmul_rn(tx.w0, x10), __dmul_rn(tx.w1, x11));
  return __dadd_rn(__dmul_rn(ty.w0, r0), __dmul_rn(ty.w1, r1));
}

// torch.clamp(p, 0.4, 10) by comparisons: NaN stays NaN
__device__ __forceinline__ double nyu_clamp(double v) {
  if (v < 0.4) v = 0.4;
  if (v > 10.0) v = 10.0;
  return v;
}

// Eigen step 2: (h, w) scaled disparity -> (224, 304), one frame per blockIdx.y
__global__ void __launch_bounds__(kNyuThreads) nyu_mid_kernel(const float* __restrict__ disp, int h, int w,
                                                              int use_disparity, double* __restrict__ mid) {
  const int f = blockIdx.y;
  const float* src = disp + static_cast<long long>(f) * h * w;
  const double sy = ac_scale(h, kNyuMidH), sx = ac_scale(w, kNyuMidW);
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < kNyuMidH * kNyuMidW; p += gridDim.x * blockDim.x) {
    const int y = p / kNyuMidW, x = p % kNyuMidW;
    const AcTap ty = ac_tap(y, h, sy), tx = ac_tap(x, w, sx);
    const float* r0 = src + static_cast<long long>(ty.i0) * w;
    const float* r1 = src + static_cast<long long>(ty.i1) * w;
    mid[static_cast<long long>(f) * kNyuMidH * kNyuMidW + p] =
        bilerp(ty, tx, nyu_scale(r0[tx.i0], use_disparity), nyu_scale(r0[tx.i1], use_disparity),
               nyu_scale(r1[tx.i0], use_disparity), nyu_scale(r1[tx.i1], use_disparity));
  }
}

// Eigen steps 3-4 at full-resolution pixel (Y, X): ReplicationPad2d(8) of the intermediate, resized to (480, 640)
__device__ __forceinline__ double nyu_full(const double* __restrict__ mid, int Y, int X, double sy, double sx) {
  const AcTap ty = ac_tap(Y, kNyuMidH + 2 * kNyuPad, sy);
  const AcTap tx = ac_tap(X, kNyuMidW + 2 * kNyuPad, sx);
  const int y0 = clamp_idx(ty.i0 - kNyuPad, kNyuMidH) * kNyuMidW, y1 = clamp_idx(ty.i1 - kNyuPad, kNyuMidH) * kNyuMidW;
  const int x0 = clamp_idx(tx.i0 - kNyuPad, kNyuMidW), x1 = clamp_idx(tx.i1 - kNyuPad, kNyuMidW);
  return bilerp(ty, tx, mid[y0 + x0], mid[y0 + x1], mid[y1 + x0], mid[y1 + x1]);
}

// ------------------------------------------------------------------------------------ metrics
// compute_errors_nyu (utils.py:85-98) terms of one pixel: y ground truth, ly its log10, x prediction
struct NyuSums {
  double rel, sq, lg;
  unsigned a1, a2, a3, n;
};
__device__ __forceinline__ void nyu_accumulate(NyuSums& s, double y, double ly, double x) {
  const double q0 = __ddiv_rn(y, x), q1 = __ddiv_rn(x, y);
  const double t = (isnan(q0) || isnan(q1)) ? q0 + q1 : fmax(q0, q1);     // torch.max propagates NaN
  s.a1 += t < 1.25;
  s.a2 += t < 1.5625;
  s.a3 += t < 1.953125;
  const double d = __dadd_rn(y, -x);
  s.rel = __dadd_rn(s.rel, __ddiv_rn(fabs(d), y));
  s.sq = __dadd_rn(s.sq, __dmul_rn(d, d));
  s.lg = __dadd_rn(s.lg, fabs(__dadd_rn(ly, -log10(x))));
  s.n += 1;
}

// fixed-order tree over the CTA's threads -> out[7] = (sum rel, sum sq, sum log, a1, a2, a3, pixels) as doubles
__device__ void nyu_block_sums(NyuSums s, double* __restrict__ out) {
  __shared__ double sd[3][kNyuThreads];
  __shared__ unsigned su[4][kNyuThreads];
  const int t = threadIdx.x;
  sd[0][t] = s.rel; sd[1][t] = s.sq; sd[2][t] = s.lg;
  su[0][t] = s.a1; su[1][t] = s.a2; su[2][t] = s.a3; su[3][t] = s.n;
  __syncthreads();
  for (int k = kNyuThreads / 2; k > 0; k >>= 1) {
    if (t < k) {
#pragma unroll
      for (int j = 0; j < 3; ++j) sd[j][t] = __dadd_rn(sd[j][t], sd[j][t + k]);
#pragma unroll
      for (int j = 0; j < 4; ++j) su[j][t] += su[j][t + k];
    }
    __syncthreads();
  }
  if (t < 7) out[t] = t < 3 ? sd[t][0] : static_cast<double>(su[t - 3][0]);
}

// one CTA per (band of output rows, frame): the chain's last steps and the band's sums -> slab[frame][band][7]
__global__ void __launch_bounds__(kNyuThreads) nyu_band_kernel(
    const float* __restrict__ disp, const double* __restrict__ mid, int mode, int use_disparity,
    const float* __restrict__ gt, const float* __restrict__ gt_log10, double* __restrict__ depth_out,
    double* __restrict__ slab) {
  const int band = blockIdx.x, f = blockIdx.y;
  const int H = nyu_out_h(mode), W = nyu_out_w(mode);
  const int r0 = band * kNyuBandRows, r1 = min(r0 + kNyuBandRows, H);
  const long long plane = static_cast<long long>(H) * W;
  const double* fmid = mid ? mid + static_cast<long long>(f) * kNyuMidH * kNyuMidW : nullptr;
  const double sy = ac_scale(kNyuMidH + 2 * kNyuPad, kNyuFullH), sx = ac_scale(kNyuMidW + 2 * kNyuPad, kNyuFullW);
  NyuSums s = {0.0, 0.0, 0.0, 0u, 0u, 0u, 0u};
  for (int p = r0 * W + threadIdx.x; p < r1 * W; p += blockDim.x) {
    const long long i = f * plane + p;
    double x;
    if (mode == WMD_EVAL_NYU_224)
      x = nyu_scale(disp[i], use_disparity);
    else
      x = nyu_full(fmid, p / W + kNyuCropY, p % W + kNyuCropX, sy, sx);
    x = nyu_clamp(x);
    if (depth_out) depth_out[i] = x;
    nyu_accumulate(s, static_cast<double>(gt[i]), static_cast<double>(gt_log10[i]), x);
  }
  nyu_block_sums(s, slab + (static_cast<long long>(f) * gridDim.x + band) * 7);
}

// out[r][j] = slab[r][0][j] + slab[r][1][j] + ... in slab order (one thread per output value)
__global__ void nyu_slab_sum_kernel(const double* __restrict__ slab, int rows, int slabs, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * 7) return;
  const int r = i / 7, j = i % 7;
  const double* s = slab + static_cast<long long>(r) * slabs * 7 + j;
  double acc = 0.0;
  for (int k = 0; k < slabs; ++k) acc = __dadd_rn(acc, s[7ll * k]);
  out[i] = acc;
}

// wmd_eval_nyu_errors_f64: CTA b sums pixels [b * chunk, (b + 1) * chunk) in a fixed tree
__global__ void __launch_bounds__(kNyuThreads) nyu_errors_kernel(const double* __restrict__ pred,
                                                                 const double* __restrict__ gt, long long n,
                                                                 double* __restrict__ slab) {
  const long long beg = static_cast<long long>(blockIdx.x) * kNyuErrChunk;
  const long long end = beg + kNyuErrChunk < n ? beg + kNyuErrChunk : n;
  NyuSums s = {0.0, 0.0, 0.0, 0u, 0u, 0u, 0u};
  for (long long i = beg + threadIdx.x; i < end; i += blockDim.x) nyu_accumulate(s, gt[i], log10(gt[i]), pred[i]);
  nyu_block_sums(s, slab + 7ll * blockIdx.x);
}

// the six means of compute_errors_nyu from the pooled sums (one thread)
__global__ void nyu_errors_finish_kernel(const double* __restrict__ sums, double* __restrict__ errors) {
  const double n = sums[6];
  errors[0] = __ddiv_rn(sums[0], n);
  errors[1] = sqrt(__ddiv_rn(sums[1], n));
  errors[2] = __ddiv_rn(sums[2], n);
  for (int k = 0; k < 3; ++k) errors[3 + k] = __ddiv_rn(sums[3 + k], n);
}

}  // namespace wmd

// ---------------------------------------------------------------------------------------- C ABI
namespace {
size_t frames_ws_bytes(int n, int mode) {
  using namespace wmd;
  const size_t mid = mode == WMD_EVAL_NYU_224 ? 0 : static_cast<size_t>(kNyuMidH) * kNyuMidW;
  return static_cast<size_t>(n) * (mid + static_cast<size_t>(nyu_bands(mode)) * 7) * sizeof(double);
}
int err_chunks(long long n) { return wmd::ceil_div(n, wmd::kNyuErrChunk); }
}  // namespace

extern "C" size_t wmd_eval_nyu_ws_bytes(int n, int mode) {
  if (n < 0 || (mode != WMD_EVAL_NYU_EIGEN && mode != WMD_EVAL_NYU_224)) return 0;
  return frames_ws_bytes(n, mode);
}

extern "C" int wmd_eval_nyu_frames(const float* disp, int n, int h, int w, int mode, int use_disparity,
                                   const float* gt, const float* gt_log10, double* depth_out, void* ws,
                                   size_t ws_bytes, double* sums, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(mode == WMD_EVAL_NYU_EIGEN || mode == WMD_EVAL_NYU_224, WMD_ERR_ARG);
  WMD_REQUIRE(n >= 0 && n <= 65535 && h > 0 && w > 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(mode != WMD_EVAL_NYU_224 || (h == 224 && w == 224), WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(n) * h * w < (1ll << 31), WMD_ERR_SHAPE);
  if (n == 0) return WMD_OK;
  WMD_REQUIRE(disp && gt && gt_log10 && ws && sums, WMD_ERR_ARG);
  WMD_REQUIRE(ws_bytes >= frames_ws_bytes(n, mode), WMD_ERR_ARG);
  cudaStream_t st = as_stream(stream);
  double* mid = nullptr;
  double* slab = static_cast<double*>(ws);
  if (mode == WMD_EVAL_NYU_EIGEN) {
    mid = slab;
    slab += static_cast<size_t>(n) * kNyuMidH * kNyuMidW;
    nyu_mid_kernel<<<dim3(ceil_div(kNyuMidH * kNyuMidW, kNyuThreads * 4), n), kNyuThreads, 0, st>>>(
        disp, h, w, use_disparity, mid);
    if (int rc = launched()) return rc;
  }
  nyu_band_kernel<<<dim3(nyu_bands(mode), n), kNyuThreads, 0, st>>>(disp, mid, mode, use_disparity, gt, gt_log10,
                                                                    depth_out, slab);
  if (int rc = launched()) return rc;
  nyu_slab_sum_kernel<<<ceil_div(7ll * n, 128), 128, 0, st>>>(slab, n, nyu_bands(mode), sums);
  return launched();
}

extern "C" size_t wmd_eval_nyu_errors_ws_bytes(long long n) {
  return n < 0 ? 0 : (static_cast<size_t>(err_chunks(n)) + 1) * 7 * sizeof(double);
}

extern "C" int wmd_eval_nyu_errors_f64(const double* pred, const double* gt, long long n, void* ws, size_t ws_bytes,
                                       double* errors, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(n >= 0 && n < (1ll << 40), WMD_ERR_SHAPE);
  WMD_REQUIRE(errors && ws && (n == 0 || (pred && gt)), WMD_ERR_ARG);
  WMD_REQUIRE(ws_bytes >= wmd_eval_nyu_errors_ws_bytes(n), WMD_ERR_ARG);
  cudaStream_t st = as_stream(stream);
  const int chunks = err_chunks(n);
  double* slab = static_cast<double*>(ws);
  double* pooled = slab + 7ll * chunks;
  if (chunks > 0) {
    nyu_errors_kernel<<<chunks, kNyuThreads, 0, st>>>(pred, gt, n, slab);
    if (int rc = launched()) return rc;
    nyu_slab_sum_kernel<<<1, 128, 0, st>>>(slab, 1, chunks, pooled);
  } else {
    cudaMemsetAsync(pooled, 0, 7 * sizeof(double), st);
  }
  if (int rc = launched()) return rc;
  nyu_errors_finish_kernel<<<1, 1, 0, st>>>(pooled, errors);
  return launched();
}
