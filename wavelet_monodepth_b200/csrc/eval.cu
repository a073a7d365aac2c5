// KITTI depth evaluation (KITTI/evaluate_depth.py): valid-pixel masks of a ground-truth split, cv2-rule bilinear
// sampling of predicted disparities at those pixels, exact per-frame medians by radix select, the seven metrics, and
// Monodepth's flip post-processing.  Everything runs in fp64 with explicit _rn intrinsics where the reference's numpy /
// cv2 arithmetic has a fixed operation order, so nvcc's FMA contraction cannot change a rounding.
#include <math.h>
#include "common.cuh"
#include "wmd_eval.h"

namespace wmd {

constexpr int kEvalThreads = 512;

// ------------------------------------------------------------------------------------ valid-pixel mask
// evaluate_depth.py:283-293.  numpy 2 compares a float32 array with a Python float in float32 (NEP 50), so the depth
// range test is done on floats; the crop bounds are float64 products truncated to int32 (.astype(np.int32)).
__global__ void eval_gt_mask_kernel(const float* __restrict__ gt, const int32_t* __restrict__ hw,
                                    uint8_t* __restrict__ mask, int Hmax, int Wmax, int split) {
  const int f = blockIdx.y;
  const int H = hw[2 * f], W = hw[2 * f + 1];
  int y0 = 0, y1 = H, x0 = 0, x1 = W;
  if (split == WMD_EVAL_EIGEN) {
    y0 = static_cast<int>(__dmul_rn(0.40810811, H));
    y1 = static_cast<int>(__dmul_rn(0.99189189, H));
    x0 = static_cast<int>(__dmul_rn(0.03594771, W));
    x1 = static_cast<int>(__dmul_rn(0.96405229, W));
  }
  const long long plane = static_cast<long long>(Hmax) * Wmax;
  for (long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; p < plane;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(p / Wmax), x = static_cast<int>(p % Wmax);
    const float g = gt[f * plane + p];
    bool ok = y < H && x < W;
    if (split == WMD_EVAL_EIGEN)
      ok = ok && g > 1e-3f && g < 80.f && y >= y0 && y < y1 && x >= x0 && x < x1;
    else
      ok = ok && g > 0.f;
    mask[f * plane + p] = ok ? 1 : 0;
  }
}

__global__ void eval_gather_kernel(const float* __restrict__ src, const int32_t* __restrict__ pixels,
                                   const int32_t* __restrict__ count, int max_rows, float* __restrict__ out) {
  const int n = min(*count, max_rows);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = src[pixels[i]];
}

// ------------------------------------------------------------------------------------ cv2 INTER_LINEAR sampling
// cv2.resize's coordinate rule for one axis: f = (d + 0.5) src / dst - 0.5, s = floor(f), weight f - s; left of the
// first sample s = 0 with weight 0; at or past the last, s = src - 1 with weight 0.
struct Tap {
  int s, s1;
  double a;
  bool last;
};
__device__ __forceinline__ Tap axis_tap(int d, int src, int dst) {
  const double f = __dadd_rn(__dmul_rn(d + 0.5, __ddiv_rn(static_cast<double>(src), static_cast<double>(dst))), -0.5);
  const double fl = floor(f);
  Tap t;
  t.s = static_cast<int>(fl);
  t.a = __dadd_rn(f, -fl);
  t.last = false;
  if (t.s < 0) { t.s = 0; t.a = 0.0; }
  if (t.s >= src - 1) { t.s = src - 1; t.a = 0.0; t.last = true; }
  t.s1 = min(t.s + 1, src - 1);
  return t;
}

template <typename T>
__device__ __forceinline__ double lerp2(const T* row, const Tap& tx) {
  // horizontal pass: the last column is copied (one tap); elsewhere both taps are weighted, a zero weight included
  const double v0 = static_cast<double>(row[tx.s]);
  if (tx.last) return v0;
  return __dadd_rn(__dmul_rn(v0, __dadd_rn(1.0, -tx.a)), __dmul_rn(static_cast<double>(row[tx.s1]), tx.a));
}

// depth = (1 / disp) * scale_factor at ground-truth pixel (y, x) of an H x W frame, disp an h x w plane
template <typename T>
__device__ __forceinline__ double sample_depth(const T* plane, int h, int w, int H, int W, int y, int x, double sf) {
  const Tap tx = axis_tap(x, w, W), ty = axis_tap(y, h, H);
  const double r0 = lerp2(plane + static_cast<long long>(ty.s) * w, tx);
  const double r1 = lerp2(plane + static_cast<long long>(ty.s1) * w, tx);
  const double v = __dadd_rn(__dmul_rn(r0, __dadd_rn(1.0, -ty.a)), __dmul_rn(r1, ty.a));
  return __dmul_rn(__ddiv_rn(1.0, v), sf);
}

// ------------------------------------------------------------------------------------ exact median
// Order-preserving key of a double: unsigned order of keys == numeric order (-Inf < ... < -0 < +0 < ... < +Inf).
__device__ __forceinline__ unsigned long long okey(double v) {
  const unsigned long long u = static_cast<unsigned long long>(__double_as_longlong(v));
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double unkey(unsigned long long k) {
  const unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
  return __longlong_as_double(static_cast<long long>(u));
}

struct SelectSmem {
  unsigned hist[256];
  unsigned digit, rank;
};

// k-th smallest (0-based) of n values, by eight 8-bit digit passes over the keys: a 256-bin shared histogram of the
// keys that match the digits found so far, then one warp finds the bin that holds rank k.  Exact; the whole CTA calls it.
template <class Load>
__device__ double select_kth(Load load, int n, unsigned k, SelectSmem& sm) {
  unsigned long long prefix = 0, pmask = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sm.hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned long long key = okey(load(i));
      if ((key & pmask) == prefix) atomicAdd(&sm.hist[(key >> shift) & 255], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      unsigned c[8], s = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c[j] = sm.hist[lane * 8 + j]; s += c[j]; }
      unsigned incl = s;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      unsigned before = incl - s;
      if (k >= before && k < incl) {
        int j = 0;
        while (k >= before + c[j]) before += c[j++];
        sm.digit = lane * 8 + j;
        sm.rank = k - before;
      }
    }
    __syncthreads();
    prefix |= static_cast<unsigned long long>(sm.digit) << shift;
    pmask |= 0xffull << shift;
    k = sm.rank;
    __syncthreads();
  }
  return unkey(prefix);
}

// np.median: the middle value, or the mean of the two middle values (in the array's own precision: float32 ground
// truth averages in float32); NaN if any value is NaN or there are none.
template <bool kF32, class Load>
__device__ double median(Load load, int n, SelectSmem& sm) {
  bool nan = false;
  for (int i = threadIdx.x; i < n; i += blockDim.x) nan |= isnan(load(i));
  nan = __syncthreads_or(nan);
  if (n == 0 || nan) return __longlong_as_double(0x7ff8000000000000ll);
  const unsigned k = static_cast<unsigned>(n - 1) / 2;
  const double a = select_kth(load, n, k, sm);
  if (n & 1) return a;
  const double b = select_kth(load, n, k + 1, sm);
  if (kF32) return static_cast<double>(__fdiv_rn(__fadd_rn(static_cast<float>(a), static_cast<float>(b)), 2.f));
  return __ddiv_rn(__dadd_rn(a, b), 2.0);
}

// ------------------------------------------------------------------------------------ metrics
// compute_errors (evaluate_depth.py:50-68) on one (gt, pred) pixel, accumulated into per-thread sums.
struct ErrSums {
  double abs_rel, sq_rel, sq, sq_log;
  unsigned a1, a2, a3;
};
__device__ __forceinline__ void accumulate(ErrSums& e, double g, double lg, double p) {
  const double q0 = __ddiv_rn(g, p), q1 = __ddiv_rn(p, g);
  const double t = (isnan(q0) || isnan(q1)) ? q0 + q1 : fmax(q0, q1);     // np.maximum propagates NaN
  e.a1 += t < 1.25;
  e.a2 += t < 1.5625;
  e.a3 += t < 1.953125;
  const double d = __dadd_rn(g, -p);
  const double d2 = __dmul_rn(d, d);
  e.sq = __dadd_rn(e.sq, d2);
  const double dl = __dadd_rn(lg, -log(p));
  e.sq_log = __dadd_rn(e.sq_log, __dmul_rn(dl, dl));
  e.abs_rel = __dadd_rn(e.abs_rel, __ddiv_rn(fabs(d), g));
  e.sq_rel = __dadd_rn(e.sq_rel, __ddiv_rn(d2, g));
}

// fixed-order tree reduction of the per-thread sums, then the seven means (0 pixels: 0 / 0 = NaN, as np.mean gives)
__device__ void finish_errors(ErrSums e, int n, double* __restrict__ out) {
  __shared__ double sd[4][kEvalThreads];
  __shared__ unsigned su[3][kEvalThreads];
  const int t = threadIdx.x;
  sd[0][t] = e.abs_rel; sd[1][t] = e.sq_rel; sd[2][t] = e.sq; sd[3][t] = e.sq_log;
  su[0][t] = e.a1; su[1][t] = e.a2; su[2][t] = e.a3;
  __syncthreads();
  for (int s = kEvalThreads / 2; s > 0; s >>= 1) {
    if (t < s) {
#pragma unroll
      for (int j = 0; j < 4; ++j) sd[j][t] = __dadd_rn(sd[j][t], sd[j][t + s]);
#pragma unroll
      for (int j = 0; j < 3; ++j) su[j][t] += su[j][t + s];
    }
    __syncthreads();
  }
  if (t == 0) {
    const double dn = static_cast<double>(n);
    out[0] = __ddiv_rn(sd[0][0], dn);
    out[1] = __ddiv_rn(sd[1][0], dn);
    out[2] = sqrt(__ddiv_rn(sd[2][0], dn));
    out[3] = sqrt(__ddiv_rn(sd[3][0], dn));
    out[4] = __ddiv_rn(static_cast<double>(su[0][0]), dn);
    out[5] = __ddiv_rn(static_cast<double>(su[1][0]), dn);
    out[6] = __ddiv_rn(static_cast<double>(su[2][0]), dn);
  }
}

// One CTA per frame f = frame0 + blockIdx.x: evaluate_depth.py:276-307 for that frame.
template <typename T>
__global__ void __launch_bounds__(kEvalThreads) eval_frames_kernel(
    const T* __restrict__ disp, int h, int w, int frame0, const int32_t* __restrict__ hw,
    const int32_t* __restrict__ pixels, const int32_t* __restrict__ offsets, const float* __restrict__ gt,
    const float* __restrict__ gt_log, int Hmax, int Wmax, double sf, int median_scaling, double* __restrict__ depth,
    double* __restrict__ errors, double* __restrict__ ratio, int32_t* __restrict__ count) {
  __shared__ SelectSmem sm;
  const int j = blockIdx.x, f = frame0 + j;
  const int beg = offsets[f], n = offsets[f + 1] - beg;
  const int H = hw[2 * f], W = hw[2 * f + 1];
  const long long plane = static_cast<long long>(Hmax) * Wmax;
  const T* src = disp + static_cast<long long>(j) * h * w;
  const float* g = gt + beg;
  double* dp = depth + beg;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const long long p = pixels[beg + i] - f * plane;
    dp[i] = sample_depth(src, h, w, H, W, static_cast<int>(p / Wmax), static_cast<int>(p % Wmax), sf);
  }
  __syncthreads();
  double r = 1.0;
  if (median_scaling) {
    const double mg = median<true>([=](int i) { return static_cast<double>(g[i]); }, n, sm);
    const double mp = median<false>([=](int i) { return dp[i]; }, n, sm);
    r = __ddiv_rn(mg, mp);
  }
  ErrSums e = {0.0, 0.0, 0.0, 0.0, 0u, 0u, 0u};
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double p = median_scaling ? __dmul_rn(dp[i], r) : dp[i];
    if (p < 1e-3) p = 1e-3;                     // boolean assignments: NaN stays NaN
    if (p > 80.0) p = 80.0;
    const double gv = static_cast<double>(g[i]);
    accumulate(e, gv, gt_log ? static_cast<double>(gt_log[beg + i]) : log(gv), p);
  }
  finish_errors(e, n, errors + 7ll * j);
  if (threadIdx.x == 0) {
    ratio[j] = r;
    count[j] = n;
  }
}

__global__ void __launch_bounds__(kEvalThreads) eval_errors_kernel(const double* __restrict__ gt,
                                                                   const double* __restrict__ pred, int n,
                                                                   double* __restrict__ out) {
  ErrSums e = {0.0, 0.0, 0.0, 0.0, 0u, 0u, 0u};
  for (int i = threadIdx.x; i < n; i += blockDim.x) accumulate(e, gt[i], log(gt[i]), pred[i]);
  finish_errors(e, n, out);
}

// ------------------------------------------------------------------------------------ flip post-processing
// evaluate_depth.py:71-79.  l = linspace(0, 1, w) as numpy forms it (x * (1 / (w - 1)), the last entry exactly 1);
// m_disp = 0.5 (l + r) is computed in the inputs' precision, as numpy does for float32 arrays.
template <typename T>
__global__ void post_process_kernel(const T* __restrict__ l, const T* __restrict__ r, double* __restrict__ out,
                                    long long total, int w) {
  const double step = w > 1 ? __ddiv_rn(1.0, static_cast<double>(w - 1)) : 0.0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % w);
    auto lmask = [&](int c) {
      const double lin = (w > 1 && c == w - 1) ? 1.0 : __dmul_rn(static_cast<double>(c), step);
      const double v = __dmul_rn(20.0, __dadd_rn(lin, -0.05));
      return __dadd_rn(1.0, -fmin(fmax(v, 0.0), 1.0));
    };
    const double lm = lmask(x), rm = lmask(w - 1 - x);
    const T lv = l[i], rv = r[i];
    const double m = static_cast<double>(static_cast<T>(static_cast<T>(0.5) * static_cast<T>(lv + rv)));
    const double a = __dadd_rn(__dmul_rn(rm, static_cast<double>(lv)), __dmul_rn(lm, static_cast<double>(rv)));
    out[i] = __dadd_rn(a, __dmul_rn(__dadd_rn(__dadd_rn(1.0, -lm), -rm), m));
  }
}

}  // namespace wmd

// ---------------------------------------------------------------------------------------- C ABI
extern "C" int wmd_eval_gt_mask(const float* gt, const int32_t* hw, uint8_t* mask, int N, int Hmax, int Wmax, int split,
                                wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(N >= 0 && Hmax > 0 && Wmax > 0 && N <= 65535, WMD_ERR_SHAPE);
  WMD_REQUIRE(split == WMD_EVAL_EIGEN || split == WMD_EVAL_GT_POSITIVE, WMD_ERR_ARG);
  if (N == 0) return WMD_OK;
  WMD_REQUIRE(gt && hw && mask, WMD_ERR_ARG);
  const long long plane = static_cast<long long>(Hmax) * Wmax;
  dim3 grid(ceil_div(plane, 256) < 1024 ? ceil_div(plane, 256) : 1024, N);
  eval_gt_mask_kernel<<<grid, 256, 0, as_stream(stream)>>>(gt, hw, mask, Hmax, Wmax, split);
  return launched();
}

extern "C" int wmd_eval_gather_f32(const float* src, const int32_t* pixels, const int32_t* count, int max_rows,
                                   float* out, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src && pixels && count && out, WMD_ERR_ARG);
  WMD_REQUIRE(max_rows >= 0, WMD_ERR_SHAPE);
  if (max_rows == 0) return WMD_OK;
  eval_gather_kernel<<<stride_grid(max_rows, 256), 256, 0, as_stream(stream)>>>(src, pixels, count, max_rows, out);
  return launched();
}

extern "C" int wmd_eval_frames(const void* disp, int disp_f64, int n, int h, int w, int frame0, const int32_t* hw,
                               const int32_t* pixels, const int32_t* offsets, const float* gt, const float* gt_log,
                               int Hmax, int Wmax, double scale_factor, int median_scaling, double* depth,
                               double* errors, double* ratio, int32_t* count, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(n >= 0 && frame0 >= 0 && h > 0 && w > 0 && Hmax > 0 && Wmax > 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(Hmax) * Wmax * (frame0 + static_cast<long long>(n)) < (1ll << 31), WMD_ERR_SHAPE);
  if (n == 0) return WMD_OK;
  WMD_REQUIRE(disp && hw && pixels && offsets && gt && depth && errors && ratio && count, WMD_ERR_ARG);
  if (disp_f64)
    eval_frames_kernel<double><<<n, kEvalThreads, 0, as_stream(stream)>>>(
        static_cast<const double*>(disp), h, w, frame0, hw, pixels, offsets, gt, gt_log, Hmax, Wmax, scale_factor,
        median_scaling, depth, errors, ratio, count);
  else
    eval_frames_kernel<float><<<n, kEvalThreads, 0, as_stream(stream)>>>(
        static_cast<const float*>(disp), h, w, frame0, hw, pixels, offsets, gt, gt_log, Hmax, Wmax, scale_factor,
        median_scaling, depth, errors, ratio, count);
  return launched();
}

extern "C" int wmd_eval_errors_f64(const double* gt, const double* pred, int n, double* errors, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(n >= 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(errors && (n == 0 || (gt && pred)), WMD_ERR_ARG);
  eval_errors_kernel<<<1, kEvalThreads, 0, as_stream(stream)>>>(gt, pred, n, errors);
  return launched();
}

extern "C" int wmd_post_process_disparity(const void* l_disp, const void* r_disp, int in_f64, double* out, int N, int h,
                                          int w, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(N >= 0 && h > 0 && w > 0, WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  WMD_REQUIRE(l_disp && r_disp && out, WMD_ERR_ARG);
  const long long total = static_cast<long long>(N) * h * w;
  if (in_f64)
    post_process_kernel<double><<<stride_grid(total, 256), 256, 0, as_stream(stream)>>>(
        static_cast<const double*>(l_disp), static_cast<const double*>(r_disp), out, total, w);
  else
    post_process_kernel<float><<<stride_grid(total, 256), 256, 0, as_stream(stream)>>>(
        static_cast<const float*>(l_disp), static_cast<const float*>(r_disp), out, total, w);
  return launched();
}
