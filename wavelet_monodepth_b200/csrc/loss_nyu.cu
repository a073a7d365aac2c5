// NYUv2's supervised training loss (NYUv2/train.py:279-327) on the device: the mean absolute difference between each
// prediction, upsampled by torch's align_corners bilinear rule, and the target, forward and backward (include/wmd_loss.h).
//
// Forward: one launch over the target grid samples every term at each target pixel, so the target is read once, and
// writes one fp64 partial per (term, CTA); a second launch adds each term's partials in CTA order.  The int8 signs of
// the differences are stored for the backward: a gather visits every target pixel about twice per axis and term, and a
// stored sign is one byte where recomputing it would re-read four taps and the target.
// Backward: one launch, one thread per low-resolution pixel of every term, sums its own footprint (gather form, no
// scatter, no atomics).  fp64 arithmetic is written with explicit _rn intrinsics so that FMA contraction cannot change a
// rounding; the fp32 weight rule with __f*_rn for the same reason.
#include <math.h>
#include "common.cuh"
#include "wmd_loss.h"

namespace wmd {

constexpr int kLossThreads = 256;
constexpr int kLossPerThread = WMD_LOSS_PIXELS_PER_CTA / kLossThreads;

struct LossTerm {
  const float* pred;
  float* grad;
  int h, w, log2_factor;
  float ry, rx;   // fp32 (in - 1) / (out - 1) per axis, 0 when out == 1
};
struct LossTable {
  LossTerm t[WMD_LOSS_MAX_TERMS];
  int n;
};

// torch's align_corners=True source taps of destination index d (UpSample.h: area_pixel_compute_scale,
// compute_source_index_and_lambda), with l0 = 1 - l1 taken exactly in fp64
struct LossTap {
  int i0, i1;
  double l0, l1;
};
__device__ __forceinline__ LossTap loss_tap(int d, int in, float r) {
  const float src = __fmul_rn(r, static_cast<float>(d));
  LossTap t;
  t.i0 = min(static_cast<int>(src), in - 1);
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  const float l1 = fminf(fmaxf(__fsub_rn(src, static_cast<float>(t.i0)), 0.f), 1.f);
  t.l1 = static_cast<double>(l1);
  t.l0 = __dadd_rn(1.0, -t.l1);
  return t;
}

// the weight with which destination d (tap t) reads source index i; false when it does not read i
__device__ __forceinline__ bool loss_weight(const LossTap& t, int i, double& wgt) {
  if (t.i0 != i && t.i1 != i) return false;
  wgt = t.i0 == i ? (t.i1 == i ? __dadd_rn(t.l0, t.l1) : t.l0) : t.l1;
  return true;
}

// destinations whose taps may read source index i: [lo, hi], a superset checked with loss_weight
__device__ __forceinline__ void loss_candidates(int i, int in, int out, int& lo, int& hi) {
  if (in == 1) {
    lo = 0;
    hi = out - 1;
    return;
  }
  const int q = in - 1, m = out - 1;
  const int a = (i - 1) * m;
  lo = max(0, (a >= 0 ? a / q : -((-a + q - 1) / q)) - 1);
  hi = min(m, (i + 1) * m / q + 1);
}

__global__ void __launch_bounds__(kLossThreads) loss_nyu_fwd_kernel(const float* __restrict__ target, int H, int W,
                                                                    long long total, LossTable tab,
                                                                    int8_t* __restrict__ signs,
                                                                    double* __restrict__ partial) {
  const long long plane = static_cast<long long>(H) * W;
  double acc[WMD_LOSS_MAX_TERMS] = {0.0, 0.0, 0.0, 0.0};
  const long long base = static_cast<long long>(blockIdx.x) * WMD_LOSS_PIXELS_PER_CTA + threadIdx.x;
#pragma unroll 1
  for (int j = 0; j < kLossPerThread; ++j) {
    const long long p = base + j * kLossThreads;
    if (p >= total) break;
    const int n = static_cast<int>(p / plane);
    const int rem = static_cast<int>(p - n * plane);
    const int Y = rem / W, X = rem % W;
    const double t = static_cast<double>(target[p]);
#pragma unroll
    for (int k = 0; k < WMD_LOSS_MAX_TERMS; ++k) {
      if (k < tab.n) {
        const LossTerm& T = tab.t[k];
        double sample;
        if (T.log2_factor == 0) {         // the identity: no neighbour is read, so none spreads a NaN
          sample = static_cast<double>(T.pred[p]);
        } else {
          const LossTap ty = loss_tap(Y, T.h, T.ry), tx = loss_tap(X, T.w, T.rx);
          const float* src = T.pred + static_cast<long long>(n) * T.h * T.w;
          const float* r0 = src + static_cast<long long>(ty.i0) * T.w;
          const float* r1 = src + static_cast<long long>(ty.i1) * T.w;
          const double a = r0[tx.i0], b = r0[tx.i1], c = r1[tx.i0], d = r1[tx.i1];
          const double top = __dadd_rn(__dmul_rn(tx.l0, a), __dmul_rn(tx.l1, b));
          const double bot = __dadd_rn(__dmul_rn(tx.l0, c), __dmul_rn(tx.l1, d));
          sample = __dadd_rn(__dmul_rn(ty.l0, top), __dmul_rn(ty.l1, bot));
        }
        const double diff = __dadd_rn(sample, -t);
        acc[k] = __dadd_rn(acc[k], fabs(diff));
        if (signs) signs[k * total + p] = static_cast<int8_t>((diff > 0.0) - (diff < 0.0));
      }
    }
  }
  __shared__ double red[WMD_LOSS_MAX_TERMS][kLossThreads];
#pragma unroll
  for (int k = 0; k < WMD_LOSS_MAX_TERMS; ++k) red[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int s = kLossThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
#pragma unroll
      for (int k = 0; k < WMD_LOSS_MAX_TERMS; ++k)
        red[k][threadIdx.x] = __dadd_rn(red[k][threadIdx.x], red[k][threadIdx.x + s]);
    }
    __syncthreads();
  }
  if (threadIdx.x < tab.n) partial[static_cast<long long>(threadIdx.x) * gridDim.x + blockIdx.x] = red[threadIdx.x][0];
}

// one CTA per term: the CTA partials in CTA order (thread t takes t, t + 256, ..., then a fixed tree), / (N H W)
__global__ void __launch_bounds__(kLossThreads) loss_nyu_mean_kernel(const double* __restrict__ partial, int ctas,
                                                                     long long total, float* __restrict__ means) {
  __shared__ double red[kLossThreads];
  const double* p = partial + static_cast<long long>(blockIdx.x) * ctas;
  double acc = 0.0;
  for (int b = threadIdx.x; b < ctas; b += kLossThreads) acc = __dadd_rn(acc, p[b]);
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = kLossThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) means[blockIdx.x] = __double2float_rn(__ddiv_rn(red[0], static_cast<double>(total)));
}

// blockIdx.y = term; one thread per pixel (n, y, x) of that term's prediction
__global__ void __launch_bounds__(kLossThreads) loss_nyu_bwd_kernel(const int8_t* __restrict__ signs, int N, int H,
                                                                    int W, LossTable tab,
                                                                    const float* __restrict__ grad_means) {
  const int k = blockIdx.y;
  const LossTerm& T = tab.t[k];
  const long long lplane = static_cast<long long>(T.h) * T.w;
  const long long p = static_cast<long long>(blockIdx.x) * kLossThreads + threadIdx.x;
  if (p >= N * lplane) return;
  const int n = static_cast<int>(p / lplane);
  const int rem = static_cast<int>(p - n * lplane);
  const int y = rem / T.w, x = rem % T.w;
  const long long plane = static_cast<long long>(H) * W;
  const int8_t* s = signs + (static_cast<long long>(k) * N + n) * plane;
  int ylo, yhi, xlo, xhi;
  loss_candidates(y, T.h, H, ylo, yhi);
  loss_candidates(x, T.w, W, xlo, xhi);
  double acc = 0.0;
  for (int Y = ylo; Y <= yhi; ++Y) {
    double wy;
    if (!loss_weight(loss_tap(Y, T.h, T.ry), y, wy)) continue;
    const int8_t* row = s + static_cast<long long>(Y) * W;
    double q = 0.0;                      // exact: the weights are multiples of 2^-27 and there are few of them
    for (int X = xlo; X <= xhi; ++X) {
      double wx;
      if (loss_weight(loss_tap(X, T.w, T.rx), x, wx)) q = __dadd_rn(q, __dmul_rn(static_cast<double>(row[X]), wx));
    }
    acc = __dadd_rn(acc, __dmul_rn(wy, q));
  }
  const double coef = __ddiv_rn(static_cast<double>(grad_means[k]), static_cast<double>(N * plane));
  T.grad[p] = __double2float_rn(__dmul_rn(coef, acc));
}

}  // namespace wmd

// ---------------------------------------------------------------------------------------- C ABI
namespace {
long long loss_total(int N, int H, int W) { return static_cast<long long>(N) * H * W; }
int loss_ctas(int N, int H, int W) { return wmd::ceil_div(loss_total(N, H, W), WMD_LOSS_PIXELS_PER_CTA); }

float loss_ratio(int in, int out) {
  return out > 1 ? static_cast<float>(in - 1) / static_cast<float>(out - 1) : 0.f;
}

// the argument checks both directions share; fills the kernel's table
int loss_table(int N, int H, int W, const wmd_loss_term* terms, int n_terms, wmd::LossTable& tab) {
  WMD_REQUIRE(terms, WMD_ERR_ARG);
  WMD_REQUIRE(n_terms >= 1 && n_terms <= WMD_LOSS_MAX_TERMS, WMD_ERR_SHAPE);
  WMD_REQUIRE(N >= 0 && N <= 65535 && H >= 1 && W >= 1, WMD_ERR_SHAPE);
  WMD_REQUIRE(loss_total(N, H, W) < (1ll << 31) / WMD_LOSS_MAX_TERMS, WMD_ERR_SHAPE);
  tab = wmd::LossTable{};
  tab.n = n_terms;
  for (int k = 0; k < n_terms; ++k) {
    const wmd_loss_term& t = terms[k];
    WMD_REQUIRE(t.log2_factor >= 0 && t.log2_factor <= 3 && t.h >= 1 && t.w >= 1, WMD_ERR_SHAPE);
    WMD_REQUIRE((static_cast<long long>(t.h) << t.log2_factor) == H, WMD_ERR_SHAPE);
    WMD_REQUIRE((static_cast<long long>(t.w) << t.log2_factor) == W, WMD_ERR_SHAPE);
    WMD_REQUIRE(N == 0 || t.pred, WMD_ERR_ARG);
    tab.t[k] = wmd::LossTerm{t.pred, nullptr, t.h, t.w, t.log2_factor, loss_ratio(t.h, H), loss_ratio(t.w, W)};
  }
  return WMD_OK;
}
}  // namespace

extern "C" size_t wmd_loss_nyu_ws_bytes(int N, int H, int W, int n_terms) {
  if (N < 0 || H < 1 || W < 1 || n_terms < 1 || n_terms > WMD_LOSS_MAX_TERMS) return 0;
  return static_cast<size_t>(loss_ctas(N, H, W)) * n_terms * sizeof(double);
}

extern "C" int wmd_loss_nyu_fwd(const float* target, int N, int H, int W, const wmd_loss_term* terms, int n_terms,
                                int8_t* signs, void* ws, size_t ws_bytes, float* means, wmd_stream_t stream) {
  using namespace wmd;
  LossTable tab;
  if (int rc = loss_table(N, H, W, terms, n_terms, tab)) return rc;
  WMD_REQUIRE(means && (N == 0 || (target && ws)), WMD_ERR_ARG);
  WMD_REQUIRE(ws_bytes >= wmd_loss_nyu_ws_bytes(N, H, W, n_terms), WMD_ERR_WORKSPACE);
  cudaStream_t st = as_stream(stream);
  const int ctas = loss_ctas(N, H, W);
  double* partial = static_cast<double*>(ws);
  if (ctas > 0) {
    loss_nyu_fwd_kernel<<<ctas, kLossThreads, 0, st>>>(target, H, W, loss_total(N, H, W), tab, signs, partial);
    if (int rc = launched()) return rc;
  }
  loss_nyu_mean_kernel<<<n_terms, kLossThreads, 0, st>>>(partial, ctas, loss_total(N, H, W), means);
  return launched();
}

extern "C" int wmd_loss_nyu_bwd(const int8_t* signs, int N, int H, int W, const wmd_loss_term* terms, int n_terms,
                                const float* grad_means, float* const* grads, wmd_stream_t stream) {
  using namespace wmd;
  LossTable tab;
  if (int rc = loss_table(N, H, W, terms, n_terms, tab)) return rc;
  WMD_REQUIRE(grads && grad_means && (N == 0 || signs), WMD_ERR_ARG);
  long long most = 0;
  for (int k = 0; k < n_terms; ++k) {
    WMD_REQUIRE(N == 0 || grads[k], WMD_ERR_ARG);
    tab.t[k].grad = grads[k];
    most = max(most, static_cast<long long>(N) * tab.t[k].h * tab.t[k].w);
  }
  if (N == 0) return WMD_OK;
  loss_nyu_bwd_kernel<<<dim3(ceil_div(most, kLossThreads), n_terms), kLossThreads, 0, as_stream(stream)>>>(
      signs, N, H, W, tab, grad_means);
  return launched();
}
