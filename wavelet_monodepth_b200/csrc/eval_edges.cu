// NYUv2 depth boundary error (NYUv2/utils.py: compute_depth_boundary_error, with scikit-image 0.16.2's canny and
// scipy's distance_transform_edt) for a batch of frames.  The arithmetic follows oracle/nyu_edges.py's restatements of
// the scipy filters and glibc's hypot, with explicit _rn intrinsics so that nvcc's FMA contraction cannot change a
// rounding; a one-ulp change in the magnitude can flip a non-maximum-suppression comparison.
//
// Launches per batch: each frame's nanmin / max - min; one tiled kernel for normalise -> gaussian -> divide -> sobel ->
// hypot -> non-maximum suppression, writing a low / high bit per pixel; union-find hysteresis (init, merge, compress,
// mark, output); the exact EDT of the Canny edges (column pass, row pass); one CTA per (band of rows, frame) for the
// score sums and one thread per frame that adds the bands in order and writes the scores.  The union-find uses atomics,
// but its result is a set (the components of `low` that hold a `high` pixel), so its bits do not depend on timing; the
// sums use none.
#include <climits>
#include <math.h>
#include <math_constants.h>
#include "common.cuh"
#include "wmd_eval.h"

namespace wmd {

constexpr int kEdgeR = 6;                         // gaussian radius: int(4 * sqrt(2) + 0.5)
constexpr int kEdgeTile = 32;                     // output pixels per tile side
constexpr int kEdgeThreads = 256;
constexpr int kEdgePH = kEdgeTile + 2 * (kEdgeR + 2);   // normalised input rows / columns: halo 6 + 1 + 1
constexpr int kEdgeSH = kEdgeTile + 4;                  // smoothed rows / columns: halo 1 + 1
constexpr int kEdgeMH = kEdgeTile + 2;                  // magnitude rows / columns: halo 1
constexpr int kEdgeBandRows = 8;
constexpr int kEdgeNone = 0x3fffffff;              // no feature in the column
constexpr double kEdgeMaxDist = 10.0;              // utils.py:144
constexpr double kDblEps = 2.220446049250313e-16;  // np.finfo(float).eps

// ------------------------------------------------------------------------------------ normalise
__device__ __forceinline__ float edge_load(const void* pred, int pred_f64, long long i) {
  return pred_f64 ? __double2float_rn(static_cast<const double*>(pred)[i]) : static_cast<const float*>(pred)[i];
}

// per frame: mm[f] = (nanmin p, fl(nanmax p - nanmin p)) over the non-zero pixels, in float32.  np.nanmax(p - min)
// equals fl(max - min) because rounding is monotonic.  An all-zero / all-NaN frame gives NaN, as numpy does.
__global__ void __launch_bounds__(kEdgeThreads) edge_minmax_kernel(const void* __restrict__ pred, int pred_f64,
                                                                   int hw, float2* __restrict__ mm) {
  __shared__ float smin[kEdgeThreads], smax[kEdgeThreads];
  const long long base = static_cast<long long>(blockIdx.x) * hw;
  float lo = __int_as_float(0x7fc00000), hi = lo;
  for (int p = threadIdx.x; p < hw; p += blockDim.x) {
    const float v = edge_load(pred, pred_f64, base + p);
    if (v != 0.0f) {                               // p[p == 0] = NaN; fminf / fmaxf skip NaN
      lo = fminf(lo, v);
      hi = fmaxf(hi, v);
    }
  }
  smin[threadIdx.x] = lo;
  smax[threadIdx.x] = hi;
  __syncthreads();
  for (int k = kEdgeThreads / 2; k > 0; k >>= 1) {
    if (threadIdx.x < k) {
      smin[threadIdx.x] = fminf(smin[threadIdx.x], smin[threadIdx.x + k]);
      smax[threadIdx.x] = fmaxf(smax[threadIdx.x], smax[threadIdx.x + k]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) mm[blockIdx.x] = make_float2(smin[0], __fsub_rn(smax[0], smin[0]));
}

// ------------------------------------------------------------------------------------ canny
// glibc e_hypot.c, the kernel without FMA (what np.hypot reaches), for finite inputs
__device__ __forceinline__ double hypot_kernel(double ax, double ay) {
  double h = __dsqrt_rn(__dadd_rn(__dmul_rn(ax, ax), __dmul_rn(ay, ay)));
  double t1, t2;
  if (h <= __dmul_rn(2.0, ay)) {
    const double delta = __dadd_rn(h, -ay);
    t1 = __dmul_rn(ax, __dadd_rn(__dmul_rn(2.0, delta), -ax));
    t2 = __dmul_rn(__dadd_rn(delta, -__dmul_rn(2.0, __dadd_rn(ax, -ay))), delta);
  } else {
    const double delta = __dadd_rn(h, -ax);
    t1 = __dmul_rn(__dmul_rn(2.0, delta), __dadd_rn(ax, -__dmul_rn(2.0, ay)));
    t2 = __dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(4.0, delta), -ay), ay), __dmul_rn(delta, delta));
  }
  return __dadd_rn(h, -__ddiv_rn(__dadd_rn(t1, t2), __dmul_rn(2.0, h)));
}

__device__ double hypot_glibc(double x, double y) {
  if (!isfinite(x) || !isfinite(y)) return (isinf(x) || isinf(y)) ? CUDART_INF : __dadd_rn(x, y);
  x = fabs(x);
  y = fabs(y);
  const double ax = x < y ? y : x, ay = x < y ? x : y;
  const double kScale = 0x1p-600, kLarge = 0x1p+511, kTiny = 0x1p-511, kEps = 0x1p-54;
  if (ax > kLarge) {
    if (ay <= __dmul_rn(ax, kEps)) return __dadd_rn(ax, ay);
    return __ddiv_rn(hypot_kernel(__dmul_rn(ax, kScale), __dmul_rn(ay, kScale)), kScale);
  }
  if (ay < kTiny) {
    if (ax >= __ddiv_rn(ay, kEps)) return __dadd_rn(ax, ay);
    return __dmul_rn(hypot_kernel(__ddiv_rn(ax, kScale), __ddiv_rn(ay, kScale)), kScale);
  }
  if (ay <= __dmul_rn(ax, kEps)) return __dadd_rn(ax, ay);
  return hypot_kernel(ax, ay);
}

// scipy's symmetric correlate1d in double: t = x[0] w0, then t += (x[-j] + x[+j]) wj for j = 6 .. 1
__device__ __forceinline__ double gauss13(const float* x, int stride, const double* w) {
  double t = __dmul_rn(static_cast<double>(x[0]), w[0]);
#pragma unroll
  for (int j = kEdgeR; j >= 1; --j)
    t = __dadd_rn(t, __dmul_rn(__dadd_rn(static_cast<double>(x[-j * stride]), static_cast<double>(x[j * stride])),
                               w[j]));
  return t;
}

// the c2 w + c1 (1 - w) <= m test of one side
__device__ __forceinline__ bool nms_side(double c1, double c2, double w, double m) {
  return __dadd_rn(__dmul_rn(c2, w), __dmul_rn(c1, __dadd_rn(1.0, -w))) <= m;
}

// one CTA per (32 x 32 tile, frame): bits[i] = low | high << 1 (both only at local maxima of the eroded mask)
__global__ void __launch_bounds__(kEdgeThreads) edge_canny_kernel(
    const void* __restrict__ pred, int pred_f64, int H, int W, const float2* __restrict__ mm,
    const double* __restrict__ taps, const double* __restrict__ bleed, double low, double high,
    uint8_t* __restrict__ bits) {
  __shared__ float P[kEdgePH][kEdgePH];           // normalised input, 0 outside the frame (mode 'constant')
  __shared__ float G[kEdgeSH][kEdgePH];           // float32 result of the axis-0 pass
  __shared__ double S[kEdgeSH][kEdgeSH];          // smoothed, in the frame only
  __shared__ double M[kEdgeMH][kEdgeMH];          // magnitude, in the frame only
  __shared__ double w[kEdgeR + 1];
  const int f = blockIdx.z, y0 = blockIdx.y * kEdgeTile, x0 = blockIdx.x * kEdgeTile;
  const long long base = static_cast<long long>(f) * H * W;
  const float mn = mm[f].x, mx = mm[f].y;
  if (threadIdx.x <= kEdgeR) w[threadIdx.x] = taps[threadIdx.x];
  for (int k = threadIdx.x; k < kEdgePH * kEdgePH; k += blockDim.x) {
    const int r = k / kEdgePH, c = k % kEdgePH, y = y0 - kEdgeR - 2 + r, x = x0 - kEdgeR - 2 + c;
    float v = 0.0f;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      v = edge_load(pred, pred_f64, base + static_cast<long long>(y) * W + x);
      v = v == 0.0f ? __int_as_float(0x7fc00000) : __fdiv_rn(__fsub_rn(v, mn), mx);
    }
    P[r][c] = v;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kEdgeSH * kEdgePH; k += blockDim.x) {
    const int r = k / kEdgePH, c = k % kEdgePH, x = x0 - kEdgeR - 2 + c;
    G[r][c] = x >= 0 && x < W ? __double2float_rn(gauss13(&P[r + kEdgeR][c], kEdgePH, w)) : 0.0f;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kEdgeSH * kEdgeSH; k += blockDim.x) {
    const int r = k / kEdgeSH, c = k % kEdgeSH, y = y0 - 2 + r, x = x0 - 2 + c;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      const float sm = __double2float_rn(gauss13(&G[r][c + kEdgeR], 1, w));
      S[r][c] = __ddiv_rn(static_cast<double>(sm), __dadd_rn(bleed[static_cast<long long>(y) * W + x], kDblEps));
    }
  }
  __syncthreads();
  // ndi.sobel with mode 'reflect' (a radius-1 filter reads the edge pixel again): axis 0 is
  // d = 0 s + (s[y+1] - s[y-1]), then 2 d + (d[x-1] + d[x+1]); axis 1 the same with the axes swapped
  auto s_at = [&](int y, int x) { return S[y - y0 + 2][x - x0 + 2]; };
  auto sobel = [&](int y, int x, double& I, double& J) {
    const int ym = max(y - 1, 0), yp = min(y + 1, H - 1), xm = max(x - 1, 0), xp = min(x + 1, W - 1);
    auto d0 = [&](int xx) { return __dadd_rn(__dmul_rn(0.0, s_at(y, xx)), __dadd_rn(s_at(yp, xx), -s_at(ym, xx))); };
    auto d1 = [&](int yy) { return __dadd_rn(__dmul_rn(0.0, s_at(yy, x)), __dadd_rn(s_at(yy, xp), -s_at(yy, xm))); };
    I = __dadd_rn(__dmul_rn(d0(x), 2.0), __dadd_rn(d0(xm), d0(xp)));
    J = __dadd_rn(__dmul_rn(d1(y), 2.0), __dadd_rn(d1(ym), d1(yp)));
  };
  for (int k = threadIdx.x; k < kEdgeMH * kEdgeMH; k += blockDim.x) {
    const int r = k / kEdgeMH, c = k % kEdgeMH, y = y0 - 1 + r, x = x0 - 1 + c;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      double I, J;
      sobel(y, x, I, J);
      M[r][c] = hypot_glibc(I, J);
    }
  }
  __syncthreads();
  auto m_at = [&](int y, int x) { return M[y - y0 + 1][x - x0 + 1]; };
  for (int k = threadIdx.x; k < kEdgeTile * kEdgeTile; k += blockDim.x) {
    const int y = y0 + k / kEdgeTile, x = x0 + k % kEdgeTile;
    if (y >= H || x >= W) continue;
    uint8_t out = 0;
    const double m = m_at(y, x);
    if (y >= 1 && y < H - 1 && x >= 1 && x < W - 1 && m > 0.0) {    // the eroded mask
      double I, J;
      sobel(y, x, I, J);
      const double aI = fabs(I), aJ = fabs(J);
      bool lm = false;
      // skimage 0.16.2's four octants in its order; where they overlap (ties) the later one's assignment stands
      if (((I >= 0 && J >= 0) || (I <= 0 && J <= 0)) && aI >= aJ) {      // 0 - 45 degrees
        const double q = __ddiv_rn(aJ, aI);
        lm = nms_side(m_at(y + 1, x), m_at(y + 1, x + 1), q, m) && nms_side(m_at(y - 1, x), m_at(y - 1, x - 1), q, m);
      }
      if (((I >= 0 && J >= 0) || (I <= 0 && J <= 0)) && aI <= aJ) {      // 45 - 90
        const double q = __ddiv_rn(aI, aJ);
        lm = nms_side(m_at(y, x + 1), m_at(y + 1, x + 1), q, m) && nms_side(m_at(y, x - 1), m_at(y - 1, x - 1), q, m);
      }
      if (((I <= 0 && J >= 0) || (I >= 0 && J <= 0)) && aI <= aJ) {      // 90 - 135
        const double q = __ddiv_rn(aI, aJ);
        lm = nms_side(m_at(y, x + 1), m_at(y - 1, x + 1), q, m) && nms_side(m_at(y, x - 1), m_at(y + 1, x - 1), q, m);
      }
      if (((I <= 0 && J >= 0) || (I >= 0 && J <= 0)) && aI >= aJ) {      // 135 - 180
        const double q = __ddiv_rn(aJ, aI);
        lm = nms_side(m_at(y - 1, x), m_at(y - 1, x + 1), q, m) && nms_side(m_at(y + 1, x), m_at(y + 1, x - 1), q, m);
      }
      if (lm) out = (m >= low ? 1 : 0) | (m >= high ? 2 : 0);
    }
    bits[base + static_cast<long long>(y) * W + x] = out;
  }
}

// ------------------------------------------------------------------------------------ hysteresis (union-find)
// label[i] <= i always points into i's own component; the atomicMin union keeps that, so find walks to the root.
__device__ __forceinline__ int uf_find(const int* L, int x) {
  int y;
  while ((y = __ldcg(L + x)) != x) x = y;
  return x;
}

__device__ void uf_union(int* L, int a, int b) {
  bool done;
  do {
    a = uf_find(L, a);
    b = uf_find(L, b);
    if (a < b) {
      const int old = atomicMin(L + b, a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const int old = atomicMin(L + a, b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  } while (!done);
}

__global__ void edge_uf_init_kernel(const uint8_t* __restrict__ bits, int total, int* __restrict__ L,
                                    uint8_t* __restrict__ hit) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    L[i] = bits[i] & 1 ? i : -1;
    hit[i] = 0;
  }
}

// 8-connectivity (ndi.label with a 3 x 3 structure): each low pixel joins its low neighbours above and to the left
__global__ void edge_uf_merge_kernel(const uint8_t* __restrict__ bits, int H, int W, int total, int* L) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    if (!(bits[i] & 1)) continue;
    const int p = i % (H * W), y = p / W, x = p % W;
    if (x > 0 && (bits[i - 1] & 1)) uf_union(L, i, i - 1);
    if (y > 0) {
      if (x > 0 && (bits[i - W - 1] & 1)) uf_union(L, i, i - W - 1);
      if (bits[i - W] & 1) uf_union(L, i, i - W);
      if (x < W - 1 && (bits[i - W + 1] & 1)) uf_union(L, i, i - W + 1);
    }
  }
}

// every low pixel points at its root; a high pixel marks its root
__global__ void edge_uf_compress_kernel(const uint8_t* __restrict__ bits, int total, int* L, uint8_t* hit) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    if (!(bits[i] & 1)) continue;
    const int r = uf_find(L, i);
    L[i] = r;
    if (bits[i] & 2) hit[r] = 1;
  }
}

__global__ void edge_uf_output_kernel(const uint8_t* __restrict__ bits, int total, const int* __restrict__ L,
                                      const uint8_t* __restrict__ hit, uint8_t* __restrict__ edges) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x)
    edges[i] = (bits[i] & 1) && hit[L[i]] ? 1 : 0;
}

// ------------------------------------------------------------------------------------ exact EDT
// one thread per (column, frame): g = rows to the nearest feature in the column (kEdgeNone: none); any[f] = 1 when
// frame f has a feature (a plain store of 1 from any thread, so the result does not depend on timing)
__global__ void edt_column_kernel(const uint8_t* __restrict__ feat, int n, int H, int W, int* __restrict__ g,
                                  int* __restrict__ any) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n * W) return;
  const int f = k / W, x = k % W;
  const long long base = static_cast<long long>(f) * H * W + x;
  int last = -1;
  bool seen = false;
  for (int y = 0; y < H; ++y) {
    if (feat[base + static_cast<long long>(y) * W]) last = y, seen = true;
    g[base + static_cast<long long>(y) * W] = last < 0 ? kEdgeNone : y - last;
  }
  last = -1;
  for (int y = H - 1; y >= 0; --y) {
    const long long i = base + static_cast<long long>(y) * W;
    if (feat[i]) last = y;
    if (last >= 0 && last - y < g[i]) g[i] = last - y;
  }
  if (seen) any[f] = 1;
}

// one CTA per (row, frame): d^2 = min over columns k of (x - k)^2 + g[k]^2, searched outwards from x until (x - k)^2
// alone reaches the best; dist = sqrt(d^2), correctly rounded as scipy's.  A frame with no feature at all gets
// scipy's result for that case, sqrt((y + 1)^2 + x^2).
__global__ void edt_row_kernel(const int* __restrict__ g, const int* __restrict__ any, int H, int W,
                               double* __restrict__ dist) {
  const int y = blockIdx.x, f = blockIdx.y;
  const long long row = (static_cast<long long>(f) * H + y) * W;
  const bool has = any[f] != 0;
  for (int x = threadIdx.x; x < W; x += blockDim.x) {
    long long best;
    if (!has) {
      best = static_cast<long long>(y + 1) * (y + 1) + static_cast<long long>(x) * x;
    } else {
      best = LLONG_MAX;
      const int reach = max(x, W - 1 - x);
      for (int d = 0; d <= reach && static_cast<long long>(d) * d < best; ++d) {
        const long long dd = static_cast<long long>(d) * d;
        if (x - d >= 0) {
          const int v = g[row + x - d];
          if (v != kEdgeNone) best = min(best, dd + static_cast<long long>(v) * v);
        }
        if (d > 0 && x + d < W) {
          const int v = g[row + x + d];
          if (v != kEdgeNone) best = min(best, dd + static_cast<long long>(v) * v);
        }
      }
    }
    dist[row + x] = __dsqrt_rn(static_cast<double>(best));
  }
}

// ------------------------------------------------------------------------------------ scores
// one CTA per (band of rows, frame) -> slab[f][band][5] = (|est|, |near|, sum_near D_gt, sum_est min(D_gt, 10),
// nansum min(D_est w, 10)), each a fixed tree over the CTA's threads
__global__ void __launch_bounds__(kEdgeThreads) edge_score_band_kernel(
    const uint8_t* __restrict__ est, const double* __restrict__ d_est, const float* __restrict__ edges_gt,
    const double* __restrict__ d_gt, int H, int W, double* __restrict__ slab) {
  __shared__ double sd[3][kEdgeThreads];
  __shared__ unsigned su[2][kEdgeThreads];
  const int band = blockIdx.x, f = blockIdx.y, t = threadIdx.x;
  const int r0 = band * kEdgeBandRows, r1 = min(r0 + kEdgeBandRows, H);
  const long long base = static_cast<long long>(f) * H * W;
  double s_near = 0.0, s_est = 0.0, s_gt = 0.0;
  unsigned n_est = 0, n_near = 0;
  for (int p = r0 * W + t; p < r1 * W; p += blockDim.x) {
    const long long i = base + p;
    const double dg = d_gt[i];
    if (est[i]) {
      ++n_est;
      s_est = __dadd_rn(s_est, dg > kEdgeMaxDist ? kEdgeMaxDist : dg);
      if (dg < kEdgeMaxDist) {
        ++n_near;
        s_near = __dadd_rn(s_near, dg);
      }
    }
    double c = __dmul_rn(d_est[i], static_cast<double>(edges_gt[i]));
    if (c > kEdgeMaxDist) c = kEdgeMaxDist;
    if (!isnan(c)) s_gt = __dadd_rn(s_gt, c);
  }
  sd[0][t] = s_near; sd[1][t] = s_est; sd[2][t] = s_gt;
  su[0][t] = n_est; su[1][t] = n_near;
  __syncthreads();
  for (int k = kEdgeThreads / 2; k > 0; k >>= 1) {
    if (t < k) {
#pragma unroll
      for (int j = 0; j < 3; ++j) sd[j][t] = __dadd_rn(sd[j][t], sd[j][t + k]);
      su[0][t] += su[0][t + k];
      su[1][t] += su[1][t + k];
    }
    __syncthreads();
  }
  double* out = slab + (static_cast<long long>(f) * gridDim.x + band) * 5;
  if (t == 0) {
    out[0] = static_cast<double>(su[0][0]);
    out[1] = static_cast<double>(su[1][0]);
    out[2] = sd[0][0];
    out[3] = sd[1][0];
    out[4] = sd[2][0];
  }
}

// one thread per frame: the band slabs added in band order, then compute_depth_boundary_error's two scores
__global__ void edge_score_finish_kernel(const double* __restrict__ slab, int n, int bands,
                                         const double* __restrict__ gt_sums, double* __restrict__ scores) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int b = 0; b < bands; ++b)
#pragma unroll
    for (int j = 0; j < 5; ++j) s[j] = __dadd_rn(s[j], slab[(static_cast<long long>(f) * bands + b) * 5 + j]);
  double acc, comp;
  if (gt_sums[2 * f] == 0.0) {                     // np.sum(edges_gt) == 0
    acc = comp = CUDART_NAN;
  } else if (s[1] == 0.0) {                        // no predicted edge within 10 pixels of a ground-truth edge
    acc = comp = kEdgeMaxDist;
  } else {
    acc = __ddiv_rn(s[2], s[1]);
    comp = __ddiv_rn(__dadd_rn(s[3], s[4]), __dadd_rn(s[0], gt_sums[2 * f + 1]));
  }
  scores[2 * f] = acc;
  scores[2 * f + 1] = comp;
}

}  // namespace wmd

// ---------------------------------------------------------------------------------------- C ABI
namespace {
size_t align256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }
int edge_bands(int h) { return wmd::ceil_div(h, wmd::kEdgeBandRows); }

struct EdgeWs {                                    // carve-up of wmd_eval_edges_frames' workspace
  float2* mm;
  uint8_t* bits;
  uint8_t* hit;
  int* labels;
  int* g;
  int* any;
  double* slab;
  size_t bytes;
};

EdgeWs edge_ws(void* ws, int n, int h, int w) {
  const size_t px = static_cast<size_t>(n) * h * w;
  char* p = static_cast<char*>(ws);
  size_t off = 0;
  EdgeWs e;
  auto take = [&](size_t b) { char* q = p ? p + off : nullptr; off += align256(b); return q; };
  e.mm = reinterpret_cast<float2*>(take(n * sizeof(float2)));
  e.bits = reinterpret_cast<uint8_t*>(take(px));
  e.hit = reinterpret_cast<uint8_t*>(take(px));
  e.labels = reinterpret_cast<int*>(take(px * sizeof(int)));
  e.g = reinterpret_cast<int*>(take(px * sizeof(int)));
  e.any = reinterpret_cast<int*>(take(n * sizeof(int)));
  e.slab = reinterpret_cast<double*>(take(static_cast<size_t>(n) * edge_bands(h) * 5 * sizeof(double)));
  e.bytes = off;
  return e;
}

bool edge_shape_ok(int n, int h, int w) {
  return n >= 0 && n <= 65535 && h > 0 && w > 0 && h <= 65535 && static_cast<long long>(n) * h * w < (1ll << 31);
}

int run_edt(const uint8_t* feat, int n, int h, int w, int* g, int* any, double* dist, cudaStream_t st) {
  using namespace wmd;
  cudaMemsetAsync(any, 0, n * sizeof(int), st);
  edt_column_kernel<<<ceil_div(static_cast<long long>(n) * w, 128), 128, 0, st>>>(feat, n, h, w, g, any);
  if (int rc = launched()) return rc;
  edt_row_kernel<<<dim3(h, n), 128, 0, st>>>(g, any, h, w, dist);
  return launched();
}
}  // namespace

extern "C" size_t wmd_eval_edges_ws_bytes(int n, int h, int w) {
  if (!edge_shape_ok(n, h, w)) return 0;
  return edge_ws(nullptr, n, h, w).bytes;
}

extern "C" int wmd_eval_edges_frames(const void* pred, int pred_f64, int n, int h, int w, const double* taps,
                                     const double* bleed, double low, double high, const float* edges_gt,
                                     const double* d_gt, const double* gt_sums, uint8_t* edges_est, double* d_est,
                                     double* scores, void* ws, size_t ws_bytes, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(edge_shape_ok(n, h, w), WMD_ERR_SHAPE);
  if (n == 0) return WMD_OK;
  WMD_REQUIRE(pred && taps && bleed && edges_gt && d_gt && gt_sums && edges_est && d_est && scores && ws,
              WMD_ERR_ARG);
  const EdgeWs e = edge_ws(ws, n, h, w);
  WMD_REQUIRE(ws_bytes >= e.bytes, WMD_ERR_WORKSPACE);
  cudaStream_t st = as_stream(stream);
  const int total = n * h * w;
  const int grid = stride_grid(total, 256);
  edge_minmax_kernel<<<n, kEdgeThreads, 0, st>>>(pred, pred_f64, h * w, e.mm);
  if (int rc = launched()) return rc;
  edge_canny_kernel<<<dim3(ceil_div(w, kEdgeTile), ceil_div(h, kEdgeTile), n), kEdgeThreads, 0, st>>>(
      pred, pred_f64, h, w, e.mm, taps, bleed, low, high, e.bits);
  if (int rc = launched()) return rc;
  edge_uf_init_kernel<<<grid, 256, 0, st>>>(e.bits, total, e.labels, e.hit);
  if (int rc = launched()) return rc;
  edge_uf_merge_kernel<<<grid, 256, 0, st>>>(e.bits, h, w, total, e.labels);
  if (int rc = launched()) return rc;
  edge_uf_compress_kernel<<<grid, 256, 0, st>>>(e.bits, total, e.labels, e.hit);
  if (int rc = launched()) return rc;
  edge_uf_output_kernel<<<grid, 256, 0, st>>>(e.bits, total, e.labels, e.hit, edges_est);
  if (int rc = launched()) return rc;
  if (int rc = run_edt(edges_est, n, h, w, e.g, e.any, d_est, st)) return rc;
  edge_score_band_kernel<<<dim3(edge_bands(h), n), kEdgeThreads, 0, st>>>(edges_est, d_est, edges_gt, d_gt, h, w,
                                                                          e.slab);
  if (int rc = launched()) return rc;
  edge_score_finish_kernel<<<ceil_div(n, 128), 128, 0, st>>>(e.slab, n, edge_bands(h), gt_sums, scores);
  return launched();
}

extern "C" size_t wmd_eval_edt_ws_bytes(int n, int h, int w) {
  if (!edge_shape_ok(n, h, w)) return 0;
  return align256(static_cast<size_t>(n) * h * w * sizeof(int)) + align256(n * sizeof(int));
}

extern "C" int wmd_eval_edt(const uint8_t* features, int n, int h, int w, double* dist, void* ws, size_t ws_bytes,
                            wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(edge_shape_ok(n, h, w), WMD_ERR_SHAPE);
  if (n == 0) return WMD_OK;
  WMD_REQUIRE(features && dist && ws, WMD_ERR_ARG);
  WMD_REQUIRE(ws_bytes >= wmd_eval_edt_ws_bytes(n, h, w), WMD_ERR_WORKSPACE);
  int* g = static_cast<int*>(ws);
  int* any = reinterpret_cast<int*>(static_cast<char*>(ws) + align256(static_cast<size_t>(n) * h * w * sizeof(int)));
  return run_edt(features, n, h, w, g, any, dist, as_stream(stream));
}
