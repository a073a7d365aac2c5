// KITTI's depth hints (KITTI/precompute_depth_hints.py) on the device (include/wmd_hints.h): OpenCV's StereoSGBM
// (MODE_SGBM) bit for bit, batched over frames, and the fusion of the twelve matchers' depths by reprojection error.
//
// Matcher, per call (one configuration, N frames), all integer:
//   prefilter: per view pixel and plane (3 clipped x-Sobel, 3 raw) the value and its half-pixel min / max, packed;
//   pixel cost: Birchfield-Tomasi over the six planes per (frame, row, column >= D, disparity), then the block sum;
//   paths: one warp per path line, the disparities spread over the lanes (ND = D / 32 consecutive ones per lane), the
//     line minimum by shuffles; the top, top-left, top-right and left-to-right kernels add their costs into S in turn
//     (one kernel per path, so every S entry has one writer per launch), the right-to-left kernel adds the last path
//     and picks the winner (uniqueness, sub-pixel) and offers it to the right view's winner of its column with an
//     atomicMin on (cost, -column), which is the pixel OpenCV's downward walk keeps;
//   then the left-right check, the 3x3 median and the speckle filter (union-find whose roots are each component's
//   least index, then sizes by integer atomics), written back mirrored for right views.
// Fusion: the views as fp32 planes, the warp of the lookup view by each matcher's depth, then per pixel the twelve
// reprojection errors, the first minimum and its depth.  The warp and the error are reproj.cuh's, shared with the loss.
#include "common.cuh"
#include "reproj.cuh"
#include "wmd_hints.h"

namespace wmd {
namespace {

constexpr int kP1 = 36, kP2 = 288, kCap = 63, kUniq = 10, kSpeckleSize = 100, kSpeckleDiff = 16 * 16;
constexpr int kMaxCost = 32767;
constexpr int kInvalid = -16;
constexpr int kT = 256;
constexpr int kWarps = 4;   // warps (path lines) per CTA
constexpr unsigned kFull = 0xffffffffu;

struct Geom {
  int N, H, W, D, W1, half;
};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// the prefiltered planes of one view, in the matcher's orientation (a right view is read mirrored): per plane the
// value, its min and its max over the half-pixel neighbours, packed v | min << 8 | max << 16
__device__ __forceinline__ int plane_val(const uint8_t* img, int H, int W, int y, int x, int p, bool rev) {
  if (x == 0 || x == W - 1) return kCap;
  const int c = p % 3;
  auto at = [&](int yy, int xx) { return static_cast<int>(img[(static_cast<long long>(yy) * W + (rev ? W - 1 - xx : xx)) * 3 + c]); };
  if (p >= 3) return at(y, x);
  const int yn = y > 0 ? y - 1 : y, ys = y < H - 1 ? y + 1 : y;
  const int g = (at(y, x + 1) - at(y, x - 1)) * 2 + at(yn, x + 1) - at(yn, x - 1) + at(ys, x + 1) - at(ys, x - 1);
  return clampi(g, -kCap, kCap) + kCap;
}

__global__ void __launch_bounds__(kT) sgbm_prefilter_kernel(const uint8_t* __restrict__ left,
                                                            const uint8_t* __restrict__ right,
                                                            const uint8_t* __restrict__ reverse, Geom g,
                                                            uint32_t* __restrict__ pre) {
  const long long plane = static_cast<long long>(g.H) * g.W, total = 2ll * g.N * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int view = static_cast<int>(i / (g.N * plane));
    const long long r = i - view * g.N * plane;
    const int n = static_cast<int>(r / plane), q = static_cast<int>(r - n * plane), y = q / g.W, x = q % g.W;
    const bool rev = reverse && reverse[n];
    const uint8_t* img = (view ? right : left) + n * plane * 3;
    for (int p = 0; p < 6; ++p) {
      const int v = plane_val(img, g.H, g.W, y, x, p, rev);
      const int vl = x > 0 ? (v + plane_val(img, g.H, g.W, y, x - 1, p, rev)) / 2 : v;
      const int vr = x < g.W - 1 ? (v + plane_val(img, g.H, g.W, y, x + 1, p, rev)) / 2 : v;
      const int lo = min(min(vl, vr), v), hi = max(max(vl, vr), v);
      pre[((static_cast<long long>(view) * g.N + n) * 6 + p) * plane + q] =
          static_cast<uint32_t>(v) | static_cast<uint32_t>(lo) << 8 | static_cast<uint32_t>(hi) << 16;
    }
  }
}

// The cost volumes are (N, H, W1, D) int16; their kernels run one CTA per (frame, row, column), N H W1 < 2^31
// (sgbm_geom), and one thread per disparity, so each CTA writes D consecutive entries.
__device__ __forceinline__ void volume_pixel(const Geom& g, int& n, int& y, int& x1) {
  const int p = blockIdx.x, ny = p / g.W1;
  x1 = p - ny * g.W1;
  n = ny / g.H;
  y = ny - n * g.H;
}

// the Birchfield-Tomasi cost of left column D + x1 against right column D + x1 - d
__global__ void __launch_bounds__(160) sgbm_pixel_cost_kernel(const uint32_t* __restrict__ pre, Geom g,
                                                              int16_t* __restrict__ out) {
  int n, y, x1;
  volume_pixel(g, n, y, x1);
  const int d = threadIdx.x, x = x1 + g.D, xr = x - d;
  const long long plane = static_cast<long long>(g.H) * g.W, row = static_cast<long long>(y) * g.W;
  int cost = 0;
#pragma unroll
  for (int p = 0; p < 6; ++p) {
    const uint32_t a = pre[(static_cast<long long>(n) * 6 + p) * plane + row + x];
    const uint32_t b = pre[((static_cast<long long>(g.N) + n) * 6 + p) * plane + row + xr];
    const int u = a & 255, u0 = (a >> 8) & 255, u1 = (a >> 16) & 255;
    const int v = b & 255, v0 = (b >> 8) & 255, v1 = (b >> 16) & 255;
    const int c0 = max(max(0, u - v1), v0 - u), c1 = max(max(0, v - u1), u0 - v);
    cost += min(c0, c1) >> (p < 3 ? 0 : 2);
  }
  out[static_cast<long long>(blockIdx.x) * g.D + d] = static_cast<int16_t>(cost);
}

// the block sum of half-width g.half, columns clamped to [0, W1 - 1] and rows to [0, H - 1]
__global__ void __launch_bounds__(160) sgbm_box_kernel(const int16_t* __restrict__ pix, Geom g,
                                                       int16_t* __restrict__ out) {
  int n, y, x1;
  volume_pixel(g, n, y, x1);
  const int d = threadIdx.x;
  int s = 0;
  for (int dy = -g.half; dy <= g.half; ++dy) {
    const long long row = (static_cast<long long>(n) * g.H + clampi(y + dy, 0, g.H - 1)) * g.W1;
    for (int dx = -g.half; dx <= g.half; ++dx) s += pix[(row + clampi(x1 + dx, 0, g.W1 - 1)) * g.D + d];
  }
  out[static_cast<long long>(blockIdx.x) * g.D + d] = static_cast<int16_t>(s);
}

__device__ __forceinline__ int warp_min(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(kFull, v, o));
  return v;
}

// path 0 left-to-right, 1 from the top-left, 2 from the top, 3 from the top-right, 4 right-to-left (with the winner)
enum { kPathLR = 0, kPathTL = 1, kPathT = 2, kPathTR = 3, kPathRL = 4 };

__host__ __device__ __forceinline__ int path_lines(int dir, int H, int W1) {
  return (dir == kPathLR || dir == kPathRL) ? H : (dir == kPathT ? W1 : W1 + H - 1);
}

template <int ND>
__global__ void __launch_bounds__(kWarps * 32) sgbm_path_kernel(const int16_t* __restrict__ C, int16_t* __restrict__ S,
                                                                Geom g, int dir, int first,
                                                                int16_t* __restrict__ disp1,
                                                                uint32_t* __restrict__ key2) {
  const int lane = threadIdx.x & 31;
  const int lines = path_lines(dir, g.H, g.W1);
  const long long gl = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5);
  if (gl >= static_cast<long long>(g.N) * lines) return;
  const int n = static_cast<int>(gl / lines), line = static_cast<int>(gl - static_cast<long long>(n) * lines);
  int x, y, sx, sy, len;
  switch (dir) {
    case kPathLR: x = 0; y = line; sx = 1; sy = 0; len = g.W1; break;
    case kPathRL: x = g.W1 - 1; y = line; sx = -1; sy = 0; len = g.W1; break;
    case kPathT: x = line; y = 0; sx = 0; sy = 1; len = g.H; break;
    case kPathTL:
      if (line < g.W1) { x = line; y = 0; } else { x = 0; y = line - g.W1 + 1; }
      sx = 1; sy = 1; len = min(g.W1 - x, g.H - y); break;
    default:
      if (line < g.W1) { x = line; y = 0; } else { x = g.W1 - 1; y = line - g.W1 + 1; }
      sx = -1; sy = 1; len = min(x + 1, g.H - y); break;
  }
  int Lp[ND];
#pragma unroll
  for (int k = 0; k < ND; ++k) Lp[k] = 0;
  int m = 0;                                  // a path starts from L' = 0, which gives L = C
  for (int t = 0; t < len; ++t, x += sx, y += sy) {
    const long long base = ((static_cast<long long>(n) * g.H + y) * g.W1 + x) * g.D + lane * ND;
    int lo = __shfl_up_sync(kFull, Lp[ND - 1], 1), hi = __shfl_down_sync(kFull, Lp[0], 1);
    if (lane == 0) lo = kMaxCost;
    if (lane == 31) hi = kMaxCost;
    int L[ND], s[ND];
#pragma unroll
    for (int k = 0; k < ND; ++k) {
      const int pm = k ? Lp[k - 1] : lo, pp = k < ND - 1 ? Lp[k + 1] : hi;
      L[k] = C[base + k] + min(min(Lp[k], pm + kP1), min(pp + kP1, m + kP2)) - m;
      s[k] = first ? L[k] : min(static_cast<int>(S[base + k]) + L[k], kMaxCost);
    }
    int lm = L[0];
#pragma unroll
    for (int k = 1; k < ND; ++k) lm = min(lm, L[k]);
    m = warp_min(lm);
#pragma unroll
    for (int k = 0; k < ND; ++k) Lp[k] = L[k];
    if (dir != kPathRL) {
#pragma unroll
      for (int k = 0; k < ND; ++k) S[base + k] = static_cast<int16_t>(s[k]);
      continue;
    }
    // the winner: the first minimum of S (key = S 256 + d), refused when a disparity two or more away is within the
    // uniqueness margin
    int key = s[0] * 256 + lane * ND;
#pragma unroll
    for (int k = 1; k < ND; ++k) key = min(key, s[k] * 256 + lane * ND + k);
    key = warp_min(key);
    const int minS = key >> 8, best = key & 255;
    bool far_low = false;
#pragma unroll
    for (int k = 0; k < ND; ++k)
      far_low |= s[k] * (100 - kUniq) < minS * 100 && abs(lane * ND + k - best) > 1;
    const bool refused = __any_sync(kFull, far_low);
    auto s_at = [&](int dd) {               // S[dd] from the lane that holds it (dd uniform over the warp)
      const int kk = dd % ND;
      int v = s[0];
#pragma unroll
      for (int k = 1; k < ND; ++k) v = kk == k ? s[k] : v;
      return __shfl_sync(kFull, v, dd / ND);
    };
    const int sm = s_at(max(best - 1, 0)), sp = s_at(min(best + 1, g.D - 1));
    if (lane == 0) {
      const int ximg = x + g.D;
      const long long row = (static_cast<long long>(n) * g.H + y) * g.W;
      int out = kInvalid;
      if (!refused) {
        atomicMin(key2 + row + ximg - best, static_cast<uint32_t>(minS) << 16 | static_cast<uint32_t>(65535 - ximg));
        if (best > 0 && best < g.D - 1) {
          const int den = max(sm + sp - 2 * minS, 1);
          out = best * 16 + ((sm - sp) * 16 + den) / (den * 2);
        } else {
          out = best * 16;
        }
      }
      disp1[row + ximg] = static_cast<int16_t>(out);
    }
  }
}

// the left-right check: refused when floor(d) and ceil(d) both land on a right-view winner more than 1 away
__device__ __forceinline__ bool lr_bad(const uint32_t* key2, long long row, int W, int x, int dd) {
  const int xx = x - dd;
  if (xx < 0 || xx >= W) return false;
  const uint32_t k = key2[row + xx];
  if (k == 0xffffffffu) return false;
  const int v = (65535 - static_cast<int>(k & 0xffffu)) - xx;
  return abs(v - dd) > 1;
}

__global__ void __launch_bounds__(kT) sgbm_lr_kernel(const int16_t* __restrict__ disp1,
                                                     const uint32_t* __restrict__ key2, Geom g,
                                                     int16_t* __restrict__ out) {
  const long long total = static_cast<long long>(g.N) * g.H * g.W;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int x = static_cast<int>(i % g.W);
    const long long row = i - x;
    int d = x < g.D ? kInvalid : disp1[i];
    if (d != kInvalid && lr_bad(key2, row, g.W, x, d >> 4) && lr_bad(key2, row, g.W, x, (d + 15) >> 4)) d = kInvalid;
    out[i] = static_cast<int16_t>(d);
  }
}

// cv::medianBlur(3): the median of the 3x3 window, edges replicated
__global__ void __launch_bounds__(kT) sgbm_median_kernel(const int16_t* __restrict__ in, Geom g,
                                                         int16_t* __restrict__ out) {
  const long long plane = static_cast<long long>(g.H) * g.W, total = g.N * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int n = static_cast<int>(i / plane), q = static_cast<int>(i - n * plane), y = q / g.W, x = q % g.W;
    int v[9];
    for (int dy = 0; dy < 3; ++dy)
      for (int dx = 0; dx < 3; ++dx)
        v[dy * 3 + dx] = in[n * plane + static_cast<long long>(clampi(y + dy - 1, 0, g.H - 1)) * g.W +
                            clampi(x + dx - 1, 0, g.W - 1)];
    for (int a = 0; a <= 4; ++a)             // selection of the five smallest; v[4] ends as the median
      for (int b = a + 1; b < 9; ++b)
        if (v[b] < v[a]) {
          const int t = v[a];
          v[a] = v[b];
          v[b] = t;
        }
    out[i] = static_cast<int16_t>(v[4]);
  }
}

// ---- speckle filter: union-find over each frame's pixels (index within the frame), every root its tree's least index
__device__ __forceinline__ int uf_find(const int* lab, int a) {
  const volatile int* l = lab;
  int p;
  while ((p = l[a]) != a) a = p;
  return a;
}
__device__ __forceinline__ void uf_unite(int* lab, int a, int b) {
  while (true) {
    a = uf_find(lab, a);
    b = uf_find(lab, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(lab + b, a);
    if (old == b) return;
    b = old;                                  // b had been linked meanwhile: join its new parent to a instead
  }
}

__device__ __forceinline__ bool joined(int a, int b) {
  return a != kInvalid && b != kInvalid && abs(a - b) <= kSpeckleDiff;
}

__global__ void __launch_bounds__(kT) sgbm_label_init_kernel(const int16_t* __restrict__ d, Geom g,
                                                             int* __restrict__ lab) {
  const long long plane = static_cast<long long>(g.H) * g.W, total = g.N * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT)
    lab[i] = d[i] == kInvalid ? -1 : static_cast<int>(i % plane);
}

__global__ void __launch_bounds__(kT) sgbm_unite_kernel(const int16_t* __restrict__ d, Geom g, int* __restrict__ lab) {
  const long long plane = static_cast<long long>(g.H) * g.W, total = g.N * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const long long f = i - i % plane;
    const int q = static_cast<int>(i - f), x = q % g.W, y = q / g.W;
    int* fl = lab + f;
    if (x + 1 < g.W && joined(d[i], d[i + 1])) uf_unite(fl, q, q + 1);
    if (y + 1 < g.H && joined(d[i], d[i + g.W])) uf_unite(fl, q, q + g.W);
  }
}

__global__ void __launch_bounds__(kT) sgbm_count_kernel(Geom g, int* __restrict__ lab, int* __restrict__ cnt) {
  const long long plane = static_cast<long long>(g.H) * g.W, total = g.N * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    if (lab[i] < 0) continue;
    const long long f = i - i % plane;
    const int r = uf_find(lab + f, static_cast<int>(i - f));
    atomicAdd(cnt + f + r, 1);
  }
}

// out = the pixel where its component has more than kSpeckleSize pixels, else invalid; mirrored back for right views
__global__ void __launch_bounds__(kT) sgbm_speckle_out_kernel(const int16_t* __restrict__ d,
                                                              const int* __restrict__ lab,
                                                              const int* __restrict__ cnt,
                                                              const uint8_t* __restrict__ reverse, Geom g,
                                                              int16_t* __restrict__ out) {
  const long long plane = static_cast<long long>(g.H) * g.W, total = g.N * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int hw = static_cast<int>(plane), n = static_cast<int>(i) / hw, q = static_cast<int>(i) - n * hw, x = q % g.W;
    const long long f = static_cast<long long>(n) * plane;        // N H W < 2^31 (sgbm_geom)
    // after the count kernel every label is its component's root
    const int v = lab[i] >= 0 && cnt[f + lab[i]] > kSpeckleSize ? d[i] : kInvalid;
    const int xo = reverse && reverse[n] ? g.W - 1 - x : x;
    out[f + (q - x) + xo] = static_cast<int16_t>(v);
  }
}

__global__ void __launch_bounds__(kT) sgbm_compress_kernel(Geom g, int* __restrict__ lab) {
  const long long plane = static_cast<long long>(g.H) * g.W, total = g.N * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    if (lab[i] < 0) continue;
    const long long f = i - i % plane;
    lab[i] = uf_find(lab + f, static_cast<int>(i - f));
  }
}

// ---- fusion
// uint8 (N, H, W, 3) -> fp32 planes (N, 3, H, W) of u / 255
__global__ void __launch_bounds__(kT) hints_planes_kernel(const uint8_t* __restrict__ img, long long npix, int hw,
                                                          float* __restrict__ out) {
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < npix;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int n = static_cast<int>(i) / hw, q = static_cast<int>(i) - n * hw;   // npix < 2^31 (hints_shape)
    for (int c = 0; c < 3; ++c)
      out[(static_cast<long long>(n) * 3 + c) * hw + q] = __fdiv_rn(static_cast<float>(img[i * 3 + c]), 255.f);
  }
}

__device__ __forceinline__ float hint_depth(int16_t raw, float k00) {
  const float disp = static_cast<float>(raw) / 16.f;      // exact
  const float q = __fdiv_rn(__fmul_rn(k00, 0.1f), __fadd_rn(disp, 1e-7f));
  return __fmul_rn(q, disp > 0.f ? 1.f : 0.f);
}

// the lookup view warped by every matcher's depth, (N, 12, 3, H, W) fp32
__global__ void __launch_bounds__(kT) hints_warp_kernel(const float* __restrict__ lookup,
                                                        const int16_t* __restrict__ disp, const float* __restrict__ K,
                                                        const float* __restrict__ iK, const float* __restrict__ T,
                                                        int N, int H, int W, float* __restrict__ warped) {
  const long long plane = static_cast<long long>(H) * W, total = static_cast<long long>(WMD_HINTS_MATCHERS) * N * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int m = static_cast<int>(i / (N * plane));
    const long long r = i - m * N * plane;
    const int n = static_cast<int>(r / plane), q = static_cast<int>(r - n * plane), Y = q / W, X = q % W;
    const Frame f = frame_ray(K + n * 16, iK + n * 16, T + n * 16, X, Y);
    const Coord c = project(f, static_cast<double>(hint_depth(disp[i], K[n * 16])), H, W);
    for (int ch = 0; ch < 3; ++ch)
      warped[((static_cast<long long>(n) * WMD_HINTS_MATCHERS + m) * 3 + ch) * plane + q] =
          __double2float_rn(sample(lookup + (static_cast<long long>(n) * 3 + ch) * plane, H, W, c).v);
  }
}

// per pixel: the twelve reprojection errors, torch.argmin (the first NaN, else the first minimum) and its depth
__global__ void __launch_bounds__(kT) hints_select_kernel(const float* __restrict__ base,
                                                          const float* __restrict__ warped,
                                                          const int16_t* __restrict__ disp,
                                                          const float* __restrict__ K, int N, int H, int W,
                                                          float* __restrict__ depth, int32_t* __restrict__ index) {
  const long long plane = static_cast<long long>(H) * W, total = static_cast<long long>(N) * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int n = static_cast<int>(i / plane), q = static_cast<int>(i - n * plane), Y = q / W, X = q % W;
    const float* tgt = base + static_cast<long long>(n) * 3 * plane;
    int k = 0;
    float bestv = 0.f;
    for (int m = 0; m < WMD_HINTS_MATCHERS; ++m) {
      const float r = reproj(warped + (static_cast<long long>(n) * WMD_HINTS_MATCHERS + m) * 3 * plane, tgt, plane, H,
                             W, Y, X);
      if (m == 0 || isnan(r) || r < bestv) {
        k = m;
        bestv = r;
        if (isnan(r)) break;
      }
    }
    depth[i] = hint_depth(disp[static_cast<long long>(k) * total + i], K[n * 16]);
    if (index) index[i] = k;
  }
}

// ---- workspace layouts
constexpr size_t kAlign = 256;
inline size_t up(size_t b) { return (b + kAlign - 1) / kAlign * kAlign; }

struct SgbmWs {
  size_t pre, pix, cost, sum, disp1, key2, lr, med, lab, cnt, total;
};

bool sgbm_geom(int N, int H, int W, int D, int bs, Geom& g) {
  if (N < 0 || H < 1 || W < 1 || H > 32767 || W > 32767) return false;
  if (D != 64 && D != 96 && D != 128 && D != 160) return false;
  if (bs < 1 || bs > 3 || W - D <= bs / 2) return false;
  // every pixel index of the batch, and every path line, fits the int grid arithmetic
  if (static_cast<long long>(N) * H * W > 0x7fffffffll) return false;
  g = Geom{N, H, W, D, W - D, bs / 2};
  return true;
}

SgbmWs sgbm_ws(const Geom& g) {
  const size_t px = static_cast<size_t>(g.N) * g.H * g.W;
  const size_t vol = static_cast<size_t>(g.N) * g.H * g.W1 * g.D * sizeof(int16_t);
  SgbmWs w;
  size_t o = 0;
  w.pre = o;   o += up(2 * 6 * px * sizeof(uint32_t));
  w.pix = o;   o += up(vol);
  w.cost = o;  o += g.half ? up(vol) : 0;
  w.sum = o;   o += up(vol);
  w.disp1 = o; o += up(px * sizeof(int16_t));
  w.key2 = o;  o += up(px * sizeof(uint32_t));
  w.lr = o;    o += up(px * sizeof(int16_t));
  w.med = o;   o += up(px * sizeof(int16_t));
  w.lab = o;   o += up(px * sizeof(int));
  w.cnt = o;   o += up(px * sizeof(int));
  w.total = o;
  return w;
}

template <int ND>
int launch_paths(const int16_t* C, int16_t* S, const Geom& g, int16_t* disp1, uint32_t* key2, cudaStream_t st) {
  const int order[5] = {kPathT, kPathTL, kPathTR, kPathLR, kPathRL};
  for (int i = 0; i < 5; ++i) {
    const long long lines = static_cast<long long>(g.N) * path_lines(order[i], g.H, g.W1);
    sgbm_path_kernel<ND><<<ceil_div(lines, kWarps), kWarps * 32, 0, st>>>(C, S, g, order[i], i == 0, disp1, key2);
    if (int rc = launched()) return rc;
  }
  return WMD_OK;
}

}  // namespace
}  // namespace wmd

extern "C" size_t wmd_sgbm_ws_bytes(int32_t N, int32_t H, int32_t W, int32_t num_disparities, int32_t block_size) {
  wmd::Geom g;
  if (!wmd::sgbm_geom(N, H, W, num_disparities, block_size, g)) return 0;
  return wmd::sgbm_ws(g).total;
}

extern "C" int wmd_sgbm_u8(const uint8_t* left, const uint8_t* right, const uint8_t* reverse, int32_t N, int32_t H,
                           int32_t W, int32_t num_disparities, int32_t block_size, void* ws, size_t ws_bytes,
                           int16_t* disp, wmd_stream_t stream) {
  using namespace wmd;
  Geom g;
  WMD_REQUIRE(sgbm_geom(N, H, W, num_disparities, block_size, g), WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  WMD_REQUIRE(left && right && ws && disp, WMD_ERR_ARG);
  const SgbmWs w = sgbm_ws(g);
  WMD_REQUIRE(ws_bytes >= w.total, WMD_ERR_WORKSPACE);
  cudaStream_t st = as_stream(stream);
  char* b = static_cast<char*>(ws);
  uint32_t* pre = reinterpret_cast<uint32_t*>(b + w.pre);
  int16_t* pix = reinterpret_cast<int16_t*>(b + w.pix);
  int16_t* cost = g.half ? reinterpret_cast<int16_t*>(b + w.cost) : pix;
  int16_t* sum = reinterpret_cast<int16_t*>(b + w.sum);
  int16_t* disp1 = reinterpret_cast<int16_t*>(b + w.disp1);
  uint32_t* key2 = reinterpret_cast<uint32_t*>(b + w.key2);
  int16_t* lr = reinterpret_cast<int16_t*>(b + w.lr);
  int16_t* med = reinterpret_cast<int16_t*>(b + w.med);
  int* lab = reinterpret_cast<int*>(b + w.lab);
  int* cnt = reinterpret_cast<int*>(b + w.cnt);
  const long long px = static_cast<long long>(N) * H * W;
  sgbm_prefilter_kernel<<<stride_grid(2 * px, kT), kT, 0, st>>>(left, right, reverse, g, pre);
  if (int rc = launched()) return rc;
  const int columns = N * H * g.W1;
  sgbm_pixel_cost_kernel<<<columns, g.D, 0, st>>>(pre, g, pix);
  if (int rc = launched()) return rc;
  if (g.half) {
    sgbm_box_kernel<<<columns, g.D, 0, st>>>(pix, g, cost);
    if (int rc = launched()) return rc;
  }
  if (int rc = record(cudaMemsetAsync(key2, 0xff, px * sizeof(uint32_t), st))) return rc;
  int rc = WMD_OK;
  switch (g.D) {
    case 64: rc = launch_paths<2>(cost, sum, g, disp1, key2, st); break;
    case 96: rc = launch_paths<3>(cost, sum, g, disp1, key2, st); break;
    case 128: rc = launch_paths<4>(cost, sum, g, disp1, key2, st); break;
    default: rc = launch_paths<5>(cost, sum, g, disp1, key2, st); break;
  }
  if (rc) return rc;
  const int grid = stride_grid(px, kT);
  sgbm_lr_kernel<<<grid, kT, 0, st>>>(disp1, key2, g, lr);
  if (int rc2 = launched()) return rc2;
  sgbm_median_kernel<<<grid, kT, 0, st>>>(lr, g, med);
  if (int rc2 = launched()) return rc2;
  sgbm_label_init_kernel<<<grid, kT, 0, st>>>(med, g, lab);
  if (int rc2 = launched()) return rc2;
  sgbm_unite_kernel<<<grid, kT, 0, st>>>(med, g, lab);
  if (int rc2 = launched()) return rc2;
  sgbm_compress_kernel<<<grid, kT, 0, st>>>(g, lab);
  if (int rc2 = launched()) return rc2;
  if (int rc2 = record(cudaMemsetAsync(cnt, 0, px * sizeof(int), st))) return rc2;
  sgbm_count_kernel<<<grid, kT, 0, st>>>(g, lab, cnt);
  if (int rc2 = launched()) return rc2;
  sgbm_speckle_out_kernel<<<grid, kT, 0, st>>>(med, lab, cnt, reverse, g, disp);
  return launched();
}

namespace {
bool hints_shape(int N, int H, int W) {
  return N >= 0 && H >= 2 && W >= 2 && H <= 32767 && W <= 32767 &&
         static_cast<long long>(N) * WMD_HINTS_MATCHERS * H * W <= 0x7fffffffll;
}
}  // namespace

extern "C" size_t wmd_depth_hints_ws_bytes(int32_t N, int32_t H, int32_t W) {
  if (!hints_shape(N, H, W)) return 0;
  const size_t px = static_cast<size_t>(N) * H * W;
  return wmd::up(2 * 3 * px * sizeof(float)) + wmd::up(WMD_HINTS_MATCHERS * 3 * px * sizeof(float));
}

extern "C" int wmd_depth_hints_f32(const uint8_t* base, const uint8_t* lookup, const int16_t* disp, const float* K,
                                   const float* inv_K, const float* T, int32_t N, int32_t H, int32_t W, void* ws,
                                   size_t ws_bytes, float* depth, int32_t* index, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(hints_shape(N, H, W), WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  WMD_REQUIRE(base && lookup && disp && K && inv_K && T && ws && depth, WMD_ERR_ARG);
  WMD_REQUIRE(ws_bytes >= wmd_depth_hints_ws_bytes(N, H, W), WMD_ERR_WORKSPACE);
  cudaStream_t st = as_stream(stream);
  const long long px = static_cast<long long>(N) * H * W;
  float* fb = static_cast<float*>(ws);
  float* fl = fb + 3 * px;
  float* warped = reinterpret_cast<float*>(static_cast<char*>(ws) + up(2 * 3 * px * sizeof(float)));
  const int grid = stride_grid(px, kT);
  hints_planes_kernel<<<grid, kT, 0, st>>>(base, px, H * W, fb);
  if (int rc = launched()) return rc;
  hints_planes_kernel<<<grid, kT, 0, st>>>(lookup, px, H * W, fl);
  if (int rc = launched()) return rc;
  hints_warp_kernel<<<stride_grid(WMD_HINTS_MATCHERS * px, kT), kT, 0, st>>>(fl, disp, K, inv_K, T, N, H, W, warped);
  if (int rc = launched()) return rc;
  hints_select_kernel<<<grid, kT, 0, st>>>(fb, warped, disp, K, N, H, W, depth, index);
  return launched();
}
