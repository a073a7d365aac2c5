// KITTI's stereo depth-hints training loss (KITTI/trainer.py: generate_images_pred + compute_losses_hints with
// frame_ids [0, "s"]) on the device, forward and backward (include/wmd_loss_kitti.h).
//
// Forward: the hint warp and the two static maps (identity, hint + 1000 (1 - mask)) once; per loss scale the warp, the
// per-pixel reprojection loss with the argmin and the masked fp64 CTA partials, the per-frame disparity mean and the
// smoothness partials; one CTA adds every partial in CTA order and writes the terms.
// Backward, per loss scale: the SSIM window coefficients of every centre, a full-resolution gather that forms dL/dD
// (fp64), the smoothness mean's per-frame correction, and one thread per low-resolution pixel that gathers its upsample
// footprint and adds the smoothness gradient.  No atomics; fp64 arithmetic through _rn intrinsics so that no FMA
// contraction changes a rounding (the numpy oracle, oracle/kitti_loss.py, evaluates the same expressions).
#include <math.h>
#include "common.cuh"
#include "reproj.cuh"
#include "wmd_loss_kitti.h"

namespace wmd {
namespace {

constexpr int kKT = 256;
constexpr int kKPer = WMD_LOSS_PIXELS_PER_CTA / kKT;
__device__ __forceinline__ double sgn(double v) { return static_cast<double>((v > 0.0) - (v < 0.0)); }

// torch's align_corners=False tap of destination d (in -> out, out = in << f): src = max((d + 0.5) in / out - 0.5, 0)
struct Tap {
  int i0, i1;
  double l0, l1;
};
__device__ __forceinline__ Tap up_tap(int d, int in, int out) {
  const double src = fmax(S_(M_(static_cast<double>(d) + 0.5, D_(static_cast<double>(in), out)), 0.5), 0.0);
  Tap t;
  t.i0 = static_cast<int>(floor(src));
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  t.l1 = S_(src, static_cast<double>(t.i0));
  t.l0 = S_(1.0, t.l1);
  return t;
}

// the upsampled disparity at (Y, X) of frame n, and depth = 1 / (lo + (hi - lo) up)
__device__ __forceinline__ double up_disp(const float* disp, int h, int w, int H, int W, int n, int Y, int X) {
  const Tap ty = up_tap(Y, h, H), tx = up_tap(X, w, W);
  const float* p = disp + static_cast<long long>(n) * h * w;
  const double a = p[ty.i0 * w + tx.i0], b = p[ty.i0 * w + tx.i1], c = p[ty.i1 * w + tx.i0], d = p[ty.i1 * w + tx.i1];
  const double top = A_(M_(tx.l0, a), M_(tx.l1, b)), bot = A_(M_(tx.l0, c), M_(tx.l1, d));
  return A_(M_(ty.l0, top), M_(ty.l1, bot));
}

// fixed-tree sum of v over the CTA (every thread gets the result in red[0])
__device__ double cta_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = kKT / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = A_(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}
// sum of n partials in index order per thread (t, t + 256, ...), then the tree
__device__ double ordered_sum(const double* p, int n, double* red) {
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += kKT) acc = A_(acc, p[i]);
  return cta_sum(acc, red);
}

struct Geo {
  int N, H, W;
  const float *tgt, *src, *K, *iK, *T, *hint, *hmask;
  double lo, hi;
};

__device__ __forceinline__ void pix(const Geo& g, long long p, int& n, int& Y, int& X) {
  const long long plane = static_cast<long long>(g.H) * g.W;
  n = static_cast<int>(p / plane);
  const int r = static_cast<int>(p - n * plane);
  Y = r / g.W;
  X = r % g.W;
}

__device__ __forceinline__ double depth_at(const Geo& g, const float* disp, int h, int w, int n, int Y, int X) {
  if (!disp) return g.hint[(static_cast<long long>(n) * g.H + Y) * g.W + X];
  const double up = up_disp(disp, h, w, g.H, g.W, n, Y, X);
  return D_(1.0, A_(g.lo, M_(S_(g.hi, g.lo), up)));
}

// the warp of the source by the hint (disp == null) or by scale disp (h, w)
__global__ void __launch_bounds__(kKT) kitti_warp_kernel(Geo g, const float* __restrict__ disp, int h, int w,
                                                         float* __restrict__ out) {
  const long long p = static_cast<long long>(blockIdx.x) * kKT + threadIdx.x;
  if (p >= static_cast<long long>(g.N) * g.H * g.W) return;
  int n, Y, X;
  pix(g, p, n, Y, X);
  const Frame f = frame_ray(g.K + n * 16, g.iK + n * 16, g.T + n * 16, X, Y);
  const Coord c = project(f, depth_at(g, disp, h, w, n, Y, X), g.H, g.W);
  const long long plane = static_cast<long long>(g.H) * g.W;
  for (int ch = 0; ch < 3; ++ch)
    out[(static_cast<long long>(n) * 3 + ch) * plane + static_cast<long long>(Y) * g.W + X] =
        __double2float_rn(sample(g.src + (static_cast<long long>(n) * 3 + ch) * plane, g.H, g.W, c).v);
}

// identity loss and hint loss + 1000 (1 - mask), fp32
__global__ void __launch_bounds__(kKT) kitti_static_kernel(Geo g, const float* __restrict__ chint,
                                                           float* __restrict__ ident, float* __restrict__ hloss) {
  const long long p = static_cast<long long>(blockIdx.x) * kKT + threadIdx.x;
  if (p >= static_cast<long long>(g.N) * g.H * g.W) return;
  int n, Y, X;
  pix(g, p, n, Y, X);
  const long long plane = static_cast<long long>(g.H) * g.W, o = static_cast<long long>(n) * 3 * plane;
  ident[p] = reproj(g.src + o, g.tgt + o, plane, g.H, g.W, Y, X);
  const float pen = __fmul_rn(1000.f, __fsub_rn(1.f, g.hmask[p]));
  hloss[p] = __fadd_rn(reproj(chint + o, g.tgt + o, plane, g.H, g.W, Y, X), pen);
}

// r, the argmin against the static maps and the noise, the masks, and the CTA partials (sum r rm, sum rm, sum hint
// term hm, sum hm), each (4, ctas) at part
__global__ void __launch_bounds__(kKT) kitti_scale_kernel(Geo g, const float* __restrict__ disp, int h, int w,
                                                          const float* __restrict__ warped,
                                                          const float* __restrict__ ident,
                                                          const float* __restrict__ hloss,
                                                          const float* __restrict__ noise, float* __restrict__ idsel,
                                                          float* __restrict__ hpix, double* __restrict__ part) {
  __shared__ double red[kKT];
  const long long total = static_cast<long long>(g.N) * g.H * g.W, plane = static_cast<long long>(g.H) * g.W;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int j = 0; j < kKPer; ++j) {
    const long long p = static_cast<long long>(blockIdx.x) * WMD_LOSS_PIXELS_PER_CTA + j * kKT + threadIdx.x;
    if (p >= total) break;
    int n, Y, X;
    pix(g, p, n, Y, X);
    const long long o = static_cast<long long>(n) * 3 * plane;
    const float r = reproj(warped + o, g.tgt + o, plane, g.H, g.W, Y, X);
    const float ids = __fadd_rn(ident[p], __fmul_rn(noise[p], 1e-5f));
    const float v[3] = {r, ids, hloss[p]};
    int k = 0;                                  // torch.argmin: the first NaN, else the first minimum
    if (!isnan(v[0])) {
      for (int i = 1; i < 3; ++i) {
        if (isnan(v[i])) {
          k = i;
          break;
        }
        if (v[i] < v[k]) k = i;
      }
    }
    const double rm = k != 1 ? 1.0 : 0.0, hm = k == 2 ? 1.0 : 0.0;
    idsel[p] = static_cast<float>(1.0 - rm);
    hpix[p] = static_cast<float>(hm);
    const double diff = S_(depth_at(g, disp, h, w, n, Y, X), static_cast<double>(g.hint[p]));
    acc[0] = A_(acc[0], M_(static_cast<double>(r), rm));
    acc[1] = A_(acc[1], rm);
    acc[2] = A_(acc[2], M_(M_(log(A_(fabs(diff), 1.0)), static_cast<double>(g.hmask[p])), hm));
    acc[3] = A_(acc[3], hm);
  }
  for (int k = 0; k < 4; ++k) {
    const double s = cta_sum(acc[k], red);
    if (threadIdx.x == 0) part[static_cast<long long>(k) * gridDim.x + blockIdx.x] = s;
  }
}

// one CTA per frame: the disparity's mean
__global__ void __launch_bounds__(kKT) kitti_mean_kernel(const float* __restrict__ disp, int hw,
                                                         double* __restrict__ mean) {
  __shared__ double red[kKT];
  const float* p = disp + static_cast<long long>(blockIdx.x) * hw;
  double acc = 0.0;
  for (int i = threadIdx.x; i < hw; i += kKT) acc = A_(acc, static_cast<double>(p[i]));
  const double s = cta_sum(acc, red);
  if (threadIdx.x == 0) mean[blockIdx.x] = D_(s, static_cast<double>(hw));
}

__device__ __forceinline__ double edge_w(const float* img, long long plane, long long a, long long b) {
  double s = 0.0;
  for (int c = 0; c < 3; ++c) s = A_(s, fabs(S_(static_cast<double>(img[c * plane + a]), img[c * plane + b])));
  return exp(M_(-2.0, D_(s, 3.0)));
}

// |nd(a) - nd(b)| e(a, b) of the x edge (dir 0) or y edge (dir 1) leaving (y, x); 0 when there is none
__device__ __forceinline__ double edge(const float* d, const float* img, long long plane, int h, int w, int y, int x,
                                       double den, int dir, double* sg) {
  const bool has = dir == 0 ? x < w - 1 : y < h - 1;
  *sg = 0.0;
  if (!has) return 0.0;
  const long long a = static_cast<long long>(y) * w + x, b = dir == 0 ? a + 1 : a + w;
  const double diff = S_(D_(static_cast<double>(d[a]), den), D_(static_cast<double>(d[b]), den));
  const double e = edge_w(img, plane, a, b);
  *sg = M_(sgn(diff), e);
  return M_(fabs(diff), e);
}

// smoothness partials (sum x edges, sum y edges) per CTA of low-resolution pixels, (2, ctas) at part
__global__ void __launch_bounds__(kKT) kitti_smooth_kernel(const float* __restrict__ disp,
                                                           const float* __restrict__ color, int N, int h, int w,
                                                           const double* __restrict__ mean, double* __restrict__ part) {
  __shared__ double red[kKT];
  const long long plane = static_cast<long long>(h) * w, total = N * plane;
  double acc[2] = {0.0, 0.0};
  for (int j = 0; j < kKPer; ++j) {
    const long long p = static_cast<long long>(blockIdx.x) * WMD_LOSS_PIXELS_PER_CTA + j * kKT + threadIdx.x;
    if (p >= total) break;
    const int n = static_cast<int>(p / plane), r = static_cast<int>(p - n * plane), y = r / w, x = r % w;
    const double den = A_(mean[n], 1e-7);
    double sg;
    for (int dir = 0; dir < 2; ++dir)
      acc[dir] = A_(acc[dir], edge(disp + n * plane, color + n * 3 * plane, plane, h, w, y, x, den, dir, &sg));
  }
  for (int k = 0; k < 2; ++k) {
    const double s = cta_sum(acc[k], red);
    if (threadIdx.x == 0) part[static_cast<long long>(k) * gridDim.x + blockIdx.x] = s;
  }
}

struct Layout {        // the forward state (fp64 words) and its pieces, per loss scale i
  int N, H, W, nl, ctas_f, ctas_l[4], h[4], w[4], shift[4];
  __host__ __device__ long long off_part_f(int i) const { return 8ll + static_cast<long long>(i) * 4 * ctas_f; }
  __host__ __device__ long long off_part_l(int i) const {
    long long o = 8ll + 4ll * nl * ctas_f;
    for (int k = 0; k < i; ++k) o += 2ll * ctas_l[k];
    return o;
  }
  __host__ __device__ long long off_mean(int i) const { return off_part_l(nl) + static_cast<long long>(i) * N; }
  __host__ __device__ long long off_static() const { return off_mean(nl); }                        // 2 N H W floats
  __host__ __device__ long long words() const { return off_static() + (static_cast<long long>(N) * H * W + 1) / 2 * 2; }
};
// word 0..7 of the state: M and Mh of each loss scale (M_i at 2 i, Mh_i at 2 i + 1)

// one CTA: every scale's partials in CTA order, the terms, and M / Mh kept for the backward
__global__ void __launch_bounds__(kKT) kitti_final_kernel(Layout L, double* __restrict__ st, int n_scales,
                                                          double dsm, float* __restrict__ terms) {
  __shared__ double red[kKT];
  double total = 0.0;
  for (int i = 0; i < L.nl; ++i) {
    double s[4], e[2];
    for (int k = 0; k < 4; ++k) s[k] = ordered_sum(st + L.off_part_f(i) + k * L.ctas_f, L.ctas_f, red);
    for (int k = 0; k < 2; ++k) e[k] = ordered_sum(st + L.off_part_l(i) + k * L.ctas_l[i], L.ctas_l[i], red);
    const int h = L.h[i], w = L.w[i];
    const double cx = static_cast<double>(L.N) * h * (w - 1), cy = static_cast<double>(L.N) * (h - 1) * w;
    const double sm = A_(D_(e[0], cx), D_(e[1], cy));
    const double rep = static_cast<double>(__double2float_rn(D_(s[0], A_(s[1], 1e-7))));
    const double hin = static_cast<double>(__double2float_rn(D_(s[2], A_(s[3], 1e-7))));
    const double ls = static_cast<double>(
        __double2float_rn(A_(A_(rep, hin), D_(M_(dsm, sm), static_cast<double>(1 << L.shift[i])))));
    total = A_(total, ls);
    if (threadIdx.x == 0) {
      terms[1 + 3 * i] = static_cast<float>(rep);
      terms[2 + 3 * i] = static_cast<float>(hin);
      terms[3 + 3 * i] = static_cast<float>(ls);
      st[2 * i] = s[1];
      st[2 * i + 1] = s[3];
    }
  }
  if (threadIdx.x == 0) terms[0] = __double2float_rn(D_(total, static_cast<double>(n_scales)));
}

// ------------------------------------------------------------------------------------------------------------ backward
struct Coefs {
  double rep, hint, smooth;   // d L / d reproj_s, d L / d depth_hint_s, d L / d smooth_s
};
__device__ __forceinline__ Coefs coefs(const float* gt, int i, int n_scales, int shift, double dsm) {
  const double gl = A_(D_(static_cast<double>(gt[0]), static_cast<double>(n_scales)), gt[3 + 3 * i]);
  Coefs c;
  c.rep = A_(gl, gt[1 + 3 * i]);
  c.hint = A_(gl, gt[2 + 3 * i]);
  c.smooth = D_(M_(gl, dsm), static_cast<double>(1 << shift));
  return c;
}

// per centre and channel: w alpha, w beta, w gamma (9 planes per frame), w = rm c.rep / (M + 1e-7) 0.85 / 3 gate
__global__ void __launch_bounds__(kKT) kitti_coef_kernel(Geo g, const float* __restrict__ warped,
                                                         const float* __restrict__ idsel, const double* __restrict__ st,
                                                         int i, const float* __restrict__ gt, int n_scales, int shift,
                                                         double dsm, double* __restrict__ cf) {
  const long long p = static_cast<long long>(blockIdx.x) * kKT + threadIdx.x;
  if (p >= static_cast<long long>(g.N) * g.H * g.W) return;
  int n, Y, X;
  pix(g, p, n, Y, X);
  const long long plane = static_cast<long long>(g.H) * g.W, o = static_cast<long long>(n) * 3 * plane;
  const long long q = static_cast<long long>(Y) * g.W + X;
  const Coefs c = coefs(gt, i, n_scales, shift, dsm);
  const double wq = M_(M_(1.0 - static_cast<double>(idsel[p]), D_(c.rep, A_(st[2 * i], 1e-7))), D_(0.85, 3.0));
  for (int ch = 0; ch < 3; ++ch) {
    const Win w = window(warped + o + ch * plane, g.tgt + o + ch * plane, g.H, g.W, Y, X);
    const double gate = (w.raw >= 0.0 && w.raw <= 1.0) ? 1.0 : 0.0;
    const double ww = M_(wq, gate), dd = M_(w.d, w.d);
    const double al = D_(-S_(D_(M_(w.my, S_(w.B, w.A)), w.d), D_(M_(M_(w.n, w.mx), S_(w.Dd, w.Cc)), dd)), 9.0);
    const double be = D_(-D_(w.A, w.d), 9.0);
    const double ga = D_(D_(M_(w.n, w.Cc), dd), 9.0);
    double* out = cf + (static_cast<long long>(n) * 9 + ch * 3) * plane + q;
    out[0] = M_(ww, al);
    out[plane] = M_(ww, be);
    out[2 * plane] = M_(ww, ga);
  }
}

// d L / d up (fp64) at every full-resolution pixel: the SSIM + L1 adjoint gathered over the reflected windows that read
// the pixel, through the sample's and the projection's derivatives, plus the hint term, times d depth / d up
__global__ void __launch_bounds__(kKT, 1) kitti_ddepth_kernel(Geo g, const float* __restrict__ disp, int h, int w,
                                                           const float* __restrict__ warped,
                                                           const float* __restrict__ idsel,
                                                           const float* __restrict__ hpix,
                                                           const double* __restrict__ st, int i,
                                                           const float* __restrict__ gt, int n_scales, int shift,
                                                           double dsm, const double* __restrict__ cf,
                                                           double* __restrict__ dup) {
  const long long p = static_cast<long long>(blockIdx.x) * kKT + threadIdx.x;
  if (p >= static_cast<long long>(g.N) * g.H * g.W) return;
  int n, Y, X;
  pix(g, p, n, Y, X);
  const long long plane = static_cast<long long>(g.H) * g.W, o = static_cast<long long>(n) * 3 * plane;
  const Coefs c = coefs(gt, i, n_scales, shift, dsm);
  const double D = depth_at(g, disp, h, w, n, Y, X);
  const Frame f = frame_ray(g.K + n * 16, g.iK + n * 16, g.T + n * 16, X, Y);
  const Coord cd = project(f, D, g.H, g.W);
  const double l1w = M_(M_(1.0 - static_cast<double>(idsel[p]), D_(c.rep, A_(st[2 * i], 1e-7))), D_(0.15, 3.0));
  double dD = 0.0;
  for (int ch = 0; ch < 3; ++ch) {
    const double* cp = cf + (static_cast<long long>(n) * 9 + ch * 3) * plane;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
#pragma unroll 1
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll 1
      for (int dx = -1; dx <= 1; ++dx)
#pragma unroll 1
        for (int qy = max(Y - 2, 0); qy <= min(Y + 2, g.H - 1); ++qy) {
          if (refl(qy + dy, g.H) != Y) continue;
#pragma unroll 1
          for (int qx = max(X - 2, 0); qx <= min(X + 2, g.W - 1); ++qx) {
            if (refl(qx + dx, g.W) != X) continue;
            const double* c = cp + static_cast<long long>(qy) * g.W + qx;
            s0 = A_(s0, c[0]);
            s1 = A_(s1, c[plane]);
            s2 = A_(s2, c[2 * plane]);
          }
        }
    const long long at = o + ch * plane + static_cast<long long>(Y) * g.W + X;
    const double x = warped[at], t = g.tgt[at];
    const double dx = A_(A_(A_(s0, M_(s1, t)), M_(s2, x)), M_(l1w, sgn(S_(x, t))));
    const Samp sp = sample(g.src + o + ch * plane, g.H, g.W, cd);
    dD = A_(dD, M_(dx, A_(M_(sp.dx, cd.dix), M_(sp.dy, cd.diy))));
  }
  const double diff = S_(D, static_cast<double>(g.hint[p]));
  const double hw = M_(M_(M_(D_(c.hint, A_(st[2 * i + 1], 1e-7)), g.hmask[p]), hpix[p]), sgn(diff));
  dD = A_(dD, D_(hw, A_(fabs(diff), 1.0)));
  dup[p] = M_(dD, -M_(M_(S_(g.hi, g.lo), D), D));
}

// d smooth / d nd at low-resolution pixel (y, x) (x edges' sign e / cx, y edges' / cy, in the oracle's order).  Only
// edges that exist add a term: a one-column map has cx = 0 and a one-row map cy = 0, and 0 / 0 would make every
// gradient of the scale NaN where the reference's mean over no edges contributes none.
__device__ __forceinline__ double smooth_G(const float* d, const float* img, long long plane, int h, int w, int y, int x, double den,
                           double cx, double cy) {
  double sg, G = 0.0;
  if (x < w - 1) {
    edge(d, img, plane, h, w, y, x, den, 0, &sg);
    G = A_(G, D_(sg, cx));
  }
  if (x > 0) {
    edge(d, img, plane, h, w, y, x - 1, den, 0, &sg);
    G = S_(G, D_(sg, cx));
  }
  if (y < h - 1) {
    edge(d, img, plane, h, w, y, x, den, 1, &sg);
    G = A_(G, D_(sg, cy));
  }
  if (y > 0) {
    edge(d, img, plane, h, w, y - 1, x, den, 1, &sg);
    G = S_(G, D_(sg, cy));
  }
  return G;
}

// one CTA per frame: corr = sum G d / (h w)
__global__ void __launch_bounds__(kKT) kitti_corr_kernel(const float* __restrict__ disp,
                                                         const float* __restrict__ color, int h, int w,
                                                         const double* __restrict__ mean, double* __restrict__ corr) {
  __shared__ double red[kKT];
  const int n = blockIdx.x;
  const long long plane = static_cast<long long>(h) * w;
  const float* d = disp + n * plane;
  const float* img = color + n * 3 * plane;
  const double den = A_(mean[n], 1e-7);
  const double cx = static_cast<double>(gridDim.x) * h * (w - 1), cy = static_cast<double>(gridDim.x) * (h - 1) * w;
  double acc = 0.0;
  for (long long q = threadIdx.x; q < plane; q += kKT) {
    const int y = static_cast<int>(q / w), x = static_cast<int>(q % w);
    acc = A_(acc, M_(smooth_G(d, img, plane, h, w, y, x, den, cx, cy), static_cast<double>(d[q])));
  }
  const double s = cta_sum(acc, red);
  if (threadIdx.x == 0) corr[n] = D_(s, static_cast<double>(plane));
}

// one thread per low-resolution pixel: the upsample adjoint of dup over its footprint (x taps then y taps, each i0
// then i1, ascending) plus c.smooth (G / den - corr / den^2)
__global__ void __launch_bounds__(kKT) kitti_grad_kernel(const double* __restrict__ dup, int N, int H, int W,
                                                         const float* __restrict__ disp,
                                                         const float* __restrict__ color, int h, int w,
                                                         const double* __restrict__ mean,
                                                         const double* __restrict__ corr, const float* __restrict__ gt,
                                                         int i, int n_scales, int shift, double dsm,
                                                         float* __restrict__ grad) {
  const long long plane = static_cast<long long>(h) * w;
  const long long p = static_cast<long long>(blockIdx.x) * kKT + threadIdx.x;
  if (p >= N * plane) return;
  const int n = static_cast<int>(p / plane), r = static_cast<int>(p - n * plane), y = r / w, x = r % w;
  const int f = H / h;
  const int Ylo = max(0, (y - 1) * f), Yhi = min(H - 1, (y + 2) * f), Xlo = max(0, (x - 1) * f),
            Xhi = min(W - 1, (x + 2) * f);
  const double* g = dup + static_cast<long long>(n) * H * W;
  double acc = 0.0;
  for (int sy = 0; sy < 2; ++sy)
    for (int Y = Ylo; Y <= Yhi; ++Y) {
      const Tap ty = up_tap(Y, h, H);
      if ((sy == 0 ? ty.i0 : ty.i1) != y) continue;
      double row = 0.0;
      for (int sx = 0; sx < 2; ++sx)
        for (int X = Xlo; X <= Xhi; ++X) {
          const Tap tx = up_tap(X, w, W);
          if ((sx == 0 ? tx.i0 : tx.i1) != x) continue;
          row = A_(row, M_(g[static_cast<long long>(Y) * W + X], sx == 0 ? tx.l0 : tx.l1));
        }
      acc = A_(acc, M_(row, sy == 0 ? ty.l0 : ty.l1));
    }
  const Coefs c = coefs(gt, i, n_scales, shift, dsm);
  const double den = A_(mean[n], 1e-7);
  const double cx = static_cast<double>(N) * h * (w - 1), cy = static_cast<double>(N) * (h - 1) * w;
  const double G = smooth_G(disp + n * plane, color + n * 3 * plane, plane, h, w, y, x, den, cx, cy);
  const double sgrad = S_(D_(G, den), D_(corr[n], M_(den, den)));
  grad[p] = __double2float_rn(A_(acc, M_(c.smooth, sgrad)));
}

}  // namespace
}  // namespace wmd

// ---------------------------------------------------------------------------------------- C ABI
namespace {
int kitti_layout(const wmd_loss_kitti_desc* d, wmd::Layout& L) {
  WMD_REQUIRE(d, WMD_ERR_ARG);
  WMD_REQUIRE(d->N >= 0 && d->N <= 65535 && d->H >= 8 && d->W >= 8 && d->H % 8 == 0 && d->W % 8 == 0,
              WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(d->N) * 9 * d->H * d->W < (1ll << 31), WMD_ERR_SHAPE);
  WMD_REQUIRE(d->n_loss >= 1 && d->n_loss <= 4 && d->n_scales >= d->n_loss && d->n_scales <= 4, WMD_ERR_SHAPE);
  WMD_REQUIRE(d->min_depth > 0.0 && d->max_depth > d->min_depth, WMD_ERR_ARG);
  L.N = d->N;
  L.H = d->H;
  L.W = d->W;
  L.nl = d->n_loss;
  L.ctas_f = wmd::ceil_div(static_cast<long long>(d->N) * d->H * d->W, WMD_LOSS_PIXELS_PER_CTA);
  for (int i = 0; i < d->n_loss; ++i) {
    WMD_REQUIRE(d->scale[i] >= 0 && d->scale[i] <= 3 && (i == 0 || d->scale[i] > d->scale[i - 1]), WMD_ERR_SHAPE);
    L.shift[i] = d->scale[i];
    L.h[i] = d->H >> d->scale[i];
    L.w[i] = d->W >> d->scale[i];
    L.ctas_l[i] = wmd::ceil_div(static_cast<long long>(d->N) * L.h[i] * L.w[i], WMD_LOSS_PIXELS_PER_CTA);
    WMD_REQUIRE(d->N == 0 || (d->disp[i] && d->color[i] && d->noise[i]), WMD_ERR_ARG);
  }
  WMD_REQUIRE(d->N == 0 || (d->target && d->source && d->K && d->inv_K && d->stereo_T && d->depth_hint &&
                            d->depth_hint_mask), WMD_ERR_ARG);
  return WMD_OK;
}

wmd::Geo kitti_geo(const wmd_loss_kitti_desc* d) {
  return wmd::Geo{d->N, d->H, d->W, d->target, d->source, d->K, d->inv_K, d->stereo_T, d->depth_hint,
                  d->depth_hint_mask, 1.0 / d->max_depth, 1.0 / d->min_depth};
}
}  // namespace

extern "C" size_t wmd_loss_kitti_ws_bytes(const wmd_loss_kitti_desc* d) {
  wmd::Layout L;
  if (kitti_layout(d, L)) return 0;
  return static_cast<size_t>(L.words()) * sizeof(double) + static_cast<size_t>(d->N) * d->H * d->W * sizeof(float);
}

extern "C" size_t wmd_loss_kitti_bwd_ws_bytes(const wmd_loss_kitti_desc* d) {
  wmd::Layout L;
  if (kitti_layout(d, L)) return 0;
  return (static_cast<size_t>(d->N) * d->H * d->W * 10 + d->N) * sizeof(double);
}

extern "C" int wmd_loss_kitti_fwd(const wmd_loss_kitti_desc* d, float* color_depth_hint, float* warped, float* idsel,
                                  float* hpix, void* ws, size_t ws_bytes, float* terms, wmd_stream_t stream) {
  using namespace wmd;
  Layout L;
  if (int rc = kitti_layout(d, L)) return rc;
  WMD_REQUIRE(terms && ws && (d->N == 0 || (color_depth_hint && warped && idsel && hpix)), WMD_ERR_ARG);
  WMD_REQUIRE(ws_bytes >= wmd_loss_kitti_ws_bytes(d), WMD_ERR_WORKSPACE);
  cudaStream_t st = as_stream(stream);
  if (d->N == 0) {
    kitti_final_kernel<<<1, kKT, 0, st>>>(L, static_cast<double*>(ws), d->n_scales, d->disparity_smoothness, terms);
    return launched();
  }
  const Geo g = kitti_geo(d);
  const long long npix = static_cast<long long>(d->N) * d->H * d->W;
  const int grid = ceil_div(npix, kKT);
  double* sw = static_cast<double*>(ws);
  float* ident = reinterpret_cast<float*>(sw + L.off_static());
  float* hloss = ident + npix;
  kitti_warp_kernel<<<grid, kKT, 0, st>>>(g, nullptr, 0, 0, color_depth_hint);
  if (int rc = launched()) return rc;
  kitti_static_kernel<<<grid, kKT, 0, st>>>(g, color_depth_hint, ident, hloss);
  if (int rc = launched()) return rc;
  for (int i = 0; i < L.nl; ++i) {
    const int h = L.h[i], w = L.w[i];
    float* wp = warped + i * 3 * npix;
    kitti_warp_kernel<<<grid, kKT, 0, st>>>(g, d->disp[i], h, w, wp);
    if (int rc = launched()) return rc;
    kitti_scale_kernel<<<L.ctas_f, kKT, 0, st>>>(g, d->disp[i], h, w, wp, ident, hloss, d->noise[i], idsel + i * npix,
                                                  hpix + i * npix, sw + L.off_part_f(i));
    if (int rc = launched()) return rc;
    kitti_mean_kernel<<<d->N, kKT, 0, st>>>(d->disp[i], h * w, sw + L.off_mean(i));
    if (int rc = launched()) return rc;
    kitti_smooth_kernel<<<L.ctas_l[i], kKT, 0, st>>>(d->disp[i], d->color[i], d->N, h, w, sw + L.off_mean(i),
                                                      sw + L.off_part_l(i));
    if (int rc = launched()) return rc;
  }
  kitti_final_kernel<<<1, kKT, 0, st>>>(L, sw, d->n_scales, d->disparity_smoothness, terms);
  return launched();
}

extern "C" int wmd_loss_kitti_bwd(const wmd_loss_kitti_desc* d, const float* warped, const float* idsel,
                                  const float* hpix, const void* fwd_ws, const float* grad_terms, void* ws,
                                  size_t ws_bytes, float* const* grads, wmd_stream_t stream) {
  using namespace wmd;
  Layout L;
  if (int rc = kitti_layout(d, L)) return rc;
  WMD_REQUIRE(grads && grad_terms, WMD_ERR_ARG);
  for (int i = 0; i < L.nl; ++i) WMD_REQUIRE(d->N == 0 || grads[i], WMD_ERR_ARG);
  WMD_REQUIRE(d->N == 0 || (warped && idsel && hpix && fwd_ws && ws), WMD_ERR_ARG);
  WMD_REQUIRE(ws_bytes >= wmd_loss_kitti_bwd_ws_bytes(d), WMD_ERR_WORKSPACE);
  if (d->N == 0) return WMD_OK;
  cudaStream_t st = as_stream(stream);
  const Geo g = kitti_geo(d);
  const long long npix = static_cast<long long>(d->N) * d->H * d->W;
  const int grid = ceil_div(npix, kKT);
  const double* sw = static_cast<const double*>(fwd_ws);
  double* cf = static_cast<double*>(ws);
  double* dup = cf + 9 * npix;
  double* corr = dup + npix;
  const double dsm = d->disparity_smoothness;
  for (int i = 0; i < L.nl; ++i) {
    const int h = L.h[i], w = L.w[i];
    const float* wp = warped + i * 3 * npix;
    kitti_coef_kernel<<<grid, kKT, 0, st>>>(g, wp, idsel + i * npix, sw, i, grad_terms, d->n_scales, L.shift[i], dsm,
                                            cf);
    if (int rc = launched()) return rc;
    kitti_ddepth_kernel<<<grid, kKT, 0, st>>>(g, d->disp[i], h, w, wp, idsel + i * npix, hpix + i * npix, sw, i,
                                              grad_terms, d->n_scales, L.shift[i], dsm, cf, dup);
    if (int rc = launched()) return rc;
    kitti_corr_kernel<<<d->N, kKT, 0, st>>>(d->disp[i], d->color[i], h, w, sw + L.off_mean(i), corr);
    if (int rc = launched()) return rc;
    kitti_grad_kernel<<<ceil_div(static_cast<long long>(d->N) * h * w, kKT), kKT, 0, st>>>(
        dup, d->N, d->H, d->W, d->disp[i], d->color[i], h, w, sw + L.off_mean(i), corr, grad_terms, i, d->n_scales,
        L.shift[i], dsm, grads[i]);
    if (int rc = launched()) return rc;
  }
  return WMD_OK;
}
