// The stereo warp and the per-pixel reprojection error shared by KITTI's depth-hints loss (loss_kitti.cu) and the depth
// hints' fusion (sgbm.cu): fp64 through _rn intrinsics, so that no FMA contraction changes a rounding; the numpy oracle
// (oracle/kitti_loss.py: project, sample, reproj) evaluates the same expressions.
#pragma once
#include <math.h>

namespace wmd {

constexpr double kC1 = 0.01 * 0.01, kC2 = 0.03 * 0.03;

__device__ __forceinline__ double A_(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double S_(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double M_(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double D_(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ int refl(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

struct Frame {          // per-frame camera: a = P[:3, :3] inv_K[:3, :3] (x, y, 1), b = P[:, 3], P = K stereo_T
  double a[3], b[3];
};
__device__ __forceinline__ Frame frame_ray(const float* K, const float* iK, const float* T, int x, int y) {
  double P[3][4];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
      P[i][j] = A_(A_(A_(M_(K[i * 4], T[j]), M_(K[i * 4 + 1], T[4 + j])), M_(K[i * 4 + 2], T[8 + j])),
                   M_(K[i * 4 + 3], T[12 + j]));
  double ray[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) ray[i] = A_(A_(M_(iK[i * 4], x), M_(iK[i * 4 + 1], y)), static_cast<double>(iK[i * 4 + 2]));
  Frame f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    f.a[i] = A_(A_(M_(P[i][0], ray[0]), M_(P[i][1], ray[1])), M_(P[i][2], ray[2]));
    f.b[i] = P[i][3];
  }
  return f;
}

struct Coord {
  double ix, iy, dix, diy;   // unclipped source coordinates and their derivatives in depth
};
__device__ __forceinline__ Coord project(const Frame& f, double D, int H, int W) {
  const double q0 = A_(M_(D, f.a[0]), f.b[0]), q1 = A_(M_(D, f.a[1]), f.b[1]), q2 = A_(M_(D, f.a[2]), f.b[2]);
  const double z = A_(q2, 1e-7);
  const double u = D_(q0, z), v = D_(q1, z);
  Coord c;
  c.ix = D_(S_(M_(A_(M_(S_(D_(u, W - 1.0), 0.5), 2.0), 1.0), static_cast<double>(W)), 1.0), 2.0);
  c.iy = D_(S_(M_(A_(M_(S_(D_(v, H - 1.0), 0.5), 2.0), 1.0), static_cast<double>(H)), 1.0), 2.0);
  const double bz = A_(f.b[2], 1e-7), zz = M_(z, z);
  c.dix = M_(D_(S_(M_(f.a[0], bz), M_(f.a[2], f.b[0])), zz), D_(static_cast<double>(W), W - 1.0));
  c.diy = M_(D_(S_(M_(f.a[1], bz), M_(f.a[2], f.b[1])), zz), D_(static_cast<double>(H), H - 1.0));
  return c;
}

// grid_sample (bilinear, border, align_corners=False) of one channel plane at c; with deriv, d/dix and d/diy (0 where
// the clamp is active or on the border)
struct Samp {
  double v, dx, dy;
};
__device__ __forceinline__ Samp sample(const float* plane, int H, int W, const Coord& c) {
  Samp s;
  if (isnan(c.ix) || isnan(c.iy)) {
    s.v = s.dx = s.dy = __longlong_as_double(0x7ff8000000000000ll);
    return s;
  }
  const double cx = fmin(fmax(c.ix, 0.0), W - 1.0), cy = fmin(fmax(c.iy, 0.0), H - 1.0);
  const double gx = (c.ix > 0.0 && c.ix < W - 1.0) ? 1.0 : 0.0, gy = (c.iy > 0.0 && c.iy < H - 1.0) ? 1.0 : 0.0;
  const int x0 = static_cast<int>(floor(cx)), y0 = static_cast<int>(floor(cy));
  const double wx1 = S_(cx, x0), wy1 = S_(cy, y0), wx0 = S_(x0 + 1.0, cx), wy0 = S_(y0 + 1.0, cy);
  const bool xin = x0 + 1 < W, yin = y0 + 1 < H;
  const double nw = plane[y0 * W + x0], ne = xin ? plane[y0 * W + x0 + 1] : 0.0;
  const double sw = yin ? plane[(y0 + 1) * W + x0] : 0.0, se = (xin && yin) ? plane[(y0 + 1) * W + x0 + 1] : 0.0;
  s.v = A_(A_(A_(M_(nw, M_(wx0, wy0)), M_(ne, M_(wx1, wy0))), M_(sw, M_(wx0, wy1))), M_(se, M_(wx1, wy1)));
  s.dx = M_(A_(M_(wy0, S_(ne, nw)), M_(wy1, S_(se, sw))), gx);
  s.dy = M_(A_(M_(wx0, S_(sw, nw)), M_(wx1, S_(se, ne))), gy);
  return s;
}

// SSIM window statistics of centre (Y, X), channel planes x (prediction) and y (target)
struct Win {
  double mx, my, A, B, Cc, Dd, n, d, raw;
};
__device__ __forceinline__ Win window(const float* x, const float* y, int H, int W, int Y, int X) {
  double r[5][3];    // per row dy: sum x, y, xx, yy, xy over dx
  for (int dy = 0; dy < 3; ++dy) {
    const int yy = refl(Y + dy - 1, H);
    double acc[5];
    for (int dx = 0; dx < 3; ++dx) {
      const int o = yy * W + refl(X + dx - 1, W);
      const double a = x[o], b = y[o];
      const double v[5] = {a, b, M_(a, a), M_(b, b), M_(a, b)};
      for (int k = 0; k < 5; ++k) acc[k] = dx == 0 ? v[k] : A_(acc[k], v[k]);
    }
    for (int k = 0; k < 5; ++k) r[k][dy] = acc[k];
  }
  double p[5];
  for (int k = 0; k < 5; ++k) p[k] = D_(A_(A_(r[k][0], r[k][1]), r[k][2]), 9.0);
  Win w;
  w.mx = p[0];
  w.my = p[1];
  const double sxx = S_(p[2], M_(w.mx, w.mx)), syy = S_(p[3], M_(w.my, w.my)), sxy = S_(p[4], M_(w.mx, w.my));
  w.A = A_(M_(M_(2.0, w.mx), w.my), kC1);
  w.B = A_(M_(2.0, sxy), kC2);
  w.Cc = A_(A_(M_(w.mx, w.mx), M_(w.my, w.my)), kC1);
  w.Dd = A_(A_(sxx, syy), kC2);
  w.n = M_(w.A, w.B);
  w.d = M_(w.Cc, w.Dd);
  w.raw = D_(S_(1.0, D_(w.n, w.d)), 2.0);
  return w;
}

// 0.85 mean_c SSIM + 0.15 mean_c |t - p| at (Y, X), rounded to fp32
__device__ __forceinline__ float reproj(const float* pred, const float* tgt, long long plane, int H, int W, int Y, int X) {
  double s[3], l[3];
  for (int c = 0; c < 3; ++c) {
    const Win w = window(pred + c * plane, tgt + c * plane, H, W, Y, X);
    s[c] = isnan(w.raw) ? w.raw : fmin(fmax(w.raw, 0.0), 1.0);
    const long long o = c * plane + static_cast<long long>(Y) * W + X;
    l[c] = fabs(S_(static_cast<double>(tgt[o]), static_cast<double>(pred[o])));
  }
  const double sm = D_(A_(A_(s[0], s[1]), s[2]), 3.0), lm = D_(A_(A_(l[0], l[1]), l[2]), 3.0);
  return __double2float_rn(A_(M_(0.85, sm), M_(0.15, lm)));
}

}  // namespace wmd
