// KITTI's training inputs (include/wmd_inputs.h): flip + Pillow's LANCZOS pyramid + ColorJitter + ToTensor, batched.
//
// Launches per call: two resample passes per stage, one clear of the contrast sums, one contrast-mean pass and one
// epilogue that writes both fp32 planes of every stage.  The resample is integer-only; the mean is an integer sum whose
// atomic additions commute, so the bits never depend on the schedule.  The colour ops keep Pillow's float and double
// sub-expressions apart with explicit round-to-nearest intrinsics, so no contraction can change a value.
#include "common.cuh"
#include "resample8.cuh"
#include "wmd_inputs.h"

namespace wmd {
namespace {

constexpr int kT = 256;
constexpr size_t kAlign = 256;

inline size_t up(size_t b) { return (b + kAlign - 1) / kAlign * kAlign; }

// One resample pass's source and tables.  Stage 0 reads per-view sizes, flips and tables from `views`.
struct Pass {
  const uint8_t* in;
  uint8_t* out;
  int in_rows, in_cols;       // the input buffer's per-view extent (stage 0: the padded source)
  int rows, cols;             // the output buffer's per-view extent
  const wmd_inputs_view* views;
  const int32_t* tab;         // stages >= 1
  int k;
};

// horizontal: out (N, rows, cols, 3) from in (N, in_rows, in_cols, 3); rows == in_rows
__global__ void __launch_bounds__(kT) inputs_resample_h_kernel(Pass p, int N) {
  const long long total = static_cast<long long>(N) * p.rows * p.cols;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int x = static_cast<int>(i % p.cols);
    const long long vy = i / p.cols;
    const int y = static_cast<int>(vy % p.rows);
    const int v = static_cast<int>(vy / p.rows);
    const int32_t* tab = p.tab;
    int k = p.k, w = p.in_cols, flip = 0;
    if (p.views) {
      const wmd_inputs_view vw = p.views[v];
      if (y >= min(vw.h, p.in_rows)) continue;
      tab = vw.xtab, k = vw.xk, w = min(vw.w, p.in_cols), flip = vw.flip;
    }
    const int32_t* row = tab + static_cast<long long>(x) * (k + 2);
    const int first = row[0], taps = min(row[1], k);
    const uint8_t* src = p.in + (static_cast<long long>(v) * p.in_rows + y) * p.in_cols * 3;
    long long a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < taps; ++t) {
      int c = min(max(first + t, 0), w - 1);
      if (flip) c = w - 1 - c;
      const long long wt = row[2 + t];
      a0 += wt * src[3 * c], a1 += wt * src[3 * c + 1], a2 += wt * src[3 * c + 2];
    }
    uint8_t* o = p.out + 3 * i;
    o[0] = static_cast<uint8_t>(acc8(a0)), o[1] = static_cast<uint8_t>(acc8(a1)), o[2] = static_cast<uint8_t>(acc8(a2));
  }
}

// vertical: out (N, rows, cols, 3) from in (N, in_rows, cols, 3)
__global__ void __launch_bounds__(kT) inputs_resample_v_kernel(Pass p, int N) {
  const long long total = static_cast<long long>(N) * p.rows * p.cols;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int x = static_cast<int>(i % p.cols);
    const long long vy = i / p.cols;
    const int y = static_cast<int>(vy % p.rows);
    const int v = static_cast<int>(vy / p.rows);
    const int32_t* tab = p.tab;
    int k = p.k, h = p.in_rows;
    if (p.views) {
      const wmd_inputs_view vw = p.views[v];
      tab = vw.ytab, k = vw.yk, h = min(vw.h, p.in_rows);
    }
    const int32_t* row = tab + static_cast<long long>(y) * (k + 2);
    const int first = row[0], taps = min(row[1], k);
    const uint8_t* src = p.in + static_cast<long long>(v) * p.in_rows * p.cols * 3 + 3 * x;
    long long a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < taps; ++t) {
      const int r = min(max(first + t, 0), h - 1);
      const uint8_t* s = src + static_cast<long long>(r) * p.cols * 3;
      const long long wt = row[2 + t];
      a0 += wt * s[0], a1 += wt * s[1], a2 += wt * s[2];
    }
    uint8_t* o = p.out + 3 * i;
    o[0] = static_cast<uint8_t>(acc8(a0)), o[1] = static_cast<uint8_t>(acc8(a1)), o[2] = static_cast<uint8_t>(acc8(a2));
  }
}

// ---- Pillow's colour operations on one pixel ---------------------------------------------------------------------
__device__ __forceinline__ int blend8(int in1, int in2, float alpha) {   // Image.blend, libImaging/Blend.c
  const float t = __fadd_rn(static_cast<float>(in1), __fmul_rn(alpha, static_cast<float>(in2 - in1)));
  return clip8(static_cast<int>(fminf(fmaxf(truncf(t), 0.f), 255.f)));
}

__device__ __forceinline__ int luma(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 0x8000) >> 16; }

// libImaging/Convert.c rgb2hsv: float where C has float, double where a double constant promotes
__device__ __forceinline__ void rgb2hsv(int r, int g, int b, int& h8, int& s8, int& v8) {
  const int maxc = max(r, max(g, b)), minc = min(r, min(g, b));
  v8 = maxc;
  if (maxc == minc) {
    h8 = 0, s8 = 0;
    return;
  }
  const float cr = static_cast<float>(maxc - minc);
  const float s = __fdiv_rn(cr, static_cast<float>(maxc));
  const float rc = __fdiv_rn(static_cast<float>(maxc - r), cr);
  const float gc = __fdiv_rn(static_cast<float>(maxc - g), cr);
  const float bc = __fdiv_rn(static_cast<float>(maxc - b), cr);
  float h;
  if (r == maxc) {
    h = __fsub_rn(bc, gc);
  } else if (g == maxc) {
    h = __double2float_rn(__dsub_rn(__dadd_rn(2.0, static_cast<double>(rc)), static_cast<double>(bc)));
  } else {
    h = __double2float_rn(__dsub_rn(__dadd_rn(4.0, static_cast<double>(gc)), static_cast<double>(rc)));
  }
  h = __double2float_rn(fmod(__dadd_rn(__ddiv_rn(static_cast<double>(h), 6.0), 1.0), 1.0));
  h8 = clip8(static_cast<int>(__dmul_rn(static_cast<double>(h), 255.0)));
  s8 = clip8(static_cast<int>(__dmul_rn(static_cast<double>(s), 255.0)));
}

// libImaging/Convert.c hsv2rgb
__device__ __forceinline__ void hsv2rgb(int h8, int s8, int v8, int& r, int& g, int& b) {
  if (s8 == 0) {
    r = g = b = v8;
    return;
  }
  const double hf = __ddiv_rn(__dmul_rn(static_cast<double>(h8), 6.0), 255.0);
  const int i = static_cast<int>(floor(hf));
  const float f = __double2float_rn(__dsub_rn(hf, static_cast<double>(i)));
  const float fs = __double2float_rn(__ddiv_rn(static_cast<double>(s8), 255.0));
  const double v = static_cast<double>(v8);
  const int p = clip8(static_cast<int>(round(__dmul_rn(v, __dsub_rn(1.0, static_cast<double>(fs))))));
  const int q = clip8(static_cast<int>(round(__dmul_rn(v, __dsub_rn(1.0, static_cast<double>(__fmul_rn(fs, f)))))));
  const int t = clip8(static_cast<int>(round(
      __dmul_rn(v, __dsub_rn(1.0, __dmul_rn(static_cast<double>(fs), __dsub_rn(1.0, static_cast<double>(f))))))));
  switch (i % 6) {
    case 0: r = v8, g = t, b = p; break;
    case 1: r = q, g = v8, b = p; break;
    case 2: r = p, g = v8, b = t; break;
    case 3: r = p, g = q, b = v8; break;
    case 4: r = t, g = p, b = v8; break;
    default: r = v8, g = p, b = q; break;
  }
}

__device__ __forceinline__ void apply_op(int op, const wmd_inputs_jitter& j, int mean, int& r, int& g, int& b) {
  switch (op) {
    case 0:
      r = blend8(0, r, j.factor[0]), g = blend8(0, g, j.factor[0]), b = blend8(0, b, j.factor[0]);
      break;
    case 1:
      r = blend8(mean, r, j.factor[1]), g = blend8(mean, g, j.factor[1]), b = blend8(mean, b, j.factor[1]);
      break;
    case 2: {
      const int l = luma(r, g, b);
      r = blend8(l, r, j.factor[2]), g = blend8(l, g, j.factor[2]), b = blend8(l, b, j.factor[2]);
      break;
    }
    default: {
      int h, s, v;
      rgb2hsv(r, g, b, h, s, v);
      hsv2rgb((h + j.hue_shift) & 255, s, v, r, g, b);
      break;
    }
  }
}

// The stages' images and outputs, indexed by blockIdx.z.
struct Stages {
  const uint8_t* img[WMD_INPUTS_MAX_SCALES];
  float* color[WMD_INPUTS_MAX_SCALES];
  float* color_aug[WMD_INPUTS_MAX_SCALES];
  int pixels[WMD_INPUTS_MAX_SCALES];
};

// sums[z][v] = sum of L over stage z's image of view v after the ops before contrast (views whose jitter has contrast)
__global__ void __launch_bounds__(kT) inputs_mean_kernel(Stages st, const wmd_inputs_jitter* __restrict__ jitter, int N,
                                                         unsigned long long* __restrict__ sums) {
  const int z = blockIdx.z, v = blockIdx.y;
  const int px = st.pixels[z];
  const wmd_inputs_jitter j = jitter[v];
  if (j.order[0] < 0 || static_cast<int>(blockIdx.x) * kT >= px) return;
  const int i = blockIdx.x * kT + threadIdx.x;
  unsigned long long l = 0;
  if (i < px) {
    const uint8_t* p = st.img[z] + (static_cast<long long>(v) * px + i) * 3;
    int r = p[0], g = p[1], b = p[2];
    for (int k = 0; k < 4 && j.order[k] != 1; ++k) apply_op(j.order[k], j, 0, r, g, b);
    l = static_cast<unsigned long long>(luma(r, g, b));
  }
  for (int o = 16; o > 0; o >>= 1) l += __shfl_down_sync(0xffffffffu, l, o);
  __shared__ unsigned long long part[kT / 32];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = l;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long s = 0;
    for (int w = 0; w < kT / 32; ++w) s += part[w];
    atomicAdd(sums + static_cast<long long>(z) * N + v, s);
  }
}

__global__ void __launch_bounds__(kT) inputs_epilogue_kernel(Stages st, const wmd_inputs_jitter* __restrict__ jitter,
                                                             int N, const unsigned long long* __restrict__ sums) {
  const int z = blockIdx.z, v = blockIdx.y;
  const int px = st.pixels[z];
  const int i = blockIdx.x * kT + threadIdx.x;
  if (i >= px) return;
  const uint8_t* p = st.img[z] + (static_cast<long long>(v) * px + i) * 3;
  int c[3] = {p[0], p[1], p[2]};
  float* plain = st.color[z] + static_cast<long long>(v) * 3 * px + i;
  float* aug = st.color_aug[z] + static_cast<long long>(v) * 3 * px + i;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) plain[static_cast<long long>(ch) * px] = __fdiv_rn(static_cast<float>(c[ch]), 255.f);
  const wmd_inputs_jitter j = jitter[v];
  if (j.order[0] >= 0) {
    const double mean = __ddiv_rn(static_cast<double>(sums[static_cast<long long>(z) * N + v]), static_cast<double>(px));
    const int m = static_cast<int>(__dadd_rn(mean, 0.5));
    for (int k = 0; k < 4; ++k) apply_op(j.order[k], j, m, c[0], c[1], c[2]);
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) aug[static_cast<long long>(ch) * px] = __fdiv_rn(static_cast<float>(c[ch]), 255.f);
}

struct InputsWs {
  size_t tmp, img[WMD_INPUTS_MAX_SCALES], sums, total;
};

bool extent_ok(int v) { return v >= 1 && v <= 32767; }

// the byte offsets of the workspace's pieces; false for a descriptor wmd_inputs_u8 refuses on shape
bool inputs_ws(const wmd_inputs_desc& d, InputsWs& w) {
  if (d.N < 0 || d.N > 65535 || d.n_scales < 1 || d.n_scales > WMD_INPUTS_MAX_SCALES) return false;
  if (!extent_ok(d.src_h) || !extent_ok(d.src_w)) return false;
  size_t tmp = 0, o = 0;
  for (int j = 0; j < d.n_scales; ++j) {
    if (!extent_ok(d.out_h[j]) || !extent_ok(d.out_w[j])) return false;
    const long long in_rows = j ? d.out_h[j - 1] : d.src_h;
    const long long h_vals = static_cast<long long>(d.N) * in_rows * d.out_w[j] * 3;
    const long long vals = static_cast<long long>(d.N) * d.out_h[j] * d.out_w[j] * 3;
    if (h_vals > 0x7fffffffll || vals > 0x7fffffffll) return false;
    tmp = h_vals > static_cast<long long>(tmp) ? static_cast<size_t>(h_vals) : tmp;
  }
  w.tmp = o, o += up(tmp);
  for (int j = 0; j < d.n_scales; ++j) {
    w.img[j] = o;
    o += up(static_cast<size_t>(d.N) * d.out_h[j] * d.out_w[j] * 3);
  }
  w.sums = o, o += up(static_cast<size_t>(d.n_scales) * d.N * sizeof(unsigned long long));
  w.total = o;
  return true;
}

}  // namespace
}  // namespace wmd

extern "C" size_t wmd_inputs_ws_bytes(const wmd_inputs_desc* d) {
  wmd::InputsWs w;
  if (!d || !wmd::inputs_ws(*d, w)) return 0;
  return w.total;
}

extern "C" int wmd_inputs_u8(const wmd_inputs_desc* d, void* ws, size_t ws_bytes, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(d, WMD_ERR_ARG);
  InputsWs w;
  WMD_REQUIRE(inputs_ws(*d, w), WMD_ERR_SHAPE);
  if (d->N == 0) return WMD_OK;
  WMD_REQUIRE(d->src && d->views && d->jitter && ws, WMD_ERR_ARG);
  for (int j = 0; j < d->n_scales; ++j) {
    WMD_REQUIRE(d->color[j] && d->color_aug[j], WMD_ERR_ARG);
    if (j) WMD_REQUIRE(d->xtab[j] && d->ytab[j] && d->xk[j] >= 1 && d->yk[j] >= 1, WMD_ERR_ARG);
  }
  WMD_REQUIRE(ws_bytes >= w.total, WMD_ERR_WORKSPACE);
  cudaStream_t s = as_stream(stream);
  char* b = static_cast<char*>(ws);
  uint8_t* tmp = reinterpret_cast<uint8_t*>(b + w.tmp);
  Stages st{};
  int max_px = 0;
  for (int j = 0; j < d->n_scales; ++j) {
    uint8_t* img = reinterpret_cast<uint8_t*>(b + w.img[j]);
    Pass p{};
    p.in = j ? st.img[j - 1] : d->src;
    p.in_rows = j ? d->out_h[j - 1] : d->src_h;
    p.in_cols = j ? d->out_w[j - 1] : d->src_w;
    p.views = j ? nullptr : d->views;
    p.tab = d->xtab[j], p.k = d->xk[j];
    p.out = tmp, p.rows = p.in_rows, p.cols = d->out_w[j];
    long long n = static_cast<long long>(d->N) * p.rows * p.cols;
    inputs_resample_h_kernel<<<stride_grid(n, kT), kT, 0, s>>>(p, d->N);
    if (int rc = launched()) return rc;
    p.in = tmp, p.in_cols = p.cols;
    p.tab = d->ytab[j], p.k = d->yk[j];
    p.out = img, p.rows = d->out_h[j];
    n = static_cast<long long>(d->N) * p.rows * p.cols;
    inputs_resample_v_kernel<<<stride_grid(n, kT), kT, 0, s>>>(p, d->N);
    if (int rc = launched()) return rc;
    st.img[j] = img;
    st.color[j] = d->color[j], st.color_aug[j] = d->color_aug[j];
    st.pixels[j] = d->out_h[j] * d->out_w[j];
    max_px = st.pixels[j] > max_px ? st.pixels[j] : max_px;
  }
  unsigned long long* sums = reinterpret_cast<unsigned long long*>(b + w.sums);
  if (int rc = record(cudaMemsetAsync(sums, 0, static_cast<size_t>(d->n_scales) * d->N * sizeof(*sums), s))) return rc;
  const dim3 grid(ceil_div(max_px, kT), d->N, d->n_scales);
  inputs_mean_kernel<<<grid, kT, 0, s>>>(st, d->jitter, d->N, sums);
  if (int rc = launched()) return rc;
  inputs_epilogue_kernel<<<grid, kT, 0, s>>>(st, d->jitter, d->N, sums);
  return launched();
}
