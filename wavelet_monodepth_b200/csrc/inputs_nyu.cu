// NYUv2's training inputs (include/wmd_inputs_nyu.h): flip + channel swap + gamma LUT + crop + Pillow resize + ToTensor.
//
// Two launches per call.  The horizontal pass reads the cropped rows of the image and the depth together, applies the
// item's flip, channel permutation and LUT to every source byte and writes uint8 intermediates; the vertical pass
// writes both fp32 outputs with the ToTensor / depth epilogue fused in.  Integer-only up to that epilogue, whose two
// depth roundings are kept apart with explicit round-to-nearest intrinsics.
#include "common.cuh"
#include "resample8.cuh"
#include "wmd_inputs_nyu.h"

namespace wmd {
namespace {

constexpr int kT = 256;
constexpr size_t kAlign = 256;
constexpr int kLo = WMD_NYU_CROP;                          // first row / column kept by the crop
constexpr int kXHi = WMD_NYU_SRC_W - WMD_NYU_CROP - 1;     // last column kept (623)
constexpr int kYHi = WMD_NYU_SRC_H - WMD_NYU_CROP - 1;     // last row kept (463)
constexpr int kRows = kYHi - kLo + 1;                      // 448 rows between the passes

inline size_t up(size_t b) { return (b + kAlign - 1) / kAlign * kAlign; }

__device__ __forceinline__ int chan(int p) { return min(max(p, 0), 2); }

// tmp_img (N, 448, image_w, 3) and tmp_depth (N, 448, depth_w): one thread per intermediate pixel of either
__global__ void __launch_bounds__(kT) nyu_inputs_h_kernel(wmd_nyu_inputs_desc d, uint8_t* __restrict__ tmp_img,
                                                          uint8_t* __restrict__ tmp_depth) {
  const int cols = d.image_w + d.depth_w;
  const long long total = static_cast<long long>(d.N) * kRows * cols;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    const int x = static_cast<int>(i % cols);
    const long long vy = i / cols;
    const int y = static_cast<int>(vy % kRows);
    const int v = static_cast<int>(vy / kRows);
    const wmd_nyu_inputs_item it = d.items[v];
    const long long src_row = static_cast<long long>(v) * WMD_NYU_SRC_H + kLo + y;
    if (x < d.image_w) {
      const int32_t* row = d.image_xtab + static_cast<long long>(x) * (d.image_xk + 2);
      const int first = row[0], taps = min(row[1], d.image_xk);
      const uint8_t* src = d.image_src + src_row * WMD_NYU_SRC_W * 3;
      const uint8_t* lut = d.lut + static_cast<long long>(v) * 256;
      const int p0 = chan(it.perm[0]), p1 = chan(it.perm[1]), p2 = chan(it.perm[2]);
      long long a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int t = 0; t < taps; ++t) {
        int c = min(max(first + t, kLo), kXHi);
        if (it.flip) c = WMD_NYU_SRC_W - 1 - c;
        const uint8_t* s = src + 3 * c;
        const long long wt = row[2 + t];
        a0 += wt * lut[s[p0]], a1 += wt * lut[s[p1]], a2 += wt * lut[s[p2]];
      }
      uint8_t* o = tmp_img + ((static_cast<long long>(v) * kRows + y) * d.image_w + x) * 3;
      o[0] = static_cast<uint8_t>(acc8(a0)), o[1] = static_cast<uint8_t>(acc8(a1)), o[2] = static_cast<uint8_t>(acc8(a2));
    } else {
      const int xd = x - d.image_w;
      const int32_t* row = d.depth_xtab + static_cast<long long>(xd) * (d.depth_xk + 2);
      const int first = row[0], taps = min(row[1], d.depth_xk);
      const uint8_t* src = d.depth_src + src_row * WMD_NYU_SRC_W;
      long long a = 1 << (kPrecisionBits - 1);
      for (int t = 0; t < taps; ++t) {
        int c = min(max(first + t, kLo), kXHi);
        if (it.flip) c = WMD_NYU_SRC_W - 1 - c;
        a += static_cast<long long>(row[2 + t]) * src[c];
      }
      tmp_depth[(static_cast<long long>(v) * kRows + y) * d.depth_w + xd] = static_cast<uint8_t>(acc8(a));
    }
  }
}

// image (N, 3, image_h, image_w) then depth (N, 1, depth_h, depth_w): one thread per output pixel of either
__global__ void __launch_bounds__(kT) nyu_inputs_v_kernel(wmd_nyu_inputs_desc d, const uint8_t* __restrict__ tmp_img,
                                                          const uint8_t* __restrict__ tmp_depth) {
  const long long n_img = static_cast<long long>(d.N) * d.image_h * d.image_w;
  const long long total = n_img + static_cast<long long>(d.N) * d.depth_h * d.depth_w;
  for (long long i = static_cast<long long>(blockIdx.x) * kT + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    if (i < n_img) {
      const int x = static_cast<int>(i % d.image_w);
      const long long vy = i / d.image_w;
      const int y = static_cast<int>(vy % d.image_h);
      const int v = static_cast<int>(vy / d.image_h);
      const int32_t* row = d.image_ytab + static_cast<long long>(y) * (d.image_yk + 2);
      const int first = row[0], taps = min(row[1], d.image_yk);
      const uint8_t* src = tmp_img + static_cast<long long>(v) * kRows * d.image_w * 3 + 3 * x;
      long long a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int t = 0; t < taps; ++t) {
        const int r = min(max(first + t, kLo), kYHi) - kLo;
        const uint8_t* s = src + static_cast<long long>(r) * d.image_w * 3;
        const long long wt = row[2 + t];
        a0 += wt * s[0], a1 += wt * s[1], a2 += wt * s[2];
      }
      const long long plane = static_cast<long long>(d.image_h) * d.image_w;
      float* o = d.image + static_cast<long long>(v) * 3 * plane + static_cast<long long>(y) * d.image_w + x;
      o[0] = __fdiv_rn(static_cast<float>(acc8(a0)), 255.f);
      o[plane] = __fdiv_rn(static_cast<float>(acc8(a1)), 255.f);
      o[2 * plane] = __fdiv_rn(static_cast<float>(acc8(a2)), 255.f);
    } else {
      const long long j = i - n_img;
      const int x = static_cast<int>(j % d.depth_w);
      const long long vy = j / d.depth_w;
      const int y = static_cast<int>(vy % d.depth_h);
      const int v = static_cast<int>(vy / d.depth_h);
      const int32_t* row = d.depth_ytab + static_cast<long long>(y) * (d.depth_yk + 2);
      const int first = row[0], taps = min(row[1], d.depth_yk);
      const uint8_t* src = tmp_depth + static_cast<long long>(v) * kRows * d.depth_w + x;
      long long a = 1 << (kPrecisionBits - 1);
      for (int t = 0; t < taps; ++t) {
        const int r = min(max(first + t, kLo), kYHi) - kLo;
        a += static_cast<long long>(row[2 + t]) * src[static_cast<long long>(r) * d.depth_w];
      }
      const float m = __fmul_rn(__fdiv_rn(static_cast<float>(acc8(a)), 255.f), 1000.f);
      d.depth[j] = fminf(fmaxf(m, 10.f), 1000.f);
    }
  }
}

struct NyuWs {
  size_t img, depth, total;
};

bool extent_ok(int v) { return v >= 1 && v <= 32767; }

// the byte offsets of the workspace's pieces; false for a descriptor wmd_nyu_inputs_u8 refuses on shape
bool nyu_ws(const wmd_nyu_inputs_desc& d, NyuWs& w) {
  if (d.N < 0 || d.N > 65535) return false;
  if (!extent_ok(d.image_h) || !extent_ok(d.image_w) || !extent_ok(d.depth_h) || !extent_ok(d.depth_w)) return false;
  const long long n = d.N;
  const long long vals[] = {n * WMD_NYU_SRC_H * WMD_NYU_SRC_W * 3, n * kRows * d.image_w * 3, n * kRows * d.depth_w,
                            n * 3 * d.image_h * d.image_w, n * d.depth_h * d.depth_w,
                            n * (kRows * (d.image_w + d.depth_w)),
                            n * (static_cast<long long>(d.image_h) * d.image_w + static_cast<long long>(d.depth_h) * d.depth_w)};
  for (long long v : vals)
    if (v > 0x7fffffffll) return false;
  size_t o = 0;
  w.img = o, o += up(static_cast<size_t>(vals[1]));
  w.depth = o, o += up(static_cast<size_t>(vals[2]));
  w.total = o;
  return true;
}

}  // namespace
}  // namespace wmd

extern "C" size_t wmd_nyu_inputs_ws_bytes(const wmd_nyu_inputs_desc* d) {
  wmd::NyuWs w;
  if (!d || !wmd::nyu_ws(*d, w)) return 0;
  return w.total;
}

extern "C" int wmd_nyu_inputs_u8(const wmd_nyu_inputs_desc* d, void* ws, size_t ws_bytes, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(d, WMD_ERR_ARG);
  NyuWs w;
  WMD_REQUIRE(nyu_ws(*d, w), WMD_ERR_SHAPE);
  if (d->N == 0) return WMD_OK;
  WMD_REQUIRE(d->image_src && d->depth_src && d->items && d->lut && d->image && d->depth && ws, WMD_ERR_ARG);
  WMD_REQUIRE(d->image_xtab && d->image_ytab && d->depth_xtab && d->depth_ytab, WMD_ERR_ARG);
  WMD_REQUIRE(d->image_xk >= 1 && d->image_yk >= 1 && d->depth_xk >= 1 && d->depth_yk >= 1, WMD_ERR_ARG);
  WMD_REQUIRE(ws_bytes >= w.total, WMD_ERR_WORKSPACE);
  cudaStream_t s = as_stream(stream);
  char* b = static_cast<char*>(ws);
  uint8_t* tmp_img = reinterpret_cast<uint8_t*>(b + w.img);
  uint8_t* tmp_depth = reinterpret_cast<uint8_t*>(b + w.depth);
  const long long nh = static_cast<long long>(d->N) * kRows * (d->image_w + d->depth_w);
  nyu_inputs_h_kernel<<<stride_grid(nh, kT), kT, 0, s>>>(*d, tmp_img, tmp_depth);
  if (int rc = launched()) return rc;
  const long long nv = static_cast<long long>(d->N) *
                       (static_cast<long long>(d->image_h) * d->image_w + static_cast<long long>(d->depth_h) * d->depth_w);
  nyu_inputs_v_kernel<<<stride_grid(nv, kT), kT, 0, s>>>(*d, tmp_img, tmp_depth);
  return launched();
}
