// KITTI's ground-truth depth maps from velodyne scans (include/wmd_gt.h): generate_depth_map of KITTI/kitti_utils.py,
// bit for bit, for a batch of frames with ragged point counts.
//
// Two passes per chunk of frames.  The point pass projects every point once and records, per pixel, the last point on
// it (atomicMax) and, per duplicate group, its first point (atomicMin), its size (atomicAdd) and its least depth
// (atomicMin of an order-preserving key).  The pixel pass recomputes the depth of each pixel's last point with the same
// code and, on the pixel of a duplicate group's first point, takes the group's least depth instead.  Integer atomics
// commute, so the result does not depend on the order the points are visited in.
#include <stdint.h>

#include "common.cuh"
#include "wmd_gt.h"

namespace wmd {
namespace {

constexpr int kT = 256;
constexpr int kChunk = 256;                          // frames per launch: their sizes travel as a kernel argument
constexpr unsigned long long kZeroKey = 1ull << 63;  // keys of zero depths start here; positive depths above 2^32 more
constexpr long long kMaxCount = 1ll << 30;           // pixels per frame and points per batch, so int loops never wrap
constexpr size_t kAlign = 256;

inline size_t up(size_t b) { return (b + kAlign - 1) / kAlign * kAlign; }

struct FrameSizes {
  int32_t hw[2 * kChunk];                            // (H, W) of the chunk's frames
};

struct VeloWs {
  size_t zmin, last, first, count, total;
};

VeloWs velo_ws(long long pixels) {
  VeloWs w;
  size_t o = 0;
  w.zmin = o;  o += up(pixels * sizeof(unsigned long long));
  w.last = o;  o += up(pixels * sizeof(int));
  w.first = o; o += up(pixels * sizeof(unsigned));
  w.count = o; o += up(pixels * sizeof(int));
  w.total = o;
  return w;
}

bool velo_shape(int N, int Hmax, int Wmax, long long total_points) {
  return N >= 0 && Hmax >= 1 && Wmax >= 1 && static_cast<long long>(Hmax) * Wmax <= kMaxCount && total_points >= 0 &&
         total_points <= kMaxCount &&
         static_cast<unsigned long long>(N) * Hmax * Wmax <= (SIZE_MAX - 4096) / 32;
}

struct Hit {
  int pixel;      // v' W + u'
  int group;      // g + 1 = v' (W - 1) + u', in [0, H W - H]
  double depth;
};

// steps 1-4 of the contract for one point; explicit round-to-nearest intrinsics, so no contraction changes the bits
__device__ __forceinline__ bool velo_project(const float4 p, const double (&P)[12], int H, int W, bool vel_depth,
                                             Hit& h) {
  const double x = p.x, y = p.y, z = p.z;
  if (!(x >= 0.0)) return false;
  double q[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    q[r] = __dadd_rn(__fma_rn(P[4 * r + 2], z, __fma_rn(P[4 * r + 1], y, __dmul_rn(P[4 * r], x))), P[4 * r + 3]);
  const double u = __dsub_rn(rint(__ddiv_rn(q[0], q[2])), 1.0);
  const double v = __dsub_rn(rint(__ddiv_rn(q[1], q[2])), 1.0);
  if (!(u >= 0.0 && v >= 0.0 && u < static_cast<double>(W) && v < static_cast<double>(H))) return false;
  const int iu = static_cast<int>(u), iv = static_cast<int>(v);
  h.pixel = iv * W + iu;
  h.group = iv * (W - 1) + iu;
  h.depth = vel_depth ? x : q[2];
  return true;
}

// Order-preserving key of a depth: negatives below every zero, zeros (either sign) below every positive.  Zeros carry
// the point instead of their sign, the later point with the smaller key, so that the minimum of a group whose least
// depth is zero is the later zero, as numpy's min returns it.
__device__ __forceinline__ unsigned long long depth_key(double d, int j) {
  const unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(d));
  if (d == 0.0) return kZeroKey + (0xffffffffull - static_cast<unsigned>(j));
  if (b >> 63) return ~b;
  return kZeroKey + (1ull << 32) + b;
}

__device__ __forceinline__ void load_camera(const double* P, int n, double (&cam)[12]) {
#pragma unroll
  for (int i = 0; i < 12; ++i) cam[i] = P[12 * static_cast<long long>(n) + i];
}

__global__ void __launch_bounds__(kT) velo_points_kernel(const float4* __restrict__ points,
                                                         const int32_t* __restrict__ offsets,
                                                         const double* __restrict__ P, const FrameSizes sz, int f0,
                                                         int nf, long long S, int vel_depth,
                                                         unsigned long long* __restrict__ zmin, int* __restrict__ last,
                                                         unsigned* __restrict__ first, int* __restrict__ count) {
  for (int k = blockIdx.y; k < nf; k += gridDim.y) {
    const int n = f0 + k, H = sz.hw[2 * k], W = sz.hw[2 * k + 1];
    double cam[12];
    load_camera(P, n, cam);
    const int b = offsets[n], e = offsets[n + 1];
    const long long base = n * S;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < e - b; j += gridDim.x * blockDim.x) {
      Hit h;
      if (!velo_project(points[static_cast<long long>(b) + j], cam, H, W, vel_depth != 0, h)) continue;
      atomicMax(last + base + h.pixel, j);
      atomicMin(first + base + h.group, static_cast<unsigned>(j));
      atomicAdd(count + base + h.group, 1);
      atomicMin(zmin + base + h.group, depth_key(h.depth, j));
    }
  }
}

__global__ void __launch_bounds__(kT) velo_pixels_kernel(const float4* __restrict__ points,
                                                         const int32_t* __restrict__ offsets,
                                                         const double* __restrict__ P, const FrameSizes sz, int f0,
                                                         int nf, int Wmax, long long S, int vel_depth,
                                                         const unsigned long long* __restrict__ zmin,
                                                         const int* __restrict__ last,
                                                         const unsigned* __restrict__ first,
                                                         const int* __restrict__ count, double* __restrict__ depth) {
  for (int k = blockIdx.y; k < nf; k += gridDim.y) {
    const int n = f0 + k, H = sz.hw[2 * k], W = sz.hw[2 * k + 1];
    double cam[12];
    load_camera(P, n, cam);
    const long long b = offsets[n], base = n * S;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < S; i += gridDim.x * blockDim.x) {
      const int y = i / Wmax, x = i - y * Wmax;
      double out = 0.0;
      const int j = (y < H && x < W) ? last[base + y * W + x] : -1;
      Hit h;
      if (j >= 0 && velo_project(points[b + j], cam, H, W, vel_depth != 0, h)) {
        out = h.depth;
        Hit hf;
        if (count[base + h.group] > 1 &&
            velo_project(points[b + first[base + h.group]], cam, H, W, vel_depth != 0, hf) && hf.pixel == h.pixel) {
          const unsigned long long key = zmin[base + h.group];
          if (key < kZeroKey) {
            out = __longlong_as_double(static_cast<long long>(~key));
          } else if (key < kZeroKey + (1ull << 32)) {          // a zero: its sign is that of the point it names
            const unsigned jz = 0xffffffffu - static_cast<unsigned>(key - kZeroKey);
            Hit hz;
            out = velo_project(points[b + jz], cam, H, W, vel_depth != 0, hz) ? hz.depth : 0.0;
          } else {
            out = __longlong_as_double(static_cast<long long>(key - kZeroKey - (1ull << 32)));
          }
        }
        if (out < 0.0) out = 0.0;
      }
      depth[base + i] = out;
    }
  }
}

}  // namespace
}  // namespace wmd

extern "C" size_t wmd_velo_depth_ws_bytes(int32_t N, int32_t Hmax, int32_t Wmax, long long total_points) {
  if (!wmd::velo_shape(N, Hmax, Wmax, total_points)) return 0;
  return wmd::velo_ws(static_cast<long long>(N) * Hmax * Wmax).total;
}

extern "C" int wmd_velo_depth_f64(const float* points, const int32_t* offsets, const double* P,
                                  const int32_t* sizes_host, int32_t N, int32_t Hmax, int32_t Wmax, int32_t vel_depth,
                                  void* ws, size_t ws_bytes, double* depth, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(velo_shape(N, Hmax, Wmax, 0), WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  WMD_REQUIRE(points && offsets && P && sizes_host && ws && depth, WMD_ERR_ARG);
  WMD_REQUIRE(reinterpret_cast<uintptr_t>(points) % 16 == 0, WMD_ERR_ARG);
  for (int n = 0; n < N; ++n) {
    const int H = sizes_host[2 * n], W = sizes_host[2 * n + 1];
    WMD_REQUIRE(H >= 1 && W >= 1 && H <= Hmax && W <= Wmax, WMD_ERR_SHAPE);
  }
  const long long S = static_cast<long long>(Hmax) * Wmax;
  const VeloWs w = velo_ws(N * S);
  WMD_REQUIRE(ws_bytes >= w.total, WMD_ERR_WORKSPACE);
  cudaStream_t st = as_stream(stream);
  char* base = static_cast<char*>(ws);
  auto* zmin = reinterpret_cast<unsigned long long*>(base + w.zmin);
  int* last = reinterpret_cast<int*>(base + w.last);
  auto* first = reinterpret_cast<unsigned*>(base + w.first);
  int* count = reinterpret_cast<int*>(base + w.count);
  // zmin, last and first start at all ones (no key, no point, no point), count at zero
  if (int rc = record(cudaMemsetAsync(base, 0xff, w.count, st))) return rc;
  if (int rc = record(cudaMemsetAsync(count, 0, w.total - w.count, st))) return rc;
  const float4* pts = reinterpret_cast<const float4*>(points);
  for (int f0 = 0; f0 < N; f0 += kChunk) {
    const int nf = N - f0 < kChunk ? N - f0 : kChunk;
    FrameSizes sz = {};
    for (int k = 0; k < 2 * nf; ++k) sz.hw[k] = sizes_host[2 * f0 + k];
    const int per_frame = ceil_div(static_cast<long long>(sm_count()) * 16, nf);
    const dim3 grid_points(per_frame, nf);
    velo_points_kernel<<<grid_points, kT, 0, st>>>(pts, offsets, P, sz, f0, nf, S, vel_depth, zmin, last, first,
                                                     count);
    if (int rc = launched()) return rc;
    const dim3 grid_pixels(ceil_div(S, kT) < per_frame ? ceil_div(S, kT) : per_frame, nf);
    velo_pixels_kernel<<<grid_pixels, kT, 0, st>>>(pts, offsets, P, sz, f0, nf, Wmax, S, vel_depth, zmin, last, first,
                                                     count, depth);
    if (int rc = launched()) return rc;
  }
  return WMD_OK;
}
