// Layout helpers: NCHW <-> pixel-major rows (batched tiled transposes through shared memory so both
// sides are coalesced), row gather/scatter at an active-pixel list, conv-weight packing.
#include "common.cuh"

namespace wmd {

constexpr int kTT = 32;

// src (N, C, HW) -> dst (N, HW, ld); columns C..ld-1 zero-filled.
// Tile = 32 channels x 128 pixels.  Read side: a warp streams 128 pixels of one channel as four coalesced 128-byte
// requests; write side: 8 lanes cover the 32 channels of one pixel as float4 (one full 128-byte
// line per pixel).  The 129-float row pitch makes the transposed shared-memory reads conflict-free.
// Tile of the two streaming moves (nchw_to_rows, gather_rows_list): LC channels x LP pixels, template parameters.  The read
// side is contiguous along pixels (LP * 4 bytes per channel row), the write side along channels (LC * 4 bytes per pixel
// row).  The dense transpose uses 32 x 128, the list gather 128 x 32 (A/B of tile shapes: scripts/layout_bench.py).
template <int LC, int LP>
struct LayoutTile {
  static constexpr int kLQ = LC / 4;             // float4 lanes that cover one pixel row of the tile
  static constexpr int kPPW = 32 / kLQ;          // pixel rows one warp store instruction covers
  static_assert(LC % 4 == 0 && kLQ <= 32 && 32 % kLQ == 0 && LP % 32 == 0 && LP % (8 * kPPW) == 0, "tile shape");
  static_assert(sizeof(float) * LC * (LP + 1) + 8 * LP <= 48 * 1024 - 64, "static shared memory");
};
constexpr int kDenseLC = 32, kDenseLP = 128;     // nchw_to_rows (plain and gated)
constexpr int kListLC = 128, kListLP = 32;       // gather_rows_list
//
// GATED: `gate` (N, HW) bytes marks the pixels whose rows a later kernel will read (the sparse decoder reads a skip
// map only under its upsample mask - sparse_upsample, KITTI/layers.py:500).  Reads are skipped per 32-pixel group
// (one 128-byte request) with no marked pixel, writes per unmarked pixel (one 128-byte line), and a tile with no
// marked pixel returns after one 128-byte look at the gate; unmarked rows of dst are left untouched.
// Not GATED, `gate` may still be given: it then only restricts amax, every row is moved.  Either way amax covers exactly
// the marked pixels, so a plain, a gated and a list-based move of the same map under the same mask report the same max.
template <bool GATED, int kLC, int kLP>
__global__ void __launch_bounds__(256) nchw_to_rows_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                           const uint8_t* __restrict__ gate, int C, long long HW,
                                                           int ld, float* __restrict__ amax) {
  constexpr int kLQ = LayoutTile<kLC, kLP>::kLQ, kPPW = LayoutTile<kLC, kLP>::kPPW;
  __shared__ float tile[kLC][kLP + 1];
  __shared__ unsigned marked[kLP / 32];
  const int n = blockIdx.z;
  const long long p0 = static_cast<long long>(blockIdx.x) * kLP;
  const int c0 = blockIdx.y * kLC;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool masked = gate != nullptr;
  if (masked) {
    if (warp < kLP / 32) {
      const long long p = p0 + 32 * warp + lane;
      const bool on = p < HW && gate[static_cast<long long>(n) * HW + p] != 0;
      const unsigned m = __ballot_sync(0xffffffffu, on);
      if (lane == 0) marked[warp] = m;
    }
    __syncthreads();
  }
  if (GATED) {
    unsigned any = 0u;
#pragma unroll
    for (int j = 0; j < kLP / 32; ++j) any |= marked[j];
    if (any == 0u) return;
  }
  const float* s = src + static_cast<long long>(n) * C * HW;
  float* d = dst + static_cast<long long>(n) * HW * ld;
  float vmax = 0.f;
  // all loads of the thread are issued before the first one is used: predicates only, no branch between two loads (a
  // `continue` per skipped group made every load wait for the previous one's shared-memory store - 4x slower than the
  // plain transpose at 35 % density)
  bool want[kLP / 32];
#pragma unroll
  for (int j = 0; j < kLP / 32; ++j) want[j] = !GATED || marked[j] != 0u;
  float v[kLC / 8][kLP / 32];
#pragma unroll
  for (int i = 0; i < kLC / 8; ++i) {
    const int c = c0 + warp + 8 * i;
    const float* row = s + static_cast<long long>(c) * HW;
#pragma unroll
    for (int j = 0; j < kLP / 32; ++j) {          // fully coalesced 128-byte requests along the channel row
      const long long p = p0 + lane + 32 * j;
      v[i][j] = (want[j] && c < C && p < HW) ? __ldg(row + p) : 0.f;
    }
  }
#pragma unroll
  for (int i = 0; i < kLC / 8; ++i) {
#pragma unroll
    for (int j = 0; j < kLP / 32; ++j) {
      tile[warp + 8 * i][lane + 32 * j] = v[i][j];
      if (!masked || ((marked[j] >> lane) & 1u)) vmax = fmaxf(vmax, finite_abs(v[i][j]));
    }
  }
  if (amax) {                                    // max |x| (of the marked pixels), for the consumers' fp16 operand scaling
    for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if (lane == 0 && vmax > __ldcg(amax)) atomicMax(reinterpret_cast<unsigned*>(amax), __float_as_uint(vmax));   // most warps skip the atomic
  }
  __syncthreads();
  const int q = lane % kLQ;                      // channel quad of this lane
  const bool vec_out = (ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(d) & 15) == 0);
#pragma unroll
  for (int it = 0; it < kLP / (8 * kPPW); ++it) {
    const int pl = it * 8 * kPPW + warp * kPPW + lane / kLQ;  // pixel within the tile
    const long long p = p0 + pl;
    const int c = c0 + 4 * q;
    if (GATED && ((marked[pl >> 5] >> (pl & 31)) & 1u) == 0u) continue;
    if (p < HW && c < ld) {
      const float4 o = make_float4(tile[4 * q][pl], tile[4 * q + 1][pl], tile[4 * q + 2][pl], tile[4 * q + 3][pl]);
      float* out = d + p * ld + c;
      if (vec_out && c + 3 < ld) {
        *reinterpret_cast<float4*>(out) = o;
      } else {
        out[0] = o.x;
        if (c + 1 < ld) out[1] = o.y;
        if (c + 2 < ld) out[2] = o.z;
        if (c + 3 < ld) out[3] = o.w;
      }
    }
  }
}

// src (N, HW, ld) -> dst (N, C, HW)
__global__ void __launch_bounds__(256) rows_to_nchw_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                           int C, long long HW, int ld) {
  __shared__ float tile[kTT][kTT + 1];
  const int n = blockIdx.z;
  const long long p0 = static_cast<long long>(blockIdx.x) * kTT;
  const int c0 = blockIdx.y * kTT;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float* s = src + static_cast<long long>(n) * HW * ld;
  float* d = dst + static_cast<long long>(n) * C * HW;
  for (int r = ty; r < kTT; r += 8) {
    const long long p = p0 + r;
    const int c = c0 + tx;
    tile[r][tx] = (p < HW && c < C) ? __ldg(s + p * ld + c) : 0.f;
  }
  __syncthreads();
  for (int r = ty; r < kTT; r += 8) {
    const int c = c0 + r;
    const long long p = p0 + tx;
    if (c < C && p < HW) d[static_cast<long long>(c) * HW + p] = tile[tx][r];
  }
}

// rows[m][c] = src[n, c, y, x] for the m-th listed pixel.  One warp handles 32 consecutive rows of one
// 32-channel slab through a shared tile so the NCHW side is read along x and the row side written along c.
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ src, float* __restrict__ rows,
                                                          int ld, int C, const int32_t* __restrict__ pixels,
                                                          const int32_t* __restrict__ count, int max_rows,
                                                          long long HW) {
  __shared__ float tile[kTT][kTT + 1];
  __shared__ int32_t pix[kTT];
  const int M = count ? min(*count, max_rows) : max_rows;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int ctiles = (C + kTT - 1) / kTT;
  const long long tiles = static_cast<long long>((M + kTT - 1) / kTT) * ctiles;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int m0 = static_cast<int>(t / ctiles) * kTT;
    const int c0 = static_cast<int>(t % ctiles) * kTT;
    if (threadIdx.x < kTT) {
      const int mm = m0 + static_cast<int>(threadIdx.x);
      pix[threadIdx.x] = mm < M ? (pixels ? pixels[mm] : mm) : -1;
    }
    __syncthreads();
    for (int r = ty; r < kTT; r += 8) {   // r: channel within slab, tx: row within tile
      const int c = c0 + r;
      const int32_t p = pix[tx];
      float v = 0.f;
      if (p >= 0 && c < C) {
        const long long n = p / HW, rem = p % HW;
        v = __ldg(src + (n * C + c) * HW + rem);
      }
      tile[r][tx] = v;
    }
    __syncthreads();
    for (int r = ty; r < kTT; r += 8) {   // r: row within tile, tx: channel
      const int m = m0 + r, c = c0 + tx;
      if (m < M && c < C) rows[static_cast<long long>(m) * ld + c] = tile[tx][r];
    }
    __syncthreads();
  }
}

// rows[m][c] = src[n, c, y, x] for the m-th listed pixel, at streaming speed for clustered lists.  Tile = 128 list entries
// x 32 channels (the shape of nchw_to_rows): the plane offsets of the 128 pixels are decoded once into shared memory; a
// warp then reads one channel of the 128 pixels as four requests (consecutive list entries are mostly consecutive pixels:
// 128-byte requests inside a run) and the write side covers each row's 32 channels with eight float4 lanes (one full
// 128-byte line per row).  Columns C..ld-1 are zero-filled.  src may be pinned host memory.
template <int kLC, int kLP>
__global__ void __launch_bounds__(256) gather_rows_list_kernel(const float* __restrict__ src, float* __restrict__ rows,
                                                               int ld, int C, const int32_t* __restrict__ pixels,
                                                               const int32_t* __restrict__ count, int max_rows,
                                                               unsigned HW, float* __restrict__ amax) {
  constexpr int kLQ = LayoutTile<kLC, kLP>::kLQ, kPPW = LayoutTile<kLC, kLP>::kPPW;
  __shared__ float tile[kLC][kLP + 1];
  __shared__ long long base[kLP];
  float vmax = 0.f;                              // (n*C)*HW + yx of the tile's pixels, -1 past the list
  const int M = count ? min(*count, max_rows) : max_rows;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ctiles = (ld + kLC - 1) / kLC;
  const long long tiles = static_cast<long long>((M + kLP - 1) / kLP) * ctiles;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int m0 = static_cast<int>(t / ctiles) * kLP;
    const int c0 = static_cast<int>(t % ctiles) * kLC;
    if (threadIdx.x < kLP) {
      const int mm = m0 + static_cast<int>(threadIdx.x);
      long long b = -1;
      if (mm < M) {
        const unsigned p = static_cast<unsigned>(pixels ? pixels[mm] : mm);
        const unsigned n = p / HW;
        b = static_cast<long long>(n) * C * HW + (p - n * HW);
      }
      base[threadIdx.x] = b;
    }
    __syncthreads();
#pragma unroll
    for (int r = warp; r < kLC; r += 8) {
      const int c = c0 + r;
      const long long coff = static_cast<long long>(c) * HW;
#pragma unroll
      for (int j = 0; j < kLP / 32; ++j) {
        const long long b = base[lane + 32 * j];
        const float v = (c < C && b >= 0) ? __ldg(src + b + coff) : 0.f;
        tile[r][lane + 32 * j] = v;
        vmax = fmaxf(vmax, finite_abs(v));
      }
    }
    __syncthreads();
    const int q = lane % kLQ;
#pragma unroll
    for (int it = 0; it < kLP / (8 * kPPW); ++it) {
      const int pl = it * 8 * kPPW + warp * kPPW + lane / kLQ;
      const int m = m0 + pl;
      const int c = c0 + 4 * q;
      if (m < M && c < ld)
        *reinterpret_cast<float4*>(rows + static_cast<long long>(m) * ld + c) =
            make_float4(tile[4 * q][pl], tile[4 * q + 1][pl], tile[4 * q + 2][pl], tile[4 * q + 3][pl]);
    }
    __syncthreads();
  }
  if (amax) {                                    // max |x| of the gathered rows, for the consumer's fp16 operand scaling
    for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if (lane == 0 && vmax > __ldcg(amax)) atomicMax(reinterpret_cast<unsigned*>(amax), __float_as_uint(vmax));   // most warps skip the atomic
  }
}

__global__ void __launch_bounds__(256) scatter_rows_kernel(const float* __restrict__ rows, int ld, int C,
                                                           const int32_t* __restrict__ pixels,
                                                           const int32_t* __restrict__ count, int max_rows,
                                                           float* __restrict__ dst, long long HW) {
  __shared__ float tile[kTT][kTT + 1];
  __shared__ int32_t pix[kTT];
  const int M = count ? min(*count, max_rows) : max_rows;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int ctiles = (C + kTT - 1) / kTT;
  const long long tiles = static_cast<long long>((M + kTT - 1) / kTT) * ctiles;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int m0 = static_cast<int>(t / ctiles) * kTT;
    const int c0 = static_cast<int>(t % ctiles) * kTT;
    if (threadIdx.x < kTT) {
      const int mm = m0 + static_cast<int>(threadIdx.x);
      pix[threadIdx.x] = mm < M ? (pixels ? pixels[mm] : mm) : -1;
    }
    __syncthreads();
    for (int r = ty; r < kTT; r += 8) {   // r: row within tile, tx: channel
      const int m = m0 + r, c = c0 + tx;
      tile[r][tx] = (m < M && c < C) ? __ldg(rows + static_cast<long long>(m) * ld + c) : 0.f;
    }
    __syncthreads();
    for (int r = ty; r < kTT; r += 8) {   // r: channel, tx: row
      const int c = c0 + r;
      const int32_t p = pix[tx];
      if (p >= 0 && c < C) {
        const long long n = p / HW, rem = p % HW;
        dst[(n * C + c) * HW + rem] = tile[tx][r];
      }
    }
    __syncthreads();
  }
}

// w (Cout, Cin, taps) -> packed [taps][Cin][ldw]
__global__ void pack_weight_kernel(const float* __restrict__ w, float* __restrict__ packed, int Cout, int Cin,
                                   int taps, int ldw) {
  const long long total = static_cast<long long>(taps) * Cin * ldw;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += step) {
    const int co = static_cast<int>(i % ldw);
    const long long r = i / ldw;
    const int ci = static_cast<int>(r % Cin);
    const int tap = static_cast<int>(r / Cin);
    packed[i] = co < Cout ? __ldg(w + (static_cast<long long>(co) * Cin + ci) * taps + tap) : 0.f;
  }
}

}  // namespace wmd

extern "C" int wmd_nchw_to_rows_f32(const float* src, float* dst, int N, int C, long long HW, int ld,
                                    wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src && dst, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && C > 0 && HW > 0 && ld >= C && N <= 65535, WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  dim3 grid(ceil_div(HW, kDenseLP), ceil_div(ld, kDenseLC), N);
  WMD_REQUIRE(grid.y <= 65535, WMD_ERR_SHAPE);
  nchw_to_rows_kernel<false, kDenseLC, kDenseLP><<<grid, 256, 0, as_stream(stream)>>>(src, dst, nullptr, C, HW, ld, nullptr);
  return launched();
}

extern "C" int wmd_nchw_to_rows_gated_f32(const float* src, float* dst, const uint8_t* gate, int N, int C,
                                          long long HW, int ld, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src && dst && gate, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && C > 0 && HW > 0 && ld >= C && N <= 65535, WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  dim3 grid(ceil_div(HW, kDenseLP), ceil_div(ld, kDenseLC), N);
  WMD_REQUIRE(grid.y <= 65535, WMD_ERR_SHAPE);
  nchw_to_rows_kernel<true, kDenseLC, kDenseLP><<<grid, 256, 0, as_stream(stream)>>>(src, dst, gate, C, HW, ld, nullptr);
  return launched();
}

extern "C" int wmd_nchw_to_rows_gated_amax_f32(const float* src, float* dst, const uint8_t* gate, int N, int C,
                                               long long HW, int ld, float* amax, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src && dst && gate, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && C > 0 && HW > 0 && ld >= C && N <= 65535, WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  dim3 grid(ceil_div(HW, kDenseLP), ceil_div(ld, kDenseLC), N);
  WMD_REQUIRE(grid.y <= 65535, WMD_ERR_SHAPE);
  nchw_to_rows_kernel<true, kDenseLC, kDenseLP><<<grid, 256, 0, as_stream(stream)>>>(src, dst, gate, C, HW, ld, amax);
  return launched();
}

extern "C" int wmd_rows_to_nchw_f32(const float* src, float* dst, int N, int C, long long HW, int ld,
                                    wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src && dst, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && C > 0 && HW > 0 && ld >= C && N <= 65535, WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  dim3 grid(ceil_div(HW, kTT), ceil_div(C, kTT), N);
  WMD_REQUIRE(grid.y <= 65535, WMD_ERR_SHAPE);
  rows_to_nchw_kernel<<<grid, 256, 0, as_stream(stream)>>>(src, dst, C, HW, ld);
  return launched();
}

extern "C" int wmd_gather_rows_nchw_f32(const float* src_nchw, float* rows, int ld, int C, const int32_t* pixels,
                                        const int32_t* count, int max_rows, int N, int H, int W,
                                        wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src_nchw && rows, WMD_ERR_ARG);
  WMD_REQUIRE(C > 0 && ld >= C && N > 0 && H > 0 && W > 0 && max_rows >= 0, WMD_ERR_SHAPE);
  if (max_rows == 0) return WMD_OK;
  const long long tiles = static_cast<long long>(ceil_div(max_rows, kTT)) * ceil_div(C, kTT);
  gather_rows_kernel<<<stride_grid(tiles * 256, 256, 4), 256, 0, as_stream(stream)>>>(
      src_nchw, rows, ld, C, pixels, count, max_rows, static_cast<long long>(H) * W);
  return launched();
}

extern "C" int wmd_gather_rows_list_f32(const float* src_nchw, float* rows, int ld, int C, const int32_t* pixels,
                                        const int32_t* count, int max_rows, int N, int H, int W, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src_nchw && rows, WMD_ERR_ARG);
  WMD_REQUIRE((pixels == nullptr) == (count == nullptr), WMD_ERR_ARG);
  WMD_REQUIRE(C > 0 && ld >= C && ld % 4 == 0 && N >= 0 && H > 0 && W > 0 && max_rows >= 0, WMD_ERR_SHAPE);
  WMD_REQUIRE((reinterpret_cast<uintptr_t>(rows) & 15) == 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(N) * H * W < (1ll << 31), WMD_ERR_SHAPE);
  if (max_rows == 0 || N == 0) return WMD_OK;
  const long long tiles = static_cast<long long>(ceil_div(max_rows, kListLP)) * ceil_div(ld, kListLC);
  gather_rows_list_kernel<kListLC, kListLP><<<stride_grid(tiles * 256, 256, 6), 256, 0, as_stream(stream)>>>(
      src_nchw, rows, ld, C, pixels, count, max_rows, static_cast<unsigned>(static_cast<long long>(H) * W), nullptr);
  return launched();
}

extern "C" int wmd_gather_rows_list_amax_f32(const float* src_nchw, float* rows, int ld, int C, const int32_t* pixels,
                                             const int32_t* count, int max_rows, int N, int H, int W, float* amax,
                                             wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src_nchw && rows, WMD_ERR_ARG);
  WMD_REQUIRE((pixels == nullptr) == (count == nullptr), WMD_ERR_ARG);
  WMD_REQUIRE(C > 0 && ld >= C && ld % 4 == 0 && N >= 0 && H > 0 && W > 0 && max_rows >= 0, WMD_ERR_SHAPE);
  WMD_REQUIRE((reinterpret_cast<uintptr_t>(rows) & 15) == 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(N) * H * W < (1ll << 31), WMD_ERR_SHAPE);
  if (max_rows == 0 || N == 0) return WMD_OK;
  const long long tiles = static_cast<long long>(ceil_div(max_rows, kListLP)) * ceil_div(ld, kListLC);
  gather_rows_list_kernel<kListLC, kListLP><<<stride_grid(tiles * 256, 256, 6), 256, 0, as_stream(stream)>>>(
      src_nchw, rows, ld, C, pixels, count, max_rows, static_cast<unsigned>(static_cast<long long>(H) * W), amax);
  return launched();
}

extern "C" int wmd_nchw_to_rows_amax_f32(const float* src, float* dst, int N, int C, long long HW, int ld, float* amax,
                                         wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src && dst, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && C > 0 && HW > 0 && ld >= C && N <= 65535, WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  dim3 grid(ceil_div(HW, kDenseLP), ceil_div(ld, kDenseLC), N);
  WMD_REQUIRE(grid.y <= 65535, WMD_ERR_SHAPE);
  nchw_to_rows_kernel<false, kDenseLC, kDenseLP><<<grid, 256, 0, as_stream(stream)>>>(src, dst, nullptr, C, HW, ld, amax);
  return launched();
}

extern "C" int wmd_nchw_to_rows_masked_amax_f32(const float* src, float* dst, const uint8_t* mask, int N, int C,
                                                long long HW, int ld, float* amax, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(src && dst && mask && amax, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && C > 0 && HW > 0 && ld >= C && N <= 65535, WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  dim3 grid(ceil_div(HW, kDenseLP), ceil_div(ld, kDenseLC), N);
  WMD_REQUIRE(grid.y <= 65535, WMD_ERR_SHAPE);
  nchw_to_rows_kernel<false, kDenseLC, kDenseLP><<<grid, 256, 0, as_stream(stream)>>>(src, dst, mask, C, HW, ld, amax);
  return launched();
}

extern "C" int wmd_scatter_rows_nchw_f32(const float* rows, int ld, int C, const int32_t* pixels, const int32_t* count,
                                         int max_rows, float* dst_nchw, int N, int H, int W, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(rows && dst_nchw, WMD_ERR_ARG);
  WMD_REQUIRE(C > 0 && ld >= C && N > 0 && H > 0 && W > 0 && max_rows >= 0, WMD_ERR_SHAPE);
  if (max_rows == 0) return WMD_OK;
  const long long tiles = static_cast<long long>(ceil_div(max_rows, kTT)) * ceil_div(C, kTT);
  scatter_rows_kernel<<<stride_grid(tiles * 256, 256, 4), 256, 0, as_stream(stream)>>>(
      rows, ld, C, pixels, count, max_rows, dst_nchw, static_cast<long long>(H) * W);
  return launched();
}

extern "C" int wmd_pack_conv_weight_f32(const float* w, float* packed, int Cout, int Cin, int taps, int ldw,
                                        wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(w && packed, WMD_ERR_ARG);
  WMD_REQUIRE(Cout > 0 && Cin > 0 && taps > 0 && ldw >= Cout, WMD_ERR_SHAPE);
  const long long total = static_cast<long long>(taps) * Cin * ldw;
  pack_weight_kernel<<<stride_grid(total, 256), 256, 0, as_stream(stream)>>>(w, packed, Cout, Cin, taps, ldw);
  return launched();
}
