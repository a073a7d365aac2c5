// K6: 3x3 stage of the wavelet coefficient heads (1..4 output channels, optional +/- head pair).
//
// With <= 4 output channels the op has ~13 flop/byte: it is bound by the gathered row reads, not by
// FMAs, so it is not routed through the GEMM tile kernel.  One warp per active output pixel: the 9 tap
// rows are resolved by lanes 0..8 (index map + border rule) and broadcast by shuffle, every lane then
// streams a channel slice of each neighbour row (128-byte coalesced requests) against weights staged
// once per CTA in shared memory, and a butterfly reduction finishes the dot products.  The epilogue
// applies the reference's  scale * (act(a) - act(b))  (depth_decoder.py:133-135,288) and scatters to the
// dense NCHW coefficient tensor (the reference's make_result=True, layers.py:473-478).
#include "common.cuh"

namespace wmd {

template <int COUT>
__global__ void __launch_bounds__(256) head_conv3x3_kernel(const wmd_head_desc d) {
  extern __shared__ __align__(16) float wsm[];
  const int C = d.c;
  const bool dual = d.off_b >= 0;
  const int wcount = 9 * C * COUT;
  float* wa = wsm;
  float* wb = wsm + wcount;
  for (int i = threadIdx.x; i < wcount; i += blockDim.x) {
    wa[i] = __ldg(d.wa + i);
    if (dual) wb[i] = __ldg(d.wb + i);
  }
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const long long HW = static_cast<long long>(d.H) * d.W;
  const int total_px = static_cast<int>(static_cast<long long>(d.N) * HW);
  int rows = d.pixels ? *d.count : total_px;
  rows = min(rows, d.max_rows);

  float ba[COUT], bb[COUT];
#pragma unroll
  for (int j = 0; j < COUT; ++j) {
    ba[j] = d.ba ? __ldg(d.ba + j) : 0.f;
    bb[j] = (dual && d.bb) ? __ldg(d.bb + j) : 0.f;
  }

  for (int m = blockIdx.x * warps_per_block + (threadIdx.x >> 5); m < rows; m += gridDim.x * warps_per_block) {
    const int p = d.pixels ? d.pixels[m] : m;
    const int n = static_cast<int>(p / HW);
    const int rem = static_cast<int>(p - n * HW);
    const int y = rem / d.W, x = rem - y * d.W;
    int my_row = -1;
    if (lane < 9) {
      int qy = y + lane / 3 - 1, qx = x + lane % 3 - 1;
      bool ok = pad_coord(qy, d.H, d.pad_mode);
      ok = pad_coord(qx, d.W, d.pad_mode) && ok;
      if (ok) {
        const int q = (n * d.H + qy) * d.W + qx;
        my_row = d.map ? d.map[q] : q;
      }
    }
    float accA[COUT], accB[COUT];
#pragma unroll
    for (int j = 0; j < COUT; ++j) { accA[j] = 0.f; accB[j] = 0.f; }
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int row = __shfl_sync(0xffffffffu, my_row, tap);
      if (row < 0) continue;   // warp-uniform
      const float* tr = d.t + static_cast<long long>(row) * d.ld;
      const float* wta = wa + tap * C * COUT;
      const float* wtb = wb + tap * C * COUT;
      for (int c = lane; c < C; c += 32) {
        const float a = __ldg(tr + d.off_a + c);
#pragma unroll
        for (int j = 0; j < COUT; ++j) accA[j] = fmaf(a, wta[c * COUT + j], accA[j]);
        if (dual) {
          const float b = __ldg(tr + d.off_b + c);
#pragma unroll
          for (int j = 0; j < COUT; ++j) accB[j] = fmaf(b, wtb[c * COUT + j], accB[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < COUT; ++j) {
      for (int o = 16; o > 0; o >>= 1) {
        accA[j] += __shfl_xor_sync(0xffffffffu, accA[j], o);
        if (dual) accB[j] += __shfl_xor_sync(0xffffffffu, accB[j], o);
      }
    }
    float v = 0.f;
#pragma unroll
    for (int j = 0; j < COUT; ++j) {
      if (lane == j) {
        const float a = activate(accA[j] + ba[j], d.act, 0.f);
        v = dual ? d.scale * (a - activate(accB[j] + bb[j], d.act, 0.f)) : d.scale * a;
      }
    }
    if (lane < COUT) d.out[(static_cast<long long>(n) * COUT + lane) * HW + rem] = v;
  }
}

template <int COUT>
static int launch_head(const wmd_head_desc& d, cudaStream_t stream) {
  const size_t smem = static_cast<size_t>(d.off_b >= 0 ? 2 : 1) * 9 * d.c * COUT * sizeof(float);
  if (smem > 220 * 1024) return WMD_ERR_UNSUPPORTED;
  int rc = record(cudaFuncSetAttribute(head_conv3x3_kernel<COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(smem)));
  if (rc != WMD_OK) return rc;
  const int per_sm = smem > 100 * 1024 ? 1 : (smem > 48 * 1024 ? 2 : 4);
  const long long need = (static_cast<long long>(d.max_rows) + 7) / 8;
  const long long cap = static_cast<long long>(sm_count()) * per_sm;
  const int grid = static_cast<int>(need < cap ? (need < 1 ? 1 : need) : cap);
  head_conv3x3_kernel<COUT><<<grid, 256, smem, stream>>>(d);
  return launched();
}

// ---- factored form of the same 3x3 stage -------------------------------------------------------------------------
// conv3x3 over a gathered neighbourhood = sum over taps of (row . W[tap]).  The row . W[tap] products for all 9 taps
// do not depend on which pixel asks for them, so they are computed ONCE per active input row by the tensor-core
// GEMM (Z = T x Wz, Wz = [tap][group] columns, wmd_conv_rows_* with taps = 1), and this kernel only gathers and adds
// 9 x G floats per output pixel (G = 6 for a +/- pair of 3-channel heads) instead of 9 x 2C: 10-80x less gather
// traffic.  One thread per output pixel; consecutive threads take consecutive active pixels, i.e. neighbours in
// x, so the nine Z rows they touch are mostly adjacent in memory.  VEC (G even, z 8-byte aligned, ldz even: decided on
// the host) reads each tap's G floats as float2 pairs; otherwise scalar loads.  The sums are the same either way.
template <int G, bool VEC>
__global__ void __launch_bounds__(256) head_gather_kernel(const float* __restrict__ z, int ldz,
                                                          const int32_t* __restrict__ map, const float* __restrict__ bias,
                                                          float scale, int act, int dual, int pad_mode,
                                                          const int32_t* __restrict__ pixels, const int32_t* __restrict__ count,
                                                          int max_rows, float* __restrict__ out, int cout, int N, int H, int W) {
  static_assert(!VEC || G % 2 == 0, "float2 loads need an even group count");
  const long long HW = static_cast<long long>(H) * W;
  const int total_px = static_cast<int>(static_cast<long long>(N) * HW);
  int rows = pixels ? *count : total_px;
  rows = min(rows, max_rows);
  float b[G];
#pragma unroll
  for (int g = 0; g < G; ++g) b[g] = bias ? __ldg(bias + g) : 0.f;
  const int step = gridDim.x * blockDim.x;
  for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < rows; m += step) {
    const int p = pixels ? pixels[m] : m;
    const int n = static_cast<int>(p / HW);
    const int rem = static_cast<int>(p - n * HW);
    const int y = rem / W, x = rem - y * W;
    float s[G];
#pragma unroll
    for (int g = 0; g < G; ++g) s[g] = b[g];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      int qy = y + tap / 3 - 1, qx = x + tap % 3 - 1;
      bool ok = pad_coord(qy, H, pad_mode);
      ok = pad_coord(qx, W, pad_mode) && ok;
      if (!ok) continue;
      const int q = (n * H + qy) * W + qx;
      const int row = map ? map[q] : q;
      if (row < 0) continue;
      const float* zr = z + static_cast<long long>(row) * ldz + tap * G;
      if (VEC) {
#pragma unroll
        for (int g = 0; g < G; g += 2) {
          const float2 v = __ldg(reinterpret_cast<const float2*>(zr + g));
          s[g] += v.x;
          s[g + 1] += v.y;
        }
      } else {
#pragma unroll
        for (int g = 0; g < G; ++g) s[g] += __ldg(zr + g);
      }
    }
    if (dual) {
#pragma unroll
      for (int j = 0; j < G / 2; ++j)
        if (j < cout)
          out[(static_cast<long long>(n) * cout + j) * HW + rem] =
              scale * (activate(s[j], act, 0.f) - activate(s[G / 2 + j], act, 0.f));
    } else {
#pragma unroll
      for (int j = 0; j < G; ++j)
        if (j < cout) out[(static_cast<long long>(n) * cout + j) * HW + rem] = scale * activate(s[j], act, 0.f);
    }
  }
}

}  // namespace wmd

extern "C" int wmd_head_gather_f32(const float* z, int ldz, int groups, const int32_t* map, const float* bias, float scale,
                                   int act, int dual, int pad_mode, const int32_t* pixels, const int32_t* count,
                                   int max_rows, float* out, int cout, int N, int H, int W, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(z && out, WMD_ERR_ARG);
  WMD_REQUIRE((pixels == nullptr) == (count == nullptr), WMD_ERR_ARG);
  WMD_REQUIRE(N > 0 && H > 0 && W > 0 && max_rows >= 0 && ldz >= 9 * groups, WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(N) * H * W < (1ll << 31), WMD_ERR_SHAPE);
  WMD_REQUIRE(pad_mode >= WMD_PAD_ZERO && pad_mode <= WMD_PAD_REPLICATE, WMD_ERR_ARG);
  WMD_REQUIRE(act >= WMD_ACT_NONE && act <= WMD_ACT_SIGMOID && act != WMD_ACT_LRELU, WMD_ERR_ARG);
  WMD_REQUIRE(dual ? (groups == 2 * cout) : (groups == cout), WMD_ERR_SHAPE);
  if (pad_mode == WMD_PAD_REFLECT) WMD_REQUIRE(H >= 2 && W >= 2, WMD_ERR_SHAPE);
  if (max_rows == 0) return WMD_OK;
  const int grid = stride_grid(max_rows, 256, 8);
  cudaStream_t st = as_stream(stream);
  // float2 loads need every row's tap block 8-byte aligned: z itself (callers pass z + col0) and an even ldz
  const bool vec = (reinterpret_cast<uintptr_t>(z) & 7) == 0 && ldz % 2 == 0;
#define WMD_LAUNCH_GATHER_V(GG, VV)                                                                                        \
  head_gather_kernel<GG, VV><<<grid, 256, 0, st>>>(z, ldz, map, bias, scale, act, dual, pad_mode, pixels, count, max_rows, \
                                                   out, cout, N, H, W)
#define WMD_LAUNCH_GATHER(GG)              \
  if (vec) WMD_LAUNCH_GATHER_V(GG, true);  \
  else WMD_LAUNCH_GATHER_V(GG, false)
  switch (groups) {
    case 1: WMD_LAUNCH_GATHER_V(1, false); break;
    case 2: WMD_LAUNCH_GATHER(2); break;
    case 3: WMD_LAUNCH_GATHER_V(3, false); break;
    case 4: WMD_LAUNCH_GATHER(4); break;
    case 6: WMD_LAUNCH_GATHER(6); break;
    case 8: WMD_LAUNCH_GATHER(8); break;
    default: return WMD_ERR_UNSUPPORTED;
  }
#undef WMD_LAUNCH_GATHER
#undef WMD_LAUNCH_GATHER_V
  return launched();
}

extern "C" int wmd_head_conv3x3_f32(const wmd_head_desc* dp, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(dp, WMD_ERR_ARG);
  const wmd_head_desc d = *dp;
  WMD_REQUIRE(d.t && d.wa && d.out, WMD_ERR_ARG);
  WMD_REQUIRE(d.off_b < 0 || d.wb, WMD_ERR_ARG);
  WMD_REQUIRE((d.pixels == nullptr) == (d.count == nullptr), WMD_ERR_ARG);
  WMD_REQUIRE(d.N > 0 && d.H > 0 && d.W > 0 && d.c > 0 && d.ld >= d.c && d.off_a >= 0 && d.max_rows >= 0,
              WMD_ERR_SHAPE);
  WMD_REQUIRE(d.off_a + d.c <= d.ld && (d.off_b < 0 || d.off_b + d.c <= d.ld), WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(d.N) * d.H * d.W < (1ll << 31), WMD_ERR_SHAPE);
  WMD_REQUIRE(d.pad_mode >= WMD_PAD_ZERO && d.pad_mode <= WMD_PAD_REPLICATE, WMD_ERR_ARG);
  WMD_REQUIRE(d.act >= WMD_ACT_NONE && d.act <= WMD_ACT_SIGMOID && d.act != WMD_ACT_LRELU, WMD_ERR_ARG);
  if (d.pad_mode == WMD_PAD_REFLECT) WMD_REQUIRE(d.H >= 2 && d.W >= 2, WMD_ERR_SHAPE);
  if (d.max_rows == 0) return WMD_OK;
  switch (d.cout) {
    case 1: return launch_head<1>(d, as_stream(stream));
    case 2: return launch_head<2>(d, as_stream(stream));
    case 3: return launch_head<3>(d, as_stream(stream));
    case 4: return launch_head<4>(d, as_stream(stream));
    default: return WMD_ERR_UNSUPPORTED;
  }
}
