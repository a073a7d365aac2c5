// K6b: the two 1x1 stages of a level's +/- coefficient heads, fused:  z = Wz . lrelu(W1 . x + b1)
//
//   x   rows (M, C)     the level's upconv(i,1) output at the active pixels          (C  = 32 / 64)
//   W1  (N1, C)         1x1 stages of the + and - heads, concatenated (depth_decoder.py:111-120), N1 = 2C
//   Wz  (54, N1)        the heads' 3x3 stages factored into per-row tap products (ops.head_tap_weight): 9 taps x 6 groups
//   z   rows (M, 56)    consumed by head_gather_kernel (9 x 6-float gather-sum, sigma difference, scatter)
//
// Run as two gather-GEMM launches these stages are per-tile-overhead bound on the tensor-core engine (4-8 chunk
// reductions: tile prologue + epilogue cost more than the MMAs) and the intermediate t (M x N1) makes a
// round trip through HBM.  Fused, a row costs C floats read + 56 written (SURVEY 8d puts the low-channel heads on the HBM
// roof); both weight matrices stay in shared memory for the life of the persistent CTA and t never leaves registers:
// the accumulator fragment of GEMM1's n8-tile j IS the A fragment of GEMM2's k-slab j (the k index of an MMA is a dummy,
// so it is permuted to match: logical k = t <- column 2t, k = t+4 <- column 2t+1 of the C fragment).
//
// Math: warp-level mma.sync m16n8k8 tf32, fp32-faithful 3xTF32 (lo*hi + hi*lo + hi*hi, x split by truncation with an
// exact remainder, weights pre-split with round-to-nearest by the pack kernel).  It is a bandwidth-side fusion: the
// tensor work per byte is small (K <= 128).
#include "common.cuh"

namespace wmd {

template <int C, int N1>
struct HeadMlpCfg {
  static constexpr int P1 = C + 16;      // W1 row pitch in floats: pitch % 32 == 16 makes the LDS.128 B loads conflict-free
  static constexpr int P2 = N1 + 8;      // Wz row pitch: pitch % 32 == 8 makes the LDS.64 B loads conflict-free
  static constexpr int NZ = 56;          // 54 outputs padded to 7 n8-tiles (rows 54, 55 of Wz are zero)
  static constexpr int W1_FLOATS = N1 * P1;
  static constexpr int WZ_FLOATS = NZ * P2;
  static constexpr int PACKED = 2 * W1_FLOATS + 2 * WZ_FLOATS + N1;   // [W1 hi | W1 lo | Wz hi | Wz lo | b1]
  static_assert(P1 % 32 == 16 && P2 % 32 == 8, "bank-conflict-free pitches");
  static_assert(C % 16 == 0 && N1 % 32 == 0, "k-steps are taken in pairs, n8-tiles four at a time");
};

__device__ __forceinline__ float tf32_round(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// x = hi + lo with hi = x truncated to tf32 (13 low mantissa bits cleared) and lo the exact remainder
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xFFFFE000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}

// 3xTF32 product accumulate: small terms first
__device__ __forceinline__ void mma3(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], float bh0, float bh1,
                                     float bl0, float bl1) {
  mma_tf32(d, al, __float_as_uint(bh0), __float_as_uint(bh1));
  mma_tf32(d, ah, __float_as_uint(bl0), __float_as_uint(bl1));
  mma_tf32(d, ah, __float_as_uint(bh0), __float_as_uint(bh1));
}

// w1 (N1, C), wz (nz, N1), b1 (N1) or NULL -> packed image the kernel copies into shared memory verbatim
template <int C, int N1>
__global__ void pack_head_mlp_kernel(const float* __restrict__ w1, const float* __restrict__ wz, const float* __restrict__ b1,
                                     int nz, float* __restrict__ out) {
  using Cfg = HeadMlpCfg<C, N1>;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Cfg::PACKED; i += gridDim.x * blockDim.x) {
    float v = 0.f;
    bool lo = false;
    int j = i;
    if (j < 2 * Cfg::W1_FLOATS) {
      lo = j >= Cfg::W1_FLOATS;
      j -= lo ? Cfg::W1_FLOATS : 0;
      const int n = j / Cfg::P1, k = j - n * Cfg::P1;
      if (k < C) v = __ldg(w1 + n * C + k);
    } else if (j < 2 * Cfg::W1_FLOATS + 2 * Cfg::WZ_FLOATS) {
      j -= 2 * Cfg::W1_FLOATS;
      lo = j >= Cfg::WZ_FLOATS;
      j -= lo ? Cfg::WZ_FLOATS : 0;
      const int n = j / Cfg::P2, k = j - n * Cfg::P2;
      if (n < nz && k < N1) v = __ldg(wz + n * N1 + k);
    } else {
      j -= 2 * Cfg::W1_FLOATS + 2 * Cfg::WZ_FLOATS;
      out[i] = b1 ? __ldg(b1 + j) : 0.f;
      continue;
    }
    const float hi = tf32_round(v);
    out[i] = lo ? tf32_round(v - hi) : hi;
  }
}

constexpr int HM_WARPS = 8;                 // 16 rows per warp: 128-row tiles
constexpr int HM_JB = 4;                    // n8-tiles of t in flight per warp (independent accumulation chains)

template <int C, int N1>
__global__ void __launch_bounds__(HM_WARPS * 32, 1)
head_mlp_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ packed, float slope,
                const int32_t* __restrict__ count, int max_rows, float* __restrict__ z, int ldz) {
  using Cfg = HeadMlpCfg<C, N1>;
  extern __shared__ __align__(16) float hm_smem[];
  const float* w1h = hm_smem;
  const float* w1l = w1h + Cfg::W1_FLOATS;
  const float* wzh = w1l + Cfg::W1_FLOATS;
  const float* wzl = wzh + Cfg::WZ_FLOATS;
  const float* b1s = wzl + Cfg::WZ_FLOATS;
  for (int i = threadIdx.x * 4; i < Cfg::PACKED; i += blockDim.x * 4)
    *reinterpret_cast<float4*>(hm_smem + i) = __ldg(reinterpret_cast<const float4*>(packed + i));
  __syncthreads();

  const int rows = count ? min(*count, max_rows) : max_rows;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  const int tiles = (rows + 16 * HM_WARPS - 1) / (16 * HM_WARPS);
  constexpr int KS = C / 8;                 // k-steps of GEMM1

  // raw rows of a warp's 16-row slab: rows g and g+8, this thread's 4 consecutive channels of every 16
  float4 ra[C / 16], rb[C / 16];
  auto load_rows = [&](int tile) {
    const int r0 = tile * (16 * HM_WARPS) + warp * 16;
    const int m_a = r0 + g, m_b = r0 + g + 8;
    const float* pa = x + static_cast<long long>(m_a) * ldx + 4 * t;
    const float* pb = x + static_cast<long long>(m_b) * ldx + 4 * t;
#pragma unroll
    for (int s = 0; s < C / 16; ++s) {
      ra[s] = m_a < rows ? __ldg(reinterpret_cast<const float4*>(pa + 16 * s)) : make_float4(0.f, 0.f, 0.f, 0.f);
      rb[s] = m_b < rows ? __ldg(reinterpret_cast<const float4*>(pb + 16 * s)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };

  int tile = blockIdx.x;
  if (tile < tiles) load_rows(tile);
  for (; tile < tiles; tile += gridDim.x) {
    // A fragments of GEMM1 for every k-step (k permuted: the pair of k-steps 2s, 2s+1 covers channels 16s + 4t + {0,1} / {2,3})
    uint32_t ah[KS][4], al[KS][4];
#pragma unroll
    for (int s = 0; s < C / 16; ++s) {
      split_tf32(ra[s].x, ah[2 * s][0], al[2 * s][0]);
      split_tf32(rb[s].x, ah[2 * s][1], al[2 * s][1]);
      split_tf32(ra[s].y, ah[2 * s][2], al[2 * s][2]);
      split_tf32(rb[s].y, ah[2 * s][3], al[2 * s][3]);
      split_tf32(ra[s].z, ah[2 * s + 1][0], al[2 * s + 1][0]);
      split_tf32(rb[s].z, ah[2 * s + 1][1], al[2 * s + 1][1]);
      split_tf32(ra[s].w, ah[2 * s + 1][2], al[2 * s + 1][2]);
      split_tf32(rb[s].w, ah[2 * s + 1][3], al[2 * s + 1][3]);
    }
    const int next = tile + gridDim.x;
    if (next < tiles) load_rows(next);                       // in flight during this tile's MMAs

    float zacc[Cfg::NZ / 8][4];
#pragma unroll
    for (int q = 0; q < Cfg::NZ / 8; ++q) zacc[q][0] = zacc[q][1] = zacc[q][2] = zacc[q][3] = 0.f;

#pragma unroll 1
    for (int j0 = 0; j0 < N1 / 8; j0 += HM_JB) {
      float tacc[HM_JB][4];
#pragma unroll
      for (int jj = 0; jj < HM_JB; ++jj) tacc[jj][0] = tacc[jj][1] = tacc[jj][2] = tacc[jj][3] = 0.f;
      // GEMM1: t[:, 8j .. 8j+7] for HM_JB n8-tiles; B fragment = W1[8j + g][channels of this thread's k positions]
#pragma unroll
      for (int s = 0; s < C / 16; ++s) {
#pragma unroll
        for (int jj = 0; jj < HM_JB; ++jj) {
          const int off = (8 * (j0 + jj) + g) * Cfg::P1 + 16 * s + 4 * t;
          const float4 bh = *reinterpret_cast<const float4*>(w1h + off);
          const float4 bl = *reinterpret_cast<const float4*>(w1l + off);
          mma3(tacc[jj], ah[2 * s], al[2 * s], bh.x, bh.y, bl.x, bl.y);
          mma3(tacc[jj], ah[2 * s + 1], al[2 * s + 1], bh.z, bh.w, bl.z, bl.w);
        }
      }
      // bias + LeakyReLU, then straight into GEMM2 as the A fragment of k-slab j
#pragma unroll
      for (int jj = 0; jj < HM_JB; ++jj) {
        const int j = j0 + jj;
        const float2 bia = *reinterpret_cast<const float2*>(b1s + 8 * j + 2 * t);
        float v0 = tacc[jj][0] + bia.x, v1 = tacc[jj][1] + bia.y, v2 = tacc[jj][2] + bia.x, v3 = tacc[jj][3] + bia.y;
        v0 = v0 > 0.f ? v0 : v0 * slope;
        v1 = v1 > 0.f ? v1 : v1 * slope;
        v2 = v2 > 0.f ? v2 : v2 * slope;
        v3 = v3 > 0.f ? v3 : v3 * slope;
        uint32_t th[4], tl[4];
        split_tf32(v0, th[0], tl[0]);      // (row g,   k = t)   <- column 2t
        split_tf32(v2, th[1], tl[1]);      // (row g+8, k = t)
        split_tf32(v1, th[2], tl[2]);      // (row g,   k = t+4) <- column 2t+1
        split_tf32(v3, th[3], tl[3]);      // (row g+8, k = t+4)
#pragma unroll
        for (int q = 0; q < Cfg::NZ / 8; ++q) {
          const int off = (8 * q + g) * Cfg::P2 + 8 * j + 2 * t;
          const float2 bh = *reinterpret_cast<const float2*>(wzh + off);
          const float2 bl = *reinterpret_cast<const float2*>(wzl + off);
          mma3(zacc[q], th, tl, bh.x, bh.y, bl.x, bl.y);
        }
      }
    }

    // z rows: fragment (row g | g+8, columns 8q + 2t, +1) -> one full 32-byte sector per 4 lanes
    const int r0 = tile * (16 * HM_WARPS) + warp * 16;
    const int m_a = r0 + g, m_b = r0 + g + 8;
#pragma unroll
    for (int q = 0; q < Cfg::NZ / 8; ++q) {
      const int col = 8 * q + 2 * t;
      if (col + 1 < ldz) {
        if (m_a < rows) *reinterpret_cast<float2*>(z + static_cast<long long>(m_a) * ldz + col) = make_float2(zacc[q][0], zacc[q][1]);
        if (m_b < rows) *reinterpret_cast<float2*>(z + static_cast<long long>(m_b) * ldz + col) = make_float2(zacc[q][2], zacc[q][3]);
      }
    }
  }
}

template <int C, int N1>
static int launch_head_mlp(const float* x, int ldx, const float* packed, float slope, const int32_t* count, int max_rows,
                           float* z, int ldz, cudaStream_t stream) {
  using Cfg = HeadMlpCfg<C, N1>;
  constexpr size_t smem = static_cast<size_t>(Cfg::PACKED) * sizeof(float);
  static bool attr_done[64] = {};                 // per device: the attribute belongs to the device's context
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    const int rc = record(cudaFuncSetAttribute(head_mlp_kernel<C, N1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem)));
    if (rc != WMD_OK) return rc;
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  const int tiles = ceil_div(max_rows, 16 * HM_WARPS);
  const int grid = tiles < sm_count() ? tiles : sm_count();
  head_mlp_kernel<C, N1><<<grid, HM_WARPS * 32, smem, stream>>>(x, ldx, packed, slope, count, max_rows, z, ldz);
  return launched();
}

}  // namespace wmd

extern "C" int wmd_head_mlp_supported(int c, int n1) { return (c == 32 && n1 == 64) || (c == 64 && n1 == 128) ? 1 : 0; }

extern "C" size_t wmd_head_mlp_weight_floats(int c, int n1) {
  using namespace wmd;
  if (c == 32 && n1 == 64) return HeadMlpCfg<32, 64>::PACKED;
  if (c == 64 && n1 == 128) return HeadMlpCfg<64, 128>::PACKED;
  return 0;
}

extern "C" int wmd_pack_head_mlp_f32(const float* w1, const float* wz, const float* b1, int c, int n1, int nz, float* packed,
                                     wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(w1 && wz && packed, WMD_ERR_ARG);
  WMD_REQUIRE(nz >= 1 && nz <= 56, WMD_ERR_SHAPE);
  if (c == 32 && n1 == 64) {
    pack_head_mlp_kernel<32, 64><<<64, 256, 0, as_stream(stream)>>>(w1, wz, b1, nz, packed);
  } else if (c == 64 && n1 == 128) {
    pack_head_mlp_kernel<64, 128><<<64, 256, 0, as_stream(stream)>>>(w1, wz, b1, nz, packed);
  } else {
    return WMD_ERR_UNSUPPORTED;
  }
  return launched();
}

extern "C" int wmd_head_mlp_f32(const float* x, int ldx, int c, const float* packed, int n1, float slope,
                                const int32_t* count, int max_rows, float* z, int ldz, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(x && packed && z, WMD_ERR_ARG);
  WMD_REQUIRE(max_rows >= 0 && ldx >= c && ldx % 4 == 0 && ldz >= 56 && ldz % 2 == 0, WMD_ERR_SHAPE);
  WMD_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(z) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(packed) & 15) == 0,
              WMD_ERR_SHAPE);
  if (max_rows == 0) return WMD_OK;
  if (c == 32 && n1 == 64) return launch_head_mlp<32, 64>(x, ldx, packed, slope, count, max_rows, z, ldz, as_stream(stream));
  if (c == 64 && n1 == 128) return launch_head_mlp<64, 128>(x, ldx, packed, slope, count, max_rows, z, ldz, as_stream(stream));
  return WMD_ERR_UNSUPPORTED;
}
