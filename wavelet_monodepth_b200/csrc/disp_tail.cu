// K7: the full-resolution tail of monodepth2's baseline decoder (depth_decoder.py:18-69, level 0), in one launch:
//
//   u    = ELU(b1 + sum up2(x) * W1)      upconv(0,1): nearest x2, 3x3 with ZERO padding, 16 -> 16 channels
//   disp = sigmoid(b2 + sum u * W2)       dispconv(0): 3x3 with REFLECT padding, 16 -> cout (1..4) channels
//
//   x     rows (N*H*W, ld >= 16) at half resolution: upconv(0,0)'s post-ELU output as wmd_conv_rows_f32 writes it
//   disp  (N, cout, 2H, 2W) NCHW
//
// As two launches the 16-channel map u is the largest tensor of the decoder (10.5 M pixels x 64 B at R50 1024x320 x 32):
// written once, then read back by the dispconv's gather.  Here it never leaves shared memory.  A persistent CTA walks
// 16 x 32 full-resolution output tiles.  Per tile it
//   1. stages the 10 x 18 half-resolution source pixels the tile needs (zeros outside the image = the zero padding of the
//      upsampled map, since up2 maps an outside coordinate to an outside source pixel);
//   2. computes u over the 18 x 34 halo on mma.sync m16n8k8 with the 3xTF32 split of head_mlp.cu (M = 612 pixels,
//      N = 16, K = 144).  A halo pixel outside the image holds u at the REFLECTED coordinate, so the dispconv's reflection
//      padding is exact and the second stage needs no border logic;
//   3. finishes every output pixel from the u halo with 144 * cout fp32 FMAs and stores it to NCHW.
#include "common.cuh"

namespace wmd {

namespace dt {
constexpr int TH = 16, TW = 32;               // output tile (full resolution)
constexpr int UH = TH + 2, UW = TW + 2;       // u halo
constexpr int UPIX = UH * UW;                 // 612
constexpr int MT = (UPIX + 15) / 16;          // 39 m16 tiles
constexpr int PH = TH / 2 + 2, PW = TW / 2 + 2;   // staged source patch (half resolution): 10 x 18
constexpr int PPIX = PH * PW;
constexpr int CP = 20;                        // channel pitch of the patch and of u: 8 consecutive pixels' float4 reads
                                              // cover all 32 banks
constexpr int KP = 148;                       // W1 row pitch: pitch % 32 == 20 makes the B fragment loads conflict-free
constexpr int W1F = 16 * KP;                  // one of the two W1 images (tf32 hi / lo), [n][k = tap*16 + ci]
constexpr int OFF_B1 = 2 * W1F;
constexpr int OFF_W2 = OFF_B1 + 16;           // W2 as [tap*16 + ci][4] (cout padded to 4 with zeros)
constexpr int OFF_B2 = OFF_W2 + 144 * 4;
constexpr int PACKED = OFF_B2 + 4;            // WMD_DISP_TAIL16_PACKED_FLOATS
constexpr int SMEM_FLOATS = PACKED + PPIX * CP + UPIX * CP;
constexpr int THREADS = 256;
static_assert(PACKED == WMD_DISP_TAIL16_PACKED_FLOATS, "wmd.h's packed size");
static_assert(PACKED % 4 == 0 && (PACKED + PPIX * CP) % 4 == 0, "16-byte aligned regions");
static_assert(TH * TW == 2 * THREADS, "two output pixels per thread");
}  // namespace dt

__device__ __forceinline__ void dt_mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// x = hi + lo: hi = x truncated to tf32, lo the exact remainder
__device__ __forceinline__ void dt_split(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xFFFFE000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}

// w1 (16, 16, 3, 3), b1 (16) or NULL, w2 (cout, 16, 3, 3), b2 (cout) or NULL -> the image the kernel copies verbatim
__global__ void pack_disp_tail16_kernel(const float* __restrict__ w1, const float* __restrict__ b1,
                                        const float* __restrict__ w2, const float* __restrict__ b2, int cout,
                                        float* __restrict__ out) {
  using namespace dt;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < PACKED; i += gridDim.x * blockDim.x) {
    float v = 0.f;
    if (i < OFF_B1) {
      const bool lo = i >= W1F;
      const int j = lo ? i - W1F : i;
      const int n = j / KP, k = j - n * KP;
      if (k < 144) {
        const int tap = k >> 4, ci = k & 15;
        const float w = __ldg(w1 + (n * 16 + ci) * 9 + tap);
        const float hi = tf32_rna_finite(w);
        v = lo ? tf32_rna_finite(w - hi) : hi;
      }
    } else if (i < OFF_W2) {
      v = b1 ? __ldg(b1 + (i - OFF_B1)) : 0.f;
    } else if (i < OFF_B2) {
      const int j = i - OFF_W2, co = j & 3, k = j >> 2, tap = k >> 4, ci = k & 15;
      if (co < cout) v = __ldg(w2 + (co * 16 + ci) * 9 + tap);
    } else {
      const int co = i - OFF_B2;
      v = (b2 && co < cout) ? __ldg(b2 + co) : 0.f;
    }
    out[i] = v;
  }
}

template <int COUT>
__global__ void __launch_bounds__(dt::THREADS, 2)
disp_tail16_kernel(const float* __restrict__ x, int ld, const float* __restrict__ packed, float* __restrict__ disp, int N,
                   int H, int W) {
  using namespace dt;
  extern __shared__ __align__(16) float dt_smem[];
  float* const wsm = dt_smem;                     // packed weights
  float* const xp = dt_smem + PACKED;             // source patch [PPIX][CP]
  float* const us = xp + PPIX * CP;               // u halo [UPIX][CP]
  for (int i = threadIdx.x * 4; i < PACKED; i += THREADS * 4)
    *reinterpret_cast<float4*>(wsm + i) = __ldg(reinterpret_cast<const float4*>(packed + i));

  const int H2 = 2 * H, W2 = 2 * W;
  const int tiles_x = (W2 + TW - 1) / TW, tiles_y = (H2 + TH - 1) / TH;
  const int tiles = N * tiles_x * tiles_y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  const float* const w1h = wsm;
  const float* const w1l = wsm + W1F;

  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int n = tile / (tiles_x * tiles_y);
    const int rem = tile - n * tiles_x * tiles_y;
    const int y0 = (rem / tiles_x) * TH, x0 = (rem % tiles_x) * TW;
    const int py0 = y0 / 2 - 1, px0 = x0 / 2 - 1;  // first staged source pixel
    __syncthreads();                               // the previous tile's readers of xp / us are done (and wsm is loaded)

    // 1. source patch, zeros outside the image
    for (int i = threadIdx.x; i < PPIX * 4; i += THREADS) {
      const int p = i >> 2, q = i & 3;
      const int sy = py0 + p / PW, sx = px0 + p % PW;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (sy >= 0 && sy < H && sx >= 0 && sx < W)
        v = __ldg(reinterpret_cast<const float4*>(x + (static_cast<long long>(n) * H * W + static_cast<long long>(sy) * W + sx) * ld) + q);
      *reinterpret_cast<float4*>(xp + p * CP + 4 * q) = v;
    }
    __syncthreads();

    // 2. u over the halo: each warp takes m16 tiles warp, warp + 8, ...
    for (int mt = warp; mt < MT; mt += THREADS / 32) {
      int base[2];                                   // patch pixel of tap (0, 0) for rows g, g + 8 of the m tile
      int lr[2], lc[2];                              // parities of the u coordinates (which source pixel each tap reads)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        int m = mt * 16 + g + 8 * h;
        m = m < UPIX ? m : UPIX - 1;                 // padding rows of the last m tile: computed, never stored
        const int r = m / UW, c = m - r * UW;
        int Y = y0 - 1 + r, X = x0 - 1 + c;
        Y = reflect_idx(Y < H2 ? Y : H2, H2);        // the halo holds u at the reflected coordinate (rows past a partial
        X = reflect_idx(X < W2 ? X : W2, W2);        // tile's edge are clamped: computed, never read)
        // taps dy = 0..2 read up2(x) at Y - 1 + dy, i.e. source row (Y - 1 + dy) >> 1 (arithmetic shift: -1 -> -1)
        lr[h] = Y;
        lc[h] = X;
        base[h] = (((Y - 1) >> 1) - py0) * PW + (((X - 1) >> 1) - px0);
      }
      float acc[2][4];
#pragma unroll
      for (int j = 0; j < 2; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int dy = tap / 3, dx = tap % 3;
        int off[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // source pixel of u(Y, X)'s tap: ((Y - 1 + dy) >> 1, (X - 1 + dx) >> 1), relative to that of tap (0, 0)
          const int ry = ((lr[h] - 1 + dy) >> 1) - ((lr[h] - 1) >> 1);
          const int rx = ((lc[h] - 1 + dx) >> 1) - ((lc[h] - 1) >> 1);
          off[h] = (base[h] + ry * PW + rx) * CP;
        }
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int ch = 8 * half + t;
          uint32_t ah[4], al[4];
          dt_split(xp[off[0] + ch], ah[0], al[0]);
          dt_split(xp[off[1] + ch], ah[1], al[1]);
          dt_split(xp[off[0] + ch + 4], ah[2], al[2]);
          dt_split(xp[off[1] + ch + 4], ah[3], al[3]);
          const int k = tap * 16 + ch;
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int wo = (8 * j + g) * KP + k;
            const float bh0 = w1h[wo], bh1 = w1h[wo + 4], bl0 = w1l[wo], bl1 = w1l[wo + 4];
            // small terms first
            dt_mma_tf32(acc[j], al, __float_as_uint(bh0), __float_as_uint(bh1));
            dt_mma_tf32(acc[j], ah, __float_as_uint(bl0), __float_as_uint(bl1));
            dt_mma_tf32(acc[j], ah, __float_as_uint(bh0), __float_as_uint(bh1));
          }
        }
      }
      // bias + ELU; fragment (row g | g + 8, channels 8j + 2t, +1)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = mt * 16 + g + 8 * h;
        if (m >= UPIX) continue;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int co = 8 * j + 2 * t;
          const float v0 = acc[j][2 * h] + wsm[OFF_B1 + co], v1 = acc[j][2 * h + 1] + wsm[OFF_B1 + co + 1];
          *reinterpret_cast<float2*>(us + m * CP + co) =
              make_float2(v0 > 0.f ? v0 : expm1_nonpos(v0), v1 > 0.f ? v1 : expm1_nonpos(v1));
        }
      }
    }
    __syncthreads();

    // 3. dispconv + sigmoid: thread -> pixels (r, c) and (r + 8, c) of the tile; a warp stores 32 consecutive x
    const int c = threadIdx.x & 31, r = threadIdx.x >> 5;
    float a0[COUT], a1[COUT];
#pragma unroll
    for (int o = 0; o < COUT; ++o) a0[o] = a1[o] = 0.f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int dy = tap / 3, dx = tap % 3;
      const float* u0 = us + ((r + dy) * UW + c + dx) * CP;
      const float* u1 = u0 + 8 * UW * CP;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 v0 = *reinterpret_cast<const float4*>(u0 + 4 * q);
        const float4 v1 = *reinterpret_cast<const float4*>(u1 + 4 * q);
        const float e0[4] = {v0.x, v0.y, v0.z, v0.w}, e1[4] = {v1.x, v1.y, v1.z, v1.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float4 wv = *reinterpret_cast<const float4*>(wsm + OFF_W2 + (tap * 16 + 4 * q + e) * 4);
          const float wr[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
          for (int o = 0; o < COUT; ++o) {
            a0[o] = fmaf(e0[e], wr[o], a0[o]);
            a1[o] = fmaf(e1[e], wr[o], a1[o]);
          }
        }
      }
    }
    const long long plane = static_cast<long long>(H2) * W2;
    const int X = x0 + c;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int Y = y0 + r + 8 * h;
      if (Y < H2 && X < W2) {
        float* const dst = disp + static_cast<long long>(n) * COUT * plane + static_cast<long long>(Y) * W2 + X;
#pragma unroll
        for (int o = 0; o < COUT; ++o) dst[o * plane] = 1.0f / (1.0f + expf(-((h ? a1[o] : a0[o]) + wsm[OFF_B2 + o])));
      }
    }
  }
}

template <int COUT>
static int launch_disp_tail16(const float* x, int ld, const float* packed, float* disp, int N, int H, int W,
                              cudaStream_t stream) {
  using namespace dt;
  constexpr size_t smem = static_cast<size_t>(SMEM_FLOATS) * sizeof(float);
  static bool attr_done[64] = {};                 // per device: the attribute belongs to the device's context
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    const int rc = record(cudaFuncSetAttribute(disp_tail16_kernel<COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem)));
    if (rc != WMD_OK) return rc;
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  const long long tiles = static_cast<long long>(N) * ceil_div(2 * H, TH) * ceil_div(2 * W, TW);
  const long long cap = 2ll * sm_count();
  const int grid = static_cast<int>(tiles < cap ? tiles : cap);
  disp_tail16_kernel<COUT><<<grid, THREADS, smem, stream>>>(x, ld, packed, disp, N, H, W);
  return launched();
}

}  // namespace wmd

extern "C" int wmd_pack_disp_tail16_f32(const float* w1, const float* b1, const float* w2, const float* b2, int cout,
                                        float* packed, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(w1 && w2 && packed, WMD_ERR_ARG);
  WMD_REQUIRE(cout >= 1 && cout <= 4, WMD_ERR_SHAPE);
  WMD_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 15) == 0, WMD_ERR_SHAPE);
  pack_disp_tail16_kernel<<<ceil_div(dt::PACKED, 256), 256, 0, as_stream(stream)>>>(w1, b1, w2, b2, cout, packed);
  return launched();
}

extern "C" int wmd_disp_tail16_f32(const float* x, int ld, const float* packed, int cout, float* disp, int N, int H, int W,
                                   wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(x && packed && disp, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && H > 0 && W > 0 && ld >= 16 && ld % 4 == 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(cout >= 1 && cout <= 4, WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(N) * H * W * ld < (1ll << 40) &&
                  static_cast<long long>(N) * cout * 4 * H * W < (1ll << 40) && static_cast<long long>(N) * H * W < (1ll << 31),
              WMD_ERR_SHAPE);
  WMD_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(packed) & 15) == 0, WMD_ERR_SHAPE);
  if (N == 0) return WMD_OK;
  switch (cout) {
    case 1: return launch_disp_tail16<1>(x, ld, packed, disp, N, H, W, as_stream(stream));
    case 2: return launch_disp_tail16<2>(x, ld, packed, disp, N, H, W, as_stream(stream));
    case 3: return launch_disp_tail16<3>(x, ld, packed, disp, N, H, W, as_stream(stream));
    default: return launch_disp_tail16<4>(x, ld, packed, disp, N, H, W, as_stream(stream));
  }
}
