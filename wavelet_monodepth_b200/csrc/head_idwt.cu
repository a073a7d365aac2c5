// K1f: the tail of a decoder level as ONE kernel - factored 3x3 head stage (gather-sum of per-tap products) ->
// sigma-difference coefficients -> Haar IDWT -> disparity plane (+ consumer epilogue, + the next level's range threshold).
//
// Replaces, per level: torch.zeros(yh) + head_gather (scatter of yh) + idwt_haar (re-read of yh) + range_thresh (re-read of
// the reconstruction): `yh` is written once and never read back, the reconstruction is reduced to its per-sample
// min / max while it is produced.  Algorithmic bytes per coefficient pixel: 4 (ll) + 1 (mask) in, 12 (yh) + 16 (out) +
// 16 (disp) out, + 9 x 24 B of tap products per ACTIVE pixel (L2-resident rows written by the kernel before).
//
// Tile = 8 coefficient rows x 128 columns per CTA (128 threads: warp w owns rows 2w, 2w+1; lane owns 4 columns).  The
// ll rows and the mask rows of the tile are staged into shared memory by the TMA (one cp.async.bulk per row segment,
// completion by mbarrier transaction bytes) while the threads fetch the index-map rows; every global store is a full
// 128-bit, 512-byte-per-warp row segment.  Arithmetic: the coefficient is  scale * (sigmoid(s+) - sigmoid(s-))  with
// s = bias + sum of the nine tap products in tap order (the order wmd_head_gather_f32 uses: results are bit-identical
// to the unfused chain), the synthesis is haar_synth of haar.cu (the dependency's separable evaluation order).
#include "common.cuh"

namespace wmd {

#define WMD_S 0.70710678118654752440f

constexpr int kFT_H = 8, kFT_W = 128, kFThreads = 128;    // small CTAs: many in flight per SM hide the gather / staging latency

__device__ __forceinline__ float fnan_min(float a, float b) { return (a != a || b != b) ? NAN : fminf(a, b); }
__device__ __forceinline__ float fnan_max(float a, float b) { return (a != a || b != b) ? NAN : fmaxf(a, b); }

__device__ __forceinline__ void synth4(float ll, float lh, float hl, float hh, float& y00, float& y01, float& y10, float& y11) {
  const float sll = __fmul_rn(WMD_S, ll), slh = __fmul_rn(WMD_S, lh);
  const float shl = __fmul_rn(WMD_S, hl), shh = __fmul_rn(WMD_S, hh);
  const float lo0 = __fadd_rn(sll, slh), lo1 = __fsub_rn(sll, slh);
  const float hi0 = __fadd_rn(shl, shh), hi1 = __fsub_rn(shl, shh);
  const float a0 = __fmul_rn(WMD_S, lo0), b0 = __fmul_rn(WMD_S, hi0);
  const float a1 = __fmul_rn(WMD_S, lo1), b1 = __fmul_rn(WMD_S, hi1);
  y00 = __fadd_rn(a0, b0); y01 = __fsub_rn(a0, b0);
  y10 = __fadd_rn(a1, b1); y11 = __fsub_rn(a1, b1);
}

__device__ __forceinline__ float disp_val(float v, float scale, int clamp01) {
  v = __fmul_rn(v, scale);
  return (clamp01 && v == v) ? fminf(fmaxf(v, 0.f), 1.f) : v;     // torch.clamp passes a NaN through; fmaxf would make it 0
}

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// consumer epilogue of the reconstruction / disparity (wmd_head_idwt_desc.epi_mode)
__device__ __forceinline__ void epilogue(const wmd_head_idwt_desc& d, long long o, float recon, float disp) {
  if (d.epi_mode == WMD_EPI_DISP_TO_DEPTH) {          // KITTI/layers.py:16-25 on the disparity plane
    const float sd = __fadd_rn(d.epi_a, __fmul_rn(d.epi_b, disp));
    d.epi_out0[o] = sd;
    if (d.epi_out1) d.epi_out1[o] = __fdiv_rn(1.f, sd);
  } else if (d.epi_mode == WMD_EPI_DIV_CLAMP) {       // NYUv2/utils.py:219,229 on the reconstruction
    // torch on CUDA evaluates `t / python_scalar` as t * (1 / scalar): what the reference's `pred_y /= 100` computes
    float v = __fmul_rn(recon, __fdiv_rn(1.f, d.epi_a));
    if (d.epi_b != 0.f && v == v) v = fminf(fmaxf(v, d.epi_lo), d.epi_hi);   // NaN stays NaN, as in torch.clamp
    d.epi_out0[o] = v;
  }
}

__global__ void __launch_bounds__(kFThreads) head_idwt_kernel(const wmd_head_idwt_desc d, unsigned* __restrict__ counters,
                                                              float* __restrict__ partial, int use_bulk) {
  __shared__ __align__(16) float s_ll[kFT_H][kFT_W];
  __shared__ __align__(16) uint8_t s_mask[kFT_H][kFT_W];
  __shared__ __align__(16) float s_yh[3][kFT_H][kFT_W];        // the tile's coefficients (phase A -> phase B)
  __shared__ uint16_t s_list[kFT_H * kFT_W];                   // the tile's active pixels
  __shared__ int s_count;
  __shared__ __align__(8) uint64_t bar;
  __shared__ float s_mn[8], s_mx[8];
  __shared__ bool is_last;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = blockIdx.y;
  const int tiles_x = (d.W + kFT_W - 1) / kFT_W;
  const int ty = blockIdx.x / tiles_x, tx = blockIdx.x - ty * tiles_x;
  const int y0 = ty * kFT_H, x0 = tx * kFT_W;
  const int th = min(kFT_H, d.H - y0), tw = min(kFT_W, d.W - x0);
  const long long HW = static_cast<long long>(d.H) * d.W;
  const float* ll_n = d.ll + static_cast<long long>(n) * HW;
  const uint8_t* mask_n = d.mask ? d.mask + static_cast<long long>(n) * HW : nullptr;

  // ---- stage ll (and the mask) rows of the tile: TMA bulk copies when every row segment is 16-byte aligned
  if (use_bulk) {
    if (tid == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_addr(&bar)), "r"(1u));
      asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    if (warp == 0) {
      const uint32_t row_bytes = static_cast<uint32_t>(tw) * 4u, mrow_bytes = mask_n ? static_cast<uint32_t>(tw) : 0u;
      if (lane == 0)
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_addr(&bar)),
                     "r"(static_cast<uint32_t>(th) * (row_bytes + mrow_bytes)) : "memory");
      __syncwarp();
      if (lane < th) {
        const long long o = static_cast<long long>(y0 + lane) * d.W + x0;
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                         smem_addr(&s_ll[lane][0])), "l"(ll_n + o), "r"(row_bytes), "r"(smem_addr(&bar)) : "memory");
        if (mask_n)
          asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                           smem_addr(&s_mask[lane][0])), "l"(mask_n + o), "r"(mrow_bytes), "r"(smem_addr(&bar)) : "memory");
      }
    }
  } else {
    for (int e = tid; e < th * tw; e += kFThreads) {
      const int r = e / tw, c = e - r * tw;
      const long long o = static_cast<long long>(y0 + r) * d.W + x0 + c;
      s_ll[r][c] = __ldg(ll_n + o);
      if (mask_n) s_mask[r][c] = __ldg(mask_n + o);
    }
  }

  float b6[6];
#pragma unroll
  for (int g = 0; g < 6; ++g) b6[g] = d.bias ? __ldg(d.bias + g) : 0.f;
  for (int e = tid; e < 3 * kFT_H * kFT_W; e += kFThreads) (&s_yh[0][0][0])[e] = 0.f;    // coefficients default to zero
  if (tid == 0) s_count = 0;

  if (use_bulk) {
    __syncthreads();                                                     // s_count / s_yh initialised
    uint32_t done = 0;
    for (uint32_t spin = 0; spin < (1u << 24) && !done; ++spin)          // bounded: a protocol bug traps instead of hanging
      asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                   : "=r"(done) : "r"(smem_addr(&bar)), "r"(0u) : "memory");
    if (!done) __trap();
  } else {
    __syncthreads();
  }

  // ---- phase A: the tile's ACTIVE pixels, dealt evenly to the threads (the gather-sum is the only irregular work: a
  // thread that owned a fixed patch would serialise up to eight 9-tap gathers while its neighbours idle)
  for (int e = tid; e < th * tw; e += kFThreads) {
    const int r = e / tw, c = e - r * tw;
    if (mask_n == nullptr || s_mask[r][c]) s_list[atomicAdd(&s_count, 1)] = static_cast<uint16_t>(r * kFT_W + c);
  }
  __syncthreads();
  const int nact = s_count;
  for (int i = tid; i < nact; i += kFThreads) {
    const int e = s_list[i];
    const int r = e / kFT_W, c = e - r * kFT_W;
    const int y = y0 + r, x = x0 + c;
    float s[6];
#pragma unroll
    for (int g = 0; g < 6; ++g) s[g] = b6[g];
    int rows9[9];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {                                  // the nine index-map lookups first: independent loads
      int qy = y + tap / 3 - 1, qx = x + tap % 3 - 1;
      bool ok = pad_coord(qy, d.H, d.pad_mode);
      ok = pad_coord(qx, d.W, d.pad_mode) && ok;
      const int q = (n * d.H + qy) * d.W + qx;
      rows9[tap] = ok ? (d.map ? __ldg(d.map + q) : q) : -1;
    }
    // all 27 loads first (a missing tap reads row 0 and is zeroed: + 0.0f leaves the sum's bits), then the sums in tap
    // order - the order of the unfused chain
    float2 v[9][3];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const float* zr = d.z + static_cast<long long>(max(rows9[tap], 0)) * d.ldz + tap * 6;
#pragma unroll
      for (int g = 0; g < 3; ++g) v[tap][g] = __ldg(reinterpret_cast<const float2*>(zr + 2 * g));
    }
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      if (rows9[tap] < 0) continue;
#pragma unroll
      for (int g = 0; g < 3; ++g) {
        s[2 * g] += v[tap][g].x;
        s[2 * g + 1] += v[tap][g].y;
      }
    }
    s_yh[0][r][c] = d.scale * (activate(s[0], WMD_ACT_SIGMOID, 0.f) - activate(s[3], WMD_ACT_SIGMOID, 0.f));
    s_yh[1][r][c] = d.scale * (activate(s[1], WMD_ACT_SIGMOID, 0.f) - activate(s[4], WMD_ACT_SIGMOID, 0.f));
    s_yh[2][r][c] = d.scale * (activate(s[2], WMD_ACT_SIGMOID, 0.f) - activate(s[5], WMD_ACT_SIGMOID, 0.f));
  }
  __syncthreads();

  // ---- phase B: the streaming part - yh rows out, synthesis, reconstruction / disparity rows out
  float mn = INFINITY, mx = -INFINITY;
  const int W2 = 2 * d.W;
  float* yh_n = d.yh + static_cast<long long>(n) * 3 * HW;
  const long long out_n = static_cast<long long>(n) * 4 * HW;
  const int cx = 4 * lane;                                  // first of this lane's four columns inside the tile
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = 2 * warp + rr;
    const int y = y0 + r;
    if (r >= th || cx >= tw) continue;
    const float4 l4 = *reinterpret_cast<const float4*>(&s_ll[r][cx]);
    const float4 a4 = *reinterpret_cast<const float4*>(&s_yh[0][r][cx]);
    const float4 h4 = *reinterpret_cast<const float4*>(&s_yh[1][r][cx]);
    const float4 d4 = *reinterpret_cast<const float4*>(&s_yh[2][r][cx]);
    const float llv[4] = {l4.x, l4.y, l4.z, l4.w}, lh[4] = {a4.x, a4.y, a4.z, a4.w};
    const float hl[4] = {h4.x, h4.y, h4.z, h4.w}, hh[4] = {d4.x, d4.y, d4.z, d4.w};
    const long long co = static_cast<long long>(y) * d.W + x0 + cx;      // W % 4 == 0: a lane's four columns are all inside
    *reinterpret_cast<float4*>(yh_n + co) = a4;
    *reinterpret_cast<float4*>(yh_n + HW + co) = h4;
    *reinterpret_cast<float4*>(yh_n + 2 * HW + co) = d4;
    float top[8], bot[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) synth4(llv[k], lh[k], hl[k], hh[k], top[2 * k], top[2 * k + 1], bot[2 * k], bot[2 * k + 1]);
    const long long oo = out_n + static_cast<long long>(2 * y) * W2 + 2 * (x0 + cx);
#pragma unroll
    for (int k = 0; k < 8; ++k) { mn = fnan_min(mn, fnan_min(top[k], bot[k])); mx = fnan_max(mx, fnan_max(top[k], bot[k])); }
    *reinterpret_cast<float4*>(d.out + oo) = make_float4(top[0], top[1], top[2], top[3]);
    *reinterpret_cast<float4*>(d.out + oo + 4) = make_float4(top[4], top[5], top[6], top[7]);
    *reinterpret_cast<float4*>(d.out + oo + W2) = make_float4(bot[0], bot[1], bot[2], bot[3]);
    *reinterpret_cast<float4*>(d.out + oo + W2 + 4) = make_float4(bot[4], bot[5], bot[6], bot[7]);
    if (d.disp || d.epi_mode) {
      float dt[8], db[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) { dt[k] = disp_val(top[k], d.disp_scale, d.clamp01); db[k] = disp_val(bot[k], d.disp_scale, d.clamp01); }
      if (d.disp) {
        *reinterpret_cast<float4*>(d.disp + oo) = make_float4(dt[0], dt[1], dt[2], dt[3]);
        *reinterpret_cast<float4*>(d.disp + oo + 4) = make_float4(dt[4], dt[5], dt[6], dt[7]);
        *reinterpret_cast<float4*>(d.disp + oo + W2) = make_float4(db[0], db[1], db[2], db[3]);
        *reinterpret_cast<float4*>(d.disp + oo + W2 + 4) = make_float4(db[4], db[5], db[6], db[7]);
      }
      if (d.epi_mode) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { epilogue(d, oo + k, top[k], dt[k]); epilogue(d, oo + W2 + k, bot[k], db[k]); }
      }
    }
  }

  // ---- per-sample range of the reconstruction -> the next level's threshold (depth_decoder.py:308), last block folds
  if (d.thresh == nullptr) return;
  for (int o = 16; o > 0; o >>= 1) {
    mn = fnan_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fnan_max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (lane == 0) { s_mn[warp] = mn; s_mx[warp] = mx; }
  __syncthreads();
  const int B = gridDim.x;
  if (tid == 0) {
    for (int w = 1; w < kFThreads / 32; ++w) { mn = fnan_min(mn, s_mn[w]); mx = fnan_max(mx, s_mx[w]); }
    volatile float* pp = partial + (static_cast<long long>(n) * B + blockIdx.x) * 2;
    pp[0] = mn; pp[1] = mx;
    __threadfence();
    const unsigned ticket = atomicAdd(&counters[n], 1u);
    is_last = (ticket == static_cast<unsigned>(B - 1));
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  mn = INFINITY; mx = -INFINITY;
  const volatile float* pr = partial + static_cast<long long>(n) * B * 2;
  for (int i = tid; i < B; i += kFThreads) { mn = fnan_min(mn, pr[2 * i]); mx = fnan_max(mx, pr[2 * i + 1]); }
  for (int o = 16; o > 0; o >>= 1) {
    mn = fnan_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fnan_max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  __syncthreads();
  if (lane == 0) { s_mn[warp] = mn; s_mx[warp] = mx; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kFThreads / 32; ++w) { mn = fnan_min(mn, s_mn[w]); mx = fnan_max(mx, s_mx[w]); }
    d.thresh[n] = __fmul_rn(__fsub_rn(mx, mn), d.thresh_ratio);
    counters[n] = 0u;                                   // workspace stays zeroed for the next call
  }
}

constexpr size_t kFCounterBytes = 16384 * sizeof(unsigned);

}  // namespace wmd

extern "C" size_t wmd_head_idwt_ws_bytes(int N, int H, int W) {
  using namespace wmd;
  const long long tiles = static_cast<long long>((H + kFT_H - 1) / kFT_H) * ((W + kFT_W - 1) / kFT_W);
  return kFCounterBytes + static_cast<size_t>(N < 1 ? 1 : N) * static_cast<size_t>(tiles) * 2 * sizeof(float);
}

extern "C" int wmd_head_idwt_f32(const wmd_head_idwt_desc* dp, void* ws, size_t ws_bytes, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(dp, WMD_ERR_ARG);
  const wmd_head_idwt_desc d = *dp;
  WMD_REQUIRE(d.z && d.ll && d.yh && d.out, WMD_ERR_ARG);
  WMD_REQUIRE(d.N >= 0 && d.H > 0 && d.W > 0 && d.ldz >= 54 && d.ldz % 2 == 0, WMD_ERR_SHAPE);
  WMD_REQUIRE((reinterpret_cast<uintptr_t>(d.z) & 7) == 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(d.N <= 16384 && static_cast<long long>(d.N) * d.H * d.W < (1ll << 31), WMD_ERR_SHAPE);
  WMD_REQUIRE(d.pad_mode >= WMD_PAD_ZERO && d.pad_mode <= WMD_PAD_REPLICATE, WMD_ERR_ARG);
  if (d.pad_mode == WMD_PAD_REFLECT) WMD_REQUIRE(d.H >= 2 && d.W >= 2, WMD_ERR_SHAPE);
  WMD_REQUIRE(d.epi_mode == WMD_EPI_NONE || d.epi_out0 != nullptr, WMD_ERR_ARG);
  WMD_REQUIRE(d.epi_mode >= WMD_EPI_NONE && d.epi_mode <= WMD_EPI_DIV_CLAMP, WMD_ERR_ARG);
  WMD_REQUIRE(d.thresh == nullptr || (ws != nullptr && ws_bytes >= wmd_head_idwt_ws_bytes(d.N, d.H, d.W)), WMD_ERR_WORKSPACE);
  // 128-bit stores: W % 4 == 0 and 16-byte aligned planes; the TMA staging additionally needs 16-byte aligned mask rows
  WMD_REQUIRE(d.W % 4 == 0 && (reinterpret_cast<uintptr_t>(d.yh) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.out) & 15) == 0 &&
                  (d.disp == nullptr || (reinterpret_cast<uintptr_t>(d.disp) & 15) == 0), WMD_ERR_SHAPE);
  if (d.N == 0) return WMD_OK;
  const int use_bulk = (d.W % 16 == 0) && (reinterpret_cast<uintptr_t>(d.ll) & 15) == 0 &&
                       (d.mask == nullptr || (reinterpret_cast<uintptr_t>(d.mask) & 15) == 0);
  const int tiles = ((d.H + kFT_H - 1) / kFT_H) * ((d.W + kFT_W - 1) / kFT_W);
  unsigned* counters = static_cast<unsigned*>(ws);
  float* partial = ws ? reinterpret_cast<float*>(static_cast<char*>(ws) + kFCounterBytes) : nullptr;
  dim3 grid(tiles, d.N);
  head_idwt_kernel<<<grid, kFThreads, 0, as_stream(stream)>>>(d, counters, partial, use_bulk);
  return launched();
}
