// Backward of the gather-GEMM convolution (training the dense decoders):
//
//   act_bwd    dz = dy * act'(y) from the saved post-activation output, the bias gradient sum_rows dz in fp64 in a fixed
//              order (rounded to fp32 once),
//              and max |dz| raised into a device scalar (the fp16-pair operand form of the data-gradient GEMM needs it);
//   wgrad      dW[tap][c][o] = sum_p A(p)[tap][c] dz(p)[o] on the tensor cores (mma.sync tf32, 3xTF32 split), A gathered
//              exactly as the forward gathers it; the pixel reduction (fp64 sums of 32-pixel chunks) is split across CTAs
//              and the partial slabs are summed in slab order by the last CTA of a tile to arrive - no float atomics, the
//              bits do not depend on timing;
//   dgrad_fold the data gradient is the forward contract itself (flipped, transposed weight, zero padding) run by the
//              forward engine over the grid extended by the one-pixel ring; this kernel adds every ring value into the pixel
//              the forward's pad mode read it from, sums the 2x2 children of a shift0 = 1 source into its low-resolution
//              rows, and writes the source-1 (skip) columns straight to NCHW.
#include "common.cuh"

namespace wmd {

// ---------------------------------------------------------------- activation backward + bias gradient
__device__ __forceinline__ float act_grad(float y, int act, float p) {   // act'(x) expressed through y = act(x)
  switch (act) {
    case WMD_ACT_ELU: return y > 0.f ? 1.f : y + 1.f;
    case WMD_ACT_LRELU: return y > 0.f ? 1.f : p;
    case WMD_ACT_SIGMOID: return y * (1.f - y);
    default: return 1.f;
  }
}

constexpr int AB_THREADS = 256;       // 8 row lanes x 32 channels
constexpr int AB_MAX_BLOCKS = 1024;
// Both kernels share one workspace layout: BWD_COUNTERS bytes of ticket / arrival counters (left zero by every launch),
// then data.  The act backward's ticket and the first weight-gradient counter are the same word; launches on one stream
// run one after the other and each leaves it zero.
constexpr size_t BWD_COUNTERS = 4096;
constexpr size_t AB_HEADER = BWD_COUNTERS;

static int ab_blocks(int rows) { return rows <= 0 ? 1 : (ceil_div(rows, 64) < AB_MAX_BLOCKS ? ceil_div(rows, 64) : AB_MAX_BLOCKS); }

__global__ void __launch_bounds__(AB_THREADS) act_bwd_kernel(const float* __restrict__ y, int ldy, const float* __restrict__ dy,
                                                             int lddy, int rows, int cout, int act, float p, float* dz,
                                                             int lddz, float* db, float* amax, double* partial,
                                                             unsigned* ticket, int rows_per_block) {
  // The bias gradient is summed in fp64 and rounded once: a column of 600 000 same-sign fp32 values summed in fp32 (a
  // per-thread chain, then up to 1024 block partials in order) drifts by ~1e-5 of the sum, 170 roundings' worth.
  __shared__ double red[8][33];
  __shared__ bool last;
  const int lane = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  float vmax = 0.f;
  for (int cb = 0; cb < cout; cb += 32) {
    const int c = cb + lane;
    double s = 0.0;
    if (c < cout) {
      for (int r = r0 + rl; r < r1; r += 8) {
        const float g = dy[static_cast<long long>(r) * lddy + c] * act_grad(y[static_cast<long long>(r) * ldy + c], act, p);
        dz[static_cast<long long>(r) * lddz + c] = g;
        s += g;
        vmax = fmaxf(vmax, finite_abs(g));
      }
    }
    red[rl][lane] = s;
    __syncthreads();
    if (rl == 0 && c < cout && db) {
      double t = red[0][lane];
#pragma unroll
      for (int k = 1; k < 8; ++k) t += red[k][lane];
      partial[static_cast<long long>(blockIdx.x) * cout + c] = t;
    }
    __syncthreads();
  }
  if (amax) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if (lane == 0 && vmax > __ldcg(amax)) atomicMax(reinterpret_cast<unsigned*>(amax), __float_as_uint(vmax));
  }
  if (!db) return;
  // the last block to finish sums the per-block partials in block order
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int c = threadIdx.x; c < cout; c += AB_THREADS) {
    double t = 0.0;
    for (int b = 0; b < static_cast<int>(gridDim.x); ++b) t += __ldcg(partial + static_cast<long long>(b) * cout + c);
    db[c] = __double2float_rn(t);
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// ---------------------------------------------------------------- weight gradient
constexpr int WG_BM = 64;             // (tap, channel) rows of a tile: 64 channels of one source at one tap
constexpr int WG_BK = 32;             // pixels per chunk
constexpr int WG_THREADS = 128;       // 4 warps, each 16 channels x BN outputs
constexpr int WG_STAGES = 3;
constexpr int WG_MIN_SPLIT_CHUNKS = 32;

template <int BN>
struct WgCfg {
  static constexpr int A_LD = WG_BM + 8;             // = 8 (mod 32): the fragment loads of a warp hit 32 distinct banks
  static constexpr int B_LD = BN <= 32 ? 40 : 72;
  static constexpr int A_STAGE = WG_BK * A_LD, B_STAGE = WG_BK * B_LD;
  static constexpr size_t SMEM = static_cast<size_t>(WG_STAGES) * (A_STAGE + B_STAGE) * sizeof(float);
  static constexpr int NT = BN / 8;
};

struct WgPlan {
  int bn, mt0, mt1, ntn, tiles, splits;
  long long nch;
};

static WgPlan wg_plan(const wmd_conv_desc& d) {
  WgPlan p;
  p.bn = d.cout >= 48 ? 64 : (d.cout > 8 ? 32 : 8);
  p.mt0 = ceil_div(d.c0, WG_BM);
  p.mt1 = d.x1 ? ceil_div(d.c1, WG_BM) : 0;
  p.ntn = ceil_div(d.cout, p.bn);
  p.tiles = d.taps * (p.mt0 + p.mt1) * p.ntn;
  const long long rows = static_cast<long long>(d.N) * d.H * d.W;
  p.nch = (rows + WG_BK - 1) / WG_BK;
  // few output tiles (a long pixel reduction into a small dW): split the pixel range until ~4 CTAs per SM are busy;
  // many tiles (a short reduction into a large dW): whole tiles
  const long long target = 4ll * sm_count();
  long long s = (target + p.tiles - 1) / p.tiles;
  const long long most = p.nch / WG_MIN_SPLIT_CHUNKS;
  if (s > most) s = most;
  if (s > 65535) s = 65535;
  if (static_cast<size_t>(p.tiles) * 4 > BWD_COUNTERS) s = 1;   // one counter per tile (split layers have < 4 x SMs tiles)
  p.splits = static_cast<int>(s < 1 ? 1 : s);
  return p;
}

__device__ __forceinline__ uint32_t to_tf32(float x) { return __float_as_uint(tf32_rna_finite(x)); }
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = to_tf32(x);
  lo = to_tf32(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// grid (tiles, splits); tile = ((mt * taps) + tap) * ntn + nt.  CTAs of one split are adjacent in launch order, so the
// taps and channel blocks that read the same pixel rows run together and share them through L2.
template <int BN>
__global__ void __launch_bounds__(WG_THREADS) conv_wgrad_kernel(const wmd_conv_desc d, const float* __restrict__ dz, int lddz,
                                                                float* __restrict__ dw, unsigned* counters, double* slabs,
                                                                int mt0, int ntn, long long nch) {
  using Cfg = WgCfg<BN>;
  constexpr int NT = Cfg::NT, A_LD = Cfg::A_LD, B_LD = Cfg::B_LD;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* As = reinterpret_cast<float*>(smem_raw);
  float* Bs = As + WG_STAGES * Cfg::A_STAGE;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int tile = blockIdx.x, split = blockIdx.y, splits = gridDim.y;
  const int nt = tile % ntn;
  const int tap = (tile / ntn) % d.taps;
  const int mt = tile / ntn / d.taps;
  const bool src1 = mt >= mt0;
  const int cbase = (src1 ? mt - mt0 : mt) * WG_BM;
  const int csrc = src1 ? d.c1 : d.c0;
  const float* xs = src1 ? d.x1 : d.x0;
  const int lds = src1 ? d.ld1 : d.ld0;
  const int nbase = nt * BN;
  const int HW = d.H * d.W;
  const int rows = d.N * HW;
  const int Hs = d.H >> d.shift0, Ws = d.W >> d.shift0;
  const int dy_tap = d.taps == 9 ? tap / 3 - 1 : 0, dx_tap = d.taps == 9 ? tap % 3 - 1 : 0;
  const long long ch_begin = nch * split / splits, ch_end = nch * (split + 1) / splits;

  // loader coordinates: A rows r = a_r0 + 8j (j < 4), 16-byte segment a_seg of the 64 channels
  const int a_seg = tid & 15, a_r0 = tid >> 4;
  const int ci = cbase + a_seg * 4;
  const int a_bytes = max(0, min(16, (csrc - ci) * 4));

  auto load_chunk = [&](long long ch, int stage) {
    const int m0 = static_cast<int>(ch * WG_BK);
    float* as = As + stage * Cfg::A_STAGE;
    // pixel of row a_r0, then step 8 pixels at a time
    int m = m0 + a_r0;
    int n = m / HW, rem = m - n * HW;
    int y = rem / d.W, x = rem - y * d.W;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int row = -1;
      if (m < rows) {
        int qy = y + dy_tap, qx = x + dx_tap;
        bool ok = pad_coord(qy, d.H, d.pad_mode);
        ok = pad_coord(qx, d.W, d.pad_mode) && ok;
        if (ok) {
          if (src1) {
            row = (n * d.H + qy) * d.W + qx;
          } else if (d.taps == 1 && d.map0 == nullptr) {
            row = m;
          } else {
            const int qs = (n * Hs + (qy >> d.shift0)) * Ws + (qx >> d.shift0);
            row = d.map0 ? d.map0[qs] : qs;
          }
        }
      }
      const bool live = row >= 0 && a_bytes > 0;
      const float* src = live ? xs + static_cast<long long>(row) * lds + ci : xs;
      cp_async16(as + (a_r0 + 8 * j) * A_LD + a_seg * 4, src, live ? a_bytes : 0);
      m += 8;
      x += 8;
      while (x >= d.W) { x -= d.W; if (++y == d.H) { y = 0; ++n; } }
    }
    float* bs = Bs + stage * Cfg::B_STAGE;
    for (int e = tid; e < WG_BK * (BN / 4); e += WG_THREADS) {
      const int r = e / (BN / 4), s = e - r * (BN / 4);
      const int o = nbase + s * 4;
      const int bytes = (m0 + r < rows) ? max(0, min(16, (d.cout - o) * 4)) : 0;
      const float* src = bytes > 0 ? dz + static_cast<long long>(m0 + r) * lddz + o : dz;
      cp_async16(bs + r * B_LD + s * 4, src, bytes);
    }
  };

  float acc[NT][4];
  double sum[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int k = 0; k < 4; ++k) { acc[j][k] = 0.f; sum[j][k] = 0.0; }

  const long long nloc = ch_end - ch_begin;
#pragma unroll
  for (int s = 0; s < WG_STAGES - 1; ++s) {
    if (s < nloc) load_chunk(ch_begin + s, s);
    cp_async_commit();
  }
  const int wm = warp * 16;
  for (long long c = 0; c < nloc; ++c) {
    cp_async_wait<WG_STAGES - 2>();
    __syncthreads();
    if (c + WG_STAGES - 1 < nloc) load_chunk(ch_begin + c + WG_STAGES - 1, static_cast<int>((c + WG_STAGES - 1) % WG_STAGES));
    cp_async_commit();
    const float* as = As + static_cast<int>(c % WG_STAGES) * Cfg::A_STAGE;
    const float* bs = Bs + static_cast<int>(c % WG_STAGES) * Cfg::B_STAGE;
#pragma unroll
    for (int kk = 0; kk < WG_BK; kk += 8) {
      // A[m][k] = As[k][m] (pixel-major in shared memory): m = channel, k = pixel
      uint32_t ah[4], al[4];
      split_tf32(as[(kk + t) * A_LD + wm + g], ah[0], al[0]);
      split_tf32(as[(kk + t) * A_LD + wm + g + 8], ah[1], al[1]);
      split_tf32(as[(kk + t + 4) * A_LD + wm + g], ah[2], al[2]);
      split_tf32(as[(kk + t + 4) * A_LD + wm + g + 8], ah[3], al[3]);
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        uint32_t bh0, bl0, bh1, bl1;
        split_tf32(bs[(kk + t) * B_LD + j * 8 + g], bh0, bl0);
        split_tf32(bs[(kk + t + 4) * B_LD + j * 8 + g], bh1, bl1);
        mma_tf32(acc[j], al, bh0, bh1);       // small terms first
        mma_tf32(acc[j], ah, bl0, bl1);
        mma_tf32(acc[j], ah, bh0, bh1);
      }
    }
    // one epoch per 32-pixel chunk: the tensor core's accumulation does not round to nearest, so each chunk's sum is
    // added into round-to-nearest sums.  On the real operands of every layer of the R18 640x192 decoder step this keeps
    // dW within 6.7e-7 of the largest fp64 element, against up to 1.0e-5 with 1024-pixel epochs.  The sums are fp64:
    // in fp32 a whole-tile reduction of 1200 chunks (NYU Decoder's up3 convA, 8 frames of 60 x 80) drifted to 2.55e-6
    // of S, over the weight gradient's bar.
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) { sum[j][k] += acc[j][k]; acc[j][k] = 0.f; }
  }
  cp_async_wait<0>();

  // element (channel cbase + wm + g + 8*(k>>1), output nbase + 8j + 2t + (k&1)) of the tile
  const int ctot = d.c0 + d.c1;
  auto store = [&](int j, int k, float v) {
    const int cl = cbase + wm + g + 8 * (k >> 1);
    const int o = nbase + j * 8 + 2 * t + (k & 1);
    if (cl < csrc && o < d.cout)
      dw[(static_cast<long long>(o) * ctot + (src1 ? d.c0 : 0) + cl) * d.taps + tap] = v;
  };
  if (splits == 1) {
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) store(j, k, __double2float_rn(sum[j][k]));
    return;
  }
  // partial slab of this split; the last split of the tile to arrive sums all of them in slab order
  constexpr int SLAB = WG_BM * BN;
  const int lidx0 = (wm + g) * BN + 2 * t;
  double* my = slabs + (static_cast<long long>(split) * gridDim.x + tile) * SLAB;
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int k = 0; k < 4; ++k) my[lidx0 + 8 * (k >> 1) * BN + j * 8 + (k & 1)] = sum[j][k];
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (tid == 0) last = atomicAdd(counters + tile, 1u) == static_cast<unsigned>(splits - 1);
  __syncthreads();
  if (!last) return;
  __threadfence();
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int li = lidx0 + 8 * (k >> 1) * BN + j * 8 + (k & 1);
      double v = 0.0;
      for (int s = 0; s < splits; ++s) v += __ldcg(slabs + (static_cast<long long>(s) * gridDim.x + tile) * SLAB + li);
      store(j, k, __double2float_rn(v));
    }
  if (tid == 0) counters[tile] = 0u;
}

template <int BN>
static int launch_wgrad(const wmd_conv_desc& d, const WgPlan& p, const float* dz, int lddz, float* dw, unsigned char* ws,
                        cudaStream_t stream) {
  static bool attr_done[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    int rc = record(cudaFuncSetAttribute(conv_wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(WgCfg<BN>::SMEM)));
    if (rc != WMD_OK) return rc;
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  unsigned* counters = reinterpret_cast<unsigned*>(ws);
  double* slabs = ws ? reinterpret_cast<double*>(ws + BWD_COUNTERS) : nullptr;
  conv_wgrad_kernel<BN><<<dim3(p.tiles, p.splits), WG_THREADS, WgCfg<BN>::SMEM, stream>>>(d, dz, lddz, dw, counters, slabs,
                                                                                         p.mt0, p.ntn, p.nch);
  return launched();
}

// ---------------------------------------------------------------- data-gradient fold
// value of the extended-grid gradient g at image pixel (y, x) plus every ring position the pad mode maps onto it
__device__ __forceinline__ float fold_px(const float* __restrict__ g, int ldg, int n, int y, int x, int H, int W, int pad,
                                         int c) {
  int ys[3], xs[3], ny = 1, nx = 1;
  ys[0] = y;
  xs[0] = x;
  if (pad != WMD_PAD_ZERO) {
    int q = -1;
    pad_coord(q, H, pad);
    if (q == y) ys[ny++] = -1;
    q = H;
    pad_coord(q, H, pad);
    if (q == y) ys[ny++] = H;
    q = -1;
    pad_coord(q, W, pad);
    if (q == x) xs[nx++] = -1;
    q = W;
    pad_coord(q, W, pad);
    if (q == x) xs[nx++] = W;
  }
  float s = 0.f;
  for (int i = 0; i < ny; ++i)
    for (int j = 0; j < nx; ++j)
      s += __ldg(g + ((static_cast<long long>(n) * (H + 2) + ys[i] + 1) * (W + 2) + xs[j] + 1) * ldg + c);
  return s;
}

// source 0: one thread per (row of x0, column); a shift0 = 1 source sums its 2x2 children in (a, b) order.  The pad
// columns c0..lddx0 are written as zeros: the rows are a gradient that autograd may add to another one whole.
__global__ void fold_src0_kernel(const float* __restrict__ g, int ldg, int N, int H, int W, int pad, int c0, int shift0,
                                 float* __restrict__ dx0, int lddx0) {
  const int Hs = H >> shift0, Ws = W >> shift0;
  const long long total = static_cast<long long>(N) * Hs * Ws * lddx0;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(e % lddx0);
    const long long r = e / lddx0;
    if (c >= c0) {
      dx0[r * lddx0 + c] = 0.f;
      continue;
    }
    const int X = static_cast<int>(r % Ws), Y = static_cast<int>((r / Ws) % Hs), n = static_cast<int>(r / (static_cast<long long>(Ws) * Hs));
    float s;
    if (shift0) {
      s = 0.f;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) s += fold_px(g, ldg, n, 2 * Y + a, 2 * X + b, H, W, pad, c);
    } else {
      s = fold_px(g, ldg, n, Y, X, H, W, pad, c);
    }
    dx0[r * lddx0 + c] = s;
  }
}

// source 1: 32 pixels x 32 channels per block through shared memory, read along channels, written along pixels (NCHW)
__global__ void fold_src1_kernel(const float* __restrict__ g, int ldg, int N, int H, int W, int pad, int c0, int c1,
                                 float* __restrict__ dx1) {
  __shared__ float tile[32][33];
  const int HW = H * W;
  const long long p0 = static_cast<long long>(blockIdx.x) * 32;
  const int cb = blockIdx.y * 32;
  const long long total = static_cast<long long>(N) * HW;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const long long p = p0 + i;
    const int c = cb + threadIdx.x;
    float v = 0.f;
    if (p < total && c < c1) {
      const int n = static_cast<int>(p / HW), rem = static_cast<int>(p - static_cast<long long>(n) * HW);
      v = fold_px(g, ldg, n, rem / W, rem % W, H, W, pad, c0 + c);
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const long long p = p0 + threadIdx.x;
    const int c = cb + i;
    if (p < total && c < c1) {
      const int n = static_cast<int>(p / HW), rem = static_cast<int>(p - static_cast<long long>(n) * HW);
      dx1[(static_cast<long long>(n) * c1 + c) * HW + rem] = tile[threadIdx.x][i];
    }
  }
}

}  // namespace wmd

extern "C" size_t wmd_act_bwd_ws_bytes(int rows, int cout) {
  return wmd::AB_HEADER + static_cast<size_t>(wmd::ab_blocks(rows)) * (cout > 0 ? cout : 0) * sizeof(double);
}

extern "C" int wmd_act_bwd_f32(const float* y, int ldy, const float* dy, int lddy, int rows, int cout, int act,
                               float act_param, float* dz, int lddz, float* db, float* amax_dz, void* ws, size_t ws_bytes,
                               wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(y && dy && dz, WMD_ERR_ARG);
  WMD_REQUIRE(act >= WMD_ACT_NONE && act <= WMD_ACT_SIGMOID, WMD_ERR_ARG);
  WMD_REQUIRE(rows >= 0 && cout > 0 && ldy >= cout && lddy >= cout && lddz >= cout, WMD_ERR_SHAPE);
  if (db) {
    WMD_REQUIRE(ws, WMD_ERR_ARG);
    WMD_REQUIRE(ws_bytes >= wmd_act_bwd_ws_bytes(rows, cout), WMD_ERR_WORKSPACE);
  }
  if (rows == 0) {
    if (db) return record(cudaMemsetAsync(db, 0, sizeof(float) * cout, as_stream(stream)));
    return WMD_OK;
  }
  const int blocks = ab_blocks(rows);
  const int per = (ceil_div(rows, blocks) + 7) / 8 * 8;
  unsigned char* w = static_cast<unsigned char*>(ws);
  act_bwd_kernel<<<ceil_div(rows, per), AB_THREADS, 0, as_stream(stream)>>>(
      y, ldy, dy, lddy, rows, cout, act, act_param, dz, lddz, db, amax_dz,
      w ? reinterpret_cast<double*>(w + AB_HEADER) : nullptr, reinterpret_cast<unsigned*>(w), per);
  return launched();
}

static int wgrad_check(const wmd_conv_desc* d) {
  WMD_REQUIRE(d && d->x0, WMD_ERR_ARG);
  WMD_REQUIRE(d->taps == 1 || d->taps == 9, WMD_ERR_ARG);
  WMD_REQUIRE(d->pad_mode >= WMD_PAD_ZERO && d->pad_mode <= WMD_PAD_REPLICATE, WMD_ERR_ARG);
  WMD_REQUIRE(d->shift0 == 0 || d->shift0 == 1, WMD_ERR_ARG);
  // a 1x1 layer without map0 reads row m of x0 itself (the forward's aligned-rows form): no upsampled source
  WMD_REQUIRE(d->taps == 9 || d->shift0 == 0, WMD_ERR_UNSUPPORTED);
  // dense layers only: the sparse decoders are inference-only
  WMD_REQUIRE(d->pixels == nullptr && d->gate == nullptr && d->map1 == nullptr, WMD_ERR_UNSUPPORTED);
  WMD_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0 && d->c0 > 0 && d->cout > 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(d->N) * d->H * d->W < (1ll << 31), WMD_ERR_SHAPE);
  WMD_REQUIRE(d->ld0 >= d->c0 && d->ld0 % 4 == 0 && (reinterpret_cast<uintptr_t>(d->x0) & 15) == 0, WMD_ERR_SHAPE);
  if (d->x1) WMD_REQUIRE(d->c1 > 0 && d->ld1 >= d->c1 && d->ld1 % 4 == 0 && (reinterpret_cast<uintptr_t>(d->x1) & 15) == 0,
                         WMD_ERR_SHAPE);
  if (d->shift0 == 1) WMD_REQUIRE(d->H % 2 == 0 && d->W % 2 == 0, WMD_ERR_SHAPE);
  if (d->pad_mode == WMD_PAD_REFLECT && d->taps == 9) WMD_REQUIRE(d->H >= 2 && d->W >= 2, WMD_ERR_SHAPE);
  return WMD_OK;
}

extern "C" size_t wmd_conv_wgrad_ws_bytes(const wmd_conv_desc* dp) {
  using namespace wmd;
  if (wgrad_check(dp) != WMD_OK) return 0;
  wmd_conv_desc d = *dp;
  if (!d.x1) d.c1 = 0;
  const WgPlan p = wg_plan(d);
  if (p.splits == 1) return 0;
  return BWD_COUNTERS + static_cast<size_t>(p.splits) * p.tiles * WG_BM * p.bn * sizeof(double);
}

extern "C" int wmd_conv_wgrad_f32(const wmd_conv_desc* dp, const float* dz, int lddz, float* dw, void* ws, size_t ws_bytes,
                                  wmd_stream_t stream) {
  using namespace wmd;
  int rc = wgrad_check(dp);
  if (rc != WMD_OK) return rc;
  WMD_REQUIRE(dz && dw, WMD_ERR_ARG);
  wmd_conv_desc d = *dp;
  if (!d.x1) { d.c1 = 0; d.ld1 = 0; }
  WMD_REQUIRE(lddz >= d.cout && lddz % 4 == 0 && (reinterpret_cast<uintptr_t>(dz) & 15) == 0, WMD_ERR_SHAPE);
  const WgPlan p = wg_plan(d);
  const size_t need = wmd_conv_wgrad_ws_bytes(&d);
  if (need) {
    WMD_REQUIRE(ws, WMD_ERR_ARG);
    WMD_REQUIRE(ws_bytes >= need, WMD_ERR_WORKSPACE);
  }
  unsigned char* w = need ? static_cast<unsigned char*>(ws) : nullptr;
  if (p.bn == 64) return launch_wgrad<64>(d, p, dz, lddz, dw, w, as_stream(stream));
  if (p.bn == 32) return launch_wgrad<32>(d, p, dz, lddz, dw, w, as_stream(stream));
  return launch_wgrad<8>(d, p, dz, lddz, dw, w, as_stream(stream));
}

extern "C" int wmd_conv_dgrad_fold_f32(const float* g, int ldg, int N, int H, int W, int pad_mode, int c0, int shift0,
                                       float* dx0, int lddx0, int c1, float* dx1_nchw, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(g && dx0, WMD_ERR_ARG);
  WMD_REQUIRE(pad_mode >= WMD_PAD_ZERO && pad_mode <= WMD_PAD_REPLICATE, WMD_ERR_ARG);
  WMD_REQUIRE(shift0 == 0 || shift0 == 1, WMD_ERR_ARG);
  WMD_REQUIRE(c1 == 0 || dx1_nchw, WMD_ERR_ARG);
  WMD_REQUIRE(N > 0 && H > 0 && W > 0 && c0 > 0 && c1 >= 0 && ldg >= c0 + c1 && lddx0 >= c0, WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(N) * (H + 2) * (W + 2) < (1ll << 31), WMD_ERR_SHAPE);
  if (shift0) WMD_REQUIRE(H % 2 == 0 && W % 2 == 0, WMD_ERR_SHAPE);
  if (pad_mode == WMD_PAD_REFLECT) WMD_REQUIRE(H >= 2 && W >= 2, WMD_ERR_SHAPE);
  const cudaStream_t s = as_stream(stream);
  const long long n0 = static_cast<long long>(N) * (H >> shift0) * (W >> shift0) * lddx0;
  fold_src0_kernel<<<stride_grid(n0, 256), 256, 0, s>>>(g, ldg, N, H, W, pad_mode, c0, shift0, dx0, lddx0);
  int rc = launched();
  if (rc != WMD_OK || c1 == 0) return rc;
  const dim3 grid(ceil_div(static_cast<long long>(N) * H * W, 32), ceil_div(c1, 32));
  fold_src1_kernel<<<grid, dim3(32, 8), 0, s>>>(g, ldg, N, H, W, pad_mode, c0, c1, dx1_nchw);
  return launched();
}
