// K5-TC: the gather-GEMM convolution on Hopper tensor cores (wgmma), fp32-faithful via 3xTF32.
//
// Same contract as conv_rows_kernel (conv.cu), different engine.  A persistent grid (at most one CTA per SM) walks
// 128 x N output tiles (N = 128 / 64 / 32); a tile's reduction K = (c0 + c1) x taps runs in 32-channel chunks, the
// taps of a channel chunk innermost (their source rows overlap: L2 hits).  256 threads = two warpgroups, warpgroup h
// owns tile rows h*64 .. h*64+63 (one wgmma M = 64 each, both share the chunk's weight tile).
//
//   gather (all 256 threads), TC_STAGES - 1 chunks ahead of the MMAs, cp.async with zero fill
//     * implicit im2col: the 128-byte channel slice of each tile row's source row (row from the per-tile tap table,
//       -1 = inactive / padded tap, and the channel tail read zeros) into a raw fp32 stage padded to 144-byte rows, so
//       that the fragment reads below are free of bank conflicts;
//     * B (weights) is pre-split, pre-swizzled by wmd_pack_conv_weight_tc_f32 into one [hi | lo] image per (n-tile,
//       chunk): K-major, 128-byte swizzled, read by the wgmma straight from shared memory through a descriptor;
//   multiply (per warpgroup)
//     * every thread reads its A fragment elements (rows g, g + 8 of its warp's 16, channels t, t + 4 of each k-step)
//       and splits x = hi + lo (hi = x with the 13 low mantissa bits cleared, lo = x - hi: exact) in registers - the
//       register-A form of wgmma, so the split never goes back to shared memory;
//     * 4 k-steps x 3 terms (lo*hi + hi*lo + hi*hi) per chunk, committed and waited as one group;
//     * the tensor core's fp32 accumulation is not round-to-nearest, a bias that grows with K.  So accumulation runs in
//       EPOCHS of kFlushChunks chunks: the first MMA of an epoch overwrites the wgmma accumulators, the epoch's end adds
//       them into per-thread fp32 registers with round-to-nearest adds;
//   epilogue: bias + activation (picked once per tile) + pair stores;
//   balanced scheduling (long reductions): whole tiles for the full rounds, the (tile, chunk) units of the remainder
//     dealt out evenly on the device (stream-K); the last segment of a cut tile to arrive sums all segments in slab
//     order, cooperatively and coalesced.
// Optional fp16-pair operand form (F16 = true, wmd_conv_desc.precision): x 2^e = h1 + h2 as fp16, f16 MMAs with K = 16
// (half the instructions), scale from the sources' max |x| (device scalars), weights' scale in the packed image's header.
#include <cuda_fp16.h>

#include "common.cuh"

namespace wmd {

constexpr int TC_BM = 128;                      // rows per CTA tile = 2 warpgroups x wgmma M = 64
constexpr int TC_BK = 32;                       // floats per chunk = one 128-byte row of a weight image
constexpr int TC_THREADS = 256;                 // two warpgroups: both gather, each multiplies its 64 rows
constexpr int TC_STAGES = 4;                    // cp.async ring: three chunks in flight while one is multiplied
constexpr int TC_A_LD = TC_BK + 4;              // raw A row pitch in floats (144 B: fragment reads hit 32 distinct banks)
constexpr int TC_A_TILE = TC_BM * TC_A_LD * 4;  // 18 KB raw fp32
constexpr int TC_TABLES = 2 * 9 * TC_BM * 4;

// Per N-tile configuration.  A stage holds the chunk's weight image first (its size is a multiple of 4 KB, so every image
// keeps the 1024-byte alignment of the 128-byte swizzle) and the raw A rows after it.
template <int BN, bool F16 = false>
struct TcCfg {
  static constexpr int B_TILE = BN * TC_BK * 4;            // bytes of one of hi / lo (tf32 form)
  // weight image of one chunk: tf32 form [hi: BN x 128 B | lo: BN x 128 B]; f16 form ONE BN x 128 B tile whose rows hold
  // [h1: 32 channels | h2: 32 channels] as fp16
  static constexpr int B_IMG = F16 ? B_TILE : 2 * B_TILE;
  static constexpr int ACC = BN / 2;                       // accumulator registers per thread (wgmma m64 x BN fragment)
  static constexpr int STAGE = B_IMG + TC_A_TILE;
  static constexpr size_t SMEM = static_cast<size_t>(TC_STAGES) * STAGE + TC_TABLES + 1024;
  static_assert(STAGE % 1024 == 0, "weight images must stay 1024-byte aligned");
  static_assert(SMEM <= 227 * 1024, "one CTA must fit the shared memory of an SM");
};
constexpr int kFlushChunks = 32;                // epoch length: K = 1024 per wgmma accumulation run
constexpr int32_t kNoRow = -1;                  // tap-table entry of an inactive / padded source: the gather writes zeros


__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// cp.async writes through the generic proxy, wgmma reads shared memory through the async proxy
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }
// keeps a register that an asynchronous wgmma reads or writes live and unmoved across the wait
__device__ __forceinline__ void reg_fence(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 wgmma); rows are 128 bytes, 8-row groups are 1024 bytes
// apart (SBO), LBO is unused by swizzled K-major operands.  A k-step inside the 128-byte row advances the start address.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// D (+)= A * B^T for one warpgroup: D = 64 x BN fp32 fragment, A = 64 x K fragment in registers (tf32: K = 8, f16: K = 16),
// B = K-major shared-memory tile behind `bdesc`.  scale_d == 0 overwrites D.
template <int BN, bool F16>
struct Wgmma;
template <> struct Wgmma<128, false> {
  static __device__ __forceinline__ void mma(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
  }
};
template <> struct Wgmma<64, false> {
  static __device__ __forceinline__ void mma(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
  }
};
template <> struct Wgmma<32, false> {
  static __device__ __forceinline__ void mma(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
        "}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
  }
};
template <> struct Wgmma<128, true> {
  static __device__ __forceinline__ void mma(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
  }
};
template <> struct Wgmma<64, true> {
  static __device__ __forceinline__ void mma(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
  }
};
template <> struct Wgmma<32, true> {
  static __device__ __forceinline__ void mma(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
        "}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
  }
};

// two floats -> packed fp16 pair, round to nearest even, saturating at +-65504 (a stray out-of-range value must not turn
// into inf - inf = NaN in the remainder piece); `lo` lands in bits 0..15 (the lower K index)
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;\n" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float f16_lo_to_f32(uint32_t pair) {
  float f;
  asm("{\n\t.reg .f16 l, h;\n\tmov.b32 {l, h}, %1;\n\tcvt.f32.f16 %0, l;\n\t}\n" : "=f"(f) : "r"(pair));
  return f;
}
__device__ __forceinline__ float f16_hi_to_f32(uint32_t pair) {
  float f;
  asm("{\n\t.reg .f16 l, h;\n\tmov.b32 {l, h}, %1;\n\tcvt.f32.f16 %0, h;\n\t}\n" : "=f"(f) : "r"(pair));
  return f;
}

__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// Balanced mode plan, shared by the conv kernel and the reduce pass (both derive it from the device-side row count).
// All but the last full round of tiles run data-parallel (whole tiles); the last full round and the partial round
// after it - between 1 and 2 x CTAs - 1 tiles - are cut stream-K style into equal ranges of U units per CTA.  Merging
// the last full round in keeps the ranges long (>= one tile's reduction), so a tile has <= 2 segments; only when
// there is no full round at all (fewer tiles than CTAs) the ranges are shorter: U >= nchunks/6, <= 7 segments.
constexpr int kBalSlabs = 8;                    // workspace slabs: CTAs x kBalSlabs tiles of TC_BM x N floats
constexpr int kBalCounterBytes = 4096;          // balanced mode: per stream-K tile arrival counters at the head of the workspace
struct BalPlan {
  long long rem_tile0;                          // first stream-K tile
  long long U;                                  // units (chunks) per CTA
  int slabs;                                    // workspace slabs per stream-K tile
};
__host__ __device__ __forceinline__ BalPlan bal_plan(long long tiles, long long grid, int nchunks) {
  BalPlan p;
  const long long rounds = tiles / grid;
  const long long dp_rounds = (tiles % grid == 0) ? rounds : (rounds > 0 ? rounds - 1 : 0);
  p.rem_tile0 = dp_rounds * grid;
  const long long rem_tiles = tiles - p.rem_tile0;
  const long long even = (rem_tiles * nchunks + grid - 1) / grid;
  const long long floor_u = (nchunks + 5) / 6;
  p.U = even > floor_u ? even : floor_u;
  p.slabs = rem_tiles >= grid ? 3 : kBalSlabs;  // rem_tiles * slabs <= grid * kBalSlabs either way (rem_tiles < 2 * grid)
  return p;
}

template <int BN, bool F16>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_rows_tc_kernel(const wmd_conv_desc d, const float* __restrict__ wtc,
                                                                     const int splits, float* __restrict__ partial) {
  using Cfg = TcCfg<BN, F16>;
  constexpr int TC_B_TILE = Cfg::B_TILE;
  constexpr int B_IMG = Cfg::B_IMG;                         // bytes of one chunk's weight image
  constexpr int ACC = Cfg::ACC;
  constexpr int STAGE = Cfg::STAGE;
  extern __shared__ unsigned char smem_dyn[];
  __shared__ int s_fixup;                                  // balanced mode: segments of the tile to reduce here (0 = not the last)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~static_cast<uintptr_t>(1023));
  int32_t* tab0 = reinterpret_cast<int32_t*>(base + TC_STAGES * STAGE);   // [tap][row]: source row in x0, -1 = none
  int32_t* tab1 = tab0 + 9 * TC_BM;                                        // ... in x1

  // F16: operands are fed as fp16 pairs.  Activations are scaled by a power of two chosen from the sources' max |x| (device
  // scalars written by their producers: layout moves, earlier convolutions) so that max |x| s lies in (2^13, 2^14] - no
  // overflow, the low piece stays normal for everything within 2^-11 .. 1 of the maximum; weights carry their own
  // power-of-two scale in the packed image's header.  Both scales are undone exactly in the epilogue.
  float ascale = 1.f, out_scale = 1.f;
  if (F16) {
    float amax = d.amax0 ? __ldg(d.amax0) : 0.f;
    if (d.c1 > 0 && d.amax1) amax = fmaxf(amax, __ldg(d.amax1));
    int e = 0;
    if (amax > 0.f && amax < INFINITY) {
      int ex;
      frexpf(amax, &ex);                         // amax = m * 2^ex, m in [0.5, 1)
      e = 14 - ex;                               // amax * 2^e in [2^13, 2^14)
    }
    e = max(-100, min(100, e));
    ascale = ldexpf(1.f, e);
    out_scale = ldexpf(1.f, -e) * __ldg(wtc);    // header word 0: 1 / weight scale
  }
  const long long HW = static_cast<long long>(d.H) * d.W;
  const int total_px = static_cast<int>(static_cast<long long>(d.N) * HW);
  int rows = d.pixels ? *d.count : total_px;
  rows = min(rows, d.max_rows);
  const int nch0 = (d.c0 + TC_BK - 1) / TC_BK, nch1 = (d.c1 + TC_BK - 1) / TC_BK;
  const int per_tap = nch0 + nch1;
  const int nchunks = d.taps * per_tap;
  const int n_tiles = (d.cout + BN - 1) / BN;
  const long long tiles = static_cast<long long>((rows + TC_BM - 1) / TC_BM) * n_tiles;
  const int Hs = d.H >> d.shift0, Ws = d.W >> d.shift0;
  const bool aligned_rows = (d.taps == 1 && d.map0 == nullptr);
  // rows each source holds: a row index past them reads zeros (a 1x1 stage over its own rows may run past x0's end)
  const long long rows_x0 = (aligned_rows && d.rows0 > 0) ? d.rows0 : static_cast<long long>(d.N) * Hs * Ws;
  const long long rows_x1 = static_cast<long long>(d.N) * HW;

  // fragment ownership: warpgroup wg, warp wq of it; rows row_a and row_a + 8 of the tile, columns 8j + 2 t4 + {0, 1}
  const int wg = warp >> 2, wq = warp & 3, t4 = lane & 3;
  const int row_a = wg * 64 + wq * 16 + (lane >> 2);

  // Work decomposition.  A "unit" is one 32-channel chunk of one output tile.
  //   splits >= 1 : every tile's reduction is cut into `splits` equal ranges (split-K); splits == 1 = whole tiles.
  //   splits == 0 : BALANCED (data-parallel + stream-K, see bal_plan): all but the last full round run whole tiles;
  //                 the units of the remaining tiles are dealt out to all CTAs in equal contiguous ranges of U
  //                 units, so the SMs finish together however many tiles the (device-side) row count yields, and
  //                 only tiles cut by a range boundary pay for partial sums.
  // Segments that do not cover a whole tile write raw partial sums to the workspace; tc_reduce_kernel sums a tile's
  // segments in a fixed order and applies bias + activation, so results stay deterministic.
  const bool balanced = (splits == 0);
  const BalPlan plan = bal_plan(tiles, gridDim.x, nchunks);
  const long long rem_tile0 = balanced ? plan.rem_tile0 : 0;            // first stream-K tile
  const long long rem_units = balanced ? (tiles - rem_tile0) * nchunks : 0;
  const long long U = plan.U;
  long long u = balanced ? static_cast<long long>(blockIdx.x) * U : 0;
  const long long u_end = balanced ? min(rem_units, u + U) : 0;
  long long item = blockIdx.x;
  const long long items = balanced ? rem_tile0 : tiles * splits;
  while (true) {
    long long tile;
    int cb, ce, slab;
    bool whole;
    long long rem_t = 0;                                                // remainder-tile index (balanced partials)
    if (balanced && item < items) {                                     // data-parallel rounds
      tile = item;
      cb = 0; ce = nchunks; slab = 0; whole = true;
      item += gridDim.x;
    } else if (balanced) {                                              // stream-K over the remainder tiles
      if (u >= u_end) break;
      rem_t = u / nchunks;
      tile = rem_tile0 + rem_t;
      cb = static_cast<int>(u - rem_t * nchunks);
      ce = static_cast<int>(min(static_cast<long long>(nchunks), cb + (u_end - u)));
      slab = static_cast<int>(blockIdx.x - (rem_t * nchunks) / U);
      whole = (cb == 0 && ce == nchunks);
      u += ce - cb;
    } else {
      if (item >= items) break;
      tile = item / splits;
      slab = static_cast<int>(item - tile * splits);
      cb = static_cast<int>(static_cast<long long>(slab) * nchunks / splits);
      ce = static_cast<int>(static_cast<long long>(slab + 1) * nchunks / splits);
      whole = (splits == 1);
      item += gridDim.x;
    }
    const int len = ce - cb;
    const int m0 = static_cast<int>(tile / n_tiles) * TC_BM;
    const int nt = static_cast<int>(tile % n_tiles);
    const int n0 = nt * BN;
    // rows / bias 8-byte aligned: the epilogue's pair form for the pairs inside cout
    const bool al_ok = (d.ldy % 2 == 0) && ((reinterpret_cast<uintptr_t>(d.y) & 7) == 0) &&
                       ((reinterpret_cast<uintptr_t>(d.bias) & 7) == 0);

    // thread t: tile row t % 128, taps [t / 128 * 5, ...): the output pixel is read and decoded once per row, the taps'
    // gate / map lookups are independent loads
    {
      const int r = tid & (TC_BM - 1);
      const int t_lo = (tid >> 7) * 5, t_hi = min(d.taps, t_lo + 5);
      const int m = m0 + r;
      int n = 0, y = 0, x = 0;
      const bool live = m < rows;
      if (live && t_lo < t_hi) {
        const unsigned p = static_cast<unsigned>(d.pixels ? d.pixels[m] : m);     // < 2^31 (checked by the host): 32-bit divisions
        const unsigned hw = static_cast<unsigned>(HW);
        n = static_cast<int>(p / hw);
        const unsigned rem = p - static_cast<unsigned>(n) * hw;
        y = static_cast<int>(rem / static_cast<unsigned>(d.W));
        x = static_cast<int>(rem - static_cast<unsigned>(y) * static_cast<unsigned>(d.W));
      }
      // Two rounds of loads for the thread's (up to) five taps instead of one dependent chain per tap: first every tap's
      // coordinates and its three look-ups (gate byte, source-0 index map, source-1 index map) are issued together - the maps
      // are read whether or not the gate turns out to be set, their indices are valid for every in-range coordinate - then
      // the results are combined.
      constexpr int kTapsPerThread = 5;
      int qv[kTapsPerThread];                        // source-1 pixel of the tap, -1 = out of range / dead row
      uint8_t gv[kTapsPerThread];
      int32_t m0v[kTapsPerThread], m1v[kTapsPerThread];
#pragma unroll
      for (int k = 0; k < kTapsPerThread; ++k) {
        const int tap = t_lo + k;
        qv[k] = -1;
        gv[k] = 1;
        m0v[k] = kNoRow;
        m1v[k] = kNoRow;
        if (live && tap < t_hi) {
          int qy = y, qx = x;
          if (d.taps == 9) { qy += tap / 3 - 1; qx += tap % 3 - 1; }
          bool ok = pad_coord(qy, d.H, d.pad_mode);
          ok = pad_coord(qx, d.W, d.pad_mode) && ok;
          if (ok) {
            const int q = (n * d.H + qy) * d.W + qx;
            qv[k] = q;
            if (d.gate) gv[k] = d.gate[q];
            m1v[k] = d.map1 ? d.map1[q] : q;        // -1 (not in the compact skip list) = kNoRow
            if (aligned_rows) {
              m0v[k] = m;
            } else {
              const int qs = (n * Hs + (qy >> d.shift0)) * Ws + (qx >> d.shift0);
              m0v[k] = d.map0 ? d.map0[qs] : qs;
            }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < kTapsPerThread; ++k) {
        const int tap = t_lo + k;
        if (tap < t_hi) {
          const bool ok = qv[k] >= 0 && gv[k] != 0;
          tab0[tap * TC_BM + r] = (ok && m0v[k] >= 0 && m0v[k] < rows_x0) ? m0v[k] : kNoRow;
          tab1[tap * TC_BM + r] = (ok && m1v[k] < rows_x1) ? m1v[k] : kNoRow;
        }
      }
    }
    __syncthreads();

    const unsigned char* wtile = reinterpret_cast<const unsigned char*>(wtc) +
                                 (F16 ? 128 : 0) + static_cast<long long>(nt) * nchunks * B_IMG;   // f16 images follow a 128-byte header

    // Chunk c of the tile into stage s: the weight image as it is, and the implicit im2col - for every tile row the
    // 32-channel slice of its tap's source row (channel chunk outermost, taps innermost: the nine taps of a chunk re-read
    // (almost) the same rows while they are hot in L2).  No row / channels past C: zero fill.
    auto load_chunk = [&](int c, int s) {
      unsigned char* st = base + s * STAGE;
      const unsigned char* wsrc = wtile + static_cast<long long>(c) * B_IMG;
#pragma unroll
      for (int i = 0; i < B_IMG / 16 / TC_THREADS; ++i) {
        const int o = (tid + i * TC_THREADS) * 16;
        cp_async16(st + o, wsrc + o, 16);
      }
      const int rr = c / d.taps;
      const int tap = c - rr * d.taps;
      const bool src1 = rr >= nch0;
      const int col = (src1 ? rr - nch0 : rr) * TC_BK;
      const float* x = src1 ? d.x1 : d.x0;
      const long long ld = src1 ? d.ld1 : d.ld0;
      const int csrc = src1 ? d.c1 : d.c0;
      const int32_t* tab = (src1 ? tab1 : tab0) + tap * TC_BM;
      float* sa = reinterpret_cast<float*>(st + B_IMG);
#pragma unroll
      for (int i = 0; i < TC_BM * 8 / TC_THREADS; ++i) {
        const int pc = tid + i * TC_THREADS, r = pc >> 3, q = pc & 7;
        const int32_t srow = tab[r];
        const int cc = col + 4 * q;
        const int bytes = srow >= 0 ? min(16, max(0, (csrc - cc) * 4)) : 0;
        cp_async16(sa + r * TC_A_LD + 4 * q, bytes ? x + srow * ld + cc : x, bytes);
      }
    };

    float acc[ACC];
#pragma unroll
    for (int j = 0; j < ACC; ++j) acc[j] = 0.f;
    float dacc[ACC];                              // the wgmma accumulators of the running epoch
#pragma unroll
    for (int j = 0; j < ACC; ++j) dacc[j] = 0.f;
    float out_max = 0.f;                          // max |y| this thread stores in this tile (-> d.amax_out)

#pragma unroll
    for (int s = 0; s < TC_STAGES - 1; ++s) {
      if (s < len) load_chunk(cb + s, s);
      cp_async_commit();                          // empty groups keep the wait counts uniform
    }
    for (int i = 0; i < len; ++i) {
      cp_async_wait<TC_STAGES - 2>();             // this thread's copies of chunk i have landed
      fence_proxy_async();
      __syncthreads();                            // everyone's have; both warpgroups are done with chunk i - 1
      if (i + TC_STAGES - 1 < len) load_chunk(cb + i + TC_STAGES - 1, (i + TC_STAGES - 1) % TC_STAGES);
      cp_async_commit();
      const unsigned char* st = base + (i % TC_STAGES) * STAGE;
      const float* sa = reinterpret_cast<const float*>(st + B_IMG);
      const uint64_t b0 = wgmma_desc_sw128(smem_u32(st));
      const uint32_t keep = (i % kFlushChunks) != 0;    // the first MMA of an epoch overwrites the accumulators
      if (F16) {
        // x * s (s a power of two: exact) = h1 + h2 with h1 = fp16(x s) and h2 = fp16(x s - h1): 22 mantissa bits, the
        // precision of the tf32 hi / lo pair.  Fragment of k-step ks: rows (r, r + 8) x channels 16 ks + 2 t4 + {0, 1}, + 8
        uint32_t h1[TC_BK / 16][4], h2[TC_BK / 16][4];
#pragma unroll
        for (int ks = 0; ks < TC_BK / 16; ++ks) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 v = *reinterpret_cast<const float2*>(sa + (row_a + (e & 1) * 8) * TC_A_LD + ks * 16 + 2 * t4 + (e >> 1) * 8);
            const float b0f = v.x * ascale, b1f = v.y * ascale;
            const uint32_t p = pack_f16x2(b0f, b1f);
            h1[ks][e] = p;
            h2[ks][e] = pack_f16x2(b0f - f16_lo_to_f32(p), b1f - f16_hi_to_f32(p));
          }
        }
        wgmma_fence();
        // rows of the weight tile: [h1: 64 B | h2: 64 B]; a k-step is 16 channels = 32 B
#pragma unroll
        for (int ks = 0; ks < TC_BK / 16; ++ks) {
          const uint64_t bh = b0 + static_cast<uint64_t>(2 * ks);
          const uint64_t bl = bh + 4u;
          Wgmma<BN, true>::mma(dacc, h2[ks], bh, ks == 0 ? keep : 1u);   // lo*hi
          Wgmma<BN, true>::mma(dacc, h1[ks], bl, 1u);                    // hi*lo
          Wgmma<BN, true>::mma(dacc, h1[ks], bh, 1u);                    // hi*hi
        }
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int ks = 0; ks < TC_BK / 16; ++ks)
#pragma unroll
          for (int e = 0; e < 4; ++e) { reg_fence(h1[ks][e]); reg_fence(h2[ks][e]); }
      } else {
        // fragment of k-step ks: rows (r, r + 8) x channels 8 ks + t4, + 4; tf32 hi by truncation, exact remainder lo
        uint32_t hi[TC_BK / 8][4], lo[TC_BK / 8][4];
#pragma unroll
        for (int ks = 0; ks < TC_BK / 8; ++ks) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float v = sa[(row_a + (e & 1) * 8) * TC_A_LD + ks * 8 + t4 + (e >> 1) * 4];
            hi[ks][e] = __float_as_uint(v) & 0xFFFFE000u;
            lo[ks][e] = __float_as_uint(v - __uint_as_float(hi[ks][e]));
          }
        }
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < TC_BK / 8; ++ks) {
          const uint64_t bh = b0 + static_cast<uint64_t>(2 * ks);
          const uint64_t bl = bh + static_cast<uint64_t>(TC_B_TILE >> 4);
          Wgmma<BN, false>::mma(dacc, lo[ks], bh, ks == 0 ? keep : 1u);  // lo*hi
          Wgmma<BN, false>::mma(dacc, hi[ks], bl, 1u);                   // hi*lo
          Wgmma<BN, false>::mma(dacc, hi[ks], bh, 1u);                   // hi*hi
        }
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int ks = 0; ks < TC_BK / 8; ++ks)
#pragma unroll
          for (int e = 0; e < 4; ++e) { reg_fence(hi[ks][e]); reg_fence(lo[ks][e]); }
      }
#pragma unroll
      for (int j = 0; j < ACC; ++j) reg_fence(dacc[j]);
      if (((i + 1) % kFlushChunks == 0) || (i == len - 1)) {
#pragma unroll
        for (int j = 0; j < ACC; ++j) acc[j] += dacc[j];
      }
    }
    cp_async_wait<0>();

    // ---- epilogue: bias, activation, pair stores.  acc[4 j + 2 h + e] = row row_a + 8 h, column 8 j + 2 t4 + e
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int my_row = row_a + 8 * h;
      const int m = m0 + my_row;
      if (m < rows && !whole) {
        // raw partial sums of this segment (bias / activation are applied by the reduce pass)
        if (balanced) {                                // compact workspace: [remainder tile][slab][TC_BM rows][BN]
          float* pr = partial + kBalCounterBytes / 4 + ((rem_t * plan.slabs + slab) * TC_BM + my_row) * BN + 2 * t4;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) __stcg(reinterpret_cast<float2*>(pr + 8 * j), make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
        } else {                                       // split-K: [slab][max_rows][ldy]
          float* pr = partial + kBalCounterBytes / 4 + (static_cast<long long>(slab) * d.max_rows + m) * d.ldy;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int co = n0 + 8 * j + 2 * t4;      // ldy % 4 == 0: a pair that starts below cout stays inside the row
            if (co < d.cout) *reinterpret_cast<float2*>(pr + co) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          }
        }
      } else if (m < rows) {
        float* yr = d.y + static_cast<long long>(m) * d.ldy;
        // The activation is picked once per tile, not per element (act is a kernel argument); pairs that lie inside cout
        // take vector bias loads and no per-element bounds.
        const float ap = d.act_param;
        auto store_all = [&](auto actf) {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int co = n0 + 8 * j + 2 * t4;
            const float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
            if (al_ok && co + 1 < d.cout) {
              const float2 bq = d.bias ? __ldg(reinterpret_cast<const float2*>(d.bias + co)) : make_float2(0.f, 0.f);
              float2 o;
              if (F16) {                               // out_scale is a power of two: the product is exact
                o.x = fmaf(a0, out_scale, bq.x); o.y = fmaf(a1, out_scale, bq.y);
              } else {
                o.x = a0 + bq.x; o.y = a1 + bq.y;
              }
              o.x = actf(o.x); o.y = actf(o.y);
              out_max = fmaxf(out_max, fmaxf(fabsf(o.x), fabsf(o.y)));
              *reinterpret_cast<float2*>(yr + co) = o;
            } else {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (co + e < d.cout) {
                  const float a = F16 ? __fmul_rn(e ? a1 : a0, out_scale) : (e ? a1 : a0);
                  const float o = actf(a + (d.bias ? __ldg(d.bias + co + e) : 0.f));
                  out_max = fmaxf(out_max, fabsf(o));
                  yr[co + e] = o;
                }
              }
            }
          }
        };
        if (d.act == WMD_ACT_ELU) store_all([](float v) { return v > 0.f ? v : expm1_nonpos(v); });
        else if (d.act == WMD_ACT_LRELU) store_all([ap](float v) { return v > 0.f ? v : v * ap; });
        else if (d.act == WMD_ACT_NONE) store_all([](float v) { return v; });
        else store_all([&](float v) { return activate(v, d.act, ap); });
      }
    }
    // ---- balanced mode, stream-K fix-up: the LAST segment of a cut tile to arrive (arrival counter per tile, left at zero
    // for the next launch) sums all segments in slab order - bias first, the order of every earlier version - applies the
    // activation and writes the rows.  No CTA waits for another one and the result does not depend on who is last.
    if (balanced && !whole) {
      __threadfence();
      __syncthreads();
      if (tid == 0) {
        const long long first = (rem_t * nchunks) / U, last = ((rem_t + 1) * nchunks - 1) / U;
        const int nseg = static_cast<int>(last - first + 1);
        unsigned* cnt = reinterpret_cast<unsigned*>(partial) + rem_t;
        const unsigned t = atomicAdd(cnt, 1u);
        s_fixup = (t == static_cast<unsigned>(nseg - 1)) ? nseg : 0;
        if (s_fixup) *cnt = 0u;
      }
      __syncthreads();
      const int nseg = s_fixup;
      if (nseg > 0) {
        __threadfence();
        // Cooperative and coalesced: the slabs are row-major [256][BN], so consecutive threads take consecutive float4s
        // (a warp reads 512 contiguous bytes per slab and writes 512 contiguous bytes of one output row); four quads per
        // thread are in flight, i.e. 4 x nseg independent L2 loads instead of one dependent load per quad.
        // tf32 form: bias first, then the slabs in slab order (the order of every earlier version); f16: slabs, scale, bias.
        const float* pb = partial + kBalCounterBytes / 4 + rem_t * plan.slabs * TC_BM * BN;
        constexpr int kQuadsPerRow = BN / 4;
        constexpr int kQuads = TC_BM * kQuadsPerRow;
        constexpr int kUnroll = 4;
        static_assert(kQuads % (TC_THREADS * kUnroll) == 0, "quads of a tile divide evenly");
        const int tile_rows = min(TC_BM, rows - m0);
        const float ap = d.act_param;
        for (int base = tid; base < kQuads; base += TC_THREADS * kUnroll) {
          float4 v[kUnroll], bq[kUnroll];
          int r[kUnroll], co[kUnroll];
          bool live[kUnroll];
#pragma unroll
          for (int q = 0; q < kUnroll; ++q) {
            const int idx = base + q * TC_THREADS;
            r[q] = idx / kQuadsPerRow;
            co[q] = n0 + 4 * (idx % kQuadsPerRow);
            live[q] = r[q] < tile_rows && co[q] < d.cout;
            bq[q] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (live[q] && d.bias) {
              if (al_ok && co[q] + 3 < d.cout) {
                bq[q] = __ldg(reinterpret_cast<const float4*>(d.bias + co[q]));
              } else {
                bq[q].x = __ldg(d.bias + co[q]);
                if (co[q] + 1 < d.cout) bq[q].y = __ldg(d.bias + co[q] + 1);
                if (co[q] + 2 < d.cout) bq[q].z = __ldg(d.bias + co[q] + 2);
                if (co[q] + 3 < d.cout) bq[q].w = __ldg(d.bias + co[q] + 3);
              }
            }
            v[q] = F16 ? make_float4(0.f, 0.f, 0.f, 0.f) : bq[q];
          }
          for (int sidx = 0; sidx < nseg; ++sidx) {
            const float4* ps = reinterpret_cast<const float4*>(pb + static_cast<long long>(sidx) * TC_BM * BN) + base;
#pragma unroll
            for (int q = 0; q < kUnroll; ++q) {
              if (live[q]) {
                const float4 pq = __ldcg(ps + q * TC_THREADS);
                v[q].x += pq.x; v[q].y += pq.y; v[q].z += pq.z; v[q].w += pq.w;
              }
            }
          }
#pragma unroll
          for (int q = 0; q < kUnroll; ++q) {
            if (live[q]) {
              float4 o = v[q];
              if (F16) {
                o.x = __fadd_rn(__fmul_rn(o.x, out_scale), bq[q].x); o.y = __fadd_rn(__fmul_rn(o.y, out_scale), bq[q].y);
                o.z = __fadd_rn(__fmul_rn(o.z, out_scale), bq[q].z); o.w = __fadd_rn(__fmul_rn(o.w, out_scale), bq[q].w);
              }
              o.x = activate(o.x, d.act, ap); o.y = activate(o.y, d.act, ap);
              o.z = activate(o.z, d.act, ap); o.w = activate(o.w, d.act, ap);
              float* yq = d.y + static_cast<long long>(m0 + r[q]) * d.ldy + co[q];
              out_max = fmaxf(out_max, fabsf(o.x));
              if (co[q] + 3 < d.cout) {                // balanced mode requires ldy % 4 == 0 and a 16-byte aligned y
                out_max = fmaxf(fmaxf(out_max, fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w)));
                *reinterpret_cast<float4*>(yq) = o;
              } else {
                yq[0] = o.x;
                if (co[q] + 1 < d.cout) { yq[1] = o.y; out_max = fmaxf(out_max, fabsf(o.y)); }
                if (co[q] + 2 < d.cout) { yq[2] = o.z; out_max = fmaxf(out_max, fabsf(o.z)); }
              }
            }
          }
        }
      }
    }
    if (d.amax_out) {                              // max |y| of the layer for its consumers' operand scaling (order independent)
      for (int o = 16; o > 0; o >>= 1) out_max = fmaxf(out_max, __shfl_xor_sync(0xffffffffu, out_max, o));
      if (lane == 0 && out_max > __ldcg(d.amax_out)) atomicMax(reinterpret_cast<unsigned*>(d.amax_out), __float_as_uint(out_max));   // most warps skip the atomic
    }
    __syncthreads();   // tap tables and stages free for the next tile
  }
}

// w (Cout, Cin, taps) fp32 -> per (n-tile, chunk) smem image [tf32 hi: BN x 32 | tf32 lo: BN x 32], K-major,
// 128B-swizzled.  Chunk order = the kernel's: source-0 channel chunks then source-1 chunks, the taps of a chunk innermost.
__global__ void pack_weight_tc_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int c0, int c1,
                                      int taps, int BN, long long total) {
  const int nch0 = (c0 + TC_BK - 1) / TC_BK, nch1 = (c1 + TC_BK - 1) / TC_BK;
  const int per_tap = nch0 + nch1;
  const int nchunks = taps * per_tap;
  const int Cin = c0 + c1;
  const long long tile_floats = static_cast<long long>(BN) * TC_BK;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += step) {
    // i indexes LOGICAL (nt, chunk, hilo, n, kk); the store address applies the swizzle
    long long t = i;
    const int kk = static_cast<int>(t % TC_BK); t /= TC_BK;
    const int n = static_cast<int>(t % BN); t /= BN;
    const int hilo = static_cast<int>(t % 2); t /= 2;
    const int c = static_cast<int>(t % nchunks);
    const int nt = static_cast<int>(t / nchunks);
    const int rr = c / taps;
    const int tap = c - rr * taps;
    const bool src1 = rr >= nch0;
    const int ci_local = (src1 ? rr - nch0 : rr) * TC_BK + kk;
    const int csrc = src1 ? c1 : c0;
    const int co = nt * BN + n;
    float v = 0.f;
    if (ci_local < csrc && co < Cout) {
      const int ci = (src1 ? c0 : 0) + ci_local;
      v = __ldg(w + (static_cast<long long>(co) * Cin + ci) * taps + tap);
    }
    const float hi = tf32_rna(v);
    const float val = hilo == 0 ? hi : tf32_rna(v - hi);
    const long long tile_base = ((static_cast<long long>(nt) * nchunks + c) * 2 + hilo) * tile_floats;
    const int piece = kk >> 2, within = kk & 3;
    out[tile_base + static_cast<long long>(n) * TC_BK + ((piece ^ (n & 7)) << 2) + within] = val;
  }
}

// y[m, co] = act(bias[co] + sum_s partial_s[m][co]) in a fixed order (deterministic).  splits >= 2: every tile has
// `splits` slabs laid out [slab][max_rows][ldy].  splits == 0 (balanced): only the remainder tiles have partial sums,
// laid out [remainder tile][slab][256][BN]; the number of segments of a tile follows from the same unit arithmetic the
// conv kernel used (grid = its CTA count); a remainder tile that one CTA covered entirely was finished there.
__global__ void tc_reduce_kernel(const float* __restrict__ partial, int splits, int grid, int BN, int nchunks,
                                 const float* __restrict__ bias, float* __restrict__ y, int ldy, int cout,
                                 const int32_t* __restrict__ count, int max_rows, int act, float act_param) {
  partial += kBalCounterBytes / 4;                   // the workspace starts with the balanced mode's arrival counters (kept zero)
  const int rows = count ? min(*count, max_rows) : max_rows;
  const long long slab_sz = static_cast<long long>(max_rows) * ldy;
  const int n_tiles = (cout + BN - 1) / BN;
  const long long tiles = static_cast<long long>((rows + TC_BM - 1) / TC_BM) * n_tiles;
  const BalPlan plan = bal_plan(tiles, grid, nchunks);
  const long long rem_tile0 = splits == 0 ? plan.rem_tile0 : 0;
  const long long U = plan.U;
  const int quads = BN >> 2;                         // float4 columns of a tile (ldy is a multiple of 4)
  // one CTA per tile per round: the slab arithmetic is per tile, the element loop has no divisions by run-time values
  for (long long tile = rem_tile0 + blockIdx.x; tile < tiles; tile += gridDim.x) {
    int nslabs = splits;
    const long long rem_t = tile - rem_tile0;
    if (splits == 0) {
      const long long first = (rem_t * nchunks) / U, last = ((rem_t + 1) * nchunks - 1) / U;
      if (first == last) continue;                   // whole tile: already written with bias + activation
      nslabs = static_cast<int>(last - first + 1);
    }
    const int m0 = static_cast<int>(tile / n_tiles) * TC_BM;
    const int co0 = static_cast<int>(tile % n_tiles) * BN;
    const int mrows = min(TC_BM, rows - m0);
    const float* pbal = partial + rem_t * plan.slabs * TC_BM * BN;
    for (int e = threadIdx.x; e < mrows * quads; e += blockDim.x) {
      const int r = e / quads, q = e - r * quads;
      const int co = co0 + (q << 2);
      if (co >= cout) continue;
      const long long o = static_cast<long long>(m0 + r) * ldy + co;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (bias) {
        v.x = __ldg(bias + co);
        if (co + 1 < cout) v.y = __ldg(bias + co + 1);
        if (co + 2 < cout) v.z = __ldg(bias + co + 2);
        if (co + 3 < cout) v.w = __ldg(bias + co + 3);
      }
      for (int sidx = 0; sidx < nslabs; ++sidx) {
        const float4 p = splits == 0 ? __ldg(reinterpret_cast<const float4*>(pbal + (static_cast<long long>(sidx) * TC_BM + r) * BN + (q << 2)))
                                     : __ldg(reinterpret_cast<const float4*>(partial + sidx * slab_sz + o));
        v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
      }
      v.x = activate(v.x, act, act_param); v.y = activate(v.y, act, act_param);
      v.z = activate(v.z, act, act_param); v.w = activate(v.w, act, act_param);
      if (co + 3 < cout) {
        *reinterpret_cast<float4*>(y + o) = v;
      } else {
        y[o] = v.x;
        if (co + 1 < cout) y[o + 1] = v.y;
        if (co + 2 < cout) y[o + 2] = v.z;
      }
    }
  }
}

// ---- fp16 weight images (precision = WMD_PREC_F16X3) -----------------------------------------------------------------
__global__ void absmax_kernel(const float* __restrict__ x, long long count, float* __restrict__ out) {
  float m = 0.f;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += step) m = fmaxf(m, fabsf(__ldg(x + i)));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > __ldcg(out)) atomicMax(reinterpret_cast<unsigned*>(out), __float_as_uint(m));
}

// header word 0 holds max |w| when this runs; it is replaced by 1 / s_w by the last block... no: by a second tiny kernel
// (finish_header) so that every pack thread reads the same maximum.
__global__ void pack_weight_tc16_kernel(const float* __restrict__ w, unsigned char* __restrict__ out, int Cout, int c0, int c1,
                                        int taps, int BN, long long total) {
  const float wmax = *reinterpret_cast<const float*>(out);        // header word 0: max |w| (absmax_kernel)
  int e = 0;
  if (wmax > 0.f && wmax < INFINITY) {
    int ex;
    frexpf(wmax, &ex);
    e = 14 - ex;
  }
  e = max(-100, min(100, e));
  const float sw = ldexpf(1.f, e);
  const int nch0 = (c0 + TC_BK - 1) / TC_BK, nch1 = (c1 + TC_BK - 1) / TC_BK;
  const int per_tap = nch0 + nch1;
  const int nchunks = taps * per_tap;
  const int Cin = c0 + c1;
  __half* img = reinterpret_cast<__half*>(out + 128);
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += step) {
    // i indexes LOGICAL (nt, chunk, n, kk); the row of a tile is 64 halves: [h1: kk 0..31 | h2: kk 0..31], 128B-swizzled
    long long t = i;
    const int kk = static_cast<int>(t % TC_BK); t /= TC_BK;
    const int n = static_cast<int>(t % BN); t /= BN;
    const int c = static_cast<int>(t % nchunks);
    const int nt = static_cast<int>(t / nchunks);
    const int rr = c / taps;
    const int tap = c - rr * taps;
    const bool src1 = rr >= nch0;
    const int ci_local = (src1 ? rr - nch0 : rr) * TC_BK + kk;
    const int csrc = src1 ? c1 : c0;
    const int co = nt * BN + n;
    float v = 0.f;
    if (ci_local < csrc && co < Cout) {
      const int ci = (src1 ? c0 : 0) + ci_local;
      v = __ldg(w + (static_cast<long long>(co) * Cin + ci) * taps + tap) * sw;
    }
    const __half h1 = __float2half_rn(v);
    const __half h2 = __float2half_rn(v - __half2float(h1));
    const long long tile_base = (static_cast<long long>(nt) * nchunks + c) * (static_cast<long long>(BN) * 64);
    // halves kk (h1) and 32 + kk (h2) of row n; 16-byte pieces (8 halves) are XOR-swizzled with the row index
    const int p1 = kk >> 3, p2 = (32 + kk) >> 3, within = kk & 7;
    img[tile_base + static_cast<long long>(n) * 64 + ((p1 ^ (n & 7)) << 3) + within] = h1;
    img[tile_base + static_cast<long long>(n) * 64 + ((p2 ^ (n & 7)) << 3) + within] = h2;
  }
}
__global__ void finish_header_tc16_kernel(unsigned char* out) {
  float* h = reinterpret_cast<float*>(out);
  const float wmax = h[0];
  int e = 0;
  if (wmax > 0.f && wmax < INFINITY) {
    int ex;
    frexpf(wmax, &ex);
    e = 14 - ex;
  }
  e = max(-100, min(100, e));
  h[1] = wmax;
  h[0] = ldexpf(1.f, -e);                          // 1 / s_w: what the conv kernel reads
}

static int tc_tile_n(int cout) { return cout >= 96 ? 128 : (cout >= 48 ? 64 : 32); }

static int g_reserved_sms = 0;     // SMs the persistent grid leaves free (for a collective's kernel on multi-GPU runs)
static int g_shared_taps = 1;      // kept for the C ABI: every tap gathers its own rows in this engine

template <int BN, bool F16>
static int launch_tc(const wmd_conv_desc& d, int splits, float* partial, cudaStream_t stream) {
  using Cfg = TcCfg<BN, F16>;
  static bool attr_done[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {   // outside the cache: set it on every launch
    int rc = record(cudaFuncSetAttribute(conv_rows_tc_kernel<BN, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(Cfg::SMEM)));
    if (rc != WMD_OK) return rc;
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  const long long tiles = static_cast<long long>(ceil_div(d.max_rows, TC_BM)) * ceil_div(d.cout, BN) * (splits > 0 ? splits : 1);
  const long long cap = sm_count() - g_reserved_sms > 1 ? sm_count() - g_reserved_sms : 1;
  const int grid = splits == 0 ? static_cast<int>(cap) : static_cast<int>(tiles < cap ? (tiles < 1 ? 1 : tiles) : cap);
  conv_rows_tc_kernel<BN, F16><<<grid, TC_THREADS, Cfg::SMEM, stream>>>(d, d.w, splits, partial);
  int rc = launched();
  if (rc != WMD_OK || splits <= 1) return rc;      // whole tiles, or balanced: the kernel's own fix-up finishes cut tiles
  const int nchunks = d.taps * ((d.c0 + TC_BK - 1) / TC_BK + (d.c1 + TC_BK - 1) / TC_BK);
  const long long all_tiles = static_cast<long long>(ceil_div(d.max_rows, TC_BM)) * ceil_div(d.cout, BN);
  const long long red_grid = all_tiles < 8 * cap ? all_tiles : 8 * cap;
  tc_reduce_kernel<<<static_cast<int>(red_grid < 1 ? 1 : red_grid), 256, 0, stream>>>(partial, splits, grid, BN, nchunks, d.bias, d.y, d.ldy, d.cout,
                                                              d.count, d.max_rows, d.act, d.act_param);
  return launched();
}

}  // namespace wmd

extern "C" int wmd_conv_tc_tile_n(int cout) { return wmd::tc_tile_n(cout); }

extern "C" int wmd_conv_tc_set_reserved_sms(int n) {
  const int was = wmd::g_reserved_sms;
  if (n >= 0) wmd::g_reserved_sms = n;
  return was;
}

extern "C" int wmd_conv_tc_set_shared_taps(int on) {
  const int was = wmd::g_shared_taps;
  if (on >= 0) wmd::g_shared_taps = on ? 1 : 0;
  return was;
}

extern "C" size_t wmd_conv_tc_weight_floats(int cout, int c0, int c1, int taps) {
  using namespace wmd;
  const int bn = tc_tile_n(cout);
  const int nchunks = taps * ((c0 + TC_BK - 1) / TC_BK + (c1 + TC_BK - 1) / TC_BK);
  return static_cast<size_t>(ceil_div(cout, bn)) * nchunks * 2 * bn * TC_BK;
}

extern "C" int wmd_pack_conv_weight_tc_f32(const float* w, float* packed, int Cout, int c0, int c1, int taps,
                                           wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(w && packed, WMD_ERR_ARG);
  WMD_REQUIRE(Cout > 0 && c0 > 0 && c1 >= 0 && (taps == 1 || taps == 9), WMD_ERR_SHAPE);
  const long long total = static_cast<long long>(wmd_conv_tc_weight_floats(Cout, c0, c1, taps));
  pack_weight_tc_kernel<<<stride_grid(total, 256), 256, 0, as_stream(stream)>>>(w, packed, Cout, c0, c1, taps,
                                                                               tc_tile_n(Cout), total);
  return launched();
}

extern "C" size_t wmd_conv_tc16_weight_bytes(int cout, int c0, int c1, int taps) {
  using namespace wmd;
  const int bn = tc_tile_n(cout);
  const int nchunks = taps * ((c0 + TC_BK - 1) / TC_BK + (c1 + TC_BK - 1) / TC_BK);
  return 128 + static_cast<size_t>(ceil_div(cout, bn)) * nchunks * bn * 128;
}

extern "C" int wmd_pack_conv_weight_tc16_f32(const float* w, void* packed, int Cout, int c0, int c1, int taps,
                                             wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(w && packed, WMD_ERR_ARG);
  WMD_REQUIRE(Cout > 0 && c0 > 0 && c1 >= 0 && (taps == 1 || taps == 9), WMD_ERR_SHAPE);
  WMD_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 127) == 0, WMD_ERR_SHAPE);
  cudaStream_t st = as_stream(stream);
  unsigned char* out = static_cast<unsigned char*>(packed);
  int rc = record(cudaMemsetAsync(out, 0, 128, st));
  if (rc != WMD_OK) return rc;
  const long long nw = static_cast<long long>(Cout) * (c0 + c1) * taps;
  absmax_kernel<<<stride_grid(nw, 256), 256, 0, st>>>(w, nw, reinterpret_cast<float*>(out));
  rc = launched();
  if (rc != WMD_OK) return rc;
  const int bn = tc_tile_n(Cout);
  const int nchunks = taps * ((c0 + TC_BK - 1) / TC_BK + (c1 + TC_BK - 1) / TC_BK);
  const long long total = static_cast<long long>(ceil_div(Cout, bn)) * nchunks * bn * TC_BK;
  pack_weight_tc16_kernel<<<stride_grid(total, 256), 256, 0, st>>>(w, out, Cout, c0, c1, taps, bn, total);
  rc = launched();
  if (rc != WMD_OK) return rc;
  finish_header_tc16_kernel<<<1, 1, 0, st>>>(out);
  return launched();
}

extern "C" int wmd_amax_f32(const float* x, long long count, float* amax, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(x && amax, WMD_ERR_ARG);
  if (count <= 0) return WMD_OK;
  absmax_kernel<<<stride_grid(count, 256, 16), 256, 0, as_stream(stream)>>>(x, count, amax);
  return launched();
}

extern "C" size_t wmd_conv_tc_splitk_ws_bytes(int max_rows, int ldy, int splits) {
  if (splits == 1) return 0;
  if (splits == 0)   // balanced: [stream-K tile][slab][256 rows][N <= 128] floats, tiles x slabs <= CTAs x kBalSlabs whatever the layer size
    return wmd::kBalCounterBytes + static_cast<size_t>(wmd::sm_count()) * wmd::kBalSlabs * wmd::TC_BM * 128 * sizeof(float);
  return wmd::kBalCounterBytes + static_cast<size_t>(splits) * static_cast<size_t>(max_rows) * static_cast<size_t>(ldy) * sizeof(float);
}

extern "C" int wmd_conv_rows_tc_f32(const wmd_conv_desc* dp, wmd_stream_t stream) {
  return wmd_conv_rows_tc_splitk_f32(dp, 1, nullptr, 0, stream);
}

extern "C" int wmd_conv_rows_tc_splitk_f32(const wmd_conv_desc* dp, int splits, void* ws, size_t ws_bytes,
                                           wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(dp, WMD_ERR_ARG);
  WMD_REQUIRE(splits >= 0 && splits <= 16, WMD_ERR_ARG);
  WMD_REQUIRE(splits == 1 || (ws != nullptr && ws_bytes >= wmd_conv_tc_splitk_ws_bytes(dp->max_rows, dp->ldy, splits)),
              WMD_ERR_WORKSPACE);
  wmd_conv_desc d = *dp;
  WMD_REQUIRE(d.x0 && d.w && d.y, WMD_ERR_ARG);
  WMD_REQUIRE(d.taps == 1 || d.taps == 9, WMD_ERR_ARG);
  WMD_REQUIRE(d.pad_mode >= WMD_PAD_ZERO && d.pad_mode <= WMD_PAD_REPLICATE, WMD_ERR_ARG);
  WMD_REQUIRE(d.act >= WMD_ACT_NONE && d.act <= WMD_ACT_SIGMOID, WMD_ERR_ARG);
  WMD_REQUIRE(d.precision == WMD_PREC_TF32X3 || d.precision == WMD_PREC_F16X3, WMD_ERR_ARG);
  WMD_REQUIRE(d.shift0 == 0 || d.shift0 == 1, WMD_ERR_ARG);
  WMD_REQUIRE((d.pixels == nullptr) == (d.count == nullptr), WMD_ERR_ARG);
  WMD_REQUIRE(d.N > 0 && d.H > 0 && d.W > 0 && d.c0 > 0 && d.cout > 0 && d.max_rows >= 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(static_cast<long long>(d.N) * d.H * d.W < (1ll << 31), WMD_ERR_SHAPE);
  if (d.x1 == nullptr) { d.c1 = 0; d.ld1 = 0; }
  WMD_REQUIRE(d.c1 >= 0 && (d.c1 == 0 || d.x1), WMD_ERR_ARG);
  WMD_REQUIRE(d.ld0 >= d.c0 && d.ld0 % 4 == 0 && (reinterpret_cast<uintptr_t>(d.x0) & 15) == 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(d.c1 == 0 || (d.ld1 >= d.c1 && d.ld1 % 4 == 0 && (reinterpret_cast<uintptr_t>(d.x1) & 15) == 0),
              WMD_ERR_SHAPE);
  WMD_REQUIRE((reinterpret_cast<uintptr_t>(d.w) & 15) == 0, WMD_ERR_SHAPE);
  WMD_REQUIRE(d.ldy >= d.cout, WMD_ERR_SHAPE);
  // the partial-sum passes move float4s
  WMD_REQUIRE(splits == 1 || (d.ldy % 4 == 0 && (reinterpret_cast<uintptr_t>(d.y) & 15) == 0 &&
                              (reinterpret_cast<uintptr_t>(ws) & 15) == 0), WMD_ERR_SHAPE);
  if (d.shift0 == 1) WMD_REQUIRE(d.H % 2 == 0 && d.W % 2 == 0, WMD_ERR_SHAPE);
  if (d.pad_mode == WMD_PAD_REFLECT && d.taps == 9) WMD_REQUIRE(d.H >= 2 && d.W >= 2, WMD_ERR_SHAPE);
  // tap tables hold 32-bit offsets in 16-byte units
  WMD_REQUIRE(static_cast<long long>(d.N) * d.H * d.W * (d.ld0 / 4) < (1ll << 32) &&
                  static_cast<long long>(d.N) * d.H * d.W * (d.ld1 / 4) < (1ll << 32),
              WMD_ERR_UNSUPPORTED);
  if (d.max_rows == 0) return WMD_OK;
  {
    const int nchunks = d.taps * ((d.c0 + TC_BK - 1) / TC_BK + (d.c1 + TC_BK - 1) / TC_BK);
    if (splits > nchunks) splits = nchunks;      // every split needs at least one chunk
    if (splits == 0 && nchunks < 2) splits = 1;   // nothing to balance inside a one-chunk reduction
  }
  float* partial = static_cast<float*>(ws);
  const bool f16 = d.precision == WMD_PREC_F16X3;
  if (f16) WMD_REQUIRE(d.amax0 != nullptr && (d.c1 == 0 || d.amax1 != nullptr), WMD_ERR_ARG);
  if (f16) WMD_REQUIRE(splits <= 1, WMD_ERR_UNSUPPORTED);   // tc_reduce_kernel sums unscaled slabs: tf32 operands only
  cudaStream_t st = as_stream(stream);
#define WMD_TC_LAUNCH(BN_) \
  return f16 ? launch_tc<BN_, true>(d, splits, partial, st) : launch_tc<BN_, false>(d, splits, partial, st)
  switch (tc_tile_n(d.cout)) {
    case 128: WMD_TC_LAUNCH(128);
    case 64: WMD_TC_LAUNCH(64);
    default: WMD_TC_LAUNCH(32);
  }
#undef WMD_TC_LAUNCH
}
