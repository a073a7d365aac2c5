// K5-TC: the gather-GEMM convolution on Hopper tensor cores (wgmma), fp32-faithful via 3xTF32.
//
// Same contract as conv_rows_kernel (conv.cu), different engine.  A persistent grid (at most one CTA per SM) walks
// 128 x N output tiles (N = 128 / 64 / 32); a tile's reduction K = (c0 + c1) x taps runs in 32-channel chunks, the
// taps of a channel chunk innermost (their source rows overlap: L2 hits).  384 threads, warp-specialised: one producer
// warpgroup fills a ring of TcCfg::STAGES shared-memory stages, two consumer warpgroups multiply; consumer warpgroup h
// owns tile rows h*64 .. h*64+63 (one wgmma M = 64 each, both share the chunk's weight tile).  Producer and consumers
// step through the same work walk (TcWalk) and hand stages over with mbarriers (full[s]: stage filled, empty[s]: both
// consumers are done with it), so the ring runs on across tile boundaries: the producer builds the next tile's tap table
// and fills its first chunks while the consumers finish the current tile and run its epilogue.
//
//   produce (warpgroup 0, setmaxnreg down to 40 registers)
//     * B (weights) is pre-split, pre-swizzled by wmd_pack_conv_weight_tc_f32 into one [hi | lo] image per (n-tile,
//       chunk): K-major, 128-byte swizzled, contiguous - one bulk copy (cp.async.bulk, completion counted in bytes on
//       full[s]); the wgmma reads it straight from shared memory through a descriptor;
//     * implicit im2col: the 128-byte channel slice of each tile row's source row (row from the per-tile tap table,
//       -1 = inactive / padded tap, and the channel tail read zeros) by cp.async with zero fill into a raw fp32 stage
//       padded to 144-byte rows, so that the fragment reads below are free of bank conflicts; each producer thread's
//       copies arrive on full[s] when they land (cp.async.mbarrier.arrive.noinc);
//   multiply (per consumer warpgroup, setmaxnreg up to 232 registers)
//     * every thread reads its A fragment elements (rows g, g + 8 of its warp's 16, channels t, t + 4 of each k-step)
//       and splits x = hi + lo (hi = x with the 13 low mantissa bits cleared, lo = x - hi: exact) in registers - the
//       register-A form of wgmma, so the split never goes back to shared memory;
//     * 4 k-steps x 3 terms (lo*hi + hi*lo + hi*hi) per chunk, committed as one group; the fragments of chunk i + 1 are
//       read and split into the other of two register sets while chunk i's group runs (wgmma.wait_group 1);
//     * the tensor core's fp32 accumulation is not round-to-nearest, a bias that grows with K.  So accumulation runs in
//       EPOCHS of kFlushChunks chunks: the first MMA of an epoch overwrites the wgmma accumulators, the epoch's end adds
//       them into per-thread fp32 registers with round-to-nearest adds;
//   epilogue (consumers only, named barriers over their 256 threads): bias + activation (picked once per tile) + pair
//     stores;
//   balanced scheduling (long reductions): whole tiles for the full rounds, the (tile, chunk) units of the remainder
//     dealt out evenly on the device (stream-K); the last segment of a cut tile to arrive sums all segments in slab
//     order, cooperatively and coalesced.
// Optional fp16-pair operand form (F16 = true, wmd_conv_desc.precision): x 2^e = h1 + h2 as fp16, f16 MMAs with K = 16
// (half the instructions), scale from the sources' max |x| (device scalars), weights' scale in the packed image's header.
// The window and row-set forms (one slot of rows per channel chunk, read by all nine taps) split in shared memory
// instead: at a slot's first step the 256 consumer threads turn its rows into fp16 pairs in place (split_slot_rows, the
// same split_f16x2 the registers use), and every k-step's fragments come from one ldmatrix.x4 per piece.
#include <cuda_fp16.h>

#include "common.cuh"

namespace wmd {

constexpr int TC_BM = 128;                      // rows per CTA tile = 2 warpgroups x wgmma M = 64
constexpr int TC_BK = 32;                       // floats per chunk = one 128-byte row of a weight image
constexpr int TC_PRODUCERS = 128;               // warpgroup 0: tap tables and copies
constexpr int TC_CONSUMERS = 256;               // warpgroups 1, 2: each multiplies its 64 rows, both run the epilogue
constexpr int TC_THREADS = TC_PRODUCERS + TC_CONSUMERS;
// setmaxnreg: every thread starts with the launch allocation (64 K registers / 384 threads, in steps of 8 = 168); the
// consumers' increase waits until the producer's decrease has returned enough registers to the pool
constexpr int TC_LAUNCH_REGS = (65536 / (TC_PRODUCERS + TC_CONSUMERS)) & ~7;
constexpr int TC_PRODUCER_REGS = 40;
constexpr int TC_CONSUMER_REGS = 232;
constexpr int TC_A_LD = TC_BK + 4;              // raw A row pitch in floats (144 B: fragment reads hit 32 distinct banks)
constexpr int TC_A_TILE = TC_BM * TC_A_LD * 4;  // 18 KB raw fp32
constexpr int TC_TABLES = 2 * 9 * TC_BM * 4;    // one tap table: [source][tap][row]
constexpr int TC_SMEM_MAX = 227 * 1024;         // dynamic shared memory one CTA may use on an SM
constexpr int TC_MAX_STAGES = 8;
static_assert(TC_PRODUCERS * (TC_LAUNCH_REGS - TC_PRODUCER_REGS) >= TC_CONSUMERS * (TC_CONSUMER_REGS - TC_LAUNCH_REGS),
              "the consumers cannot take more registers than the producer gives back");

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
  // Ring depth: as many stages as fit beside the tap tables, the two barriers per stage and the 1 KB alignment slack, at
  // most TC_MAX_STAGES.  The gather's latency is the same for every configuration while a smaller stage drains faster
  // (the f16 form issues half the MMAs), so the small stages need more chunks in flight: 4 for tf32 N = 128, 6 for f16
  // N = 128 and tf32 N = 64, 8 for the rest.
  static constexpr int FIT = (TC_SMEM_MAX - TC_TABLES - 1024) / (STAGE + 2 * 8);
  static constexpr int STAGES = FIT < TC_MAX_STAGES ? FIT : TC_MAX_STAGES;
  static constexpr int BARRIERS = 2 * STAGES * 8;          // full[s], empty[s]
  static constexpr size_t SMEM = static_cast<size_t>(STAGES) * STAGE + TC_TABLES + BARRIERS + 1024;
  static_assert(STAGE % 1024 == 0, "weight images must stay 1024-byte aligned");
  static_assert(STAGES >= 2, "the ring needs two stages");
  static_assert(SMEM <= TC_SMEM_MAX, "one CTA must fit the shared memory of an SM");
};
// Window mode (conv_rows_tc_kernel_window): a dense 3x3 layer (no pixel list, no index maps, no gate) reads, for one tile
// and one source, a CONTIGUOUS range of source rows, and every tap's rows lie inside it.  So the producer loads that
// range's 32-channel slices once per channel chunk into a window slot, and the consumers read tap `t` of tile row r at
// window row tab[t][r] (a window-relative uint16 table that travels with the slot); the nine taps stop fetching (and
// storing) the same rows nine times.  Window of a 128-row tile starting at output row m0, for an output width W (pad
// modes keep every tap within one row / column of its pixel, inside the image):
//   shift 0 (x1, and x0 at full resolution): the tap rows of output row m lie in [m - W - 1, m + W + 1], so the window
//     is [m0 - W - 1, m0 + 127 + W + 1]: 128 + 2 (W + 1) rows;
//   shift 1 (x0 at half resolution, Ws = W / 2, H even): output row Y (global, n H + y) reads source rows
//     ((Y - 1) >> 1) .. ((Y + 1) >> 1), any column.  A tile spans output rows Y0 .. Y0 + D with D <= (W + 126) / W
//     (128 pixels from any column), so the window is the whole source rows ((Y0 - 1) >> 1) .. ((Y0 + D + 1) >> 1): at
//     most ((D + 1) >> 1) + 2 rows of Ws (the count for Y0 even; Y0 odd gives (D >> 1) + 2), starting at
//     ((Y0 - 1) >> 1) Ws.
// Slots hold TC_WIN_ROWS rows plus one row of zeros (padded taps and dead rows point at it); a launch whose window is
// larger keeps the gather path.  After the rows and the table a slot has a 16-byte header: word 0 the row-set form's
// per-tap flag, word 1 the number of rows loaded (the rows the f16 form's consumers split in place).
constexpr int TC_WIN_ROWS = 288;                                   // shift 0: W <= 79
constexpr int TC_WIN_DATA = (TC_WIN_ROWS + 1) * TC_A_LD * 4;       // rows + the zero row, 144-byte pitch
constexpr int TC_WIN_TAB = 9 * TC_BM * 2;                          // [tap][row] uint16 window rows
constexpr int TC_SLOT_HDR = 16;
constexpr int TC_WIN_SLOT = TC_WIN_DATA + TC_WIN_TAB + TC_SLOT_HDR;
static_assert(TC_WIN_DATA % 16 == 0 && TC_WIN_SLOT % 16 == 0, "window rows take 16-byte cp.async");
__host__ __device__ __forceinline__ int win_rows(int W, int shift) {
  if (shift == 0) return TC_BM + 2 * (W + 1);
  const int D = (W + TC_BM - 2) / W;
  return (((D + 1) >> 1) + 2) * (W >> 1);
}
__host__ __device__ __forceinline__ int win_base(int m0, int W, int shift) {
  if (shift == 0) return m0 - (W + 1);
  const int Y0 = m0 / W;
  return (Y0 > 0 ? (Y0 - 1) >> 1 : -1) * (W >> 1);
}

// Row-set mode (conv_rows_tc_kernel_rowset): a 3x3 launch through a pixel list, index maps or a gate reads no contiguous
// range, but the 9 x 128 tap rows a tile reads from one source repeat heavily (a 128-pixel tile of the KITTI decoder's
// sparse levels reads 100 - 470 distinct rows of a source in its 1152 tap slots).  So once per tile and source the
// producer collects the distinct rows - a bitmap over the tile's [min, max] row range, thread t owning word t, then
// popcount ranks: ascending order, whatever the thread timing - and a uint16 table [tap][row] of ranks (dead and padded
// taps: the zero row).  Per channel chunk it then loads the distinct rows' 32-channel slices into a slot, as the window
// form does, and the consumers read the slot through the same table form.  A source whose range exceeds the bitmap
// (TC_SET_SPAN) or whose distinct rows exceed the slot (TC_SET_ROWS) stages one slot per tap instead - the tap's 128
// gathered rows, identity table - and says so in the slot's flag word, so the consumers wait for a slot at every step.
// The rows a step reads, and so the bits, are the same either way.
constexpr int TC_SET_ROWS = 480;
constexpr int TC_SET_SPAN = 32 * TC_PRODUCERS;                     // bitmap rows: one 32-bit word per producer thread
constexpr int TC_SET_DATA = (TC_SET_ROWS + 1) * TC_A_LD * 4;
constexpr int TC_SET_SLOT = TC_SET_DATA + TC_WIN_TAB + TC_SLOT_HDR;   // rows + zero row, the table, the header
// the producer's per-source scratch: rank tables, distinct rows, bitmap words, their rank bases; then 128 B of reductions
constexpr int TC_SET_SCRATCH = 2 * (TC_WIN_TAB + TC_SET_ROWS * 4 + 2 * TC_PRODUCERS * 4) + 128;
static_assert(TC_SET_DATA % 16 == 0 && TC_SET_SLOT % 16 == 0 && TC_SET_SCRATCH % 16 == 0, "slot rows take 16-byte cp.async");

// Window and row-set modes: a ring of weight-only stages beside two slots, the producer's tap tables (and the row-set
// scratch), the barriers (full[s], empty[s] of the ring, then full / empty of the two slots) and the alignment slack.
// Window: 4 stages for tf32 N = 128, 8 for the rest; row set: 4 for the 16 KB weight images (f16 N = 128, tf32
// N = 64), 8 for the smaller ones (tf32 N = 128, two stages, is not built: tc_rowset_takes).
template <int BN, bool F16, bool SET = false>
struct TcWinCfg {
  static constexpr int B_IMG = TcCfg<BN, F16>::B_IMG;
  static constexpr int FIXED = 2 * (SET ? TC_SET_SLOT : TC_WIN_SLOT) + TC_TABLES + (SET ? TC_SET_SCRATCH : 0) + 4 * 8 + 1024;
  static constexpr int FIT = (TC_SMEM_MAX - FIXED) / (B_IMG + 2 * 8);
  static constexpr int STAGES = FIT < TC_MAX_STAGES ? FIT : TC_MAX_STAGES;
  static constexpr size_t SMEM = static_cast<size_t>(STAGES) * B_IMG + FIXED + 2 * STAGES * 8;
  static_assert(STAGES >= 2, "the ring needs two stages");
  static_assert(SMEM <= TC_SMEM_MAX, "one CTA must fit the shared memory of an SM");
};

constexpr int kFlushChunks = 32;                // epoch length: K = 1024 per wgmma accumulation run
static_assert(kFlushChunks % 2 == 0, "an epoch starts on register set 0");
constexpr int32_t kNoRow = -1;                  // tap-table entry of an inactive / padded source: the gather writes zeros


__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>   // until at most N committed groups of this warpgroup are pending
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }

// mbarriers in shared memory (phase parity waits), the bulk copy that counts its bytes on one, and named barriers
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n"
      "WMD_MBAR_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra WMD_MBAR_WAIT;\n}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// arrives on `bar` once every cp.async this thread has issued so far has landed; .noinc: the arrival is one of the
// barrier's expected count
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(threads) : "memory");
}
// named barrier ids (0 is __syncthreads): the producer warpgroup's, the consumers' epilogue, the consumers' slot split
constexpr int kProducerBar = 1, kConsumerBar = 2, kSplitBar = 3;
// the four 8 x 8 b16 matrices whose rows lanes 8i .. 8i + 7 address, into r[i] (the mma fragment layout)
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(saddr) : "memory");
}
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

// two floats -> packed fp16 pair, round to nearest even; `lo` lands in bits 0..15 (the lower K index).  Not saturating:
// the operand scale keeps every finite value below 2^14, and an infinite one must stay infinite (its remainder piece is
// then Inf - Inf = NaN, so the output is non-finite where the contract's is; saturation made it a finite 131008 2^-e)
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;\n" : "=r"(r) : "f"(hi), "f"(lo));
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
// The fp16-pair split of two adjacent channels: x s (s a power of two: exact) = h1 + h2 with h1 = fp16(x s) and
// h2 = fp16(x s - h1), 22 mantissa bits, the precision of the tf32 hi / lo pair; each piece packed with the lower
// channel in bits 0..15.  The gather kernel splits its fragment elements in registers, the window and row-set kernels
// split their slots' rows in place (split_slot_rows): both through this function, so the two give the same bits.
__device__ __forceinline__ void split_f16x2(float x0, float x1, float s, uint32_t& h1, uint32_t& h2) {
  const float b0f = x0 * s, b1f = x1 * s;
  h1 = pack_f16x2(b0f, b1f);
  h2 = pack_f16x2(b0f - f16_lo_to_f32(h1), b1f - f16_hi_to_f32(h1));
}
// The window and row-set kernels' f16 form: the consumers (thread ctid of TC_CONSUMERS) split the first `rows` rows of a
// slot in place, once per slot instead of once per tap that reads them.  Each 32-byte group of 8 fp32 channels becomes
// [h1: 8 x fp16 | h2: 8 x fp16]: channels 8 q .. 8 q + 7 of a row keep bytes 32 q .. 32 q + 31, and the pitch stays
// 144 bytes.  The zero row needs no split: fp32 zeros are fp16 zeros.
__device__ __forceinline__ void split_slot_rows(unsigned char* slot, int rows, float s, int ctid) {
#pragma unroll 1
  for (int q = ctid; q < rows * 4; q += TC_CONSUMERS) {
    uint4* p = reinterpret_cast<uint4*>(slot + (q >> 2) * (TC_A_LD * 4) + (q & 3) * 32);
    const uint4 u = p[0], v = p[1];
    uint4 h1, h2;
    split_f16x2(__uint_as_float(u.x), __uint_as_float(u.y), s, h1.x, h2.x);
    split_f16x2(__uint_as_float(u.z), __uint_as_float(u.w), s, h1.y, h2.y);
    split_f16x2(__uint_as_float(v.x), __uint_as_float(v.y), s, h1.z, h2.z);
    split_f16x2(__uint_as_float(v.z), __uint_as_float(v.w), s, h1.w, h2.w);
    p[0] = h1;
    p[1] = h2;
  }
}

// Exponent e of the power-of-two scale of an fp16-pair operand whose (finite-value) maximum is m: m 2^e in [2^13, 2^14),
// so no finite operand overflows fp16 and the low piece h2 = fp16(v 2^e - h1) stays normal for every |v| >= 2^-11 m.
// e is clamped to [-126, 127], where 2^e is a normal float: for finite m only the upper end is reached (m < 2^-113),
// and then m 2^e < 2^14 still.  m = 0 or non-finite: e = 0.
__host__ __device__ __forceinline__ int f16_scale_exp(float m) {
  int e = 0;
  if (m > 0.f && m < INFINITY) {
    int ex;
    frexpf(m, &ex);                              // m = f * 2^ex, f in [0.5, 1)
    e = 14 - ex;
  }
  return e < -126 ? -126 : (e > 127 ? 127 : e);
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

// Work decomposition of one CTA.  A "unit" is one 32-channel chunk of one output tile.
//   splits >= 1 : every tile's reduction is cut into `splits` equal ranges (split-K); splits == 1 = whole tiles.
//   splits == 0 : BALANCED (data-parallel + stream-K, see bal_plan): all but the last full round run whole tiles;
//                 the units of the remaining tiles are dealt out to all CTAs in equal contiguous ranges of U
//                 units, so the SMs finish together however many tiles the (device-side) row count yields, and
//                 only tiles cut by a range boundary pay for partial sums.
// Segments that do not cover a whole tile write raw partial sums to the workspace; tc_reduce_kernel sums a tile's
// segments in a fixed order and applies bias + activation, so results stay deterministic.
// The producer and the consumers each step through their own copy of the walk: the same items in the same order.
struct TcItem {
  long long tile;
  long long rem_t;                              // remainder-tile index (balanced partials)
  int cb, ce;                                   // chunk range [cb, ce) of the tile's reduction
  int slab;                                     // workspace slab of a partial segment
  bool whole;                                   // the range is the whole reduction: the output rows are written here
};
struct TcWalk {
  long long U, u, u_end, item, items, rem_tile0;
  int splits, nchunks;
  __device__ __forceinline__ TcWalk(long long tiles, int splits_, int nchunks_, const BalPlan& plan)
      : splits(splits_), nchunks(nchunks_) {
    const bool balanced = splits == 0;
    rem_tile0 = balanced ? plan.rem_tile0 : 0;                          // first stream-K tile
    const long long rem_units = balanced ? (tiles - rem_tile0) * nchunks : 0;
    U = plan.U;
    u = balanced ? static_cast<long long>(blockIdx.x) * U : 0;
    u_end = balanced ? min(rem_units, u + U) : 0;
    item = blockIdx.x;
    items = balanced ? rem_tile0 : tiles * splits;
  }
  __device__ __forceinline__ bool next(TcItem& w) {
    w.rem_t = 0;
    if (splits == 0 && item < items) {                                  // data-parallel rounds
      w.tile = item;
      w.cb = 0; w.ce = nchunks; w.slab = 0; w.whole = true;
      item += gridDim.x;
    } else if (splits == 0) {                                           // stream-K over the remainder tiles
      if (u >= u_end) return false;
      w.rem_t = u / nchunks;
      w.tile = rem_tile0 + w.rem_t;
      w.cb = static_cast<int>(u - w.rem_t * nchunks);
      w.ce = static_cast<int>(min(static_cast<long long>(nchunks), w.cb + (u_end - u)));
      w.slab = static_cast<int>(blockIdx.x - (w.rem_t * nchunks) / U);
      w.whole = (w.cb == 0 && w.ce == nchunks);
      u += w.ce - w.cb;
    } else {
      if (item >= items) return false;
      w.tile = item / splits;
      w.slab = static_cast<int>(item - w.tile * splits);
      w.cb = static_cast<int>(static_cast<long long>(w.slab) * nchunks / splits);
      w.ce = static_cast<int>(static_cast<long long>(w.slab + 1) * nchunks / splits);
      w.whole = (splits == 1);
      item += gridDim.x;
    }
    return true;
  }
};

template <int V>
struct Ic { static constexpr int value = V; };   // a compile-time register-set index

// How A reaches shared memory: gathered per (chunk, tap) into the stage, or loaded once per channel chunk into a slot as
// a window (dense 3x3 layers, see TC_WIN_ROWS) or as a tile's distinct rows (the other 3x3 layers, see TC_SET_ROWS).
enum TcFeed { kFeedGather = 0, kFeedWindow = 1, kFeedRowset = 2 };

template <int BN, bool F16, int FEED>
__device__ __forceinline__ void conv_rows_tc_body(const wmd_conv_desc& d, const float* __restrict__ wtc, const int splits,
                                                  float* __restrict__ partial) {
  using Cfg = TcCfg<BN, F16>;
  constexpr bool WIN = FEED != kFeedGather;                 // stages hold weights only, A comes from the two slots
  constexpr bool SET = FEED == kFeedRowset;
  constexpr int TC_B_TILE = Cfg::B_TILE;
  constexpr int B_IMG = Cfg::B_IMG;                         // bytes of one chunk's weight image
  constexpr int ACC = Cfg::ACC;
  constexpr int STAGE = WIN ? B_IMG : Cfg::STAGE;
  constexpr int STAGES = WIN ? TcWinCfg<BN, F16, SET>::STAGES : Cfg::STAGES;
  constexpr int SLOT_ROWS = SET ? TC_SET_ROWS : TC_WIN_ROWS;  // slot row SLOT_ROWS holds zeros
  constexpr int SLOT_DATA = SET ? TC_SET_DATA : TC_WIN_DATA;
  constexpr int SLOT = SET ? TC_SET_SLOT : TC_WIN_SLOT;
  constexpr int SLOTS = WIN ? 2 * SLOT : 0;
  constexpr int SCRATCH = SET ? TC_SET_SCRATCH : 0;
  extern __shared__ unsigned char smem_dyn[];
  __shared__ int s_fixup;                                  // balanced mode: segments of the tile to reduce here (0 = not the last)

  const int tid = threadIdx.x, lane = tid & 31;
  // the role as a warp-uniform value (a lane-0 broadcast): the consumers' wgmma run on paths the compiler knows do not
  // diverge inside a warp, and are not serialised
  const int warpgroup = __shfl_sync(0xffffffffu, tid / 128, 0);
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~static_cast<uintptr_t>(1023));
  unsigned char* wslot = base + STAGES * STAGE;                            // slots j = 0, 1: rows, the table (, the flag)
  int32_t* tab0 = reinterpret_cast<int32_t*>(base + STAGES * STAGE + SLOTS);   // [tap][row]: source row in x0, -1 = none
  int32_t* tab1 = tab0 + 9 * TC_BM;                                        // ... in x1
  // row-set scratch (producer only), per source: rank tables [tap][row], distinct rows, bitmap words, their rank bases
  unsigned char* sx = base + STAGES * STAGE + SLOTS + TC_TABLES;
  uint16_t* set_tab = reinterpret_cast<uint16_t*>(sx);
  int32_t* set_rows = reinterpret_cast<int32_t*>(sx + 2 * TC_WIN_TAB);
  uint32_t* set_bits = reinterpret_cast<uint32_t*>(set_rows + 2 * TC_SET_ROWS);
  int32_t* set_rank = reinterpret_cast<int32_t*>(set_bits + 2 * TC_PRODUCERS);
  int32_t* set_red = set_rank + 2 * TC_PRODUCERS;          // [0, 8): warp min / max, [8, 12): warp counts, [12, 16): per source staged, count
  uint64_t* full = reinterpret_cast<uint64_t*>(sx + SCRATCH);   // stage s holds its chunk
  uint64_t* empty = full + STAGES;                                                       // both consumers are done with s
  uint64_t* wfull = empty + STAGES;                        // window / row set: slot j holds its channel chunk's rows and table
  uint64_t* wempty = wfull + 2;                            // ... every consumer warp has read slot j for the last time

  const long long HW = static_cast<long long>(d.H) * d.W;
  const int total_px = static_cast<int>(static_cast<long long>(d.N) * HW);
  int rows = d.pixels ? *d.count : total_px;
  rows = __shfl_sync(0xffffffffu, min(rows, d.max_rows), 0);   // warp-uniform, and so is the whole work walk
  const int nch0 = (d.c0 + TC_BK - 1) / TC_BK, nch1 = (d.c1 + TC_BK - 1) / TC_BK;
  const int per_tap = nch0 + nch1;
  const int nchunks = d.taps * per_tap;
  const int n_tiles = (d.cout + BN - 1) / BN;
  const long long tiles = static_cast<long long>((rows + TC_BM - 1) / TC_BM) * n_tiles;
  const bool balanced = (splits == 0);
  const BalPlan plan = bal_plan(tiles, gridDim.x, nchunks);
  TcWalk walk(tiles, splits, nchunks, plan);
  TcItem it;

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full + s, WIN ? 1 : TC_PRODUCERS + 1);     // every producer thread's copies (gather) + the weight image's bytes
      mbar_init(empty + s, TC_CONSUMERS / 32);             // one arrival per consumer warp
    }
    if (WIN) {
      for (int j = 0; j < 2; ++j) {
        // two arrivals per producer thread: its copies (noinc) and a plain arrive that releases its table stores
        mbar_init(wfull + j, 2 * TC_PRODUCERS);
        mbar_init(wempty + j, TC_CONSUMERS / 32);
      }
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  if (WIN && tid < 2 * TC_A_LD) {                          // the zero row of each slot, never overwritten
    const int j = tid / TC_A_LD;
    reinterpret_cast<float*>(wslot + j * SLOT)[SLOT_ROWS * TC_A_LD + tid % TC_A_LD] = 0.f;
  }
  __syncthreads();

  if (warpgroup == 0) {
    // ================================================================ producer: tap tables, weight images, A rows
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(TC_PRODUCER_REGS));
    const int Hs = d.H >> d.shift0, Ws = d.W >> d.shift0;
    const bool aligned_rows = (d.taps == 1 && d.map0 == nullptr);
    // rows each source holds: a row index past them reads zeros (a 1x1 stage over its own rows may run past x0's end)
    const long long rows_x0 = (aligned_rows && d.rows0 > 0) ? d.rows0 : static_cast<long long>(d.N) * Hs * Ws;
    const long long rows_x1 = static_cast<long long>(d.N) * HW;
    const unsigned char* wimg = reinterpret_cast<const unsigned char*>(wtc) + (F16 ? 128 : 0);   // f16 images follow a 128-byte header
    uint32_t g = 0;                                        // chunks this CTA has issued: stage g % STAGES, use g / STAGES
    uint32_t wi = 0;                                       // window mode: windows issued: slot wi & 1, use wi >> 1
    while (walk.next(it)) {
      const int m0 = static_cast<int>(it.tile / n_tiles) * TC_BM;
      const int nt = static_cast<int>(it.tile % n_tiles);
      // The previous tile's copies have all been issued (they read the table when they are issued): one table is enough,
      // and it is built while the consumers still multiply the previous tile's last chunks.
      named_bar_sync(kProducerBar, TC_PRODUCERS);
      // thread t: tile row t; the output pixel is read and decoded once per row.  Taps in rounds of two: first every
      // tap's coordinates and its three look-ups (gate byte, source-0 index map, source-1 index map) are issued together -
      // the maps are read whether or not the gate turns out to be set, their indices are valid for every in-range
      // coordinate - then the results are combined.
      {
        const int r = tid;
        const int m = m0 + r;
        int n = 0, y = 0, x = 0;
        const bool live = m < rows;
        if (live) {
          const unsigned p = static_cast<unsigned>(d.pixels ? d.pixels[m] : m);     // < 2^31 (checked by the host): 32-bit divisions
          const unsigned hw = static_cast<unsigned>(HW);
          n = static_cast<int>(p / hw);
          const unsigned rem = p - static_cast<unsigned>(n) * hw;
          y = static_cast<int>(rem / static_cast<unsigned>(d.W));
          x = static_cast<int>(rem - static_cast<unsigned>(y) * static_cast<unsigned>(d.W));
        }
        constexpr int kTapsPerRound = 2;
#pragma unroll 1
        for (int t_lo = 0; t_lo < d.taps; t_lo += kTapsPerRound) {
          const int t_hi = min(d.taps, t_lo + kTapsPerRound);
          int qv[kTapsPerRound];                   // source-1 pixel of the tap, -1 = out of range / dead row
          uint8_t gv[kTapsPerRound];
          int32_t m0v[kTapsPerRound], m1v[kTapsPerRound];
#pragma unroll
          for (int k = 0; k < kTapsPerRound; ++k) {
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
                m1v[k] = d.map1 ? d.map1[q] : q;    // -1 (not in the compact skip list) = kNoRow
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
          for (int k = 0; k < kTapsPerRound; ++k) {
            const int tap = t_lo + k;
            if (tap < t_hi) {
              const bool ok = qv[k] >= 0 && gv[k] != 0;
              tab0[tap * TC_BM + r] = (ok && m0v[k] >= 0 && m0v[k] < rows_x0) ? m0v[k] : kNoRow;
              tab1[tap * TC_BM + r] = (ok && m1v[k] < rows_x1) ? m1v[k] : kNoRow;
            }
          }
        }
      }
      named_bar_sync(kProducerBar, TC_PRODUCERS);
      if constexpr (SET) {
        // Row-set mode: each source's distinct rows in ascending order and the rank table (see TC_SET_ROWS).  Thread t
        // owns bitmap word t and tile row t of the tables; the scratch is free again for the same reason the tap table is.
        const int warp = tid >> 5;
#pragma unroll 1
        for (int s = 0; s < (d.c1 > 0 ? 2 : 1); ++s) {
          const int32_t* tab = s ? tab1 : tab0;
          uint32_t* bits = set_bits + s * TC_PRODUCERS;
          int32_t* rank = set_rank + s * TC_PRODUCERS;
          int lo = 0x7fffffff, hi = -1;                    // the tile's row range in this source
#pragma unroll 1
          for (int t = 0; t < 9; ++t) {
            const int32_t a = tab[t * TC_BM + tid];
            if (a >= 0) { lo = min(lo, a); hi = max(hi, a); }
          }
          lo = __reduce_min_sync(0xffffffffu, lo);
          hi = __reduce_max_sync(0xffffffffu, hi);
          if (lane == 0) { set_red[2 * warp] = lo; set_red[2 * warp + 1] = hi; }
          bits[tid] = 0u;
          named_bar_sync(kProducerBar, TC_PRODUCERS);
#pragma unroll
          for (int k = 0; k < TC_PRODUCERS / 32; ++k) { lo = min(lo, set_red[2 * k]); hi = max(hi, set_red[2 * k + 1]); }
          const bool fits = hi < lo || hi - lo < TC_SET_SPAN;   // hi < lo: no live tap
          if (fits) {
#pragma unroll 1
            for (int t = 0; t < 9; ++t) {
              const int32_t a = tab[t * TC_BM + tid];
              if (a >= 0) atomicOr(bits + ((a - lo) >> 5), 1u << ((a - lo) & 31));
            }
          }
          named_bar_sync(kProducerBar, TC_PRODUCERS);
          const uint32_t w = bits[tid];
          int incl = __popc(w);                            // inclusive prefix of the words' popcounts
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
          }
          if (lane == 31) set_red[8 + warp] = incl;
          named_bar_sync(kProducerBar, TC_PRODUCERS);
          int r = incl - __popc(w), total = 0;
#pragma unroll
          for (int k = 0; k < TC_PRODUCERS / 32; ++k) {
            const int n = set_red[8 + k];
            total += n;
            if (k < warp) r += n;
          }
          const bool staged = fits && total <= TC_SET_ROWS;
          if (tid == 0) { set_red[12 + 2 * s] = staged; set_red[13 + 2 * s] = total; }
          if (staged) {
            rank[tid] = r;
            int32_t* rows_s = set_rows + s * TC_SET_ROWS;
            for (uint32_t m = w; m; m &= m - 1) rows_s[r++] = lo + 32 * tid + (__ffs(m) - 1);
          }
          named_bar_sync(kProducerBar, TC_PRODUCERS);
          if (staged) {
            uint16_t* st = set_tab + s * 9 * TC_BM;
#pragma unroll 1
            for (int t = 0; t < 9; ++t) {
              const int32_t a = tab[t * TC_BM + tid];
              int v = TC_SET_ROWS;
              if (a >= 0) {
                const int o = a - lo;
                v = rank[o >> 5] + __popc(bits[o >> 5] & ((1u << (o & 31)) - 1u));
              }
              st[t * TC_BM + tid] = static_cast<uint16_t>(v);
            }
          }
        }
      }

      // Chunk c of the tile into stage s: the weight image as it is (one bulk copy), and the implicit im2col - for every
      // tile row the 32-channel slice of its tap's source row (channel chunk outermost, taps innermost: the nine taps of
      // a chunk re-read (almost) the same rows while they are hot in L2).  No row / channels past C: zero fill.
      const unsigned char* wtile = wimg + static_cast<long long>(nt) * nchunks * B_IMG;
#pragma unroll 1
      for (int c = it.cb; c < it.ce; ++c, ++g) {
        const int s = static_cast<int>(g % STAGES);
        if (g >= STAGES) mbar_wait(empty + s, ((g / STAGES) - 1) & 1);
        unsigned char* st = base + s * STAGE;
        if (tid == 0) {
          mbar_arrive_expect_tx(full + s, B_IMG);
          bulk_copy_g2s(st, wtile + static_cast<long long>(c) * B_IMG, B_IMG, full + s);
        }
        const int taps = WIN ? 9 : d.taps;
        const int rr = c / taps;
        const int tap = c - rr * taps;
        const bool src1 = rr >= nch0;
        const int col = (src1 ? rr - nch0 : rr) * TC_BK;
        const float* x = src1 ? d.x1 : d.x0;
        const long long ld = src1 ? d.ld1 : d.ld0;
        const int csrc = src1 ? d.c1 : d.c0;
        if constexpr (WIN) {
          // A channel chunk's first step in this segment (a stream-K segment may start at any tap) loads its window or
          // row set into the next slot: the table, then the rows, zero filled as the gather does.  A row-set source
          // staged per tap loads a slot at every step: the tap's 128 gathered rows, identity table.
          const bool tap_slots = SET && !set_red[12 + 2 * src1];
          if (c != it.cb && tap != 0 && !tap_slots) continue;
          const int j = static_cast<int>(wi & 1);
          if (wi >= 2) mbar_wait(wempty + j, ((wi >> 1) - 1) & 1);
          float* sw = reinterpret_cast<float*>(wslot + j * SLOT);
          uint16_t* wt = reinterpret_cast<uint16_t*>(wslot + j * SLOT + SLOT_DATA);
          uint32_t* hdr = reinterpret_cast<uint32_t*>(wslot + j * SLOT + SLOT_DATA + TC_WIN_TAB);
          if constexpr (SET) {
            // slot row r holds source row rows_s[r] (-1: zeros): the distinct rows and their rank table, or the tap's
            // gathered rows and the identity
            const int32_t* rows_s = tab0 + (src1 * 9 + tap) * TC_BM;
            int n = TC_BM;
            if (tap_slots) {
              wt[tap * TC_BM + tid] = static_cast<uint16_t>(tid);
            } else {
              const uint16_t* stb = set_tab + src1 * 9 * TC_BM;
#pragma unroll 1
              for (int t = 0; t < 9; ++t) wt[t * TC_BM + tid] = stb[t * TC_BM + tid];
              rows_s = set_rows + src1 * TC_SET_ROWS;
              n = set_red[13 + 2 * src1];
            }
            if (tid == 0) { hdr[0] = tap_slots; hdr[1] = n; }
#pragma unroll 1
            for (int pc = tid; pc < n * 8; pc += TC_PRODUCERS) {
              const int r = pc >> 3, q = pc & 7;
              const int32_t srow = rows_s[r];
              const int cc = col + 4 * q;
              const int bytes = srow >= 0 ? min(16, max(0, (csrc - cc) * 4)) : 0;
              cp_async16(sw + r * TC_A_LD + 4 * q, bytes ? x + static_cast<long long>(srow) * ld + cc : x, bytes);
            }
          } else {
            const int32_t* tab = src1 ? tab1 : tab0;
            const int shift = src1 ? 0 : d.shift0;
            const int wb = win_base(m0, d.W, shift), wn = win_rows(d.W, shift);
            const long long nrows = src1 ? rows_x1 : rows_x0;
            if (tid == 0) hdr[1] = wn;
#pragma unroll
            for (int t = 0; t < 9; ++t) {
              const int32_t a = tab[t * TC_BM + tid];
              const int o = a - wb;
              wt[t * TC_BM + tid] = static_cast<uint16_t>(a != kNoRow && o >= 0 && o < wn ? o : TC_WIN_ROWS);
            }
#pragma unroll 1
            for (int pc = tid; pc < wn * 8; pc += TC_PRODUCERS) {
              const int r = pc >> 3, q = pc & 7;
              const long long srow = static_cast<long long>(wb) + r;
              const int cc = col + 4 * q;
              const int bytes = (srow >= 0 && srow < nrows) ? min(16, max(0, (csrc - cc) * 4)) : 0;
              cp_async16(sw + r * TC_A_LD + 4 * q, bytes ? x + srow * ld + cc : x, bytes);
            }
          }
          // cp.async's arrival tracks only its copies; the plain arrive (release) publishes this thread's table (and
          // header) stores to the consumers' wait (acquire)
          cp_async_mbar_arrive(wfull + j);
          mbar_arrive(wfull + j);
          ++wi;
          continue;
        }
        const int32_t* tab = (src1 ? tab1 : tab0) + tap * TC_BM;
        float* sa = reinterpret_cast<float*>(st + B_IMG);
#pragma unroll
        for (int i = 0; i < TC_BM * 8 / TC_PRODUCERS; ++i) {
          const int pc = tid + i * TC_PRODUCERS, r = pc >> 3, q = pc & 7;
          const int32_t srow = tab[r];
          const int cc = col + 4 * q;
          const int bytes = srow >= 0 ? min(16, max(0, (csrc - cc) * 4)) : 0;
          cp_async16(sa + r * TC_A_LD + 4 * q, bytes ? x + srow * ld + cc : x, bytes);
        }
        cp_async_mbar_arrive(full + s);
      }
    }
    asm volatile("cp.async.wait_all;\n" ::: "memory");
    return;
  }

  // ================================================================== consumers: multiply, epilogue, stream-K fix-up
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(TC_CONSUMER_REGS));
  const int ctid = tid - TC_PRODUCERS;

  // F16: operands are fed as fp16 pairs.  Activations are scaled by a power of two chosen from the sources' max |x| (device
  // scalars written by their producers: layout moves, earlier convolutions) so that max |x| s lies in [2^13, 2^14)
  // (f16_scale_exp) - no overflow, the low piece stays normal for everything within 2^-11 .. 1 of the maximum; weights
  // carry their own power-of-two scale in the packed image's header.  Both scales are undone exactly in the epilogue:
  // y = acc 2^-(e + e_w) + bias = fma(acc, out_scale, bias) with out_scale = 2^k2, k2 = -(e + e_w) clamped to the
  // float powers of two [2^-149, 2^127]; the rest, 2^k1, is applied to the sums first (out_pre), in a branch off the
  // per-element path.  For finite maxima e and e_w lie in [-114, 127], so k is in [-254, 228] and k1 in [-105, 101];
  // k1 < 0 needs the product of the two maxima below about 2^-121, k1 > 0 needs it above about 2^154: there the
  // largest terms x w leave fp32, and so does the exact result of any row that reads them.
  float ascale = 1.f, out_scale = 1.f, out_pre = 1.f;
  if (F16) {
    float amax = d.amax0 ? __ldg(d.amax0) : 0.f;
    if (d.c1 > 0 && d.amax1) amax = fmaxf(amax, __ldg(d.amax1));
    const int e = f16_scale_exp(amax);
    ascale = ldexpf(1.f, e);
    const int k = -(e + __ldg(reinterpret_cast<const int*>(wtc) + 2));   // header word 2: e_w, the weight scale's exponent
    const int k2 = max(-149, min(127, k));
    out_scale = ldexpf(1.f, k2);
    out_pre = ldexpf(1.f, k - k2);
  }

  // fragment ownership: consumer warpgroup wg, warp wq of it; rows row_a and row_a + 8 of the tile, columns 8j + 2 t4 + {0, 1}
  const int wg = ctid >> 7, wq = (ctid >> 5) & 3, t4 = lane & 3;
  const int row_a = wg * 64 + wq * 16 + (lane >> 2);
  const int row_l = wg * 64 + wq * 16 + (lane & 15);       // the row whose address the lane gives ldmatrix
  // rows / bias 8-byte aligned: the epilogue's pair form for the pairs inside cout
  const bool al_ok = (d.ldy % 2 == 0) && ((reinterpret_cast<uintptr_t>(d.y) & 7) == 0) &&
                     ((reinterpret_cast<uintptr_t>(d.bias) & 7) == 0);

  // A fragments of a chunk, two register sets: the next chunk's are read and split while the current one's MMAs run.
  // tf32: fa = hi, fb = lo; f16: fa = h1, fb = h2.
  constexpr int KS = F16 ? TC_BK / 16 : TC_BK / 8;          // k-steps per chunk
  uint32_t fa[2][KS][4], fb[2][KS][4];
  float acc[ACC];
  float dacc[ACC];                                         // the wgmma accumulators of the running epoch
#pragma unroll
  for (int j = 0; j < ACC; ++j) dacc[j] = 0.f;

  // Window and row-set modes: a segment's first chunk and every channel chunk's first tap start the next slot (slot
  // number & 1), and so does every step of a row-set source staged per tap (the flag word of the slot in use).
  uint32_t wnext = 0, wcur = 0;                            // slots this CTA has started; the slot of the chunk last loaded
  bool tap_slots = false;
  int seg_cb = 0;

  // wait for stage gi % STAGES to hold chunk gi (and in window / row-set mode, at a slot's first step, for its slot),
  // then read this thread's fragment elements (chunk i of the segment) into register set B
  auto load_frag = [&](auto B, uint32_t gi, int i) {
    constexpr int b = decltype(B)::value;
    const int s = static_cast<int>(gi % STAGES);
    mbar_wait(full + s, (gi / STAGES) & 1);
    const float* sa = reinterpret_cast<const float*>(base + s * STAGE + B_IMG);
    int pr0 = row_a * TC_A_LD, pr1 = (row_a + 8) * TC_A_LD;   // float offsets of this thread's two fragment rows
    if constexpr (WIN) {
      const int tap = (seg_cb + i) % 9;
      const bool start = i == 0 || tap == 0 || tap_slots;
      if (start) wcur = wnext++;
      const int j = static_cast<int>(wcur & 1);
      unsigned char* slot = wslot + j * SLOT;
      if (start) {
        mbar_wait(wfull + j, (wcur >> 1) & 1);
        [[maybe_unused]] const uint32_t* hdr = reinterpret_cast<const uint32_t*>(slot + SLOT_DATA + TC_WIN_TAB);
        if constexpr (SET) tap_slots = hdr[0] != 0u;
        if constexpr (F16) {
          // the slot's rows become fp16 pairs once, for every tap that reads them; both consumer warpgroups walk the
          // same chunks, so all 256 threads start every slot together
          split_slot_rows(slot, static_cast<int>(hdr[1]), ascale, ctid);
          named_bar_sync(kSplitBar, TC_CONSUMERS);
        }
      }
      const uint16_t* wt = reinterpret_cast<const uint16_t*>(slot + SLOT_DATA) + tap * TC_BM;
      if constexpr (F16) {
        // Fragment of k-step ks from the split rows: per piece one ldmatrix.x4 over the warp's 16 rows, lane l giving
        // the address of row l & 15 in channels 16 ks + 8 (l >> 4) .. + 7: h1 at byte 32 g of its group g, h2 at 32 g + 16
        const uint32_t pa = smem_u32(slot) + wt[row_l] * (TC_A_LD * 4) + (lane >> 4) * 32;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          ldmatrix_x4(fa[b][ks], pa + 64 * ks);
          ldmatrix_x4(fb[b][ks], pa + 64 * ks + 16);
        }
        return;
      }
      sa = reinterpret_cast<const float*>(slot);
      pr0 = wt[row_a] * TC_A_LD;
      pr1 = wt[row_a + 8] * TC_A_LD;
    }
    if (F16) {
      // Fragment of k-step ks: rows (r, r + 8) x channels 16 ks + 2 t4 + {0, 1}, + 8, split in registers
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 v = *reinterpret_cast<const float2*>(sa + ((e & 1) ? pr1 : pr0) + ks * 16 + 2 * t4 + (e >> 1) * 8);
          split_f16x2(v.x, v.y, ascale, fa[b][ks][e], fb[b][ks][e]);
        }
      }
    } else {
      // fragment of k-step ks: rows (r, r + 8) x channels 8 ks + t4, + 4; tf32 hi by truncation, exact remainder lo
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float v = sa[((e & 1) ? pr1 : pr0) + ks * 8 + t4 + (e >> 1) * 4];
          fa[b][ks][e] = __float_as_uint(v) & 0xFFFFE000u;
          fb[b][ks][e] = __float_as_uint(v - __uint_as_float(fa[b][ks][e]));
        }
      }
    }
  };
  auto fence_frag = [&](auto B) {                           // the set stays live and unmoved until its MMAs have retired
    constexpr int b = decltype(B)::value;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
      for (int e = 0; e < 4; ++e) { reg_fence(fa[b][ks][e]); reg_fence(fb[b][ks][e]); }
  };
  auto release = [&](uint32_t gi) {                          // this warp is done with the stage of chunk gi
    if (lane == 0) mbar_arrive(empty + gi % STAGES);
  };

  uint32_t g = 0;                                          // chunks this CTA has consumed
  while (walk.next(it)) {
    const int len = it.ce - it.cb;
    const int m0 = static_cast<int>(it.tile / n_tiles) * TC_BM;
    const int n0 = static_cast<int>(it.tile % n_tiles) * BN;
    const long long rem_t = it.rem_t;
    const int slab = it.slab;
    const bool whole = it.whole;
#pragma unroll
    for (int j = 0; j < ACC; ++j) acc[j] = 0.f;
    float out_max = 0.f;                                   // max |y| this thread stores in this tile (-> d.amax_out)

    // Chunk i of the segment from register set B: its MMAs are issued, then the previous chunk's group is waited for: its
    // stage goes back to the producer, its register set takes chunk i + 1's fragments.  The first MMA of an epoch
    // overwrites the accumulators.
    auto step = [&](auto B, int i) {
      constexpr int b = decltype(B)::value;
      const uint32_t gi = g + i;
      const uint64_t b0 = wgmma_desc_sw128(smem_u32(base + (gi % STAGES) * STAGE));
      const uint32_t keep = (i % kFlushChunks) != 0;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        if (F16) {
          // rows of the weight tile: [h1: 64 B | h2: 64 B]; a k-step is 16 channels = 32 B
          const uint64_t bh = b0 + static_cast<uint64_t>(2 * ks);
          const uint64_t bl = bh + 4u;
          Wgmma<BN, true>::mma(dacc, fb[b][ks], bh, ks == 0 ? keep : 1u);   // lo*hi
          Wgmma<BN, true>::mma(dacc, fa[b][ks], bl, 1u);                    // hi*lo
          Wgmma<BN, true>::mma(dacc, fa[b][ks], bh, 1u);                    // hi*hi
        } else {
          const uint64_t bh = b0 + static_cast<uint64_t>(2 * ks);
          const uint64_t bl = bh + static_cast<uint64_t>(TC_B_TILE >> 4);
          Wgmma<BN, false>::mma(dacc, fb[b][ks], bh, ks == 0 ? keep : 1u);  // lo*hi
          Wgmma<BN, false>::mma(dacc, fa[b][ks], bl, 1u);                   // hi*lo
          Wgmma<BN, false>::mma(dacc, fa[b][ks], bh, 1u);                   // hi*hi
        }
      }
      wgmma_commit();
      if constexpr (WIN) {
        // chunk i's fragments are in registers (its MMAs are issued): after the slot's last step in this segment, the
        // slot goes back to the producer
        if ((seg_cb + i) % 9 == 8 || i + 1 == len || tap_slots) {
          __syncwarp();
          if (lane == 0) mbar_arrive(wempty + (wcur & 1));
        }
      }
      wgmma_wait<1>();                                     // chunk i - 1 has retired
      fence_frag(Ic<1 - b>());
      if (i > 0) release(gi - 1);
      if (i + 1 < len) load_frag(Ic<1 - b>(), gi + 1, i + 1);
    };
    // Epochs of kFlushChunks chunks counted from the segment start (even: chunk i always uses register set i % 2).  The
    // accumulators are read only after an epoch's last group has retired, outside any branch, so the compiler keeps the
    // wgmma of the epoch asynchronous.
    seg_cb = it.cb;
    load_frag(Ic<0>(), g, 0);
#pragma unroll 1
    for (int e0 = 0; e0 < len; e0 += kFlushChunks) {
      const int e1 = min(len, e0 + kFlushChunks);
#pragma unroll 1
      for (int i = e0; i < e1; i += 2) {
        step(Ic<0>(), i);
        if (i + 1 < e1) step(Ic<1>(), i + 1);
      }
      wgmma_wait<0>();
      fence_frag(Ic<0>());
      fence_frag(Ic<1>());
#pragma unroll
      for (int j = 0; j < ACC; ++j) reg_fence(dacc[j]);
#pragma unroll
      for (int j = 0; j < ACC; ++j) acc[j] += dacc[j];
    }
    release(g + len - 1);
    g += len;

    if (F16 && whole && out_pre != 1.f) {
#pragma unroll
      for (int j = 0; j < ACC; ++j) acc[j] *= out_pre;
    }
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
              out_max = fmaxf(out_max, fmaxf(finite_abs(o.x), finite_abs(o.y)));
              *reinterpret_cast<float2*>(yr + co) = o;
            } else {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (co + e < d.cout) {
                  const float a = F16 ? __fmul_rn(e ? a1 : a0, out_scale) : (e ? a1 : a0);
                  const float o = actf(a + (d.bias ? __ldg(d.bias + co + e) : 0.f));
                  out_max = fmaxf(out_max, finite_abs(o));
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
      named_bar_sync(kConsumerBar, TC_CONSUMERS);
      if (ctid == 0) {
        const long long first = (rem_t * nchunks) / plan.U, last = ((rem_t + 1) * nchunks - 1) / plan.U;
        const int nseg = static_cast<int>(last - first + 1);
        unsigned* cnt = reinterpret_cast<unsigned*>(partial) + rem_t;
        const unsigned t = atomicAdd(cnt, 1u);
        s_fixup = (t == static_cast<unsigned>(nseg - 1)) ? nseg : 0;
        if (s_fixup) *cnt = 0u;
      }
      named_bar_sync(kConsumerBar, TC_CONSUMERS);
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
        static_assert(kQuads % (TC_CONSUMERS * kUnroll) == 0, "quads of a tile divide evenly");
        const int tile_rows = min(TC_BM, rows - m0);
        const float ap = d.act_param;
        // co is a multiple of 4: the quad load needs a 16-byte aligned bias (the ABI only asks for 4 bytes)
        const bool bias16 = (reinterpret_cast<uintptr_t>(d.bias) & 15) == 0;
        for (int qbase = ctid; qbase < kQuads; qbase += TC_CONSUMERS * kUnroll) {
          float4 v[kUnroll], bq[kUnroll];
          int r[kUnroll], co[kUnroll];
          bool live[kUnroll];
#pragma unroll
          for (int q = 0; q < kUnroll; ++q) {
            const int idx = qbase + q * TC_CONSUMERS;
            r[q] = idx / kQuadsPerRow;
            co[q] = n0 + 4 * (idx % kQuadsPerRow);
            live[q] = r[q] < tile_rows && co[q] < d.cout;
            bq[q] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (live[q] && d.bias) {
              if (bias16 && co[q] + 3 < d.cout) {
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
            const float4* ps = reinterpret_cast<const float4*>(pb + static_cast<long long>(sidx) * TC_BM * BN) + qbase;
#pragma unroll
            for (int q = 0; q < kUnroll; ++q) {
              if (live[q]) {
                const float4 pq = __ldcg(ps + q * TC_CONSUMERS);
                v[q].x += pq.x; v[q].y += pq.y; v[q].z += pq.z; v[q].w += pq.w;
              }
            }
          }
#pragma unroll
          for (int q = 0; q < kUnroll; ++q) {
            if (live[q]) {
              float4 o = v[q];
              if (F16) {
                if (out_pre != 1.f) { o.x *= out_pre; o.y *= out_pre; o.z *= out_pre; o.w *= out_pre; }
                o.x = __fadd_rn(__fmul_rn(o.x, out_scale), bq[q].x); o.y = __fadd_rn(__fmul_rn(o.y, out_scale), bq[q].y);
                o.z = __fadd_rn(__fmul_rn(o.z, out_scale), bq[q].z); o.w = __fadd_rn(__fmul_rn(o.w, out_scale), bq[q].w);
              }
              o.x = activate(o.x, d.act, ap); o.y = activate(o.y, d.act, ap);
              o.z = activate(o.z, d.act, ap); o.w = activate(o.w, d.act, ap);
              float* yq = d.y + static_cast<long long>(m0 + r[q]) * d.ldy + co[q];
              out_max = fmaxf(out_max, finite_abs(o.x));
              if (co[q] + 3 < d.cout) {                // balanced mode requires ldy % 4 == 0 and a 16-byte aligned y
                out_max = fmaxf(fmaxf(out_max, finite_abs(o.y)), fmaxf(finite_abs(o.z), finite_abs(o.w)));
                *reinterpret_cast<float4*>(yq) = o;
              } else {
                yq[0] = o.x;
                if (co[q] + 1 < d.cout) { yq[1] = o.y; out_max = fmaxf(out_max, finite_abs(o.y)); }
                if (co[q] + 2 < d.cout) { yq[2] = o.z; out_max = fmaxf(out_max, finite_abs(o.z)); }
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
  }
}

// Three kernels with their own names, so that a profile tells them apart; the window and row-set forms' names extend the
// gather form's, so a search for the tensor-core engine by name finds all three.  The window form runs the dense 3x3
// launches whose windows fit (tc_window_fits), the row-set form the other 3x3 launches that are not split
// (tc_rowset_takes), the gather form every other launch.  All three give the same bits.
template <int BN, bool F16>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_rows_tc_kernel(const wmd_conv_desc d, const float* __restrict__ wtc,
                                                                     const int splits, float* __restrict__ partial) {
  conv_rows_tc_body<BN, F16, kFeedGather>(d, wtc, splits, partial);
}
template <int BN, bool F16>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_rows_tc_kernel_window(const wmd_conv_desc d, const float* __restrict__ wtc,
                                                                         const int splits, float* __restrict__ partial) {
  conv_rows_tc_body<BN, F16, kFeedWindow>(d, wtc, splits, partial);
}
template <int BN, bool F16>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_rows_tc_kernel_rowset(const wmd_conv_desc d, const float* __restrict__ wtc,
                                                                         const int splits, float* __restrict__ partial) {
  conv_rows_tc_body<BN, F16, kFeedRowset>(d, wtc, splits, partial);
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
    const float hi = tf32_rna_finite(v);
    const float val = hilo == 0 ? hi : tf32_rna_finite(v - hi);
    const long long tile_base = ((static_cast<long long>(nt) * nchunks + c) * 2 + hilo) * tile_floats;
    const int piece = kk >> 2, within = kk & 3;
    out[tile_base + static_cast<long long>(n) * TC_BK + ((piece ^ (n & 7)) << 2) + within] = val;
  }
}

// y[m, co] = act(bias[co] + sum_s partial_s[m][co]) in a fixed order (deterministic).  splits >= 2: every tile has
// `splits` slabs laid out [slab][max_rows][ldy].  splits == 0 (balanced): only the remainder tiles have partial sums,
// laid out [remainder tile][slab][256][BN]; the number of segments of a tile follows from the same unit arithmetic the
// conv kernel used (grid = its CTA count); a remainder tile that one CTA covered entirely was finished there.
// amax_out (nullable) is raised to max |y| of the rows written here, as the conv kernel does for the rows it writes.
__global__ void tc_reduce_kernel(const float* __restrict__ partial, int splits, int grid, int BN, int nchunks,
                                 const float* __restrict__ bias, float* __restrict__ y, int ldy, int cout,
                                 const int32_t* __restrict__ count, int total_px, int max_rows, int act, float act_param,
                                 float* __restrict__ amax_out) {
  partial += kBalCounterBytes / 4;                   // the workspace starts with the balanced mode's arrival counters (kept zero)
  const int rows = min(count ? *count : total_px, max_rows);   // the conv kernel's row count
  float out_max = 0.f;                               // max |y| this thread writes (-> amax_out)
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
      out_max = fmaxf(out_max, finite_abs(v.x));
      if (co + 3 < cout) {
        out_max = fmaxf(fmaxf(out_max, finite_abs(v.y)), fmaxf(finite_abs(v.z), finite_abs(v.w)));
        *reinterpret_cast<float4*>(y + o) = v;
      } else {
        y[o] = v.x;
        if (co + 1 < cout) { y[o + 1] = v.y; out_max = fmaxf(out_max, finite_abs(v.y)); }
        if (co + 2 < cout) { y[o + 2] = v.z; out_max = fmaxf(out_max, finite_abs(v.z)); }
      }
    }
  }
  if (amax_out) {                                    // as in the conv kernel: order independent, most warps skip the atomic
    for (int o = 16; o > 0; o >>= 1) out_max = fmaxf(out_max, __shfl_xor_sync(0xffffffffu, out_max, o));
    if ((threadIdx.x & 31) == 0 && out_max > __ldcg(amax_out)) atomicMax(reinterpret_cast<unsigned*>(amax_out), __float_as_uint(out_max));
  }
}

// ---- fp16 weight images (precision = WMD_PREC_F16X3) -----------------------------------------------------------------
__global__ void absmax_kernel(const float* __restrict__ x, long long count, float* __restrict__ out) {
  float m = 0.f;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += step) m = fmaxf(m, finite_abs(__ldg(x + i)));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > __ldcg(out)) atomicMax(reinterpret_cast<unsigned*>(out), __float_as_uint(m));
}

// max |x| over the rows r of x (rows x cols, contiguous) with mask[r] != 0.  A warp takes 32 rows at a time: one
// coalesced read of their mask bytes, then the marked rows only, the lanes along each row (unmarked rows cost no traffic).
__global__ void absmax_rows_masked_kernel(const float* __restrict__ x, long long rows, int cols,
                                          const uint8_t* __restrict__ mask, float* __restrict__ out) {
  float m = 0.f;
  const int lane = threadIdx.x & 31;
  const long long groups = (rows + 31) / 32;
  const long long warps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long gi = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; gi < groups; gi += warps) {
    const long long r0 = gi * 32;
    unsigned marked = __ballot_sync(0xffffffffu, r0 + lane < rows && mask[r0 + lane] != 0);
    while (marked) {
      const int b = __ffs(marked) - 1;
      marked &= marked - 1;
      const float* row = x + (r0 + b) * cols;
      for (int c = lane; c < cols; c += 32) m = fmaxf(m, finite_abs(__ldg(row + c)));
    }
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0 && m > __ldcg(out)) atomicMax(reinterpret_cast<unsigned*>(out), __float_as_uint(m));
}

// header word 0 holds max |w| when this runs; it is replaced by 1 / s_w by the last block... no: by a second tiny kernel
// (finish_header) so that every pack thread reads the same maximum.
__global__ void pack_weight_tc16_kernel(const float* __restrict__ w, unsigned char* __restrict__ out, int Cout, int c0, int c1,
                                        int taps, int BN, long long total) {
  const float wmax = *reinterpret_cast<const float*>(out);        // header word 0: max |w| over finite w (absmax_kernel)
  const float sw = ldexpf(1.f, f16_scale_exp(wmax));
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
  const int e = f16_scale_exp(wmax);
  h[1] = wmax;
  h[0] = ldexpf(1.f, -e);                          // 1 / s_w (subnormal for e = 127)
  reinterpret_cast<int*>(out)[2] = e;              // e_w: what the conv kernel reads
}

static int tc_tile_n(int cout) { return cout >= 96 ? 128 : (cout >= 48 ? 64 : 32); }

static int g_reserved_sms = 0;     // SMs the persistent grid leaves free (for a collective's kernel on multi-GPU runs)

// Window mode (TC_WIN_ROWS) takes a launch when its rows are the dense grid, its taps read no index map or gate, its
// tiles are not split (whole tiles or balanced) and every source's window fits a slot.
static bool tc_window_fits(const wmd_conv_desc& d, int splits) {
  if (d.taps != 9 || d.pixels || d.map0 || d.map1 || d.gate || splits > 1 || d.W > TC_WIN_ROWS) return false;
  return win_rows(d.W, d.shift0) <= TC_WIN_ROWS && (d.c1 == 0 || win_rows(d.W, 0) <= TC_WIN_ROWS);
}
// Row-set mode (TC_SET_ROWS) takes the 3x3 launches that read through a pixel list, an index map or a gate, when their
// tiles are not split (whole tiles or balanced).  tf32 N = 128 keeps the gather form: beside the two row-set slots its
// ring holds only two 32 KB weight images, and the NYU decoder's sparse launches (all of that form) ran ~9 % slower so.
static bool tc_rowset_takes(const wmd_conv_desc& d, int splits) {
  if (d.precision == WMD_PREC_TF32X3 && tc_tile_n(d.cout) == 128) return false;
  return d.taps == 9 && (d.pixels || d.map0 || d.map1 || d.gate) && splits <= 1;
}

template <int BN, bool F16, int FEED>
static int launch_tc(const wmd_conv_desc& d, int splits, float* partial, cudaStream_t stream) {
  const size_t smem = FEED == kFeedGather ? TcCfg<BN, F16>::SMEM : TcWinCfg<BN, F16, FEED == kFeedRowset>::SMEM;
  auto kernel = [] {                               // only the form launched here is instantiated
    if constexpr (FEED == kFeedWindow) return conv_rows_tc_kernel_window<BN, F16>;
    else if constexpr (FEED == kFeedRowset) return conv_rows_tc_kernel_rowset<BN, F16>;
    else return conv_rows_tc_kernel<BN, F16>;
  }();
  static bool attr_done[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {   // outside the cache: set it on every launch
    int rc = record(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    if (rc != WMD_OK) return rc;
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  const long long tiles = static_cast<long long>(ceil_div(d.max_rows, TC_BM)) * ceil_div(d.cout, BN) * (splits > 0 ? splits : 1);
  const long long cap = sm_count() - g_reserved_sms > 1 ? sm_count() - g_reserved_sms : 1;
  const int grid = splits == 0 ? static_cast<int>(cap) : static_cast<int>(tiles < cap ? (tiles < 1 ? 1 : tiles) : cap);
  kernel<<<grid, TC_THREADS, smem, stream>>>(d, d.w, splits, partial);
  int rc = launched();
  if (rc != WMD_OK || splits <= 1) return rc;      // whole tiles, or balanced: the kernel's own fix-up finishes cut tiles
  const int nchunks = d.taps * ((d.c0 + TC_BK - 1) / TC_BK + (d.c1 + TC_BK - 1) / TC_BK);
  const long long all_tiles = static_cast<long long>(ceil_div(d.max_rows, TC_BM)) * ceil_div(d.cout, BN);
  const long long red_grid = all_tiles < 8 * cap ? all_tiles : 8 * cap;
  tc_reduce_kernel<<<static_cast<int>(red_grid < 1 ? 1 : red_grid), 256, 0, stream>>>(partial, splits, grid, BN, nchunks, d.bias, d.y, d.ldy, d.cout,
                                                              d.count, d.N * d.H * d.W, d.max_rows,
                                                              d.act, d.act_param, d.amax_out);
  return launched();
}
// The launch's feed form; tf32 N = 128 has no row-set build (tc_rowset_takes never picks it)
template <int BN, bool F16>
static int launch_feed(int feed, const wmd_conv_desc& d, int splits, float* partial, cudaStream_t stream) {
  if (feed == kFeedWindow) return launch_tc<BN, F16, kFeedWindow>(d, splits, partial, stream);
  if constexpr (F16 || BN != 128) {
    if (feed == kFeedRowset) return launch_tc<BN, F16, kFeedRowset>(d, splits, partial, stream);
  }
  return launch_tc<BN, F16, kFeedGather>(d, splits, partial, stream);
}

}  // namespace wmd

extern "C" int wmd_conv_tc_tile_n(int cout) { return wmd::tc_tile_n(cout); }

extern "C" int wmd_conv_tc_set_reserved_sms(int n) {
  const int was = wmd::g_reserved_sms;
  if (n >= 0) wmd::g_reserved_sms = n;
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

extern "C" int wmd_amax_rows_masked_f32(const float* x, long long rows, int cols, const uint8_t* mask, float* amax,
                                        wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(x && mask && amax, WMD_ERR_ARG);
  WMD_REQUIRE(rows >= 0 && cols > 0, WMD_ERR_SHAPE);
  if (rows == 0) return WMD_OK;
  absmax_rows_masked_kernel<<<stride_grid(rows, 256, 16), 256, 0, as_stream(stream)>>>(x, rows, cols, mask, amax);
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
  const int feed = tc_window_fits(d, splits) ? kFeedWindow : (tc_rowset_takes(d, splits) ? kFeedRowset : kFeedGather);
  switch (tc_tile_n(d.cout)) {
    case 128: return f16 ? launch_feed<128, true>(feed, d, splits, partial, st) : launch_feed<128, false>(feed, d, splits, partial, st);
    case 64: return f16 ? launch_feed<64, true>(feed, d, splits, partial, st) : launch_feed<64, false>(feed, d, splits, partial, st);
    default: return f16 ? launch_feed<32, true>(feed, d, splits, partial, st) : launch_feed<32, false>(feed, d, splits, partial, st);
  }
}
