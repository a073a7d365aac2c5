// Shared helpers for libwmd (sm_90a).  Host-side error plumbing + small device utilities.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "wmd.h"

namespace wmd {

// ---- host side -------------------------------------------------------------------------------
extern thread_local int g_last_cuda_error;
extern thread_local long long g_launches;

inline int record(cudaError_t e) {
  if (e == cudaSuccess) return WMD_OK;
  g_last_cuda_error = static_cast<int>(e);
  return WMD_ERR_CUDA;
}

// call right after a kernel launch
inline int launched() {
  ++g_launches;
  return record(cudaPeekAtLastError());
}

inline cudaStream_t as_stream(wmd_stream_t s) { return static_cast<cudaStream_t>(s); }

int sm_count();          // SMs of the current device (cached per device)

inline int ceil_div(long long a, long long b) { return static_cast<int>((a + b - 1) / b); }

// grid for a grid-stride elementwise kernel: enough CTAs to cover `work` items, capped at `waves` x SMs x per_sm
inline int stride_grid(long long work, int block, int per_sm = 8) {
  long long need = (work + block - 1) / block;
  long long cap = static_cast<long long>(sm_count()) * per_sm;
  if (need < 1) need = 1;
  return static_cast<int>(need < cap ? need : cap);
}

// ---- device side -----------------------------------------------------------------------------
__device__ __forceinline__ int reflect_idx(int q, int n) {   // ReflectionPad(1) semantics, n >= 2
  q = q < 0 ? -q : q;
  return q >= n ? 2 * (n - 1) - q : q;
}
__device__ __forceinline__ int clamp_idx(int q, int n) { return q < 0 ? 0 : (q >= n ? n - 1 : q); }

// maps tap coordinate q into [0,n) under pad_mode; returns false if the tap reads the zero padding
__device__ __forceinline__ bool pad_coord(int& q, int n, int pad_mode) {
  if (pad_mode == WMD_PAD_REFLECT) { q = reflect_idx(q, n); return true; }
  if (pad_mode == WMD_PAD_REPLICATE) { q = clamp_idx(q, n); return true; }
  return q >= 0 && q < n;
}

// e^v - 1 for v <= 0 in a dozen branch-free instructions (the library expm1f is ~80 with its range handling, and the
// tile epilogues apply it to every output element): Taylor series to v^7 above -0.25 (truncation < 4e-10), below that
// 2^(v log2 e) - 1 on the SFU, whose ~2e-7 absolute error sits on a result of magnitude >= 0.22.
__device__ __forceinline__ float expm1_nonpos(float v) {
  float t = fmaf(v, 1.f / 5040.f, 1.f / 720.f);
  t = fmaf(v, t, 1.f / 120.f);
  t = fmaf(v, t, 1.f / 24.f);
  t = fmaf(v, t, 1.f / 6.f);
  t = fmaf(v, t, 0.5f);
  const float near0 = fmaf(v * v, t, v);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(e) : "f"(v * 1.4426950408889634f));
  return v > -0.25f ? near0 : e - 1.f;
}

// |v| for finite v, 0 for +-Inf and NaN: the operand of every max |x| that sets an fp16-pair scale.  One non-finite value
// must not change the scale, and with it the bits, of every other value in the launch (an Inf max would leave the whole
// launch unscaled); the non-finite value itself still reaches the output through the split (wmd.h, precision).
__device__ __forceinline__ float finite_abs(float v) {
  const float a = fabsf(v);
  return a < INFINITY ? a : 0.f;
}

// v rounded to tf32 to nearest (cvt.rna), the hi piece of a round-to-nearest tf32 split.  A finite |v| >= (2 - 2^-11)
// 2^127 rounds up to Inf, and its remainder v - hi would be -Inf: there hi is v truncated to tf32 instead, which never
// overflows and leaves an exact finite remainder.  Every other v keeps cvt.rna's bits.
__device__ __forceinline__ float tf32_rna_finite(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(v));
  const float hi = __uint_as_float(r);
  return (fabsf(hi) == INFINITY && fabsf(v) < INFINITY) ? __uint_as_float(__float_as_uint(v) & 0xFFFFE000u) : hi;
}

__device__ __forceinline__ float activate(float v, int act, float p) {
  switch (act) {
    case WMD_ACT_ELU: return v > 0.f ? v : expm1_nonpos(v);
    case WMD_ACT_LRELU: return v > 0.f ? v : v * p;
    case WMD_ACT_SIGMOID: return 1.0f / (1.0f + expf(-v));
    default: return v;
  }
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, int src_bytes) {
  // 16-byte async copy global->shared, bytes beyond src_bytes are zero-filled (src_bytes in [0,16])
  unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gmem_src), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

}  // namespace wmd

#define WMD_REQUIRE(cond, code) \
  do {                          \
    if (!(cond)) return (code); \
  } while (0)
