// K1 / K2: one-level 2-D Haar synthesis (IDWT) and analysis (DWT), fp32, NCHW planes.
//
// HBM-bound streaming kernels: every coefficient is read once and every output written once
// (algorithmic bytes 32*N*C*H*W for the IDWT, +16*N*C*H*W with the fused disp plane), 128-bit
// coalesced accesses, no shared memory (no reuse to exploit), grid-stride over a grid sized in
// multiples of the SM count.  The arithmetic follows the dependency's separable evaluation order
// (oracle/haar.py) with explicit roundings (no FMA contraction) so results are bit-identical to it.
#include "common.cuh"

namespace wmd {

#define WMD_S 0.70710678118654752440f

struct Quad { float y00, y01, y10, y11; };

__device__ __forceinline__ Quad haar_synth(float ll, float lh, float hl, float hh) {
  // column pass (height): lo = g0*ll + g1*lh, hi = g0*hl + g1*hh ; then row pass (width)
  const float sll = __fmul_rn(WMD_S, ll), slh = __fmul_rn(WMD_S, lh);
  const float shl = __fmul_rn(WMD_S, hl), shh = __fmul_rn(WMD_S, hh);
  const float lo0 = __fadd_rn(sll, slh), lo1 = __fsub_rn(sll, slh);   // rows 2i, 2i+1 of the low band
  const float hi0 = __fadd_rn(shl, shh), hi1 = __fsub_rn(shl, shh);
  const float a0 = __fmul_rn(WMD_S, lo0), b0 = __fmul_rn(WMD_S, hi0);
  const float a1 = __fmul_rn(WMD_S, lo1), b1 = __fmul_rn(WMD_S, hi1);
  Quad q;
  q.y00 = __fadd_rn(a0, b0); q.y01 = __fsub_rn(a0, b0);
  q.y10 = __fadd_rn(a1, b1); q.y11 = __fsub_rn(a1, b1);
  return q;
}

__device__ __forceinline__ float disp_of(float v, float scale, int clamp01) {
  v = __fmul_rn(v, scale);
  return (clamp01 && v == v) ? fminf(fmaxf(v, 0.f), 1.f) : v;     // torch.clamp passes a NaN through; fmaxf would make it 0
}

// consumer epilogue of the reconstruction / its disparity plane (WMD_EPI_*, see wmd_head_idwt_desc)
struct EpiArgs {
  int mode;
  float a, b, lo, hi;
  float* out0;
  float* out1;
};
__device__ __forceinline__ void epi_store(const EpiArgs& e, long long o, float recon, float dispv) {
  if (e.mode == WMD_EPI_DISP_TO_DEPTH) {             // KITTI/layers.py:16-25
    const float sd = __fadd_rn(e.a, __fmul_rn(e.b, dispv));
    e.out0[o] = sd;
    if (e.out1) e.out1[o] = __fdiv_rn(1.f, sd);
  } else if (e.mode == WMD_EPI_DIV_CLAMP) {          // NYUv2/utils.py:219,229
    // torch on CUDA evaluates `t / python_scalar` as t * (1 / scalar) (one IEEE division of the scalar, then a multiply):
    // that is what the reference's `pred_y /= 100` computes where it runs (NYUv2/utils.py:219 after model.cuda())
    float v = __fmul_rn(recon, __fdiv_rn(1.f, e.a));
    if (e.b != 0.f && v == v) v = fminf(fmaxf(v, e.lo), e.hi);   // NaN stays NaN, as in torch.clamp
    e.out0[o] = v;
  }
}

// VEC: W even; one thread = two coefficient columns = a 2x4 output patch (two float4 stores per plane).
template <bool VEC>
__global__ void __launch_bounds__(256) idwt_haar_kernel(const float* __restrict__ ll, const float* __restrict__ hf,
                                                        float* __restrict__ out, float* __restrict__ disp,
                                                        float disp_scale, int clamp01, long long planes, int H, int W,
                                                        const EpiArgs epi) {
  const long long HW = static_cast<long long>(H) * W;
  const int Wv = VEC ? (W >> 1) : W;
  const long long total = planes * H * Wv;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += step) {
    const int jv = static_cast<int>(idx % Wv);
    const long long t = idx / Wv;
    const int i = static_cast<int>(t % H);
    const long long p = t / H;
    const long long cofs = static_cast<long long>(i) * W + (VEC ? 2 * jv : jv);
    const float* pl = ll + p * HW + cofs;
    const float* ph = hf + p * 3 * HW + cofs;
    const long long oofs = p * 4 * HW + static_cast<long long>(2 * i) * (2 * W) + (VEC ? 4 * jv : 2 * jv);
    if (VEC) {
      const float2 vll = __ldg(reinterpret_cast<const float2*>(pl));
      const float2 vlh = __ldg(reinterpret_cast<const float2*>(ph));
      const float2 vhl = __ldg(reinterpret_cast<const float2*>(ph + HW));
      const float2 vhh = __ldg(reinterpret_cast<const float2*>(ph + 2 * HW));
      const Quad q0 = haar_synth(vll.x, vlh.x, vhl.x, vhh.x);
      const Quad q1 = haar_synth(vll.y, vlh.y, vhl.y, vhh.y);
      const float4 r0 = make_float4(q0.y00, q0.y01, q1.y00, q1.y01);
      const float4 r1 = make_float4(q0.y10, q0.y11, q1.y10, q1.y11);
      *reinterpret_cast<float4*>(out + oofs) = r0;
      *reinterpret_cast<float4*>(out + oofs + 2 * W) = r1;
      if (disp) {
        *reinterpret_cast<float4*>(disp + oofs) =
            make_float4(disp_of(r0.x, disp_scale, clamp01), disp_of(r0.y, disp_scale, clamp01),
                        disp_of(r0.z, disp_scale, clamp01), disp_of(r0.w, disp_scale, clamp01));
        *reinterpret_cast<float4*>(disp + oofs + 2 * W) =
            make_float4(disp_of(r1.x, disp_scale, clamp01), disp_of(r1.y, disp_scale, clamp01),
                        disp_of(r1.z, disp_scale, clamp01), disp_of(r1.w, disp_scale, clamp01));
      }
      if (epi.mode) {
        const float t4[4] = {r0.x, r0.y, r0.z, r0.w}, b4[4] = {r1.x, r1.y, r1.z, r1.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          epi_store(epi, oofs + k, t4[k], disp_of(t4[k], disp_scale, clamp01));
          epi_store(epi, oofs + 2 * W + k, b4[k], disp_of(b4[k], disp_scale, clamp01));
        }
      }
    } else {
      const Quad q = haar_synth(__ldg(pl), __ldg(ph), __ldg(ph + HW), __ldg(ph + 2 * HW));
      out[oofs] = q.y00; out[oofs + 1] = q.y01;
      out[oofs + 2 * W] = q.y10; out[oofs + 2 * W + 1] = q.y11;
      if (disp) {
        disp[oofs] = disp_of(q.y00, disp_scale, clamp01);
        disp[oofs + 1] = disp_of(q.y01, disp_scale, clamp01);
        disp[oofs + 2 * W] = disp_of(q.y10, disp_scale, clamp01);
        disp[oofs + 2 * W + 1] = disp_of(q.y11, disp_scale, clamp01);
      }
      if (epi.mode) {
        epi_store(epi, oofs, q.y00, disp_of(q.y00, disp_scale, clamp01));
        epi_store(epi, oofs + 1, q.y01, disp_of(q.y01, disp_scale, clamp01));
        epi_store(epi, oofs + 2 * W, q.y10, disp_of(q.y10, disp_scale, clamp01));
        epi_store(epi, oofs + 2 * W + 1, q.y11, disp_of(q.y11, disp_scale, clamp01));
      }
    }
  }
}

// x (planes,H,W) with H,W even -> ll (planes,H/2,W/2), hf (planes,3,H/2,W/2).  One thread per output pixel.
__global__ void __launch_bounds__(256) dwt_haar_kernel(const float* __restrict__ x, float* __restrict__ ll,
                                                       float* __restrict__ hf, long long planes, int H, int W) {
  const int Ho = H >> 1, Wo = W >> 1;
  const long long HWo = static_cast<long long>(Ho) * Wo;
  const long long total = planes * HWo;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += step) {
    const int j = static_cast<int>(idx % Wo);
    const long long t = idx / Wo;
    const int i = static_cast<int>(t % Ho);
    const long long p = t / Ho;
    const float* px = x + p * static_cast<long long>(H) * W + static_cast<long long>(2 * i) * W + 2 * j;
    const float2 r0 = __ldg(reinterpret_cast<const float2*>(px));
    const float2 r1 = __ldg(reinterpret_cast<const float2*>(px + W));
    // row pass (width): lo = s*x0 + s*x1, hi = s*x0 - s*x1
    const float lo0 = __fadd_rn(__fmul_rn(WMD_S, r0.x), __fmul_rn(WMD_S, r0.y));
    const float hi0 = __fsub_rn(__fmul_rn(WMD_S, r0.x), __fmul_rn(WMD_S, r0.y));
    const float lo1 = __fadd_rn(__fmul_rn(WMD_S, r1.x), __fmul_rn(WMD_S, r1.y));
    const float hi1 = __fsub_rn(__fmul_rn(WMD_S, r1.x), __fmul_rn(WMD_S, r1.y));
    // column pass (height)
    const long long o = static_cast<long long>(i) * Wo + j;
    ll[p * HWo + o] = __fadd_rn(__fmul_rn(WMD_S, lo0), __fmul_rn(WMD_S, lo1));
    float* ph = hf + p * 3 * HWo + o;
    ph[0] = __fsub_rn(__fmul_rn(WMD_S, lo0), __fmul_rn(WMD_S, lo1));        // LH: low along width, high along height
    ph[HWo] = __fadd_rn(__fmul_rn(WMD_S, hi0), __fmul_rn(WMD_S, hi1));      // HL
    ph[2 * HWo] = __fsub_rn(__fmul_rn(WMD_S, hi0), __fmul_rn(WMD_S, hi1));  // HH
  }
}

// Fused IDWT + disparity epilogue + bilinear resize to the full-resolution plane (the consumer of ("disp", s) in
// KITTI/trainer.py:338-339 and NYUv2/utils.py:223-227).  The upsampled plane is produced straight from the
// coefficients: a CTA owns a 32 x 128 tile of the FULL-resolution output, synthesises the (tile/f + 2)^2 patch of
// disp it interpolates from into shared memory (each source pixel = one quadrant of one Haar butterfly, coefficient
// reads are L1/L2 hits shared by the four quadrants), then every thread blends its outputs.  The disp plane itself
// is never read back from HBM: 16*H*W coefficient bytes in, 4*Hf*Wf bytes out.
constexpr int kBT_H = 32, kBT_W = 128;
constexpr int kBS_MAX = 2048;   // floats of shared source patch: (32/f + 4) * (128/f + 4) fits for f >= ~1.6 per axis

__device__ __forceinline__ float src_index(float scale, int dst, bool align_corners) {
  if (align_corners) return scale * static_cast<float>(dst);
  const float s = scale * (static_cast<float>(dst) + 0.5f) - 0.5f;
  return s < 0.f ? 0.f : s;
}

__global__ void __launch_bounds__(256) idwt_bilinear_kernel(const float* __restrict__ ll, const float* __restrict__ hf,
                                                            float* __restrict__ full, float disp_scale, int clamp01,
                                                            int H, int W, int Hf, int Wf, float sy, float sx,
                                                            int align_corners) {
  __shared__ float patch[kBS_MAX];
  const long long plane = blockIdx.z;
  const int Y0 = blockIdx.y * kBT_H, X0 = blockIdx.x * kBT_W;
  const int Hs = 2 * H, Ws = 2 * W;                       // source (disp) plane
  const int Y1 = min(Y0 + kBT_H, Hf) - 1, X1 = min(X0 + kBT_W, Wf) - 1;
  // source rows / cols this tile interpolates from
  const int ys0 = static_cast<int>(src_index(sy, Y0, align_corners));
  const int ys1 = min(static_cast<int>(src_index(sy, Y1, align_corners)) + 1, Hs - 1);
  const int xs0 = static_cast<int>(src_index(sx, X0, align_corners));
  const int xs1 = min(static_cast<int>(src_index(sx, X1, align_corners)) + 1, Ws - 1);
  const int ph = ys1 - ys0 + 1, pw = xs1 - xs0 + 1;
  const long long HW = static_cast<long long>(H) * W;
  const float* pl = ll + plane * HW;
  const float* phf = hf + plane * 3 * HW;
  for (int e = threadIdx.x; e < ph * pw; e += blockDim.x) {
    const int y = ys0 + e / pw, x = xs0 + e % pw;
    const long long o = static_cast<long long>(y >> 1) * W + (x >> 1);
    const Quad q = haar_synth(__ldg(pl + o), __ldg(phf + o), __ldg(phf + HW + o), __ldg(phf + 2 * HW + o));
    const float v = (y & 1) ? ((x & 1) ? q.y11 : q.y10) : ((x & 1) ? q.y01 : q.y00);
    patch[e] = disp_of(v, disp_scale, clamp01);
  }
  __syncthreads();
  float* out = full + plane * static_cast<long long>(Hf) * Wf;
  for (int e = threadIdx.x; e < kBT_H * kBT_W; e += blockDim.x) {
    const int Y = Y0 + e / kBT_W, X = X0 + e % kBT_W;
    if (Y >= Hf || X >= Wf) continue;
    const float fy = src_index(sy, Y, align_corners), fx = src_index(sx, X, align_corners);
    const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
    const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
    const float ly = fy - static_cast<float>(y0), lx = fx - static_cast<float>(x0);
    const float* r0 = patch + (y0 - ys0) * pw - xs0;
    const float* r1 = patch + (y1 - ys0) * pw - xs0;
    out[static_cast<long long>(Y) * Wf + X] =
        (1.f - ly) * ((1.f - lx) * r0[x0] + lx * r0[x1]) + ly * ((1.f - lx) * r1[x0] + lx * r1[x1]);
  }
}

}  // namespace wmd

extern "C" int wmd_idwt_bilinear_f32(const float* ll, const float* hf, float* full, float disp_scale, int clamp01,
                                     int full_h, int full_w, int align_corners, int N, int C, int H, int W,
                                     wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(ll && hf && full, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && C > 0 && H > 0 && W > 0 && full_h > 0 && full_w > 0, WMD_ERR_SHAPE);
  const long long planes = static_cast<long long>(N) * C;
  if (planes == 0) return WMD_OK;
  WMD_REQUIRE(planes <= 65535, WMD_ERR_SHAPE);
  const int Hs = 2 * H, Ws = 2 * W;
  // PyTorch's area_pixel_compute_scale: in/out, or (in-1)/(out-1) with align_corners
  const float sy = align_corners ? (full_h > 1 ? static_cast<float>(Hs - 1) / static_cast<float>(full_h - 1) : 0.f)
                                 : static_cast<float>(Hs) / static_cast<float>(full_h);
  const float sx = align_corners ? (full_w > 1 ? static_cast<float>(Ws - 1) / static_cast<float>(full_w - 1) : 0.f)
                                 : static_cast<float>(Ws) / static_cast<float>(full_w);
  // shared patch must hold the tile's source footprint (upsampling by ~1.6x or more only)
  const long long need = (static_cast<long long>(kBT_H * sy) + 4) * (static_cast<long long>(kBT_W * sx) + 4);
  WMD_REQUIRE(need <= kBS_MAX, WMD_ERR_UNSUPPORTED);
  dim3 grid(ceil_div(full_w, kBT_W), ceil_div(full_h, kBT_H), static_cast<unsigned>(planes));
  idwt_bilinear_kernel<<<grid, 256, 0, as_stream(stream)>>>(ll, hf, full, disp_scale, clamp01, H, W, full_h, full_w, sy, sx,
                                                          align_corners);
  return launched();
}

static int launch_idwt(const float* ll, const float* hf, float* out, float* disp, float disp_scale, int clamp01, int N,
                       int C, int H, int W, const wmd::EpiArgs& epi, wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(ll && hf && out, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && C > 0 && H > 0 && W > 0, WMD_ERR_SHAPE);
  const long long planes = static_cast<long long>(N) * C;
  if (planes == 0) return WMD_OK;
  const bool vec = (W % 2) == 0;
  const long long work = planes * H * (vec ? W / 2 : W);
  const int grid = stride_grid(work, 256);
  if (vec)
    idwt_haar_kernel<true><<<grid, 256, 0, as_stream(stream)>>>(ll, hf, out, disp, disp_scale, clamp01, planes, H, W, epi);
  else
    idwt_haar_kernel<false><<<grid, 256, 0, as_stream(stream)>>>(ll, hf, out, disp, disp_scale, clamp01, planes, H, W, epi);
  return launched();
}

extern "C" int wmd_idwt_haar_f32(const float* ll, const float* hf, float* out, float* disp, float disp_scale,
                                 int clamp01, int N, int C, int H, int W, wmd_stream_t stream) {
  const wmd::EpiArgs none = {WMD_EPI_NONE, 0.f, 0.f, 0.f, 0.f, nullptr, nullptr};
  return launch_idwt(ll, hf, out, disp, disp_scale, clamp01, N, C, H, W, none, stream);
}

extern "C" int wmd_idwt_haar_epi_f32(const float* ll, const float* hf, float* out, float* disp, float disp_scale,
                                     int clamp01, int epi_mode, float epi_a, float epi_b, float epi_lo, float epi_hi,
                                     float* epi_out0, float* epi_out1, int N, int C, int H, int W, wmd_stream_t stream) {
  WMD_REQUIRE(epi_mode >= WMD_EPI_NONE && epi_mode <= WMD_EPI_DIV_CLAMP, WMD_ERR_ARG);
  WMD_REQUIRE(epi_mode == WMD_EPI_NONE || epi_out0 != nullptr, WMD_ERR_ARG);
  const wmd::EpiArgs epi = {epi_mode, epi_a, epi_b, epi_lo, epi_hi, epi_out0, epi_out1};
  return launch_idwt(ll, hf, out, disp, disp_scale, clamp01, N, C, H, W, epi, stream);
}

extern "C" int wmd_dwt_haar_f32(const float* x, float* ll, float* hf, int N, int C, int H, int W,
                                wmd_stream_t stream) {
  using namespace wmd;
  WMD_REQUIRE(x && ll && hf, WMD_ERR_ARG);
  WMD_REQUIRE(N >= 0 && C > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, WMD_ERR_SHAPE);
  const long long planes = static_cast<long long>(N) * C;
  if (planes == 0) return WMD_OK;
  const long long work = planes * (H / 2) * (W / 2);
  dwt_haar_kernel<<<stride_grid(work, 256), 256, 0, as_stream(stream)>>>(x, ll, hf, planes, H, W);
  return launched();
}
