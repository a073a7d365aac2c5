// Pillow's 8-bit resample arithmetic (libImaging/Resample.c), shared by KITTI's and NYUv2's input kernels: each pass
// accumulates 22-bit fixed-point taps from 1 << 21 and keeps clip(acc >> 22, 0, 255).
#pragma once

namespace wmd {

constexpr int kPrecisionBits = 22;

__device__ __forceinline__ int clip8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

__device__ __forceinline__ int acc8(long long acc) {   // Pillow's clip8 of a 22-bit fixed-point sum
  return clip8(static_cast<int>(acc >> kPrecisionBits));
}

}  // namespace wmd
