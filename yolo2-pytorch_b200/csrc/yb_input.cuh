// Input forms of the first-layer kernels, the layout boundary where the caller's image enters the network:
//   kInF32  fp32 NCHW [B,3,H,W], already transformed (what the reference's model takes);
//   kInU8   uint8 NHWC [B,H,W,3] times 1/255, torchvision's ToTensor (Darknet's frame path without a configured transform);
//   kInLut  uint8 NHWC [B,H,W,3] through a per-channel table lut[3][256] fp32, the configured ToTensor + Normalize chain compiled by
//           transform.TensorTransform.  Zero padding stays 0 in the transformed domain, as the reference's conv pads its normalised input.
// Only the load differs between the forms: every kernel computes on the same fp32 value with the same code after it.
#pragma once
#include <stdint.h>

namespace yb {

enum InputMode { kInF32 = 0, kInU8 = 1, kInLut = 2 };

// byte (img, iy, ix, c) of the uint8 NHWC frame batch x through the table (read through the L1: 3 KB, shared by every CTA of the SM; a copy
// in shared memory measured no faster for the stems)
__device__ __forceinline__ float lut_pixel(const void* x, const float* lut, long long img, int c, int iy, int ix, int height, int width) {
  return __ldg(lut + c * 256 + __ldg(reinterpret_cast<const uint8_t*>(x) + ((img * height + iy) * width + ix) * 3 + c));
}

}  // namespace yb
