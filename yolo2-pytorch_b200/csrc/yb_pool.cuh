// nn.MaxPool2d(kernel_size=3, stride=2, padding=1) window on fp16 NHWC, shared by the ResNet pool (resnet_ops.cu) and the DenseNet stem
// pool that writes into a channel slice of a wider buffer (densenet_ops.cu).  A window holding a NaN gives NaN (__hmax2_nan), as torch's
// max_pool2d does and as the backward kernels' winner rule (a NaN replaces the running maximum) assumes.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace yb {

__device__ __forceinline__ uint4 hmax8_(uint4 a, uint4 b) {
  uint4 r;
  const __half2* pa = reinterpret_cast<const __half2*>(&a);
  const __half2* pb = reinterpret_cast<const __half2*>(&b);
  __half2* pr = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) pr[i] = __hmax2_nan(pa[i], pb[i]);
  return r;
}

// max over the in-range pixels of rows 2py-1..2py+1, columns 2px-1..2px+1 of image img, channels [8 cg, 8 cg + 8)
__device__ __forceinline__ uint4 maxpool3x3_s2_window(const __half* __restrict__ x, long long img, int py, int px, int cg, int height, int width,
                                                      int channels) {
  bool any = false;
  uint4 m = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int iy = 2 * py - 1 + r;
    if (iy < 0 || iy >= height) continue;
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int ix = 2 * px - 1 + s;
      if (ix < 0 || ix >= width) continue;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + ((img * height + iy) * width + ix) * channels + cg * 8));
      m = any ? hmax8_(m, v) : v;
      any = true;
    }
  }
  return m;
}

}  // namespace yb
