// DenseNet plugin kernels (model/densenet.py of the reference, torchvision's _Transition / features.pool0), inference.
//   bn_relu_avgpool2x2  a transition's norm -> relu -> AvgPool2d(2), with the pooling moved in front of its 1x1 conv: pooling and a
//                       1x1 conv commute in exact arithmetic, and pooling first cuts that conv's work 4x.  The rounding differs from the
//                       reference's order (conv on the full-resolution activation, then pool) by fp32 summation order only.
//   maxpool3x3_s2_ld    nn.MaxPool2d(3, 2, 1) (features.pool0) writing into a channel slice of a wider buffer: the stem's pool lands
//                       directly in channels [0, 64) of the first dense block's buffer, so no concatenation copy follows.
// The dense layers' convs are yb_conv1x1_preact_fwd (norm1 + relu1 + conv1) and yb_conv_bn_act_fwd (conv2); the stem is the
// ResNet stem kernel.
#include "yb_common.h"
#include "yb_pool.cuh"
#include <cuda_fp16.h>
#include <stdint.h>

namespace yb {

// y[b, oy, ox, c] = fp16(((r(2oy, 2ox) + r(2oy, 2ox+1)) + (r(2oy+1, 2ox) + r(2oy+1, 2ox+1))) * 0.25), r = max(fmaf(scale[c], x, shift[c]), 0)
// in fp32.  One thread per output pixel and 8 channels.
__global__ void bn_relu_avgpool2x2_kernel(const __half* __restrict__ x, int x_ld, const float* __restrict__ scale, const float* __restrict__ shift,
                                          __half* __restrict__ y, int batch, int height, int width, int channels) {
  const int c8 = channels >> 3;
  const int oh = height >> 1, ow = width >> 1;
  const long long total = static_cast<long long>(batch) * oh * ow * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int px = static_cast<int>(t % ow); t /= ow;
  const int py = static_cast<int>(t % oh);
  const long long img = t / oh;
  float sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { sc[e] = __ldg(scale + cg * 8 + e); sh[e] = __ldg(shift + cg * 8 + e); }
  float r[4][8];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const long long pix = (img * height + 2 * py + (q >> 1)) * width + 2 * px + (q & 1);
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + pix * x_ld + cg * 8));
    const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
    for (int e = 0; e < 8; ++e) r[q][e] = fmaxf(__fmaf_rn(sc[e], __half2float(hv[e]), sh[e]), 0.f);
  }
  uint4 out;
  __half2* ho = reinterpret_cast<__half2*>(&out);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float a = ((r[0][2 * e] + r[1][2 * e]) + (r[2][2 * e] + r[3][2 * e])) * 0.25f;
    const float b = ((r[0][2 * e + 1] + r[1][2 * e + 1]) + (r[2][2 * e + 1] + r[3][2 * e + 1])) * 0.25f;
    ho[e] = __floats2half2_rn(a, b);
  }
  reinterpret_cast<uint4*>(y)[idx] = out;
}

int bn_relu_avgpool2x2(const void* x, int x_ld, const float* scale, const float* shift, void* y, int batch, int height, int width, int channels,
                       cudaStream_t stream) {
  YB_REQUIRE(x && scale && shift && y && batch > 0 && height > 1 && width > 1, "bn_relu_avgpool2x2: bad argument");
  YB_REQUIRE(height % 2 == 0 && width % 2 == 0, "bn_relu_avgpool2x2: H=%d, W=%d must be even", height, width);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "bn_relu_avgpool2x2: x / y must be 16B aligned");
  YB_REQUIRE(channels % 8 == 0 && x_ld % 8 == 0 && x_ld >= channels, "bn_relu_avgpool2x2: channels=%d, x_ld=%d (multiples of 8, x_ld >= channels)",
             channels, x_ld);
  const long long total = static_cast<long long>(batch) * (height / 2) * (width / 2) * (channels / 8);
  bn_relu_avgpool2x2_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x), x_ld, scale, shift,
                                                                                           reinterpret_cast<__half*>(y), batch, height, width, channels);
  return check_launch("bn_relu_avgpool2x2_kernel");
}

// nn.MaxPool2d(kernel_size=3, stride=2, padding=1) on x [B,H,W,C] into channels [y_ch_off, y_ch_off + C) of y [B,(H+1)/2,(W+1)/2,y_ld]
__global__ void maxpool3x3_s2_ld_kernel(const __half* __restrict__ x, __half* __restrict__ y, int y_ld, int y_ch_off, int batch, int height,
                                        int width, int channels) {
  const int c8 = channels >> 3;
  const int oh = (height + 1) / 2, ow = (width + 1) / 2;
  const long long total = static_cast<long long>(batch) * oh * ow * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  const long long opix = idx / c8;
  const int px = static_cast<int>(opix % ow);
  const long long t = opix / ow;
  const int py = static_cast<int>(t % oh);
  const long long img = t / oh;
  const uint4 m = maxpool3x3_s2_window(x, img, py, px, cg, height, width, channels);
  *reinterpret_cast<uint4*>(y + opix * y_ld + y_ch_off + cg * 8) = m;
}

int maxpool3x3_s2_ld(const void* x, void* y, int y_ld, int y_ch_off, int batch, int height, int width, int channels, cudaStream_t stream) {
  YB_REQUIRE(x && y && batch > 0 && height > 0 && width > 0 && channels % 8 == 0, "maxpool3x3_s2_ld: bad argument");
  YB_REQUIRE(y_ld % 8 == 0 && y_ch_off % 8 == 0 && y_ch_off >= 0 && y_ch_off + channels <= y_ld,
             "maxpool3x3_s2_ld: channels [%d, %d) do not fit y_ld=%d (offsets multiples of 8)", y_ch_off, y_ch_off + channels, y_ld);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "maxpool3x3_s2_ld: x / y must be 16B aligned");
  const long long total = static_cast<long long>(batch) * ((height + 1) / 2) * ((width + 1) / 2) * (channels / 8);
  maxpool3x3_s2_ld_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y),
                                                                                         y_ld, y_ch_off, batch, height, width, channels);
  return check_launch("maxpool3x3_s2_ld_kernel");
}

}  // namespace yb
