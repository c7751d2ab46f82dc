// Inception-v3 and Inception-v4 plugin kernels (model/inception3.py of the reference over torchvision's BasicConv2d / InceptionA-E, and
// model/inception4.py), inference.
//   pack_weight_khw       fp32 OIHW [Cout][Cin][kh][kw] -> fp16 [cout_pad][kh][kw][cin_pad], zeros in the padding: the B operand of the
//                         general-geometry conv (yb_conv2d_bn_act_fwd), with Cout / Cin rounded up to what the tensor-core conv needs
//                         (Inception's 80- and 48-channel layers run as 96 / 64 channels whose extra filters and inputs are zero).
//   maxpool3x3_s2_valid   F.max_pool2d(x, 3, stride=2) (pad 0, floor) into a channel slice of a wider buffer: the pool branch of
//                         Mixed_6a / Mixed_7a lands directly in its block's concatenation buffer.
//   avgpool3x3_s1         F.avg_pool2d(x, 3, stride=1, padding=1) with count_include_pad=True (torchvision's Inception blocks): the
//                         divisor is 9 at every pixel, borders included.  The branch's 1x1 conv then runs on the pooled tensor.
//   avgpool3x3_s1_excl    nn.AvgPool2d(3, stride=1, padding=1, count_include_pad=False) (the branch3 pools of model/inception4.py's
//                         Inception_A / B / C): the divisor is the number of in-range taps, 4 in a corner, 6 on an edge, 9 inside.
//                         Same kernel as avgpool3x3_s1 with the divisor chosen by a template parameter, so interior pixels are
//                         bit-identical between the two.
// The first conv (3 -> 32, 3x3, stride 2, pad 0) is mb_conv0_kernel<0> (mobilenet_ops.cu); every other conv is the implicit GEMM.
#include "yb_common.h"
#include "yb_pool.cuh"
#include <cuda_fp16.h>
#include <stdint.h>

namespace yb {

__global__ void pack_weight_khw_kernel(const float* __restrict__ w, __half* __restrict__ out, int cout, int cin, int kh, int kw, int cout_pad,
                                       int cin_pad) {
  const int taps = kh * kw;
  const long long total = static_cast<long long>(cout_pad) * taps * cin_pad;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ci = static_cast<int>(idx % cin_pad);
  const long long t = idx / cin_pad;
  const int tap = static_cast<int>(t % taps);
  const int co = static_cast<int>(t / taps);
  const float v = (co < cout && ci < cin) ? __ldg(w + (static_cast<long long>(co) * cin + ci) * taps + tap) : 0.f;
  out[idx] = __float2half_rn(v);
}

int pack_weight_khw(const float* w, void* out, int cout, int cin, int kh, int kw, int cout_pad, int cin_pad, cudaStream_t stream) {
  YB_REQUIRE(w && out && cout > 0 && cin > 0 && kh >= 1 && kh <= 7 && kw >= 1 && kw <= 7 && cout_pad >= cout && cin_pad >= cin,
             "pack_weight_khw: bad argument (cout %d, cin %d, kernel %d x %d, padded to %d x %d)", cout, cin, kh, kw, cout_pad, cin_pad);
  const long long total = static_cast<long long>(cout_pad) * kh * kw * cin_pad;
  pack_weight_khw_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(w, reinterpret_cast<__half*>(out), cout, cin, kh, kw,
                                                                                        cout_pad, cin_pad);
  return check_launch("pack_weight_khw_kernel");
}

// y[b, oy, ox, y_ch_off + c] = max over rows 2oy..2oy+2, columns 2ox..2ox+2 of x[b, :, :, c]; one thread per output pixel and 8 channels
__global__ void maxpool3x3_s2_valid_kernel(const __half* __restrict__ x, __half* __restrict__ y, int y_ld, int y_ch_off, int batch, int height,
                                           int width, int channels) {
  const int c8 = channels >> 3;
  const int oh = (height - 3) / 2 + 1, ow = (width - 3) / 2 + 1;
  const long long total = static_cast<long long>(batch) * oh * ow * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  const long long opix = idx / c8;
  const int px = static_cast<int>(opix % ow);
  const long long t = opix / ow;
  const int py = static_cast<int>(t % oh);
  const long long img = t / oh;
  uint4 m = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + ((img * height + 2 * py + r) * width + 2 * px + s) * channels + cg * 8));
      m = (r | s) ? hmax8_(m, v) : v;
    }
  *reinterpret_cast<uint4*>(y + opix * y_ld + y_ch_off + cg * 8) = m;
}

int maxpool3x3_s2_valid(const void* x, void* y, int y_ld, int y_ch_off, int batch, int height, int width, int channels, cudaStream_t stream) {
  YB_REQUIRE(x && y && batch > 0 && height >= 3 && width >= 3 && channels > 0 && channels % 8 == 0,
             "maxpool3x3_s2_valid: bad argument (H, W >= 3, C a multiple of 8)");
  YB_REQUIRE(y_ld % 8 == 0 && y_ch_off % 8 == 0 && y_ch_off >= 0 && y_ch_off + channels <= y_ld,
             "maxpool3x3_s2_valid: channels [%d, %d) do not fit y_ld=%d (offsets multiples of 8)", y_ch_off, y_ch_off + channels, y_ld);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "maxpool3x3_s2_valid: x / y must be 16B aligned");
  const long long total = static_cast<long long>(batch) * ((height - 3) / 2 + 1) * ((width - 3) / 2 + 1) * (channels / 8);
  maxpool3x3_s2_valid_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x),
                                                                                            reinterpret_cast<__half*>(y), y_ld, y_ch_off, batch,
                                                                                            height, width, channels);
  return check_launch("maxpool3x3_s2_valid_kernel");
}

// y[b, oy, ox, c] = fp16((sum of the in-range pixels of rows oy-1..oy+1, columns ox-1..ox+1 in fp32, row-major order) / n), one division
// rounded to nearest; n = 9 (kExclPad false: count_include_pad) or the number of in-range pixels (kExclPad true)
template <bool kExclPad>
__global__ void avgpool3x3_s1_kernel(const __half* __restrict__ x, __half* __restrict__ y, int batch, int height, int width, int channels) {
  const int c8 = channels >> 3;
  const long long total = static_cast<long long>(batch) * height * width * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  const long long pix = idx / c8;
  const int px = static_cast<int>(pix % width);
  const long long t = pix / width;
  const int py = static_cast<int>(t % height);
  const long long img = t / height;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
  for (int r = -1; r <= 1; ++r) {
    const int iy = py + r;
    if (iy < 0 || iy >= height) continue;
#pragma unroll
    for (int s = -1; s <= 1; ++s) {
      const int ix = px + s;
      if (ix < 0 || ix >= width) continue;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + ((img * height + iy) * width + ix) * channels + cg * 8));
      const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += __half2float(hv[e]);
    }
  }
  float n = 9.f;
  if (kExclPad) {
    const int rows = 3 - (py == 0) - (py == height - 1), cols = 3 - (px == 0) - (px == width - 1);
    n = static_cast<float>(rows * cols);
  }
  uint4 out;
  __half2* ho = reinterpret_cast<__half2*>(&out);
#pragma unroll
  for (int e = 0; e < 4; ++e) ho[e] = __floats2half2_rn(__fdiv_rn(acc[2 * e], n), __fdiv_rn(acc[2 * e + 1], n));
  reinterpret_cast<uint4*>(y)[idx] = out;
}

template <bool kExclPad>
static int avgpool3x3_s1_launch(const void* x, void* y, int batch, int height, int width, int channels, cudaStream_t stream, const char* name) {
  YB_REQUIRE(x && y && batch > 0 && height > 0 && width > 0 && channels > 0 && channels % 8 == 0, "%s: bad argument (C a multiple of 8)", name);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "%s: x / y must be 16B aligned", name);
  const long long total = static_cast<long long>(batch) * height * width * (channels / 8);
  avgpool3x3_s1_kernel<kExclPad><<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x),
                                                                                                 reinterpret_cast<__half*>(y), batch, height,
                                                                                                 width, channels);
  return check_launch(kExclPad ? "avgpool3x3_s1_kernel<excl>" : "avgpool3x3_s1_kernel");
}

int avgpool3x3_s1(const void* x, void* y, int batch, int height, int width, int channels, cudaStream_t stream) {
  return avgpool3x3_s1_launch<false>(x, y, batch, height, width, channels, stream, "avgpool3x3_s1");
}

int avgpool3x3_s1_excl(const void* x, void* y, int batch, int height, int width, int channels, cudaStream_t stream) {
  return avgpool3x3_s1_launch<true>(x, y, batch, height, width, channels, stream, "avgpool3x3_s1_excl");
}

}  // namespace yb
