// ResNet plugin kernels (SURVEY 8f rank 4; /root/reference model/resnet.py:28-147), inference and training.
//   stem7x7     nn.Conv2d(3, 64, 7, stride 2, pad 3) + BatchNorm2d + ReLU (:107-109): fp32 NCHW image in, fp16 NHWC out -- the layout boundary.
//               Train mode: the raw conv output (stem7x7 raw = 1) and its weight gradient (stem7x7_wgrad).
//   maxpool3x3  nn.MaxPool2d(3, stride 2, pad 1) (:110) on fp16 NHWC, and its backward.
//   subsample2  x[:, ::2, ::2, :]: a stride-2 conv with "same" padding equals its stride-1 form at the even pixels, so the three stride-2 3x3
//               convs and the 1x1 stride-2 downsample convs (:33,:39,:65,:73) run on the stride-1 wgmma kernel + this selection.
//               upsample2_zero is its transpose (the backward of the selection).
//   add_relu    out += residual; relu (:58-59, :100-101); residual_bwd is the gradient at a block boundary.
// The 3x3 / 1x1 convs themselves (with folded BN and ReLU or identity) are yb_conv_bn_act_fwd.
#include "yb_common.h"
#include "yb_input.cuh"
#include "yb_pool.cuh"
#include <cuda_fp16.h>
#include <stdint.h>

namespace yb {

constexpr int kStemOut = 64, kStemTaps = 147;

// one thread per output pixel, all 64 channels in registers; weights [tap][64] in shared memory (tap = ci*49 + r*7 + s).
// kRaw: the train-mode form, the conv output z itself (no BatchNorm, no ReLU; scale / shift unused).
// kIn: kInF32 (x fp32 NCHW) or kInLut (x_u8 uint8 NHWC through lut[3][256]; yb_input.cuh).
template <bool kRaw, int kIn>
__global__ void __launch_bounds__(128) stem7x7_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ scale,
                                                      const float* __restrict__ shift, __half* __restrict__ y, int batch, int height, int width,
                                                      const uint8_t* __restrict__ x_u8, const float* __restrict__ lut) {
  extern __shared__ float ws[];            // [147][64]
  for (int i = threadIdx.x; i < kStemTaps * kStemOut; i += blockDim.x) ws[i] = w[(i % kStemOut) * kStemTaps + i / kStemOut];
  __syncthreads();
  const int oh = height >> 1, ow = width >> 1;
  const long long total = static_cast<long long>(batch) * oh * ow;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int px = static_cast<int>(idx % ow);
  const long long t = idx / ow;
  const int py = static_cast<int>(t % oh);
  const long long img = t / oh;
  float acc[kStemOut];
#pragma unroll
  for (int i = 0; i < kStemOut; ++i) acc[i] = 0.f;
  for (int ci = 0; ci < 3; ++ci) {
    const float* xp = x + (img * 3 + ci) * height * width;
    for (int r = 0; r < 7; ++r) {
      const int iy = 2 * py - 3 + r;
      if (iy < 0 || iy >= height) continue;
#pragma unroll
      for (int s = 0; s < 7; ++s) {
        const int ix = 2 * px - 3 + s;
        float v;
        if (kIn == kInLut) v = (ix >= 0 && ix < width) ? lut_pixel(x_u8, lut, img, ci, iy, ix, height, width) : 0.f;
        else v = (ix >= 0 && ix < width) ? __ldg(xp + static_cast<long long>(iy) * width + ix) : 0.f;
        const float4* wp = reinterpret_cast<const float4*>(ws + (ci * 49 + r * 7 + s) * kStemOut);
#pragma unroll
        for (int q = 0; q < kStemOut / 4; ++q) {
          const float4 wv = wp[q];
          acc[4 * q] = fmaf(v, wv.x, acc[4 * q]); acc[4 * q + 1] = fmaf(v, wv.y, acc[4 * q + 1]);
          acc[4 * q + 2] = fmaf(v, wv.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(v, wv.w, acc[4 * q + 3]);
        }
      }
    }
  }
  uint4* dst = reinterpret_cast<uint4*>(y + idx * kStemOut);
#pragma unroll
  for (int q = 0; q < kStemOut / 8; ++q) {
    uint4 pk;
    __half2* h = reinterpret_cast<__half2*>(&pk);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = q * 8 + 2 * e;
      if (kRaw)
        h[e] = __floats2half2_rn(acc[c], acc[c + 1]);
      else
        h[e] = __floats2half2_rn(fmaxf(acc[c] * __ldg(scale + c) + __ldg(shift + c), 0.f), fmaxf(acc[c + 1] * __ldg(scale + c + 1) + __ldg(shift + c + 1), 0.f));
    }
    dst[q] = pk;
  }
}

// raw = 1: the train-mode form (scale / shift may be NULL).  lut == nullptr: x is fp32 NCHW; otherwise uint8 NHWC read through lut[3][256] (not
// with raw)
int stem7x7(const void* x, const float* lut, const float* w, const float* scale, const float* shift, void* y, int batch, int height, int width, int raw,
            cudaStream_t stream) {
  YB_REQUIRE(x && w && (raw || (scale && shift)) && y && batch > 0 && height % 2 == 0 && width % 2 == 0 && !(raw && lut), "stem7x7: bad argument");
  const int smem = kStemTaps * kStemOut * static_cast<int>(sizeof(float));
  const int form = lut ? 2 : raw ? 1 : 0;
  static bool attr_set[3] = {false, false, false};
  if (!attr_set[form]) {
    YB_CUDA(cudaFuncSetAttribute(lut ? stem7x7_kernel<false, kInLut> : raw ? stem7x7_kernel<true, kInF32> : stem7x7_kernel<false, kInF32>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set[form] = true;
  }
  const long long total = static_cast<long long>(batch) * (height / 2) * (width / 2);
  const unsigned grid = static_cast<unsigned>((total + 127) / 128);
  const float* xf = lut ? nullptr : static_cast<const float*>(x);
  const uint8_t* xu = lut ? static_cast<const uint8_t*>(x) : nullptr;
  if (lut)
    stem7x7_kernel<false, kInLut><<<grid, 128, smem, stream>>>(xf, w, scale, shift, reinterpret_cast<__half*>(y), batch, height, width, xu, lut);
  else if (raw)
    stem7x7_kernel<true, kInF32><<<grid, 128, smem, stream>>>(xf, w, scale, shift, reinterpret_cast<__half*>(y), batch, height, width, xu, lut);
  else
    stem7x7_kernel<false, kInF32><<<grid, 128, smem, stream>>>(xf, w, scale, shift, reinterpret_cast<__half*>(y), batch, height, width, xu, lut);
  return check_launch("stem7x7_kernel");
}

// Weight gradient of the stem (model/resnet.py:107, nn.Conv2d(3, 64, 7, stride 2, pad 3)): dw[co][ci][r][s] = sum over output pixels p of
// x[b, ci, 2oy - 3 + r, 2ox - 3 + s] * dz[p, co], fp32 OIHW [64,3,7,7] (ADDED to dw, zeroed by the host first).  192 threads = 64 output channels x
// 3 input channels; a thread keeps the 49 sums of its (co, ci) in registers.  Each CTA walks a grid-strided sequence of slabs of kWgSlab pixels:
// the slab's image patches (kWgSlab x 147 fp32) and dz rows (kWgSlab x 64) are staged in shared memory, where a warp's patch reads are broadcasts.
// One fp32 atomic per weight per CTA at the end.
constexpr int kWgSlab = 16;
__global__ void __launch_bounds__(192) stem7x7_wgrad_kernel(const float* __restrict__ x, const __half* __restrict__ dz, float* __restrict__ dw, int batch,
                                                            int height, int width) {
  __shared__ float s_x[kWgSlab][kStemTaps];
  __shared__ float s_g[kWgSlab][kStemOut];
  const int co = threadIdx.x & 63, ci = threadIdx.x >> 6;
  const int oh = height >> 1, ow = width >> 1;
  const long long pixels = static_cast<long long>(batch) * oh * ow;
  float acc[49];
#pragma unroll
  for (int k = 0; k < 49; ++k) acc[k] = 0.f;
  for (long long p0 = static_cast<long long>(blockIdx.x) * kWgSlab; p0 < pixels; p0 += static_cast<long long>(gridDim.x) * kWgSlab) {
    __syncthreads();                       // the previous slab is consumed
    for (int i = threadIdx.x; i < kWgSlab * kStemTaps; i += blockDim.x) {
      const int j = i / kStemTaps, tap = i - j * kStemTaps;
      const long long p = p0 + j;
      float v = 0.f;
      if (p < pixels) {
        const int px = static_cast<int>(p % ow);
        const long long t = p / ow;
        const int py = static_cast<int>(t % oh);
        const long long img = t / oh;
        const int c = tap / 49, rs = tap - c * 49, r = rs / 7, s = rs - r * 7;
        const int iy = 2 * py - 3 + r, ix = 2 * px - 3 + s;
        if (iy >= 0 && iy < height && ix >= 0 && ix < width) v = __ldg(x + ((img * 3 + c) * height + iy) * width + ix);
      }
      s_x[j][tap] = v;
    }
    for (int i = threadIdx.x; i < kWgSlab * kStemOut; i += blockDim.x) {
      const int j = i >> 6;
      const long long p = p0 + j;
      s_g[j][i & 63] = p < pixels ? __half2float(dz[p * kStemOut + (i & 63)]) : 0.f;
    }
    __syncthreads();
#pragma unroll 2
    for (int j = 0; j < kWgSlab; ++j) {
      const float g = s_g[j][co];
      const float* xp = &s_x[j][ci * 49];
#pragma unroll
      for (int k = 0; k < 49; ++k) acc[k] = fmaf(xp[k], g, acc[k]);
    }
  }
  float* dst = dw + (co * 3 + ci) * 49;
#pragma unroll
  for (int k = 0; k < 49; ++k) atomicAdd(dst + k, acc[k]);
}

int stem7x7_wgrad(const float* x, const void* dz, float* dw, int batch, int height, int width, cudaStream_t stream) {
  YB_REQUIRE(x && dz && dw && batch > 0 && height % 2 == 0 && width % 2 == 0, "stem7x7_wgrad: bad argument");
  YB_CUDA(cudaMemsetAsync(dw, 0, kStemOut * kStemTaps * sizeof(float), stream));
  const long long pixels = static_cast<long long>(batch) * (height / 2) * (width / 2);
  const long long blocks = (pixels + kWgSlab * 16 - 1) / (kWgSlab * 16);       // at least 16 slabs per CTA before the grid is capped
  const int cap = sm_count() * 4;
  const int grid = static_cast<int>(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
  stem7x7_wgrad_kernel<<<grid, 192, 0, stream>>>(x, reinterpret_cast<const __half*>(dz), dw, batch, height, width);
  return check_launch("stem7x7_wgrad_kernel");
}

// nn.MaxPool2d(kernel_size=3, stride=2, padding=1): out[oy, ox] = max over the in-range pixels of rows 2oy-1..2oy+1, columns 2ox-1..2ox+1
__global__ void maxpool3x3_s2_kernel(const __half* __restrict__ x, __half* __restrict__ y, int batch, int height, int width, int channels) {
  const int c8 = channels >> 3;
  const int oh = (height + 1) / 2, ow = (width + 1) / 2;
  const long long total = static_cast<long long>(batch) * oh * ow * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int px = static_cast<int>(t % ow); t /= ow;
  const int py = static_cast<int>(t % oh);
  const long long img = t / oh;
  const uint4 m = maxpool3x3_s2_window(x, img, py, px, cg, height, width, channels);
  reinterpret_cast<uint4*>(y)[idx] = m;
}

int maxpool3x3_s2(const void* x, void* y, int batch, int height, int width, int channels, cudaStream_t stream) {
  YB_REQUIRE(x && y && batch > 0 && height > 0 && width > 0 && channels % 8 == 0, "maxpool3x3_s2: bad argument");
  const long long total = static_cast<long long>(batch) * ((height + 1) / 2) * ((width + 1) / 2) * (channels / 8);
  maxpool3x3_s2_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), batch, height,
                                                                                      width, channels);
  return check_launch("maxpool3x3_s2_kernel");
}

// Backward of nn.MaxPool2d(3, 2, 1) (model/resnet.py:110): every output's gradient goes to the FIRST maximum of its window in scan order (rows, then
// columns; a later element replaces the running maximum only if strictly greater, or NaN), as torch's CPU kernel does.  The argmax is recomputed
// from the saved input x.  One thread per input pixel and 8 channels gathers from the at most 2 x 2 windows that contain the pixel, sums in fp32
// and rounds once: no atomics, deterministic.
__global__ void maxpool3x3_s2_bwd_kernel(const __half* __restrict__ x, const __half* __restrict__ dy, __half* __restrict__ dx, int batch, int height, int width,
                                         int channels) {
  const int c8 = channels >> 3;
  const int oh = (height + 1) / 2, ow = (width + 1) / 2;
  const long long total = static_cast<long long>(batch) * height * width * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int ix = static_cast<int>(t % width); t /= width;
  const int iy = static_cast<int>(t % height);
  const long long img = t / height;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  // windows oy with 2oy - 1 <= iy <= 2oy + 1
  const int oy0 = iy / 2, oy1 = min((iy + 1) / 2, oh - 1);
  const int ox0 = ix / 2, ox1 = min((ix + 1) / 2, ow - 1);
  for (int oy = oy0; oy <= oy1; ++oy) {
    for (int ox = ox0; ox <= ox1; ++ox) {
      float best[8];
      int arg[8];
      bool any = false;
      for (int r = 0; r < 3; ++r) {
        const int yy = 2 * oy - 1 + r;
        if (yy < 0 || yy >= height) continue;
        for (int s = 0; s < 3; ++s) {
          const int xx = 2 * ox - 1 + s;
          if (xx < 0 || xx >= width) continue;
          const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + ((img * height + yy) * width + xx) * channels + cg * 8));
          const __half* hv = reinterpret_cast<const __half*>(&v);
          const int pos = yy * width + xx;
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const float f = __half2float(hv[e]);
            if (!any || f > best[e] || isnan(f)) {
              best[e] = f;
              arg[e] = pos;
            }
          }
          any = true;
        }
      }
      const uint4 g = __ldg(reinterpret_cast<const uint4*>(dy + ((img * oh + oy) * ow + ox) * channels + cg * 8));
      const __half* hg = reinterpret_cast<const __half*>(&g);
      const int me = iy * width + ix;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (arg[e] == me) acc[e] += __half2float(hg[e]);
    }
  }
  uint4 out;
  __half2* ho = reinterpret_cast<__half2*>(&out);
#pragma unroll
  for (int e = 0; e < 4; ++e) ho[e] = __floats2half2_rn(acc[2 * e], acc[2 * e + 1]);
  reinterpret_cast<uint4*>(dx)[idx] = out;
}

int maxpool3x3_s2_bwd(const void* x, const void* dy, void* dx, int batch, int height, int width, int channels, cudaStream_t stream) {
  YB_REQUIRE(x && dy && dx && batch > 0 && height > 0 && width > 0 && channels % 8 == 0, "maxpool3x3_s2_bwd: bad argument");
  const long long total = static_cast<long long>(batch) * height * width * (channels / 8);
  maxpool3x3_s2_bwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x), reinterpret_cast<const __half*>(dy),
                                                                                          reinterpret_cast<__half*>(dx), batch, height, width, channels);
  return check_launch("maxpool3x3_s2_bwd_kernel");
}

// y[b, oy, ox, :] = x[b, 2oy, 2ox, :]
__global__ void subsample2_kernel(const __half* __restrict__ x, __half* __restrict__ y, int batch, int height, int width, int channels) {
  const int c8 = channels >> 3;
  const int oh = (height + 1) / 2, ow = (width + 1) / 2;
  const long long total = static_cast<long long>(batch) * oh * ow * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int px = static_cast<int>(t % ow); t /= ow;
  const int py = static_cast<int>(t % oh);
  const long long img = t / oh;
  reinterpret_cast<uint4*>(y)[idx] = __ldg(reinterpret_cast<const uint4*>(x + ((img * height + 2 * py) * width + 2 * px) * channels + cg * 8));
}

int subsample2(const void* x, void* y, int batch, int height, int width, int channels, cudaStream_t stream) {
  YB_REQUIRE(x && y && batch > 0 && height > 0 && width > 0 && channels % 8 == 0, "subsample2: bad argument");
  const long long total = static_cast<long long>(batch) * ((height + 1) / 2) * ((width + 1) / 2) * (channels / 8);
  subsample2_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), batch, height, width,
                                                                                   channels);
  return check_launch("subsample2_kernel");
}

// The transpose of subsample2: y[b, 2oy, 2ox, :] = x[b, oy, ox, :], zero at the odd rows / columns.  height / width are those of y (full resolution).
// The backward of a stride-2 conv computed as subsample2 o (stride-1 conv): dz at half resolution goes through this, then the stride-1 gradients.
__global__ void upsample2_zero_kernel(const __half* __restrict__ x, __half* __restrict__ y, int batch, int height, int width, int channels) {
  const int c8 = channels >> 3;
  const int xh = (height + 1) / 2, xw = (width + 1) / 2;
  const long long total = static_cast<long long>(batch) * height * width * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int ix = static_cast<int>(t % width); t /= width;
  const int iy = static_cast<int>(t % height);
  const long long img = t / height;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (((iy | ix) & 1) == 0) v = __ldg(reinterpret_cast<const uint4*>(x + ((img * xh + (iy >> 1)) * xw + (ix >> 1)) * channels + cg * 8));
  reinterpret_cast<uint4*>(y)[idx] = v;
}

int upsample2_zero(const void* x, void* y, int batch, int height, int width, int channels, cudaStream_t stream) {
  YB_REQUIRE(x && y && batch > 0 && height > 0 && width > 0 && channels % 8 == 0, "upsample2_zero: bad argument");
  const long long total = static_cast<long long>(batch) * height * width * (channels / 8);
  upsample2_zero_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), batch, height,
                                                                                       width, channels);
  return check_launch("upsample2_zero_kernel");
}

// Gradient at a block boundary (model/resnet.py:44-61, 82-103 in reverse): out = (y > 0) ? g_a + S^T g_b : 0, fp32 sum, one rounding.  y is the
// block input (the previous block's ReLU output; NULL = no mask, the max-pool output in front of layer1.0), g_a the main path's data gradient at
// y's resolution, g_b the skip path's (NULL = none): the identity skip at stride 1, the downsample conv's data gradient at half resolution with
// stride_b = 2 (S^T = zero insertion).
__global__ void residual_bwd_kernel(const __half* __restrict__ y, const __half* __restrict__ ga, const __half* __restrict__ gb, int stride_b,
                                    __half* __restrict__ out, int batch, int height, int width, int channels) {
  const int c8 = channels >> 3;
  const long long total = static_cast<long long>(batch) * height * width * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const uint4 va = __ldg(reinterpret_cast<const uint4*>(ga) + idx);
  const __half2* pa = reinterpret_cast<const __half2*>(&va);
  float f[8];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 a = __half22float2(pa[e]);
    f[2 * e] = a.x;
    f[2 * e + 1] = a.y;
  }
  if (gb != nullptr) {
    long long bi = idx;
    bool hit = true;
    if (stride_b == 2) {
      const int cg = static_cast<int>(idx % c8);
      long long t = idx / c8;
      const int ix = static_cast<int>(t % width); t /= width;
      const int iy = static_cast<int>(t % height);
      const long long img = t / height;
      hit = ((iy | ix) & 1) == 0;
      bi = ((img * ((height + 1) / 2) + (iy >> 1)) * ((width + 1) / 2) + (ix >> 1)) * c8 + cg;
    }
    if (hit) {
      const uint4 vb = __ldg(reinterpret_cast<const uint4*>(gb) + bi);
      const __half2* pb = reinterpret_cast<const __half2*>(&vb);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 b = __half22float2(pb[e]);
        f[2 * e] += b.x;
        f[2 * e + 1] += b.y;
      }
    }
  }
  if (y != nullptr) {
    const uint4 vy = __ldg(reinterpret_cast<const uint4*>(y) + idx);
    const __half* hy = reinterpret_cast<const __half*>(&vy);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (!(__half2float(hy[e]) > 0.f)) f[e] = 0.f;
  }
  uint4 r;
  __half2* pr = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int e = 0; e < 4; ++e) pr[e] = __floats2half2_rn(f[2 * e], f[2 * e + 1]);
  reinterpret_cast<uint4*>(out)[idx] = r;
}

int residual_bwd(const void* y, const void* ga, const void* gb, int stride_b, void* out, int batch, int height, int width, int channels, cudaStream_t stream) {
  YB_REQUIRE(ga && out && batch > 0 && height > 0 && width > 0 && channels % 8 == 0 && (stride_b == 1 || stride_b == 2), "residual_bwd: bad argument");
  const long long total = static_cast<long long>(batch) * height * width * (channels / 8);
  residual_bwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(y), reinterpret_cast<const __half*>(ga),
                                                                                     reinterpret_cast<const __half*>(gb), stride_b, reinterpret_cast<__half*>(out), batch,
                                                                                     height, width, channels);
  return check_launch("residual_bwd_kernel");
}

// out = relu(a + b), fp16, fp32 add, 8 elements per thread
__global__ void add_relu_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ out, long long n8) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n8) return;
  const uint4 va = __ldg(a + idx), vb = __ldg(b + idx);
  const __half2* pa = reinterpret_cast<const __half2*>(&va);
  const __half2* pb = reinterpret_cast<const __half2*>(&vb);
  uint4 r;
  __half2* pr = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 fa = __half22float2(pa[i]), fb = __half22float2(pb[i]);
    pr[i] = __floats2half2_rn(fmaxf(fa.x + fb.x, 0.f), fmaxf(fa.y + fb.y, 0.f));
  }
  out[idx] = r;
}

int add_relu(const void* a, const void* b, void* out, long long count, cudaStream_t stream) {
  YB_REQUIRE(a && b && out && count > 0 && count % 8 == 0, "add_relu: count must be a positive multiple of 8");
  const long long n8 = count / 8;
  add_relu_kernel<<<static_cast<unsigned>((n8 + 255) / 256), 256, 0, stream>>>(static_cast<const uint4*>(a), static_cast<const uint4*>(b), static_cast<uint4*>(out), n8);
  return check_launch("add_relu_kernel");
}

}  // namespace yb
