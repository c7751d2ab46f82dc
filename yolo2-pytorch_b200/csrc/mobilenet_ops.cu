// MobileNet plugin kernels (BASELINE configs[4], "C5"; /root/reference model/mobilenet.py:25-85), inference only.
//   mb_conv0   conv_bn(3, 32, stride 2): nn.Conv2d(3,32,3,2,1) + BatchNorm2d + ReLU  (:25-30), fp32 NCHW image in,
//              fp16 NHWC out -- the layout boundary of this backbone.  kPad = 0 is Inception-v3's Conv2d_1a_3x3 (the same conv without
//              padding, any H, W >= 3).
//   dwconv3x3  conv_dw: depthwise nn.Conv2d(C,C,3,stride,1,groups=C) + BatchNorm2d + ReLU (:33-38) on fp16 NHWC.
//              HBM-bound: one thread = 8 channels (16 B) of one output pixel, 9 vector loads, fp32 FMA, 16 B store.
// The pointwise convs (conv_pw, :41-46) and the 1x1 head reuse the wgmma implicit-GEMM kernel (slope = 0 -> ReLU).
#include "yb_common.h"
#include <cuda_fp16.h>
#include <stdint.h>

namespace yb {

template <int kPad>
__global__ void __launch_bounds__(256) mb_conv0_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ scale,
                                                       const float* __restrict__ shift, __half* __restrict__ y, int batch, int height, int width, int raw,
                                                       int split) {
  __shared__ __align__(16) float ws[27][32];
  __shared__ float sc[32], sh[32];
  for (int i = threadIdx.x; i < 27 * 32; i += blockDim.x) ws[i / 32][i % 32] = w[(i % 32) * 27 + i / 32];
  if (threadIdx.x < 32) { sc[threadIdx.x] = raw ? 1.f : scale[threadIdx.x]; sh[threadIdx.x] = raw ? 0.f : shift[threadIdx.x]; }
  __syncthreads();
  const int oh = (height + 2 * kPad - 3) / 2 + 1, ow = (width + 2 * kPad - 3) / 2 + 1;
  const long long total = static_cast<long long>(batch) * oh * ow;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int px = static_cast<int>(idx % ow);
  const long long t = idx / ow;
  const int py = static_cast<int>(t % oh);
  const int img = static_cast<int>(t / oh);
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int iy = 2 * py - kPad + r;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ix = 2 * px - kPad + s;
        const float v = (iy >= 0 && iy < height && ix >= 0 && ix < width) ? __ldg(x + ((static_cast<long long>(img) * 3 + c) * height + iy) * width + ix) : 0.f;
        const float4* wp = reinterpret_cast<const float4*>(&ws[c * 9 + r * 3 + s][0]);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 wv = wp[q];
          acc[4 * q] = fmaf(v, wv.x, acc[4 * q]); acc[4 * q + 1] = fmaf(v, wv.y, acc[4 * q + 1]);
          acc[4 * q + 2] = fmaf(v, wv.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(v, wv.w, acc[4 * q + 3]);
        }
      }
    }
  // split (strict precision): the pixel holds [hi 32 | lo 32], lo = fp16(v - fp32(hi)): the next layer reads hi + lo
  uint4* dst = reinterpret_cast<uint4*>(y + idx * (split ? 64 : 32));
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 pk, pl;
    __half2* h = reinterpret_cast<__half2*>(&pk);
    __half2* hl = reinterpret_cast<__half2*>(&pl);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = q * 8 + 2 * e;
      const float lo = raw ? -INFINITY : 0.f;          // raw (training forward): the conv output itself, BatchNorm / ReLU come later
      const float v0 = fmaxf(acc[c] * sc[c] + sh[c], lo), v1 = fmaxf(acc[c + 1] * sc[c + 1] + sh[c + 1], lo);
      h[e] = __floats2half2_rn(v0, v1);
      const float2 r = __half22float2(h[e]);
      hl[e] = __floats2half2_rn(v0 - r.x, v1 - r.y);
    }
    dst[q] = pk;
    if (split) dst[4 + q] = pl;
  }
}

int mb_conv0(const float* x, const float* w, const float* scale, const float* shift, void* y, int batch, int height, int width, int raw, int split,
             cudaStream_t stream) {
  YB_REQUIRE(x && w && (raw || (scale && shift)) && y && batch > 0 && height % 2 == 0 && width % 2 == 0 && !(raw && split), "mb_conv0: bad argument");
  const long long total = static_cast<long long>(batch) * (height / 2) * (width / 2);
  mb_conv0_kernel<1><<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(x, w, raw ? w : scale, raw ? w : shift, reinterpret_cast<__half*>(y), batch, height, width,
                                                                                    raw, split);
  return check_launch("mb_conv0_kernel");
}

// Inception-v3 Conv2d_1a_3x3: nn.Conv2d(3, 32, 3, stride 2, pad `pad`) + folded BatchNorm + ReLU, x fp32 NCHW [B,3,H,W] -> y fp16 NHWC
// [B,(H+2pad-3)/2+1,(W+2pad-3)/2+1,32].  pad = 1 is the MobileNet instantiation (same bits as mb_conv0 at even H, W).
int stem3x3_s2(const float* x, const float* w, const float* scale, const float* shift, void* y, int batch, int height, int width, int pad,
               cudaStream_t stream) {
  YB_REQUIRE(x && w && scale && shift && y && batch > 0 && (pad == 0 || pad == 1), "stem3x3_s2: bad argument (pad 0 or 1)");
  YB_REQUIRE(height + 2 * pad >= 3 && width + 2 * pad >= 3, "stem3x3_s2: %d x %d input gives an empty output", height, width);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(y) & 15) == 0, "stem3x3_s2: y must be 16B aligned");
  const long long total = static_cast<long long>(batch) * ((height + 2 * pad - 3) / 2 + 1) * ((width + 2 * pad - 3) / 2 + 1);
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  if (pad == 0) mb_conv0_kernel<0><<<grid, 256, 0, stream>>>(x, w, scale, shift, reinterpret_cast<__half*>(y), batch, height, width, 0, 0);
  else mb_conv0_kernel<1><<<grid, 256, 0, stream>>>(x, w, scale, shift, reinterpret_cast<__half*>(y), batch, height, width, 0, 0);
  return check_launch("mb_conv0_kernel");
}

// w: fp32 [C][9] (the [C,1,3,3] depthwise weight), scale/shift: folded BN.
// One thread = 8 channels (16 B) of TX consecutive output pixels of one row.  Its 72 weights are 288 contiguous bytes (18 x LDG.128,
// once), the 3 x 3 input window slides along the row in registers (3 new 16 B loads per output pixel at stride 1, 6 at stride 2), so
// the kernel issues ~1/4 of the load instructions of the one-pixel-per-thread form (which ncu showed issue-bound at 0.10 of HBM peak).
template <int STRIDE, int TX>
__global__ void __launch_bounds__(128) dwconv3x3_kernel(const __half* __restrict__ x, const float* __restrict__ w, const float* __restrict__ scale,
                                                        const float* __restrict__ shift, __half* __restrict__ y, int batch, int height, int width,
                                                        int channels, int raw) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int c8 = channels >> 3;
  const int oh = height / STRIDE, ow = width / STRIDE;
  const int strips = (ow + TX - 1) / TX;
  const long long total = static_cast<long long>(batch) * oh * strips * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int strip = static_cast<int>(t % strips); t /= strips;
  const int py = static_cast<int>(t % oh);
  const int img = static_cast<int>(t / oh);
  float wr[72];
  {
    const float4* wp = reinterpret_cast<const float4*>(w + static_cast<long long>(cg) * 72);
#pragma unroll
    for (int i = 0; i < 18; ++i) {
      const float4 v = __ldg(wp + i);
      wr[4 * i] = v.x; wr[4 * i + 1] = v.y; wr[4 * i + 2] = v.z; wr[4 * i + 3] = v.w;
    }
  }
  float sc[8], sh[8];
  {
    float4 a0 = make_float4(1.f, 1.f, 1.f, 1.f), a1 = a0, b0 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = b0;
    if (!raw) {
      a0 = __ldg(reinterpret_cast<const float4*>(scale + cg * 8)); a1 = __ldg(reinterpret_cast<const float4*>(scale + cg * 8) + 1);
      b0 = __ldg(reinterpret_cast<const float4*>(shift + cg * 8)); b1 = __ldg(reinterpret_cast<const float4*>(shift + cg * 8) + 1);
    }
    sc[0] = a0.x; sc[1] = a0.y; sc[2] = a0.z; sc[3] = a0.w; sc[4] = a1.x; sc[5] = a1.y; sc[6] = a1.z; sc[7] = a1.w;
    sh[0] = b0.x; sh[1] = b0.y; sh[2] = b0.z; sh[3] = b0.w; sh[4] = b1.x; sh[5] = b1.y; sh[6] = b1.z; sh[7] = b1.w;
  }
  const int px0 = strip * TX;
  const int iy0 = py * STRIDE - 1;
  const __half* xrow[3];
  bool rok[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int iy = iy0 + r;
    rok[r] = iy >= 0 && iy < height;
    xrow[r] = x + ((static_cast<long long>(img) * height + (rok[r] ? iy : 0)) * width) * channels + cg * 8;
  }
  auto load_col = [&](int ix, uint4 (&col)[3]) {
    const bool cok = ix >= 0 && ix < width;
#pragma unroll
    for (int r = 0; r < 3; ++r)
      col[r] = (cok && rok[r]) ? __ldg(reinterpret_cast<const uint4*>(xrow[r] + static_cast<long long>(ix) * channels)) : make_uint4(0u, 0u, 0u, 0u);
  };
  uint4 win[3][3];                                   // [column s][row r]
  load_col(px0 * STRIDE - 1, win[0]);
  if (STRIDE == 1) load_col(px0 * STRIDE, win[1]);
#pragma unroll
  for (int j = 0; j < TX; ++j) {
    const int px = px0 + j;
    if (px >= ow) break;
    if (STRIDE == 1) {
      load_col(px + 1, win[2]);
    } else {
      load_col(2 * px, win[1]);
      load_col(2 * px + 1, win[2]);
    }
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
    for (int s = 0; s < 3; ++s)
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const __half2* h = reinterpret_cast<const __half2*>(&win[s][r]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(h[e]);
          acc[2 * e] = fmaf(f.x, wr[(2 * e) * 9 + r * 3 + s], acc[2 * e]);
          acc[2 * e + 1] = fmaf(f.y, wr[(2 * e + 1) * 9 + r * 3 + s], acc[2 * e + 1]);
        }
      }
    uint4 pk;
    __half2* ho = reinterpret_cast<__half2*>(&pk);
#pragma unroll
    const float lo = raw ? -INFINITY : 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e)
      ho[e] = __floats2half2_rn(fmaxf(acc[2 * e] * sc[2 * e] + sh[2 * e], lo), fmaxf(acc[2 * e + 1] * sc[2 * e + 1] + sh[2 * e + 1], lo));
    *reinterpret_cast<uint4*>(y + ((static_cast<long long>(img) * oh + py) * ow + px) * channels + cg * 8) = pk;
    // slide: stride 1 keeps two columns, stride 2 keeps one
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      if (STRIDE == 1) { win[0][r] = win[1][r]; win[1][r] = win[2][r]; }
      else win[0][r] = win[2][r];
    }
  }
}

int dwconv3x3(const void* x, const float* w, const float* scale, const float* shift, void* y, int batch, int height, int width, int channels,
              int stride, int raw, cudaStream_t stream) {
  YB_REQUIRE(x && w && (raw || (scale && shift)) && y && batch > 0 && channels % 8 == 0 && (stride == 1 || stride == 2) && height % stride == 0 &&
                 width % stride == 0,
             "dwconv3x3: bad argument");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(w) & 15) == 0 && (raw || ((reinterpret_cast<uintptr_t>(scale) & 15) == 0 && (reinterpret_cast<uintptr_t>(shift) & 15) == 0)),
             "dwconv3x3: weights / scale / shift must be 16 B aligned");
  const int oh = height / stride, ow = width / stride;
  // pixels per thread: long strips amortise the 72-weight preload, but the grid must still cover the SMs on the 13 x 13 layers
  const int tx = ow >= 52 ? 8 : 4;
  const long long total = static_cast<long long>(batch) * oh * ((ow + tx - 1) / tx) * (channels / 8);
  const unsigned grid = static_cast<unsigned>((total + 127) / 128);
  const __half* xp = reinterpret_cast<const __half*>(x);
  __half* yp = reinterpret_cast<__half*>(y);
  if (stride == 1) {
    if (tx == 8) dwconv3x3_kernel<1, 8><<<grid, 128, 0, stream>>>(xp, w, scale, shift, yp, batch, height, width, channels, raw);
    else dwconv3x3_kernel<1, 4><<<grid, 128, 0, stream>>>(xp, w, scale, shift, yp, batch, height, width, channels, raw);
  } else {
    if (tx == 8) dwconv3x3_kernel<2, 8><<<grid, 128, 0, stream>>>(xp, w, scale, shift, yp, batch, height, width, channels, raw);
    else dwconv3x3_kernel<2, 4><<<grid, 128, 0, stream>>>(xp, w, scale, shift, yp, batch, height, width, channels, raw);
  }
  return check_launch("dwconv3x3_kernel");
}

// Strict-precision form (the plugin's `precision = strict`): activations travel as [hi | lo] fp16 pairs (x: [B,H,W,2C], y: [B,OH,OW,2C]), the
// depthwise sum runs on hi + lo in fp32 and the result is split again, so a depthwise layer adds no fp16 rounding of its own.
// One thread = 8 channels of one output pixel (18 loads); this mode trades speed for the 1e-3 contract.
__global__ void __launch_bounds__(128) dwconv3x3_split_kernel(const __half* __restrict__ x, const float* __restrict__ w, const float* __restrict__ scale,
                                                              const float* __restrict__ shift, __half* __restrict__ y, int batch, int height, int width,
                                                              int channels, int stride) {
  const int c8 = channels >> 3;
  const int oh = height / stride, ow = width / stride;
  const long long total = static_cast<long long>(batch) * oh * ow * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int px = static_cast<int>(t % ow); t /= ow;
  const int py = static_cast<int>(t % oh);
  const long long img = t / oh;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  const float* wp = w + static_cast<long long>(cg) * 72;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int iy = py * stride - 1 + r;
    if (iy < 0 || iy >= height) continue;
#pragma unroll
    for (int s2 = 0; s2 < 3; ++s2) {
      const int ix = px * stride - 1 + s2;
      if (ix < 0 || ix >= width) continue;
      const __half* src = x + ((img * height + iy) * width + ix) * (2 * channels) + cg * 8;
      const uint4 qh = __ldg(reinterpret_cast<const uint4*>(src)), ql = __ldg(reinterpret_cast<const uint4*>(src + channels));
      const __half2* hh = reinterpret_cast<const __half2*>(&qh);
      const __half2* hl = reinterpret_cast<const __half2*>(&ql);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = __half22float2(hh[e]), b = __half22float2(hl[e]);
        acc[2 * e] = fmaf(a.x + b.x, __ldg(wp + (2 * e) * 9 + r * 3 + s2), acc[2 * e]);
        acc[2 * e + 1] = fmaf(a.y + b.y, __ldg(wp + (2 * e + 1) * 9 + r * 3 + s2), acc[2 * e + 1]);
      }
    }
  }
  uint4 pk, pl;
  __half2* ho = reinterpret_cast<__half2*>(&pk);
  __half2* lo = reinterpret_cast<__half2*>(&pl);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int c = cg * 8 + 2 * e;
    const float v0 = fmaxf(acc[2 * e] * __ldg(scale + c) + __ldg(shift + c), 0.f), v1 = fmaxf(acc[2 * e + 1] * __ldg(scale + c + 1) + __ldg(shift + c + 1), 0.f);
    ho[e] = __floats2half2_rn(v0, v1);
    const float2 rr = __half22float2(ho[e]);
    lo[e] = __floats2half2_rn(v0 - rr.x, v1 - rr.y);
  }
  __half* dst = y + ((img * oh + py) * ow + px) * (2 * channels) + cg * 8;
  *reinterpret_cast<uint4*>(dst) = pk;
  *reinterpret_cast<uint4*>(dst + channels) = pl;
}

int dwconv3x3_split(const void* x, const float* w, const float* scale, const float* shift, void* y, int batch, int height, int width, int channels, int stride,
                    cudaStream_t stream) {
  YB_REQUIRE(x && w && scale && shift && y && batch > 0 && channels % 8 == 0 && (stride == 1 || stride == 2) && height % stride == 0 && width % stride == 0,
             "dwconv3x3_split: bad argument");
  const long long total = static_cast<long long>(batch) * (height / stride) * (width / stride) * (channels / 8);
  dwconv3x3_split_kernel<<<static_cast<unsigned>((total + 127) / 128), 128, 0, stream>>>(reinterpret_cast<const __half*>(x), w, scale, shift,
                                                                                        reinterpret_cast<__half*>(y), batch, height, width, channels, stride);
  return check_launch("dwconv3x3_split_kernel");
}

// ------------------------------------------------------------------------------------------------
// Training of the MobileNet plugin (what torch autograd does for conv_bn / conv_dw in the reference, model/mobilenet.py:25-38).
// Depthwise data gradient, both strides: forward z[oy, ox] = sum_{r,s} a[oy*st - 1 + r, ox*st - 1 + s] * w[r, s], hence
// da[y, x] = sum over the taps with (y + 1 - r) and (x + 1 - s) divisible by st of dz[(y + 1 - r)/st, (x + 1 - s)/st] * w[r, s].
// thread = 8 channels of one input pixel.
__global__ void __launch_bounds__(128) dw_dgrad_kernel(const __half* __restrict__ dz, const float* __restrict__ w, __half* __restrict__ da, int batch, int height,
                                                       int width, int channels, int stride) {
  const int c8 = channels >> 3;
  const long long total = static_cast<long long>(batch) * height * width * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int px = static_cast<int>(t % width); t /= width;
  const int py = static_cast<int>(t % height);
  const long long img = t / height;
  const int oh = height / stride, ow = width / stride;
  float wr[72];
  {
    const float4* wp = reinterpret_cast<const float4*>(w + static_cast<long long>(cg) * 72);
#pragma unroll
    for (int i = 0; i < 18; ++i) { const float4 v = __ldg(wp + i); wr[4 * i] = v.x; wr[4 * i + 1] = v.y; wr[4 * i + 2] = v.z; wr[4 * i + 3] = v.w; }
  }
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  const __half* zb = dz + img * oh * ow * channels + cg * 8;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int ty = py + 1 - r;
    if (ty < 0 || ty % stride != 0) continue;
    const int oy = ty / stride;
    if (oy >= oh) continue;
#pragma unroll
    for (int s2 = 0; s2 < 3; ++s2) {
      const int tx = px + 1 - s2;
      if (tx < 0 || tx % stride != 0) continue;
      const int ox = tx / stride;
      if (ox >= ow) continue;
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(zb + (static_cast<long long>(oy) * ow + ox) * channels));
      const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h[e]);
        acc[2 * e] = fmaf(f.x, wr[(2 * e) * 9 + r * 3 + s2], acc[2 * e]);
        acc[2 * e + 1] = fmaf(f.y, wr[(2 * e + 1) * 9 + r * 3 + s2], acc[2 * e + 1]);
      }
    }
  }
  uint4 out;
  __half2* ho = reinterpret_cast<__half2*>(&out);
#pragma unroll
  for (int e = 0; e < 4; ++e) ho[e] = __floats2half2_rn(acc[2 * e], acc[2 * e + 1]);
  reinterpret_cast<uint4*>(da)[idx] = out;
}

int dw_dgrad(const void* dz, const float* w, void* da, int batch, int height, int width, int channels, int stride, cudaStream_t stream) {
  YB_REQUIRE(dz && w && da && batch > 0 && channels % 8 == 0 && (stride == 1 || stride == 2) && height % stride == 0 && width % stride == 0 &&
                 (reinterpret_cast<uintptr_t>(w) & 15) == 0, "dw_dgrad: bad argument");
  const long long total = static_cast<long long>(batch) * height * width * (channels / 8);
  dw_dgrad_kernel<<<static_cast<unsigned>((total + 127) / 128), 128, 0, stream>>>(reinterpret_cast<const __half*>(dz), w, reinterpret_cast<__half*>(da), batch, height,
                                                                                width, channels, stride);
  return check_launch("dw_dgrad_kernel");
}

// Depthwise weight gradient: dw[c][r][s] = sum over images and output pixels of dz[oy, ox, c] * a[oy*st - 1 + r, ox*st - 1 + s, c]  (fp32 [C][9],
// ADDED to dw, which the host zeroes first).  A thread owns 8 channels and walks output pixels with the block's stride; its 72 partial sums are
// combined across the block's pixel lanes in shared memory and leave as one atomicAdd per (channel, tap) and block.
__global__ void __launch_bounds__(256) dw_wgrad_kernel(const __half* __restrict__ a, const __half* __restrict__ dz, float* __restrict__ dw, int batch, int height,
                                                       int width, int channels, int stride) {
  extern __shared__ float s_dw[];            // [channels][9]
  for (int i = threadIdx.x; i < channels * 9; i += blockDim.x) s_dw[i] = 0.f;
  __syncthreads();
  const int c8 = channels >> 3;
  const int cg = threadIdx.x % c8;
  const int lane = threadIdx.x / c8, lanes = blockDim.x / c8;
  const int oh = height / stride, ow = width / stride;
  const long long pixels = static_cast<long long>(batch) * oh * ow;
  float acc[9][8];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[t][e] = 0.f;
  for (long long p = static_cast<long long>(blockIdx.x) * lanes + lane; p < pixels; p += static_cast<long long>(gridDim.x) * lanes) {
    const int ox = static_cast<int>(p % ow);
    const long long t2 = p / ow;
    const int oy = static_cast<int>(t2 % oh);
    const long long img = t2 / oh;
    const uint4 qz = __ldg(reinterpret_cast<const uint4*>(dz + p * channels + cg * 8));
    float g[8];
    {
      const __half2* h = reinterpret_cast<const __half2*>(&qz);
#pragma unroll
      for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(h[e]); g[2 * e] = f.x; g[2 * e + 1] = f.y; }
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int iy = oy * stride - 1 + r;
      if (iy < 0 || iy >= height) continue;
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) {
        const int ix = ox * stride - 1 + s2;
        if (ix < 0 || ix >= width) continue;
        const uint4 qa = __ldg(reinterpret_cast<const uint4*>(a + ((img * height + iy) * width + ix) * channels + cg * 8));
        const __half2* h = reinterpret_cast<const __half2*>(&qa);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(h[e]);
          acc[r * 3 + s2][2 * e] = fmaf(f.x, g[2 * e], acc[r * 3 + s2][2 * e]);
          acc[r * 3 + s2][2 * e + 1] = fmaf(f.y, g[2 * e + 1], acc[r * 3 + s2][2 * e + 1]);
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int e = 0; e < 8; ++e) atomicAdd(&s_dw[(cg * 8 + e) * 9 + t], acc[t][e]);
  __syncthreads();
  for (int i = threadIdx.x; i < channels * 9; i += blockDim.x) atomicAdd(&dw[i], s_dw[i]);
}

int dw_wgrad(const void* a, const void* dz, float* dw, int batch, int height, int width, int channels, int stride, cudaStream_t stream) {
  YB_REQUIRE(a && dz && dw && batch > 0 && channels % 8 == 0 && channels <= 1024 && 256 % (channels / 8) == 0 && (stride == 1 || stride == 2) &&
                 height % stride == 0 && width % stride == 0, "dw_wgrad: bad argument (C=%d)", channels);
  YB_CUDA(cudaMemsetAsync(dw, 0, static_cast<size_t>(channels) * 9 * sizeof(float), stream));
  const long long pixels = static_cast<long long>(batch) * (height / stride) * (width / stride);
  const int lanes = 256 / (channels / 8);
  long long blocks = (pixels + lanes * 16 - 1) / (lanes * 16);            // ~16 pixels per thread: the 72 atomics per thread amortise
  const int cap = sm_count() * 4;
  const int grid = static_cast<int>(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
  dw_wgrad_kernel<<<grid, 256, channels * 9 * sizeof(float), stream>>>(reinterpret_cast<const __half*>(a), reinterpret_cast<const __half*>(dz), dw, batch, height, width,
                                                                       channels, stride);
  return check_launch("dw_wgrad_kernel");
}

// Weight gradient of the stride-2 first layer: dw[co][ci][r][s] = sum x[b, ci, 2*oy - kPad + r, 2*ox - kPad + s] * dz[b, oy, ox, co]  (fp32 OIHW
// [32,3,3,3], ADDED to dw, zeroed by the host first).  kPad = 1: MobileNet (even H, W); kPad = 0: Inception-v3's Conv2d_1a_3x3 (any H, W >= 3).  256 threads = 32 output channels x 8 pixel lanes; a thread keeps its channel's 27 sums in registers.
template <int kPad>
__global__ void __launch_bounds__(256) mb_conv0_wgrad_kernel(const float* __restrict__ x, const __half* __restrict__ dz, float* __restrict__ dw, int batch,
                                                             int height, int width) {
  __shared__ float s_dw[32 * 27];
  for (int i = threadIdx.x; i < 32 * 27; i += blockDim.x) s_dw[i] = 0.f;
  __syncthreads();
  const int co = threadIdx.x & 31, lane = threadIdx.x >> 5;
  const int oh = (height + 2 * kPad - 3) / 2 + 1, ow = (width + 2 * kPad - 3) / 2 + 1;
  const long long pixels = static_cast<long long>(batch) * oh * ow;
  float acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0.f;
  for (long long p = static_cast<long long>(blockIdx.x) * 8 + lane; p < pixels; p += static_cast<long long>(gridDim.x) * 8) {
    const int ox = static_cast<int>(p % ow);
    const long long t2 = p / ow;
    const int oy = static_cast<int>(t2 % oh);
    const long long img = t2 / oh;
    const float g = __half2float(dz[p * 32 + co]);
#pragma unroll
    for (int ci = 0; ci < 3; ++ci)
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int iy = 2 * oy - kPad + r;
#pragma unroll
        for (int s2 = 0; s2 < 3; ++s2) {
          const int ix = 2 * ox - kPad + s2;
          const float v = (iy >= 0 && iy < height && ix >= 0 && ix < width) ? __ldg(x + ((img * 3 + ci) * height + iy) * width + ix) : 0.f;
          acc[ci * 9 + r * 3 + s2] = fmaf(v, g, acc[ci * 9 + r * 3 + s2]);
        }
      }
  }
#pragma unroll
  for (int k = 0; k < 27; ++k) atomicAdd(&s_dw[co * 27 + k], acc[k]);
  __syncthreads();
  for (int i = threadIdx.x; i < 32 * 27; i += blockDim.x) atomicAdd(&dw[i], s_dw[i]);
}

int mb_conv0_wgrad(const float* x, const void* dz, float* dw, int batch, int height, int width, cudaStream_t stream) {
  YB_REQUIRE(x && dz && dw && batch > 0 && height % 2 == 0 && width % 2 == 0, "mb_conv0_wgrad: bad argument");
  YB_CUDA(cudaMemsetAsync(dw, 0, 32 * 27 * sizeof(float), stream));
  const long long pixels = static_cast<long long>(batch) * (height / 2) * (width / 2);
  long long blocks = (pixels + 8 * 32 - 1) / (8 * 32);
  const int cap = sm_count() * 6;
  const int grid = static_cast<int>(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
  mb_conv0_wgrad_kernel<1><<<grid, 256, 0, stream>>>(x, reinterpret_cast<const __half*>(dz), dw, batch, height, width);
  return check_launch("mb_conv0_wgrad_kernel");
}

// Inception-v3's Conv2d_1a_3x3 in training: the raw conv output z (no BatchNorm, no ReLU) and the weight gradient from the fp32 image, at
// padding `pad` (0 for Inception; 1 gives the bits of the MobileNet forms).
int stem3x3_s2_raw(const float* x, const float* w, void* z, int batch, int height, int width, int pad, cudaStream_t stream) {
  YB_REQUIRE(x && w && z && batch > 0 && (pad == 0 || pad == 1), "stem3x3_s2_raw: bad argument (pad 0 or 1)");
  YB_REQUIRE(height + 2 * pad >= 3 && width + 2 * pad >= 3, "stem3x3_s2_raw: %d x %d input gives an empty output", height, width);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(z) & 15) == 0, "stem3x3_s2_raw: z must be 16B aligned");
  const long long total = static_cast<long long>(batch) * ((height + 2 * pad - 3) / 2 + 1) * ((width + 2 * pad - 3) / 2 + 1);
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  if (pad == 0) mb_conv0_kernel<0><<<grid, 256, 0, stream>>>(x, w, w, w, reinterpret_cast<__half*>(z), batch, height, width, 1, 0);
  else mb_conv0_kernel<1><<<grid, 256, 0, stream>>>(x, w, w, w, reinterpret_cast<__half*>(z), batch, height, width, 1, 0);
  return check_launch("mb_conv0_kernel");
}

int stem3x3_s2_wgrad(const float* x, const void* dz, float* dw, int batch, int height, int width, int pad, cudaStream_t stream) {
  YB_REQUIRE(x && dz && dw && batch > 0 && (pad == 0 || pad == 1), "stem3x3_s2_wgrad: bad argument (pad 0 or 1)");
  YB_REQUIRE(height + 2 * pad >= 3 && width + 2 * pad >= 3, "stem3x3_s2_wgrad: %d x %d input gives an empty output", height, width);
  YB_CUDA(cudaMemsetAsync(dw, 0, 32 * 27 * sizeof(float), stream));
  const long long pixels = static_cast<long long>(batch) * ((height + 2 * pad - 3) / 2 + 1) * ((width + 2 * pad - 3) / 2 + 1);
  long long blocks = (pixels + 8 * 32 - 1) / (8 * 32);
  const int cap = sm_count() * 6;
  const int grid = static_cast<int>(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
  if (pad == 0) mb_conv0_wgrad_kernel<0><<<grid, 256, 0, stream>>>(x, reinterpret_cast<const __half*>(dz), dw, batch, height, width);
  else mb_conv0_wgrad_kernel<1><<<grid, 256, 0, stream>>>(x, reinterpret_cast<const __half*>(dz), dw, batch, height, width);
  return check_launch("mb_conv0_wgrad_kernel");
}

}  // namespace yb
