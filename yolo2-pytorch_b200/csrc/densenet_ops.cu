// DenseNet plugin kernels (model/densenet.py of the reference, torchvision's _Transition / features.pool0), inference.
//   bn_relu_avgpool2x2  a transition's norm -> relu -> AvgPool2d(2), with the pooling moved in front of its 1x1 conv: pooling and a
//                       1x1 conv commute in exact arithmetic, and pooling first cuts that conv's work 4x.  The rounding differs from the
//                       reference's order (conv on the full-resolution activation, then pool) by fp32 summation order only.
//   maxpool3x3_s2_ld    nn.MaxPool2d(3, 2, 1) (features.pool0) writing into a channel slice of a wider buffer: the stem's pool lands
//                       directly in channels [0, 64) of the first dense block's buffer, so no concatenation copy follows.
// The dense layers' convs are yb_conv1x1_preact_fwd (norm1 + relu1 + conv1) and yb_conv_bn_act_fwd (conv2); the stem is the
// ResNet stem kernel.
// Training (b200.train_engine.DenseNetTrainer): every norm that reads a block channel shares that channel's batch statistics, so
//   bn_batch_fold       one norm's (pre_scale, pre_shift) from the shared mean / invstd and its own gamma / beta
//   bn_running_update   every norm of a block updates its running statistics from the shared batch mean / variance, in one launch
//   bn_preact_bwd       a pre-activation norm's backward over channels [0, C) of the block buffer, its incoming gradient at full
//                       resolution or through the transition's 2x2 average pool; the apply pass adds dx into the block's fp32 gradient
//                       buffer and rounds the slice that this contribution completes to fp16 in the same pass
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

// ---- training ------------------------------------------------------------------------------------------------------------------------
// The (scale, shift) of a train-mode norm from the shared batch statistics: y = fmaf(sc, x, sh), sc = gamma * invstd, sh = beta - mean * sc
// with one rounding (fmaf).  The forward pre-activation and the backward below both use exactly these values, so the ReLU mask of the
// backward is the forward's.
__device__ __forceinline__ void preact_coef(const float* mean, const float* invstd, const float* gamma, const float* beta, int c, float& sc, float& sh) {
  sc = __fmul_rn(__ldg(gamma + c), __ldg(invstd + c));
  sh = __fmaf_rn(-__ldg(mean + c), sc, __ldg(beta + c));
}

__global__ void bn_batch_fold_kernel(const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, float* __restrict__ scale, float* __restrict__ shift, int channels) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= channels) return;
  float sc, sh;
  preact_coef(mean, invstd, gamma, beta, c, sc, sh);
  scale[c] = sc;
  shift[c] = sh;
}

int bn_batch_fold(const float* mean, const float* invstd, const float* gamma, const float* beta, float* scale, float* shift, int channels,
                  cudaStream_t stream) {
  YB_REQUIRE(mean && invstd && gamma && beta && scale && shift && channels > 0, "bn_batch_fold: bad argument");
  bn_batch_fold_kernel<<<(channels + 255) / 256, 256, 0, stream>>>(mean, invstd, gamma, beta, scale, shift, channels);
  return check_launch("bn_batch_fold_kernel");
}

// Mirror of yb_bn_running (include/yolo2_b200.h).
struct BnRunning {
  float* running_mean;
  float* running_var;
  int channels;
  float momentum;
};
static_assert(sizeof(BnRunning) == 24, "yb_bn_running layout");

// norm k (blockIdx.y) over channels [0, channels_k): running = (1 - momentum_k) * running + momentum_k * batch, in double as yb_bn_finalize
__global__ void bn_running_update_kernel(const float* __restrict__ batch_mean, const float* __restrict__ batch_var, const BnRunning* __restrict__ norms) {
  const BnRunning n = norms[blockIdx.y];
  const double m = static_cast<double>(n.momentum);
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n.channels; c += gridDim.x * blockDim.x) {
    n.running_mean[c] = static_cast<float>((1.0 - m) * n.running_mean[c] + m * batch_mean[c]);
    n.running_var[c] = static_cast<float>((1.0 - m) * n.running_var[c] + m * batch_var[c]);
  }
}

int bn_running_update(const float* batch_mean, const float* batch_var, const void* norms, int count, int max_channels, cudaStream_t stream) {
  YB_REQUIRE(batch_mean && batch_var && norms && count > 0 && count <= 65535 && max_channels > 0, "bn_running_update: bad argument");
  const dim3 grid((max_channels + 255) / 256, count);
  bn_running_update_kernel<<<grid, 256, 0, stream>>>(batch_mean, batch_var, reinterpret_cast<const BnRunning*>(norms));
  return check_launch("bn_running_update_kernel");
}

struct PreBwd {
  const __half* x; long long x_ld;
  const float* mean; const float* invstd; const float* gamma; const float* beta;
  int relu;
  const __half* da; long long da_ld;
  int batch, height, width, channels;
  double* sums;
  float* dx; long long dx_ld;
  __half* dx16; long long dx16_ld; int dx16_ch0;
};

// Backward of one pre-activation norm a = act(fmaf(sc, x, sh)) over channels [0, C) of the block buffer x.  A block covers up to 32 groups
// of 8 channels (blockIdx.y selects which) and 256 / groups pixel rows; every thread keeps its 8 channels for the whole grid-stride loop.
// kPool = 1: the gradient arrives at the output of the transition's AvgPool2d(2): d(a) = 0.25 * da at each of the window's 4 pixels.
// mode 0: sums[0..C) += sum dy, sums[C..2C) += sum dy * xhat.   mode 1: dx += sc * dy - k1 - k2 * xhat (fp32, at dx_ld), and channels
// >= dx16_ch0 also go to dx16 as fp16 (the slice this contribution completes).
template <int kMode, int kPool>
__global__ void __launch_bounds__(256) bn_preact_bwd_kernel(const PreBwd a) {
  __shared__ float s_acc[2][256];
  const int groups = min(32, (a.channels >> 3) - 32 * static_cast<int>(blockIdx.y));
  const int rows = 256 / groups;
  const int lane = threadIdx.x % groups, row = threadIdx.x / groups;
  const int c0 = (32 * static_cast<int>(blockIdx.y) + lane) * 8;
  const float inv_n = 1.f / static_cast<float>(static_cast<long long>(a.batch) * a.height * a.width);
  float sc[8], sh[8], xa[8], xb[8], k1[8], k2[8], acc1[8], acc2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    preact_coef(a.mean, a.invstd, a.gamma, a.beta, c0 + i, sc[i], sh[i]);
    xa[i] = __ldg(a.invstd + c0 + i);
    xb[i] = -__ldg(a.mean + c0 + i) * xa[i];
    k1[i] = kMode == 1 ? sc[i] * (static_cast<float>(a.sums[c0 + i]) * inv_n) : 0.f;
    k2[i] = kMode == 1 ? sc[i] * (static_cast<float>(a.sums[a.channels + c0 + i]) * inv_n) : 0.f;
    acc1[i] = 0.f; acc2[i] = 0.f;
  }
  if (kMode == 0) {
    for (int i = threadIdx.x; i < 512; i += 256) (&s_acc[0][0])[i] = 0.f;
    __syncthreads();
  }
  const bool to16 = kMode == 1 && a.dx16 != nullptr && c0 >= a.dx16_ch0;
  const int oh = kPool ? a.height >> 1 : a.height, ow = kPool ? a.width >> 1 : a.width;
  const long long items = static_cast<long long>(a.batch) * oh * ow;
  if (row < rows) {
    for (long long it = static_cast<long long>(blockIdx.x) * rows + row; it < items; it += static_cast<long long>(gridDim.x) * rows) {
      long long pix0;
      float gpool[8];
      if (kPool) {
        const long long px = it % ow, t = it / ow;
        const long long py = t % oh, img = t / oh;
        pix0 = (img * a.height + 2 * py) * a.width + 2 * px;
        const uint4 g = __ldg(reinterpret_cast<const uint4*>(a.da + it * a.da_ld + c0));
        const __half2* hg = reinterpret_cast<const __half2*>(&g);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __half22float2(hg[i]);
          gpool[2 * i] = 0.25f * f.x; gpool[2 * i + 1] = 0.25f * f.y;
        }
      } else {
        pix0 = it;
      }
#pragma unroll
      for (int q = 0; q < (kPool ? 4 : 1); ++q) {
        const long long pix = kPool ? pix0 + (q >> 1) * a.width + (q & 1) : pix0;
        const uint4 xv = __ldg(reinterpret_cast<const uint4*>(a.x + pix * a.x_ld + c0));
        const __half2* hx = reinterpret_cast<const __half2*>(&xv);
        float g[8];
        if (kPool) {
#pragma unroll
          for (int i = 0; i < 8; ++i) g[i] = gpool[i];
        } else {
          const uint4 dv = __ldg(reinterpret_cast<const uint4*>(a.da + pix * a.da_ld + c0));
          const __half2* hd = reinterpret_cast<const __half2*>(&dv);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = __half22float2(hd[i]);
            g[2 * i] = f.x; g[2 * i + 1] = f.y;
          }
        }
        float out[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __half22float2(hx[i]);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int j = 2 * i + e;
            const float xf = e ? f.y : f.x;
            const float y = __fmaf_rn(sc[j], xf, sh[j]);
            const float dy = (!a.relu || y > 0.f) ? g[j] : 0.f;
            const float xhat = fmaf(xf, xa[j], xb[j]);
            if (kMode == 0) { acc1[j] += dy; acc2[j] = fmaf(dy, xhat, acc2[j]); }
            else out[j] = fmaf(sc[j], dy, -fmaf(k2[j], xhat, k1[j]));
          }
        }
        if (kMode == 1) {
          float4* d = reinterpret_cast<float4*>(a.dx + pix * a.dx_ld + c0);
          float4 v0 = d[0], v1 = d[1];
          v0.x += out[0]; v0.y += out[1]; v0.z += out[2]; v0.w += out[3];
          v1.x += out[4]; v1.y += out[5]; v1.z += out[6]; v1.w += out[7];
          d[0] = v0; d[1] = v1;
          if (to16) {
            uint4 h;
            __half2* hh = reinterpret_cast<__half2*>(&h);
            hh[0] = __floats2half2_rn(v0.x, v0.y); hh[1] = __floats2half2_rn(v0.z, v0.w);
            hh[2] = __floats2half2_rn(v1.x, v1.y); hh[3] = __floats2half2_rn(v1.z, v1.w);
            *reinterpret_cast<uint4*>(a.dx16 + pix * a.dx16_ld + (c0 - a.dx16_ch0)) = h;
          }
        }
      }
    }
  }
  if (kMode == 0) {
    if (row < rows) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        atomicAdd(&s_acc[0][lane * 8 + i], acc1[i]);
        atomicAdd(&s_acc[1][lane * 8 + i], acc2[i]);
      }
    }
    __syncthreads();
    const int base = 256 * static_cast<int>(blockIdx.y);
    for (int i = threadIdx.x; i < groups * 8; i += 256) {
      atomicAdd(&a.sums[base + i], static_cast<double>(s_acc[0][i]));
      atomicAdd(&a.sums[a.channels + base + i], static_cast<double>(s_acc[1][i]));
    }
  }
}

int bn_preact_bwd(int mode, const void* x, long long x_ld, const float* mean, const float* invstd, const float* gamma, const float* beta, int relu,
                  const void* da, long long da_ld, int pool, int batch, int height, int width, int channels, double* sums, float* dx, long long dx_ld,
                  void* dx16, long long dx16_ld, int dx16_ch0, cudaStream_t stream) {
  YB_REQUIRE(x && mean && invstd && gamma && beta && da && sums && (mode == 0 || mode == 1) && (relu == 0 || relu == 1) && (pool == 0 || pool == 1),
             "bn_preact_bwd: bad argument");
  YB_REQUIRE(batch > 0 && height > 0 && width > 0 && channels > 0 && channels % 8 == 0 && x_ld % 8 == 0 && x_ld >= channels && da_ld % 8 == 0 &&
             da_ld >= channels, "bn_preact_bwd: C=%d, x_ld=%lld, da_ld=%lld (multiples of 8, pitches >= C)", channels, x_ld, da_ld);
  YB_REQUIRE(!pool || (height % 2 == 0 && width % 2 == 0), "bn_preact_bwd: the average-pool route needs even H, W");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(da) & 15) == 0, "bn_preact_bwd: x / da must be 16B aligned");
  if (mode == 1) {
    YB_REQUIRE(dx && dx_ld % 4 == 0 && dx_ld >= channels && (reinterpret_cast<uintptr_t>(dx) & 15) == 0, "bn_preact_bwd: dx (16B aligned, dx_ld >= C)");
    YB_REQUIRE(dx16 == nullptr || (dx16_ch0 >= 0 && dx16_ch0 < channels && dx16_ch0 % 8 == 0 && dx16_ld % 8 == 0 && dx16_ld >= channels - dx16_ch0 &&
                                   (reinterpret_cast<uintptr_t>(dx16) & 15) == 0),
               "bn_preact_bwd: dx16 slice [%d, %d) (offset a multiple of 8, dx16_ld >= its width, 16B aligned)", dx16_ch0, channels);
  }
  PreBwd a{reinterpret_cast<const __half*>(x), x_ld, mean, invstd, gamma, beta, relu, reinterpret_cast<const __half*>(da), da_ld, batch, height, width,
           channels, sums, dx, dx_ld, reinterpret_cast<__half*>(dx16), dx16_ld, dx16_ch0};
  const int gy = (channels / 8 + 31) / 32;
  const int groups = channels / 8 < 32 ? channels / 8 : 32;
  const long long items = static_cast<long long>(batch) * (pool ? height / 2 : height) * (pool ? width / 2 : width);
  long long gx = (items + (256 / groups) * 16 - 1) / ((256 / groups) * 16);          // ~16 items per thread: 2C double atomics per block
  const long long cap = (static_cast<long long>(sm_count()) * 8 + gy - 1) / gy;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  const dim3 grid(static_cast<unsigned>(gx), gy);
  if (mode == 0 && pool) bn_preact_bwd_kernel<0, 1><<<grid, 256, 0, stream>>>(a);
  else if (mode == 0) bn_preact_bwd_kernel<0, 0><<<grid, 256, 0, stream>>>(a);
  else if (pool) bn_preact_bwd_kernel<1, 1><<<grid, 256, 0, stream>>>(a);
  else bn_preact_bwd_kernel<1, 0><<<grid, 256, 0, stream>>>(a);
  return check_launch("bn_preact_bwd_kernel");
}

}  // namespace yb
