// Training-mode companions of the conv kernel (HBM-bound, 16-byte vectorised, fp16 NHWC activations):
//   bn_stats / bn_finalize      batch statistics of the raw conv output z and running-stat update
//                               (nn.BatchNorm2d(momentum=0.01) in train mode, model/yolo2.py:58)
//   bn_act_apply                a = leaky(gamma * (z - mean) * invstd + beta) [+ fused MaxPool2d(2)]   (yolo2.py:58-59,79)
//   bn_act_bwd_reduce / _apply  backward of leaky + BN (+ max-pool routing, + a second unpooled gradient for
//                               the passthrough branch point): dgamma, dbeta and dz
//   reorg_bwd, head_grad_prepare, conv0_wgrad, unpack_wgrad
// Everything the reference gets from torch autograd over nn.BatchNorm2d / LeakyReLU / MaxPool2d / reorg / cat.
#include "yb_common.h"
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdlib.h>

namespace yb {

constexpr int kTrainThreads = 256;

__device__ __forceinline__ void h8_to_f(const uint4& v, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h[i]);
    f[2 * i] = t.x; f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 f_to_h8(const float (&f)[8]) {
  uint4 v;
  __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return v;
}

// ------------------------------------------------------------------------------------------------
// sums[0..C) += sum_rows z, sums[C..2C) += sum_rows z^2   (double accumulators, zero on entry).  Each trip's four rows are added in fp32,
// everything after that in double: the fp32 part stays three roundings deep at any row count, which matters because bn_finalize's
// var = sum z^2 / n - mean^2 amplifies the error of the sums by 1 + (mean / std)^2.
__global__ void __launch_bounds__(kTrainThreads) bn_stats_kernel(const __half* __restrict__ z, long long ld, long long rows, int channels,
                                                                 double* __restrict__ sums) {
  extern __shared__ double s_sum[];  // [2][channels]
  for (int i = threadIdx.x; i < 2 * channels; i += blockDim.x) s_sum[i] = 0.0;
  __syncthreads();
  const int c8 = channels >> 3;
  const int cg = threadIdx.x % c8;
  const int rpi = blockDim.x / c8;                 // rows per iteration
  const int rib = threadIdx.x / c8;
  double s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.0; q[i] = 0.0; }
  if (rib < rpi) {
    const long long rstride = static_cast<long long>(gridDim.x) * rpi;
    for (long long r0 = static_cast<long long>(blockIdx.x) * rpi + rib; r0 < rows; r0 += 4 * rstride) {
      uint4 raw[4];                                    // four rows per trip, loads first (latency-bound otherwise)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long r = r0 + u * rstride;
        raw[u] = r < rows ? __ldg(reinterpret_cast<const uint4*>(z + r * ld + cg * 8)) : make_uint4(0u, 0u, 0u, 0u);   // fp16 zeros add nothing
      }
      float ts[8], tq[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) { ts[i] = 0.f; tq[i] = 0.f; }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float f[8];
        h8_to_f(raw[u], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) { ts[i] += f[i]; tq[i] = fmaf(f[i], f[i], tq[i]); }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) { s[i] += static_cast<double>(ts[i]); q[i] += static_cast<double>(tq[i]); }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      atomicAdd(&s_sum[cg * 8 + i], s[i]);
      atomicAdd(&s_sum[channels + cg * 8 + i], q[i]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * channels; i += blockDim.x) atomicAdd(&sums[i], s_sum[i]);
}

// mean/invstd for this batch, running-stat update (unbiased variance, like torch), sums reset to 0
__global__ void bn_finalize_kernel(double* __restrict__ sums, long long rows, int channels, float eps, float momentum,
                                   float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ mean_out,
                                   float* __restrict__ invstd_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= channels) return;
  const double m = sums[c] / static_cast<double>(rows);
  double var = sums[channels + c] / static_cast<double>(rows) - m * m;
  if (var < 0.0) var = 0.0;
  mean_out[c] = static_cast<float>(m);
  invstd_out[c] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  if (running_mean != nullptr) {
    const double unbiased = rows > 1 ? var * static_cast<double>(rows) / static_cast<double>(rows - 1) : var;
    running_mean[c] = static_cast<float>((1.0 - momentum) * running_mean[c] + momentum * m);
    running_var[c] = static_cast<float>((1.0 - momentum) * running_var[c] + momentum * unbiased);
  }
  sums[c] = 0.0;
  sums[channels + c] = 0.0;
}

struct BnParams {
  const float* mean;
  const float* invstd;
  const float* gamma;
  const float* beta;
  float slope;
  int channels;
};

// Per-thread channel constants.  Every thread of these kernels owns the same 8 channels for its whole grid-stride loop
// (blockDim and the total stride are multiples of C/8), so the folded BatchNorm terms live in registers: the loop body
// is ~8 instructions per element (convert, FMA, select, ...) with no shared-memory or index-division traffic, which
// is what lets the kernels run at HBM speed instead of being issue-bound.
struct Ch8 {
  float sc[8], sh[8];   // y = z * sc + sh          (sc = gamma * invstd, sh = beta - mean * sc; 1 / 0 without BN)
};
__device__ __forceinline__ void load_ch8(const BnParams& bn, int cg, bool has_bn, Ch8& k) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = cg * 8 + i;
    if (has_bn) {
      const float sc = __ldg(bn.gamma + c) * __ldg(bn.invstd + c);
      k.sc[i] = sc;
      k.sh[i] = __ldg(bn.beta + c) - __ldg(bn.mean + c) * sc;
    } else {
      k.sc[i] = 1.f; k.sh[i] = 0.f;
    }
  }
}

// a = leaky(scale * z + shift); pool = 1 additionally takes the 2x2 max (thread = 8 channels of one OUTPUT pixel)
template <int kPool>
__global__ void __launch_bounds__(kTrainThreads) bn_act_apply_kernel(const __half* __restrict__ z, long long ld_z, BnParams bn,
                                                                     __half* __restrict__ a, long long ld_a, int a_ch_off, int batch, int height,
                                                                     int width) {
  const unsigned c8 = static_cast<unsigned>(bn.channels) >> 3;
  const unsigned cg = threadIdx.x % c8;
  Ch8 k;
  load_ch8(bn, static_cast<int>(cg), true, k);
  const unsigned oh = kPool ? height >> 1 : height, ow = kPool ? width >> 1 : width;
  const unsigned npix = static_cast<unsigned>(batch) * oh * ow;                 // output pixels (< 2^31, checked on the host)
  const unsigned pstride = gridDim.x * (blockDim.x / c8);
  constexpr int nwin = kPool ? 4 : 1;
  if constexpr (!kPool) {
    // four pixels per trip, loads first: these kernels are latency-bound (see bn_act_bwd_kernel)
    constexpr int U = 4;
    for (unsigned p0 = blockIdx.x * (blockDim.x / c8) + threadIdx.x / c8; p0 < npix; p0 += U * pstride) {
      uint4 raw[U];
      bool ok[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const unsigned q = p0 + u * pstride;
        ok[u] = q < npix;
        raw[u] = __ldg(reinterpret_cast<const uint4*>(z + static_cast<long long>(ok[u] ? q : p0) * ld_z + cg * 8));
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (!ok[u]) continue;
        float f[8], y[8];
        h8_to_f(raw[u], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float v = fmaf(f[i], k.sc[i], k.sh[i]);
          y[i] = v > 0.f ? v : v * bn.slope;
        }
        *reinterpret_cast<uint4*>(a + static_cast<long long>(p0 + u * pstride) * ld_a + a_ch_off + cg * 8) = f_to_h8(y);
      }
    }
  } else
#pragma unroll 2
  for (unsigned p = blockIdx.x * (blockDim.x / c8) + threadIdx.x / c8; p < npix; p += pstride) {
    long long in0;
    if (kPool) {
      const unsigned px = p % ow, t = p / ow;
      const unsigned py = t % oh, img = t / oh;
      in0 = (static_cast<long long>(img) * height + 2 * py) * width + 2 * px;
    } else {
      in0 = p;
    }
    uint4 raw[nwin];
#pragma unroll
    for (int w = 0; w < nwin; ++w)
      raw[w] = __ldg(reinterpret_cast<const uint4*>(z + (in0 + (w >> 1) * width + (w & 1)) * ld_z + cg * 8));
    float best[8];
#pragma unroll
    for (int w = 0; w < nwin; ++w) {
      float f[8];
      h8_to_f(raw[w], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float y = fmaf(f[i], k.sc[i], k.sh[i]);
        y = y > 0.f ? y : y * bn.slope;
        best[i] = (w == 0) ? y : fmaxf(best[i], y);
      }
    }
    *reinterpret_cast<uint4*>(a + static_cast<long long>(p) * ld_a + a_ch_off + cg * 8) = f_to_h8(best);
  }
}

// Gradient arriving at the activated output of one unit: optional unpooled part (da) plus optional part that
// arrives through the unit's 2x2 max-pool (dap, routed to the window's first maximum as torch does).
struct GradIn {
  const __half* da;   long long ld_da;  int da_off;     // [B,H,W,*]
  const __half* dap;  long long ld_dap; int dap_off;    // [B,H/2,W/2,*]
};

// One thread handles 8 channels of one 2x2 window (pool / branch layers) or of one pixel (window = 0).
// mode 0: accumulate sum(dy), sum(dy * xhat) ; mode 1: write dz = sc * (dy - mean(dy) - xhat * mean(dy xhat)).
// kHasDa = 0 (only valid with kWin = 1): the gradient arrives through the max-pool alone, so exactly one pixel of the
// window (the first maximum) has a non-zero dy -- the reduction touches one element per window and the dz of the
// other three is just -(k1 + k2 * xhat): about a third of the instructions of the general path.
template <int kMode, int kWin, int kHasDa>
__global__ void __launch_bounds__(kTrainThreads) bn_act_bwd_kernel(const __half* __restrict__ z, long long ld_z, BnParams bn, GradIn g, int batch,
                                                                   int height, int width, double* __restrict__ sums,
                                                                   __half* __restrict__ dz, long long ld_dz, int has_bn) {
  constexpr int nwin = kWin ? 4 : 1;
  extern __shared__ float s_acc[];                // mode 0: [2][C] block accumulators
  const unsigned c8 = static_cast<unsigned>(bn.channels) >> 3;
  const unsigned cg = threadIdx.x % c8;
  const float inv_rows = 1.f / static_cast<float>(static_cast<long long>(batch) * height * width);
  Ch8 k;
  load_ch8(bn, static_cast<int>(cg), has_bn != 0, k);
  float xa[8], xb[8];                             // xhat = z * xa + xb
  float k1[8], k2[8];                             // mode 1: dz = sc * dy - k1 - k2 * xhat
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = static_cast<int>(cg) * 8 + i;
    if (has_bn) {
      xa[i] = __ldg(bn.invstd + c);
      xb[i] = -__ldg(bn.mean + c) * xa[i];
    } else {
      xa[i] = 0.f; xb[i] = 0.f;
    }
    if (kMode == 1 && has_bn) {
      k1[i] = k.sc[i] * (static_cast<float>(sums[c]) * inv_rows);
      k2[i] = k.sc[i] * (static_cast<float>(sums[bn.channels + c]) * inv_rows);
    } else {
      k1[i] = 0.f; k2[i] = 0.f;
    }
  }
  if (kMode == 0) {
    for (int i = threadIdx.x; i < 2 * bn.channels; i += blockDim.x) s_acc[i] = 0.f;
    __syncthreads();
  }
  const unsigned oh = kWin ? height >> 1 : height, ow = kWin ? width >> 1 : width;
  const unsigned npix = static_cast<unsigned>(batch) * oh * ow;
  const unsigned pstride = gridDim.x * (blockDim.x / c8);
  float acc1[8], acc2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { acc1[i] = 0.f; acc2[i] = 0.f; }
  if constexpr (!kWin) {
    // ---- plain units (no pooling window; the gradient is `da`): four pixels per trip, all eight 16-byte loads issued
    // before any arithmetic -- the kernel is latency-bound, not issue-bound, so memory-level parallelism is what counts
    constexpr int U = 4;
    for (unsigned p0 = blockIdx.x * (blockDim.x / c8) + threadIdx.x / c8; p0 < npix; p0 += U * pstride) {
      uint4 zr[U], dr[U];
      bool ok[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const unsigned q = p0 + u * pstride;
        ok[u] = q < npix;
        const long long pix = ok[u] ? q : p0;
        zr[u] = __ldg(reinterpret_cast<const uint4*>(z + pix * ld_z + cg * 8));
        dr[u] = __ldg(reinterpret_cast<const uint4*>(g.da + pix * g.ld_da + g.da_off + cg * 8));
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (!ok[u]) continue;
        float zf[8], gd[8], out[8];
        h8_to_f(zr[u], zf);
        h8_to_f(dr[u], gd);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float y = fmaf(zf[i], k.sc[i], k.sh[i]);
          const float dy = y > 0.f ? gd[i] : gd[i] * bn.slope;
          const float xhat = fmaf(zf[i], xa[i], xb[i]);
          if (kMode == 0) { acc1[i] += dy; acc2[i] = fmaf(dy, xhat, acc2[i]); }
          else out[i] = fmaf(k.sc[i], dy, -fmaf(k2[i], xhat, k1[i]));
        }
        if (kMode == 1) *reinterpret_cast<uint4*>(dz + static_cast<long long>(p0 + u * pstride) * ld_dz + cg * 8) = f_to_h8(out);
      }
    }
  } else
#pragma unroll 1
  for (unsigned p = blockIdx.x * (blockDim.x / c8) + threadIdx.x / c8; p < npix; p += pstride) {
    long long in0;
    if (kWin) {
      const unsigned px = p % ow, t = p / ow;
      const unsigned py = t % oh, img = t / oh;
      in0 = (static_cast<long long>(img) * height + 2 * py) * width + 2 * px;
    } else {
      in0 = p;
    }
    // all loads of this item first (memory-level parallelism), then the math
    uint4 zr[nwin], dr[nwin], pr = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int w = 0; w < nwin; ++w) {
      const long long pix = in0 + (w >> 1) * width + (w & 1);
      zr[w] = __ldg(reinterpret_cast<const uint4*>(z + pix * ld_z + cg * 8));
      if (kHasDa) dr[w] = (g.da != nullptr) ? __ldg(reinterpret_cast<const uint4*>(g.da + pix * g.ld_da + g.da_off + cg * 8)) : make_uint4(0u, 0u, 0u, 0u);
    }
    if (g.dap != nullptr) pr = __ldg(reinterpret_cast<const uint4*>(g.dap + static_cast<long long>(p) * g.ld_dap + g.dap_off + cg * 8));
    float gp[8];
    h8_to_f(pr, gp);
    if constexpr (!kHasDa) {
      // ---- pooled gradient only: one live element per window and channel ----
      float zf[nwin][8];
#pragma unroll
      for (int w = 0; w < nwin; ++w) h8_to_f(zr[w], zf[w]);
      float dyb[8];
      int arg[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float besty = fmaf(zf[0][i], k.sc[i], k.sh[i]);
        float bestz = zf[0][i];
        arg[i] = 0;
#pragma unroll
        for (int w = 1; w < nwin; ++w) {
          const float y = fmaf(zf[w][i], k.sc[i], k.sh[i]);
          if (y > besty) { besty = y; bestz = zf[w][i]; arg[i] = w; }   // first maximum wins (leaky is strictly increasing)
        }
        dyb[i] = besty > 0.f ? gp[i] : gp[i] * bn.slope;
        if (kMode == 0) {
          acc1[i] += dyb[i];
          acc2[i] = fmaf(dyb[i], fmaf(bestz, xa[i], xb[i]), acc2[i]);
        }
      }
      if (kMode == 1) {
#pragma unroll
        for (int w = 0; w < nwin; ++w) {
          float out[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float base = -fmaf(k2[i], fmaf(zf[w][i], xa[i], xb[i]), k1[i]);
            out[i] = arg[i] == w ? fmaf(k.sc[i], dyb[i], base) : base;
          }
          *reinterpret_cast<uint4*>(dz + (in0 + (w >> 1) * width + (w & 1)) * ld_dz + cg * 8) = f_to_h8(out);
        }
      }
    } else {
    float zf[nwin][8], yv[nwin][8];
    int arg[8];
#pragma unroll
    for (int w = 0; w < nwin; ++w) {
      h8_to_f(zr[w], zf[w]);
#pragma unroll
      for (int i = 0; i < 8; ++i) yv[w][i] = fmaf(zf[w][i], k.sc[i], k.sh[i]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      arg[i] = 0;
      if (kWin) {
        float besty = yv[0][i];
#pragma unroll
        for (int w = 1; w < nwin; ++w)
          if (yv[w][i] > besty) { besty = yv[w][i]; arg[i] = w; }      // first maximum wins (leaky is strictly increasing)
      }
    }
#pragma unroll
    for (int w = 0; w < nwin; ++w) {
      float gd[8], out[8];
      h8_to_f(dr[w], gd);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float gin = gd[i];
        if (!kWin || arg[i] == w) gin += gp[i];          // gp is zero when there is no pooled gradient
        const float dy = yv[w][i] > 0.f ? gin : gin * bn.slope;
        const float xhat = fmaf(zf[w][i], xa[i], xb[i]);
        if (kMode == 0) { acc1[i] += dy; acc2[i] = fmaf(dy, xhat, acc2[i]); }
        else out[i] = fmaf(k.sc[i], dy, -fmaf(k2[i], xhat, k1[i]));
      }
      if (kMode == 1) *reinterpret_cast<uint4*>(dz + (in0 + (w >> 1) * width + (w & 1)) * ld_dz + cg * 8) = f_to_h8(out);
    }
    }
  }
  if (kMode == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      atomicAdd(&s_acc[cg * 8 + i], acc1[i]);
      atomicAdd(&s_acc[bn.channels + cg * 8 + i], acc2[i]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * bn.channels; i += blockDim.x) atomicAdd(&sums[i], static_cast<double>(s_acc[i]));
  }
}

// dgamma = scale * sum(dy xhat), dbeta = scale * sum(dy)  (fp32 parameter gradients; scale = 1 / loss scale) ; optionally reset the accumulators
__global__ void bn_param_grad_kernel(double* __restrict__ sums, int channels, float* __restrict__ dgamma, float* __restrict__ dbeta, int reset,
                                     float scale) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= channels) return;
  if (dbeta) dbeta[c] = static_cast<float>(sums[c] * static_cast<double>(scale));
  if (dgamma) dgamma[c] = static_cast<float>(sums[channels + c] * static_cast<double>(scale));
  if (reset) { sums[c] = 0.0; sums[channels + c] = 0.0; }
}

static int grid_for(long long work_items, int items_per_thread = 1) {
  long long blocks = (work_items + static_cast<long long>(kTrainThreads) * items_per_thread - 1) / (static_cast<long long>(kTrainThreads) * items_per_thread);
  const long long cap = static_cast<long long>(sm_count()) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

// keep cg = threadIdx % c8 constant along the grid stride: total stride must be a multiple of c8
static int grid_for_groups(long long work_items, int c8) {
  static const int items = getenv("YB_BN_ITEMS") ? atoi(getenv("YB_BN_ITEMS")) : 16;   // tuning knob (tools): work items per thread
  int g = grid_for(work_items, items > 0 ? items : 16);    // every block pays ~50 parameter loads per thread and 2C global double atomics
  (void)c8;  // blockDim (256) is a multiple of every supported c8 (4..256), so any grid size works
  return g;
}

int bn_stats(const void* z, long long ld, long long rows, int channels, double* sums, cudaStream_t stream) {
  YB_REQUIRE(z && sums && rows > 0 && channels >= 8 && channels % 8 == 0 && channels <= 2048 && kTrainThreads % (channels / 8) == 0 && ld % 8 == 0,
             "bn_stats: unsupported shape (C=%d)", channels);
  const int rpi = kTrainThreads / (channels / 8);
  long long blocks = (rows + static_cast<long long>(rpi) * 16 - 1) / (static_cast<long long>(rpi) * 16);   // >= 16 rows per thread: 2C double atomics per block
  const long long cap = static_cast<long long>(sm_count()) * 8;
  if (blocks > cap) blocks = cap;
  bn_stats_kernel<<<static_cast<int>(blocks), kTrainThreads, 2 * channels * sizeof(double), stream>>>(reinterpret_cast<const __half*>(z), ld, rows,
                                                                                                  channels, sums);
  return check_launch("bn_stats_kernel");
}

int bn_finalize(double* sums, long long rows, int channels, float eps, float momentum, float* running_mean, float* running_var, float* mean,
                float* invstd, cudaStream_t stream) {
  YB_REQUIRE(sums && mean && invstd && rows > 0 && channels > 0, "bn_finalize: bad argument");
  bn_finalize_kernel<<<(channels + 127) / 128, 128, 0, stream>>>(sums, rows, channels, eps, momentum, running_mean, running_var, mean, invstd);
  return check_launch("bn_finalize_kernel");
}

int bn_act_apply(const void* z, long long ld_z, const float* mean, const float* invstd, const float* gamma, const float* beta, float slope,
                 void* a, long long ld_a, int a_ch_off, int batch, int height, int width, int channels, int pool, cudaStream_t stream) {
  YB_REQUIRE(z && mean && invstd && gamma && beta && a && channels % 8 == 0 && channels <= 2048 && ld_z % 8 == 0 && ld_a % 8 == 0 && a_ch_off % 8 == 0,
             "bn_act_apply: bad argument");
  YB_REQUIRE(!pool || (height % 2 == 0 && width % 2 == 0), "bn_act_apply: pooling needs even H, W");
  BnParams bn{mean, invstd, gamma, beta, slope, channels};
  YB_REQUIRE(kTrainThreads % (channels / 8) == 0, "bn_act_apply: C/8 must divide %d (C=%d)", kTrainThreads, channels);
  const long long total = static_cast<long long>(batch) * (pool ? height / 2 : height) * (pool ? width / 2 : width) * (channels / 8);
  YB_REQUIRE(total / (channels / 8) < (1ll << 31), "bn_act_apply: too many pixels");
  if (pool) bn_act_apply_kernel<1><<<grid_for(total), kTrainThreads, 0, stream>>>(reinterpret_cast<const __half*>(z), ld_z, bn, reinterpret_cast<__half*>(a),
                                                                                 ld_a, a_ch_off, batch, height, width);
  else bn_act_apply_kernel<0><<<grid_for(total), kTrainThreads, 0, stream>>>(reinterpret_cast<const __half*>(z), ld_z, bn, reinterpret_cast<__half*>(a), ld_a,
                                                                            a_ch_off, batch, height, width);
  return check_launch("bn_act_apply_kernel");
}

// mode 0: reduce into sums ; mode 1: write dz.  has_bn = 0: plain leaky/bias unit (mean..beta may be null).
int bn_act_bwd(int mode, const void* z, long long ld_z, const float* mean, const float* invstd, const float* gamma, const float* beta,
               float slope, const void* da, long long ld_da, int da_off, const void* dap, long long ld_dap, int dap_off, int batch, int height,
               int width, int channels, int window, double* sums, void* dz, long long ld_dz, int has_bn, cudaStream_t stream) {
  YB_REQUIRE(z && sums && (da || dap) && channels % 8 == 0 && channels <= 2048 && kTrainThreads % (channels / 8) == 0, "bn_act_bwd: bad argument (C=%d)", channels);
  YB_REQUIRE(!has_bn || (mean && invstd && gamma && beta), "bn_act_bwd: BN parameters missing");
  YB_REQUIRE(mode == 0 || dz != nullptr, "bn_act_bwd: dz missing");
  YB_REQUIRE(!window || (height % 2 == 0 && width % 2 == 0), "bn_act_bwd: window mode needs even H, W");
  YB_REQUIRE(dap == nullptr || window, "bn_act_bwd: a pooled gradient needs window mode");
  BnParams bn{mean, invstd, gamma, beta, slope, channels};
  GradIn g{reinterpret_cast<const __half*>(da), ld_da, da_off, reinterpret_cast<const __half*>(dap), ld_dap, dap_off};
  const long long total = static_cast<long long>(batch) * (window ? height / 2 : height) * (window ? width / 2 : width) * (channels / 8);
  YB_REQUIRE(total / (channels / 8) < (1ll << 31), "bn_act_bwd: too many pixels");
  const int grid = grid_for_groups(total, channels / 8);
  const size_t smem = mode == 0 ? 2 * channels * sizeof(float) : 0;
  const __half* zp = reinterpret_cast<const __half*>(z);
  __half* dzp = reinterpret_cast<__half*>(dz);
  const bool pooled_only = window && da == nullptr;
  if (mode == 0 && pooled_only) bn_act_bwd_kernel<0, 1, 0><<<grid, kTrainThreads, smem, stream>>>(zp, ld_z, bn, g, batch, height, width, sums, nullptr, 0, has_bn);
  else if (mode == 0 && window) bn_act_bwd_kernel<0, 1, 1><<<grid, kTrainThreads, smem, stream>>>(zp, ld_z, bn, g, batch, height, width, sums, nullptr, 0, has_bn);
  else if (mode == 0) bn_act_bwd_kernel<0, 0, 1><<<grid, kTrainThreads, smem, stream>>>(zp, ld_z, bn, g, batch, height, width, sums, nullptr, 0, has_bn);
  else if (pooled_only) bn_act_bwd_kernel<1, 1, 0><<<grid, kTrainThreads, smem, stream>>>(zp, ld_z, bn, g, batch, height, width, sums, dzp, ld_dz, has_bn);
  else if (window) bn_act_bwd_kernel<1, 1, 1><<<grid, kTrainThreads, smem, stream>>>(zp, ld_z, bn, g, batch, height, width, sums, dzp, ld_dz, has_bn);
  else bn_act_bwd_kernel<1, 0, 1><<<grid, kTrainThreads, smem, stream>>>(zp, ld_z, bn, g, batch, height, width, sums, dzp, ld_dz, has_bn);
  return check_launch("bn_act_bwd_kernel");
}

int bn_param_grad(double* sums, int channels, float* dgamma, float* dbeta, int reset, float scale, cudaStream_t stream) {
  YB_REQUIRE(sums && channels > 0, "bn_param_grad: bad argument");
  bn_param_grad_kernel<<<(channels + 127) / 128, 128, 0, stream>>>(sums, channels, dgamma, dbeta, reset, scale);
  return check_launch("bn_param_grad_kernel");
}

// ------------------------------------------------------------------------------------------------
// reorg backward: d_in[b, 2h'+sh, 2w'+sw, c] = d_out[b, h', w', off + (sh*2+sw)*C + c]
__global__ void reorg_bwd_kernel(const __half* __restrict__ dy, long long ld_dy, int dy_off, __half* __restrict__ dx, int batch, int height, int width,
                                 int channels) {
  const int c8 = channels >> 3;
  const int oh = height >> 1, ow = width >> 1;
  const long long total = static_cast<long long>(batch) * oh * ow * 4 * c8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int off = static_cast<int>(t % 4); t /= 4;
  const int px = static_cast<int>(t % ow); t /= ow;
  const int py = static_cast<int>(t % oh);
  const int img = static_cast<int>(t / oh);
  const uint4 v = __ldg(reinterpret_cast<const uint4*>(dy + ((static_cast<long long>(img) * oh + py) * ow + px) * ld_dy + dy_off + off * channels + cg * 8));
  *reinterpret_cast<uint4*>(dx + ((static_cast<long long>(img) * height + 2 * py + (off >> 1)) * width + 2 * px + (off & 1)) * channels + cg * 8) = v;
}

int reorg_bwd(const void* dy, long long ld_dy, int dy_off, void* dx, int batch, int height, int width, int channels, cudaStream_t stream) {
  YB_REQUIRE(dy && dx && batch > 0 && height % 2 == 0 && width % 2 == 0 && channels % 8 == 0 && ld_dy % 8 == 0 && dy_off % 8 == 0, "reorg_bwd: bad argument");
  const long long total = static_cast<long long>(batch) * (height / 2) * (width / 2) * 4 * (channels / 8);
  reorg_bwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(dy), ld_dy, dy_off,
                                                                                   reinterpret_cast<__half*>(dx), batch, height, width, channels);
  return check_launch("reorg_bwd_kernel");
}

// ------------------------------------------------------------------------------------------------
// Head gradient: dfeature fp32 NCHW [B,C,S,S] -> fp16 NHWC [B,S,S,Cpad] (zero padded) and bias gradient db[C]
__global__ void head_grad_kernel(const float* __restrict__ df, __half* __restrict__ dz, float* __restrict__ dbias, int batch, int channels, int cpad,
                                 int cells) {
  // block = one channel; threads stride over (b, cell)
  const int c = blockIdx.x;
  float acc = 0.f;
  const long long n = static_cast<long long>(batch) * cells;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const long long b = i / cells, cell = i - b * cells;
    float v = 0.f;
    if (c < channels) { v = df[(b * channels + c) * cells + cell]; acc += v; }
    dz[i * cpad + c] = __float2half_rn(v);
  }
  __shared__ float red[32];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0 && c < channels && dbias != nullptr) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x + 31) / 32; ++w) t += red[w];
    dbias[c] = t;
  }
}

int head_grad_prepare(const float* dfeature, void* dz, float* dbias, int batch, int channels, int cpad, int cells, cudaStream_t stream) {
  YB_REQUIRE(dfeature && dz && batch > 0 && channels > 0 && cpad >= channels && cpad % 8 == 0, "head_grad_prepare: bad argument");
  head_grad_kernel<<<cpad, 256, 0, stream>>>(dfeature, reinterpret_cast<__half*>(dz), dbias, batch, channels, cpad, cells);
  return check_launch("head_grad_kernel");
}

// ------------------------------------------------------------------------------------------------
// conv0 weight gradient: dW[co][ci][r][s] = sum_{b,y,x} dz[b,y,x,co] * x[b,ci,y+r-1,x+s-1]   (Cout = 32, Cin = 3)
// A [27 taps (padded to 32) x pixels] x [pixels x 32 co] product with the pixels as the reduction dimension.  K = 27 is
// far too thin for a wgmma tile, and the op is HBM-bound (709 MB of dz at batch 64), so this uses warp-level
// mma.sync.m16n8k16 (fp16 in, fp32 accumulate): persistent blocks over 8x32-pixel tiles, the haloed fp32 input patch
// and the fp16 dz tile staged in shared memory; warp w owns image row w of the tile (2 K-steps of 16 pixels), builds
// the tap-major A fragments from the patch (two adjacent pixels -> one half2 register) and reads the dz fragments
// with ldmatrix.trans.  Each warp keeps the whole 32 x 32 result in 32 fp32 registers per thread until the end.
constexpr int kW0Rows = 8, kW0Cols = 32;
constexpr int kW0DzStride = 40;      // halves per staged dz pixel row (32 + 8 pad: conflict-free ldmatrix)

__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gmem_src, bool valid) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  const int n = valid ? 4 : 0;                                   // src-size 0: the 4 destination bytes are zero-filled
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(gmem_src), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gmem_src) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}

struct W0Smem {
  float patch[2][3][kW0Rows + 2][kW0Cols + 2];
  __align__(16) __half dzs[2][kW0Rows * kW0Cols][kW0DzStride];
  float s_dw[32 * 32];            // [tap (padded)][co]
};
// fused form: dz is never in memory.  The staged tile holds the raw conv output z; the gradient arriving through the unit's 2x2 max-pool
// (one 64-byte row per window) is staged next to it and the BatchNorm + leaky + pool backward (bn_act_bwd_kernel<1, 1, 0>'s arithmetic)
// turns z into dz in place, in shared memory, before the tensor-core pass.
struct W0SmemFused {
  W0Smem base;
  __align__(16) __half dap[2][(kW0Rows / 2) * (kW0Cols / 2)][32];
  float k[6][32];                 // sc, sh, xa, xb, k1, k2 per channel
};
struct W0Fuse {
  const __half* z;                // [B,H,W,32] raw conv output of the forward pass
  const __half* dap; long long ld_dap; int dap_off;     // [B,H/2,W/2,*] gradient of the pooled activation
  const float *mean, *invstd, *gamma, *beta;
  float slope;
  const double* sums;             // pass-1 sums of this unit (sum dy, sum dy * xhat)
};

template <bool kFused>
__global__ void __launch_bounds__(256, kFused ? 3 : 1) conv0_wgrad_kernel(const float* __restrict__ x, const __half* __restrict__ dz, float* __restrict__ dw, int batch,
                                                          int height, int width, int tiles_x, int tiles_y, int num_tiles, const W0Fuse fz) {
  extern __shared__ __align__(16) uint8_t w0_raw[];
  W0Smem& sm = *reinterpret_cast<W0Smem*>(w0_raw);
  W0SmemFused& smf = *reinterpret_cast<W0SmemFused*>(w0_raw);       // only touched when kFused
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  for (int i = tid; i < 32 * 32; i += 256) sm.s_dw[i] = 0.f;
  if (kFused) {
    if (tid < 32) {
      const float inv_rows = 1.f / static_cast<float>(static_cast<long long>(batch) * height * width);
      const float istd = __ldg(fz.invstd + tid), sc = __ldg(fz.gamma + tid) * istd, mu = __ldg(fz.mean + tid);
      smf.k[0][tid] = sc;
      smf.k[1][tid] = __ldg(fz.beta + tid) - mu * sc;
      smf.k[2][tid] = istd;
      smf.k[3][tid] = -mu * istd;
      smf.k[4][tid] = sc * (static_cast<float>(fz.sums[tid]) * inv_rows);
      smf.k[5][tid] = sc * (static_cast<float>(fz.sums[32 + tid]) * inv_rows);
    }
    dz = fz.z;                     // the staged tile starts as z
  }
  float acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
  // A-fragment rows of this thread: taps g, g+8, g+16, g+24 -> patch plane / row / column offsets (tap >= 27: zero)
  int a_off[4];
  bool a_ok[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int tap = g + 8 * j;
    a_ok[j] = tap < 27;
    const int tc = a_ok[j] ? tap / 9 : 0, tr = a_ok[j] ? (tap % 9) / 3 : 0, ts = a_ok[j] ? tap % 3 : 0;
    a_off[j] = (tc * (kW0Rows + 2) + warp + tr) * (kW0Cols + 2) + ts;
  }
  // ldmatrix.x4.trans row addresses: matrix j = lane >> 3: K-half (j & 1), co block (j >> 1) (+2 for the second load)
  const int lm_row = (lane & 7) + ((lane >> 3) & 1) * 8;
  const int lm_col = (lane >> 4) * 8;

  // stage one tile (haloed fp32 patch + fp16 dz tile) into buffer `buf` with cp.async: the copy of tile i+1 overlaps the
  // tensor-core work on tile i
  auto stage = [&](int tile, int buf) {
    const int tx = tile % tiles_x;
    const int t2 = tile / tiles_x;
    const int ty = t2 % tiles_y;
    const int img = t2 / tiles_y;
    const int y0 = ty * kW0Rows, x0 = tx * kW0Cols;
    for (int i = tid; i < 3 * (kW0Rows + 2) * (kW0Cols + 2); i += 256) {
      const int c = i / ((kW0Rows + 2) * (kW0Cols + 2));
      const int rem = i - c * ((kW0Rows + 2) * (kW0Cols + 2));
      const int r = rem / (kW0Cols + 2), col = rem - r * (kW0Cols + 2);
      const int iy = y0 - 1 + r, ix = x0 - 1 + col;
      const bool ok = iy >= 0 && iy < height && ix >= 0 && ix < width;
      const float* src = x + ((static_cast<long long>(img) * 3 + c) * height + (ok ? iy : 0)) * width + (ok ? ix : 0);
      cp_async_4(&sm.patch[buf][c][r][col], src, ok);
    }
    for (int i = tid; i < kW0Rows * kW0Cols * 4; i += 256) {        // 4 x 16 B per pixel
      const int pix = i >> 2, part = i & 3;
      const int py = pix / kW0Cols, pxx = pix % kW0Cols;
      cp_async_16(&sm.dzs[buf][pix][part * 8], dz + ((static_cast<long long>(img) * height + y0 + py) * width + x0 + pxx) * 32 + part * 8);
    }
    if (kFused) {                                                    // one 16-byte piece per thread: 64 windows x 4
      const int win = tid >> 2, part = tid & 3;
      const int wy = win / (kW0Cols / 2), wx = win % (kW0Cols / 2);
      cp_async_16(&smf.dap[buf][win][part * 8],
                  fz.dap + ((static_cast<long long>(img) * (height >> 1) + (y0 >> 1) + wy) * (width >> 1) + (x0 >> 1) + wx) * fz.ld_dap + fz.dap_off + part * 8);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  int buf = 0;
  if (static_cast<int>(blockIdx.x) < num_tiles) stage(blockIdx.x, 0);
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int next = tile + gridDim.x;
    if (next < num_tiles) {
      stage(next, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    if (kFused) {
      // thread = 8 channels (cg) of one pool window: z -> dz in place (first maximum takes the pooled gradient, as torch routes it)
      const int win = tid >> 2, cg = tid & 3;
      const int wy = win / (kW0Cols / 2), wx = win % (kW0Cols / 2);
      float zf[4][8], gp[8];
      __half* zp[4];
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        zp[w] = &sm.dzs[buf][(2 * wy + (w >> 1)) * kW0Cols + 2 * wx + (w & 1)][cg * 8];
        h8_to_f(*reinterpret_cast<const uint4*>(zp[w]), zf[w]);
      }
      h8_to_f(*reinterpret_cast<const uint4*>(&smf.dap[buf][win][cg * 8]), gp);
      // per channel: which pixel of the window holds the maximum (2 bits each), and the routed gradient times sc (kept in gp)
      uint32_t argbits = 0u;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = cg * 8 + i;
        const float sc = smf.k[0][c], sh = smf.k[1][c];
        float besty = fmaf(zf[0][i], sc, sh);
        uint32_t arg = 0u;
#pragma unroll
        for (int w = 1; w < 4; ++w) {
          const float y = fmaf(zf[w][i], sc, sh);
          if (y > besty) { besty = y; arg = static_cast<uint32_t>(w); }
        }
        argbits |= arg << (2 * i);
        gp[i] = sc * (besty > 0.f ? gp[i] : gp[i] * fz.slope);
      }
      // one pixel at a time (keeps the live registers low: this kernel wants three blocks per SM)
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        float out[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = cg * 8 + i;
          const float base = -fmaf(smf.k[5][c], fmaf(zf[w][i], smf.k[2][c], smf.k[3][c]), smf.k[4][c]);
          out[i] = ((argbits >> (2 * i)) & 3u) == static_cast<uint32_t>(w) ? gp[i] + base : base;
        }
        *reinterpret_cast<uint4*>(zp[w]) = f_to_h8(out);
      }
      __syncthreads();
    }
    const float* pflat = &sm.patch[buf][0][0][0];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      // B fragments (dz): b[n-tile][0..1]
      uint32_t bfr[4][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t addr = static_cast<uint32_t>(__cvta_generic_to_shared(&sm.dzs[buf][warp * kW0Cols + ks * 16 + lm_row][h * 16 + lm_col]));
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                     : "=r"(bfr[2 * h][0]), "=r"(bfr[2 * h][1]), "=r"(bfr[2 * h + 1][0]), "=r"(bfr[2 * h + 1][1]) : "r"(addr));
      }
      // A fragments (taps x pixels) from the fp32 patch
      const int k0 = ks * 16 + t * 2;
      uint32_t afr[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int j0 = 2 * mt, j1 = 2 * mt + 1;       // rows g + 16 mt and g + 16 mt + 8
        const float* r0 = pflat + a_off[j0] + k0;
        const float* r1 = pflat + a_off[j1] + k0;
        afr[mt][0] = a_ok[j0] ? pack_h2(r0[0], r0[1]) : 0u;
        afr[mt][1] = a_ok[j1] ? pack_h2(r1[0], r1[1]) : 0u;
        afr[mt][2] = a_ok[j0] ? pack_h2(r0[8], r0[9]) : 0u;
        afr[mt][3] = a_ok[j1] ? pack_h2(r1[8], r1[9]) : 0u;
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
          asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                       : "+f"(acc[mt][nt][0]), "+f"(acc[mt][nt][1]), "+f"(acc[mt][nt][2]), "+f"(acc[mt][nt][3])
                       : "r"(afr[mt][0]), "r"(afr[mt][1]), "r"(afr[mt][2]), "r"(afr[mt][3]), "r"(bfr[nt][0]), "r"(bfr[nt][1]));
    }
    __syncthreads();                 // everyone is done with `buf` before the next iteration's prefetch overwrites it
    buf ^= 1;
  }
  __syncthreads();
  // D fragment: (row g, cols 2t, 2t+1), (row g + 8, same cols) of each 16 x 8 tile
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int r0 = mt * 16 + g, c0 = nt * 8 + t * 2;
      atomicAdd(&sm.s_dw[r0 * 32 + c0], acc[mt][nt][0]);
      atomicAdd(&sm.s_dw[r0 * 32 + c0 + 1], acc[mt][nt][1]);
      atomicAdd(&sm.s_dw[(r0 + 8) * 32 + c0], acc[mt][nt][2]);
      atomicAdd(&sm.s_dw[(r0 + 8) * 32 + c0 + 1], acc[mt][nt][3]);
    }
  __syncthreads();
  for (int i = tid; i < 27 * 32; i += 256) {
    const int k = i / 32, co = i % 32;                 // k = ci*9 + r*3 + s  -> OIHW flat index co*27 + k
    atomicAdd(&dw[co * 27 + k], sm.s_dw[i]);
  }
}

static int conv0_wgrad_launch(const float* x, const void* dz, float* dw, int batch, int height, int width, const W0Fuse* fz, cudaStream_t stream) {
  YB_REQUIRE(x && dw && batch > 0 && height % kW0Rows == 0 && width % kW0Cols == 0, "conv0_wgrad: H %% 8 == 0 and W %% 32 == 0 required");
  YB_CUDA(cudaMemsetAsync(dw, 0, 27 * 32 * sizeof(float), stream));
  const int tiles_x = width / kW0Cols, tiles_y = height / kW0Rows;
  const long long tiles = static_cast<long long>(tiles_x) * tiles_y * batch;
  static int resident[2] = {0, 0};               // persistent blocks: exactly what fits (a partial second wave would double the time)
  const int fused = fz != nullptr;
  const int smem = static_cast<int>(fused ? sizeof(W0SmemFused) : sizeof(W0Smem));
  if (resident[fused] == 0) {
    if (fused) {
      YB_CUDA(cudaFuncSetAttribute(conv0_wgrad_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      YB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident[1], conv0_wgrad_kernel<true>, 256, smem));
    } else {
      YB_CUDA(cudaFuncSetAttribute(conv0_wgrad_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      YB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident[0], conv0_wgrad_kernel<false>, 256, smem));
    }
    if (resident[fused] < 1) resident[fused] = 1;
  }
  const int cap = sm_count() * resident[fused];
  const int grid = tiles < cap ? static_cast<int>(tiles) : cap;
  if (fused)
    conv0_wgrad_kernel<true><<<grid, 256, smem, stream>>>(x, nullptr, dw, batch, height, width, tiles_x, tiles_y, static_cast<int>(tiles), *fz);
  else
    conv0_wgrad_kernel<false><<<grid, 256, smem, stream>>>(x, reinterpret_cast<const __half*>(dz), dw, batch, height, width, tiles_x, tiles_y,
                                                          static_cast<int>(tiles), W0Fuse{});
  return check_launch("conv0_wgrad_kernel");
}

int conv0_wgrad(const float* x, const void* dz, float* dw, int batch, int height, int width, cudaStream_t stream) {
  YB_REQUIRE(dz, "conv0_wgrad: dz missing");
  return conv0_wgrad_launch(x, dz, dw, batch, height, width, nullptr, stream);
}

// Weight gradient of the first layer with the BatchNorm + leaky + 2x2 max-pool backward of that layer fused in (second pass: `sums` already
// holds sum dy, sum dy * xhat from bn_act_bwd mode 0): reads z and the pooled gradient, never writes dz (no data gradient is needed for the image).
int conv0_wgrad_bn(const float* x, const void* z, const void* dap, long long ld_dap, int dap_off, const float* mean, const float* invstd,
                   const float* gamma, const float* beta, float slope, const double* sums, float* dw, int batch, int height, int width,
                   cudaStream_t stream) {
  YB_REQUIRE(z && dap && mean && invstd && gamma && beta && sums && ld_dap >= 32 && ld_dap % 8 == 0 && dap_off % 8 == 0, "conv0_wgrad_bn: bad argument");
  W0Fuse fz{reinterpret_cast<const __half*>(z), reinterpret_cast<const __half*>(dap), ld_dap, dap_off, mean, invstd, gamma, beta, slope, sums};
  return conv0_wgrad_launch(x, nullptr, dw, batch, height, width, &fz, stream);
}

// ------------------------------------------------------------------------------------------------
// fp32 [Cout][k][k][Cin] (the wgrad kernel's accumulation layout) -> fp32 OIHW parameter gradient, times `scale`
// (the inverse loss scale).  One block per (Cout row, 128-channel chunk): coalesced reads of the k*k tap rows into
// shared memory, coalesced writes of the [128][k*k] output run.
__global__ void __launch_bounds__(128) unpack_wgrad_kernel(const float* __restrict__ g, float* __restrict__ out, int cout, int cin, int k, float scale) {
  __shared__ float tile[9][129];
  const int k2 = k * k;
  const int co = blockIdx.y, ci0 = blockIdx.x * 128, t = threadIdx.x;
  const int nci = cin - ci0 < 128 ? cin - ci0 : 128;
  if (t < nci)
    for (int tap = 0; tap < k2; ++tap) tile[tap][t] = g[(static_cast<long long>(co) * k2 + tap) * cin + ci0 + t];
  __syncthreads();
  float* dst = out + (static_cast<long long>(co) * cin + ci0) * k2;
  for (int j = t; j < nci * k2; j += 128) dst[j] = tile[j % k2][j / k2] * scale;
}

// ------------------------------------------------------------------------------------------------
// Gradient guard.  Activation gradients travel in fp16 under a static loss scale; an overflow there (huge hparams, a tiny
// running_var) would write inf / NaN into the parameter gradients and poison the optimizer state for good.  Pass 1 raises
// found[0] (float, zeroed here first) if any of the `count` fp32 values is not finite; pass 2 (zero_if_found) clears the
// whole buffer in that case, so a plain optimizer takes a null step.  Optimizers that understand `found_inf` (torch's fused
// Adam / SGD) can skip the step outright from the same flag.  No host synchronisation; capturable.
__global__ void grad_guard_detect_kernel(const float4* __restrict__ buf, long long count4, const float* __restrict__ tail, int ntail,
                                         float* __restrict__ found) {
  bool bad = false;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < count4; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = __ldg(buf + i);
    // x - x is 0 for finite x and NaN for inf / NaN
    const float t = (v.x - v.x) + (v.y - v.y) + (v.z - v.z) + (v.w - v.w);
    bad = bad || !(t == 0.f);
  }
  if (blockIdx.x == 0 && static_cast<int>(threadIdx.x) < ntail) {
    const float x = tail[threadIdx.x];
    bad = bad || !((x - x) == 0.f);
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) *found = 1.f;
}

__global__ void grad_guard_zero_kernel(float4* __restrict__ buf, long long count4, float* __restrict__ tail, int ntail, const float* __restrict__ found) {
  if (*found == 0.f) return;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < count4; i += static_cast<long long>(gridDim.x) * blockDim.x)
    buf[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (blockIdx.x == 0 && static_cast<int>(threadIdx.x) < ntail) tail[threadIdx.x] = 0.f;
}

int grad_guard(float* buf, long long count, float* found, int zero_if_found, cudaStream_t stream) {
  YB_REQUIRE(buf && found && count > 0 && (reinterpret_cast<uintptr_t>(buf) & 15) == 0, "grad_guard: bad argument (16 B aligned buffer)");
  YB_CUDA(cudaMemsetAsync(found, 0, sizeof(float), stream));
  const long long count4 = count / 4;
  const int ntail = static_cast<int>(count - count4 * 4);
  const int grid = sm_count() * 8;
  grad_guard_detect_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const float4*>(buf), count4, buf + count4 * 4, ntail, found);
  int rc = check_launch("grad_guard_detect_kernel");
  if (rc || !zero_if_found) return rc;
  grad_guard_zero_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<float4*>(buf), count4, buf + count4 * 4, ntail, found);
  return check_launch("grad_guard_zero_kernel");
}

// ------------------------------------------------------------------------------------------------
// Gradient guard of dynamic loss scaling.  The backward ran at grad_scale * f, where f (device float, a power of two) is the
// dynamic factor, and un-scaled by 1 / grad_scale only; this pass finishes the un-scaling and moves f.  Detection is the guard's
// pass 1 (grad_guard_detect_kernel); then, if found, the buffer is zeroed, else multiplied by 1 / f -- exact, a power of two -- and
// left unwritten when f == 1.  Last, one thread applies GradScaler's rule to f and the growth tracker: backoff 0.5 on overflow,
// growth 2 after `growth_interval` clean steps in a row, clamped to [2^-24, 2^24] so that a gradient no factor can bring into
// fp16 range cannot drive f to 0.  It runs after every block has read f, hence a launch of its own.  No host sync; capturable.
__global__ void grad_unscale_apply_kernel(float4* __restrict__ buf, long long count4, float* __restrict__ tail, int ntail,
                                          const float* __restrict__ found, const float* __restrict__ factor) {
  const bool bad = *found != 0.f;
  const float f = *factor;
  if (!bad && f == 1.f) return;
  const float s = bad ? 0.f : 1.f / f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < count4; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float4 v = bad ? make_float4(0.f, 0.f, 0.f, 0.f) : buf[i];
    v.x *= s; v.y *= s; v.z *= s; v.w *= s;
    buf[i] = v;
  }
  if (blockIdx.x == 0 && static_cast<int>(threadIdx.x) < ntail) tail[threadIdx.x] = bad ? 0.f : tail[threadIdx.x] * s;
}

__global__ void loss_scale_update_kernel(const float* __restrict__ found, float* __restrict__ factor, int* __restrict__ tracker, int growth_interval) {
  float f = *factor;
  int t = *tracker;
  if (*found != 0.f) {
    f *= 0.5f;
    t = 0;
  } else if (++t >= growth_interval) {
    f *= 2.f;
    t = 0;
  }
  *factor = fminf(fmaxf(f, 0x1p-24f), 0x1p24f);
  *tracker = t;
}

int grad_unscale_guard(float* buf, long long count, float* found, float* factor, int* tracker, int growth_interval, cudaStream_t stream) {
  YB_REQUIRE(buf && found && factor && tracker && count > 0 && growth_interval > 0 && (reinterpret_cast<uintptr_t>(buf) & 15) == 0,
             "grad_unscale_guard: bad argument (16 B aligned buffer, growth_interval > 0)");
  YB_CUDA(cudaMemsetAsync(found, 0, sizeof(float), stream));
  const long long count4 = count / 4;
  const int ntail = static_cast<int>(count - count4 * 4);
  const int grid = sm_count() * 8;
  grad_guard_detect_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const float4*>(buf), count4, buf + count4 * 4, ntail, found);
  int rc = check_launch("grad_guard_detect_kernel");
  if (rc) return rc;
  grad_unscale_apply_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<float4*>(buf), count4, buf + count4 * 4, ntail, found, factor);
  rc = check_launch("grad_unscale_apply_kernel");
  if (rc) return rc;
  loss_scale_update_kernel<<<1, 1, 0, stream>>>(found, factor, tracker, growth_interval);
  return check_launch("loss_scale_update_kernel");
}

int unpack_wgrad(const float* g_krsc, float* out_oihw, int cout, int cin, int k, float scale, cudaStream_t stream) {
  YB_REQUIRE(g_krsc && out_oihw && cout > 0 && cin > 0 && (k == 1 || k == 3), "unpack_wgrad: bad argument");
  unpack_wgrad_kernel<<<dim3((cin + 127) / 128, cout), 128, 0, stream>>>(g_krsc, out_oihw, cout, cin, k, scale);
  return check_launch("unpack_wgrad_kernel");
}

}  // namespace yb
