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
// Training (Inception-v3):
//   pack_weight_dgrad_khw      the data-gradient operand: rotated by 180 degrees, transposed, zero-padded.
//   maxpool3x3_s2_valid_bwd    the backward of maxpool3x3_s2_valid, dy read from a channel slice of a block's output gradient.
//   join_f16                   the gradient at a tensor read by several units: the sum of up to four contributions.
// Training (Inception-v4):
//   avgpool3x3_s1_excl_bwd     the backward of avgpool3x3_s1_excl: each output's gradient divided by that output's own divisor.
#include "yb_common.h"
#include "yb_pool.cuh"
#include <cuda_fp16.h>
#include <stdint.h>

namespace yb {

// element idx of the forward operand [cout_pad][kh][kw][cin_pad]
__device__ __forceinline__ __half khw_fwd_elem(const float* __restrict__ w, long long idx, int cout, int cin, int taps, int cin_pad) {
  const int ci = static_cast<int>(idx % cin_pad);
  const long long t = idx / cin_pad;
  const int tap = static_cast<int>(t % taps);
  const int co = static_cast<int>(t / taps);
  return __float2half_rn((co < cout && ci < cin) ? __ldg(w + (static_cast<long long>(co) * cin + ci) * taps + tap) : 0.f);
}

// element idx of the data-gradient operand [cin_pad][kh][kw][cout_pad]: out[ci][tap][co] = w[co][ci][taps-1-tap] (rotated by 180 degrees)
__device__ __forceinline__ __half khw_dgrad_elem(const float* __restrict__ w, long long idx, int cout, int cin, int taps, int cout_pad) {
  const int co = static_cast<int>(idx % cout_pad);
  const long long t = idx / cout_pad;
  const int tap = static_cast<int>(t % taps);
  const int ci = static_cast<int>(t / taps);
  return __float2half_rn((co < cout && ci < cin) ? __ldg(w + (static_cast<long long>(co) * cin + ci) * taps + (taps - 1 - tap)) : 0.f);
}

__global__ void pack_weight_khw_kernel(const float* __restrict__ w, __half* __restrict__ out, int cout, int cin, int kh, int kw, int cout_pad,
                                       int cin_pad) {
  const long long total = static_cast<long long>(cout_pad) * kh * kw * cin_pad;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  out[idx] = khw_fwd_elem(w, idx, cout, cin, kh * kw, cin_pad);
}

int pack_weight_khw(const float* w, void* out, int cout, int cin, int kh, int kw, int cout_pad, int cin_pad, cudaStream_t stream) {
  YB_REQUIRE(w && out && cout > 0 && cin > 0 && kh >= 1 && kh <= 7 && kw >= 1 && kw <= 7 && cout_pad >= cout && cin_pad >= cin,
             "pack_weight_khw: bad argument (cout %d, cin %d, kernel %d x %d, padded to %d x %d)", cout, cin, kh, kw, cout_pad, cin_pad);
  const long long total = static_cast<long long>(cout_pad) * kh * kw * cin_pad;
  pack_weight_khw_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(w, reinterpret_cast<__half*>(out), cout, cin, kh, kw,
                                                                                        cout_pad, cin_pad);
  return check_launch("pack_weight_khw_kernel");
}

// Data-gradient operand of a kh x kw conv: out[ci][r][s][co] = w[co][ci][kh-1-r][kw-1-s], fp16 [cin_pad][kh][kw][cout_pad], zeros in the
// padding.  The data gradient is then yb_conv2d_bn_act_fwd on dz (cout_pad channels) at padding (kh-1-pad_h, kw-1-pad_w), stride 1; the
// zero rows of padded input channels give exact-zero gradients there.
__global__ void pack_weight_dgrad_khw_kernel(const float* __restrict__ w, __half* __restrict__ out, int cout, int cin, int kh, int kw, int cout_pad,
                                             int cin_pad) {
  const long long total = static_cast<long long>(cin_pad) * kh * kw * cout_pad;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  out[idx] = khw_dgrad_elem(w, idx, cout, cin, kh * kw, cout_pad);
}

int pack_weight_dgrad_khw(const float* w, void* out, int cout, int cin, int kh, int kw, int cout_pad, int cin_pad, cudaStream_t stream) {
  YB_REQUIRE(w && out && cout > 0 && cin > 0 && kh >= 1 && kh <= 7 && kw >= 1 && kw <= 7 && cout_pad >= cout && cin_pad >= cin,
             "pack_weight_dgrad_khw: bad argument (cout %d, cin %d, kernel %d x %d, padded to %d x %d)", cout, cin, kh, kw, cout_pad, cin_pad);
  const long long total = static_cast<long long>(cin_pad) * kh * kw * cout_pad;
  pack_weight_dgrad_khw_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(w, reinterpret_cast<__half*>(out), cout, cin, kh, kw,
                                                                                              cout_pad, cin_pad);
  return check_launch("pack_weight_dgrad_khw_kernel");
}

// Both operands of many kh x kw units in ONE launch (yb_pack_weights_khw_batch): a training step re-packs every weight, and one launch per
// operand and unit is 187 launches per Inception-v3 step.  The work is one flat range: unit u owns elements [elem0, elem0 + 2n), n =
// cout_pad * kh * kw * cin_pad, the first n its forward operand, the next n its data-gradient operand, each element written by the same
// expression as the single-unit packs above (so the bits are theirs).  The unit table is staged in shared memory and searched per element.
struct PackKhwUnit {
  const float* w;
  __half* out_f;
  __half* out_d;
  long long elem0;
  int cout, cin, kh, kw, cout_pad, cin_pad;
};
constexpr int kPackKhwMaxUnits = 256;

__global__ void __launch_bounds__(256) pack_weights_khw_batch_kernel(const PackKhwUnit* __restrict__ units, int num_units, long long total) {
  __shared__ PackKhwUnit s_units[kPackKhwMaxUnits];
  for (int i = threadIdx.x; i < num_units; i += blockDim.x) s_units[i] = units[i];
  __syncthreads();
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    int lo = 0, hi = num_units - 1;                 // the last unit whose elem0 <= idx
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_units[mid].elem0 <= idx) lo = mid; else hi = mid - 1;
    }
    const PackKhwUnit& u = s_units[lo];
    const int taps = u.kh * u.kw;
    const long long n = static_cast<long long>(u.cout_pad) * taps * u.cin_pad;
    const long long local = idx - u.elem0;
    if (local < n) {
      if (u.out_f != nullptr) u.out_f[local] = khw_fwd_elem(u.w, local, u.cout, u.cin, taps, u.cin_pad);
    } else if (u.out_d != nullptr) {
      u.out_d[local - n] = khw_dgrad_elem(u.w, local - n, u.cout, u.cin, taps, u.cout_pad);
    }
  }
}

int pack_weights_khw_batch(const void* units_dev, int num_units, long long total, cudaStream_t stream) {
  static_assert(sizeof(PackKhwUnit) == 56, "PackKhwUnit must match yb_pack_khw_unit");
  YB_REQUIRE(units_dev && num_units > 0 && num_units <= kPackKhwMaxUnits && total > 0,
             "pack_weights_khw_batch: bad argument (1..%d units)", kPackKhwMaxUnits);
  const long long blocks = (total + 255) / 256;
  const long long cap = static_cast<long long>(sm_count()) * 16;
  pack_weights_khw_batch_kernel<<<static_cast<unsigned>(blocks < cap ? blocks : cap), 256, 0, stream>>>(static_cast<const PackKhwUnit*>(units_dev),
                                                                                                        num_units, total);
  return check_launch("pack_weights_khw_batch_kernel");
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

// Backward of maxpool3x3_s2_valid (F.max_pool2d(x, 3, stride=2)): every output's gradient goes to the FIRST maximum of its window in scan
// order (rows, then columns; a later element replaces the running maximum only if strictly greater, or NaN), torch's rule.  The winner is
// recomputed from x.  One thread per input pixel and 8 channels gathers from the at most 2 x 2 windows that contain the pixel, sums in fp32
// and rounds once: no atomics, deterministic.  dy is channels [dy_ch_off, dy_ch_off + C) of [B,OH,OW,dy_ld]; dx is [B,H,W,C].
__global__ void maxpool3x3_s2_valid_bwd_kernel(const __half* __restrict__ x, const __half* __restrict__ dy, int dy_ld, int dy_ch_off,
                                               __half* __restrict__ dx, int batch, int height, int width, int channels) {
  const int c8 = channels >> 3;
  const int oh = (height - 3) / 2 + 1, ow = (width - 3) / 2 + 1;
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
  // windows o with 2o <= i <= 2o + 2
  const int oy0 = iy >= 2 ? (iy - 1) / 2 : 0, oy1 = min(iy / 2, oh - 1);
  const int ox0 = ix >= 2 ? (ix - 1) / 2 : 0, ox1 = min(ix / 2, ow - 1);
  const int me = iy * width + ix;
  for (int oy = oy0; oy <= oy1; ++oy) {
    for (int ox = ox0; ox <= ox1; ++ox) {
      float best[8];
      int arg[8];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int yy = 2 * oy + r, xx = 2 * ox + s;
          const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + ((img * height + yy) * width + xx) * channels + cg * 8));
          const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const float f = __half2float(hv[e]);
            if ((r | s) == 0 || f > best[e] || isnan(f)) {
              best[e] = f;
              arg[e] = yy * width + xx;
            }
          }
        }
      }
      const uint4 g = __ldg(reinterpret_cast<const uint4*>(dy + ((img * oh + oy) * ow + ox) * dy_ld + dy_ch_off + cg * 8));
      const __half* hg = reinterpret_cast<const __half*>(&g);
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

int maxpool3x3_s2_valid_bwd(const void* x, const void* dy, int dy_ld, int dy_ch_off, void* dx, int batch, int height, int width, int channels,
                            cudaStream_t stream) {
  YB_REQUIRE(x && dy && dx && batch > 0 && height >= 3 && width >= 3 && channels > 0 && channels % 8 == 0,
             "maxpool3x3_s2_valid_bwd: bad argument (H, W >= 3, C a multiple of 8)");
  YB_REQUIRE(dy_ld % 8 == 0 && dy_ch_off % 8 == 0 && dy_ch_off >= 0 && dy_ch_off + channels <= dy_ld,
             "maxpool3x3_s2_valid_bwd: channels [%d, %d) do not fit dy_ld=%d (offsets multiples of 8)", dy_ch_off, dy_ch_off + channels, dy_ld);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(dy) & 15) == 0 && (reinterpret_cast<uintptr_t>(dx) & 15) == 0,
             "maxpool3x3_s2_valid_bwd: x / dy / dx must be 16B aligned");
  const long long total = static_cast<long long>(batch) * height * width * (channels / 8);
  maxpool3x3_s2_valid_bwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const __half*>(x), reinterpret_cast<const __half*>(dy), dy_ld, dy_ch_off, reinterpret_cast<__half*>(dx), batch, height, width,
      channels);
  return check_launch("maxpool3x3_s2_valid_bwd_kernel");
}

// out = fp16(a + b + c + d), summed in fp32 in that order and rounded once; c and d may be NULL.  The gradient at a tensor read by several
// units (a Mixed block's input, the branch point of Mixed_7b / 7c's 3x3 branches).
__global__ void join_f16_kernel(const __half* __restrict__ a, const __half* __restrict__ b, const __half* __restrict__ c, const __half* __restrict__ d,
                                __half* __restrict__ out, long long n8) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n8) return;
  const __half* src[4] = {a, b, c, d};
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (src[i] == nullptr) continue;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src[i]) + idx);
    const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += __half2float(hv[e]);
  }
  uint4 o;
  __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int e = 0; e < 4; ++e) ho[e] = __floats2half2_rn(acc[2 * e], acc[2 * e + 1]);
  reinterpret_cast<uint4*>(out)[idx] = o;
}

int join_f16(const void* a, const void* b, const void* c, const void* d, void* out, long long count, cudaStream_t stream) {
  YB_REQUIRE(a && b && out && count > 0 && count % 8 == 0 && (c || !d), "join_f16: bad argument (a, b required, count a multiple of 8)");
  const void* ptrs[5] = {a, b, c, d, out};
  for (const void* q : ptrs) YB_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0, "join_f16: operands must be 16B aligned");
  const long long n8 = count / 8;
  join_f16_kernel<<<static_cast<unsigned>((n8 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const __half*>(a), reinterpret_cast<const __half*>(b), reinterpret_cast<const __half*>(c), reinterpret_cast<const __half*>(d),
      reinterpret_cast<__half*>(out), n8);
  return check_launch("join_f16_kernel");
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

// Backward of avgpool3x3_s1_excl: dx[b, iy, ix, c] = fp16(sum over the in-range outputs (oy, ox) of rows iy-1..iy+1, columns ix-1..ix+1 in
// row-major order of dy[b, oy, ox, c] / n(oy, ox)), each term one round-to-nearest fp32 division by that output's own in-range count, summed
// in fp32 and rounded once.  The pool is not its own transpose: the divisor belongs to the output, not to the input pixel.  One thread per
// pixel and 8 channels gathers; no atomics, deterministic.
__global__ void avgpool3x3_s1_excl_bwd_kernel(const __half* __restrict__ dy, __half* __restrict__ dx, int batch, int height, int width,
                                              int channels) {
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
    const int oy = py + r;
    if (oy < 0 || oy >= height) continue;
    const int rows = 3 - (oy == 0) - (oy == height - 1);
#pragma unroll
    for (int s = -1; s <= 1; ++s) {
      const int ox = px + s;
      if (ox < 0 || ox >= width) continue;
      const float n = static_cast<float>(rows * (3 - (ox == 0) - (ox == width - 1)));
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(dy + ((img * height + oy) * width + ox) * channels + cg * 8));
      const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += __fdiv_rn(__half2float(hv[e]), n);
    }
  }
  uint4 out;
  __half2* ho = reinterpret_cast<__half2*>(&out);
#pragma unroll
  for (int e = 0; e < 4; ++e) ho[e] = __floats2half2_rn(acc[2 * e], acc[2 * e + 1]);
  reinterpret_cast<uint4*>(dx)[idx] = out;
}

int avgpool3x3_s1_excl_bwd(const void* dy, void* dx, int batch, int height, int width, int channels, cudaStream_t stream) {
  YB_REQUIRE(dy && dx && batch > 0 && height > 0 && width > 0 && channels > 0 && channels % 8 == 0,
             "avgpool3x3_s1_excl_bwd: bad argument (C a multiple of 8)");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(dy) & 15) == 0 && (reinterpret_cast<uintptr_t>(dx) & 15) == 0,
             "avgpool3x3_s1_excl_bwd: dy / dx must be 16B aligned");
  const long long total = static_cast<long long>(batch) * height * width * (channels / 8);
  avgpool3x3_s1_excl_bwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(dy),
                                                                                               reinterpret_cast<__half*>(dx), batch, height,
                                                                                               width, channels);
  return check_launch("avgpool3x3_s1_excl_bwd_kernel");
}

}  // namespace yb
