// conv0 (layers1.0): 3x3 conv, Cin = 3 -> Cout = 32, + folded BN + leaky-ReLU + 2x2 max-pool, on the
// tensor cores.  Replaces nn.Conv2d(3,32,3,pad 1) -> BatchNorm2d -> LeakyReLU -> MaxPool2d(2)
// (reference model/yolo2.py:78-79) and doubles as the layout boundary: it reads the caller's
// image batch (fp32 NCHW as the reference's ToTensor produces it, raw uint8 NHWC frames scaled
// by 1/255 == torchvision ToTensor, or uint8 NHWC frames through a ToTensor + Normalize table; yb_input.cuh) and writes the first fp16
// NHWC activation.
//
// K = 27 is far too small for a TMA-fed pipeline (one pixel's im2col row is 54 bytes), so the CTA
// builds the A operand itself: a 16x32-pixel conv tile (+1 halo) is staged in shared memory once,
// each of the 128 threads converts the 4x4x3 patch of ONE 2x2 pool window to fp16 and writes the
// four im2col rows (K padded to 32, 64-byte rows, 64B-swizzled exactly like a TMA box would be)
// into four 128-row M-tiles -- M-tile j holds pixel j of every window.  The CTA (one warpgroup)
// issues 4 x 2 x 2 wgmma (M=64, N=32, K=16) into four register accumulators; every accumulator
// has the same row -> thread mapping, so a thread holds the four conv outputs of each window row
// it owns, applies scale/shift + leaky, takes the max in registers and stores the pooled pixel's
// channels.  Persistent CTAs (2 per SM), weights (B operand) built once per CTA.
#include "yb_common.h"
#include "yb_ptx.cuh"
#include "yb_input.cuh"
#include <stdlib.h>

namespace yb {

constexpr int kT0Rows = 16, kT0Cols = 32;          // conv pixels per tile (8 x 16 pool windows = 128)
constexpr int kPatchRows = kT0Rows + 2, kPatchCols = kT0Cols + 2, kPatchPitch = 48;
constexpr int kC0Out = 32;

// CTAs per SM: each thread keeps 4 x 2 x 16 fp32 accumulators in registers
constexpr int kC0CtasPerSm = 2;

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

struct Conv0Params {
  const void* x;        // fp32 NCHW [B,3,H,W] or uint8 NHWC [B,H,W,3] (InputMode)
  const float* lut;     // kInLut: fp32 [3][256]
  const float* w;       // fp32 OIHW [32,3,3,3]
  const float* scale;
  const float* shift;
  float slope;
  __half* y;            // fp16 NHWC [B,H/2,W/2,32]
  int batch, height, width;
  int tiles_x, tiles_y, num_tiles;
  int raw;              // 1: write the raw conv output, unpooled fp16 NHWC [B,H,W,32] (training forward)
  double* stats;        // raw form of conv0_k16_kernel: += sum z, sum z^2 per channel ([2][32]); may be null
  int* dbg;
};

template <int kIn>
__global__ void __launch_bounds__(128, kC0CtasPerSm) conv0_tc_kernel(const Conv0Params p) {
  __shared__ __align__(1024) uint8_t a_smem[4 * 128 * 64];          // 4 M-tiles x 128 rows x 64 B (SW64)
  __shared__ __align__(1024) uint8_t b_smem[kC0Out * 64];           // 32 rows (Cout) x 64 B (SW64)
  __shared__ __align__(16) float patch[3][kPatchRows][kPatchPitch];
  __shared__ __align__(16) float sc[kC0Out], sh[kC0Out];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t a_base = smem_u32(a_smem), b_base = smem_u32(b_smem);

  if (tid < kC0Out) { sc[tid] = p.scale[tid]; sh[tid] = p.shift[tid]; }
  {
    // B operand: row n = output channel, k = ci*9 + r*3 + s (the OIHW flattening), zero padded to 32
    const int n = tid >> 2, j = tid & 3;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = j * 8 + e;
      v[e] = (k < 27) ? __ldg(p.w + n * 27 + k) : 0.f;
    }
    const uint4 pk = make_uint4(pack_h2(v[0], v[1]), pack_h2(v[2], v[3]), pack_h2(v[4], v[5]), pack_h2(v[6], v[7]));
    *reinterpret_cast<uint4*>(b_smem + n * 64 + ((j ^ ((n >> 1) & 3)) << 4)) = pk;
  }
  __syncthreads();
  pdl_trigger();        // lets a PDL successor (the next conv) set up while this grid drains

  const int wy = tid >> 4, wx = tid & 15;        // the pool window whose im2col rows this thread builds
  const int oh = p.height >> 1, ow = p.width >> 1;

  constexpr int kPatchElems = 3 * kPatchRows * kPatchCols;
  constexpr int kPatchIters = (kPatchElems + 127) / 128;
  // All of a tile's patch loads are issued back to back into registers (one exposed memory latency,
  // not kPatchIters of them) and, from the second tile on, while the previous tile's MMAs and
  // epilogue are still running.
  auto prefetch = [&](int t, float (&v)[kPatchIters]) {
    const int ptx = t % p.tiles_x;
    const int pt2 = t / p.tiles_x;
    const int pty = pt2 % p.tiles_y;
    const int pimg = pt2 / p.tiles_y;
    const int y0 = pty * kT0Rows - 1, x0 = ptx * kT0Cols - 1;
#pragma unroll
    for (int k = 0; k < kPatchIters; ++k) {
      const int i = tid + k * 128;
      const int c = i / (kPatchRows * kPatchCols);
      const int rem = i - c * (kPatchRows * kPatchCols);
      const int r = rem / kPatchCols, col = rem - r * kPatchCols;
      const int iy = y0 + r, ix = x0 + col;
      float val = 0.f;
      if (i < kPatchElems && iy >= 0 && iy < p.height && ix >= 0 && ix < p.width) {
        if (kIn == kInLut) {
          val = lut_pixel(p.x, p.lut, pimg, c, iy, ix, p.height, p.width);
        } else if (kIn == kInU8) {
          val = static_cast<float>(__ldg(reinterpret_cast<const uint8_t*>(p.x) + ((static_cast<long long>(pimg) * p.height + iy) * p.width + ix) * 3 + c)) *
                (1.f / 255.f);
        } else {
          val = __ldg(reinterpret_cast<const float*>(p.x) + ((static_cast<long long>(pimg) * 3 + c) * p.height + iy) * p.width + ix);
        }
      }
      v[k] = val;
    }
  };
  float pre[kPatchIters];
  if (static_cast<int>(blockIdx.x) < p.num_tiles) prefetch(blockIdx.x, pre);

  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int tx = tile % p.tiles_x;
    const int t2 = tile / p.tiles_x;
    const int ty = t2 % p.tiles_y;
    const int img = t2 / p.tiles_y;
    // ---- 1. stage the haloed input patch (zeros outside the image) from the prefetched registers ----
#pragma unroll
    for (int k = 0; k < kPatchIters; ++k) {
      const int i = tid + k * 128;
      if (i < kPatchElems) {
        const int c = i / (kPatchRows * kPatchCols);
        const int rem = i - c * (kPatchRows * kPatchCols);
        const int r = rem / kPatchCols, col = rem - r * kPatchCols;
        patch[c][r][col] = pre[k];
      }
    }
    __syncthreads();
    // ---- 2. build the four im2col rows of this thread's window ----
    float in[3][4][4];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float2 lo = *reinterpret_cast<const float2*>(&patch[c][2 * wy + r][2 * wx]);
        const float2 hi = *reinterpret_cast<const float2*>(&patch[c][2 * wy + r][2 * wx + 2]);
        in[c][r][0] = lo.x; in[c][r][1] = lo.y; in[c][r][2] = hi.x; in[c][r][3] = hi.y;
      }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int dy = j >> 1, dx = j & 1;
      float k[32];
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int s = 0; s < 3; ++s) k[c * 9 + r * 3 + s] = in[c][dy + r][dx + s];
#pragma unroll
      for (int e = 27; e < 32; ++e) k[e] = 0.f;
      uint8_t* row = a_smem + j * (128 * 64) + tid * 64;
      const int sw = (tid >> 1) & 3;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint4 pk = make_uint4(pack_h2(k[q * 8 + 0], k[q * 8 + 1]), pack_h2(k[q * 8 + 2], k[q * 8 + 3]),
                                    pack_h2(k[q * 8 + 4], k[q * 8 + 5]), pack_h2(k[q * 8 + 6], k[q * 8 + 7]));
        *reinterpret_cast<uint4*>(row + ((q ^ sw) << 4)) = pk;
      }
    }
    // generic-proxy smem writes -> visible to the tensor core (async proxy)
    fence_proxy_async_smem();
    __syncthreads();
    // ---- 3. MMA: 4 accumulators x 2 row halves x (K = 32 = 2 x 16) ----
    float acc[4][2][16];
    {
      const uint64_t bdesc = make_kmajor_desc<64>(b_base);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t adesc = make_kmajor_desc<64>(a_base + j * (128 * 64) + h * (64 * 64));
          wgmma_f16<kC0Out>(acc[j][h], adesc, bdesc, 0);
          wgmma_f16<kC0Out>(acc[j][h], adesc + 2, bdesc + 2, 1);
        }
      }
      wgmma_commit();
    }
    {
      const int next = tile + gridDim.x;          // overlap the next tile's input fetch with the MMAs
      if (next < p.num_tiles) prefetch(next, pre);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 4; ++j) { fence_regs(acc[j][0]); fence_regs(acc[j][1]); }
    // ---- 4. epilogue: scale/shift + leaky on the 4 pixels of each window, max, fp16 NHWC store ----
    // accumulator row m (= pool window m of the tile) of fragment half (h, hh), channels 8 jj + 2 (lane % 4) + {0, 1}
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int m = 64 * h + 16 * warp + (lane >> 2) + 8 * hh;
        const int my = m >> 4, mx = m & 15;
        const int py = ty * (kT0Rows / 2) + my, px = tx * (kT0Cols / 2) + mx;
        __half* dst = p.y + ((static_cast<long long>(img) * oh + py) * ow + px) * kC0Out;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int c = 8 * jj + 2 * (lane & 3);
          if (p.raw) {
            // training mode: the raw (pre-BatchNorm) conv output of the 4 pixels of this window, unpooled
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int yy = ty * kT0Rows + 2 * my + (j >> 1), xx = tx * kT0Cols + 2 * mx + (j & 1);
              *reinterpret_cast<uint32_t*>(p.y + ((static_cast<long long>(img) * p.height + yy) * p.width + xx) * kC0Out + c) =
                  pack_h2(acc[j][h][4 * jj + 2 * hh], acc[j][h][4 * jj + 2 * hh + 1]);
            }
            continue;
          }
          float mm[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float s = sc[c + e], b = sh[c + e];
            float best = -INFINITY;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float t = acc[j][h][4 * jj + 2 * hh + e] * s + b;
              t = t > 0.f ? t : t * p.slope;
              best = fmaxf(best, t);
            }
            mm[e] = best;
          }
          *reinterpret_cast<uint32_t*>(dst + c) = pack_h2(mm[0], mm[1]);
        }
      }
    }
    // The next tile's barrier (after patch staging, before its MMAs) orders this tile's smem reads before anything is
    // overwritten.
  }
}

// ---------------------------------------------------------------------------------------------
// Second form of the same layer: NO thread-built im2col rows.  The first form above spends most of its instruction issue writing four
// 64-byte im2col rows per thread while the tensor core and HBM sit mostly idle.  Here the haloed input patch is
// kept in shared memory as fp16 pixels of 4 channels (r, g, b, 0 = 8 bytes) and the tensor core reads every operand IN PLACE through
// un-swizzled K-major descriptors: one filter ROW (3 taps x 4 channels = 12, padded to K = 16) of output pixel (y, x) is the 32
// contiguous bytes starting at patch pixel (y + r, x); pixels two columns apart are 16 bytes apart, which is exactly the row pitch of
// an 8 x 16 B core matrix.  So with M-tile (dy, dx) = pixel (dy, dx) of every 2x2 pool window, the 8 windows of a window row form one
// core matrix (LBO = 16 B to the second K chunk, which overlaps the next window's first -- it is only ever read), the next window row
// is two patch rows further (SBO = 288 B), and a second copy of the patch shifted by one pixel gives the odd columns their 16-byte
// alignment.  3 MMAs (one per filter row, K = 16) per accumulator instead of 2, and the threads only convert + store 8 B per pixel.
// K-pad lanes read the neighbouring pixel and meet zero weights (finite inputs assumed; an inf / NaN pixel would reach x - 3 .. x + 1
// instead of x - 1 .. x + 1).
constexpr int kV2Rows = 32, kV2Cols = 16;                       // conv pixels per tile = 16 x 8 pool windows
constexpr int kV2PR = kV2Rows + 2, kV2PC = kV2Cols + 2;         // 34 x 18 pixel patch
constexpr int kV2Pitch = kV2PC * 8;                             // 144 B per patch row
constexpr int kV2Copy = kV2PR * kV2Pitch;                       // 4896 B
constexpr int kV2Pixels = kV2PR * kV2PC;                        // 612
constexpr int kV2Iters = (kV2Pixels + 127) / 128;               // 5 pixels per thread

// kRaw (training forward): the un-normalised conv output z goes out at full resolution.  Written straight from the accumulator layout, every
// store instruction would touch many different 128-byte lines (bound by L2 write transactions); instead the tile is staged in shared memory
// (swizzled) and leaves as 512 contiguous bytes per warp instruction.  The copy-out loop hands every thread
// the same 8 channels on every trip, so the BatchNorm batch statistics (sum z, sum z^2 of the fp16 values that are stored) accumulate in 16
// fp32 registers over one tile (16 rows per thread), are reduced across the warp and added into a double shared accumulator per tile, and
// leave once at the end (p.stats: double [2][32], as yb_bn_stats).  Keeping the fp32 part to one tile bounds its rounding error by 19 fp32
// roundings of sum |z| however many tiles a CTA runs: the variance var = sum z^2 / n - mean^2 amplifies that error by 1 + (mean / std)^2.
constexpr int kV2StageBytes = kV2Rows * kV2Cols * kC0Out * 2;   // 32 KB

template <int kIn, bool kRaw>
__global__ void __launch_bounds__(128, kC0CtasPerSm) conv0_k16_kernel(const Conv0Params p) {
  __shared__ __align__(128) uint8_t stage[kRaw ? kV2StageBytes : 16];
  __shared__ double s_stats[2 * kC0Out];
  __shared__ __align__(128) uint8_t patch_e[kV2Copy + 48];      // pixel (r, c) at (r * 18 + c) * 8: even columns 16 B aligned
  __shared__ __align__(128) uint8_t patch_o[kV2Copy + 48];      // the same pixels at + 8 B: odd columns 16 B aligned
  __shared__ __align__(128) uint8_t b_smem[3 * 1024];           // per filter row: [n / 8][k / 8][n % 8][k % 8] fp16 (32 x 16)
  __shared__ __align__(16) float sc[kC0Out], sh[kC0Out];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t e_base = smem_u32(patch_e), o_base = smem_u32(patch_o), b_base = smem_u32(b_smem);

  if (tid < kC0Out) { sc[tid] = p.scale[tid]; sh[tid] = p.shift[tid]; }
  // the bytes past the last patch pixel are read by the K-pad lanes of the last row: keep them finite
  if (tid < 12) {
    reinterpret_cast<uint32_t*>(patch_e + kV2Copy)[tid] = 0u;
    reinterpret_cast<uint32_t*>(patch_o + kV2Copy)[tid] = 0u;
  }
  if (tid < 2) reinterpret_cast<uint32_t*>(patch_o)[tid] = 0u;
  {
    // B operand, filter row r: element (n, k = s * 4 + c) = w[n][c][r][s] for s, c < 3, else 0
    const int n = tid >> 2, s4 = tid & 3;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float v[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) v[c] = (s4 < 3 && c < 3) ? __ldg(p.w + n * 27 + c * 9 + r * 3 + s4) : 0.f;
      const uint2 pk = make_uint2(pack_h2(v[0], v[1]), pack_h2(v[2], v[3]));
      *reinterpret_cast<uint2*>(b_smem + r * 1024 + (n >> 3) * 256 + (s4 >> 1) * 128 + (n & 7) * 16 + (s4 & 1) * 8) = pk;
    }
  }
  __syncthreads();
  pdl_trigger();

  const int oh = p.height >> 1, ow = p.width >> 1;

  auto prefetch = [&](int t, float (&v)[kV2Iters][3]) {
    const int ptx = t % p.tiles_x;
    const int pt2 = t / p.tiles_x;
    const int pty = pt2 % p.tiles_y;
    const int pimg = pt2 / p.tiles_y;
    const int y0 = pty * kV2Rows - 1, x0 = ptx * kV2Cols - 1;
#pragma unroll
    for (int k = 0; k < kV2Iters; ++k) {
      const int i = tid + k * 128;
      const int r = i / kV2PC, c = i - r * kV2PC;
      const int iy = y0 + r, ix = x0 + c;
      const bool ok = i < kV2Pixels && iy >= 0 && iy < p.height && ix >= 0 && ix < p.width;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        float val = 0.f;
        if (ok) {
          if (kIn == kInLut) val = lut_pixel(p.x, p.lut, pimg, ch, iy, ix, p.height, p.width);
          else if (kIn == kInU8) val = static_cast<float>(__ldg(reinterpret_cast<const uint8_t*>(p.x) + ((static_cast<long long>(pimg) * p.height + iy) * p.width + ix) * 3 + ch)) * (1.f / 255.f);
          else val = __ldg(reinterpret_cast<const float*>(p.x) + ((static_cast<long long>(pimg) * 3 + ch) * p.height + iy) * p.width + ix);
        }
        v[k][ch] = val;
      }
    }
  };
  float pre[kV2Iters][3];
  if (static_cast<int>(blockIdx.x) < p.num_tiles) prefetch(blockIdx.x, pre);
  float st1[8], st2[8];                           // kRaw: statistics of channels (tid & 3) * 8 .. + 7
#pragma unroll
  for (int e = 0; e < 8; ++e) { st1[e] = 0.f; st2[e] = 0.f; }
  if (kRaw && tid < 2 * kC0Out) s_stats[tid] = 0.0;

  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int tx = tile % p.tiles_x;
    const int t2 = tile / p.tiles_x;
    const int ty = t2 % p.tiles_y;
    const int img = t2 / p.tiles_y;
    // every warp's wgmma of the previous tile has retired (each warp waited on its own part) before any thread overwrites the
    // operands it read
    __syncthreads();
    // ---- 1. the patch, twice (8 B per pixel each) ----
#pragma unroll
    for (int k = 0; k < kV2Iters; ++k) {
      const int i = tid + k * 128;
      if (i < kV2Pixels) {
        const uint2 pk = make_uint2(pack_h2(pre[k][0], pre[k][1]), pack_h2(pre[k][2], 0.f));
        *reinterpret_cast<uint2*>(patch_e + i * 8) = pk;
        *reinterpret_cast<uint2*>(patch_o + 8 + i * 8) = pk;
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    // ---- 2. MMA: accumulator (dy, dx) += sum over filter rows, operands read in place.  Accumulator rows = pool windows
    // (8 per window row, window rows 2 patch rows apart); rows 64..127 start 8 window rows further down ----
    float acc[4][2][16];
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int dy = j >> 1, dx = j & 1;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const uint32_t a_addr = (dx ? o_base + 8 : e_base) + ((dy + r) * kV2PC + dx) * 8 + h * 8 * (2 * kV2Pitch);
          wgmma_f16<kC0Out>(acc[j][h], make_kmajor_desc_noswz(a_addr, 16, 2 * kV2Pitch), make_kmajor_desc_noswz(b_base + r * 1024, 128, 256), r != 0);
        }
      }
    }
    wgmma_commit();
    {
      const int next = tile + gridDim.x;
      if (next < p.num_tiles) prefetch(next, pre);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 4; ++j) { fence_regs(acc[j][0]); fence_regs(acc[j][1]); }
    // ---- 3. epilogue: as the first form, window m = accumulator row ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int m = 64 * h + 16 * warp + (lane >> 2) + 8 * hh;
        const int wy = m >> 3, wx = m & 7;
        const int py = ty * (kV2Rows / 2) + wy, px = tx * (kV2Cols / 2) + wx;
        __half* dst = p.y + ((static_cast<long long>(img) * oh + py) * ow + px) * kC0Out;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int c = 8 * jj + 2 * (lane & 3);
          if constexpr (kRaw) {
            // pixel (row, col) of the tile lives at slot col' = col / 2 + (col & 1) * 8 of its row (the eight windows of a window row
            // then fill eight consecutive 64-byte slots), 16-byte chunk jj at jj ^ ((col / 4) & 3)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int row = 2 * wy + (j >> 1), slot = wx + (j & 1) * 8;
              *reinterpret_cast<uint32_t*>(stage + (row * kV2Cols + slot) * (kC0Out * 2) + ((jj ^ ((wx >> 1) & 3)) << 4) + (lane & 3) * 4) =
                  pack_h2(acc[j][h][4 * jj + 2 * hh], acc[j][h][4 * jj + 2 * hh + 1]);
            }
            continue;
          }
          float mm[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float s = sc[c + e], b = sh[c + e];
            float best = -INFINITY;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float t = acc[j][h][4 * jj + 2 * hh + e] * s + b;
              t = t > 0.f ? t : t * p.slope;
              best = fmaxf(best, t);
            }
            mm[e] = best;
          }
          *reinterpret_cast<uint32_t*>(dst + c) = pack_h2(mm[0], mm[1]);
        }
      }
    }
    if constexpr (kRaw) {
      __syncthreads();                              // the whole tile is staged
      // 2048 chunks of 16 B: chunk c = i * 128 + tid -> row c / 64, (col, g) = c % 64 = tid % 64 on every trip
      const int cr = tid & 63, col = cr >> 2, gq = cr & 3;
      const int src_off = ((col >> 1) + (col & 1) * 8) * (kC0Out * 2) + ((gq ^ ((col >> 2) & 3)) << 4);
      __half* dst = p.y + ((static_cast<long long>(img) * p.height + ty * kV2Rows) * p.width + tx * kV2Cols) * kC0Out + cr * 8;
#pragma unroll 4
      for (int i = 0; i < kV2Rows / 2; ++i) {
        const int row = 2 * i + (tid >> 6);
        const uint4 q = *reinterpret_cast<const uint4*>(stage + row * (kV2Cols * kC0Out * 2) + src_off);
        *reinterpret_cast<uint4*>(dst + static_cast<long long>(row) * p.width * kC0Out) = q;
        if (p.stats != nullptr) {
          const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h[e]);
            st1[2 * e] += f.x; st2[2 * e] = fmaf(f.x, f.x, st2[2 * e]);
            st1[2 * e + 1] += f.y; st2[2 * e + 1] = fmaf(f.y, f.y, st2[2 * e + 1]);
          }
        }
      }
      if (p.stats != nullptr) {
        // this tile's partials: lanes with equal (lane & 3) hold the same 8 channels; their warp sum goes into the double accumulator
#pragma unroll
        for (int e = 0; e < 8; ++e) {
#pragma unroll
          for (int sft = 4; sft <= 16; sft <<= 1) {
            st1[e] += __shfl_xor_sync(0xffffffffu, st1[e], sft);
            st2[e] += __shfl_xor_sync(0xffffffffu, st2[e], sft);
          }
        }
        if ((tid & 31) < 4) {
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            atomicAdd(&s_stats[(tid & 3) * 8 + e], static_cast<double>(st1[e]));
            atomicAdd(&s_stats[kC0Out + (tid & 3) * 8 + e], static_cast<double>(st2[e]));
          }
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) { st1[e] = 0.f; st2[e] = 0.f; }
      }
      // the next iteration's __syncthreads (after the patch is written) orders this copy-out before the next tile's staging stores
    }
  }
  if (kRaw && p.stats != nullptr) {
    __syncthreads();
    if (tid < 2 * kC0Out) atomicAdd(p.stats + tid, s_stats[tid]);
  }
}

// in_mode: InputMode; lut is read in kInLut only
int conv0_tc_forward(const void* x, int in_mode, const float* lut, const float* w, const float* scale, const float* shift, float slope, void* y, int batch,
                     int height, int width, int cout, int raw, double* stats, cudaStream_t stream) {
  YB_REQUIRE(x && w && y && (raw || (scale && shift)), "conv0: null pointer");
  YB_REQUIRE(cout == kC0Out, "conv0: Cout=%d unsupported (32)", cout);
  YB_REQUIRE(in_mode == kInF32 || in_mode == kInU8 || (in_mode == kInLut && lut), "conv0: bad input mode %d (or a null table)", in_mode);
  const bool x_is_u8 = in_mode != kInF32;
  // operands-in-place form when the shape tiles 32 x 16 (every multiple of 32, i.e. every Darknet input); YB_CONV0_V1=1 forces the first form
  static const int force_v1 = getenv("YB_CONV0_V1") ? atoi(getenv("YB_CONV0_V1")) : 0;
  const bool v2 = !force_v1 && batch > 0 && height > 0 && width > 0 && height % kV2Rows == 0 && width % kV2Cols == 0;
  YB_REQUIRE(v2 || (batch > 0 && height > 0 && width > 0 && height % kT0Rows == 0 && width % kT0Cols == 0),
             "conv0: H must be a multiple of %d and W of %d, or H of %d and W of %d (got %dx%d)", kV2Rows, kV2Cols, kT0Rows, kT0Cols, height,
             width);
  Conv0Params p;
  p.x = x; p.lut = lut; p.w = w; p.scale = scale; p.shift = shift; p.slope = slope; p.y = reinterpret_cast<__half*>(y);
  p.batch = batch; p.height = height; p.width = width;
  p.tiles_x = v2 ? width / kV2Cols : width / kT0Cols;
  p.tiles_y = v2 ? height / kV2Rows : height / kT0Rows;
  const long long tiles = static_cast<long long>(p.tiles_x) * p.tiles_y * batch;
  YB_REQUIRE(tiles < (1ll << 31), "conv0: too many tiles");
  p.num_tiles = static_cast<int>(tiles);
  p.raw = raw;
  p.stats = stats;
  YB_REQUIRE(stats == nullptr || (raw && v2 && !x_is_u8), "conv0: fused statistics need the raw fp32-input form on a 32 x 16-tileable image");
  if (raw) { p.scale = w; p.shift = w; }   // unused in raw mode, must be readable
  p.dbg = debug_word_device();
  const int max_ctas = sm_count() * kC0CtasPerSm;
  const int grid = p.num_tiles < max_ctas ? p.num_tiles : max_ctas;
  if (v2) {
    if (x_is_u8) {
      YB_REQUIRE(!raw, "conv0: the uint8 input form has no raw output");
      if (in_mode == kInLut) conv0_k16_kernel<kInLut, false><<<grid, 128, 0, stream>>>(p);
      else conv0_k16_kernel<kInU8, false><<<grid, 128, 0, stream>>>(p);
    } else if (raw) {
      conv0_k16_kernel<kInF32, true><<<grid, 128, 0, stream>>>(p);
    } else {
      conv0_k16_kernel<kInF32, false><<<grid, 128, 0, stream>>>(p);
    }
    return check_launch("conv0_k16_kernel");
  }
  if (in_mode == kInLut) conv0_tc_kernel<kInLut><<<grid, 128, 0, stream>>>(p);
  else if (in_mode == kInU8) conv0_tc_kernel<kInU8><<<grid, 128, 0, stream>>>(p);
  else conv0_tc_kernel<kInF32><<<grid, 128, 0, stream>>>(p);
  return check_launch("conv0_tc_kernel");
}

// ---------------------------------------------------------------------------------------------
// 64-filter form of conv0_k16_kernel: VGG's features.0, Conv2d(3, 64, 3, padding 1) + bias or folded BatchNorm + ReLU, optionally followed by
// MaxPool2d(2, 2) (model/vgg.py make_layers).  Same 32 x 16 tiles and operands read in place (patch_e / patch_o, per-filter-row B), N = 64.
// A whole tile's accumulators at N = 64 would be 4 x 2 x 32 = 256 registers per thread, so the tile runs as two passes over accumulator
// rows 0..63 (window rows 0..7, pixel rows 0..15) and 64..127: per pass 4 x 3 wgmma (M 64, N 64, K 16) into 4 x 32 registers, then that
// pass's epilogue.  kPool: scale/shift + activation on the four pixels of each window, their max stored from registers as the 32-filter form.
// Otherwise the pass's 16 x 16 pixels x 64 channels are staged in shared memory (32 KB; pixel col at slot col / 2 + (col & 1) * 8 of its row,
// 16-byte chunk jj at jj ^ (col / 2)) and leave as 2 KB contiguous rows.  scale / shift are read through the L1 (the static shared memory is
// at its 48 KB limit).
constexpr int kC64Out = 64;
constexpr int kC64StageBytes = (kV2Rows / 2) * kV2Cols * kC64Out * 2;   // 32 KB

template <int kIn, bool kPool>
__global__ void __launch_bounds__(128, kC0CtasPerSm) conv0_c64_kernel(const Conv0Params p) {
  __shared__ __align__(128) uint8_t stage[kPool ? 16 : kC64StageBytes];
  __shared__ __align__(128) uint8_t patch_e[kV2Copy + 48];
  __shared__ __align__(128) uint8_t patch_o[kV2Copy + 48];
  __shared__ __align__(128) uint8_t b_smem[3 * 2048];           // per filter row: [n / 8][k / 8][n % 8][k % 8] fp16 (64 x 16)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t e_base = smem_u32(patch_e), o_base = smem_u32(patch_o), b_base = smem_u32(b_smem);

  if (tid < 12) {
    reinterpret_cast<uint32_t*>(patch_e + kV2Copy)[tid] = 0u;
    reinterpret_cast<uint32_t*>(patch_o + kV2Copy)[tid] = 0u;
  }
  if (tid < 2) reinterpret_cast<uint32_t*>(patch_o)[tid] = 0u;
#pragma unroll
  for (int n0 = 0; n0 < kC64Out; n0 += 32) {
    // B operand, filter row r: element (n, k = s * 4 + c) = w[n][c][r][s] for s, c < 3, else 0
    const int n = n0 + (tid >> 2), s4 = tid & 3;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float v[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) v[c] = (s4 < 3 && c < 3) ? __ldg(p.w + n * 27 + c * 9 + r * 3 + s4) : 0.f;
      const uint2 pk = make_uint2(pack_h2(v[0], v[1]), pack_h2(v[2], v[3]));
      *reinterpret_cast<uint2*>(b_smem + r * 2048 + (n >> 3) * 256 + (s4 >> 1) * 128 + (n & 7) * 16 + (s4 & 1) * 8) = pk;
    }
  }
  __syncthreads();
  pdl_trigger();

  const int oh = p.height >> 1, ow = p.width >> 1;
  auto prefetch = [&](int t, float (&v)[kV2Iters][3]) {
    const int ptx = t % p.tiles_x;
    const int pt2 = t / p.tiles_x;
    const int pty = pt2 % p.tiles_y;
    const int pimg = pt2 / p.tiles_y;
    const int y0 = pty * kV2Rows - 1, x0 = ptx * kV2Cols - 1;
#pragma unroll
    for (int k = 0; k < kV2Iters; ++k) {
      const int i = tid + k * 128;
      const int r = i / kV2PC, c = i - r * kV2PC;
      const int iy = y0 + r, ix = x0 + c;
      const bool ok = i < kV2Pixels && iy >= 0 && iy < p.height && ix >= 0 && ix < p.width;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        if (kIn == kInLut) v[k][ch] = ok ? lut_pixel(p.x, p.lut, pimg, ch, iy, ix, p.height, p.width) : 0.f;
        else v[k][ch] = ok ? __ldg(reinterpret_cast<const float*>(p.x) + ((static_cast<long long>(pimg) * 3 + ch) * p.height + iy) * p.width + ix) : 0.f;
      }
    }
  };
  float pre[kV2Iters][3];
  if (static_cast<int>(blockIdx.x) < p.num_tiles) prefetch(blockIdx.x, pre);

  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int tx = tile % p.tiles_x;
    const int t2 = tile / p.tiles_x;
    const int ty = t2 % p.tiles_y;
    const int img = t2 / p.tiles_y;
    __syncthreads();                                // the previous tile's wgmma and copy-out are done with the patch and the stage
#pragma unroll
    for (int k = 0; k < kV2Iters; ++k) {
      const int i = tid + k * 128;
      if (i < kV2Pixels) {
        const uint2 pk = make_uint2(pack_h2(pre[k][0], pre[k][1]), pack_h2(pre[k][2], 0.f));
        *reinterpret_cast<uint2*>(patch_e + i * 8) = pk;
        *reinterpret_cast<uint2*>(patch_o + 8 + i * 8) = pk;
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      float acc[4][32];
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int dy = j >> 1, dx = j & 1;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const uint32_t a_addr = (dx ? o_base + 8 : e_base) + ((dy + r) * kV2PC + dx) * 8 + h * 8 * (2 * kV2Pitch);
          wgmma_f16<kC64Out>(acc[j], make_kmajor_desc_noswz(a_addr, 16, 2 * kV2Pitch), make_kmajor_desc_noswz(b_base + r * 2048, 128, 256), r != 0);
        }
      }
      wgmma_commit();
      if (h == 0) {
        const int next = tile + gridDim.x;
        if (next < p.num_tiles) prefetch(next, pre);
      }
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < 4; ++j) fence_regs(acc[j]);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int m = 64 * h + 16 * warp + (lane >> 2) + 8 * hh;
        const int wy = m >> 3, wx = m & 7;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int c = 8 * jj + 2 * (lane & 3);
          const float s0 = __ldg(p.scale + c), s1 = __ldg(p.scale + c + 1), b0 = __ldg(p.shift + c), b1 = __ldg(p.shift + c + 1);
          if constexpr (kPool) {
            float best0 = -INFINITY, best1 = -INFINITY;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float t0 = acc[j][4 * jj + 2 * hh] * s0 + b0, t1 = acc[j][4 * jj + 2 * hh + 1] * s1 + b1;
              t0 = t0 > 0.f ? t0 : t0 * p.slope;
              t1 = t1 > 0.f ? t1 : t1 * p.slope;
              best0 = fmaxf(best0, t0);
              best1 = fmaxf(best1, t1);
            }
            const int py = ty * (kV2Rows / 2) + wy, px = tx * (kV2Cols / 2) + wx;
            *reinterpret_cast<uint32_t*>(p.y + ((static_cast<long long>(img) * oh + py) * ow + px) * kC64Out + c) = pack_h2(best0, best1);
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float t0 = acc[j][4 * jj + 2 * hh] * s0 + b0, t1 = acc[j][4 * jj + 2 * hh + 1] * s1 + b1;
              t0 = t0 > 0.f ? t0 : t0 * p.slope;
              t1 = t1 > 0.f ? t1 : t1 * p.slope;
              const int row = 2 * (wy - 8 * h) + (j >> 1), slot = wx + (j & 1) * 8;
              *reinterpret_cast<uint32_t*>(stage + (row * kV2Cols + slot) * (kC64Out * 2) + ((jj ^ wx) << 4) + (lane & 3) * 4) = pack_h2(t0, t1);
            }
          }
        }
      }
      if constexpr (!kPool) {
        __syncthreads();                            // the pass is staged
        // 16 rows x 128 chunks of 16 B: on every trip thread tid copies chunk g = tid % 8 of pixel col = tid / 8 of one row
        const int col = tid >> 3, g = tid & 7;
        const int src_off = ((col >> 1) + (col & 1) * 8) * (kC64Out * 2) + ((g ^ (col >> 1)) << 4);
        __half* dst = p.y + ((static_cast<long long>(img) * p.height + ty * kV2Rows + 16 * h) * p.width + tx * kV2Cols + col) * kC64Out + g * 8;
#pragma unroll 4
        for (int row = 0; row < kV2Rows / 2; ++row) {
          const uint4 q = *reinterpret_cast<const uint4*>(stage + row * (kV2Cols * kC64Out * 2) + src_off);
          *reinterpret_cast<uint4*>(dst + static_cast<long long>(row) * p.width * kC64Out) = q;
        }
        __syncthreads();                            // copied out before the next pass stages over it
      }
    }
  }
}

// lut == nullptr: x is fp32 NCHW; otherwise uint8 NHWC read through lut[3][256]
int conv0_c64_forward(const void* x, const float* lut, const float* w, const float* scale, const float* shift, float slope, void* y, int batch,
                      int height, int width, int pool, cudaStream_t stream) {
  YB_REQUIRE(x && w && scale && shift && y, "conv0_c64: null pointer");
  YB_REQUIRE(batch > 0 && height > 0 && width > 0 && height % kV2Rows == 0 && width % kV2Cols == 0,
             "conv0_c64: H must be a multiple of %d and W of %d (got %dx%d)", kV2Rows, kV2Cols, height, width);
  Conv0Params p;
  p.x = x; p.lut = lut; p.w = w; p.scale = scale; p.shift = shift; p.slope = slope; p.y = reinterpret_cast<__half*>(y);
  p.batch = batch; p.height = height; p.width = width;
  p.tiles_x = width / kV2Cols;
  p.tiles_y = height / kV2Rows;
  const long long tiles = static_cast<long long>(p.tiles_x) * p.tiles_y * batch;
  YB_REQUIRE(tiles < (1ll << 31), "conv0_c64: too many tiles");
  p.num_tiles = static_cast<int>(tiles);
  p.raw = 0;
  p.stats = nullptr;
  p.dbg = debug_word_device();
  const int max_ctas = sm_count() * kC0CtasPerSm;
  const int grid = p.num_tiles < max_ctas ? p.num_tiles : max_ctas;
  if (lut) {
    if (pool) conv0_c64_kernel<kInLut, true><<<grid, 128, 0, stream>>>(p);
    else conv0_c64_kernel<kInLut, false><<<grid, 128, 0, stream>>>(p);
  } else {
    if (pool) conv0_c64_kernel<kInF32, true><<<grid, 128, 0, stream>>>(p);
    else conv0_c64_kernel<kInF32, false><<<grid, 128, 0, stream>>>(p);
  }
  return check_launch("conv0_c64_kernel");
}

// ---------------------------------------------------------------------------------------------
// Weight gradient of the 64-filter first layer: dw[co][ci][r][s] = sum over (b, y, x) of x[b][ci][y + r - 1][x + s - 1] * dz[b][y][x][co], from
// the caller's fp32 NCHW image and the fp16 NHWC gradient of the layer's conv output.  The reduction runs over B*H*W pixels in 8 x 32 pixel
// tiles spread over persistent CTAs (4 per SM).  A CTA stages the haloed fp32 patch and the tile's dz (32 KB) in shared memory; thread
// (co = tid % 64, tap group tid / 64) owns the taps g, g + 4, ... (7 or 6 of the 27) of filter co and accumulates them in fp32 registers
// over all its tiles: per pixel one dz load (a warp reads 32 consecutive channels) and one broadcast patch load per tap.  The 27 x 64
// partial sums of every CTA are added into dw (zeroed first) with atomics.
constexpr int kCW0Rows = 8, kCW0Cols = 32, kCW0Pix = kCW0Rows * kCW0Cols;
constexpr int kCW0PR = kCW0Rows + 2, kCW0PC = kCW0Cols + 2;
constexpr int kCW0CtasPerSm = 4;

__global__ void __launch_bounds__(256, kCW0CtasPerSm) conv0_c64_wgrad_kernel(const float* __restrict__ x, const __half* __restrict__ dz,
                                                                            float* __restrict__ dw, int height, int width, int tiles_x,
                                                                            int tiles_y, int num_tiles) {
  __shared__ __align__(16) __half dzs[kCW0Pix * kC64Out];
  __shared__ float patch[3 * kCW0PR * kCW0PC];
  const int tid = threadIdx.x, co = tid & 63, tg = tid >> 6;
  int off[7];
#pragma unroll
  for (int j = 0; j < 7; ++j) {
    const int tap = tg + 4 * j < 27 ? tg + 4 * j : 0;
    off[j] = ((tap / 9) * kCW0PR + (tap % 9) / 3) * kCW0PC + tap % 3;
  }
  float acc[7];
#pragma unroll
  for (int j = 0; j < 7; ++j) acc[j] = 0.f;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int tx = tile % tiles_x;
    const int t2 = tile / tiles_x;
    const int ty = t2 % tiles_y;
    const int img = t2 / tiles_y;
    const int y0 = ty * kCW0Rows, x0 = tx * kCW0Cols;
    __syncthreads();                              // the previous tile's reads are done
    for (int i = tid; i < 3 * kCW0PR * kCW0PC; i += 256) {
      const int c = i / (kCW0PR * kCW0PC);
      const int rem = i - c * (kCW0PR * kCW0PC);
      const int r = rem / kCW0PC, col = rem - r * kCW0PC;
      const int iy = y0 - 1 + r, ix = x0 - 1 + col;
      patch[i] = (iy >= 0 && iy < height && ix >= 0 && ix < width)
                     ? __ldg(x + ((static_cast<long long>(img) * 3 + c) * height + iy) * width + ix) : 0.f;
    }
    // dz tile: 8 rows of 32 pixels x 128 B, each row contiguous in memory
#pragma unroll
    for (int k = 0; k < kCW0Pix * kC64Out / 8 / 256; ++k) {
      const int i = tid + k * 256;                // 16-byte chunk: row i / 256, chunk i % 256 of that row
      const int r = i >> 8, q = i & 255;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(dz + ((static_cast<long long>(img) * height + y0 + r) * width + x0) * kC64Out) + q);
      reinterpret_cast<uint4*>(dzs)[i] = v;
    }
    __syncthreads();
#pragma unroll 2
    for (int p = 0; p < kCW0Pix; ++p) {
      const float d = __half2float(dzs[p * kC64Out + co]);
      const int po = (p >> 5) * kCW0PC + (p & 31);
#pragma unroll
      for (int j = 0; j < 7; ++j) acc[j] = fmaf(patch[off[j] + po], d, acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 7; ++j)
    if (tg + 4 * j < 27) atomicAdd(dw + co * 27 + tg + 4 * j, acc[j]);
}

int conv0_c64_wgrad(const float* x, const void* dz, float* dw, int batch, int height, int width, cudaStream_t stream) {
  YB_REQUIRE(x && dz && dw, "conv0_c64_wgrad: null pointer");
  YB_REQUIRE(batch > 0 && height > 0 && width > 0 && height % kCW0Rows == 0 && width % kCW0Cols == 0,
             "conv0_c64_wgrad: H must be a multiple of %d and W of %d (got %dx%d)", kCW0Rows, kCW0Cols, height, width);
  YB_CUDA(cudaMemsetAsync(dw, 0, 64 * 27 * sizeof(float), stream));
  const int tiles_x = width / kCW0Cols, tiles_y = height / kCW0Rows;
  const long long tiles = static_cast<long long>(tiles_x) * tiles_y * batch;
  YB_REQUIRE(tiles < (1ll << 31), "conv0_c64_wgrad: too many tiles");
  const int cap = sm_count() * kCW0CtasPerSm;
  const int grid = tiles < cap ? static_cast<int>(tiles) : cap;
  conv0_c64_wgrad_kernel<<<grid, 256, 0, stream>>>(x, reinterpret_cast<const __half*>(dz), dw, height, width, tiles_x, tiles_y,
                                                   static_cast<int>(tiles));
  return check_launch("conv0_c64_wgrad_kernel");
}

}  // namespace yb
