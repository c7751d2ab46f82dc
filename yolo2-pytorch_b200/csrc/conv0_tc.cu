// conv0 (layers1.0): 3x3 conv, Cin = 3 -> Cout = 32, + folded BN + leaky-ReLU + 2x2 max-pool, on the
// tensor cores.  Replaces nn.Conv2d(3,32,3,pad 1) -> BatchNorm2d -> LeakyReLU -> MaxPool2d(2)
// (reference model/yolo2.py:78-79) and doubles as the layout boundary: it reads the caller's
// image batch (fp32 NCHW as the reference's ToTensor produces it, or raw uint8 NHWC frames scaled
// by 1/255 == torchvision ToTensor) and writes the first fp16 NHWC activation.
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
  const void* x;        // fp32 NCHW [B,3,H,W] or uint8 NHWC [B,H,W,3]
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

template <bool kU8>
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
        if (kU8) {
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
// registers over all of the CTA's tiles and are reduced once at the end (p.stats: double [2][32], as yb_bn_stats).
constexpr int kV2StageBytes = kV2Rows * kV2Cols * kC0Out * 2;   // 32 KB

template <bool kU8, bool kRaw>
__global__ void __launch_bounds__(128, kC0CtasPerSm) conv0_k16_kernel(const Conv0Params p) {
  __shared__ __align__(128) uint8_t stage[kRaw ? kV2StageBytes : 16];
  __shared__ float s_stats[2 * kC0Out];
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
          if (kU8) val = static_cast<float>(__ldg(reinterpret_cast<const uint8_t*>(p.x) + ((static_cast<long long>(pimg) * p.height + iy) * p.width + ix) * 3 + ch)) * (1.f / 255.f);
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
  if (kRaw && tid < 2 * kC0Out) s_stats[tid] = 0.f;

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
      // the next iteration's __syncthreads (after the patch is written) orders this copy-out before the next tile's staging stores
    }
  }
  if (kRaw && p.stats != nullptr) {
    // lanes with equal (lane & 3) hold the same 8 channels
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
        atomicAdd(&s_stats[(tid & 3) * 8 + e], st1[e]);
        atomicAdd(&s_stats[kC0Out + (tid & 3) * 8 + e], st2[e]);
      }
    }
    __syncthreads();
    if (tid < 2 * kC0Out) atomicAdd(p.stats + tid, static_cast<double>(s_stats[tid]));
  }
}

int conv0_tc_forward(const void* x, int x_is_u8, const float* w, const float* scale, const float* shift, float slope, void* y, int batch,
                     int height, int width, int cout, int raw, double* stats, cudaStream_t stream) {
  YB_REQUIRE(x && w && y && (raw || (scale && shift)), "conv0: null pointer");
  YB_REQUIRE(cout == kC0Out, "conv0: Cout=%d unsupported (32)", cout);
  YB_REQUIRE(batch > 0 && height > 0 && width > 0 && height % kT0Rows == 0 && width % kT0Cols == 0,
             "conv0: H must be a multiple of %d and W of %d (got %dx%d)", kT0Rows, kT0Cols, height, width);
  // operands-in-place form when the shape tiles 32 x 16 (every multiple of 32, i.e. every Darknet input); YB_CONV0_V1=1 forces the first form
  static const int force_v1 = getenv("YB_CONV0_V1") ? atoi(getenv("YB_CONV0_V1")) : 0;
  const bool v2 = !force_v1 && height % kV2Rows == 0 && width % kV2Cols == 0;
  Conv0Params p;
  p.x = x; p.w = w; p.scale = scale; p.shift = shift; p.slope = slope; p.y = reinterpret_cast<__half*>(y);
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
      conv0_k16_kernel<true, false><<<grid, 128, 0, stream>>>(p);
    } else if (raw) {
      conv0_k16_kernel<false, true><<<grid, 128, 0, stream>>>(p);
    } else {
      conv0_k16_kernel<false, false><<<grid, 128, 0, stream>>>(p);
    }
    return check_launch("conv0_k16_kernel");
  }
  if (x_is_u8) conv0_tc_kernel<true><<<grid, 128, 0, stream>>>(p);
  else conv0_tc_kernel<false><<<grid, 128, 0, stream>>>(p);
  return check_launch("conv0_tc_kernel");
}

}  // namespace yb
