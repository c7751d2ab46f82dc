// K1: convolution as an implicit GEMM on the Hopper tensor cores (wgmma), sm_90a.
//
// Replaces the reference's  nn.Conv2d -> nn.BatchNorm2d(eval) -> nn.LeakyReLU(0.1)  unit
// (reference model/yolo2.py:49-65) for k in {1,3}, stride 1, pad (k-1)/2.
//
//   D[M = B*H*W pixels, N = Cout] = A[M, K = k*k*Cin] * W[N, K]^T
//
//   * A is never materialised: each K-block (one filter tap, BK input channels) of a 128-pixel
//     M-tile is fetched by ONE im2col-mode TMA (cp.async.bulk.tensor.4d...im2col) straight from
//     the NHWC fp16 activation into 128B- (or 64B-) swizzled shared memory; halo pixels are
//     zero-filled by the TMA unit.  W (KRSC fp16, K-major) comes in by a tiled 2D TMA.
//   * one warpgroup issues wgmma (M=64 x2, N=BN, K=16) with the fp32 accumulator in registers, then
//     parks the finished tile in a shared-memory accumulator (yb_ptx.cuh) and starts the next tile,
//     so the epilogue of tile i overlaps the mainloop of tile i+1;
//   * the epilogue warps read that tile one pixel row per thread, apply the folded BatchNorm (fp32
//     scale/shift per channel) + leaky-ReLU and store fp16 NHWC (optionally into a channel slice of a
//     wider buffer, which is how torch.cat at yolo2.py:129 disappears) or fp32 NCHW (the head, the
//     tensor the reference hands to the decoder).
//   * persistent: grid = min(#tiles, #SMs); warps 0..3 = MMA warpgroup, warp 4 = TMA producer,
//     warps 5..8 = epilogue (rows 32 * (warp - 5) .. + 31 of the tile).
#include "yb_common.h"
#include "yb_ptx.cuh"
#include <stdlib.h>

namespace yb {

struct ConvParams {
  int m_total;      // B*H*W
  int height, width;
  int cin, cout;
  int ksize, pad;
  int kb_per_tap;   // Cin / BK
  int num_kb;       // ksize*ksize*kb_per_tap
  int m_tiles, n_tiles;
  int a_im2col;     // 1: im2col TMA, 0: plain 2D tiled TMA over [M, Cin] (1x1 only)
  const float* scale;
  const float* shift;
  float slope;
  void* y;
  long long y_ld;   // fp16 NHWC: elements per pixel row of the destination buffer
  int y_ch_off;     // fp16 NHWC: first destination channel
  int out_mode;     // 0: fp16 NHWC, 1: fp32 NCHW
  int hw;           // H*W
  int skip;         // profiling ablation (results are garbage): 1 = no A loads, 2 = no B loads, 4 = no MMA, 8 = no stores
  int* dbg;
  // stream-K (streamk != 0): the tiles x K-blocks iteration space is cut into gridDim.x equal contiguous ranges, so a
  // layer whose tile count does not fill the SMs (13x13 at batch 32: 169 tiles of 128 x 128 on 132 SMs) still keeps every SM busy.  A CTA
  // whose range ends inside a tile dumps that partial fp32 accumulator to ws[blockIdx] and raises flags[blockIdx];
  // the CTA that holds the tile's last K-block adds the partials of the (lower-numbered) CTAs and runs the epilogue.
  int streamk;
  int sk_base, sk_rem;         // units per CTA = sk_base (+1 for the first sk_rem CTAs)
  float* ws;                   // [gridDim.x][MT][BN/32][128][32] fp32
  unsigned* flags;             // [gridDim.x], 0 = empty, 1 = partial ready (reset by the consumer)
  unsigned long long* trace;   // optional (yb_conv_set_trace): block 0 records clock64() per pipeline event, 3 roles x 256 slots
  // optional (training): per-channel sum and sum of squares of the STORED (fp16-rounded) outputs, added into
  // stats[0..Cout) / stats[Cout..2Cout) -- the batch statistics of train-mode BatchNorm without a second pass over z
  double* stats;
  // split-precision ("strict") mode.  The reduction dimension of the GEMM is a concatenation of fp16 terms,
  //   A = [a_hi | a_lo | a_hi] (channels of one pixel),  W = [w_hi | w_hi | w_lo] (per tap),
  // so a_hi*w_hi + a_lo*w_hi + a_hi*w_lo accumulate into ONE fp32 accumulator: the fp16 rounding of either operand
  // (2^-11 relative, the source of the 1.6e-3 end-to-end drift) drops to ~2^-22.  `cin` is then the concatenated width,
  // `a_wrap` the number of channels the activation tensor really holds (C or 2C): channel offsets past it wrap around.
  // `lo_off` != 0: the epilogue also stores lo = fp16(v - fp32(fp16(v))) at y + lo_off (fp16 NHWC only).
  int a_wrap;
  long long lo_off;
  // fp16 NHWC output through shared memory + TMA store (tmap_y): each epilogue warp stages 32 rows x 64 channels (128B-swizzled) and
  // one lane ships them with a single bulk store, instead of per-thread 16 B stores that write 32 half-used sectors per instruction
  // (lanes = pixels, 2*y_ld bytes apart).
  int tma_store;
};

// role 0 = TMA producer, 1 = MMA issuer, 2 = epilogue thread 0; slot = running event index of that role
#define YB_TRACE(role, slot) do { if (p.trace != nullptr && blockIdx.x == 0 && (slot) < 256) p.trace[(role) * 256 + (slot)] = clock64(); } while (0)


constexpr int BM = 128;

constexpr int UMMA_K = 16;
constexpr int kMmaThreads = 128;                // warps 0..3: the MMA warpgroup
constexpr int kProducerWarp = 4;
constexpr int kEpiWarp0 = 5;                    // warps 5..8: epilogue
constexpr int kEpiThreads = 128;
constexpr int kThreads = kMmaThreads + 32 + kEpiThreads;
constexpr int kSmemLimit = 232448;              // 227 KB: the per-block opt-in maximum of sm_90

// Work iteration shared by the three warp roles.  Plain mode: whole tiles, strided over the CTAs.  Stream-K mode: the
// CTA's unit range [s, e) (unit = one K-block of one tile) is walked from its END backwards, one tile segment at a
// time, so that the only segment that can stop short of its tile's last K-block is the first one processed -- its
// partial sums are needed by a HIGHER-numbered CTA, which reaches that tile last.  Waits therefore only ever point at
// lower block ids and at work those CTAs do first.
struct WorkIter {
  int tile, kb0, kb1;
  int streamk, num_kb, num_tiles, stride, s, cur_end;
  __device__ __forceinline__ static int sk_start(int c, int base, int rem) { return c * base + (c < rem ? c : rem); }
  __device__ __forceinline__ WorkIter(const ConvParams& p, int unit_id, int num_units, int ntiles) {
    streamk = p.streamk; num_kb = p.num_kb; num_tiles = ntiles; stride = num_units;
    if (streamk) {
      s = sk_start(unit_id, p.sk_base, p.sk_rem);
      cur_end = sk_start(unit_id + 1, p.sk_base, p.sk_rem);
      tile = 0; kb0 = 0; kb1 = 0;
      advance();
    } else {
      tile = unit_id; kb0 = 0; kb1 = num_kb; s = 0; cur_end = 0;
    }
  }
  __device__ __forceinline__ void advance() {   // stream-K only
    if (cur_end <= s) { tile = num_tiles; return; }
    tile = (cur_end - 1) / num_kb;
    const int tile_start = tile * num_kb;
    const int seg_start = s > tile_start ? s : tile_start;
    kb0 = seg_start - tile_start;
    kb1 = cur_end - tile_start;
    cur_end = seg_start;
  }
  __device__ __forceinline__ bool valid() const { return tile < num_tiles; }
  __device__ __forceinline__ void next() { if (streamk) advance(); else tile += stride; }
};

__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// MT = number of 128-pixel M-subtiles per CTA tile (1 or 2).  MT = 2 makes the CTA tile 256 x BN: both
// subtiles reuse the same weight (B) tile from shared memory, halving the L2->SM weight traffic per MAC.
// The MMA warpgroup holds MT * BN fp32 accumulators per thread, so MT * BN <= 128.
template <int BN, int BK, int MT>
struct ConvCfg {
  static constexpr int kSwizzle = BK * 2;                       // bytes per smem row
  static constexpr int kASubBytes = BM * BK * 2;
  static constexpr int kABytes = MT * kASubBytes;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccCols = MT * BN;                      // columns of the shared-memory accumulator tile
  static constexpr int kAccBytes = kAccCols * kAccPitch * 4;
  static constexpr bool kMergedA = (MT == 2);                   // A tile fetched by one 256-pixel TMA box
  static constexpr int kRowsPerTile = BM * MT;
  static constexpr int kOutBytes = BM * 128;                    // TMA-store staging: one 32-row x 64-channel fp16 slice (4 KB) per epilogue warp
  static constexpr int kFixedBytes = kAccBytes + kOutBytes + 1024 /*align slack*/ + 2 * 2 * BN * 4 /*scale/shift x2*/ + 2 * BN * 4 /*stats*/ + 256 /*barriers*/;
  static constexpr int kStages = ((kSmemLimit - kFixedBytes) / kStageBytes) > 8 ? 8 : ((kSmemLimit - kFixedBytes) / kStageBytes);
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(kAccCols <= 128, "accumulator does not fit the MMA warpgroup's registers");
  static_assert(kStages >= 2, "shared memory budget");
};

template <int BN, int BK, int MT>
__global__ void __launch_bounds__(kThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_y, const ConvParams p) {
  using Cfg = ConvCfg<BN, BK, MT>;
  constexpr int kStages = Cfg::kStages;
  constexpr bool kMergedA = Cfg::kMergedA;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the swizzle atoms
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t smem_a = smem_base;
  const uint32_t smem_b = smem_base + kStages * Cfg::kABytes;
  const uint32_t smem_o = smem_base + kStages * Cfg::kStageBytes;                       // 1024-aligned: stage sizes are multiples of 1 KB
  float* sacc = reinterpret_cast<float*>(smem_gen + kStages * Cfg::kStageBytes + Cfg::kOutBytes);
  float* ep_scale = sacc + Cfg::kAccCols * kAccPitch;                                   // [2][BN]
  float* ep_shift = ep_scale + 2 * BN;                                                  // [2][BN]
  float* ep_stats = ep_shift + 2 * BN;                                                  // [2][BN] sum, sum of squares of this tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(ep_stats + 2 * BN);
  const uint32_t bar_full = smem_u32(bars);                 // [kStages]
  const uint32_t bar_empty = bar_full + 8 * kStages;        // [kStages]
  const uint32_t bar_tfull = bar_empty + 8 * kStages;       // accumulator tile written
  const uint32_t bar_tempty = bar_tfull + 8;                // accumulator tile read

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.m_tiles * p.n_tiles;
  const int unit_id = static_cast<int>(blockIdx.x);
  const int num_units = static_cast<int>(gridDim.x);

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, 4);                      // one arrival per MMA warp
    }
    mbar_init(bar_tfull, 4);
    mbar_init(bar_tempty, 4);
    fence_mbar_init();
    fence_proxy_async_smem();
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (p.tma_store) tma_prefetch_desc(&tmap_y);
  }
  __syncthreads();
  // PDL: everything above (barrier init, descriptor prefetch) overlapped the tail of the previous kernel of the
  // stream; nothing below may run before that kernel's outputs (our activations / the stream-K workspace) are complete
  pdl_trigger();
  pdl_wait();

  if (warp == kProducerWarp) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      int tr_p = 0;
      for (WorkIter it(p, unit_id, num_units, num_tiles); it.valid(); it.next()) {
        const int tile = it.tile;
        const int n_tile = tile % p.n_tiles;
        const int m_tile = tile / p.n_tiles;
        const int m_cta = m_tile * Cfg::kRowsPerTile;
        int img[MT], h0[MT], w0[MT];
        int nsub = 0;                      // subtiles that start inside the tensor (the rest are skipped)
#pragma unroll
        for (int t = 0; t < MT; ++t) {
          const int ms = m_cta + t * BM;
          if (ms < p.m_total) nsub = t + 1;
          img[t] = ms / p.hw;
          const int rem = ms - img[t] * p.hw;
          h0[t] = rem / p.width;
          w0[t] = rem - h0[t] * p.width;
        }
        if (p.skip & 1) nsub = 0;
        if (kMergedA && nsub) nsub = MT;      // the merged box always transfers (and zero-fills) both subtiles
        const uint32_t tx_bytes = nsub * Cfg::kASubBytes + ((p.skip & 2) ? 0 : Cfg::kBBytes);
        for (int kb = it.kb0; kb < it.kb1; ++kb) {
          const int tap = kb / p.kb_per_tap;
          const int c0 = (kb - tap * p.kb_per_tap) * BK;    // offset inside the (possibly concatenated) weight row of this tap
          const int ca = c0 >= p.a_wrap ? c0 - p.a_wrap : c0;   // activation channel (split mode: the hi part is read twice)
          const int r = tap / p.ksize;
          const int s = tap - r * p.ksize;
          mbar_wait(bar_empty + 8 * stage, phase ^ 1, p.dbg, 0x100 | stage);
          YB_TRACE(0, tr_p); ++tr_p;
          const uint32_t full = bar_full + 8 * stage;
          mbar_arrive_expect_tx(full, tx_bytes);
          if (kMergedA) {
            // one TMA box covers both 128-pixel subtiles (the tensor map's box is BM * MT pixels): the im2col-mode TMA has
            // a large per-instruction cost, rows past the tensor end are zero-filled
            if (!(p.skip & 1)) {
              const uint32_t dst = smem_a + stage * Cfg::kABytes;
              if (p.a_im2col) tma_load_im2col_4d(dst, &tmap_a, full, ca, w0[0] - p.pad, h0[0] - p.pad, img[0], static_cast<uint16_t>(s), static_cast<uint16_t>(r));
              else tma_load_2d(dst, &tmap_a, full, ca, m_cta);
            }
          } else {
#pragma unroll
          for (int t = 0; t < MT; ++t) {
            if (t < nsub) {
              const uint32_t dst = smem_a + stage * Cfg::kABytes + t * Cfg::kASubBytes;
              if (p.a_im2col) tma_load_im2col_4d(dst, &tmap_a, full, ca, w0[t] - p.pad, h0[t] - p.pad, img[t], static_cast<uint16_t>(s), static_cast<uint16_t>(r));
              else tma_load_2d(dst, &tmap_a, full, ca, m_cta + t * BM);
            }
          }
          }
          if (!(p.skip & 2)) tma_load_2d(smem_b + stage * Cfg::kBBytes, &tmap_b, full, tap * p.cin + c0, n_tile * BN);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp < kProducerWarp) {
    // ===================== MMA warpgroup =====================
    float acc[MT][2][BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    uint32_t acc_phase = 0;
    int tr_m = 0;
    for (WorkIter it(p, unit_id, num_units, num_tiles); it.valid(); it.next()) {
      const int kb_first = it.kb0, kb_last = it.kb1 - 1;
      int prev = -1;
      for (int kb = kb_first; kb <= kb_last; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase, p.dbg, 0x300 | stage);
        if (threadIdx.x == 0) { YB_TRACE(1, tr_m); ++tr_m; }
        if (!(p.skip & 4)) {
          const uint64_t bdesc = make_kmajor_desc<Cfg::kSwizzle>(smem_b + stage * Cfg::kBBytes);
          wgmma_fence();
#pragma unroll
          for (int t = 0; t < MT; ++t) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint64_t adesc = make_kmajor_desc<Cfg::kSwizzle>(smem_a + stage * Cfg::kABytes + t * Cfg::kASubBytes + h * 64 * Cfg::kSwizzle);
#pragma unroll
              for (int k = 0; k < BK / UMMA_K; ++k)      // advance 16 fp16 = 32 bytes inside the swizzled row: +2 in the 16-byte address field
                wgmma_f16<BN>(acc[t][h], adesc + 2 * k, bdesc + 2 * k, ((kb - kb_first) | k) != 0);
            }
          }
          wgmma_commit();
          // one group in flight: the previous K-block's MMAs have retired, so its smem slot can be refilled
          wgmma_wait<1>();
        }
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(bar_empty + 8 * prev); }
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int t = 0; t < MT; ++t)
#pragma unroll
        for (int h = 0; h < 2; ++h) fence_regs(acc[t][h]);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
      // park the tile for the epilogue once it has drained the previous one
      mbar_wait(bar_tempty, acc_phase ^ 1, p.dbg, 0x200);
#pragma unroll
      for (int t = 0; t < MT; ++t)
#pragma unroll
        for (int h = 0; h < 2; ++h) sacc_store<BN>(sacc, h * 64, t * BN, acc[t][h]);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_tfull);
      acc_phase ^= 1;
    }
  } else {
    // ===================== epilogue (warps 5..8) =====================
    const int q = warp - kEpiWarp0;            // tile rows 32 q .. 32 q + 31
    const int et = threadIdx.x - kEpiWarp0 * 32;   // 0 .. kEpiThreads - 1
    uint32_t acc_phase = 0;
    int buf = 0;
    for (WorkIter it(p, unit_id, num_units, num_tiles); it.valid(); it.next()) {
      const int tile = it.tile;
      const int n_tile = tile % p.n_tiles;
      const int m_tile = tile / p.n_tiles;
      const int n0 = n_tile * BN;
      // stream-K roles of this segment: it either stops short of the tile's last K-block (dump the partial sums), or
      // finishes a tile whose first K-blocks were summed by lower-numbered CTAs (collect their partials first)
      const bool sk_dump = it.kb1 < p.num_kb;
      const bool sk_collect = !sk_dump && it.kb0 > 0;
      int sk_lo = 0;                           // partials come from CTAs [sk_lo, blockIdx.x)
      const int m_cta = m_tile * Cfg::kRowsPerTile;
      // stage this tile's per-channel scale/shift (double-buffered: a warp can be one tile ahead)
      float* sc = ep_scale + buf * BN;
      float* sh = ep_shift + buf * BN;
      buf ^= 1;
      for (int i = et; i < BN; i += kEpiThreads) {
        const int c = n0 + i;
        sc[i] = (c < p.cout) ? __ldg(p.scale + c) : 0.f;
        sh[i] = (c < p.cout) ? __ldg(p.shift + c) : 0.f;
        if (p.stats != nullptr) { ep_stats[i] = 0.f; ep_stats[BN + i] = 0.f; }
      }
      if (sk_collect) {
        // the CTA whose range contains this tile's first unit, by inverting sk_start()
        const int u = tile * p.num_kb;
        const int wide = p.sk_rem * (p.sk_base + 1);
        sk_lo = u < wide ? u / (p.sk_base + 1) : p.sk_rem + (u - wide) / p.sk_base;
        if (et == 0) {
          for (int j = sk_lo; j < static_cast<int>(blockIdx.x); ++j) {
            uint32_t spins = 0;
            uint64_t t0 = 0;
            while (ld_acquire_gpu(p.flags + j) == 0u) {
              if ((++spins & 0x3FFu) == 0) {
                const uint64_t now = globaltimer_ns();
                if (t0 == 0) t0 = now;
                if (now - t0 > 4000000000ull) {
                  if (p.dbg != nullptr) { p.dbg[0] = 0x0BAD0500; p.dbg[1] = static_cast<int>(blockIdx.x); p.dbg[2] = j; p.dbg[3] = tile; __threadfence_system(); }
                  __trap();
                }
              }
            }
          }
        }
      }
      asm volatile("bar.sync 1, %0;" :: "n"(kEpiThreads) : "memory");
      mbar_wait(bar_tfull, acc_phase, p.dbg, 0x400);
      if (sk_dump) {
        float* wsp = p.ws + static_cast<size_t>(blockIdx.x) * (MT * BN * 128);
#pragma unroll 1
        for (int t = 0; t < MT; ++t) {
          if (m_cta + t * BM >= p.m_total) break;
#pragma unroll 1
          for (int cc = 0; cc < BN / 32; ++cc) {
            if (n0 + cc * 32 >= p.cout) break;
            uint32_t v[32];
            sacc_ld_x32(sacc, q * 32 + lane, t * BN + cc * 32, v);
            float4* dst = reinterpret_cast<float4*>(wsp + (static_cast<size_t>(t * (BN / 32) + cc) * 128 + q * 32 + lane) * 32);
#pragma unroll
            for (int g = 0; g < 8; ++g)
              dst[g] = make_float4(__uint_as_float(v[4 * g]), __uint_as_float(v[4 * g + 1]), __uint_as_float(v[4 * g + 2]), __uint_as_float(v[4 * g + 3]));
          }
        }
        __threadfence();
        asm volatile("bar.sync 1, %0;" :: "n"(kEpiThreads) : "memory");
        if (et == 0) st_release_gpu(p.flags + blockIdx.x, 1u);
        if (lane == 0) mbar_arrive(bar_tempty);
        acc_phase ^= 1;
        continue;
      }
#pragma unroll 1
      for (int t = 0; t < MT; ++t) {
        if (m_cta + t * BM >= p.m_total) break;   // warp-uniform: subtile entirely past the end
        const int row = m_cta + t * BM + q * 32 + lane;
        const bool row_ok = row < p.m_total;
        int img = 0, pix = 0;
        if (p.out_mode == 1) { img = row / p.hw; pix = row - img * p.hw; }
        if (p.tma_store) {
          // ---- fp16 NHWC through the staging buffer: 64 channels per bulk store ----
#pragma unroll 1
          for (int c2 = 0; c2 < BN / 64; ++c2) {
            if (n0 + c2 * 64 >= p.cout) break;
            uint4 pk[8];
            uint32_t vv[2][32];
            sacc_ld_x32(sacc, q * 32 + lane, t * BN + (c2 * 2) * 32, vv[0]);
            sacc_ld_x32(sacc, q * 32 + lane, t * BN + (c2 * 2 + 1) * 32, vv[1]);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int cc = c2 * 2 + hh;
              uint32_t (&v)[32] = vv[hh];
              const int cbase = n0 + cc * 32;
              if (sk_collect && cbase < p.cout) {
                for (int j = sk_lo; j < static_cast<int>(blockIdx.x); ++j) {
                  const float4* src = reinterpret_cast<const float4*>(p.ws + static_cast<size_t>(j) * (MT * BN * 128) +
                                                                      (static_cast<size_t>(t * (BN / 32) + cc) * 128 + q * 32 + lane) * 32);
#pragma unroll
                  for (int g = 0; g < 8; ++g) {
                    const float4 a = __ldcg(src + g);
                    v[4 * g] = __float_as_uint(__uint_as_float(v[4 * g]) + a.x);
                    v[4 * g + 1] = __float_as_uint(__uint_as_float(v[4 * g + 1]) + a.y);
                    v[4 * g + 2] = __float_as_uint(__uint_as_float(v[4 * g + 2]) + a.z);
                    v[4 * g + 3] = __float_as_uint(__uint_as_float(v[4 * g + 3]) + a.w);
                  }
                }
              }
              float f[32];
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                float x = __uint_as_float(v[j]) * sc[cc * 32 + j] + sh[cc * 32 + j];
                f[j] = x > 0.f ? x : x * p.slope;
              }
              if (p.stats != nullptr && cbase < p.cout) {
                float a1[32], a2[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                  const float r = row_ok ? __half2float(__float2half_rn(f[j])) : 0.f;
                  a1[j] = r; a2[j] = r * r;
                }
#pragma unroll
                for (int s = 16; s >= 1; s >>= 1) {
                  const bool up = (lane & s) != 0;
#pragma unroll
                  for (int j = 0; j < s; ++j) {
                    const float k1 = up ? a1[j + s] : a1[j], g1 = up ? a1[j] : a1[j + s];
                    const float k2 = up ? a2[j + s] : a2[j], g2 = up ? a2[j] : a2[j + s];
                    a1[j] = k1 + __shfl_xor_sync(0xffffffffu, g1, s);
                    a2[j] = k2 + __shfl_xor_sync(0xffffffffu, g2, s);
                  }
                }
                atomicAdd(&ep_stats[cc * 32 + lane], a1[0]);
                atomicAdd(&ep_stats[BN + cc * 32 + lane], a2[0]);
              }
#pragma unroll
              for (int g = 0; g < 4; ++g) {
                __half2 h0 = __floats2half2_rn(f[g * 8 + 0], f[g * 8 + 1]);
                __half2 h1 = __floats2half2_rn(f[g * 8 + 2], f[g * 8 + 3]);
                __half2 h2 = __floats2half2_rn(f[g * 8 + 4], f[g * 8 + 5]);
                __half2 h3 = __floats2half2_rn(f[g * 8 + 6], f[g * 8 + 7]);
                pk[hh * 4 + g].x = *reinterpret_cast<uint32_t*>(&h0);
                pk[hh * 4 + g].y = *reinterpret_cast<uint32_t*>(&h1);
                pk[hh * 4 + g].z = *reinterpret_cast<uint32_t*>(&h2);
                pk[hh * 4 + g].w = *reinterpret_cast<uint32_t*>(&h3);
              }
            }
            // Each epilogue warp ships its own 32 rows (4 KB of the staging tile) with its own bulk store: no block-level barrier in the
            // epilogue, so while one warp waits the others convert / store.  The warp's previous store must have drained its slice.
            if (lane == 0) tma_store_wait_read<0>();
            __syncwarp();
            {
              const uint32_t slice = smem_o + q * 4096 + lane * 128;
#pragma unroll
              for (int c = 0; c < 8; ++c) st_shared_v4(slice + ((c ^ (lane & 7)) << 4), pk[c]);
            }
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0 && !(p.skip & 8)) {
              tma_store_2d(&tmap_y, smem_o + q * 4096, n0 + c2 * 64, m_cta + t * BM + q * 32);      // rows >= M and channels >= Cout are clipped by the tensor map
              tma_store_commit();
            }
          }
          continue;
        }
#pragma unroll 1
        for (int cc = 0; cc < BN / 32; ++cc) {
          uint32_t v[32];
          sacc_ld_x32(sacc, q * 32 + lane, t * BN + cc * 32, v);
          const int cbase = n0 + cc * 32;
          if (cbase >= p.cout) continue;           // warp-uniform
          if (sk_collect) {
            for (int j = sk_lo; j < static_cast<int>(blockIdx.x); ++j) {
              const float4* src = reinterpret_cast<const float4*>(p.ws + static_cast<size_t>(j) * (MT * BN * 128) +
                                                                  (static_cast<size_t>(t * (BN / 32) + cc) * 128 + q * 32 + lane) * 32);
#pragma unroll
              for (int g = 0; g < 8; ++g) {
                const float4 a = __ldcg(src + g);
                v[4 * g] = __float_as_uint(__uint_as_float(v[4 * g]) + a.x);
                v[4 * g + 1] = __float_as_uint(__uint_as_float(v[4 * g + 1]) + a.y);
                v[4 * g + 2] = __float_as_uint(__uint_as_float(v[4 * g + 2]) + a.z);
                v[4 * g + 3] = __float_as_uint(__uint_as_float(v[4 * g + 3]) + a.w);
              }
            }
          }
          float f[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            float x = __uint_as_float(v[j]) * sc[cc * 32 + j] + sh[cc * 32 + j];
            f[j] = x > 0.f ? x : x * p.slope;
          }
          if (p.skip & 8) continue;
          if (p.stats != nullptr) {
            // column sums over this warp's 32 rows by recursive halving: after step s a lane keeps the half of its values
            // whose column bit s equals its lane bit s (31 shuffles per quantity); lane l ends up with column cbase + l
            float a1[32], a2[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const float r = row_ok ? __half2float(__float2half_rn(f[j])) : 0.f;      // statistics of the value that is stored
              a1[j] = r; a2[j] = r * r;
            }
#pragma unroll
            for (int s = 16; s >= 1; s >>= 1) {
              const bool up = (lane & s) != 0;
#pragma unroll
              for (int j = 0; j < s; ++j) {
                const float k1 = up ? a1[j + s] : a1[j], g1 = up ? a1[j] : a1[j + s];
                const float k2 = up ? a2[j + s] : a2[j], g2 = up ? a2[j] : a2[j + s];
                a1[j] = k1 + __shfl_xor_sync(0xffffffffu, g1, s);
                a2[j] = k2 + __shfl_xor_sync(0xffffffffu, g2, s);
              }
            }
            atomicAdd(&ep_stats[cc * 32 + lane], a1[0]);
            atomicAdd(&ep_stats[BN + cc * 32 + lane], a2[0]);
          }
          if (p.out_mode == 0) {
            if (row_ok) {
              __half* dst = reinterpret_cast<__half*>(p.y) + static_cast<long long>(row) * p.y_ld + p.y_ch_off + cbase;
#pragma unroll
              for (int g = 0; g < 4; ++g) {
                if (cbase + g * 8 < p.cout) {
                  uint4 pk;
                  __half2 h0 = __floats2half2_rn(f[g * 8 + 0], f[g * 8 + 1]);
                  __half2 h1 = __floats2half2_rn(f[g * 8 + 2], f[g * 8 + 3]);
                  __half2 h2 = __floats2half2_rn(f[g * 8 + 4], f[g * 8 + 5]);
                  __half2 h3 = __floats2half2_rn(f[g * 8 + 6], f[g * 8 + 7]);
                  pk.x = *reinterpret_cast<uint32_t*>(&h0);
                  pk.y = *reinterpret_cast<uint32_t*>(&h1);
                  pk.z = *reinterpret_cast<uint32_t*>(&h2);
                  pk.w = *reinterpret_cast<uint32_t*>(&h3);
                  *reinterpret_cast<uint4*>(dst + g * 8) = pk;
                  if (p.lo_off != 0) {
                    // residual of the fp16 rounding, itself rounded to fp16: hi + lo carries ~22 mantissa bits
                    const float2 r0 = __half22float2(h0), r1 = __half22float2(h1), r2 = __half22float2(h2), r3 = __half22float2(h3);
                    __half2 l0 = __floats2half2_rn(f[g * 8 + 0] - r0.x, f[g * 8 + 1] - r0.y);
                    __half2 l1 = __floats2half2_rn(f[g * 8 + 2] - r1.x, f[g * 8 + 3] - r1.y);
                    __half2 l2 = __floats2half2_rn(f[g * 8 + 4] - r2.x, f[g * 8 + 5] - r2.y);
                    __half2 l3 = __floats2half2_rn(f[g * 8 + 6] - r3.x, f[g * 8 + 7] - r3.y);
                    uint4 pl;
                    pl.x = *reinterpret_cast<uint32_t*>(&l0);
                    pl.y = *reinterpret_cast<uint32_t*>(&l1);
                    pl.z = *reinterpret_cast<uint32_t*>(&l2);
                    pl.w = *reinterpret_cast<uint32_t*>(&l3);
                    *reinterpret_cast<uint4*>(dst + p.lo_off + g * 8) = pl;
                  }
                }
              }
            }
          } else {
            if (row_ok) {
              float* dst = reinterpret_cast<float*>(p.y) + (static_cast<long long>(img) * p.cout + cbase) * p.hw + pix;
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                if (cbase + j < p.cout) dst[static_cast<long long>(j) * p.hw] = f[j];
              }
            }
          }
        }
      }  // M-subtiles
      // hand the accumulator tile back to the MMA warpgroup
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_tempty);
      if (p.stats != nullptr) {
        // this tile's column sums -> the global double accumulators (the bar.sync at the top of the next tile orders the
        // re-zeroing of ep_stats after these reads)
        asm volatile("bar.sync 1, %0;" :: "n"(kEpiThreads) : "memory");
        for (int i = et; i < BN; i += kEpiThreads) {
          if (n0 + i < p.cout) {
            atomicAdd(p.stats + n0 + i, static_cast<double>(ep_stats[i]));
            atomicAdd(p.stats + p.cout + n0 + i, static_cast<double>(ep_stats[BN + i]));
          }
        }
        asm volatile("bar.sync 1, %0;" :: "n"(kEpiThreads) : "memory");
      }
      if (sk_collect) {
        // every reader is done with the partials: hand the slots back (the next writer is a later launch)
        asm volatile("bar.sync 1, %0;" :: "n"(kEpiThreads) : "memory");
        for (int j = sk_lo + et; j < static_cast<int>(blockIdx.x); j += kEpiThreads) p.flags[j] = 0u;
      }
      acc_phase ^= 1;
    }
    if (p.tma_store && lane == 0) tma_store_wait<0>();     // every bulk store of this warp has landed before the CTA's shared memory goes away
  }
}

// ---------------------------------------------------------------------------------------------
// Halo-tile kernel for 3x3, Cin = 32 (layers1.2).  The im2col formulation above pulls every input pixel through the
// L2 -> SM path nine times (once per tap): 779 MB for 88 MB of input at batch 32.  Here an output tile is a 16 x 8 pixel
// rectangle and its 18 x 10 x 32ch input halo is fetched ONCE (11.5 KB instead of 72 KB) as four 8-channel planes
// [pixel][16 B].  In that layout a 3x3 tap is just a shifted window: 8 consecutive pixels of a halo row form one 8 x 16 B
// core matrix of the un-swizzled K-major operand format, the next output row is +10 pixels (SBO = 160 B) and the second
// K chunk is the next plane (LBO), so wgmma reads all nine taps straight out of the halo tile by moving the
// descriptor's start address by (r * 10 + s) * 16 B.  Weights stay resident in shared memory; the epilogue can
// apply the 2x2 max-pool that follows this layer (lane ^ 1 and lane ^ 8 hold the horizontal / vertical neighbours) and
// ships the tile with one TMA store, so the un-pooled activation never reaches HBM in inference.
// ---------------------------------------------------------------------------------------------
struct C32Params {
  int batch, height, width, cout;
  int tiles_w, tiles_h, num_tiles;
  const float* scale;
  const float* shift;
  float slope;
  int pool;
  int swap_lbo;   // testing: exchange LBO / SBO in the A descriptor
  int skip;
  int* dbg;
  unsigned long long* trace;
  double* stats;  // training forward: += per-channel sum / sum of squares of the stored values ([2][cout]); needs exact tiling, no pool
};

struct C32Cfg {
  static constexpr int TH = 16, TW = 8, HH = TH + 2, HW = TW + 2;
  static constexpr int kPlaneData = HH * HW * 16;                 // 2880 B written by one TMA box
  static constexpr int kPlane = (kPlaneData + 127) / 128 * 128;   // 2944: TMA destinations are 128 B aligned
  static constexpr int kHalo = 4 * kPlane;                        // 11776
  static constexpr int kStages = 4;
  static constexpr int BN = 64;
  static constexpr int kBTap = BN * 32 * 2;                       // 4 KB
  static constexpr int kBBytes = 9 * kBTap;                       // 36 KB resident
  static constexpr int kOutBytes = 128 * 128;                     // staging tile for the TMA store (2 per epilogue group)
  static constexpr int kGroups = 2;                               // epilogue groups of four warps, one accumulator tile each
  static constexpr int kAccBytes = BN * kAccPitch * 4;
  static constexpr int kEpiThreads = kGroups * 128;
  static constexpr int kThreads = 128 + 32 + kEpiThreads;         // MMA warpgroup, TMA warp, epilogue groups
  static constexpr int kSmemBytes = 1024 + kBBytes + 2 * kGroups * kOutBytes + kStages * kHalo + kGroups * kAccBytes + 2 * BN * 4 + 256 + 2 * BN * 4 /*stats*/;
  static_assert(kSmemBytes <= kSmemLimit, "c32: shared memory budget");
};

__global__ void __launch_bounds__(C32Cfg::kThreads, 1)
conv_c32_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                const __grid_constant__ CUtensorMap tmap_y, const C32Params p) {
  using Cfg = C32Cfg;
  constexpr int BN = Cfg::BN;
  constexpr int kGroups = Cfg::kGroups;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t smem_b = smem_base;
  const uint32_t smem_o = smem_b + Cfg::kBBytes;
  const uint32_t smem_h = smem_o + 2 * kGroups * Cfg::kOutBytes;
  float* sacc = reinterpret_cast<float*>(smem_gen + Cfg::kBBytes + 2 * kGroups * Cfg::kOutBytes + Cfg::kStages * Cfg::kHalo);  // [kGroups] tiles
  float* ep_scale = sacc + kGroups * BN * kAccPitch;
  float* ep_shift = ep_scale + BN;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ep_shift + BN);
  const uint32_t bar_full = smem_u32(bars);
  const uint32_t bar_empty = bar_full + 8 * Cfg::kStages;
  const uint32_t bar_tfull = bar_empty + 8 * Cfg::kStages;
  const uint32_t bar_tempty = bar_tfull + 8 * kGroups;
  const uint32_t bar_w = bar_tempty + 8 * kGroups;
  float* ep_stats = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);      // [2][BN], accumulated over all of this CTA's tiles
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < Cfg::kStages; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 4); }
    for (int i = 0; i < kGroups; ++i) { mbar_init(bar_tfull + 8 * i, 4); mbar_init(bar_tempty + 8 * i, 4); }
    mbar_init(bar_w, 1);
    fence_mbar_init();
    fence_proxy_async_smem();
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_y);
  }
  __syncthreads();
  pdl_trigger();        // an ordinary launch itself; lets a PDL successor set up while this grid drains

  if (warp == kProducerWarp) {
    if (lane == 0) {
      mbar_arrive_expect_tx(bar_w, Cfg::kBBytes);
      for (int t = 0; t < 9; ++t) tma_load_2d(smem_b + t * Cfg::kBTap, &tmap_w, bar_w, t * 32, 0);
      int stage = 0; uint32_t phase = 0; int tr = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int tw = tile % p.tiles_w;
        const int rest = tile / p.tiles_w;
        const int th = rest % p.tiles_h;
        const int n = rest / p.tiles_h;
        mbar_wait(bar_empty + 8 * stage, phase ^ 1, p.dbg, 0xB00 | stage);
        YB_TRACE(0, tr); ++tr;
        if (p.skip & 1) {
          mbar_arrive(bar_full + 8 * stage);
        } else {
          mbar_arrive_expect_tx(bar_full + 8 * stage, 4 * Cfg::kPlaneData);
          for (int c = 0; c < 4; ++c)
            tma_load_4d(smem_h + stage * Cfg::kHalo + c * Cfg::kPlane, &tmap_x, bar_full + 8 * stage, c * 8, tw * Cfg::TW - 1, th * Cfg::TH - 1, n);
        }
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp < kProducerWarp) {
    // MMA warpgroup: rows 0..63 of the 16 x 8 tile are output rows 0..7 (one 8-pixel core matrix each), rows 64..127 start
    // 8 halo rows further down
    const uint32_t lbo = p.swap_lbo ? Cfg::HW * 16 : Cfg::kPlane;
    const uint32_t sbo = p.swap_lbo ? Cfg::kPlane : Cfg::HW * 16;
    float acc[2][BN / 2];
    int stage = 0; uint32_t phase = 0; int tr = 0;
    mbar_wait(bar_w, 0, p.dbg, 0xB10);
    int local = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++local) {
      mbar_wait(bar_full + 8 * stage, phase, p.dbg, 0xB30 | stage);
      if (threadIdx.x == 0) { YB_TRACE(1, tr); ++tr; }
      const uint32_t halo = smem_h + stage * Cfg::kHalo;
      if (!(p.skip & 4)) {
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int t = 0; t < 9; ++t) {
            const uint32_t win = halo + ((h * 8 + t / 3) * Cfg::HW + (t % 3)) * 16;      // tap (r, s): window shifted by r rows, s pixels
            const uint64_t bdesc = make_kmajor_desc<64>(smem_b + t * Cfg::kBTap);
            wgmma_f16<BN>(acc[h], make_kmajor_desc_noswz(win, lbo, sbo), bdesc, t != 0);
            wgmma_f16<BN>(acc[h], make_kmajor_desc_noswz(win + 2 * Cfg::kPlane, lbo, sbo), bdesc + 2, 1);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
      }
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * stage);
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      // tile `local` goes to epilogue group local % kGroups, through that group's accumulator tile
      const int grp = local % kGroups;
      const uint32_t use = static_cast<uint32_t>(local / kGroups);
      mbar_wait(bar_tempty + 8 * grp, (use & 1) ^ 1, p.dbg, 0xB20 | grp);
      float* tile_acc = sacc + grp * BN * kAccPitch;
      sacc_store<BN>(tile_acc, 0, 0, acc[0]);
      sacc_store<BN>(tile_acc, 64, 0, acc[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_tfull + 8 * grp);
    }
  } else {
    // Independent epilogue groups of four warps take the tiles round-robin: one tile's epilogue is a chain of latencies
    // (accumulator reads, two named barriers, the async-proxy fence, the TMA store issue), so kGroups of them in flight
    // multiply the tile rate.
    const int ew = warp - kEpiWarp0;
    const int q = ew & 3;                   // tile pixels 32 q .. 32 q + 31: rows 4q .. 4q+3
    const int grp = ew >> 2;
    const int gt = (threadIdx.x - kEpiWarp0 * 32) & 127;
    const int et = threadIdx.x - kEpiWarp0 * 32;
    const float* tile_acc = sacc + grp * BN * kAccPitch;
    int tr = 0;
    for (int i = et; i < BN; i += Cfg::kEpiThreads) {
      ep_scale[i] = (i < p.cout) ? __ldg(p.scale + i) : 0.f;
      ep_shift[i] = (i < p.cout) ? __ldg(p.shift + i) : 0.f;
      ep_stats[i] = 0.f; ep_stats[BN + i] = 0.f;
    }
    asm volatile("bar.sync 8, %0;" :: "n"(Cfg::kEpiThreads) : "memory");
    const int m = q * 32 + lane;            // tile-local pixel: row m >> 3, column m & 7
    int srow = m;
    bool writer = true;
    if (p.pool) {
      writer = ((lane & 1) == 0) && ((lane & 8) == 0);
      srow = (q * 2 + (lane >> 4)) * 4 + ((lane & 7) >> 1);       // pooled pixel: row (m >> 3) / 2, column (m & 7) / 2
    }
    int local = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++local) {
      if (local % kGroups != grp) continue;
      const uint32_t use = static_cast<uint32_t>(local / kGroups);
      const int tw = tile % p.tiles_w;
      const int rest = tile / p.tiles_w;
      const int th = rest % p.tiles_h;
      const int n = rest / p.tiles_h;
      mbar_wait(bar_tfull + 8 * grp, use & 1, p.dbg, 0xB40 | grp);
      if (et == 0) { YB_TRACE(2, tr); ++tr; }
      uint4 pk[8];
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        uint32_t v[32];
        sacc_ld_x32(tile_acc, m, half * 32, v);
        if (half == 1) {                      // both halves are in registers: hand the accumulator tile back
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_tempty + 8 * grp);
        }
        float f[32];
#pragma unroll
        for (int j4 = 0; j4 < 8; ++j4) {
          const float4 s4 = *reinterpret_cast<const float4*>(ep_scale + half * 32 + j4 * 4);
          const float4 h4 = *reinterpret_cast<const float4*>(ep_shift + half * 32 + j4 * 4);
          const float x0 = __uint_as_float(v[j4 * 4 + 0]) * s4.x + h4.x, x1 = __uint_as_float(v[j4 * 4 + 1]) * s4.y + h4.y;
          const float x2 = __uint_as_float(v[j4 * 4 + 2]) * s4.z + h4.z, x3 = __uint_as_float(v[j4 * 4 + 3]) * s4.w + h4.w;
          f[j4 * 4 + 0] = x0 > 0.f ? x0 : x0 * p.slope; f[j4 * 4 + 1] = x1 > 0.f ? x1 : x1 * p.slope;
          f[j4 * 4 + 2] = x2 > 0.f ? x2 : x2 * p.slope; f[j4 * 4 + 3] = x3 > 0.f ? x3 : x3 * p.slope;
        }
        if (p.stats != nullptr) {
          // column sums over this warp's 32 pixels by recursive halving (as conv_igemm_kernel): lane l ends up with channel half * 32 + l
          float a1[32], a2[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float r = __half2float(__float2half_rn(f[j]));          // statistics of the value that is stored
            a1[j] = r; a2[j] = r * r;
          }
#pragma unroll
          for (int sft = 16; sft >= 1; sft >>= 1) {
            const bool up = (lane & sft) != 0;
#pragma unroll
            for (int j = 0; j < sft; ++j) {
              const float k1 = up ? a1[j + sft] : a1[j], g1 = up ? a1[j] : a1[j + sft];
              const float k2 = up ? a2[j + sft] : a2[j], g2 = up ? a2[j] : a2[j + sft];
              a1[j] = k1 + __shfl_xor_sync(0xffffffffu, g1, sft);
              a2[j] = k2 + __shfl_xor_sync(0xffffffffu, g2, sft);
            }
          }
          atomicAdd(&ep_stats[half * 32 + lane], a1[0]);
          atomicAdd(&ep_stats[BN + half * 32 + lane], a2[0]);
        }
        if (p.pool) {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            f[j] = fmaxf(f[j], __shfl_xor_sync(0xffffffffu, f[j], 1));
            f[j] = fmaxf(f[j], __shfl_xor_sync(0xffffffffu, f[j], 8));
          }
        }
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          __half2 h0 = __floats2half2_rn(f[g * 8 + 0], f[g * 8 + 1]), h1 = __floats2half2_rn(f[g * 8 + 2], f[g * 8 + 3]);
          __half2 h2 = __floats2half2_rn(f[g * 8 + 4], f[g * 8 + 5]), h3 = __floats2half2_rn(f[g * 8 + 6], f[g * 8 + 7]);
          pk[half * 4 + g].x = *reinterpret_cast<uint32_t*>(&h0); pk[half * 4 + g].y = *reinterpret_cast<uint32_t*>(&h1);
          pk[half * 4 + g].z = *reinterpret_cast<uint32_t*>(&h2); pk[half * 4 + g].w = *reinterpret_cast<uint32_t*>(&h3);
        }
      }
      const uint32_t obuf = smem_o + (grp * 2 + (use & 1)) * Cfg::kOutBytes;
      if (gt == 0) tma_store_wait_read<1>();      // this group's store from two of its tiles ago has drained the buffer
      asm volatile("bar.sync %0, 128;" :: "r"(1 + grp) : "memory");
      if (et == 0) { YB_TRACE(2, tr); ++tr; }
      if (writer) {
#pragma unroll
        for (int c = 0; c < 8; ++c) st_shared_v4(obuf + srow * 128 + ((c ^ (srow & 7)) << 4), pk[c]);
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" :: "r"(1 + grp) : "memory");
      if (gt == 0 && !(p.skip & 8)) {
        if (p.pool) tma_store_4d(&tmap_y, obuf, 0, tw * (Cfg::TW / 2), th * (Cfg::TH / 2), n);
        else tma_store_4d(&tmap_y, obuf, 0, tw * Cfg::TW, th * Cfg::TH, n);
        tma_store_commit();
      }
      if (et == 0) { YB_TRACE(2, tr); ++tr; }
    }
    if (gt == 0) tma_store_wait<0>();
    if (p.stats != nullptr) {
      asm volatile("bar.sync 8, %0;" :: "n"(Cfg::kEpiThreads) : "memory");       // every group has added its last tile
      for (int i = et; i < p.cout; i += Cfg::kEpiThreads) {
        atomicAdd(p.stats + i, static_cast<double>(ep_stats[i]));
        atomicAdd(p.stats + p.cout + i, static_cast<double>(ep_stats[BN + i]));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Host side: tensor-map encoding through the driver entry points (no link-time libcuda dependency)
// ---------------------------------------------------------------------------------------------
constexpr long long kSkFlagBytes = 4096;          // room for 1024 CTA flags
constexpr long long kSkSlotBytes = 128 * 128 * 4;  // one CTA's largest partial accumulator (MT*BN = 128 columns x 128 rows x fp32)
long long conv_workspace_bytes() { return kSkFlagBytes + kSkSlotBytes * sm_count(); }

static unsigned long long* g_conv_trace = nullptr;
void conv_set_trace(void* dev_ptr) { g_conv_trace = static_cast<unsigned long long*>(dev_ptr); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int get_encoders(EncodeTiledFn* tiled, EncodeIm2colFn* im2col) {
  static EncodeTiledFn s_tiled = nullptr;
  static EncodeIm2colFn s_im2col = nullptr;
  if (s_tiled == nullptr || s_im2col == nullptr) {
    void* f0 = nullptr;
    void* f1 = nullptr;
    cudaDriverEntryPointQueryResult q0, q1;
    YB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f0, cudaEnableDefault, &q0));
    YB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f1, cudaEnableDefault, &q1));
    if (f0 == nullptr || f1 == nullptr || q0 != cudaDriverEntryPointSuccess || q1 != cudaDriverEntryPointSuccess)
      return fail(YB_ERR_DRIVER, "cuTensorMapEncode* driver entry points unavailable");
    s_tiled = reinterpret_cast<EncodeTiledFn>(f0);
    s_im2col = reinterpret_cast<EncodeIm2colFn>(f1);
  }
  *tiled = s_tiled;
  *im2col = s_im2col;
  return 0;
}

int get_tensor_map_encoders(EncodeTiledFn* tiled, EncodeIm2colFn* im2col) { return get_encoders(tiled, im2col); }

template <int BN, int BK, int MT>
static int launch_conv(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ty, const ConvParams& p, cudaStream_t stream) {
  using Cfg = ConvCfg<BN, BK, MT>;
  static bool attr_set = false;
  if (!attr_set) {
    YB_CUDA(cudaFuncSetAttribute(conv_igemm_kernel<BN, BK, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  const int tiles = p.m_tiles * p.n_tiles;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cudaLaunchAttribute attr[1];
  int nattr = 0;
  // Programmatic dependent launch: this kernel's prologue may overlap the previous kernel's tail.  Off by default (the prologue is
  // a small share of a conv, and early-resident CTAs spinning in griddepcontrol.wait hold SMs another stream's kernels could use);
  // YB_PDL=1 switches it on for A/B runs.
  static const int use_pdl = getenv("YB_PDL") ? atoi(getenv("YB_PDL")) : 0;
  if (use_pdl) {
    attr[nattr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[nattr].val.programmaticStreamSerializationAllowed = 1;
    ++nattr;
  }
  if (p.streamk) cfg.gridDim = dim3(sm_count());          // sk_base / sk_rem were computed for exactly this many CTAs
  else cfg.gridDim = dim3(tiles < sm_count() ? tiles : sm_count());
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = nattr;
  YB_CUDA(cudaLaunchKernelEx(&cfg, conv_igemm_kernel<BN, BK, MT>, ta, tb, ty, p));
  return check_launch("conv_igemm_kernel");
}

// CTA tile shapes (BLOCK_N, M-subtiles): the MMA warpgroup keeps MT * BLOCK_N <= 128 accumulators per thread
template <int BK>
static int dispatch_conv(int bn, int mt, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ty, const ConvParams& p, cudaStream_t stream) {
  if (mt == 2) return launch_conv<64, BK, 2>(ta, tb, ty, p, stream);
  if (bn == 64) return launch_conv<64, BK, 1>(ta, tb, ty, p, stream);
  return launch_conv<128, BK, 1>(ta, tb, ty, p, stream);
}

static int conv_c32_forward(const void* x, const void* w, const float* scale, const float* shift, float slope, void* y, int batch,
                            int height, int width, int cout, int x_ld, long long y_ld, int y_ch_off, int pool, int flags, double* stats,
                            cudaStream_t stream) {
  using Cfg = C32Cfg;
  EncodeTiledFn enc_tiled;
  EncodeIm2colFn enc_im2col;
  int rc = get_encoders(&enc_tiled, &enc_im2col);
  if (rc) return rc;
  YB_REQUIRE(!pool || (height % 2 == 0 && width % 2 == 0), "conv: fused 2x2 max-pool needs even H and W");
  C32Params p;
  p.batch = batch; p.height = height; p.width = width; p.cout = cout;
  p.tiles_w = (width + Cfg::TW - 1) / Cfg::TW;
  p.tiles_h = (height + Cfg::TH - 1) / Cfg::TH;
  const long long nt = static_cast<long long>(batch) * p.tiles_w * p.tiles_h;
  YB_REQUIRE(nt < (1ll << 31), "conv: too many tiles");
  p.num_tiles = static_cast<int>(nt);
  p.scale = scale; p.shift = shift; p.slope = slope;
  p.pool = pool;
  p.swap_lbo = (flags >> 6) & 1;
  p.skip = (flags >> 24) & 0xF;
  p.dbg = debug_word_device();
  p.trace = g_conv_trace;
  p.stats = stats;
  YB_REQUIRE(stats == nullptr || (!pool && height % Cfg::TH == 0 && width % Cfg::TW == 0),
             "conv: fused statistics on the Cin = 32 kernel need H %% 16 == 0, W %% 8 == 0 and no fused pool");
  alignas(64) CUtensorMap tx, tw, ty;
  CUresult cr;
  {
    const cuuint64_t dims[4] = {32, static_cast<cuuint64_t>(width), static_cast<cuuint64_t>(height), static_cast<cuuint64_t>(batch)};
    const cuuint64_t strides[3] = {static_cast<cuuint64_t>(x_ld) * 2, static_cast<cuuint64_t>(x_ld) * 2 * width,
                                   static_cast<cuuint64_t>(x_ld) * 2 * width * height};
    const cuuint32_t box[4] = {8, Cfg::HW, Cfg::HH, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    cr = enc_tiled(&tx, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeTiled(halo) failed (%d)", static_cast<int>(cr));
  }
  {
    const cuuint64_t dims[2] = {9 * 32, static_cast<cuuint64_t>(cout)};
    const cuuint64_t strides[1] = {9 * 32 * 2};
    const cuuint32_t box[2] = {32, 64};
    const cuuint32_t estr[2] = {1, 1};
    cr = enc_tiled(&tw, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeTiled(W) failed (%d)", static_cast<int>(cr));
  }
  {
    const int oh = pool ? height / 2 : height, ow = pool ? width / 2 : width;
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(cout), static_cast<cuuint64_t>(ow), static_cast<cuuint64_t>(oh), static_cast<cuuint64_t>(batch)};
    const cuuint64_t strides[3] = {static_cast<cuuint64_t>(y_ld) * 2, static_cast<cuuint64_t>(y_ld) * 2 * ow, static_cast<cuuint64_t>(y_ld) * 2 * ow * oh};
    const cuuint32_t box[4] = {64, static_cast<cuuint32_t>(pool ? Cfg::TW / 2 : Cfg::TW), static_cast<cuuint32_t>(pool ? Cfg::TH / 2 : Cfg::TH), 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    cr = enc_tiled(&ty, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, static_cast<__half*>(y) + y_ch_off, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeTiled(Y) failed (%d)", static_cast<int>(cr));
  }
  static bool attr_set = false;
  if (!attr_set) {
    YB_CUDA(cudaFuncSetAttribute(conv_c32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  const int grid = p.num_tiles < sm_count() ? p.num_tiles : sm_count();
  conv_c32_kernel<<<grid, Cfg::kThreads, Cfg::kSmemBytes, stream>>>(tx, tw, ty, p);
  return check_launch("conv_c32_kernel");
}

int conv_igemm_forward(const void* x, const void* w, const float* scale, const float* shift, float slope, void* y, int batch,
                       int height, int width, int cin, int cout, int ksize, int x_ld, long long y_ld, int y_ch_off, int out_mode,
                       int flags, void* workspace, long long workspace_bytes, double* stats, int a_channels, int lo_ch_off, cudaStream_t stream) {
  YB_REQUIRE(x && w && scale && shift && y, "conv: null pointer");
  // split-precision operands (see ConvParams::a_wrap): cin is the concatenated reduction width, a_channels what x really holds
  if (a_channels <= 0) a_channels = cin;
  const bool split = a_channels != cin || lo_ch_off >= 0;
  YB_REQUIRE(a_channels <= cin && a_channels % 32 == 0 && cin - a_channels <= a_channels, "conv: a_channels=%d does not fit cin=%d", a_channels, cin);
  YB_REQUIRE(lo_ch_off < 0 || (out_mode == 0 && stats == nullptr && lo_ch_off % 8 == 0 && lo_ch_off >= y_ch_off + cout && lo_ch_off + cout <= y_ld),
             "conv: lo_ch_off=%d (needs fp16 NHWC output with room for a second Cout-wide slice)", lo_ch_off);
  YB_REQUIRE(stats == nullptr || out_mode == 0, "conv: fused statistics need the fp16 NHWC output");
  YB_REQUIRE(ksize == 1 || ksize == 3, "conv: ksize %d unsupported (1 or 3)", ksize);
  YB_REQUIRE(batch > 0 && height > 0 && width > 0, "conv: bad shape");
  YB_REQUIRE(cin % 32 == 0, "conv: Cin=%d must be a multiple of 32 (layer 0 uses yb_conv0_*)", cin);
  YB_REQUIRE(x_ld >= a_channels && x_ld % 8 == 0, "conv: x_ld=%d", x_ld);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0, "conv: x/w must be 16B aligned");
  YB_REQUIRE(out_mode == 0 || out_mode == 1, "conv: out_mode");
  if (out_mode == 0) {
    YB_REQUIRE(cout % 8 == 0 && y_ld % 8 == 0 && y_ch_off % 8 == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0,
               "conv: fp16 NHWC output needs Cout, y_ld, y_ch_off multiples of 8 and a 16B aligned pointer");
  }
  const long long m_total_ll = static_cast<long long>(batch) * height * width;
  YB_REQUIRE(m_total_ll < (1ll << 31) - BM, "conv: too many pixels");
  const int pool = (flags >> 4) & 1;        // YB_CONV_POOL2X2
  // 3x3, Cin = 32, Cout <= 64 (layers1.2): halo-tile kernel unless a test asks for one of the im2col kernels
  if (!split && cin == 32 && ksize == 3 && cout <= 64 && out_mode == 0 && ((flags >> 28) & 1) == 0 && ((flags >> 5) & 1) == 0 && ((flags >> 8) & 0xFFFF) == 0)
    return conv_c32_forward(x, w, scale, shift, slope, y, batch, height, width, cout, x_ld, y_ld, y_ch_off, pool, flags, stats, stream);
  if (pool) return fail(YB_ERR_UNSUPPORTED, "conv: YB_CONV_POOL2X2 is only implemented for the Cin = 32 3x3 layer");
  const int bk = (cin % 64 == 0 && a_channels % 64 == 0) ? 64 : 32;     // K-blocks never straddle the wrap point
  // tile shape: flags may force BLOCK_N (bits 8..17) and the number of M-subtiles (bits 20..21); otherwise pick the
  // (BLOCK_N, M-subtiles) pair with the lowest modelled time.  The model treats the kernel as bound by the L2->SM operand
  // feed (a tile costs its operand bytes at a per-SM rate, or its MMA time if larger, and tiles run in ceil(tiles/SMs)
  // rounds, capped by a chip-wide L2 rate); its rates are estimates for H100, not fitted measurements.
  int bn = 0, mt = 0, streamk = 0;
  // stream-K needs the caller's workspace (one per stream: partial sums + flags); flags bit 3 forbids, bit 30 forces it
  const bool sk_possible = stats == nullptr && workspace != nullptr && workspace_bytes >= conv_workspace_bytes() && (flags & 8) == 0 &&
                           (reinterpret_cast<uintptr_t>(workspace) & 255) == 0;
  const bool sk_force = sk_possible && ((flags >> 30) & 1);
  const int force_bn = (flags >> 8) & 0x3FF;
  const int force_mt = (flags >> 20) & 0x3;
  const int force_pair = (flags >> 22) & 0x3;      // 0 = auto, 1 = single-CTA tiles (the only form), 2 = CTA pair (not on sm_90)
  YB_REQUIRE(force_pair != 2, "conv: CTA-pair tiles need two-CTA tensor-core instructions, which sm_90 does not have");
  YB_REQUIRE(!force_bn || ((force_bn == 64 || force_bn == 128) && (force_mt != 2 || force_bn == 64)),
             "conv: BLOCK_N=%d x %d M-subtiles is not a tile shape of this kernel (64 x 1, 128 x 1, 64 x 2)", force_bn, force_mt ? force_mt : 1);
  {
    double best = 1e300;
    const int sms = sm_count();
    const int num_kb = ksize * ksize * (cin / bk);
    for (int cbn = 64; cbn <= 128; cbn *= 2) {
      if (force_bn && cbn != force_bn) continue;
      if (!force_bn && cbn > 64 && cbn / 2 >= cout) continue;       // do not pad Cout by more than 2x
      for (int cmt = 1; cmt <= 2; ++cmt) {
        if (force_mt && cmt != force_mt) continue;
        if (cmt * cbn > 128) continue;
        const int rows_tile = BM * cmt;
        const double tiles = static_cast<double>((m_total_ll + rows_tile - 1) / rows_tile) * ((cout + cbn - 1) / cbn);
        const double rounds = static_cast<double>((static_cast<long long>(tiles) + sms - 1) / sms);
        const double bytes_kb = (cmt * BM + cbn) * bk * 2.0;        // per CTA
        const double mma_ns_kb = cmt * BM * cbn * bk * 2.0 / 7000.0;  // ~7 TFLOP/s per SM of dense fp16
        const double kb_ns = bytes_kb / 60.0 > mma_ns_kb ? bytes_kb / 60.0 : mma_ns_kb;
        const double tile_ns = num_kb * kb_ns + 500.0;
        const double agg_ns = tiles * num_kb * bytes_kb / 7000.0;
        double t = rounds * tile_ns;
        if (agg_ns > t) t = agg_ns;
        int csk = 0;
        if (sk_possible) {
          // stream-K: every SM gets units/SMs K-blocks; on top, roughly one partial dump + one collecting epilogue per CTA
          const double units = tiles * num_kb;
          const double per_cta = static_cast<double>((static_cast<long long>(units) + sms - 1) / sms);
          const double epi_ns = 8000.0 * (cmt * cbn / 512.0);
          double tsk = per_cta * kb_ns + epi_ns + 1500.0;
          if (agg_ns > tsk) tsk = agg_ns;
          // stream-K pays when the layer leaves most of the GPU idle (single images, small batches); layers that already fill
          // the chip gain nothing from the spread
          const bool ok = per_cta >= 4.0 && num_kb >= 2;
          const bool idle = tiles <= sms / 2;
          if (ok && (sk_force || (idle && tsk < 0.93 * t))) { t = tsk; csk = 1; }
        }
        if (sk_force && !csk) continue;
        // ties go to the wider-N shape (more reuse of each A tile)
        if (t < best * 0.9999 || (t <= best * 1.0001 && cbn > bn)) { best = t; bn = cbn; mt = cmt; streamk = csk; }
      }
    }
    if (bn == 0) { bn = force_bn ? force_bn : 128; mt = force_mt ? force_mt : 1; streamk = 0; }
  }
  YB_REQUIRE((bn == 64 || bn == 128) && (mt == 1 || mt == 2) && mt * bn <= 128, "conv: tile %d x %d", bn, mt);
  // 1x1 layers read A as a plain [pixels, Cin] matrix (2-D tiled TMA: cheaper per instruction than im2col mode);
  // YB_CONV_1X1_IM2COL=1 switches back for A/B runs
  static const int k1x1_im2col = getenv("YB_CONV_1X1_IM2COL") ? atoi(getenv("YB_CONV_1X1_IM2COL")) : 0;
  const int a_im2col = (ksize == 3) ? 1 : ((k1x1_im2col && !(flags & 1)) ? 1 : 0);

  EncodeTiledFn enc_tiled;
  EncodeIm2colFn enc_im2col;
  int rc = get_encoders(&enc_tiled, &enc_im2col);
  if (rc) return rc;

  ConvParams p;
  p.m_total = static_cast<int>(m_total_ll);
  p.height = height; p.width = width; p.cin = cin; p.cout = cout; p.ksize = ksize; p.pad = (ksize - 1) / 2;
  p.kb_per_tap = cin / bk;
  p.num_kb = ksize * ksize * p.kb_per_tap;
  const int rows_tile = BM * mt;
  p.m_tiles = (p.m_total + rows_tile - 1) / rows_tile;
  p.n_tiles = (cout + bn - 1) / bn;
  p.a_im2col = a_im2col;
  p.scale = scale; p.shift = shift; p.slope = slope;
  p.y = y; p.y_ld = y_ld; p.y_ch_off = y_ch_off; p.out_mode = out_mode;
  p.hw = height * width;
  p.dbg = debug_word_device();
  p.trace = g_conv_trace;
  p.skip = (flags >> 24) & 0xF;
  p.streamk = streamk;
  p.stats = stats;
  p.tma_store = 0;
  p.a_wrap = a_channels;
  p.lo_off = lo_ch_off >= 0 ? static_cast<long long>(lo_ch_off - y_ch_off) : 0;
  p.sk_base = 0; p.sk_rem = 0; p.ws = nullptr; p.flags = nullptr;
  if (streamk) {
    const long long units = static_cast<long long>(p.m_tiles) * p.n_tiles * p.num_kb;
    YB_REQUIRE(units < (1ll << 31), "conv: stream-K unit count overflows");
    p.sk_base = static_cast<int>(units / sm_count());
    p.sk_rem = static_cast<int>(units % sm_count());
    p.flags = static_cast<unsigned*>(workspace);
    p.ws = reinterpret_cast<float*>(static_cast<char*>(workspace) + kSkFlagBytes);
  }

  const CUtensorMapSwizzle swz = (bk == 64) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  alignas(64) CUtensorMap ta, tb;
  CUresult cr;
  const int a_rows = BM * mt;     // pixels per A box (ConvCfg::kMergedA)
  if (a_im2col) {
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(a_channels), static_cast<cuuint64_t>(width), static_cast<cuuint64_t>(height),
                                static_cast<cuuint64_t>(batch)};
    const cuuint64_t strides[3] = {static_cast<cuuint64_t>(x_ld) * 2, static_cast<cuuint64_t>(x_ld) * 2 * width,
                                   static_cast<cuuint64_t>(x_ld) * 2 * width * height};
    const int lower[2] = {-p.pad, -p.pad};                    // {W, H}
    const int upper[2] = {p.pad - (ksize - 1), p.pad - (ksize - 1)};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    cr = enc_im2col(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(x), dims, strides, lower, upper,
                    static_cast<cuuint32_t>(bk), static_cast<cuuint32_t>(a_rows), estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeIm2col failed (%d)", static_cast<int>(cr));
    // Driver workaround (same one CUTLASS carries, cute/atom/copy_traits_sm90_im2col.hpp): for
    // tensors smaller than 128 KiB drivers <= 13.1 set a descriptor bit that breaks im2col loads.
    int drv = 0;
    cudaDriverGetVersion(&drv);
    const unsigned long long span_bytes = static_cast<unsigned long long>(x_ld) * 2ull * width * height * batch;
    if (drv <= 13010 && span_bytes < 131072ull) reinterpret_cast<uint64_t*>(&ta)[1] &= ~(1ull << 21);
  } else {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(a_channels), static_cast<cuuint64_t>(p.m_total)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(x_ld) * 2};
    const cuuint32_t box[2] = {static_cast<cuuint32_t>(bk), static_cast<cuuint32_t>(a_rows)};
    const cuuint32_t estr[2] = {1, 1};
    cr = enc_tiled(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(x), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeTiled(A) failed (%d)", static_cast<int>(cr));
  }
  {
    const cuuint64_t k_total = static_cast<cuuint64_t>(ksize) * ksize * cin;
    const cuuint64_t dims[2] = {k_total, static_cast<cuuint64_t>(cout)};
    const cuuint64_t strides[1] = {k_total * 2};
    const cuuint32_t box[2] = {static_cast<cuuint32_t>(bk), static_cast<cuuint32_t>(bn)};
    const cuuint32_t estr[2] = {1, 1};
    cr = enc_tiled(&tb, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(w), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeTiled(W) failed (%d)", static_cast<int>(cr));
  }

  // output tensor map of the TMA-store epilogue (fp16 NHWC, no residual output); flags bit 29 (YB_CONV_PLAIN_STORE) keeps the
  // per-thread stores for A/B runs
  alignas(64) CUtensorMap ty;
  memset(&ty, 0, sizeof(ty));
  p.tma_store = (out_mode == 0 && lo_ch_off < 0 && ((flags >> 29) & 1) == 0) ? 1 : 0;
  if (p.tma_store) {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cout), static_cast<cuuint64_t>(p.m_total)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(y_ld) * 2};
    const cuuint32_t box[2] = {64, 32};                 // one epilogue warp's rows
    const cuuint32_t estr[2] = {1, 1};
    cr = enc_tiled(&ty, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, static_cast<__half*>(y) + y_ch_off, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeTiled(Y) failed (%d)", static_cast<int>(cr));
  }
  if (bk == 64) return dispatch_conv<64>(bn, mt, ta, tb, ty, p, stream);
  return dispatch_conv<32>(bn, mt, ta, tb, ty, p, stream);
}

// ---------------------------------------------------------------------------------------------
// CUDA-core reference of the same unit: test / bisect utility only (never on the product path).
// One thread per (pixel, cout); fp16 inputs, fp32 accumulate, identical epilogue and outputs.
// ---------------------------------------------------------------------------------------------
__global__ void conv_ref_kernel(const __half* __restrict__ x, const __half* __restrict__ w, ConvParams p, int x_ld) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(p.m_total) * p.cout;
  if (idx >= total) return;
  const int co = static_cast<int>(idx % p.cout);
  const int row = static_cast<int>(idx / p.cout);
  const int img = row / p.hw;
  const int pix = row - img * p.hw;
  const int h = pix / p.width;
  const int wq = pix - h * p.width;
  float acc = 0.f;
  for (int r = 0; r < p.ksize; ++r) {
    const int hi = h + r - p.pad;
    if (hi < 0 || hi >= p.height) continue;
    for (int s = 0; s < p.ksize; ++s) {
      const int wi = wq + s - p.pad;
      if (wi < 0 || wi >= p.width) continue;
      const __half* xp = x + (static_cast<long long>(img) * p.hw + static_cast<long long>(hi) * p.width + wi) * x_ld;
      const __half* wp = w + (static_cast<long long>(co) * p.ksize * p.ksize + r * p.ksize + s) * p.cin;
      for (int c = 0; c < p.cin; ++c) acc += __half2float(xp[c]) * __half2float(wp[c]);
    }
  }
  float v = acc * p.scale[co] + p.shift[co];
  v = v > 0.f ? v : v * p.slope;
  if (p.out_mode == 0) {
    reinterpret_cast<__half*>(p.y)[static_cast<long long>(row) * p.y_ld + p.y_ch_off + co] = __float2half_rn(v);
  } else {
    reinterpret_cast<float*>(p.y)[(static_cast<long long>(img) * p.cout + co) * p.hw + pix] = v;
  }
}

int conv_ref_forward(const void* x, const void* w, const float* scale, const float* shift, float slope, void* y, int batch,
                     int height, int width, int cin, int cout, int ksize, int x_ld, long long y_ld, int y_ch_off, int out_mode,
                     cudaStream_t stream) {
  YB_REQUIRE(x && w && scale && shift && y, "conv_ref: null pointer");
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.m_total = batch * height * width;
  p.height = height; p.width = width; p.cin = cin; p.cout = cout; p.ksize = ksize; p.pad = (ksize - 1) / 2;
  p.scale = scale; p.shift = shift; p.slope = slope; p.y = y; p.y_ld = y_ld; p.y_ch_off = y_ch_off; p.out_mode = out_mode;
  p.hw = height * width;
  const long long total = static_cast<long long>(p.m_total) * cout;
  conv_ref_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x),
                                                                                  reinterpret_cast<const __half*>(w), p, x_ld);
  return check_launch("conv_ref_kernel");
}

}  // namespace yb
