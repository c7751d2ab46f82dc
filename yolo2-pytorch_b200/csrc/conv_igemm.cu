// K1: convolution as an implicit GEMM on the Hopper tensor cores (wgmma), sm_90a.
//
// Replaces the reference's  nn.Conv2d -> nn.BatchNorm2d(eval) -> nn.LeakyReLU(0.1)  unit
// (reference model/yolo2.py:49-65) for k in {1,3}, stride 1, pad (k-1)/2, and the general geometry of Inception-v3
// (kh x kw filters up to 7 x 7, stride 1 or 2, any padding below the filter size; yb_conv2d_bn_act_fwd).
//
//   D[M = B*OH*OW output pixels, N = Cout] = A[M, K = kh*kw*Cin] * W[N, K]^T
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
  int m_total;      // B*OH*OW
  int height, width;  // OUTPUT rows / columns: they drive the M enumeration and the fp32 NCHW epilogue
  int cin, cout;
  int kh, kw, pad_h, pad_w, stride;
  int in_h, in_w;   // input rows / columns
  int kb_per_tap;   // Cin / BK
  int num_kb;       // kh*kw*kb_per_tap
  int m_tiles, n_tiles;
  int a_im2col;     // 1: im2col TMA, 0: plain 2D tiled TMA over [M, Cin] (1x1, stride 1 only)
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
  // chained form (conv_wide_chain_kernel): the 1x1 unit that consumes this conv's output inside the tile -- its scale / shift /
  // slope and Cout; y / tmap_y are that unit's output
  const float* scale2;
  const float* shift2;
  float slope2;
  int cout2;
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
// kPreCh > 0 (the pre-activation form, conv_preact_kernel): room for a per-input-channel scale / shift table of up to kPreCh channels.
template <int BN, int BK, int MT, int kPreCh = 0>
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
  static constexpr int kFixedBytes = kAccBytes + kOutBytes + 1024 /*align slack*/ + 2 * 2 * BN * 4 /*scale/shift x2*/ + 2 * BN * 4 /*stats*/ + 256 /*barriers*/ +
                                     2 * kPreCh * 4 /*pre-activation scale / shift*/;
  static constexpr int kStages = ((kSmemLimit - kFixedBytes) / kStageBytes) > 8 ? 8 : ((kSmemLimit - kFixedBytes) / kStageBytes);
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(kAccCols <= 128, "accumulator does not fit the MMA warpgroup's registers");
  static_assert(kStages >= 2, "shared memory budget");
};

// Pre-activation of the A operand (DenseNet's norm -> relu -> 1x1 conv, conv_preact_kernel):
//   a[p][c] = fp16_rn(act(fmaf(scale[c], x[p][c], shift[c]))), act = ReLU (relu = 1) or identity (0).
struct PreAct {
  const float* scale;
  const float* shift;
  int relu;
};
constexpr int kPreMaxCh = 1920;                 // DenseNet-201's widest block input; the table is staged whole, once per CTA

// Applies the pre-activation in place to one swizzled A stage (MT * 128 pixel rows x BK channels starting at channel c0).  The TMA
// swizzle permutes 16-byte chunks inside a row: logical chunk c of row r sits at chunk c ^ (r % 8) (BK = 64, 128-byte rows) or
// c ^ ((r / 2) % 4) (BK = 32, 64-byte rows).  A thread keeps one chunk column, so its scale / shift values stay in registers, and a
// warp covers 512 contiguous bytes per pass.  A thread handles its chunk in two 8-byte halves; threads whose rows fall on alternate
// 128-byte lines take the halves in opposite order, so each instruction of a warp touches all 32 banks twice (2 wavefronts per 256 B).
template <int BK, int MT>
__device__ __forceinline__ void preact_stage(uint32_t a, const float* tab_scale, const float* tab_shift, int c0, int relu) {
  constexpr int kChunks = BK / 8;
  constexpr int kRowsPerPass = kMmaThreads / kChunks;
  const int c = threadIdx.x % kChunks;
  const int r0 = threadIdx.x / kChunks;
  // two passes of 4 channels (8 bytes) per chunk: 8 table values live next to the 128 accumulators of the widest tile without spilling
#pragma unroll 1
  for (int pass = 0; pass < 2; ++pass) {
    const int half = pass ^ ((r0 / (64 / BK)) & 1);
    const int ch = c0 + c * 8 + half * 4;
    const float4 sc = *reinterpret_cast<const float4*>(tab_scale + ch);
    const float4 sh = *reinterpret_cast<const float4*>(tab_shift + ch);
#pragma unroll 1
    for (int i = 0; i < MT * BM / kRowsPerPass; ++i) {
      const int r = r0 + i * kRowsPerPass;
      const int pc = (BK == 64) ? (c ^ (r & 7)) : (c ^ ((r >> 1) & 3));
      const uint32_t addr = a + r * (BK * 2) + pc * 16 + half * 8;
      uint32_t v0, v1;
      asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(v0), "=r"(v1) : "r"(addr) : "memory");
      const float2 f0 = __half22float2(*reinterpret_cast<__half2*>(&v0));
      const float2 f1 = __half22float2(*reinterpret_cast<__half2*>(&v1));
      float y0 = __fmaf_rn(sc.x, f0.x, sh.x), y1 = __fmaf_rn(sc.y, f0.y, sh.y);
      float y2 = __fmaf_rn(sc.z, f1.x, sh.z), y3 = __fmaf_rn(sc.w, f1.y, sh.w);
      if (relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); y2 = fmaxf(y2, 0.f); y3 = fmaxf(y3, 0.f); }
      __half2 h0 = __floats2half2_rn(y0, y1), h1 = __floats2half2_rn(y2, y3);
      asm volatile("st.shared.v2.b32 [%0], {%1, %2};" :: "r"(addr), "r"(*reinterpret_cast<uint32_t*>(&h0)), "r"(*reinterpret_cast<uint32_t*>(&h1))
                   : "memory");
    }
  }
}

// The body of both implicit-GEMM kernels of this family.  kPre = false is conv_igemm_kernel; kPre = true (1x1 only) is
// conv_preact_kernel, whose MMA warpgroup applies `pre` to every A stage in shared memory before issuing the unchanged
// shared-memory wgmma.
template <int BN, int BK, int MT, bool kPre>
__device__ __forceinline__ void conv_igemm_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, const CUtensorMap& tmap_y,
                                                const ConvParams p, const PreAct pre) {
  using Cfg = ConvCfg<BN, BK, MT, kPre ? kPreMaxCh : 0>;
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
        int img[MT], h0[MT], w0[MT];       // input coordinates of the first output pixel's window corner, per subtile
        int nsub = 0;                      // subtiles that start inside the tensor (the rest are skipped)
#pragma unroll
        for (int t = 0; t < MT; ++t) {
          const int ms = m_cta + t * BM;
          if (ms < p.m_total) nsub = t + 1;
          img[t] = ms / p.hw;
          const int rem = ms - img[t] * p.hw;
          const int oh = rem / p.width;
          h0[t] = oh * p.stride - p.pad_h;
          w0[t] = (rem - oh * p.width) * p.stride - p.pad_w;
        }
        if (p.skip & 1) nsub = 0;
        if (kMergedA && nsub) nsub = MT;      // the merged box always transfers (and zero-fills) both subtiles
        const uint32_t tx_bytes = nsub * Cfg::kASubBytes + ((p.skip & 2) ? 0 : Cfg::kBBytes);
        for (int kb = it.kb0; kb < it.kb1; ++kb) {
          const int tap = kb / p.kb_per_tap;
          const int c0 = (kb - tap * p.kb_per_tap) * BK;    // offset inside the (possibly concatenated) weight row of this tap
          const int ca = c0 >= p.a_wrap ? c0 - p.a_wrap : c0;   // activation channel (split mode: the hi part is read twice)
          const int r = tap / p.kw;
          const int s = tap - r * p.kw;
          mbar_wait(bar_empty + 8 * stage, phase ^ 1, p.dbg, 0x100 | stage);
          YB_TRACE(0, tr_p); ++tr_p;
          const uint32_t full = bar_full + 8 * stage;
          mbar_arrive_expect_tx(full, tx_bytes);
          if (kMergedA) {
            // one TMA box covers both 128-pixel subtiles (the tensor map's box is BM * MT pixels): the im2col-mode TMA has
            // a large per-instruction cost, rows past the tensor end are zero-filled
            if (!(p.skip & 1)) {
              const uint32_t dst = smem_a + stage * Cfg::kABytes;
              if (p.a_im2col) tma_load_im2col_4d(dst, &tmap_a, full, ca, w0[0], h0[0], img[0], static_cast<uint16_t>(s), static_cast<uint16_t>(r));
              else tma_load_2d(dst, &tmap_a, full, ca, m_cta);
            }
          } else {
#pragma unroll
          for (int t = 0; t < MT; ++t) {
            if (t < nsub) {
              const uint32_t dst = smem_a + stage * Cfg::kABytes + t * Cfg::kASubBytes;
              if (p.a_im2col) tma_load_im2col_4d(dst, &tmap_a, full, ca, w0[t], h0[t], img[t], static_cast<uint16_t>(s), static_cast<uint16_t>(r));
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
    float* pre_scale = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);     // [kPreMaxCh] (kPre only)
    float* pre_shift = pre_scale + kPreMaxCh;
    if constexpr (kPre) {
      for (int i = threadIdx.x; i < p.cin; i += kMmaThreads) { pre_scale[i] = __ldg(pre.scale + i); pre_shift[i] = __ldg(pre.shift + i); }
      asm volatile("bar.sync 2, %0;" :: "n"(kMmaThreads) : "memory");
    }
    for (WorkIter it(p, unit_id, num_units, num_tiles); it.valid(); it.next()) {
      const int kb_first = it.kb0, kb_last = it.kb1 - 1;
      int prev = -1;
      for (int kb = kb_first; kb <= kb_last; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase, p.dbg, 0x300 | stage);
        if (threadIdx.x == 0) { YB_TRACE(1, tr_m); ++tr_m; }
        if constexpr (kPre) {
          // 1x1: K-block kb is channels [kb * BK, kb * BK + BK).  The generic-proxy writes are made visible to the wgmma (async
          // proxy) by the fence, and the whole tile is transformed before any warp issues its MMAs.
          preact_stage<BK, MT>(smem_a + stage * Cfg::kABytes, pre_scale, pre_shift, kb * BK, pre.relu);
          fence_proxy_async_smem();
          asm volatile("bar.sync 2, %0;" :: "n"(kMmaThreads) : "memory");
        }
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

template <int BN, int BK, int MT>
__global__ void __launch_bounds__(kThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_y, const ConvParams p) {
  conv_igemm_body<BN, BK, MT, false>(tmap_a, tmap_b, tmap_y, p, PreAct{nullptr, nullptr, 0});
}

template <int BN, int BK, int MT>
__global__ void __launch_bounds__(kThreads, 1)
conv_preact_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const __grid_constant__ CUtensorMap tmap_y, const ConvParams p, const PreAct pre) {
  conv_igemm_body<BN, BK, MT, true>(tmap_a, tmap_b, tmap_y, p, pre);
}

// ---------------------------------------------------------------------------------------------
// Wide family: a 256 x 128 CTA tile on two consumer warpgroups.  Warpgroup 0 is the producer (one thread issues the TMA loads,
// one thread per consumer issues that consumer's TMA stores; the group gives its registers back), warpgroups 1 and 2 each
// accumulate 128 pixels x 128 channels in registers (128 fp32 per thread) from the same stage: A is one 256-pixel box, B is read
// by both.  Per FLOP that moves 2/3 of the operand bytes of the 128 x 128 tile.  The epilogue runs from the registers (scale /
// shift, leaky, fp16, a 128B-swizzled staging slice, TMA store), so there is no accumulator park; stream-K partials go to and
// come from `ws` out of the registers.  Each accumulator sees the same K-blocks and k16 steps in the same order as in the
// 128 x 128 kernel, so a launch without stream-K is bit-identical to it.  fp16 NHWC output only: the head, the residual (lo)
// output and the training statistics stay on conv_igemm_kernel.
//
// Epilogue overlap.  The tensor cores idle from a tile's last MMA to the next tile's first one, so the consumers keep that
// stretch down to the conversion arithmetic:
//   * the last K-block is committed as two groups, and rows 0..63 of a consumer's tile are converted while the MMAs into rows
//     64..127 still run;
//   * the tile's scale / shift sit in a shared-memory table (one float per consumer thread, loaded when the tile starts and
//     stored there at its end), so the conversion reads one 16-byte word per column pair instead of waiting on global loads;
//   * each 64-row half goes through the consumer's 16 KB staging slice, and a thread of the producer warpgroup issues its TMA
//     stores and waits for them to read the slice (mbarriers slice_full / slice_empty): the consumer converts the second half
//     into registers while the first half's stores drain, and starts the next tile as soon as the second half is staged.
// ---------------------------------------------------------------------------------------------
constexpr int kWideThreads = 384;
constexpr int kWideRows = 256;
constexpr int kWideBN = 128;
constexpr int kWidePoolRows = kWideRows / 4;   // pooled form: output rows (pool windows) per tile

__device__ __forceinline__ uint32_t hmax2_u32(uint32_t a, uint32_t b) {
  const __half2 m = __hmax2(*reinterpret_cast<const __half2*>(&a), *reinterpret_cast<const __half2*>(&b));
  return *reinterpret_cast<const uint32_t*>(&m);
}

template <int BK>
struct WideCfg {
  static constexpr int kSwizzle = BK * 2;
  static constexpr int kABytes = kWideRows * BK * 2;
  static constexpr int kBBytes = kWideBN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kOutBytes = 128 * 128;                   // per consumer: 64 rows x 128 channels fp16 as two [64][128 B] blocks, 128B-swizzled
  static constexpr int kTableBytes = kWideBN * 2 * 4;           // the tile's scale / shift: float4 {sc[2i], sc[2i + 1], sh[2i], sh[2i + 1]} per column pair
  static constexpr int kFixedBytes = 2 * kOutBytes + kTableBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int kStages = ((kSmemLimit - kFixedBytes) / kStageBytes) > 8 ? 8 : ((kSmemLimit - kFixedBytes) / kStageBytes);
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static constexpr int kWsFloats = kWideRows * kWideBN;         // one CTA's stream-K partial tile
  static_assert(kStages >= (BK == 64 ? 4 : 8), "shared memory budget: the epilogue's slices and table must not cost a pipeline stage");
  // chained form: the second unit's scale / shift table (float4 per column pair of its 64 channels) after the barriers
  static constexpr int kChainTableBytes = 64 * 2 * 4;
  static constexpr int kChainSmemBytes = kSmemBytes + kChainTableBytes;
  static_assert(kChainSmemBytes <= kSmemLimit, "shared memory budget: the chained form must not cost a pipeline stage");
};
constexpr int kChainN = 64;       // chained form: output channels of the second (1x1) unit per tile

// kPool: the pooled form (conv_wide_pool_kernel), kChain: the chained form (conv_wide_chain_kernel), see below.  tmap_a[0] is the A map
// of the plain form; the pooled form reads one map per pool-window position.  tmap_w2: the chained form's second weight.
template <int BK, bool kPool, bool kChain>
__device__ __forceinline__ void conv_wide_body(const CUtensorMap* const (&tmap_a)[4], const CUtensorMap& tmap_b, const CUtensorMap& tmap_y,
                                               const CUtensorMap* tmap_w2, const ConvParams p) {
  static_assert(!(kPool && kChain), "one fused epilogue at a time");
  using Cfg = WideCfg<BK>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_a = smem_base;
  const uint32_t smem_b = smem_base + kStages * Cfg::kABytes;
  const uint32_t smem_o = smem_base + kStages * Cfg::kStageBytes;         // [2 consumers][kOutBytes]
  const uint32_t table = smem_o + 2 * Cfg::kOutBytes;                     // [kWideBN / 2] float4
  const uint32_t bar_full = table + Cfg::kTableBytes;                     // [kStages]
  const uint32_t bar_empty = bar_full + 8 * kStages;                      // [kStages]
  const uint32_t bar_slice_full = bar_empty + 8 * kStages;                // [2 consumers]: a 64-row half is staged
  const uint32_t bar_slice_empty = bar_slice_full + 16;                   // [2 consumers]: its stores have read the slice
  // chained form: the second unit's [64][128] fp16 weight is resident as two K-blocks of [64 rows][128 B] (128B-swizzled), in the
  // upper 8 KB of consumer kb2's staging slice -- its 64-channel output only uses the lower half.  One load per CTA on bar_w.
  const uint32_t bar_w = bar_slice_empty + 16;
  const uint32_t table2 = table + Cfg::kTableBytes + 256;                 // [kChainN / 2] float4
  const int num_tiles = p.m_tiles * p.n_tiles;
  const int unit_id = static_cast<int>(blockIdx.x);
  const int num_units = static_cast<int>(gridDim.x);

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, 8);                     // one arrival per consumer warp
    }
    for (int c = 0; c < 2; ++c) {
      mbar_init(bar_slice_full + 8 * c, 4);                // one arrival per warp of consumer c
      if constexpr (kPool) mbar_init(bar_slice_empty + 8 * c, c == 1 ? 4 : 1);   // pooled: consumer 1's slice is read by consumer 0's warps
      else mbar_init(bar_slice_empty + 8 * c, 1);          // its store thread
    }
    if constexpr (kChain) mbar_init(bar_w, 1);
    fence_mbar_init();
    fence_proxy_async_smem();
    tma_prefetch_desc(tmap_a[0]);
    if constexpr (kPool) {
      for (int b = 1; b < 4; ++b) tma_prefetch_desc(tmap_a[b]);
    }
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_y);
    if constexpr (kChain) tma_prefetch_desc(tmap_w2);
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();

  if (threadIdx.x < 128) {
    // ===================== producer warpgroup =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      int tr_p = 0;
      if constexpr (kChain) {
        mbar_arrive_expect_tx(bar_w, 2 * kChainN * 128);    // rows >= Cout2 are zero-filled and still counted
        for (int kb2 = 0; kb2 < 2; ++kb2) tma_load_2d(smem_o + kb2 * Cfg::kOutBytes + 8192, tmap_w2, bar_w, kb2 * 64, 0);
      }
      for (WorkIter it(p, unit_id, num_units, num_tiles); it.valid(); it.next()) {
        const int n_tile = it.tile % p.n_tiles;
        const int m_cta = (it.tile / p.n_tiles) * (kPool ? kWidePoolRows : kWideRows);
        const int img = m_cta / p.hw;
        const int rem = m_cta - img * p.hw;
        const int oh = rem / p.width;
        const int h0 = oh * p.stride - p.pad_h;                // input coordinates of the first output pixel's window corner
        const int w0 = (rem - oh * p.width) * p.stride - p.pad_w;
        for (int kb = it.kb0; kb < it.kb1; ++kb) {
          const int tap = kb / p.kb_per_tap;
          const int c0 = (kb - tap * p.kb_per_tap) * BK;
          const int ca = c0 >= p.a_wrap ? c0 - p.a_wrap : c0;
          const int r = tap / p.kw;
          const int s = tap - r * p.kw;
          mbar_wait(bar_empty + 8 * stage, phase ^ 1, p.dbg, 0x600 | stage);
          YB_TRACE(0, tr_p); ++tr_p;
          const uint32_t full = bar_full + 8 * stage;
          mbar_arrive_expect_tx(full, Cfg::kStageBytes);      // the A box always transfers (and zero-fills) all 256 rows
          const uint32_t dst = smem_a + stage * Cfg::kABytes;
          if constexpr (kPool) {
            // box b = 2 dy + dx: window position (dy, dx) of the tile's 64 pool windows, stage rows 64 b .. 64 b + 63
#pragma unroll
            for (int b = 0; b < 4; ++b)
              tma_load_im2col_4d(dst + b * kWidePoolRows * BK * 2, tmap_a[b], full, ca, w0 + (b & 1), h0 + (b >> 1), img, static_cast<uint16_t>(s),
                                 static_cast<uint16_t>(r));
          } else {
            if (p.a_im2col) tma_load_im2col_4d(dst, tmap_a[0], full, ca, w0, h0, img, static_cast<uint16_t>(s), static_cast<uint16_t>(r));
            else tma_load_2d(dst, tmap_a[0], full, ca, m_cta);
          }
          tma_load_2d(smem_b + stage * Cfg::kBBytes, &tmap_b, full, tap * p.cin + c0, n_tile * kWideBN);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    } else if (threadIdx.x == 32 || (!kPool && threadIdx.x == 64)) {
      // store thread of consumer c: ships each staged 64-row half (rows >= M and channels >= Cout are clipped by the tensor map); the
      // pooled form stores once per tile, the 64 pooled rows consumer 0 staged
      const int c = (threadIdx.x >> 5) - 1;
      const uint32_t slice = smem_o + c * Cfg::kOutBytes;
      uint32_t sph = 0;
      for (WorkIter it(p, unit_id, num_units, num_tiles); it.valid(); it.next()) {
        if (it.kb1 < p.num_kb) continue;                      // stream-K dump: nothing to store
        const int n0 = (it.tile % p.n_tiles) * kWideBN;
        const int m_base = kPool ? (it.tile / p.n_tiles) * kWidePoolRows : (it.tile / p.n_tiles) * kWideRows + c * 128;
        for (int h = 0; h < (kPool ? 1 : 2); ++h) {
          mbar_wait(bar_slice_full + 8 * c, sph, p.dbg, 0x900 | c);
#pragma unroll
          for (int c2 = 0; c2 < (kChain ? 1 : 2); ++c2) {       // chained: the 64 channels of the second unit
            if (kChain || n0 + c2 * 64 < p.cout) {
#pragma unroll
              for (int g = 0; g < 2; ++g) {
                const int row = m_base + h * 64 + g * 32;
                if (row < p.m_total) tma_store_2d(&tmap_y, slice + c2 * 8192 + g * 4096, n0 + c2 * 64, row);
              }
            }
          }
          tma_store_commit();
          tma_store_wait_read<0>();
          mbar_arrive(bar_slice_empty + 8 * c);
          sph ^= 1;
        }
      }
      tma_store_wait<0>();     // every bulk store has landed before the CTA's shared memory goes away
    }
    return;
  }
  // ===================== consumer warpgroups =====================
  setmaxnreg_inc<232>();
  const int cw = (threadIdx.x >> 7) - 1;       // consumer 0: tile rows 0..127, consumer 1: rows 128..255
  const int t = threadIdx.x & 127;
  const int warp = t >> 5;
  const int lane = t & 31;
  const bool leader = threadIdx.x == 128;
  const uint32_t slice = smem_o + cw * Cfg::kOutBytes;
  const int te = cw * 128 + t;                 // this thread's entry of the scale / shift table
  const float4* tab4 = reinterpret_cast<const float4*>(smem_raw + (table - smem_u32(smem_raw)));
  float acc[2][64];
  int stage = 0;
  uint32_t phase = 0;
  uint32_t sph = 0;                            // staging slice phase
  if constexpr (kChain) {
    // the second unit's table, once per CTA (read after the first tile's table barriers): entry te < 128 is column pair te / 4,
    // {scale, scale, shift, shift}[te % 4]
    if (te < 2 * kChainN) {
      const int col = 2 * (te >> 2) + (te & 1);
      const float v = col < p.cout2 ? __ldg(((te & 2) ? p.shift2 : p.scale2) + col) : 0.f;
      asm volatile("st.shared.f32 [%0], %1;" :: "r"(table2 + 4 * te), "f"(v) : "memory");
    }
  }
  // trace (yb_conv_set_trace; block 0, consumer 0's first thread), tile i of the CTA: role 1 slot 2i = its last full-barrier wait,
  // 2i + 1 = its first wgmma issue; role 2 slot 2i = its K-loop end (every MMA retired), 2i + 1 = its epilogue end.  tr_t = 2i
  int tr_t = 0;
  for (WorkIter it(p, unit_id, num_units, num_tiles); it.valid(); it.next(), tr_t += 2) {
    const int kb_first = it.kb0, kb_last = it.kb1 - 1;
    const int tile = it.tile;
    const int n0 = (tile % p.n_tiles) * kWideBN;
    // stream-K roles of this segment: it stops short of the tile's last K-block (dump the partial sums), or finishes a tile whose
    // first K-blocks were summed by lower-numbered CTAs (collect their partials first)
    const bool sk_dump = !kChain && it.kb1 < p.num_kb;      // the chained form has no stream-K
    const bool sk_collect = !kChain && !sk_dump && it.kb0 > 0;
    float tab = 0.f;                           // table entry te: column pair te / 4, {scale, scale, shift, shift}[te % 4]
    {
      const int col = n0 + 2 * (te >> 2) + (te & 1);
      if (!sk_dump && col < p.cout) tab = __ldg(((te & 2) ? p.shift : p.scale) + col);
    }
    // waits for K-block kb's stage and returns its B descriptor
    auto stage_ready = [&](int kb) {
      mbar_wait(bar_full + 8 * stage, phase, p.dbg, 0x700 | stage);
      if (leader) {
        if (kb == kb_last) YB_TRACE(1, tr_t);
        if (kb == kb_first) YB_TRACE(1, tr_t + 1);
      }
      wgmma_fence();
      return make_kmajor_desc<Cfg::kSwizzle>(smem_b + stage * Cfg::kBBytes);
    };
    // one K-block of MMAs into the accumulator rows 64 h .. 64 h + 63
    auto mma_rows = [&](float (&d)[64], int h, uint64_t bdesc, bool first_kb) {
      const uint64_t adesc = make_kmajor_desc<Cfg::kSwizzle>(smem_a + stage * Cfg::kABytes + (cw * 128 + h * 64) * Cfg::kSwizzle);
#pragma unroll
      for (int k = 0; k < BK / UMMA_K; ++k) wgmma_f16<kWideBN>(d, adesc + 2 * k, bdesc + 2 * k, !first_kb || k != 0);
    };
    // the MMAs of the stage before `stage` have retired: hand it back to the producer
    auto release_prev = [&]() {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * (stage == 0 ? kStages - 1 : stage - 1));
    };
    auto next_stage = [&](int kb) {
      if (kb != kb_first) release_prev();
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    };
    for (int kb = kb_first; kb < kb_last; ++kb) {
      const uint64_t bdesc = stage_ready(kb);
      mma_rows(acc[0], 0, bdesc, kb == kb_first);
      mma_rows(acc[1], 1, bdesc, kb == kb_first);
      wgmma_commit();
      wgmma_wait<1>();      // one group in flight: the previous K-block's MMAs have retired, so its stage can be refilled
      next_stage(kb);
    }
    {
      // the last K-block, committed as two groups: rows 0..63 retire first
      const uint64_t bdesc = stage_ready(kb_last);
      mma_rows(acc[0], 0, bdesc, kb_last == kb_first);
      wgmma_commit();
      mma_rows(acc[1], 1, bdesc, kb_last == kb_first);
      wgmma_commit();
      wgmma_wait<1>();
      fence_regs(acc[0]);
      next_stage(kb_last);
    }

    int sk_lo = 0;
    if (sk_collect) {
      const int u = tile * p.num_kb;
      const int wide = p.sk_rem * (p.sk_base + 1);
      sk_lo = u < wide ? u / (p.sk_base + 1) : p.sk_rem + (u - wide) / p.sk_base;
      if (leader) {
        for (int j = sk_lo; j < static_cast<int>(blockIdx.x); ++j) {
          uint32_t spins = 0;
          uint64_t t0 = 0;
          while (ld_acquire_gpu(p.flags + j) == 0u) {
            if ((++spins & 0x3FFu) == 0) {
              const uint64_t now = globaltimer_ns();
              if (t0 == 0) t0 = now;
              if (now - t0 > 4000000000ull) {
                if (p.dbg != nullptr) { p.dbg[0] = 0x0BAD0800; p.dbg[1] = static_cast<int>(blockIdx.x); p.dbg[2] = j; p.dbg[3] = tile; __threadfence_system(); }
                __trap();
              }
            }
          }
        }
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    if (!sk_dump) {
      // every consumer thread is done with the previous tile's table before it is overwritten, and reads this one after
      asm volatile("bar.sync 1, 256;" ::: "memory");
      asm volatile("st.shared.f32 [%0], %1;" :: "r"(table + 4 * te), "f"(tab) : "memory");
      asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    // per-thread partial layout: float4 g of thread t of consumer cw at ((cw * 32 + g) * 128 + t) * 4 -- coalesced both ways;
    // g / 16 is the accumulator row half h
    uint32_t pk_dx0[kPool ? 32 : 1];           // pooled form: the converted h = 0 half (window column dx = 0), kept for the dx max
    // chained form: converted half h is the register A operand of the second GEMM into acc2[h]; it stays live until that GEMM retires
    uint32_t pk_a[kChain ? 2 : 1][kChain ? 32 : 1];
    float acc2[kChain ? 2 : 1][kChain ? 32 : 1];
    // chained form: scale / shift, leaky, fp16 of the second unit for one 64-row half, staged for its 64-channel store
    auto chain_store = [&](const float (&d)[kChain ? 32 : 1]) {
      if constexpr (kChain) {
        const float4* tab2 = reinterpret_cast<const float4*>(smem_raw + (table2 - smem_u32(smem_raw)));
        uint32_t pk2[16];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const float4 ss = tab2[4 * jj + (lane & 3)];
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            float x0 = d[4 * jj + 2 * hh] * ss.x + ss.z;
            float x1 = d[4 * jj + 2 * hh + 1] * ss.y + ss.w;
            x0 = x0 > 0.f ? x0 : x0 * p.slope2;
            x1 = x1 > 0.f ? x1 : x1 * p.slope2;
            __half2 v = __floats2half2_rn(x0, x1);
            pk2[2 * jj + hh] = *reinterpret_cast<uint32_t*>(&v);
          }
        }
        mbar_wait(bar_slice_empty + 8 * cw, sph ^ 1, p.dbg, 0xA00 | cw);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int r = warp * 16 + (lane >> 2) + hh * 8;
            const uint32_t addr = slice + r * 128 + ((jj ^ (r & 7)) << 4) + 4 * (lane & 3);
            asm volatile("st.shared.b32 [%0], %1;" :: "r"(addr), "r"(pk2[2 * jj + hh]) : "memory");
          }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_slice_full + 8 * cw);
        sph ^= 1;
      }
    };
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1) {
        wgmma_wait<0>();                       // chained: also the second GEMM of rows 0..63, committed after these MMAs
        fence_regs(acc[1]);
        if (leader) YB_TRACE(2, tr_t);
        release_prev();
        if constexpr (kChain) {
          // rows 0..63 of the second unit go out before rows 64..127 are converted (keeping both halves' second-GEMM operands live
          // at once would spill); the last stage is already back with the producer
          fence_regs(acc2[0]);
          fence_regs_u32(pk_a[0]);
          chain_store(acc2[0]);
        }
      }
      if (sk_dump) {
        float4* dst = reinterpret_cast<float4*>(p.ws + static_cast<size_t>(blockIdx.x) * Cfg::kWsFloats) + (cw * 32 + 16 * h) * 128 + t;
#pragma unroll
        for (int g = 0; g < 16; ++g) dst[g * 128] = make_float4(acc[h][4 * g], acc[h][4 * g + 1], acc[h][4 * g + 2], acc[h][4 * g + 3]);
        continue;
      }
      for (int j = sk_lo; j < (sk_collect ? static_cast<int>(blockIdx.x) : 0); ++j) {
        const float4* src = reinterpret_cast<const float4*>(p.ws + static_cast<size_t>(j) * Cfg::kWsFloats) + (cw * 32 + 16 * h) * 128 + t;
#pragma unroll
        for (int g = 0; g < 16; ++g) {
          const float4 a = __ldcg(src + g * 128);
          acc[h][4 * g] += a.x; acc[h][4 * g + 1] += a.y; acc[h][4 * g + 2] += a.z; acc[h][4 * g + 3] += a.w;
        }
      }
      // scale / shift, leaky, fp16.  Fragment of thread t: acc[h][4 j + 2 hh + e] is tile row 64 h + 16 warp + lane / 4 + 8 hh,
      // column 8 j + 2 (lane % 4) + e; pk[16 c2 + 2 jj + hh] holds the pair of j = 8 c2 + jj
      uint32_t pk[32];
#pragma unroll
      for (int c2 = 0; c2 < 2; ++c2) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const float4 ss = tab4[c2 * 32 + 4 * jj + (lane & 3)];
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int j = c2 * 8 + jj;
            float x0 = acc[h][4 * j + 2 * hh] * ss.x + ss.z;
            float x1 = acc[h][4 * j + 2 * hh + 1] * ss.y + ss.w;
            x0 = x0 > 0.f ? x0 : x0 * p.slope;
            x1 = x1 > 0.f ? x1 : x1 * p.slope;
            __half2 v = __floats2half2_rn(x0, x1);
            pk[16 * c2 + 2 * jj + hh] = *reinterpret_cast<uint32_t*>(&v);
          }
        }
      }
      if constexpr (kPool) {
        if (h == 0) {
#pragma unroll
          for (int i = 0; i < 32; ++i) pk_dx0[i] = pk[i];
          continue;
        }
        // fp16 max in maxpool2x2_kernel's order: max(max(dx 0, dx 1) of row dy 0, the same of row dy 1), pair by pair
#pragma unroll
        for (int i = 0; i < 32; ++i) pk[i] = hmax2_u32(pk_dx0[i], pk[i]);
        if (cw == 0) {
          // consumer 1 staged row dy = 1 at the same slice positions this thread stages: take the dy max, then hand its slice back
          mbar_wait(bar_slice_full + 8, sph, p.dbg, 0xB00);
#pragma unroll
          for (int c2 = 0; c2 < 2; ++c2)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int hh = 0; hh < 2; ++hh) {
                const int r = warp * 16 + (lane >> 2) + hh * 8;
                const uint32_t addr = smem_o + Cfg::kOutBytes + c2 * 8192 + r * 128 + ((jj ^ (r & 7)) << 4) + 4 * (lane & 3);
                uint32_t v;
                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
                pk[16 * c2 + 2 * jj + hh] = hmax2_u32(pk[16 * c2 + 2 * jj + hh], v);
              }
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_slice_empty + 8);
        }
      }
      if constexpr (kChain) {
        // the 1x1 unit that follows: its 128 input channels of these 64 rows are pk, which is exactly the A fragment of an
        // m64 x 16 step -- k-step kk (channels 16 kk .. 16 kk + 15) is pk[4 kk .. 4 kk + 3].  The k16 steps run in channel order
        // from scale-d = 0, as in the plain launch of that unit.
#pragma unroll
        for (int i = 0; i < 32; ++i) pk_a[h][i] = pk[i];
        mbar_wait(bar_w, 0, p.dbg, 0xC00);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          const uint32_t a[4] = {pk_a[h][4 * kk], pk_a[h][4 * kk + 1], pk_a[h][4 * kk + 2], pk_a[h][4 * kk + 3]};
          const uint64_t bdesc = make_kmajor_desc<128>(smem_o + (kk >> 2) * Cfg::kOutBytes + 8192) + 2 * (kk & 3);
          wgmma_f16_rs_n64(acc2[h], a, bdesc, kk != 0);
        }
        wgmma_commit();
        if (h == 0) continue;                  // rows 0..63's second GEMM queues behind the MMAs of rows 64..127
        wgmma_wait<0>();
        fence_regs(acc2[1]);
        fence_regs_u32(pk_a[1]);
        chain_store(acc2[1]);
        continue;
      }
      // the slice is free once the store thread (pooled, consumer 1: consumer 0) has seen the previous half's stores read it
      mbar_wait(bar_slice_empty + 8 * cw, sph ^ 1, p.dbg, 0xA00 | cw);
#pragma unroll
      for (int c2 = 0; c2 < 2; ++c2)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int r = warp * 16 + (lane >> 2) + hh * 8;       // row inside the half
            const uint32_t addr = slice + c2 * 8192 + r * 128 + ((jj ^ (r & 7)) << 4) + 4 * (lane & 3);
            asm volatile("st.shared.b32 [%0], %1;" :: "r"(addr), "r"(pk[16 * c2 + 2 * jj + hh]) : "memory");
          }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_slice_full + 8 * cw);
      sph ^= 1;
    }
    if (sk_dump) {
      __threadfence();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (leader) st_release_gpu(p.flags + blockIdx.x, 1u);
      continue;
    }
    if (leader) YB_TRACE(2, tr_t + 1);
    if (sk_collect) {
      // every reader is done with the partials: hand the slots back (the next writer is a later launch)
      asm volatile("bar.sync 1, 256;" ::: "memory");
      for (int j = sk_lo + t + 128 * cw; j < static_cast<int>(blockIdx.x); j += 256) p.flags[j] = 0u;
    }
  }
}

template <int BK>
__global__ void __launch_bounds__(kWideThreads, 1)
conv_wide_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_y, const ConvParams p) {
  const CUtensorMap* const ta[4] = {&tmap_a, &tmap_a, &tmap_a, &tmap_a};
  conv_wide_body<BK, false, false>(ta, tmap_b, tmap_y, nullptr, p);
}

// The same tile with the 2x2 max-pool that follows a 3x3 same-padded layer fused into its epilogue (YB_CONV_POOL2X2): a tile is 64 pool
// windows x their 4 positions, and only the 64 x 128 pooled outputs are stored.  Position (dy, dx) of window (i, j) is output pixel
// (2 i + dy, 2 j + dx), so each position is a stride-2 conv whose window corners start at (dy - 1, dx - 1): tmap_a<2 dy + dx> is that
// im2col map and fills stage rows 64 (2 dy + dx) .. + 63.  Consumer dy thus holds positions (dy, 0) and (dy, 1) of the same window in
// its two accumulator halves, on the same thread: it takes the dx max in registers after the fp16 rounding, consumer 1 stages its
// result, consumer 0 takes the dy max against it and stages the pooled slice for one TMA store.  Every output is the fp32 sum of the
// plain tile (same K-blocks, same k16 steps), so the result equals conv_wide_kernel + maxpool2x2_kernel bit for bit.  No stream-K.
template <int BK>
__global__ void __launch_bounds__(kWideThreads, 1)
conv_wide_pool_kernel(const __grid_constant__ CUtensorMap tmap_a0, const __grid_constant__ CUtensorMap tmap_a1,
                      const __grid_constant__ CUtensorMap tmap_a2, const __grid_constant__ CUtensorMap tmap_a3,
                      const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ CUtensorMap tmap_y, const ConvParams p) {
  const CUtensorMap* const ta[4] = {&tmap_a0, &tmap_a1, &tmap_a2, &tmap_a3};
  conv_wide_body<BK, true, false>(ta, tmap_b, tmap_y, nullptr, p);
}

// The same tile with the 1x1 unit that follows the layer run in its epilogue (YB_CONV_CHAIN1X1): after a 64-row half of the tile is
// converted to fp16, its 128 channels (the layer's whole Cout, one N tile) are the A operand of a second GEMM against the unit's
// [Cout2 <= 64][128] weight, straight from the registers.  Only that unit's scale / shift / leaky output is stored; the layer's own
// output never leaves the SM.  The second GEMM runs the same k16 steps in the same channel order from scale-d = 0 on the same fp16
// operands as the unit's plain launch, and the epilogue arithmetic is the same, so the result equals conv_wide_kernel followed by
// the unit's launch bit for bit.  BK = 64, no stream-K.
template <int BK>
__global__ void __launch_bounds__(kWideThreads, 1)
conv_wide_chain_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_y, const __grid_constant__ CUtensorMap tmap_w2, const ConvParams p) {
  static_assert(BK == 64, "chained form: instantiated for producers with Cin % 64 == 0 only (conv_choose refuses the others)");
  const CUtensorMap* const ta[4] = {&tmap_a, &tmap_a, &tmap_a, &tmap_a};
  conv_wide_body<BK, false, true>(ta, tmap_b, tmap_y, &tmap_w2, p);
}

// ---------------------------------------------------------------------------------------------
// Halo-tile kernel for 3x3, Cin = 32 (layers1.2).  The im2col formulation above pulls every input pixel through the
// L2 -> SM path nine times (once per tap): 779 MB for 88 MB of input at batch 32.  Here an output tile is a 16 x 8 pixel
// rectangle and its 18 x 10 x 32ch input halo is fetched ONCE (11.5 KB instead of 72 KB) as four 8-channel planes
// [pixel][16 B].  In that layout a 3x3 tap is just a shifted window: 8 consecutive pixels of a halo row form one 8 x 16 B
// core matrix of the un-swizzled K-major operand format, the next output row is +10 pixels (SBO = 160 B) and the second
// K chunk is the next plane (LBO), so wgmma reads all nine taps straight out of the halo tile by moving the
// descriptor's start address by (r * 10 + s) * 16 B.  The epilogue can apply the 2x2 max-pool that follows this layer
// and ships the tile with one TMA store, so the un-pooled activation never reaches HBM in inference.  The first form
// (conv_c32_kernel_v1) keeps the weights resident in shared memory and pools across lanes (lane ^ 1 and lane ^ 8 hold the
// horizontal / vertical neighbours); conv_c32_kernel below holds them in registers and pools within a thread.
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
  static constexpr int kSmemBytes = 1024 + kBBytes + 2 * kGroups * kOutBytes + kStages * kHalo + kGroups * kAccBytes + 2 * BN * 4 + 256 + 2 * BN * 8 /*stats*/;
  static_assert(kSmemBytes <= kSmemLimit, "c32: shared memory budget");
};

// The first form (YB_CONV_C32_V1=1 for A/B runs, and the training forward with statistics): one MMA warpgroup with both operands in
// shared memory, the accumulator handed through a shared-memory tile to two epilogue groups.
__global__ void __launch_bounds__(C32Cfg::kThreads, 1)
conv_c32_kernel_v1(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
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
  // [2][BN] double, accumulated over all of this CTA's tiles: each warp's 32-pixel fp32 column sum is added in double, so the fp32 part of the
  // statistics is five roundings deep however many tiles the CTA runs (the variance amplifies it by 1 + (mean / std)^2)
  double* ep_stats = reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(bars) + 256);
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
      ep_stats[i] = 0.0; ep_stats[BN + i] = 0.0;
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
          atomicAdd(&ep_stats[half * 32 + lane], static_cast<double>(a1[0]));
          atomicAdd(&ep_stats[BN + half * 32 + lane], static_cast<double>(a2[0]));
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
        atomicAdd(p.stats + i, ep_stats[i]);
        atomicAdd(p.stats + p.cout + i, ep_stats[BN + i]);
      }
    }
  }
}

// The halo tile computed transposed, D^T[64 channels x 128 pixels] = W . X^T, so shared memory is off the critical path:
//   * A is the weight, held in registers for the whole kernel (18 k16 steps x 4 registers per thread, loaded once per CTA);
//   * B is the halo window, read by one m64n128k16 per k16 step with the same descriptor form as the first form's A (K-major, no
//     swizzle, LBO = plane, SBO = one halo row; tap (r, s) = start shifted by (r * 10 + s) * 16 B), so a tile reads 72 KB of shared
//     memory for its MMAs instead of 144 KB;
//   * warpgroup 0 is the TMA producer (one thread); warpgroups 1 and 2 each take alternate tiles of the CTA's list and run their own
//     epilogue from the registers, so one consumer's epilogue runs under the other's MMAs.
// The k16 steps run in the first form's order (per tap, channels 0-15 then 16-31; taps 0..8) on the same fp16 operands and the
// epilogue arithmetic is the same (scale / shift and leaky in fp32, the 2x2 max on the fp32 values in the first form's operand
// order, then RN to fp16), so the output equals conv_c32_kernel_v1's bit for bit.  Thread l of warp w holds channels
// 16 w + l / 4 (+ 8) of tile pixels (row j, columns 2 (l % 4) + {0, 1}) for all 16 rows j: a 2x2 pool window is in one thread.
struct C32RegCfg {
  static constexpr int kStages = 8;
  static constexpr int kOutBytes = 128 * 128;                     // one tile's staged output: 128 pixels x 64 channels fp16, 128B-swizzled
  static constexpr int kSmemBytes = 1024 + 4 * kOutBytes + kStages * C32Cfg::kHalo + 256;    // 2 staging buffers per consumer, barriers
  static_assert(kSmemBytes <= kSmemLimit, "c32: shared memory budget");
};

__global__ void __launch_bounds__(kWideThreads, 1)
conv_c32_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_y, const __half* __restrict__ w,
                const C32Params p) {
  using Cfg = C32Cfg;
  constexpr int kStages = C32RegCfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_o = smem_base;                                      // [2 consumers][2 buffers][kOutBytes]
  const uint32_t smem_h = smem_o + 4 * C32RegCfg::kOutBytes;              // [kStages][kHalo]
  const uint32_t bar_full = smem_h + kStages * Cfg::kHalo;
  const uint32_t bar_empty = bar_full + 8 * kStages;
  const uint32_t bar_turn = bar_empty + 8 * kStages;                      // [2 consumers]: the other consumer's MMAs have retired

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 4); }   // one arrival per consumer warp
    for (int c = 0; c < 2; ++c) mbar_init(bar_turn + 8 * c, 4);
    fence_mbar_init();
    fence_proxy_async_smem();
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_y);
  }
  __syncthreads();
  pdl_trigger();        // an ordinary launch itself; lets a PDL successor set up while this grid drains

  // trace (yb_conv_set_trace; block 0), tile i of the CTA: role 0 slot i = its halo load issue, role 1 slot i = its first wgmma issue;
  // role 2 slot 2i = its MMAs retired, 2i + 1 = its epilogue end (store issued)
  if (threadIdx.x < 128) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0; int tr = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int tw = tile % p.tiles_w;
        const int rest = tile / p.tiles_w;
        const int th = rest % p.tiles_h;
        const int n = rest / p.tiles_h;
        mbar_wait(bar_empty + 8 * stage, phase ^ 1, p.dbg, 0xB50 | stage);
        YB_TRACE(0, tr); ++tr;
        if (p.skip & 1) {
          mbar_arrive(bar_full + 8 * stage);
        } else {
          mbar_arrive_expect_tx(bar_full + 8 * stage, 4 * Cfg::kPlaneData);
          for (int c = 0; c < 4; ++c)
            tma_load_4d(smem_h + stage * Cfg::kHalo + c * Cfg::kPlane, &tmap_x, bar_full + 8 * stage, c * 8, tw * Cfg::TW - 1, th * Cfg::TH - 1, n);
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int cw = (threadIdx.x >> 7) - 1;        // consumer cw takes the CTA's tiles cw, cw + 2, ...
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const int ch0 = 16 * warp + (lane >> 2);      // this thread's channels: ch0 (h = 0) and ch0 + 8 (h = 1)
  // the weight as the A fragment of every k16 step ks (tap ks / 2, channels 16 (ks % 2) ..): rows ch0 / ch0 + 8, K columns
  // 2 (l % 4) + {0, 1} and 8 + the same.  Rows >= Cout are zero.
  uint32_t wa[18][4];
  {
    const unsigned int* wrow[2];
    bool live[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      live[h] = ch0 + 8 * h < p.cout;
      wrow[h] = reinterpret_cast<const unsigned int*>(w + (live[h] ? ch0 + 8 * h : 0) * 288 + 2 * (lane & 3));
    }
#pragma unroll
    for (int ks = 0; ks < 18; ++ks)
#pragma unroll
      for (int i = 0; i < 4; ++i) wa[ks][i] = live[i & 1] ? __ldg(wrow[i & 1] + ks * 8 + 4 * (i >> 1)) : 0u;
  }
  float sc[2], sh[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    sc[h] = ch0 + 8 * h < p.cout ? __ldg(p.scale + ch0 + 8 * h) : 0.f;
    sh[h] = ch0 + 8 * h < p.cout ? __ldg(p.shift + ch0 + 8 * h) : 0.f;
  }
  const uint32_t lbo = p.swap_lbo ? Cfg::HW * 16 : Cfg::kPlane;
  const uint32_t sbo = p.swap_lbo ? Cfg::kPlane : Cfg::HW * 16;
  const int mi = lane >> 3, mr = lane & 7;       // stmatrix: this thread addresses row mr of matrix mi
  float acc[64];
  int use = 0;                                   // tiles this consumer has staged
  for (int local = cw, tile = blockIdx.x + cw * gridDim.x; tile < p.num_tiles; local += 2, tile += 2 * gridDim.x, ++use) {
    const int stage = local % kStages;
    // the consumers take turns on the tensor cores (tile local - 1's MMAs have retired), so one's epilogue runs under the other's
    // MMAs instead of both issuing together and then both converting
    if (local > 0) mbar_wait(bar_turn + 8 * cw, ((local - 1) >> 1) & 1, p.dbg, 0xB70 | cw);
    mbar_wait(bar_full + 8 * stage, (local / kStages) & 1, p.dbg, 0xB60 | stage);
    if (t == 0) YB_TRACE(1, local);
    const uint32_t halo = smem_h + stage * Cfg::kHalo;
    if (!(p.skip & 4)) {
      wgmma_fence();
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const uint32_t win = halo + ((tap / 3) * Cfg::HW + (tap % 3)) * 16;      // tap (r, s): window shifted by r rows, s pixels
        wgmma_f16_rs_n128(acc, wa[2 * tap], make_kmajor_desc_noswz(win, lbo, sbo), tap != 0);
        wgmma_f16_rs_n128(acc, wa[2 * tap + 1], make_kmajor_desc_noswz(win + 2 * Cfg::kPlane, lbo, sbo), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
    }
    fence_regs(acc);
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(bar_empty + 8 * stage);
      mbar_arrive(bar_turn + 8 * (cw ^ 1));
    }
    if (t == 0) YB_TRACE(2, 2 * local);
    const int tw = tile % p.tiles_w;
    const int rest = tile / p.tiles_w;
    const int th = rest % p.tiles_h;
    const int n = rest / p.tiles_h;
    // scale / shift, leaky: acc[4 j + 2 h + e] is channel ch0 + 8 h, pixel (row j, column 2 (l % 4) + e)
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = acc[4 * j + 2 * h + e] * sc[h] + sh[h];
          acc[4 * j + 2 * h + e] = x > 0.f ? x : x * p.slope;
        }
    const uint32_t obuf = smem_o + (cw * 2 + (use & 1)) * C32RegCfg::kOutBytes;
    if (t == 0) tma_store_wait_read<1>();        // this consumer's store from two of its tiles ago has drained the buffer
    asm volatile("bar.sync %0, 128;" :: "r"(1 + cw) : "memory");
    // staged as [pixel][64 channels], 16-byte chunk c of pixel row px at (c ^ (px & 7)): the TMA store's 128B swizzle.  The matrices of
    // one stmatrix are (rows = channels ch0 - lane / 4 + 8 h, columns = 8 pixels); chunk 2 warp + h of the pixels they cover.
    if (p.pool) {
      // window (i, l % 4) is rows 2 i, 2 i + 1, columns 2 (l % 4) + {0, 1}: max(max(row 2 i), max(row 2 i + 1)) in the first form's order.
      // Matrix (i2, h): fragment column 2 (l % 4) + e is pooled pixel (2 i2 + e, l % 4), stored at pooled row (2 i2 + e) * 4 + l % 4.
      float pm[8][2];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          pm[i][h] = fmaxf(fmaxf(acc[4 * (2 * i) + 2 * h], acc[4 * (2 * i) + 2 * h + 1]),
                           fmaxf(acc[4 * (2 * i + 1) + 2 * h], acc[4 * (2 * i + 1) + 2 * h + 1]));
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        uint32_t r[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int i2 = 2 * k + (m >> 1), h = m & 1;
          __half2 v = __floats2half2_rn(pm[2 * i2][h], pm[2 * i2 + 1][h]);
          r[m] = *reinterpret_cast<uint32_t*>(&v);
        }
        const int px = 8 * (2 * k + (mi >> 1)) + 4 * (mr & 1) + (mr >> 1);
        stmatrix_x4_trans(obuf + px * 128 + (((2 * warp + (mi & 1)) ^ (px & 7)) << 4), r[0], r[1], r[2], r[3]);
      }
    } else {
      // matrix (j, h): fragment column 2 (l % 4) + e is pixel 8 j + 2 (l % 4) + e
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        uint32_t r[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int j = 2 * k + (m >> 1), h = m & 1;
          __half2 v = __floats2half2_rn(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          r[m] = *reinterpret_cast<uint32_t*>(&v);
        }
        const int px = 8 * (2 * k + (mi >> 1)) + mr;
        stmatrix_x4_trans(obuf + px * 128 + (((2 * warp + (mi & 1)) ^ (px & 7)) << 4), r[0], r[1], r[2], r[3]);
      }
    }
    fence_proxy_async_smem();
    asm volatile("bar.sync %0, 128;" :: "r"(1 + cw) : "memory");
    if (t == 0) {
      if (!(p.skip & 8)) {
        if (p.pool) tma_store_4d(&tmap_y, obuf, 0, tw * (Cfg::TW / 2), th * (Cfg::TH / 2), n);
        else tma_store_4d(&tmap_y, obuf, 0, tw * Cfg::TW, th * Cfg::TH, n);
      }
      tma_store_commit();
      YB_TRACE(2, 2 * local + 1);
    }
  }
  if (t == 0) tma_store_wait<0>();
}

// ---------------------------------------------------------------------------------------------
// Host side: tensor-map encoding through the driver entry points (no link-time libcuda dependency)
// ---------------------------------------------------------------------------------------------
constexpr long long kSkFlagBytes = 4096;          // room for 1024 CTA flags
constexpr long long kSkSlotBytes = kWideRows * kWideBN * 4;  // one CTA's largest partial accumulator (the 256 x 128 fp32 tile)
long long conv_workspace_bytes() { return kSkFlagBytes + kSkSlotBytes * sm_count(); }

constexpr int kKernelIgemm = 0;      // conv_igemm_kernel (one MMA warpgroup, shared-memory accumulator)
constexpr int kKernelWide = 1;       // conv_wide_kernel (256 x 128, two consumer warpgroups)
constexpr int kKernelC32 = 2;        // conv_c32_kernel (3x3, Cin = 32 halo tiles)
struct ConvChoice {
  int kernel, bk, bn, mt, streamk, grid;
  int pool;        // the 2x2 max-pool is fused (conv_c32_kernel, conv_wide_pool_kernel)
  int chain;       // the following 1x1 unit is fused (conv_wide_chain_kernel)
};
constexpr int kFlagChain = 1 << 7;   // YB_CONV_CHAIN1X1

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
static int launch_conv(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ty, const ConvParams& p, const PreAct* pre,
                       cudaStream_t stream) {
  using Cfg = ConvCfg<BN, BK, MT>;
  using PreCfg = ConvCfg<BN, BK, MT, kPreMaxCh>;
  static bool attr_set = false, pre_attr_set = false;
  if (pre == nullptr && !attr_set) {
    YB_CUDA(cudaFuncSetAttribute(conv_igemm_kernel<BN, BK, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  if (pre != nullptr && !pre_attr_set) {
    YB_CUDA(cudaFuncSetAttribute(conv_preact_kernel<BN, BK, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, PreCfg::kSmemBytes));
    pre_attr_set = true;
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
  cfg.dynamicSmemBytes = pre != nullptr ? PreCfg::kSmemBytes : Cfg::kSmemBytes;
  cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = nattr;
  if (pre != nullptr) {
    YB_CUDA(cudaLaunchKernelEx(&cfg, conv_preact_kernel<BN, BK, MT>, ta, tb, ty, p, *pre));
    return check_launch("conv_preact_kernel");
  }
  YB_CUDA(cudaLaunchKernelEx(&cfg, conv_igemm_kernel<BN, BK, MT>, ta, tb, ty, p));
  return check_launch("conv_igemm_kernel");
}

template <int BK>
static int launch_wide(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ty, const ConvParams& p, int grid, cudaStream_t stream) {
  using Cfg = WideCfg<BK>;
  static bool attr_set = false;
  if (!attr_set) {
    YB_CUDA(cudaFuncSetAttribute(conv_wide_kernel<BK>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cudaLaunchAttribute attr[1];
  int nattr = 0;
  static const int use_pdl = getenv("YB_PDL") ? atoi(getenv("YB_PDL")) : 0;     // as launch_conv: A/B runs only
  if (use_pdl) {
    attr[nattr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[nattr].val.programmaticStreamSerializationAllowed = 1;
    ++nattr;
  }
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kWideThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = nattr;
  YB_CUDA(cudaLaunchKernelEx(&cfg, conv_wide_kernel<BK>, ta, tb, ty, p));
  return check_launch("conv_wide_kernel");
}

// the pooled form: ta[2 dy + dx] is the A map of window position (dy, dx)
template <int BK>
static int launch_wide_pool(const CUtensorMap (&ta)[4], const CUtensorMap& tb, const CUtensorMap& ty, const ConvParams& p, int grid,
                            cudaStream_t stream) {
  using Cfg = WideCfg<BK>;
  static bool attr_set = false;
  if (!attr_set) {
    YB_CUDA(cudaFuncSetAttribute(conv_wide_pool_kernel<BK>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  conv_wide_pool_kernel<BK><<<grid, kWideThreads, Cfg::kSmemBytes, stream>>>(ta[0], ta[1], ta[2], ta[3], tb, ty, p);
  return check_launch("conv_wide_pool_kernel");
}

// the chained form: ty is the second unit's output, tw2 its weight
static int launch_wide_chain(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ty, const CUtensorMap& tw2, const ConvParams& p,
                             int grid, cudaStream_t stream) {
  using Cfg = WideCfg<64>;
  static bool attr_set = false;
  if (!attr_set) {
    YB_CUDA(cudaFuncSetAttribute(conv_wide_chain_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kChainSmemBytes));
    attr_set = true;
  }
  conv_wide_chain_kernel<64><<<grid, kWideThreads, Cfg::kChainSmemBytes, stream>>>(ta, tb, ty, tw2, p);
  return check_launch("conv_wide_chain_kernel");
}

// CTA tile shapes (BLOCK_N, M-subtiles): the one-warpgroup kernel keeps MT * BLOCK_N <= 128 accumulators per thread; 128 x 2 is
// the two-consumer kernel
// the two-consumer shape has no pre-activation form (conv_choose never picks it when `pre` is set)
template <int BK>
static int dispatch_conv(int bn, int mt, int grid, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ty, const ConvParams& p,
                         const PreAct* pre, cudaStream_t stream) {
  if (mt == 2 && bn == 128) return launch_wide<BK>(ta, tb, ty, p, grid, stream);
  if (mt == 2) return launch_conv<64, BK, 2>(ta, tb, ty, p, pre, stream);
  if (bn == 64) return launch_conv<64, BK, 1>(ta, tb, ty, p, pre, stream);
  return launch_conv<128, BK, 1>(ta, tb, ty, p, pre, stream);
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
  // the first form (conv_c32_kernel_v1) for the training forward's statistics, and for every launch with YB_CONV_C32_V1=1 (A/B runs)
  static const int force_v1 = getenv("YB_CONV_C32_V1") ? atoi(getenv("YB_CONV_C32_V1")) : 0;
  const bool v1 = force_v1 != 0 || stats != nullptr;
  if (v1) {
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
  const int grid = p.num_tiles < sm_count() ? p.num_tiles : sm_count();
  if (v1) {
    static bool attr_set = false;
    if (!attr_set) {
      YB_CUDA(cudaFuncSetAttribute(conv_c32_kernel_v1, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
      attr_set = true;
    }
    conv_c32_kernel_v1<<<grid, Cfg::kThreads, Cfg::kSmemBytes, stream>>>(tx, tw, ty, p);
    return check_launch("conv_c32_kernel_v1");
  }
  static bool attr_set = false;
  if (!attr_set) {
    YB_CUDA(cudaFuncSetAttribute(conv_c32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C32RegCfg::kSmemBytes));
    attr_set = true;
  }
  conv_c32_kernel<<<grid, kWideThreads, C32RegCfg::kSmemBytes, stream>>>(tx, ty, static_cast<const __half*>(w), p);
  return check_launch("conv_c32_kernel");
}

// Kernel and tile shape of one conv launch.  flags may force BLOCK_N (bits 8..17) and the number of 128-row M-subtiles
// (bits 20..21), forbid (bit 3) or force (bit 30) stream-K; otherwise the (BLOCK_N, M-subtiles, stream-K) triple with the lowest
// modelled time wins.  Model (constants fitted to profiles/conv_layers_h100.json: every shape of the 21 implicit-GEMM launches of
// C2 timed alone on an H100 SXM at a 700 W power limit, median of three runs): tiles run in ceil(tiles / SMs) rounds; a K-block costs a fixed issue latency (im2col boxes cost
// more than plain tiled ones) plus its operand bytes at a per-SM L2->SM rate; the one-warpgroup kernel's epilogue overlaps the
// next main loop (a tile costs the larger of the two), the two-consumer kernel's register epilogue mostly does not (they add).  With
// these constants the model picks, on each of those 21 launches, a shape within 3 % of the fastest one measured.
constexpr double kKbNsIm2col = 240.0;     // ns per K-block, every conv but 1x1 stride 1 (im2col-mode A box)
constexpr double kKbNsTiled = 100.0;      // ns per K-block, 1x1 stride-1 layers (plain 2-D tiled A box)
constexpr double kFeedBytesPerNs = 130.0; // L2 -> SM operand bytes per ns per SM
constexpr double kEpiNsPerOut = 0.15;     // one-warpgroup epilogue, ns per output element (overlapped with the main loop)
constexpr double kWideEpiNsPerOut = 0.04; // two-consumer register epilogue, ns per output element (what the next tile's MMAs do not hide)
constexpr double kSkNs = 16000.0;         // stream-K partial dump + collect, one-warpgroup kernel
constexpr double kSkNsWide = 9000.0;      // the same from registers, two-consumer kernel
// height / width are the OUTPUT dims (M counts output pixels); a K-block of every conv but 1x1 stride 1 pays the im2col box cost.
int conv_choose(int batch, int height, int width, int cin, int cout, int kh, int kw, int stride, int pad_h, int pad_w, int a_channels, int out_mode,
                int flags, bool workspace_ok, bool stats, bool lo, bool pre, ConvChoice* out) {
  ConvChoice c;
  memset(&c, 0, sizeof(c));
  const int sms = sm_count();
  const bool split = a_channels != cin || lo;
  const bool same3x3 = kh == 3 && kw == 3 && stride == 1 && pad_h == 1 && pad_w == 1;
  const bool im2col_cost = !(kh == 1 && kw == 1 && stride == 1);
  // 3x3 same-padded stride 1, Cin = 32, Cout <= 64 (layers1.2): halo-tile kernel unless a test asks for one of the im2col kernels
  if (!split && cin == 32 && same3x3 && cout <= 64 && out_mode == 0 && ((flags >> 28) & 1) == 0 && ((flags >> 5) & 1) == 0 && ((flags >> 7) & 1) == 0 &&
      ((flags >> 8) & 0xFFFF) == 0) {
    const long long tiles = static_cast<long long>(batch) * ((width + C32Cfg::TW - 1) / C32Cfg::TW) * ((height + C32Cfg::TH - 1) / C32Cfg::TH);
    c.kernel = kKernelC32; c.bk = 32; c.bn = C32Cfg::BN; c.mt = 1; c.pool = (flags >> 4) & 1;
    c.grid = static_cast<int>(tiles < sms ? tiles : sms);
    *out = c;
    return 0;
  }
  // the fused 2x2 max-pool outside the Cin = 32 kernel: the two-consumer tile's pooled form, on the layers whose selection is that tile
  const bool pool = (flags >> 4) & 1;
  if (pool) {
    if (!(same3x3 && height % 2 == 0 && width % 2 == 0 && out_mode == 0 && !split && !stats && !pre))
      return fail(YB_ERR_UNSUPPORTED, "conv: YB_CONV_POOL2X2 needs a 3x3 same-padded stride-1 layer with even H and W, fp16 NHWC output and "
                                      "plain operands");
    if ((flags >> 30) & 1) return fail(YB_ERR_UNSUPPORTED, "conv: the fused 2x2 max-pool has no stream-K form");
  }
  const int bk = (cin % 64 == 0 && a_channels % 64 == 0) ? 64 : 32;     // K-blocks never straddle the wrap point
  // the following 1x1 unit fused into the epilogue: the two-consumer tile whose one N tile is the layer's whole Cout = 128
  const bool chain = (flags >> 7) & 1;
  if (chain) {
    if (!(out_mode == 0 && !split && !stats && !pre && !pool && bk == 64 && cout == kWideBN))
      return fail(YB_ERR_UNSUPPORTED, "conv: YB_CONV_CHAIN1X1 needs Cout = %d, Cin %% 64 == 0, fp16 NHWC output, plain operands and no fused "
                                      "pool (Cout %d, Cin %d)", kWideBN, cout, cin);
    if ((flags >> 30) & 1) return fail(YB_ERR_UNSUPPORTED, "conv: the chained form has no stream-K form");
  }
  const bool sk_possible = !stats && !pool && !chain && workspace_ok && (flags & 8) == 0;
  const bool sk_force = sk_possible && ((flags >> 30) & 1);
  // the two-consumer kernel: fp16 NHWC through the TMA store, no residual output, statistics or profiling ablation
  // (the pre-activation form exists only for the one-warpgroup kernel)
  const bool wide_ok = out_mode == 0 && !lo && !stats && !pre && ((flags >> 24) & 0xF) == 0 && ((flags >> 29) & 1) == 0;
  const int force_bn = (flags >> 8) & 0x3FF;
  const int force_mt = (flags >> 20) & 0x3;
  const int force_pair = (flags >> 22) & 0x3;      // 0 = auto, 1 = single-CTA tiles (the only form), 2 = CTA pair (not on sm_90)
  YB_REQUIRE(force_pair != 2, "conv: CTA-pair tiles need two-CTA tensor-core instructions, which sm_90 does not have");
  YB_REQUIRE(!force_bn || ((force_bn == 64 || force_bn == 128) && (force_mt != 2 || force_bn == 64 || wide_ok)),
             "conv: BLOCK_N=%d x %d M-subtiles is not a tile shape of this launch (64 x 1, 128 x 1, 64 x 2; 128 x 2 for fp16 NHWC "
             "outputs without residual or statistics)", force_bn, force_mt ? force_mt : 1);
  const long long m_total = static_cast<long long>(batch) * height * width;
  const int num_kb = kh * kw * (cin / bk);
  double best = 1e300;
  for (int cbn = 64; cbn <= 128; cbn *= 2) {
    if (force_bn && cbn != force_bn) continue;
    if (!force_bn && cbn > 64 && cbn / 2 >= cout) continue;       // do not pad Cout by more than 2x
    for (int cmt = 1; cmt <= 2; ++cmt) {
      if (force_mt && cmt != force_mt) continue;
      const bool cwide = cmt * cbn > 128;
      if (cwide && !wide_ok) continue;
      const int rows_tile = BM * cmt;
      const double tiles = static_cast<double>((m_total + rows_tile - 1) / rows_tile) * ((cout + cbn - 1) / cbn);
      const double rounds = static_cast<double>((static_cast<long long>(tiles) + sms - 1) / sms);
      const double kb_ns = (im2col_cost ? kKbNsIm2col : kKbNsTiled) + (cmt * BM + cbn) * bk * 2.0 / kFeedBytesPerNs;
      const double main_ns = num_kb * kb_ns;
      const double outs = static_cast<double>(rows_tile) * cbn;
      const double tile_ns = cwide ? main_ns + outs * kWideEpiNsPerOut : (main_ns > outs * kEpiNsPerOut ? main_ns : outs * kEpiNsPerOut);
      double t = rounds * tile_ns;
      int csk = 0;
      if (sk_possible) {
        // stream-K: every SM gets units/SMs K-blocks, plus one partial dump / collect
        const double units = tiles * num_kb;
        const double per_cta = static_cast<double>((static_cast<long long>(units) + sms - 1) / sms);
        const double tsk = per_cta * kb_ns + (cwide ? kSkNsWide : kSkNs);
        // stream-K only spreads layers that leave most of the GPU idle (single images, small batches).  On layers that fill
        // the chip it changes the fp32 summation order of most outputs, which the fp16 activations of the next layers turn
        // into a head-feature difference of ~1.2e-3 (max|d| / max|y|) at C2.
        const bool ok = per_cta >= 4.0 && num_kb >= 2;
        const bool idle = tiles <= sms / 2;
        if (ok && (sk_force || (idle && tsk < 0.93 * t))) { t = tsk; csk = 1; }
      }
      if (sk_force && !csk) continue;
      // ties go to the wider-N shape (more reuse of each A tile)
      if (t < best * 0.9999 || (t <= best * 1.0001 && cbn > c.bn)) { best = t; c.bn = cbn; c.mt = cmt; c.streamk = csk; }
    }
  }
  if (c.bn == 0) { c.bn = force_bn ? force_bn : 128; c.mt = force_mt ? force_mt : 1; c.streamk = 0; }
  YB_REQUIRE((c.bn == 64 || c.bn == 128) && (c.mt == 1 || c.mt == 2) && (c.mt * c.bn <= 128 || wide_ok), "conv: tile %d x %d", c.bn, c.mt);
  c.kernel = c.mt * c.bn > 128 ? kKernelWide : kKernelIgemm;
  c.bk = bk;
  if (pool && c.kernel != kKernelWide)
    return fail(YB_ERR_UNSUPPORTED, "conv: the fused 2x2 max-pool runs on the 256 x 128 two-consumer tile only; this launch takes %d x %d tiles",
                BM * c.mt, c.bn);
  c.pool = pool;
  if (chain && c.kernel != kKernelWide)
    return fail(YB_ERR_UNSUPPORTED, "conv: the chained form runs on the 256 x 128 two-consumer tile only; this launch takes %d x %d tiles",
                BM * c.mt, c.bn);
  c.chain = chain;
  const long long tiles = ((m_total + BM * c.mt - 1) / (BM * c.mt)) * ((cout + c.bn - 1) / c.bn);
  c.grid = c.streamk ? sms : static_cast<int>(tiles < sms ? tiles : sms);      // sk_base / sk_rem are computed for exactly sms CTAs
  *out = c;
  return 0;
}

// The general geometry accepted by yb_conv2d_bn_act_fwd / yb_conv2d_choice; writes the output dims.
static int conv_geometry(int in_h, int in_w, int kh, int kw, int stride, int pad_h, int pad_w, int* out_h, int* out_w) {
  YB_REQUIRE(kh >= 1 && kh <= 7 && kw >= 1 && kw <= 7, "conv2d: kernel %d x %d (1..7 on each axis)", kh, kw);
  YB_REQUIRE(stride == 1 || stride == 2, "conv2d: stride %d (1 or 2)", stride);
  YB_REQUIRE(pad_h >= 0 && pad_h < kh && pad_w >= 0 && pad_w < kw, "conv2d: padding (%d, %d) for a %d x %d kernel (0 <= pad < k)", pad_h, pad_w, kh,
             kw);
  YB_REQUIRE(in_h > 0 && in_w > 0 && in_h + 2 * pad_h >= kh && in_w + 2 * pad_w >= kw, "conv2d: %d x %d input gives an empty output", in_h, in_w);
  *out_h = (in_h + 2 * pad_h - kh) / stride + 1;
  *out_w = (in_w + 2 * pad_w - kw) / stride + 1;
  return 0;
}

// out = {kernel (kKernel*), BK, BLOCK_N, rows per CTA tile, stream-K, grid} of a yb_conv2d_bn_act_fwd launch
int conv2d_choice(int batch, int in_h, int in_w, int cin, int cout, int kh, int kw, int stride, int pad_h, int pad_w, int out_mode, int flags,
                  int with_workspace, int* out) {
  YB_REQUIRE(out != nullptr && batch > 0 && cin > 0 && cin % 32 == 0 && cout > 0, "conv_choice: bad shape");
  int oh = 0, ow = 0;
  int rc = conv_geometry(in_h, in_w, kh, kw, stride, pad_h, pad_w, &oh, &ow);
  if (rc) return rc;
  ConvChoice c;
  rc = conv_choose(batch, oh, ow, cin, cout, kh, kw, stride, pad_h, pad_w, cin, out_mode, flags, with_workspace != 0, false, false, false, &c);
  if (rc) return rc;
  out[0] = c.kernel; out[1] = c.bk; out[2] = c.bn; out[3] = c.kernel == kKernelC32 ? C32Cfg::TH * C32Cfg::TW : BM * c.mt;
  out[4] = c.streamk; out[5] = c.grid;
  return 0;
}

// the same for a yb_conv_bn_act_fwd(_ws) launch: k x k, stride 1, pad (k-1)/2
int conv_choice(int batch, int height, int width, int cin, int cout, int ksize, int out_mode, int flags, int with_workspace, int* out) {
  YB_REQUIRE(out != nullptr && batch > 0 && height > 0 && width > 0 && cin % 32 == 0 && cout > 0 && (ksize == 1 || ksize == 3),
             "conv_choice: bad shape");
  return conv2d_choice(batch, height, width, cin, cout, ksize, ksize, 1, (ksize - 1) / 2, (ksize - 1) / 2, out_mode, flags, with_workspace, out);
}

// a_extent > 0: the A tensor maps cover only channels [0, a_extent) of each pixel; the TMA fills the rest of every K-block with
// zeros (yb_conv_bn_act_tail_fwd).  0: they cover a_channels.
static int conv2d_launch(const void* x, const void* w, const float* scale, const float* shift, float slope, void* y, int batch, int in_h, int in_w,
                         int cin, int cout, int kh, int kw, int stride, int pad_h, int pad_w, int x_ld, long long y_ld, int y_ch_off, int out_mode,
                         int flags, void* workspace, long long workspace_bytes, double* stats, int a_channels, int lo_ch_off,
                         const float* pre_scale, const float* pre_shift, int pre_relu, const ConvChain* chain, int a_extent, cudaStream_t stream) {
  YB_REQUIRE(x && w && scale && shift && y, "conv: null pointer");
  // the chained form: y is the second unit's output, Cout2 channels at y_ch_off
  if (chain != nullptr) flags |= kFlagChain;
  YB_REQUIRE(chain != nullptr || !(flags & kFlagChain), "conv: YB_CONV_CHAIN1X1 needs the second unit (yb_conv_bn_act_chain_fwd)");
  if (chain != nullptr) {
    YB_REQUIRE(chain->w && chain->scale && chain->shift && (reinterpret_cast<uintptr_t>(chain->w) & 15) == 0,
               "conv chain: null or misaligned second-unit operand");
    YB_REQUIRE(chain->cout > 0 && chain->cout <= kChainN && chain->cout % 8 == 0, "conv chain: the second unit's Cout=%d (8 .. %d, multiple of 8)",
               chain->cout, kChainN);
  }
  const int y_cout = chain != nullptr ? chain->cout : cout;
  YB_REQUIRE(batch > 0, "conv: bad shape");
  int height = 0, width = 0;      // output dims
  int rc = conv_geometry(in_h, in_w, kh, kw, stride, pad_h, pad_w, &height, &width);
  if (rc) return rc;
  const bool plain_1x1 = kh == 1 && kw == 1 && stride == 1;
  // pre-activation form (pre_scale != NULL): 1x1, plain fp16 operands; fused statistics are the training form (yb_conv1x1_preact_stats_fwd)
  const bool pre = pre_scale != nullptr;
  if (pre) {
    YB_REQUIRE(pre_shift != nullptr && (pre_relu == 0 || pre_relu == 1), "conv_preact: pre_shift must be given, pre_relu 0 or 1");
    YB_REQUIRE(plain_1x1, "conv_preact: k=%d x %d, stride %d: the pre-activation form is 1x1 stride 1 only", kh, kw, stride);
    YB_REQUIRE(a_channels <= 0 || a_channels == cin, "conv_preact: split-precision operands are not supported");
    YB_REQUIRE(lo_ch_off < 0, "conv_preact: no residual output");
    YB_REQUIRE(cin <= kPreMaxCh, "conv_preact: Cin=%d exceeds the %d-channel pre-activation table", cin, kPreMaxCh);
  }
  const PreAct pre_act{pre_scale, pre_shift, pre_relu};
  // split-precision operands (see ConvParams::a_wrap): cin is the concatenated reduction width, a_channels what x really holds
  if (a_channels <= 0) a_channels = cin;
  YB_REQUIRE(a_channels <= cin && a_channels % 32 == 0 && cin - a_channels <= a_channels, "conv: a_channels=%d does not fit cin=%d", a_channels, cin);
  YB_REQUIRE(lo_ch_off < 0 || (out_mode == 0 && stats == nullptr && lo_ch_off % 8 == 0 && lo_ch_off >= y_ch_off + cout && lo_ch_off + cout <= y_ld),
             "conv: lo_ch_off=%d (needs fp16 NHWC output with room for a second Cout-wide slice)", lo_ch_off);
  YB_REQUIRE(stats == nullptr || out_mode == 0, "conv: fused statistics need the fp16 NHWC output");
  YB_REQUIRE(cin > 0 && cin % 32 == 0, "conv: Cin=%d must be a multiple of 32 (layer 0 uses yb_conv0_*)", cin);
  const int a_ext = a_extent > 0 ? a_extent : a_channels;
  YB_REQUIRE(x_ld >= a_ext && x_ld % 8 == 0, "conv: x_ld=%d", x_ld);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0, "conv: x/w must be 16B aligned");
  YB_REQUIRE(out_mode == 0 || out_mode == 1, "conv: out_mode");
  if (out_mode == 0) {
    YB_REQUIRE(y_cout % 8 == 0 && y_ld % 8 == 0 && y_ch_off % 8 == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0,
               "conv: fp16 NHWC output needs Cout, y_ld, y_ch_off multiples of 8 and a 16B aligned pointer");
  }
  const long long m_total_ll = static_cast<long long>(batch) * height * width;
  YB_REQUIRE(m_total_ll < (1ll << 31) - kWideRows && static_cast<long long>(batch) * in_h * in_w < (1ll << 31), "conv: too many pixels");
  // stream-K needs the caller's workspace (one per stream: partial sums + flags)
  const bool ws_ok = workspace != nullptr && workspace_bytes >= conv_workspace_bytes() && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0;
  ConvChoice ch;
  rc = conv_choose(batch, height, width, cin, cout, kh, kw, stride, pad_h, pad_w, a_channels, out_mode, flags, ws_ok, stats != nullptr, lo_ch_off >= 0,
                   pre, &ch);
  if (rc) return rc;
  YB_REQUIRE(!pre || ch.kernel == kKernelIgemm, "conv_preact: no pre-activation form of kernel %d", ch.kernel);
  if (ch.kernel == kKernelC32)
    return conv_c32_forward(x, w, scale, shift, slope, y, batch, height, width, cout, x_ld, y_ld, y_ch_off, (flags >> 4) & 1, flags, stats, stream);
  const int bk = ch.bk, bn = ch.bn, mt = ch.mt, streamk = ch.streamk;
  // 1x1 stride-1 layers read A as a plain [pixels, Cin] matrix (2-D tiled TMA: cheaper per instruction than im2col mode);
  // YB_CONV_1X1_IM2COL=1 switches back for A/B runs
  static const int k1x1_im2col = getenv("YB_CONV_1X1_IM2COL") ? atoi(getenv("YB_CONV_1X1_IM2COL")) : 0;
  const int a_im2col = !plain_1x1 ? 1 : ((k1x1_im2col && !(flags & 1) && !pre) ? 1 : 0);

  EncodeTiledFn enc_tiled;
  EncodeIm2colFn enc_im2col;
  rc = get_encoders(&enc_tiled, &enc_im2col);
  if (rc) return rc;

  // the pooled form enumerates pool windows: M, H and W are the pooled output's, and each window position is a stride-2 conv
  // (conv_wide_pool_kernel), so the producer's window corners are 2 i - 1, 2 j - 1 plus the position
  const bool pooled = ch.pool != 0;
  if (pooled) { height /= 2; width /= 2; }
  ConvParams p;
  p.m_total = static_cast<int>(static_cast<long long>(batch) * height * width);
  p.height = height; p.width = width; p.cin = cin; p.cout = cout;
  p.kh = kh; p.kw = kw; p.pad_h = pad_h; p.pad_w = pad_w; p.stride = pooled ? 2 : stride; p.in_h = in_h; p.in_w = in_w;
  p.kb_per_tap = cin / bk;
  p.num_kb = kh * kw * p.kb_per_tap;
  const int rows_tile = pooled ? kWidePoolRows : BM * mt;
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
  p.scale2 = chain ? chain->scale : nullptr; p.shift2 = chain ? chain->shift : nullptr;
  p.slope2 = chain ? chain->slope : 0.f; p.cout2 = chain ? chain->cout : 0;
  if (streamk) {
    const long long units = static_cast<long long>(p.m_tiles) * p.n_tiles * p.num_kb;
    YB_REQUIRE(units < (1ll << 31), "conv: stream-K unit count overflows");
    p.sk_base = static_cast<int>(units / sm_count());
    p.sk_rem = static_cast<int>(units % sm_count());
    p.flags = static_cast<unsigned*>(workspace);
    p.ws = reinterpret_cast<float*>(static_cast<char*>(workspace) + kSkFlagBytes);
  }

  const CUtensorMapSwizzle swz = (bk == 64) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  alignas(64) CUtensorMap ta_pos[4];   // ta_pos[0] is the A map; the pooled form has one per window position
  alignas(64) CUtensorMap tb;
  CUtensorMap& ta = ta_pos[0];
  CUresult cr;
  const int a_rows = pooled ? kWidePoolRows : BM * mt;     // pixels per A box (ConvCfg::kMergedA)
  if (a_im2col) {
    // the input tensor; the bounding box of window corners is [-pad, in + pad - k] on each axis, walked with the conv's stride, so
    // consecutive box pixels are consecutive output pixels (row-major, then the next image).  Pooled, position (dy, dx): corners
    // [d - 1, in + d - 3] walked with stride 2, one per pool window
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(a_ext), static_cast<cuuint64_t>(in_w), static_cast<cuuint64_t>(in_h),
                                static_cast<cuuint64_t>(batch)};
    const cuuint64_t strides[3] = {static_cast<cuuint64_t>(x_ld) * 2, static_cast<cuuint64_t>(x_ld) * 2 * in_w,
                                   static_cast<cuuint64_t>(x_ld) * 2 * in_w * in_h};
    const cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(p.stride), static_cast<cuuint32_t>(p.stride), 1};
    int drv = 0;
    cudaDriverGetVersion(&drv);
    for (int b = 0; b < (pooled ? 4 : 1); ++b) {
      const int dx = pooled ? (b & 1) : 0, dy = pooled ? (b >> 1) : 0;
      const int lower[2] = {dx - pad_w, dy - pad_h};                    // {W, H}
      const int upper[2] = {dx + pad_w - (kw - 1) - (pooled ? 1 : 0), dy + pad_h - (kh - 1) - (pooled ? 1 : 0)};
      cr = enc_im2col(&ta_pos[b], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(x), dims, strides, lower, upper,
                      static_cast<cuuint32_t>(bk), static_cast<cuuint32_t>(a_rows), estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeIm2col failed (%d)", static_cast<int>(cr));
      // Driver workaround (same one CUTLASS carries, cute/atom/copy_traits_sm90_im2col.hpp): for
      // tensors smaller than 128 KiB drivers <= 13.1 set a descriptor bit that breaks im2col loads.
      const unsigned long long span_bytes = static_cast<unsigned long long>(x_ld) * 2ull * in_w * in_h * batch;
      if (drv <= 13010 && span_bytes < 131072ull) reinterpret_cast<uint64_t*>(&ta_pos[b])[1] &= ~(1ull << 21);
    }
  } else {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(a_ext), static_cast<cuuint64_t>(p.m_total)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(x_ld) * 2};
    const cuuint32_t box[2] = {static_cast<cuuint32_t>(bk), static_cast<cuuint32_t>(a_rows)};
    const cuuint32_t estr[2] = {1, 1};
    cr = enc_tiled(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(x), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeTiled(A) failed (%d)", static_cast<int>(cr));
  }
  {
    const cuuint64_t k_total = static_cast<cuuint64_t>(kh) * kw * cin;
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
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(y_cout), static_cast<cuuint64_t>(p.m_total)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(y_ld) * 2};
    const cuuint32_t box[2] = {64, 32};                 // one epilogue warp's rows
    const cuuint32_t estr[2] = {1, 1};
    cr = enc_tiled(&ty, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, static_cast<__half*>(y) + y_ch_off, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeTiled(Y) failed (%d)", static_cast<int>(cr));
  }
  if (ch.chain) {
    // the second unit's weight [Cout2][Cin2 = 128] as two 64-channel K-blocks of 64 rows (rows >= Cout2 zero-filled)
    alignas(64) CUtensorMap tw2;
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cout), static_cast<cuuint64_t>(chain->cout)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(cout) * 2};
    const cuuint32_t box[2] = {64, static_cast<cuuint32_t>(kChainN)};
    const cuuint32_t estr[2] = {1, 1};
    cr = enc_tiled(&tw2, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(chain->w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(YB_ERR_DRIVER, "cuTensorMapEncodeTiled(W2) failed (%d)", static_cast<int>(cr));
    return launch_wide_chain(ta, tb, ty, tw2, p, ch.grid, stream);
  }
  if (pooled) return bk == 64 ? launch_wide_pool<64>(ta_pos, tb, ty, p, ch.grid, stream) : launch_wide_pool<32>(ta_pos, tb, ty, p, ch.grid, stream);
  if (bk == 64) return dispatch_conv<64>(bn, mt, ch.grid, ta, tb, ty, p, pre ? &pre_act : nullptr, stream);
  return dispatch_conv<32>(bn, mt, ch.grid, ta, tb, ty, p, pre ? &pre_act : nullptr, stream);
}

int conv2d_forward(const void* x, const void* w, const float* scale, const float* shift, float slope, void* y, int batch, int in_h, int in_w,
                   int cin, int cout, int kh, int kw, int stride, int pad_h, int pad_w, int x_ld, long long y_ld, int y_ch_off, int out_mode,
                   int flags, void* workspace, long long workspace_bytes, double* stats, int a_channels, int lo_ch_off,
                   const float* pre_scale, const float* pre_shift, int pre_relu, const ConvChain* chain, cudaStream_t stream) {
  return conv2d_launch(x, w, scale, shift, slope, y, batch, in_h, in_w, cin, cout, kh, kw, stride, pad_h, pad_w, x_ld, y_ld, y_ch_off, out_mode, flags,
                       workspace, workspace_bytes, stats, a_channels, lo_ch_off, pre_scale, pre_shift, pre_relu, chain, 0, stream);
}

// k x k, stride 1, pad (k-1)/2 with cin % 8 == 0 (yb_conv_bn_act_tail_fwd).  The GEMM runs over cin_pad = round_up(cin, 32) channels per
// tap -- the K-blocks of the plain conv on a zero-padded operand -- while the A maps cover channels [0, cin) only, so the TMA zero-fills
// [cin, cin_pad) of each tap's last K-block and never reads x past channel cin.  w holds zeros there.  The TMA still delivers whole boxes,
// so every stage's transaction byte count is the plain conv's.  No stream-K, fused pool, chained 1x1 or Cin = 32 halo-tile form.
int conv_tail_forward(const void* x, const void* w, const float* scale, const float* shift, float slope, void* y, int batch, int height,
                      int width, int cin, int cin_pad, int cout, int ksize, int x_ld, long long y_ld, int y_ch_off, int out_mode, int flags,
                      cudaStream_t stream) {
  YB_REQUIRE(ksize == 1 || ksize == 3, "conv tail: ksize %d unsupported (1 or 3)", ksize);
  YB_REQUIRE(cin > 0 && cin % 8 == 0, "conv tail: Cin=%d must be a positive multiple of 8", cin);
  YB_REQUIRE(cin_pad == (cin + 31) / 32 * 32, "conv tail: cin_pad=%d must be round_up(Cin=%d, 32)", cin_pad, cin);
  YB_REQUIRE(x_ld >= cin && x_ld % 8 == 0, "conv tail: x_ld=%d (needs x_ld >= Cin=%d, multiple of 8)", x_ld, cin);
  if (flags & ((1 << 4) | kFlagChain | (1 << 30)))
    return fail(YB_ERR_UNSUPPORTED, "conv tail: no fused pool, chained 1x1 or stream-K form (flags 0x%x)", flags);
  flags |= 1 << 28;      // YB_CONV_NO_SMALLK: never the Cin = 32 halo-tile kernel
  return conv2d_launch(x, w, scale, shift, slope, y, batch, height, width, cin_pad, cout, ksize, ksize, 1, (ksize - 1) / 2, (ksize - 1) / 2, x_ld,
                       y_ld, y_ch_off, out_mode, flags, nullptr, 0, nullptr, 0, -1, nullptr, nullptr, 0, nullptr, cin, stream);
}

// k x k, stride 1, pad (k-1)/2: yb_conv_bn_act_fwd(_ws) and its statistics, split and pre-activation forms
int conv_igemm_forward(const void* x, const void* w, const float* scale, const float* shift, float slope, void* y, int batch,
                       int height, int width, int cin, int cout, int ksize, int x_ld, long long y_ld, int y_ch_off, int out_mode,
                       int flags, void* workspace, long long workspace_bytes, double* stats, int a_channels, int lo_ch_off,
                       const float* pre_scale, const float* pre_shift, int pre_relu, cudaStream_t stream) {
  YB_REQUIRE(ksize == 1 || ksize == 3, "conv: ksize %d unsupported (1 or 3)", ksize);
  return conv2d_forward(x, w, scale, shift, slope, y, batch, height, width, cin, cout, ksize, ksize, 1, (ksize - 1) / 2, (ksize - 1) / 2, x_ld, y_ld,
                        y_ch_off, out_mode, flags, workspace, workspace_bytes, stats, a_channels, lo_ch_off, pre_scale, pre_shift, pre_relu, nullptr,
                        stream);
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
  for (int r = 0; r < p.kh; ++r) {
    const int hi = h * p.stride + r - p.pad_h;
    if (hi < 0 || hi >= p.in_h) continue;
    for (int s = 0; s < p.kw; ++s) {
      const int wi = wq * p.stride + s - p.pad_w;
      if (wi < 0 || wi >= p.in_w) continue;
      const __half* xp = x + ((static_cast<long long>(img) * p.in_h + hi) * p.in_w + wi) * x_ld;
      const __half* wp = w + (static_cast<long long>(co) * p.kh * p.kw + r * p.kw + s) * p.cin;
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
  p.height = height; p.width = width; p.cin = cin; p.cout = cout;
  p.kh = ksize; p.kw = ksize; p.pad_h = (ksize - 1) / 2; p.pad_w = (ksize - 1) / 2; p.stride = 1; p.in_h = height; p.in_w = width;
  p.scale = scale; p.shift = shift; p.slope = slope; p.y = y; p.y_ld = y_ld; p.y_ch_off = y_ch_off; p.out_mode = out_mode;
  p.hw = height * width;
  const long long total = static_cast<long long>(p.m_total) * cout;
  conv_ref_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __half*>(x),
                                                                                  reinterpret_cast<const __half*>(w), p, x_ld);
  return check_launch("conv_ref_kernel");
}

}  // namespace yb
