// Implicit-GEMM convolution on Hopper wgmma tensor cores (sm_90a).
//
//   out[pixel, co] = sum_{tap, ci} A[pixel + tap, ci] * W[tap, co, ci]  (+ fused 1x1 operand)
//                    + bias (+ bias2) (+ residual)
//
//   * M tile = 128 output pixels = a (TW x TH x TB) box of the NHWC tensor; N tile = BN couts (64 or 128);
//     K block = 64 input channels of one filter tap.
//   * Channel counts are multiples of 32.  A K block that runs past Cin (Cin2) reads zeros: the TMA zero-fills the
//     activation and weight boxes past the end of their channel dimension.  The last N block may run 32 or 96 couts
//     past Cout; an epilogue slice (BN / 4 columns: 16 or 32) then lies wholly inside or wholly past Cout, and the
//     slices past it are skipped.
//   * Operands are split planes (hi, lo) in bf16 or fp16.  passes=3 issues A_lo.W_hi + A_hi.W_lo + A_hi.W_hi
//     into the same accumulator (fp32-class accuracy); passes=1 issues A_hi.W_hi only.
//   * TMA (cp.async.bulk.tensor, 4-D tiled map, SWIZZLE_128B) stages the shifted pixel box of a
//     tap straight from the activation tensor; out-of-image coordinates are zero-filled by the
//     TMA unit, which IS the conv padding -- no im2col buffer, no halo logic.
//   * Warp-specialised persistent CTA: warps 0-7 = two consumer warpgroups (wgmma m64nBNk16 on rows
//     0-63 / 64-127 of the tile, register accumulators, epilogue straight from the fragment), warps 8-11 =
//     producer warpgroup whose first lane feeds a STAGES-deep shared-memory ring with TMA.  384 threads cap
//     every thread at 168 registers, so the producer warpgroup gives registers to the consumers (setmaxnreg).
//   * Software-pipelined epilogue: a finished tile's promoted accumulator stays in registers while the
//     next tile's first chunk runs; after each of that chunk's K blocks is issued, the consumers run one
//     slice (a group of columns) of the finished tile's epilogue, so it overlaps the tensor core.  Each
//     element's arithmetic is the same as in a serial epilogue.
//   * fp32-faithful accumulation: the tensor core's accumulator add truncates (round-toward-zero),
//     so a K = 9216 chain accumulated entirely inside wgmma drifts by ~3e-5.  The K loop is therefore
//     cut into chunks of `kb_per_chunk` K-blocks; each chunk starts from a zero wgmma accumulator and is
//     added into a second fp32 register accumulator with round-to-nearest.
//   * Every mbarrier wait has a clock-based watchdog: on expiry a device fault word is set and
//     the CTA drains without deadlocking the GPU (bbdm_check_device_fault reports it).
#include "tc_common.cuh"
#include <stdlib.h>

namespace bbdm {

constexpr int UM_BM = 128;       // pixels per tile (two m64 warpgroups)
constexpr int UM_BK = 64;        // K block: 64 input channels of one tap = one 128-byte SWIZZLE_128B row
constexpr int UM_THREADS = 384;  // 2 consumer warpgroups + 1 producer warpgroup
// register split (65,536 per SM): 128 x 40 for the producer warpgroup + 256 x 232 for the consumers
constexpr int UM_PRODUCER_REGS = 40, UM_CONSUMER_REGS = 232;
static_assert(128 * UM_PRODUCER_REGS + 256 * UM_CONSUMER_REGS <= 65536, "conv_umma: register split");
constexpr int UM_SLICES = 4;     // epilogue slices per tile, each BN / 32 column blocks of 8

struct ConvParams {
  int B, H, W, Cout;
  int TW, TH, TB, tiles_w, tiles_h, tiles_b, n_tiles;
  int kb_per_tap;   // ceil(Cin / 64)
  int K1;           // taps * kb_per_tap
  int K2;           // ceil(Cin2 / 64)
  int taps;
  int up2;           // 1: fused nearest-2x upsample (4 output phases x 2x2 taps on the low-res input)
  int origin;        // taps == 4: first row / column of the 2x2 window (0 or -1)
  int w_per_image;   // 1: the weight "tap" index is the image index of the tile (36 Winograd position GEMMs in one launch)
  int kb_per_chunk;  // K blocks accumulated inside wgmma before promotion to the fp32 register accumulator
  const float* bias; const float* bias2;
  const float* residual; int res_mode;
  float* out; __nv_bfloat16* out_hi; __nv_bfloat16* out_lo;
  int out_nchw_c;    // > 0: out is NCHW with this many channels (UNet head)
  float* stats;      // fused GroupNorm partial sums (see BbdmConvArgs.stats_partial) or nullptr
  unsigned long long* fault;
};

template <int BN>
struct UmmaCfg {
  static constexpr uint32_t A_BYTES = UM_BM * UM_BK * 2;     // per plane per stage
  static constexpr uint32_t W_BYTES = BN * UM_BK * 2;
  static constexpr uint32_t STAGE3 = 2 * A_BYTES + 2 * W_BYTES;  // hi+lo planes
  static constexpr uint32_t STAGE1 = A_BYTES + W_BYTES;
  static constexpr uint32_t SMEM_BUDGET = 200 * 1024;
  static constexpr int STAGES3 = (SMEM_BUDGET / STAGE3) > 6 ? 6 : (SMEM_BUDGET / STAGE3);
  static constexpr int STAGES1 = (SMEM_BUDGET / STAGE1) > 8 ? 8 : (SMEM_BUDGET / STAGE1);
};

template <int BN, bool F16>
__device__ __forceinline__ void conv_mma(float* d, uint64_t da, uint64_t db) {
  if (F16) {
    if (BN == 128) wgmma_n128_f16<0>(d, da, db, 1u); else wgmma_n64_f16<0>(d, da, db, 1u);
  } else {
    if (BN == 128) wgmma_n128_bf16<0>(d, da, db, 1u); else wgmma_n64_bf16<0>(d, da, db, 1u);
  }
}

// ---- tile epilogue: bias / fused-skip bias / residual / store, straight from the fragment ----------------
// Where a consumer thread's two fragment rows (ri = 0, 1) of a tile land; computed once per tile, kept while
// the epilogue's slices run.
struct EpiTile {
  int nb, tw, th, tb, phase;
  int bb[2], hh[2], ww[2];
  bool valid[2];
  int64_t pix[2];
};

__device__ __forceinline__ EpiTile epi_tile(const ConvParams& p, int tile, int n_blocks, int warp, int lane) {
  EpiTile e;
  e.nb = tile % n_blocks;
  int mt = tile / n_blocks;
  e.phase = 0;
  if (p.up2) { e.phase = mt & 3; mt >>= 2; }
  e.tw = mt % p.tiles_w; mt /= p.tiles_w;
  e.th = mt % p.tiles_h;
  e.tb = mt / p.tiles_h;
  const int OH = p.up2 ? 2 * p.H : p.H, OW = p.up2 ? 2 * p.W : p.W;
#pragma unroll
  for (int ri = 0; ri < 2; ++ri) {
    const int row = 16 * warp + (lane >> 2) + 8 * ri;        // tile row (warp 0-7 -> rows 0-127)
    const int ws = e.tw * p.TW + row % p.TW;                  // coordinates in the conv INPUT grid
    const int hs = e.th * p.TH + (row / p.TW) % p.TH;
    e.bb[ri] = e.tb * p.TB + row / (p.TW * p.TH);
    e.valid[ri] = ws < p.W && hs < p.H && e.bb[ri] < p.B;
    e.hh[ri] = p.up2 ? 2 * hs + (e.phase >> 1) : hs;         // output grid (fused upsample: 2x with phase offset)
    e.ww[ri] = p.up2 ? 2 * ws + (e.phase & 1) : ws;
    e.pix[ri] = ((int64_t)e.bb[ri] * OH + e.hh[ri]) * OW + e.ww[ri];
  }
  return e;
}

// Slice s of the epilogue: column blocks jj = JS*s .. JS*s + JS-1 (8 columns each) of both fragment rows.
// Every bias and residual load of the slice is issued before its first store; each element's residual is
// read by the thread that writes that element, so out == residual works.  With fused GroupNorm statistics,
// the slice's per-warp column (sum, sum sq) go to stats_s (sum order: row ri 0, ri 1, lanes xor 4/8/16).
template <int BN>
__device__ __forceinline__ void epi_slice(const ConvParams& p, const float* racc, EpiTile e, int s, int warp,
                                          int lane, float (*stats_s)[BN][2]) {
  constexpr int JS = BN / 8 / UM_SLICES;
  if (e.nb * BN + s * (BN / UM_SLICES) >= p.Cout) return;   // past the last cout (warp-uniform)
  // opaque tile coordinates: otherwise the compiler hoists every slice's address arithmetic out of the K loop the
  // slice runs in, and those addresses would occupy registers (and spill) for the whole loop
  asm volatile("" : "+r"(e.nb), "+r"(e.bb[0]), "+r"(e.bb[1]), "+r"(e.hh[0]), "+r"(e.hh[1]), "+r"(e.ww[0]),
               "+r"(e.ww[1]), "+l"(e.pix[0]), "+l"(e.pix[1]));
  const int OH = p.up2 ? 2 * p.H : p.H, OW = p.up2 ? 2 * p.W : p.W;
  const int n0 = e.nb * BN + 2 * (lane & 3);
  // bias terms first, then the residual: the same per-element order of adds as a serial epilogue, with the
  // residual mode branched on once per slice so that all of its loads can be in flight together
  float2 v[2][JS];
#pragma unroll
  for (int ri = 0; ri < 2; ++ri) {
#pragma unroll
    for (int j = 0; j < JS; ++j) {
      const int jj = JS * s + j;
      const int nc = n0 + 8 * jj;
      v[ri][j] = make_float2(racc[4 * jj + 2 * ri], racc[4 * jj + 2 * ri + 1]);
      if (p.bias) { const float2 b = *reinterpret_cast<const float2*>(p.bias + nc); v[ri][j].x += b.x; v[ri][j].y += b.y; }
      if (p.bias2) { const float2 b = *reinterpret_cast<const float2*>(p.bias2 + nc); v[ri][j].x += b.x; v[ri][j].y += b.y; }
    }
  }
  if (p.res_mode == BBDM_RES_SAME || p.res_mode == BBDM_RES_UP2) {
#pragma unroll
    for (int ri = 0; ri < 2; ++ri) {
      if (!e.valid[ri]) continue;
      const int64_t rpix = p.res_mode == BBDM_RES_SAME
                               ? e.pix[ri]
                               : ((int64_t)e.bb[ri] * (OH >> 1) + (e.hh[ri] >> 1)) * (OW >> 1) + (e.ww[ri] >> 1);
      const float* rp = p.residual + rpix * p.Cout + n0 + 8 * JS * s;
#pragma unroll
      for (int j = 0; j < JS; ++j) {
        const float2 t = *reinterpret_cast<const float2*>(rp + 8 * j);
        v[ri][j].x += t.x; v[ri][j].y += t.y;
      }
    }
  } else if (p.res_mode == BBDM_RES_DOWN2) {
    const int64_t W2 = (int64_t)OW * 2;
#pragma unroll
    for (int ri = 0; ri < 2; ++ri) {
      if (!e.valid[ri]) continue;
      const float* rp0 = p.residual + (((int64_t)e.bb[ri] * OH * 2 + e.hh[ri] * 2) * W2 + e.ww[ri] * 2) * p.Cout +
                         n0 + 8 * JS * s;
#pragma unroll
      for (int j = 0; j < JS; ++j) {
        const float* rp = rp0 + 8 * j;
        const float2 t0 = *reinterpret_cast<const float2*>(rp), t1 = *reinterpret_cast<const float2*>(rp + p.Cout);
        const float2 t2 = *reinterpret_cast<const float2*>(rp + W2 * p.Cout);
        const float2 t3 = *reinterpret_cast<const float2*>(rp + (W2 + 1) * p.Cout);
        v[ri][j].x += 0.25f * (((t0.x + t1.x) + t2.x) + t3.x);
        v[ri][j].y += 0.25f * (((t0.y + t1.y) + t2.y) + t3.y);
      }
    }
  }
  float ssum[2 * JS], ssq[2 * JS];           // per (column block, parity): sums over this thread's 2 rows
#pragma unroll
  for (int j = 0; j < 2 * JS; ++j) { ssum[j] = 0.f; ssq[j] = 0.f; }
#pragma unroll
  for (int ri = 0; ri < 2; ++ri) {
    if (!e.valid[ri]) continue;
    const int bb = e.bb[ri], hh = e.hh[ri], ww = e.ww[ri];
    const int64_t pix = e.pix[ri];
#pragma unroll
    for (int j = 0; j < JS; ++j) {
      const int nc = n0 + 8 * (JS * s + j);
      const float2 w = v[ri][j];
      if (p.out_nchw_c > 0) {
        // head: first out_nchw_c couts straight into the NCHW result
        if (nc < p.out_nchw_c) p.out[(((int64_t)bb * p.out_nchw_c + nc) * OH + hh) * OW + ww] = w.x;
        if (nc + 1 < p.out_nchw_c) p.out[(((int64_t)bb * p.out_nchw_c + nc + 1) * OH + hh) * OW + ww] = w.y;
      } else if (p.out) {
        *reinterpret_cast<float2*>(p.out + pix * p.Cout + nc) = w;
      }
      if (p.out_hi) {
        uint32_t h, l;
        split2x(w.x, w.y, h, l);
        *reinterpret_cast<uint32_t*>(p.out_hi + pix * p.Cout + nc) = h;
        *reinterpret_cast<uint32_t*>(p.out_lo + pix * p.Cout + nc) = l;
      }
      ssum[2 * j] += w.x; ssq[2 * j] += w.x * w.x;
      ssum[2 * j + 1] += w.y; ssq[2 * j + 1] += w.y * w.y;
    }
  }
  if (p.stats) {
    // rows of a warp: lanes with equal lane % 4 hold the same columns
#pragma unroll
    for (int j = 0; j < 2 * JS; ++j) {
#pragma unroll
      for (int off = 4; off < 32; off <<= 1) {
        ssum[j] += __shfl_xor_sync(0xffffffffu, ssum[j], off);
        ssq[j] += __shfl_xor_sync(0xffffffffu, ssq[j], off);
      }
    }
    if (lane < 4) {
#pragma unroll
      for (int j = 0; j < 2 * JS; ++j) {
        const int c = 8 * (JS * s + (j >> 1)) + 2 * lane + (j & 1);
        stats_s[warp][c][0] = ssum[j];
        stats_s[warp][c][1] = ssq[j];
      }
    }
  }
}

// After a tile's last slice: fused GroupNorm statistics of the tensor just written, per-channel (sum, sum sq)
// over each 32-row quarter of the tile (tile lies inside one image: TB == 1); a quarter is warps (2q, 2q + 1).
template <int BN>
__device__ __forceinline__ void epi_stats_out(const ConvParams& p, const EpiTile& e, float (*stats_s)[BN][2]) {
  if (!p.stats) return;
  asm volatile("bar.sync 1, 256;" ::: "memory");
  const int64_t tile_lin =
      (((int64_t)e.tb * p.tiles_w * p.tiles_h + e.th * p.tiles_w + e.tw) * (p.up2 ? 4 : 1) + e.phase) * 4;
  int i0 = threadIdx.x;
  asm volatile("" : "+r"(i0));   // keeps this loop's per-thread indices from being held across the tile loop
  for (int i = i0; i < 4 * BN; i += 256) {
    const int q = i / BN, c = i % BN;
    if (e.nb * BN + c >= p.Cout) continue;
    const float s = stats_s[2 * q][c][0] + stats_s[2 * q + 1][c][0];
    const float sq = stats_s[2 * q][c][1] + stats_s[2 * q + 1][c][1];
    *reinterpret_cast<float2*>(p.stats + ((tile_lin + q) * p.Cout + e.nb * BN + c) * 2) = make_float2(s, sq);
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

// slices s_begin .. s_end - 1 (s is a run-time index; each slice's register indices must be compile-time)
template <int BN>
__device__ __forceinline__ void epi_slices(const ConvParams& p, const float* racc, const EpiTile& e, int s_begin,
                                           int s_end, int warp, int lane, float (*stats_s)[BN][2]) {
#pragma unroll
  for (int s = 0; s < UM_SLICES; ++s)
    if (s >= s_begin && s < s_end) epi_slice<BN>(p, racc, e, s, warp, lane, stats_s);
}

template <int BN, int PASSES, bool F16>
__global__ void __launch_bounds__(UM_THREADS, 1)
conv_umma_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                 const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                 const __grid_constant__ CUtensorMap map_a2_hi, const __grid_constant__ CUtensorMap map_a2_lo,
                 const __grid_constant__ CUtensorMap map_w2_hi, const __grid_constant__ CUtensorMap map_w2_lo,
                 const ConvParams p) {
  using Cfg = UmmaCfg<BN>;
  constexpr int STAGES = PASSES == 3 ? Cfg::STAGES3 : Cfg::STAGES1;
  constexpr uint32_t STAGE_BYTES = PASSES == 3 ? Cfg::STAGE3 : Cfg::STAGE1;
  constexpr uint32_t OFF_ALO = Cfg::A_BYTES;
  constexpr uint32_t OFF_WHI = PASSES == 3 ? 2 * Cfg::A_BYTES : Cfg::A_BYTES;
  constexpr uint32_t OFF_WLO = OFF_WHI + Cfg::W_BYTES;
  constexpr int NR = BN / 2;                  // accumulator registers per thread
  static_assert(STAGES >= 2, "need at least a double buffer");

  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bars[2 * 8];
  __shared__ int abort_s;
  // fused GroupNorm statistics: per-warp column (sum, sum sq) over its 16 rows
  __shared__ __align__(16) float stats_s[8][BN][2];

  const uint32_t tiles_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar_full = smem_u32(&bars[0]);        // [STAGES]
  const uint32_t bar_empty = smem_u32(&bars[8]);       // [STAGES]
  volatile int* abort_flag = &abort_s;

  if (threadIdx.x == 0) {
    abort_s = 0;
    for (int i = 0; i < STAGES; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int n_blocks = (p.Cout + BN - 1) / BN;
  const int total_tiles = p.n_tiles * n_blocks * (p.up2 ? 4 : 1);
  const int KB = p.K1 + p.K2;

  if (warp >= 8) {
    // ================================ TMA producer ==========================================
    setmaxnreg_dec<UM_PRODUCER_REGS>();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase_bit = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nb = tile % n_blocks;
        int mt = tile / n_blocks;
        int phase = 0;
        if (p.up2) { phase = mt & 3; mt >>= 2; }
        const int tw = mt % p.tiles_w; mt /= p.tiles_w;
        const int th = mt % p.tiles_h;
        const int tb = mt / p.tiles_h;
        const int w0 = tw * p.TW, h0 = th * p.TH, b0 = tb * p.TB, n0 = nb * BN;
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(bar_empty + 8 * stage, phase_bit ^ 1, abort_flag, p.fault, 0xE0000000ull | (unsigned)kb);
          const uint32_t sbase = tiles_base + stage * STAGE_BYTES;
          const uint32_t full = bar_full + 8 * stage;
          mbar_expect_tx(full, STAGE_BYTES);
          if (kb < p.K1) {
            const int tap = kb / p.kb_per_tap, cb = kb - tap * p.kb_per_tap;
            int dy = 0, dx = 0, wtap = tap;
            if (p.up2) {
              // output phase (a, b) = (phase>>1, phase&1); 2x2 taps (r, c) on the low-res source
              const int r = tap >> 1, c = tap & 1;
              dy = (phase >> 1) ? r : r - 1;
              dx = (phase & 1) ? c : c - 1;
              wtap = phase * 4 + tap;
            } else if (p.taps == 9) { dy = tap / 3 - 1; dx = tap % 3 - 1; }
            else if (p.taps == 4) { dy = (tap >> 1) + p.origin; dx = (tap & 1) + p.origin; }   // 2x2 window at rows/cols
                                                                     // origin..origin+1: zero fill bottom/right (0) or top/left (-1)
            else if (p.w_per_image) wtap = tb;                       // taps == 1: weights of transform position tb
            tma_load_4d(sbase, &map_a_hi, full, cb * UM_BK, w0 + dx, h0 + dy, b0);
            if (PASSES == 3) tma_load_4d(sbase + OFF_ALO, &map_a_lo, full, cb * UM_BK, w0 + dx, h0 + dy, b0);
            tma_load_3d(sbase + OFF_WHI, &map_w_hi, full, cb * UM_BK, n0, wtap);
            if (PASSES == 3) tma_load_3d(sbase + OFF_WLO, &map_w_lo, full, cb * UM_BK, n0, wtap);
          } else {
            const int cb = kb - p.K1;
            tma_load_4d(sbase, &map_a2_hi, full, cb * UM_BK, w0, h0, b0);
            if (PASSES == 3) tma_load_4d(sbase + OFF_ALO, &map_a2_lo, full, cb * UM_BK, w0, h0, b0);
            tma_load_3d(sbase + OFF_WHI, &map_w2_hi, full, cb * UM_BK, n0, 0);
            if (PASSES == 3) tma_load_3d(sbase + OFF_WLO, &map_w2_lo, full, cb * UM_BK, n0, 0);
          }
          if (++stage == STAGES) { stage = 0; phase_bit ^= 1; }
        }
      }
    }
    return;
  }

  // ================================ consumer warpgroups: MMA + epilogue ========================
  setmaxnreg_inc<UM_CONSUMER_REGS>();
  const int wg = warp >> 2;                    // rows 64*wg .. 64*wg + 63 of the tile
  const uint32_t a_off = (uint32_t)wg * 64 * 128;
  int stage = 0;
  uint32_t phase_bit = 0;
  // racc: the tile's fp32 accumulator.  From the end of a tile until the end of the next tile's first chunk it
  // holds the finished tile (epilogue `pend`, slices done so far `slice`).
  float racc[NR];
  EpiTile pend;
  bool pending = false;
  int slice = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    for (int kb0 = 0; kb0 < KB; kb0 += p.kb_per_chunk) {
      const int kb1 = kb0 + p.kb_per_chunk < KB ? kb0 + p.kb_per_chunk : KB;
      float acc[NR];
#pragma unroll
      for (int j = 0; j < NR; ++j) acc[j] = 0.f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase_bit, abort_flag, p.fault, 0xF0000000ull | (unsigned)kb);
        const uint32_t sbase = tiles_base + stage * STAGE_BYTES;
        const uint64_t da_hi = make_sw128_desc(sbase + a_off);
        const uint64_t da_lo = make_sw128_desc(sbase + OFF_ALO + a_off);
        const uint64_t db_hi = make_sw128_desc(sbase + OFF_WHI);
        const uint64_t db_lo = make_sw128_desc(sbase + OFF_WLO);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < UM_BK / 16; ++k) {
          const uint64_t ko = (uint64_t)(k * 32 >> 4);   // +32 B per k16 inside the swizzle atom
          if (PASSES == 3) {
            conv_mma<BN, F16>(acc, da_lo + ko, db_hi + ko);
            conv_mma<BN, F16>(acc, da_hi + ko, db_lo + ko);
          }
          conv_mma<BN, F16>(acc, da_hi + ko, db_hi + ko);
        }
        wgmma_commit();
        wgmma_wait<1>();                       // the previous K block's products have retired: free its slot
        if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase_bit ^= 1; }
        if (pending) {
          // the previous tile's epilogue, one slice per K block while its wgmmas run; the chunk's last K block
          // takes the slices left over
          const int s_end = kb + 1 < kb1 ? slice + 1 : UM_SLICES;
          epi_slices<BN>(p, racc, pend, slice, s_end, warp, lane, stats_s);
          slice = s_end;
        }
      }
      if (pending) {
        epi_stats_out<BN>(p, pend, stats_s);
        pending = false;
      }
      wgmma_wait<0>();
      reg_fence<NR>(acc);
      if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
      if (kb0 == 0) {
#pragma unroll
        for (int j = 0; j < NR; ++j) racc[j] = 0.f + acc[j];
      } else {
#pragma unroll
        for (int j = 0; j < NR; ++j) racc[j] += acc[j];
      }
    }
    pend = epi_tile(p, tile, n_blocks, warp, lane);
    pending = true;
    slice = 0;
  }
  if (pending) {
    // a CTA's last tile: nothing left to overlap with
    epi_slices<BN>(p, racc, pend, 0, UM_SLICES, warp, lane, stats_s);
    epi_stats_out<BN>(p, pend, stats_s);
  }
}

// ---- Winograd position GEMMs (weights_per_image, fp32 NHWC store + optional bias) ---------------------------------
// Same tiles, ring, products, chunk boundaries and fold order as conv_umma_kernel, so the result is bit-identical; two
// things differ.  A finished tile needs no epilogue state (no residual, statistics or split outputs): the consumers
// store it straight from the fp32 sum and keep nothing across the next tile.  The registers that frees hold a second
// chunk accumulator: chunk c + 1 is issued into one while chunk c, in the other, waits for its fold.  The fold runs
// after chunk c + 1's first K block is committed and `wgmma_wait<1>` has retired chunk c, so the tensor core is never
// drained at a chunk boundary; only a CTA's last tile ends in `wgmma_wait<0>`.

template <int BN, bool F16>
__device__ __forceinline__ void wino_mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  if (F16) {
    if (BN == 128) wgmma_n128_f16<0>(d, da, db, scale_d); else wgmma_n64_f16<0>(d, da, db, scale_d);
  } else {
    if (BN == 128) wgmma_n128_bf16<0>(d, da, db, scale_d); else wgmma_n64_bf16<0>(d, da, db, scale_d);
  }
}

// One row block of a finished tile: out[pix, n] = racc (+ bias), columns nb * BN .. nb * BN + BN - 1 (BN divides
// Cout on this route).
template <int BN>
__device__ __forceinline__ void wino_store(const ConvParams& p, const float* racc, int tile, int n_blocks, int warp,
                                           int lane) {
  const int nb = tile % n_blocks;
  int mt = tile / n_blocks;
  const int tw = mt % p.tiles_w; mt /= p.tiles_w;
  const int th = mt % p.tiles_h;
  const int tb = mt / p.tiles_h;                 // transform position (TB == 1: a tile lies inside one position)
  const int n0 = nb * BN + 2 * (lane & 3);
#pragma unroll
  for (int ri = 0; ri < 2; ++ri) {
    const int row = 16 * warp + (lane >> 2) + 8 * ri;
    const int ws = tw * p.TW + row % p.TW, hs = th * p.TH + row / p.TW;
    if (ws >= p.W || hs >= p.H) continue;
    float* op = p.out + (((int64_t)tb * p.H + hs) * p.W + ws) * p.Cout + n0;
#pragma unroll
    for (int jj = 0; jj < BN / 8; ++jj) {
      float2 v = make_float2(racc[4 * jj + 2 * ri], racc[4 * jj + 2 * ri + 1]);
      if (p.bias) { const float2 b = *reinterpret_cast<const float2*>(p.bias + n0 + 8 * jj); v.x += b.x; v.y += b.y; }
      *reinterpret_cast<float2*>(op + 8 * jj) = v;
    }
  }
}

// Consumer side of the position-GEMM kernel: where the chunk stream stands.  `tile`, `kb0`: the next chunk to issue;
// the pending chunk (issued, not yet folded) belongs to `pend_tile` and starts (`pend_first`) or ends (`pend_last`)
// that tile's K loop.
struct WinoStream {
  int tile, kb0, stage, prev, pend_tile;
  uint32_t phase_bit;
  bool pend, pend_first, pend_last;
};

// Folds the pending chunk's accumulator into racc (round-to-nearest, the order of conv_umma_kernel) and stores a
// finished tile.  The caller has retired the chunk's wgmmas.
template <int BN>
__device__ __forceinline__ void wino_fold(const ConvParams& p, WinoStream& s, float* racc, float* acc, int n_blocks,
                                          int warp, int lane) {
  constexpr int NR = BN / 2;
  reg_fence<NR>(acc);
  if (s.pend_first) {
#pragma unroll
    for (int j = 0; j < NR; ++j) racc[j] = 0.f + acc[j];
  } else {
#pragma unroll
    for (int j = 0; j < NR; ++j) racc[j] += acc[j];
  }
  if (s.pend_last) wino_store<BN>(p, racc, s.pend_tile, n_blocks, warp, lane);
  s.pend = false;
}

// Issues the next chunk into `acc` and folds the pending one (in `other`) once the chunk's first K block is in
// flight.  Returns false when the CTA has no chunk left (nothing issued; the pending chunk is still in `other`).
template <int BN, int PASSES, bool F16, uint32_t STAGE_BYTES, int STAGES>
__device__ __forceinline__ bool wino_chunk(const ConvParams& p, WinoStream& s, float* racc, float* acc, float* other,
                                           uint32_t tiles_base, uint32_t bar_full, uint32_t bar_empty,
                                           volatile int* abort_flag, int total_tiles, int n_blocks, int KB, int warp,
                                           int lane) {
  constexpr int NR = BN / 2;
  constexpr uint32_t OFF_ALO = UmmaCfg<BN>::A_BYTES;
  constexpr uint32_t OFF_WHI = PASSES == 3 ? 2 * UmmaCfg<BN>::A_BYTES : UmmaCfg<BN>::A_BYTES;
  constexpr uint32_t OFF_WLO = OFF_WHI + UmmaCfg<BN>::W_BYTES;
  if (s.tile >= total_tiles) return false;
  const uint32_t a_off = (uint32_t)(warp >> 2) * 64 * 128;
  const int kb1 = s.kb0 + p.kb_per_chunk < KB ? s.kb0 + p.kb_per_chunk : KB;
  for (int kb = s.kb0; kb < kb1; ++kb) {
    mbar_wait(bar_full + 8 * s.stage, s.phase_bit, abort_flag, p.fault, 0xF6000000ull | (unsigned)kb);
    const uint32_t sbase = tiles_base + s.stage * STAGE_BYTES;
    const uint64_t da_hi = make_sw128_desc(sbase + a_off);
    const uint64_t da_lo = make_sw128_desc(sbase + OFF_ALO + a_off);
    const uint64_t db_hi = make_sw128_desc(sbase + OFF_WHI);
    const uint64_t db_lo = make_sw128_desc(sbase + OFF_WLO);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < UM_BK / 16; ++k) {
      const uint64_t ko = (uint64_t)(k * 32 >> 4);
      // the chunk's first product overwrites the accumulator (scale-d = 0): the chunk starts from zero without a
      // register write that the tensor core would have to wait for
      const uint32_t keep = (k == 0 && kb == s.kb0) ? 0u : 1u;
      if (PASSES == 3) {
        wino_mma<BN, F16>(acc, da_lo + ko, db_hi + ko, keep);
        wino_mma<BN, F16>(acc, da_hi + ko, db_lo + ko, 1u);
      }
      wino_mma<BN, F16>(acc, da_hi + ko, db_hi + ko, PASSES == 3 ? 1u : keep);
    }
    wgmma_commit();
    wgmma_wait<1>();                         // everything before this K block has retired: free the previous slot
    if (s.prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * s.prev);
    s.prev = s.stage;
    if (++s.stage == STAGES) { s.stage = 0; s.phase_bit ^= 1; }
    if (s.pend) wino_fold<BN>(p, s, racc, other, n_blocks, warp, lane);
  }
  s.pend = true;
  s.pend_tile = s.tile;
  s.pend_first = s.kb0 == 0;
  s.pend_last = kb1 == KB;
  s.kb0 = kb1;
  if (s.kb0 == KB) { s.kb0 = 0; s.tile += gridDim.x; }
  return true;
}

template <int BN, int PASSES, bool F16>
__device__ __forceinline__ void wino_drain(const ConvParams& p, WinoStream& s, float* racc, float* acc,
                                           uint32_t bar_empty, int n_blocks, int warp, int lane) {
  if (!s.pend) return;
  wgmma_wait<0>();
  if (lane == 0) mbar_arrive(bar_empty + 8 * s.prev);
  wino_fold<BN>(p, s, racc, acc, n_blocks, warp, lane);
}

template <int BN, int PASSES, bool F16>
__global__ void __launch_bounds__(UM_THREADS, 1)
wino_gemm_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                 const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                 const ConvParams p) {
  using Cfg = UmmaCfg<BN>;
  constexpr int STAGES = PASSES == 3 ? Cfg::STAGES3 : Cfg::STAGES1;
  constexpr uint32_t STAGE_BYTES = PASSES == 3 ? Cfg::STAGE3 : Cfg::STAGE1;
  constexpr uint32_t OFF_ALO = Cfg::A_BYTES;
  constexpr uint32_t OFF_WHI = PASSES == 3 ? 2 * Cfg::A_BYTES : Cfg::A_BYTES;
  constexpr uint32_t OFF_WLO = OFF_WHI + Cfg::W_BYTES;
  constexpr int NR = BN / 2;
  static_assert(STAGES >= 2, "need at least a double buffer");

  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bars[2 * 8];
  __shared__ int abort_s;

  const uint32_t tiles_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar_full = smem_u32(&bars[0]);
  const uint32_t bar_empty = smem_u32(&bars[8]);
  volatile int* abort_flag = &abort_s;

  if (threadIdx.x == 0) {
    abort_s = 0;
    for (int i = 0; i < STAGES; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int n_blocks = p.Cout / BN;
  const int total_tiles = p.n_tiles * n_blocks;
  const int KB = p.K1;

  if (warp >= 8) {
    setmaxnreg_dec<UM_PRODUCER_REGS>();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase_bit = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nb = tile % n_blocks;
        int mt = tile / n_blocks;
        const int tw = mt % p.tiles_w; mt /= p.tiles_w;
        const int th = mt % p.tiles_h;
        const int tb = mt / p.tiles_h;
        const int w0 = tw * p.TW, h0 = th * p.TH, n0 = nb * BN;
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(bar_empty + 8 * stage, phase_bit ^ 1, abort_flag, p.fault, 0xE6000000ull | (unsigned)kb);
          const uint32_t sbase = tiles_base + stage * STAGE_BYTES;
          const uint32_t full = bar_full + 8 * stage;
          mbar_expect_tx(full, STAGE_BYTES);
          tma_load_4d(sbase, &map_a_hi, full, kb * UM_BK, w0, h0, tb);
          if (PASSES == 3) tma_load_4d(sbase + OFF_ALO, &map_a_lo, full, kb * UM_BK, w0, h0, tb);
          tma_load_3d(sbase + OFF_WHI, &map_w_hi, full, kb * UM_BK, n0, tb);
          if (PASSES == 3) tma_load_3d(sbase + OFF_WLO, &map_w_lo, full, kb * UM_BK, n0, tb);
          if (++stage == STAGES) { stage = 0; phase_bit ^= 1; }
        }
      }
    }
    return;
  }

  setmaxnreg_inc<UM_CONSUMER_REGS>();
  float racc[NR], acc0[NR], acc1[NR];
  WinoStream s;
  s.tile = blockIdx.x; s.kb0 = 0; s.stage = 0; s.prev = -1; s.pend_tile = -1; s.phase_bit = 0;
  s.pend = s.pend_first = s.pend_last = false;
  // chunks alternate between the two accumulators; each call folds the chunk the other one holds
  for (;;) {
    if (!wino_chunk<BN, PASSES, F16, STAGE_BYTES, STAGES>(p, s, racc, acc0, acc1, tiles_base, bar_full, bar_empty,
                                                          abort_flag, total_tiles, n_blocks, KB, warp, lane)) {
      wino_drain<BN, PASSES, F16>(p, s, racc, acc1, bar_empty, n_blocks, warp, lane);
      break;
    }
    if (!wino_chunk<BN, PASSES, F16, STAGE_BYTES, STAGES>(p, s, racc, acc1, acc0, tiles_base, bar_full, bar_empty,
                                                          abort_flag, total_tiles, n_blocks, KB, warp, lane)) {
      wino_drain<BN, PASSES, F16>(p, s, racc, acc0, bar_empty, n_blocks, warp, lane);
      break;
    }
  }
}

// ------------------------------------------------------------------------------- host side
// bf16 NHWC activation [B,H,W,C] -> 4-D map (C, W, H, B), box (64, TW, TH, TB), SWIZZLE_128B
static int make_act_map(CUtensorMap* m, const void* ptr, int B, int H, int W, int C, int TW, int TH, int TB,
                        bool f16) {
  EncodeTiledFn enc = get_encode();
  BBDM_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)UM_BK, (cuuint32_t)TW, (cuuint32_t)TH, (cuuint32_t)TB};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  BBDM_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(activation) failed: %d (B=%d H=%d W=%d C=%d box=%dx%dx%d)",
               (int)r, B, H, W, C, TW, TH, TB);
  return BBDM_OK;
}

// bf16 weights [taps][Cout][Cin] -> 3-D map (Cin, Cout, taps), box (64, BN, 1)
static int make_w_map(CUtensorMap* m, const void* ptr, int taps, int Cout, int Cin, int BN, bool f16) {
  EncodeTiledFn enc = get_encode();
  BBDM_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)Cout, (cuuint64_t)taps};
  cuuint64_t strides[2] = {(cuuint64_t)Cin * 2, (cuuint64_t)Cout * Cin * 2};
  cuuint32_t box[3] = {(cuuint32_t)UM_BK, (cuuint32_t)BN, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = enc(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  BBDM_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(weight) failed: %d (taps=%d Cout=%d Cin=%d BN=%d)", (int)r,
               taps, Cout, Cin, BN);
  return BBDM_OK;
}

static int pow2_floor(int x) { int p = 1; while (p * 2 <= x) p *= 2; return p; }
static int pow2_ceil(int x) { int p = 1; while (p < x) p *= 2; return p; }

template <int BN, int PASSES, bool F16>
static int launch_conv(const CUtensorMap* maps, const ConvParams& p, int grid, cudaStream_t s) {
  using Cfg = UmmaCfg<BN>;
  constexpr int STAGES = PASSES == 3 ? Cfg::STAGES3 : Cfg::STAGES1;
  constexpr uint32_t STAGE_BYTES = PASSES == 3 ? Cfg::STAGE3 : Cfg::STAGE1;
  const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024;
  static DeviceOnce configured;
  if (configured.need()) {
    BBDM_CUDA_CHECK(cudaFuncSetAttribute(conv_umma_kernel<BN, PASSES, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured.mark();
  }
  conv_umma_kernel<BN, PASSES, F16><<<grid, UM_THREADS, smem, s>>>(maps[0], maps[1], maps[2], maps[3], maps[4], maps[5],
                                                                  maps[6], maps[7], p);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

template <int BN, int PASSES, bool F16>
static int launch_wino(const CUtensorMap* maps, const ConvParams& p, int grid, cudaStream_t s) {
  using Cfg = UmmaCfg<BN>;
  constexpr int STAGES = PASSES == 3 ? Cfg::STAGES3 : Cfg::STAGES1;
  constexpr uint32_t STAGE_BYTES = PASSES == 3 ? Cfg::STAGE3 : Cfg::STAGE1;
  const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024;
  static DeviceOnce configured;
  if (configured.need()) {
    BBDM_CUDA_CHECK(cudaFuncSetAttribute(wino_gemm_kernel<BN, PASSES, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured.mark();
  }
  wino_gemm_kernel<BN, PASSES, F16><<<grid, UM_THREADS, smem, s>>>(maps[0], maps[1], maps[2], maps[3], p);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // namespace bbdm

using namespace bbdm;

static void tile_geometry(int H, int W, int* TW, int* TH, int* TB) {
  *TW = pow2_floor(W) < 16 ? pow2_floor(W) : 16;
  const int th = pow2_ceil(H);
  *TH = th < UM_BM / *TW ? th : UM_BM / *TW;
  *TB = UM_BM / (*TW * *TH);
}

// (for an upsample2x conv call this with the INPUT H, W and multiply rows_per_image by 4)
extern "C" int bbdm_conv_umma_geometry(int H, int W, int* TW, int* TH, int* TB, int* rows_per_image) {
  BBDM_REQUIRE(H > 0 && W >= 4, "conv_umma_geometry: need H > 0, W >= 4");
  int tw, th, tb;
  tile_geometry(H, W, &tw, &th, &tb);
  if (TW) *TW = tw;
  if (TH) *TH = th;
  if (TB) *TB = tb;
  if (rows_per_image) *rows_per_image = tb == 1 ? 4 * ((W + tw - 1) / tw) * ((H + th - 1) / th) : 0;
  return BBDM_OK;
}

extern "C" int bbdm_conv_umma(const BbdmConvArgs* a, void* stream) {
  BBDM_REQUIRE(a != nullptr, "conv_umma: null args");
  BBDM_REQUIRE(a->B > 0 && a->H > 0 && a->W > 0, "conv_umma: bad spatial shape");
  BBDM_REQUIRE(a->taps == 1 || a->taps == 9 || a->taps == 4, "conv_umma: taps must be 1, 4 or 9 (got %d)", a->taps);
  BBDM_REQUIRE(!a->upsample2x || (a->taps == 4 && a->Cin2 == 0), "conv_umma: upsample2x needs the 16 phase taps and no fused 1x1");
  BBDM_REQUIRE(a->Cin > 0 && a->Cin % 32 == 0, "conv_umma: Cin %% 32 != 0 (Cin=%d)", a->Cin);
  BBDM_REQUIRE(a->Cout > 0 && a->Cout % 32 == 0, "conv_umma: Cout %% 32 != 0 (Cout=%d)", a->Cout);
  BBDM_REQUIRE(a->Cin2 >= 0 && a->Cin2 % 32 == 0, "conv_umma: Cin2 %% 32 != 0 (Cin2=%d)", a->Cin2);
  BBDM_REQUIRE(a->passes == 1 || a->passes == 3, "conv_umma: passes must be 1 or 3");
  BBDM_REQUIRE(a->a_hi && a->w_hi && (a->passes == 1 || (a->a_lo && a->w_lo)), "conv_umma: missing operand plane");
  if (a->Cin2) BBDM_REQUIRE(a->a2_hi && a->w2_hi && (a->passes == 1 || (a->a2_lo && a->w2_lo)), "conv_umma: missing 1x1 operand plane");
  BBDM_REQUIRE(a->out || (a->out_hi && a->out_lo), "conv_umma: no output");
  BBDM_REQUIRE((a->out_hi == nullptr) == (a->out_lo == nullptr), "conv_umma: out hi/lo must come in pairs");
  BBDM_REQUIRE(a->res_mode >= 0 && a->res_mode <= 3 && (a->res_mode == 0 || a->residual), "conv_umma: bad residual");
  if (a->res_mode == BBDM_RES_UP2 && !a->upsample2x) BBDM_REQUIRE(a->H % 2 == 0 && a->W % 2 == 0, "conv_umma: RES_UP2 needs even H, W");
  BBDM_REQUIRE(a->W >= 4, "conv_umma: W < 4 not supported (use conv_direct)");
  BBDM_REQUIRE(a->window_origin == 0 || a->window_origin == -1, "conv_umma: window_origin must be 0 or -1 (got %d)",
               a->window_origin);
  BBDM_REQUIRE(a->window_origin == 0 || (a->taps == 4 && !a->upsample2x),
               "conv_umma: window_origin -1 needs taps == 4 and no upsample2x");
  const bool wpi = a->weights_per_image != 0, f16 = a->operand_f16 != 0;
  if (wpi) BBDM_REQUIRE(a->taps == 1 && a->Cin2 == 0 && !a->upsample2x, "conv_umma: weights_per_image needs taps == 1 and no fused operand");
  if (wpi) BBDM_REQUIRE(a->Cin % 64 == 0 && a->Cout % 64 == 0, "conv_umma: weights_per_image needs Cin, Cout %% 64 == 0");

  ConvParams p;
  p.B = a->B; p.H = a->H; p.W = a->W; p.Cout = a->Cout;
  tile_geometry(a->H, a->W, &p.TW, &p.TH, &p.TB);
  p.tiles_w = (a->W + p.TW - 1) / p.TW;
  p.tiles_h = (a->H + p.TH - 1) / p.TH;
  p.tiles_b = (a->B + p.TB - 1) / p.TB;
  p.n_tiles = p.tiles_w * p.tiles_h * p.tiles_b;
  // N tile: 128 couts where 128-wide blocks cover Cout with no more padding columns than 64-wide ones (64 accumulator +
  // 64 promotion registers per thread; each A box is then loaded once per 128 couts): Cout % 128 in {0, 96}.  At
  // Cout % 128 in {32, 64} the last 128-wide block would compute 96 or 64 zero columns, so 64-wide ones pad at most
  // 32.  Either way 64-wide tiles when 128-wide ones leave most SMs without a tile (small spatial extents / batches):
  // more CTAs finish sooner.
  int BN = (a->Cout + 127) / 128 * 128 == (a->Cout + 63) / 64 * 64 ? 128 : 64;
  {
    const int64_t m_tiles = (int64_t)p.n_tiles * (a->upsample2x ? 4 : 1);
    const int64_t want = (int64_t)(0.7 * num_sms());
    if (BN > 64 && m_tiles * ((a->Cout + BN - 1) / BN) < want) BN = 64;
  }
  p.kb_per_tap = (a->Cin + UM_BK - 1) / UM_BK;
  p.K1 = a->taps * p.kb_per_tap;
  p.K2 = (a->Cin2 + UM_BK - 1) / UM_BK;
  p.taps = a->taps;
  p.up2 = a->upsample2x ? 1 : 0;
  p.origin = a->window_origin;
  p.w_per_image = wpi ? 1 : 0;
  // chunk length: 4 K-blocks (direct conv, split operands), 8 (single pass).  The Winograd position GEMMs promote
  // more often, because their output transform amplifies the truncation error of the tensor core's accumulator:
  // every 2 K-blocks below 512 input channels, every 4 from 512 on.  BBDM_WINO_CHUNK overrides (A/B switch).
  static int wino_chunk = -1;
  if (wino_chunk < 0) { const char* e = getenv("BBDM_WINO_CHUNK"); wino_chunk = (e && atoi(e) > 0) ? atoi(e) : 0; }
  const int wchunk = wino_chunk ? wino_chunk : (a->Cin >= 512 ? 4 : 2);
  p.kb_per_chunk = wpi ? wchunk : (a->passes == 3 ? 4 : 8);
  if (wpi) BBDM_REQUIRE(p.TB == 1, "conv_umma: weights_per_image needs 128-pixel tiles inside one image (H*W >= 128)");
  p.bias = a->bias; p.bias2 = a->Cin2 ? a->bias2 : nullptr;
  p.residual = a->residual; p.res_mode = a->res_mode;
  p.out = a->out; p.out_hi = (__nv_bfloat16*)a->out_hi; p.out_lo = (__nv_bfloat16*)a->out_lo;
  p.out_nchw_c = a->out_nchw_channels;
  p.stats = a->stats_partial;
  BBDM_REQUIRE(p.out_nchw_c >= 0 && p.out_nchw_c <= a->Cout && (p.out_nchw_c == 0 || (a->out && !a->out_hi)),
               "conv_umma: bad out_nchw_channels");
  p.fault = device_fault_ptr();
  BBDM_REQUIRE(p.fault != nullptr, "conv_umma: device fault word unavailable");

  BBDM_REQUIRE(p.stats == nullptr || (p.TB == 1 && p.out_nchw_c == 0),
               "conv_umma: stats_partial needs a tile inside one image (H*W >= 128) and NHWC output");
  CUtensorMap maps[8];
  int rc;
  if ((rc = make_act_map(&maps[0], a->a_hi, a->B, a->H, a->W, a->Cin, p.TW, p.TH, p.TB, f16))) return rc;
  if ((rc = make_act_map(&maps[1], a->passes == 3 ? a->a_lo : a->a_hi, a->B, a->H, a->W, a->Cin, p.TW, p.TH, p.TB, f16))) return rc;
  const int wtaps = a->upsample2x ? 16 : (wpi ? a->B : a->taps);
  if ((rc = make_w_map(&maps[2], a->w_hi, wtaps, a->Cout, a->Cin, BN, f16))) return rc;
  if ((rc = make_w_map(&maps[3], a->passes == 3 ? a->w_lo : a->w_hi, wtaps, a->Cout, a->Cin, BN, f16))) return rc;
  if (a->Cin2) {
    if ((rc = make_act_map(&maps[4], a->a2_hi, a->B, a->H, a->W, a->Cin2, p.TW, p.TH, p.TB, f16))) return rc;
    if ((rc = make_act_map(&maps[5], a->passes == 3 ? a->a2_lo : a->a2_hi, a->B, a->H, a->W, a->Cin2, p.TW, p.TH, p.TB, f16))) return rc;
    if ((rc = make_w_map(&maps[6], a->w2_hi, 1, a->Cout, a->Cin2, BN, f16))) return rc;
    if ((rc = make_w_map(&maps[7], a->passes == 3 ? a->w2_lo : a->w2_hi, 1, a->Cout, a->Cin2, BN, f16))) return rc;
  } else {
    maps[4] = maps[0]; maps[5] = maps[1]; maps[6] = maps[2]; maps[7] = maps[3];
  }
  const int64_t total = (int64_t)p.n_tiles * ((a->Cout + BN - 1) / BN) * (p.up2 ? 4 : 1);
  BBDM_REQUIRE(total < (1ll << 30), "conv_umma: too many tiles");
  const int grid = (int)(total < num_sms() ? total : num_sms());
  cudaStream_t s = (cudaStream_t)stream;
  const bool p3 = a->passes == 3;
  // position GEMMs whose epilogue is a plain store (+ bias): the kernel without epilogue state (the Winograd route)
  if (wpi && p.res_mode == BBDM_RES_NONE && !p.stats && !p.out_hi && !p.out_nchw_c && p.out) {
    if (BN == 128) {
      if (f16) return p3 ? launch_wino<128, 3, true>(maps, p, grid, s) : launch_wino<128, 1, true>(maps, p, grid, s);
      return p3 ? launch_wino<128, 3, false>(maps, p, grid, s) : launch_wino<128, 1, false>(maps, p, grid, s);
    }
    if (f16) return p3 ? launch_wino<64, 3, true>(maps, p, grid, s) : launch_wino<64, 1, true>(maps, p, grid, s);
    return p3 ? launch_wino<64, 3, false>(maps, p, grid, s) : launch_wino<64, 1, false>(maps, p, grid, s);
  }
  if (BN == 128) {
    if (f16) return p3 ? launch_conv<128, 3, true>(maps, p, grid, s) : launch_conv<128, 1, true>(maps, p, grid, s);
    return p3 ? launch_conv<128, 3, false>(maps, p, grid, s) : launch_conv<128, 1, false>(maps, p, grid, s);
  }
  if (f16) return p3 ? launch_conv<64, 3, true>(maps, p, grid, s) : launch_conv<64, 1, true>(maps, p, grid, s);
  return p3 ? launch_conv<64, 3, false>(maps, p, grid, s) : launch_conv<64, 1, false>(maps, p, grid, s);
}
