// Weight gradient of the stride-1 "same" convolution on Hopper wgmma tensor cores (sm_90a).
//
//   dW[tap][co][ci] = sum over pixels p of  dY[p][co] * A[p + tap][ci]
//
// taps: 1 (1x1), 9 (3x3 window at offsets -1..1), or 4 (2x2 window at offsets origin..origin+1, origin 0 or -1: the
// stride-2 3x3 conv on a space-to-depth operand, and its adjoint).
//
// GEMM view per filter tap:  M = Cout (tile 128), N = Cin (tile BN), K = pixels (blocks of 64).
//   * A operand  = dY^T planes [Cout][P] with a row pitch of ld_g >= P pixels (K-major: 64 consecutive pixels = one
//     128-byte row), written by bbdm_split_grad; 2-D TMA map, SWIZZLE_128B, OOB zero fill past pixel P.
//   * B operand  = the forward conv's input planes [B,H,W,Cin], loaded in TMA im2col mode: K block kb is the pixels
//     [64 kb, 64 kb + 64) of the flattened (b, h, w) index, wherever the run wraps across rows or images, each read
//     at the filter tap's offset (the im2col offsets; OOB zero fill = the conv padding and everything past the last
//     image).  64 channels per pixel = one 128-byte SWIZZLE_128B row, so the shared-memory image is the one a
//     tiled box of the same 64 pixels gives.  Consumed as an MN-major operand (channels contiguous); BN/64 swizzle
//     atoms side by side, LBO = one atom (8 KiB).
//   * two consumer warpgroups (couts 0-63 / 64-127 of the tile) + one TMA producer warp; split-bf16 x3
//     products, chunked wgmma -> fp32-register promotion (as conv_umma.cu).
//   * Cin and Cout are multiples of 32.  The last Cin tile may run past Cin: a channel past the end only reaches the
//     accumulator column of that channel, and columns past Cin are not stored, so the result does not depend on what
//     the im2col load puts there.  Likewise rows past Cout of the last Cout tile (the dY^T map zero-fills them).
//   * K is split across CTAs (the pixel range); every CTA writes its partial [split][tap][Cout][Cin]
//     tile, bbdm's reduce kernel sums the splits in a fixed order (deterministic) into OIHW.
#include "tc_common.cuh"

namespace bbdm {

constexpr int WG_BM = 128;   // couts per tile
constexpr int WG_BK = 64;    // pixels per K block
constexpr int WG_THREADS = 288;

struct WgradParams {
  int Cout, Cin, taps, origin;
  int n_co, n_ci;            // tiles along Cout / Cin
  int H, W;                  // map geometry (the K block's first pixel -> im2col coordinates)
  int lo;                    // im2col bounding-box corner: the window's first row / column offset (-1, 0)
  int kblocks;               // total K blocks = ceil(P / 64)
  int splits, kb_per_split;
  int kb_per_chunk;
  float* partial;            // [splits][taps][Cout][Cin]
  unsigned long long* fault;
};

// N tile along Cin: 128 where 128-wide tiles cover Cin with no more padding channels than 64-wide ones (64 accumulator
// + 64 promotion registers per thread), i.e. Cin % 128 in {0, 96}
static inline int wgrad_bn(int Cin) { return (Cin + 127) / 128 * 128 == (Cin + 63) / 64 * 64 ? 128 : 64; }

template <int BN>
__global__ void __launch_bounds__(WG_THREADS, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap map_g_hi, const __grid_constant__ CUtensorMap map_g_lo,
                  const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                  const WgradParams p) {
  constexpr uint32_t G_BYTES = WG_BM * WG_BK * 2;       // 16 KiB per plane (dY^T tile)
  constexpr uint32_t A_ATOM = WG_BK * 64 * 2;           // 8 KiB: 64 pixels x 64 channels
  constexpr uint32_t A_BYTES = (BN / 64) * A_ATOM;      // per plane
  constexpr uint32_t STAGE_BYTES = 2 * G_BYTES + 2 * A_BYTES;
  constexpr int STAGES = (200 * 1024 / STAGE_BYTES) > 6 ? 6 : (200 * 1024 / STAGE_BYTES);
  constexpr int NR = BN / 2;
  static_assert(STAGES >= 2, "stage too large");

  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bars[2 * 8];
  __shared__ int abort_s;
  const uint32_t tiles_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar_full = smem_u32(&bars[0]), bar_empty = smem_u32(&bars[8]);
  volatile int* abort_flag = &abort_s;

  if (threadIdx.x == 0) {
    abort_s = 0;
    for (int i = 0; i < STAGES; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // work item = (split, tap, co tile, ci tile); persistent over the grid
  const int total = p.splits * p.taps * p.n_co * p.n_ci;

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < total; item += gridDim.x) {
        int r = item;
        const int ci_t = r % p.n_ci; r /= p.n_ci;
        const int co_t = r % p.n_co; r /= p.n_co;
        const int tap = r % p.taps;
        const int split = r / p.taps;
        // tap offset within the window, counted from its first row / column (the map's bounding-box corner p.lo)
        uint16_t oy = 0, ox = 0;
        if (p.taps == 9) { oy = (uint16_t)(tap / 3); ox = (uint16_t)(tap % 3); }
        else if (p.taps == 4) { oy = (uint16_t)(tap >> 1); ox = (uint16_t)(tap & 1); }
        const int kb0 = split * p.kb_per_split;
        const int kb1 = kb0 + p.kb_per_split < p.kblocks ? kb0 + p.kb_per_split : p.kblocks;
        for (int kb = kb0; kb < kb1; ++kb) {
          const int px = kb * WG_BK;                   // first pixel of the K block
          const int pw = px % p.W, ph = (px / p.W) % p.H, pb = px / (p.W * p.H);
          mbar_wait(bar_empty + 8 * stage, phase ^ 1, abort_flag, p.fault, 0xC5000000ull | (unsigned)kb);
          const uint32_t sb = tiles_base + stage * STAGE_BYTES, full = bar_full + 8 * stage;
          mbar_expect_tx(full, STAGE_BYTES);
          // dY^T tile: rows = 128 couts, 64 consecutive pixels (flattened index kb*64)
          tma_load_2d(sb, &map_g_hi, full, kb * WG_BK, co_t * WG_BM);
          tma_load_2d(sb + G_BYTES, &map_g_lo, full, kb * WG_BK, co_t * WG_BM);
#pragma unroll
          for (int at = 0; at < BN / 64; ++at) {
            const int c0 = ci_t * BN + at * 64;
            tma_load_4d_im2col(sb + 2 * G_BYTES + at * A_ATOM, &map_a_hi, full, c0, pw + p.lo, ph + p.lo, pb, ox, oy);
            tma_load_4d_im2col(sb + 2 * G_BYTES + A_BYTES + at * A_ATOM, &map_a_lo, full, c0, pw + p.lo, ph + p.lo, pb,
                               ox, oy);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // consumer warpgroups: wgmma + promotion + store (rows = couts 64*wg .. 64*wg + 63 of the tile)
  const uint32_t g_off = (uint32_t)(warp >> 2) * 64 * 128;
  int stage = 0;
  uint32_t phase = 0;
  for (int item = blockIdx.x; item < total; item += gridDim.x) {
    int r = item;
    const int ci_t = r % p.n_ci; r /= p.n_ci;
    const int co_t = r % p.n_co; r /= p.n_co;
    const int tap = r % p.taps;
    const int split = r / p.taps;
    const int kb0 = split * p.kb_per_split;
    const int kb1 = kb0 + p.kb_per_split < p.kblocks ? kb0 + p.kb_per_split : p.kblocks;
    float racc[NR];
#pragma unroll
    for (int j = 0; j < NR; ++j) racc[j] = 0.f;
    for (int c0 = kb0; c0 < kb1; c0 += p.kb_per_chunk) {
      const int c1 = c0 + p.kb_per_chunk < kb1 ? c0 + p.kb_per_chunk : kb1;
      float acc[NR];
#pragma unroll
      for (int j = 0; j < NR; ++j) acc[j] = 0.f;
      int prev = -1;
      for (int kb = c0; kb < c1; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase, abort_flag, p.fault, 0xC3000000ull | (unsigned)kb);
        const uint32_t sb = tiles_base + stage * STAGE_BYTES;
        const uint64_t dg_hi = make_sw128_desc(sb + g_off), dg_lo = make_sw128_desc(sb + G_BYTES + g_off);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < WG_BK / 16; ++k) {
          const uint64_t ka = (uint64_t)(k * 32 >> 4);                   // A: +32 B per 16 pixels (K-major)
          const uint32_t ab = sb + 2 * G_BYTES + k * 16 * 128;            // B: +16 pixel rows of 128 B
          const uint64_t da_hi = make_sw128_desc(ab, A_ATOM), da_lo = make_sw128_desc(ab + A_BYTES, A_ATOM);
          if (BN == 128) {
            wgmma_n128_bf16<1>(acc, dg_lo + ka, da_hi, 1u);
            wgmma_n128_bf16<1>(acc, dg_hi + ka, da_lo, 1u);
            wgmma_n128_bf16<1>(acc, dg_hi + ka, da_hi, 1u);
          } else {
            wgmma_n64_bf16<1>(acc, dg_lo + ka, da_hi, 1u);
            wgmma_n64_bf16<1>(acc, dg_hi + ka, da_lo, 1u);
            wgmma_n64_bf16<1>(acc, dg_hi + ka, da_hi, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence<NR>(acc);
      if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
#pragma unroll
      for (int j = 0; j < NR; ++j) racc[j] += acc[j];
    }
#pragma unroll
    for (int ri = 0; ri < 2; ++ri) {
      const int co = co_t * WG_BM + 16 * warp + (lane >> 2) + 8 * ri;
      if (co < p.Cout) {
        float* op = p.partial + (((int64_t)split * p.taps + tap) * p.Cout + co) * p.Cin + ci_t * BN + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < BN / 8; ++jj)
          if (ci_t * BN + 8 * jj < p.Cin)     // Cin % 32 == 0: a block of 8 columns lies wholly inside or past Cin
            *reinterpret_cast<float2*>(op + 8 * jj) = make_float2(racc[4 * jj + 2 * ri], racc[4 * jj + 2 * ri + 1]);
      }
    }
  }
}

// sum the split-K partials in a fixed order; write OIHW:  dW[co][ci][tap].
// thread = one (co, ci) pair, all taps: partial reads coalesced along ci, each thread writes its
// `taps` consecutive output floats.
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ partial, int splits, int taps, int Cout, int Cin, float* __restrict__ dw) {
  const int64_t pairs = (int64_t)Cout * Cin;
  const int64_t n = pairs * taps;
  for (int64_t pr = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pr < pairs; pr += (int64_t)gridDim.x * blockDim.x) {
    for (int t = 0; t < taps; ++t) {
      float s = 0.f;
      for (int k = 0; k < splits; ++k) s += partial[(int64_t)k * n + (int64_t)t * pairs + pr];
      dw[pr * taps + t] = s;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// fp32 NHWC gradient [P][C] -> split planes in both orientations + per-channel sums (bias grad):
//   hi/lo   [P][C]  (K = channel major: A operand of the data-gradient conv)
//   hi_t/lo_t [C][P] with row pitch ld_t (K = pixel major: A operand of the weight-gradient GEMM)
// 32x32 tiles through shared memory; colsum partials per tile row-block, reduced in fixed order.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
split_grad_kernel(const float* __restrict__ src, int64_t P, int C, __nv_bfloat16* __restrict__ hi,
                  __nv_bfloat16* __restrict__ lo, __nv_bfloat16* __restrict__ hi_t, __nv_bfloat16* __restrict__ lo_t,
                  int64_t ld_t, float* __restrict__ colsum_part) {
  __shared__ float tile[64][65];
  const int64_t p0 = (int64_t)blockIdx.x * 64;
  const int c0 = blockIdx.y * 64;
  const int tx = threadIdx.x % 64, ty = threadIdx.x / 64;   // 64 x 4
  for (int r = ty; r < 64; r += 4) {
    const int64_t pp = p0 + r;
    float v = 0.f;
    if (pp < P && c0 + tx < C) v = src[pp * C + c0 + tx];
    tile[r][tx] = v;
    if (pp < P && c0 + tx < C && hi) {
      __nv_bfloat16 h, l;
      split_bf16(v, h, l);
      hi[pp * C + c0 + tx] = h;
      lo[pp * C + c0 + tx] = l;
    }
  }
  __syncthreads();
  // transposed planes: thread tx walks pixels (contiguous in the [C][P] layout)
  for (int r = ty; r < 64; r += 4) {
    const int c = c0 + r;
    const int64_t pp = p0 + tx;
    if (c < C && pp < P) {
      __nv_bfloat16 h, l;
      split_bf16(tile[tx][r], h, l);
      hi_t[(int64_t)c * ld_t + pp] = h;
      lo_t[(int64_t)c * ld_t + pp] = l;
    }
  }
  if (colsum_part && ty == 0 && c0 + tx < C) {
    float s = 0.f;
    for (int r = 0; r < 64; ++r) s += tile[r][tx];
    colsum_part[(int64_t)blockIdx.x * C + c0 + tx] = s;
  }
}

// one CTA per 32 channels: 8 row-lanes x 32 channels, fixed-order fp64 tree => deterministic
__global__ void __launch_bounds__(256)
colsum_reduce_kernel(const float* __restrict__ part, int64_t nblk, int C, float* __restrict__ out) {
  __shared__ double sm[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  double s = 0.0;
  if (c < C)
    for (int64_t b = ry; b < nblk; b += 8) s += (double)part[b * C + c];
  sm[ry][cx] = s;
  __syncthreads();
  if (ry == 0 && c < C) {
    double t = 0.0;
#pragma unroll
    for (int r = 0; r < 8; ++r) t += sm[r][cx];
    out[c] = (float)t;
  }
}

static int make_gt_map(CUtensorMap* m, const void* ptr, int Cout, int64_t P, int64_t ld) {
  EncodeTiledFn enc = get_encode();
  BBDM_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)P, (cuuint64_t)Cout};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)WG_BK, (cuuint32_t)WG_BM};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  BBDM_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(dY^T) failed: %d", (int)r);
  return BBDM_OK;
}

// im2col map of the activation planes: 64 pixels x 64 channels per load.  The bounding box of each image runs from
// row / column lo to H-1+lo / W-1+lo (H x W positions, one per output pixel); a load's coordinates are the first output
// pixel shifted by lo, and the tap's offset within the window (0..2) is the im2col offset.
static int make_act_im2col_map(CUtensorMap* m, const void* ptr, int B, int H, int W, int C, int lo) {
  EncodeIm2colFn enc = get_encode_im2col();
  BBDM_REQUIRE(enc != nullptr, "cuTensorMapEncodeIm2col entry point not available");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const int lower[2] = {lo, lo}, upper[2] = {lo, lo};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, lower, upper, 64,
                   (cuuint32_t)WG_BK, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  BBDM_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeIm2col(wgrad activation) failed: %d (B=%d H=%d W=%d C=%d)", (int)r,
               B, H, W, C);
  return BBDM_OK;
}

template <int BN>
static int launch_wgrad(const CUtensorMap* maps, const WgradParams& p, int grid, cudaStream_t s) {
  constexpr uint32_t STAGE_BYTES = 2 * (WG_BM * WG_BK * 2) + 2 * (BN / 64) * (WG_BK * 64 * 2);
  constexpr int STAGES = (200 * 1024 / STAGE_BYTES) > 6 ? 6 : (200 * 1024 / STAGE_BYTES);
  const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024;
  static DeviceOnce configured;
  if (configured.need()) {
    BBDM_CUDA_CHECK(cudaFuncSetAttribute(conv_wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured.mark();
  }
  conv_wgrad_kernel<BN><<<grid, WG_THREADS, smem, s>>>(maps[0], maps[1], maps[2], maps[3], p);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // namespace bbdm

using namespace bbdm;

extern "C" {

int bbdm_split_grad(const float* src, int64_t P, int C, void* hi, void* lo, void* hi_t, void* lo_t, int64_t ld_t,
                    float* colsum, float* workspace, void* stream) {
  BBDM_REQUIRE(src && hi_t && lo_t && P > 0 && C > 0, "split_grad: bad args");
  BBDM_REQUIRE(ld_t >= P, "split_grad: row pitch %lld of the transposed planes < P = %lld", (long long)ld_t,
               (long long)P);
  BBDM_REQUIRE((hi == nullptr) == (lo == nullptr), "split_grad: hi/lo in pairs");
  BBDM_REQUIRE(colsum == nullptr || workspace != nullptr, "split_grad: colsum needs a workspace of ceil(P/64)*C floats");
  const int64_t nb = (P + 63) / 64;
  BBDM_REQUIRE(nb < (1ll << 31), "split_grad: too many pixels");
  dim3 grid((unsigned)nb, (C + 63) / 64);
  cudaStream_t s = (cudaStream_t)stream;
  split_grad_kernel<<<grid, 256, 0, s>>>(src, P, C, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, (__nv_bfloat16*)hi_t,
                                         (__nv_bfloat16*)lo_t, ld_t, colsum ? workspace : nullptr);
  BBDM_LAUNCH_CHECK();
  if (colsum) {
    colsum_reduce_kernel<<<(C + 31) / 32, 256, 0, s>>>(workspace, nb, C, colsum);
    BBDM_LAUNCH_CHECK();
  }
  return BBDM_OK;
}

int bbdm_conv_wgrad_workspace(int B, int H, int W, int Cin, int Cout, int taps, int* splits, int64_t* floats) {
  BBDM_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && Cin % 32 == 0 && Cout > 0 && Cout % 32 == 0 &&
               (taps == 1 || taps == 4 || taps == 9), "wgrad_workspace: bad shape");
  const int64_t P = (int64_t)B * H * W;
  const int64_t kblocks = (P + 63) / 64;
  const int BN = wgrad_bn(Cin);
  const int64_t tiles = (int64_t)taps * ((Cout + 127) / 128) * ((Cin + BN - 1) / BN);
  int64_t sp = (3 * (int64_t)num_sms() + tiles - 1) / tiles;
  if (sp > kblocks / 8) sp = kblocks / 8;
  if (sp < 1) sp = 1;
  if (sp > 64) sp = 64;
  if (splits) *splits = (int)sp;
  if (floats) *floats = sp * taps * (int64_t)Cout * Cin;
  return BBDM_OK;
}

int bbdm_conv_wgrad(const void* g_hi_t, const void* g_lo_t, int64_t ld_g, const void* a_hi, const void* a_lo, int B,
                    int H, int W, int Cin, int Cout, int taps, int window_origin, float* dw, float* workspace,
                    void* stream) {
  BBDM_REQUIRE(g_hi_t && g_lo_t && a_hi && a_lo && dw && workspace, "conv_wgrad: null pointer");
  BBDM_REQUIRE(Cin > 0 && Cin % 32 == 0 && Cout > 0 && Cout % 32 == 0 && (taps == 1 || taps == 4 || taps == 9) && W >= 4,
               "conv_wgrad: unsupported shape");
  BBDM_REQUIRE(window_origin == 0 || (taps == 4 && window_origin == -1),
               "conv_wgrad: window_origin -1 needs taps == 4 (got origin %d, taps %d)", window_origin, taps);
  const int64_t P = (int64_t)B * H * W;
  BBDM_REQUIRE(B > 0 && H > 0 && P < (1ll << 31) - WG_BK, "conv_wgrad: bad pixel count (B=%d H=%d W=%d)", B, H, W);
  // TMA global strides are multiples of 16 bytes: the dY^T rows need a pitch of a multiple of 8 pixels
  BBDM_REQUIRE(ld_g >= P && ld_g % 8 == 0, "conv_wgrad: dY^T row pitch %lld must be >= P = %lld and a multiple of 8",
               (long long)ld_g, (long long)P);
  WgradParams p;
  p.Cout = Cout; p.Cin = Cin; p.taps = taps; p.origin = window_origin;
  p.H = H; p.W = W;
  p.lo = taps == 9 ? -1 : (taps == 4 ? window_origin : 0);
  p.kblocks = (int)((P + WG_BK - 1) / WG_BK);
  int splits; int64_t fl;
  int rc = bbdm_conv_wgrad_workspace(B, H, W, Cin, Cout, taps, &splits, &fl);
  if (rc) return rc;
  p.splits = splits;
  p.kb_per_split = (p.kblocks + splits - 1) / splits;
  p.splits = (p.kblocks + p.kb_per_split - 1) / p.kb_per_split;      // no empty splits
  p.kb_per_chunk = 4;
  p.partial = workspace;
  p.fault = device_fault_ptr();
  BBDM_REQUIRE(p.fault != nullptr, "conv_wgrad: device fault word unavailable");
  const int BN = wgrad_bn(Cin);
  p.n_co = (Cout + WG_BM - 1) / WG_BM;
  p.n_ci = (Cin + BN - 1) / BN;
  CUtensorMap maps[4];
  if ((rc = make_gt_map(&maps[0], g_hi_t, Cout, P, ld_g))) return rc;
  if ((rc = make_gt_map(&maps[1], g_lo_t, Cout, P, ld_g))) return rc;
  if ((rc = make_act_im2col_map(&maps[2], a_hi, B, H, W, Cin, p.lo))) return rc;
  if ((rc = make_act_im2col_map(&maps[3], a_lo, B, H, W, Cin, p.lo))) return rc;
  const int64_t total = (int64_t)p.splits * taps * p.n_co * p.n_ci;
  const int grid = (int)(total < num_sms() ? total : num_sms());
  cudaStream_t s = (cudaStream_t)stream;
  if (BN == 128) rc = launch_wgrad<128>(maps, p, grid, s);
  else rc = launch_wgrad<64>(maps, p, grid, s);
  if (rc) return rc;
  const int64_t n = (int64_t)Cout * Cin;
  int64_t g = (n + 255) / 256;
  if (g > (int64_t)num_sms() * 8) g = (int64_t)num_sms() * 8;
  wgrad_reduce_kernel<<<(int)g, 256, 0, s>>>(workspace, p.splits, taps, Cout, Cin, dw);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // extern "C"
