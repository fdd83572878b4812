// Winograd F(4x4, 3x3) for the stride-1 3x3 convolutions of the ResBlocks (openaimodel.py:207,233):
// 4x fewer tensor-core MACs than the direct implicit GEMM.
//
//   Y = A^T [ sum_ci (G g G^T) .* (B^T d B) ] A        per 4x4 output tile / 6x6 input tile
//
// Three kernels around the wgmma GEMM (bbdm_conv_umma, weights_per_image mode: 36 independent
// [tiles x Cin] . [Cin x Cout] products, one per transform position):
//   wino_input_kernel   x (fp32 NHWC, optionally a channel concat) -> GroupNorm affine (+FiLM) -> SiLU ->
//                       V = B^T d B per 6x6 tile (zero padding applies to the ACTIVATED tensor) ->
//                       split-fp16 planes V_hi, V_lo [36][tiles][C]; optionally also the split-bf16 planes of
//                       the raw input (A operand of the ResBlock's 1x1 skip conv).  HBM-bound:
//                       4 B read + 36/16 * 4 B written per input element.
//   wino_weight_kernel  U = s * G g G^T (fp64 from the fp32 OIHW weight) -> split-fp16 [36][Cout][Cin], with the
//                       per-tensor power of two s = 2^(14 - ceil(log2 max|w|)) (wino_wmax_kernel reduces max|w|).
//   wino_output_kernel  M [36][tiles][Cout] fp32 -> Y = (1/s) * A^T M A + bias (+ residual: same / nearest-up /
//                       2x2-avg addressed) -> fp32 NHWC + fused GroupNorm partial sums of the result.
//                       HBM-bound: 36/16 * 4 B read + 4 B written per output element.
//
// F(6x6, 3x3) (interpolation points 0, +-1, +-2, +-1/2; bbdm_wino6_*): the same three kernels over 8x8 input tiles at
// stride 6 and 64 position GEMMs -- 64/36 positions per 36/16 output pixels, 0.79x the MACs and the V / M bytes of
// F(4,3), for the large maps of the UNet sampling executor (convs.wino_tile).  Its transforms amplify rounding more
// (tools/studies/winograd_f63_accuracy.py: the chain sits at the direct split-bf16 kernel's deviation, about 1.5x
// F(4,3)'s) and B^T d B grows a tile by up to 225 (F(4,3): 100), so fp16 V is finite for max|act| <= 291.
//
// Numerics (tools/studies/split_formats_accuracy.py): split-FP16 operands carry 22 mantissa bits (bf16 pairs: 16),
// which pays for the F(4,3) transforms' error amplification; the GEMM promotes the tensor core's truncating
// accumulator into fp32 registers every 2-4 K-blocks (conv_umma.cu), and tests/test_gpu_winograd.py bounds the chain's
// deviation from the fp64 conv.  The weight planes are pre-scaled by the power of two s (exact): every entry of
// G g G^T is bounded by max|g| (the absolute row sums of G are at most 1), so |s U| <= 2^14 < 65504 and the hi and lo
// planes of the largest entries stay normal fp16 numbers at any weight magnitude (a fixed scale loses the lo planes to
// fp16's subnormal range for small weights: 2.5e-5 instead of 6e-6 at weight std 1e-3).  The scale stays on the device
// (1/s in a caller-provided float that the output transform reads): training repacks every step without a host
// synchronisation, and sampling replays a captured graph.
#include "common.cuh"
#include <cuda_fp16.h>
#include <stdlib.h>

namespace bbdm {

constexpr float WINO_WSCALE_FIXED = 256.0f;    // scale without a scale buffer, and of an all-zero weight tensor

// s = 2^(14 - ceil(log2 m)) from the bit pattern of m = max|w| (a non-negative float), exponent clamped to +-100
__host__ __device__ inline float wino_wscale(uint32_t mbits) {
  if (mbits == 0) return WINO_WSCALE_FIXED;
  const int e = (int)(mbits >> 23) - 127;                  // m = 1.f * 2^e (subnormals: e = -127)
  int k = 14 - (e + ((mbits & 0x7fffffu) != 0 ? 1 : 0));
  k = k < -100 ? -100 : (k > 100 ? 100 : k);
  float s = 1.0f;
  for (; k > 0; --k) s *= 2.0f;
  for (; k < 0; ++k) s *= 0.5f;
  return s;
}

// ---- 1-D transforms (interpolation points 0, +-1, +-2; Lavin & Gray) -----------------------------
// B^T (6x6) applied to d[0..5] with stride S in a register array
template <int S>
__device__ __forceinline__ void wino_bt6(float* d) {
  const float d0 = d[0], d1 = d[S], d2 = d[2 * S], d3 = d[3 * S], d4 = d[4 * S], d5 = d[5 * S];
  d[0] = fmaf(4.0f, d0, fmaf(-5.0f, d2, d4));
  d[S] = fmaf(-4.0f, d1 + d2, d3 + d4);
  d[2 * S] = fmaf(4.0f, d1 - d2, d4 - d3);
  d[3 * S] = fmaf(2.0f, d3 - d1, d4 - d2);
  d[4 * S] = fmaf(2.0f, d1 - d3, d4 - d2);
  d[5 * S] = fmaf(4.0f, d1, fmaf(-5.0f, d3, d5));
}
// A^T (4x6) applied to m[0..5] (stride S) -> y[0..3] (stride T)
template <int S, int T>
__host__ __device__ __forceinline__ void wino_at6(const float* m, float* y) {
  const float s12 = m[S] + m[2 * S], d12 = m[S] - m[2 * S];
  const float s34 = m[3 * S] + m[4 * S], d34 = m[3 * S] - m[4 * S];
  y[0] = (m[0] + s12) + s34;
  y[T] = fmaf(2.0f, d34, d12);
  y[2 * T] = fmaf(4.0f, s34, s12);
  y[3 * T] = fmaf(8.0f, d34, d12) + m[5 * S];
}

// ---- F(6x6,3x3): interpolation points 0, +-1, +-2, +-1/2 (and infinity) -----------------------
// B^T (8x8) applied to d[0..7] with stride S.  Absolute row sums reach 15 (F(4,3): 10): |V| <= 225 max|d|.
template <int S>
__device__ __forceinline__ void wino_bt8(float* d) {
  const float d0 = d[0], d1 = d[S], d2 = d[2 * S], d3 = d[3 * S], d4 = d[4 * S], d5 = d[5 * S], d6 = d[6 * S],
              d7 = d[7 * S];
  const float e1 = fmaf(-4.25f, d4, d2 + d6), o1 = fmaf(-4.25f, d3, d1 + d5);
  const float e3 = fmaf(0.25f, d2, fmaf(-1.25f, d4, d6)), o3 = fmaf(0.5f, d1, fmaf(-2.5f, d3, 2.0f * d5));
  const float e5 = fmaf(4.0f, d2, fmaf(-5.0f, d4, d6)), o5 = fmaf(2.0f, d1, fmaf(-2.5f, d3, 0.5f * d5));
  d[0] = fmaf(5.25f, d4 - d2, d0 - d6);
  d[S] = e1 + o1;
  d[2 * S] = e1 - o1;
  d[3 * S] = e3 + o3;
  d[4 * S] = e3 - o3;
  d[5 * S] = e5 + o5;
  d[6 * S] = e5 - o5;
  d[7 * S] = fmaf(5.25f, d3 - d5, d7 - d1);
}
// A^T (6x8) applied to m[0..7] (stride S) -> y[0..5] (stride T)
template <int S, int T>
__host__ __device__ __forceinline__ void wino_at8(const float* m, float* y) {
  const float a = m[S] + m[2 * S], b = m[S] - m[2 * S];
  const float c = m[3 * S] + m[4 * S], d = m[3 * S] - m[4 * S];
  const float e = m[5 * S] + m[6 * S], f = m[5 * S] - m[6 * S];
  y[0] = ((m[0] + a) + c) + e;
  y[T] = fmaf(2.0f, d, fmaf(0.5f, f, b));
  y[2 * T] = fmaf(4.0f, c, fmaf(0.25f, e, a));
  y[3 * T] = fmaf(8.0f, d, fmaf(0.125f, f, b));
  y[4 * T] = fmaf(16.0f, c, fmaf(0.0625f, e, a));
  y[5 * T] = fmaf(32.0f, d, fmaf(0.03125f, f, b)) + m[7 * S];
}

__device__ __forceinline__ void split2_f16(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// ------------------------------------------------------------------------------------------
struct WinoInParams {
  const float* src1; int c1;
  const float* src2; int c2;
  int B, H, W, C, groups, cpg, th, tw;   // H x W: the conv's map
  int sH, sW;                // the sources' map: H x W, or 2H(+1) x 2W(+1) for the 2x2-pooled form (down2)
  int64_t Mtot;              // rows of the V planes: B*th*tw tiles (F(6,3): padded to a multiple of 16, zero rows)
  const float* mean; const float* rstd; const float* gamma; const float* beta;
  const float* fscale; const float* fshift; int64_t fstride;
  int silu;
  __half* v_hi; __half* v_lo;
  __nv_bfloat16* raw_hi; __nv_bfloat16* raw_lo;
  __nv_bfloat16* act_hi; __nv_bfloat16* act_lo;   // optional split-bf16 planes of the ACTIVATED tensor (wgrad operand)
  unsigned long long* fault;   // F(6,3): device fault word, set when a V value is not a finite fp16 number
};

constexpr unsigned long long WINO6_RANGE_FAULT = 0xC0000000ull;   // | C: channel count of the failing launch

// One CTA per (sample b, tile row ty, chunk of 256*VEC channels): every thread owns VEC channels and walks the tile
// row left to right, keeping the two activated pixel columns it shares with the next tile in registers (24 instead of
// 36 loads + activations per tile).  A warp reads 128*VEC contiguous bytes per pixel and writes 64*VEC contiguous
// bytes per (position, tile) and plane.
template <int VEC>
__global__ void __launch_bounds__(256)
wino_input_kernel(const WinoInParams p) {
  const int b = blockIdx.x / p.th, ty = blockIdx.x % p.th;
  const int c = (blockIdx.y * 256 + threadIdx.x) * VEC;
  if (c >= p.C) return;
  // GroupNorm affine x FiLM of this sample for this thread's channels
  float sc[VEC], sh[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) {
    const int g = (c + v) / p.cpg;
    const float s0 = p.rstd[b * p.groups + g] * p.gamma[c + v];
    const float h0 = p.beta[c + v] - p.mean[b * p.groups + g] * s0;
    float f1 = 1.0f, f0 = 0.0f;
    if (p.fscale) { f1 = 1.0f + p.fscale[(int64_t)b * p.fstride + c + v]; f0 = p.fshift[(int64_t)b * p.fstride + c + v]; }
    sc[v] = s0 * f1;
    sh[v] = fmaf(h0, f1, f0);
  }
  const float* base;
  int cs, cc;
  if (c < p.c1) { base = p.src1; cs = p.c1; cc = c; } else { base = p.src2; cs = p.c2; cc = c - p.c1; }
  const int y0 = 4 * ty - 1;
  float act[VEC][36];      // activated 6x6 tile, [row][col]
  // load + activate columns [j0, 6) of the tile whose first input column is x0
  auto fill = [&](int x0, int j0) {
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      const int iy = y0 + i;
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        if (j < j0) continue;
        const int ix = x0 + j;
        const bool in = iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
        float x[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) x[v] = 0.f;
        if (in) {
          const float* ptr = base + (((int64_t)b * p.H + iy) * p.W + ix) * cs + cc;
          if (VEC == 2) { const float2 t = *reinterpret_cast<const float2*>(ptr); x[0] = t.x; x[VEC - 1] = t.y; }
          else x[0] = *ptr;
        }
        if (p.raw_hi && i >= 1 && i <= 4 && j >= 2) {
          // pixels this pass owns (tile interior rows; columns not seen by the previous tile): raw split-bf16 planes
          // for the 1x1 skip conv.  Column j >= 2 of tile tx is input column 4*tx+1.. : every pixel exactly once,
          // except input column 0 (j == 1 of tile 0), handled by j0 == 0 below.
          const int64_t off = (((int64_t)b * p.H + iy) * p.W + ix) * p.C + c;
          if (in) {
            if (VEC == 2) {
              uint32_t h, l;
              split2x(x[0], x[VEC - 1], h, l);
              *reinterpret_cast<uint32_t*>(p.raw_hi + off) = h;
              *reinterpret_cast<uint32_t*>(p.raw_lo + off) = l;
            } else {
              split_bf16(x[0], p.raw_hi[off], p.raw_lo[off]);
            }
          }
        } else if (p.raw_hi && i >= 1 && i <= 4 && j == 1 && j0 == 0 && in) {
          const int64_t off = (((int64_t)b * p.H + iy) * p.W + ix) * p.C + c;
          if (VEC == 2) {
            uint32_t h, l;
            split2x(x[0], x[VEC - 1], h, l);
            *reinterpret_cast<uint32_t*>(p.raw_hi + off) = h;
            *reinterpret_cast<uint32_t*>(p.raw_lo + off) = l;
          } else {
            split_bf16(x[0], p.raw_hi[off], p.raw_lo[off]);
          }
        }
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          float a = fmaf(x[v], sc[v], sh[v]);
          if (p.silu) a = __fdividef(a, 1.0f + __expf(-a));
          act[v][i * 6 + j] = in ? a : 0.f;       // the conv zero-pads the ACTIVATED tensor
        }
      }
    }
  };
  for (int tx = 0; tx < p.tw; ++tx) {
    if (tx == 0) fill(-1, 0);
    else {
      // columns 4, 5 of the previous tile are columns 0, 1 of this one
#pragma unroll
      for (int v = 0; v < VEC; ++v)
#pragma unroll
        for (int i = 0; i < 6; ++i) { act[v][i * 6] = act[v][i * 6 + 4]; act[v][i * 6 + 1] = act[v][i * 6 + 5]; }
      fill(4 * tx - 1, 2);
    }
    // V = B^T d B: columns, then rows (on a copy: `act` carries over to the next tile)
    float t[VEC][36];
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
#pragma unroll
      for (int q = 0; q < 36; ++q) t[v][q] = act[v][q];
#pragma unroll
      for (int j = 0; j < 6; ++j) wino_bt6<6>(t[v] + j);
#pragma unroll
      for (int i = 0; i < 6; ++i) wino_bt6<1>(t[v] + 6 * i);
    }
    const int64_t m = ((int64_t)b * p.th + ty) * p.tw + tx;
#pragma unroll
    for (int q = 0; q < 36; ++q) {
      const int64_t off = ((int64_t)q * p.Mtot + m) * p.C + c;
      if (VEC == 2) {
        uint32_t h, l;
        split2_f16(t[0][q], t[VEC - 1][q], h, l);
        *reinterpret_cast<uint32_t*>(p.v_hi + off) = h;
        *reinterpret_cast<uint32_t*>(p.v_lo + off) = l;
      } else {
        const __half h = __float2half_rn(t[0][q]);
        p.v_hi[off] = h;
        p.v_lo[off] = __float2half_rn(t[0][q] - __half2float(h));
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Shared-memory staged input transform (the default): one CTA per (sample b, tile row ty, 64-channel chunk) walks the
// tile row in segments of TX tiles.  Per segment: (1) cp.async stages the N x (T*TX+2) pixel x 64 channel input patch
// (N = T+2 rows; double buffered: the next segment's loads fly while this one is transformed -- the register variant
// above is bound by exposed load latency, ncu: 65 % long-scoreboard stalls, 29 % issue utilisation); (2) every pixel is
// activated ONCE in place (GroupNorm affine x FiLM, SiLU; out-of-image pixels become exact zeros = the conv padding
// of the activated tensor); (3) F(4,3): thread (tile, channel pair) reads its 6x6 tile with conflict-free 8-byte LDS,
// transforms, splits to fp16 hi/lo and stores (128 contiguous bytes per warp, position and plane).  F(6,3): thread
// (tile, channel) does the same for its 8x8 tile (64 floats of state, not 128: the kernel stays spill-free at 2 CTAs
// per SM), 64 contiguous bytes per warp, position and plane.
// POOL (F(6,3), the down-ResBlock's conv1): the conv's input is the 2x2 average of the ACTIVATED 2H x 2W sources
// (GroupNorm + SiLU, then the pool: the reference order).  Phase 2 reads the four source pixels of each patch pixel
// itself, activates each and stores their average; nothing is staged by cp.async (a full-resolution patch would not
// fit twice per CTA at 2 CTAs per SM).
template <int T>
struct WinoIn {
  static constexpr int N = T + 2;                    // input tile side
  static constexpr int CC = 64;                      // channels per CTA
  static constexpr int TX = T == 4 ? 8 : 4;          // tiles per segment: 256 threads in phase 3, 2 buffers x 2 CTAs/SM
  static constexpr int COLS = T * TX + 2;            // patch columns (>= 16: phases 1/2 step 16 pixels at a time)
  static constexpr int PATCH = N * COLS * CC;        // floats per buffer
  static constexpr size_t SMEM = 2 * (size_t)PATCH * sizeof(float);
};
static_assert(WinoIn<4>::SMEM == 2 * 6 * 34 * 64 * 4 && WinoIn<6>::SMEM * 2 <= 227 * 1024, "staged patch budget");

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(g) : "memory");
}

template <int T, bool POOL>
__global__ void __launch_bounds__(256, 2)
wino_input_smem_kernel(const WinoInParams p) {
  static_assert(!POOL || T == 6, "the pooled input form is F(6,3) only");
  using K = WinoIn<T>;
  constexpr int N = K::N, CC = K::CC, TX = K::TX, COLS = K::COLS;
  extern __shared__ __align__(16) float patch[];          // [2][N][COLS][CC]
  const int b = blockIdx.x / p.th, ty = blockIdx.x % p.th;
  const int cbase = blockIdx.y * CC;                       // first channel of this CTA (in the concatenation)
  const float* base;
  int cs, cc0;
  if (cbase < p.c1) { base = p.src1; cs = p.c1; cc0 = cbase; } else { base = p.src2; cs = p.c2; cc0 = cbase - p.c1; }
  const int y0 = T * ty - 1;
  const int tid = threadIdx.x;
  const int ch4 = tid & 15;                                // this thread's 4-channel group in phases 1/2
  const int pix0 = tid >> 4;                               // first patch pixel of this thread (stride 16 pixels)
  constexpr int NPIX = N * COLS;                           // pixels per patch

  if constexpr (T == 6) {
    // the GEMM's padding rows (tile count rounded up to 16): exact zeros, written by the CTAs of tile row 0
    if (blockIdx.x == 0) {
      const int64_t tiles = (int64_t)p.B * p.th * p.tw;
      const int npad = (int)(p.Mtot - tiles);
      for (int k = tid; k < N * N * npad * CC; k += 256) {
        const int c = k % CC, r = (k / CC) % npad, q = k / (CC * npad);
        const int64_t off = ((int64_t)q * p.Mtot + tiles + r) * p.C + cbase + c;
        p.v_hi[off] = __float2half_rn(0.f);
        p.v_lo[off] = __float2half_rn(0.f);
      }
    }
  }

  // GroupNorm affine x FiLM for the 4 channels this thread activates
  float sc[4], sh[4];
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    sc[v] = 1.0f; sh[v] = 0.0f;            // mean == nullptr: identity (the data-gradient conv transforms dY as is)
    if (p.mean) {
      const int c = cbase + ch4 * 4 + v;
      const int g = c / p.cpg;
      const float s0 = p.rstd[b * p.groups + g] * p.gamma[c];
      const float h0 = p.beta[c] - p.mean[b * p.groups + g] * s0;
      float f1 = 1.0f, f0 = 0.0f;
      if (p.fscale) { f1 = 1.0f + p.fscale[(int64_t)b * p.fstride + c]; f0 = p.fshift[(int64_t)b * p.fstride + c]; }
      sc[v] = s0 * f1;
      sh[v] = fmaf(h0, f1, f0);
    }
  }
  const int nseg = (p.tw + TX - 1) / TX;
  const uint32_t patch_s = (uint32_t)__cvta_generic_to_shared(patch);

  auto stage = [&](int seg, int buf) {
    if constexpr (!POOL) {
      const int x0 = T * TX * seg - 1;
      int i = 0, j = pix0;                                // pix0 < 16 <= COLS: row 0
      for (int px = pix0; px < NPIX; px += 16, j += 16) {
        if (j >= COLS) { j -= COLS; ++i; }
        const int iy = y0 + i, ix = x0 + j;
        if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W)
          cp_async16(patch_s + (uint32_t)(((buf * NPIX + px) * CC + ch4 * 4) * 4),
                     base + (((int64_t)b * p.H + iy) * p.W + ix) * cs + cc0 + ch4 * 4);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  auto activate = [&](const float4 x) {
    float4 a = make_float4(fmaf(x.x, sc[0], sh[0]), fmaf(x.y, sc[1], sh[1]), fmaf(x.z, sc[2], sh[2]),
                           fmaf(x.w, sc[3], sh[3]));
    if (p.silu) {
      a.x = __fdividef(a.x, 1.0f + __expf(-a.x)); a.y = __fdividef(a.y, 1.0f + __expf(-a.y));
      a.z = __fdividef(a.z, 1.0f + __expf(-a.z)); a.w = __fdividef(a.w, 1.0f + __expf(-a.w));
    }
    return a;
  };

  stage(0, 0);
  for (int seg = 0; seg < nseg; ++seg) {
    const int buf = seg & 1;
    if (seg + 1 < nseg) {
      stage(seg + 1, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    float* pb = patch + buf * K::PATCH;
    const int x0 = T * TX * seg - 1;
    // ---- phase 2: activate every staged pixel once, in place ------------------------------------------------
    int i = 0, j = pix0;
    for (int px = pix0; px < NPIX; px += 16, j += 16) {
      if (j >= COLS) { j -= COLS; ++i; }
      const int iy = y0 + i, ix = x0 + j;
      float4* q = reinterpret_cast<float4*>(pb + px * CC + ch4 * 4);
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      if (POOL && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
        const float* s = base + (((int64_t)b * p.sH + 2 * iy) * p.sW + 2 * ix) * cs + cc0 + ch4 * 4;
        const int64_t rs = (int64_t)p.sW * cs;
        const float4 a0 = activate(__ldg(reinterpret_cast<const float4*>(s)));
        const float4 a1 = activate(__ldg(reinterpret_cast<const float4*>(s + cs)));
        const float4 a2 = activate(__ldg(reinterpret_cast<const float4*>(s + rs)));
        const float4 a3 = activate(__ldg(reinterpret_cast<const float4*>(s + rs + cs)));
        a = make_float4(0.25f * (((a0.x + a1.x) + a2.x) + a3.x), 0.25f * (((a0.y + a1.y) + a2.y) + a3.y),
                        0.25f * (((a0.z + a1.z) + a2.z) + a3.z), 0.25f * (((a0.w + a1.w) + a2.w) + a3.w));
      } else if (!POOL && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
        const float4 x = *q;
        if (p.raw_hi && i >= 1 && i <= T && j >= 1 && j <= T * TX) {
          // pixels this segment owns: raw split-bf16 planes for the 1x1 skip conv
          uint2 h, l;
          split4(x, h, l);
          const int64_t off = (((int64_t)b * p.H + iy) * p.W + ix) * p.C + cbase + ch4 * 4;
          *reinterpret_cast<uint2*>(p.raw_hi + off) = h;
          *reinterpret_cast<uint2*>(p.raw_lo + off) = l;
        }
        a = activate(x);
        if (p.act_hi && i >= 1 && i <= T && j >= 1 && j <= T * TX) {
          // training: the activated tensor's split-bf16 planes are the weight-gradient GEMM's operand
          uint2 h, l;
          split4(a, h, l);
          const int64_t off = (((int64_t)b * p.H + iy) * p.W + ix) * p.C + cbase + ch4 * 4;
          *reinterpret_cast<uint2*>(p.act_hi + off) = h;
          *reinterpret_cast<uint2*>(p.act_lo + off) = l;
        }
      }
      *q = a;                                              // out of the image: exact zero (padding of the activation)
    }
    __syncthreads();
    // ---- phase 3: one (tile, channel pair) [F(4,3)] or (tile, channel) [F(6,3)] per thread ----------------------
    const int64_t plane = p.Mtot * p.C;
    if constexpr (T == 4) {
      const int txl = tid >> 5, c0 = (tid & 31) * 2;
      const int tx = TX * seg + txl;
      if (tx < p.tw) {
        float t0[36], t1[36];
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
          for (int j = 0; j < 6; ++j) {
            const float2 v = *reinterpret_cast<const float2*>(pb + ((i * COLS + 4 * txl + j) * CC + c0));
            t0[i * 6 + j] = v.x;
            t1[i * 6 + j] = v.y;
          }
#pragma unroll
        for (int j = 0; j < 6; ++j) { wino_bt6<6>(t0 + j); wino_bt6<6>(t1 + j); }
#pragma unroll
        for (int i = 0; i < 6; ++i) { wino_bt6<1>(t0 + 6 * i); wino_bt6<1>(t1 + 6 * i); }
        const int64_t m = ((int64_t)b * p.th + ty) * p.tw + tx;
        __half* ph = p.v_hi + m * p.C + cbase + c0;
        __half* pl = p.v_lo + m * p.C + cbase + c0;
#pragma unroll
        for (int q = 0; q < 36; ++q) {
          uint32_t h, l;
          split2_f16(t0[q], t1[q], h, l);
          *reinterpret_cast<uint32_t*>(ph) = h;
          *reinterpret_cast<uint32_t*>(pl) = l;
          ph += plane;
          pl += plane;
        }
      }
    } else {
      const int txl = tid >> 6, c = tid & 63;
      const int tx = TX * seg + txl;
      if (tx < p.tw) {
        float t[64];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) t[i * 8 + j] = pb[(i * COLS + 6 * txl + j) * CC + c];
#pragma unroll
        for (int j = 0; j < 8; ++j) wino_bt8<8>(t + j);
#pragma unroll
        for (int i = 0; i < 8; ++i) wino_bt8<1>(t + 8 * i);
        const int64_t m = ((int64_t)b * p.th + ty) * p.tw + tx;
        __half* ph = p.v_hi + m * p.C + cbase + c;
        __half* pl = p.v_lo + m * p.C + cbase + c;
        // |V| <= 225 max|act|: past max|act| ~ 291 the fp16 planes overflow -- reported, never silent
        bool finite = true;
#pragma unroll
        for (int q = 0; q < 64; ++q) {
          const __half h = __float2half_rn(t[q]);
          finite &= fabsf(t[q]) < 65520.0f;              // rounds to at most 65504 (false for NaN too)
          *ph = h;
          *pl = __float2half_rn(t[q] - __half2float(h));
          ph += plane;
          pl += plane;
        }
        if (!finite) atomicExch(p.fault, WINO6_RANGE_FAULT | (unsigned)(p.C & 0xFFFFFFF));
      }
    }
    __syncthreads();          // all reads of this buffer done before the cp.async of segment seg+2 lands in it
  }
}

// ------------------------------------------------------------------------------------------
struct WinoOutParams {
  const float* m; int64_t Mtot;
  const float* inv_wscale;   // 1/s of the weight planes (device scalar written by bbdm_wino_pack_weight), or nullptr: 2^-8
  int B, H, W, Cout, th, tw;
  const float* bias;
  const float* residual; int res_mode;
  float* out;
  float* stats;      // [B*th][Cout][2] or nullptr
};

// One CTA per (64-channel group, tile row ty, sample b): 32 channel pairs x 8 tile-column lanes.
// RES is a template parameter: the residual values of a tile are fetched as ONE batch of independent loads right after
// the 36 loads of M (a load placed between the stores of the result cannot be moved ahead of them by the compiler --
// `out` may alias `residual` -- and serialises 16 load -> add -> store round trips per tile: the first version ran the
// "+ skip" layers 2.5x slower than the plain ones, profiles/r02_conv_layers_cfg2_closing.md), and the variant without a
// residual keeps its register budget.
// One output tile (4x4 pixels) of one channel pair.  __host__ __device__: tools/host_check_wino_output.cu runs exactly
// this code on the CPU against a direct fp64 evaluation (tests/test_wino_output_host.py).
template <int RES>
__host__ __device__ __forceinline__ void wino_output_tile(const WinoOutParams& p, int b, int ty, int tx, int c, float2 bv,
                                                          float inv, float& sum0, float& sum1, float& sq0, float& sq1) {
  const int64_t m = ((int64_t)b * p.th + ty) * p.tw + tx;
  float mx[36], my[36];
#pragma unroll
  for (int q = 0; q < 36; ++q) {
    const float2 v = *reinterpret_cast<const float2*>(p.m + ((int64_t)q * p.Mtot + m) * p.Cout + c);
    mx[q] = v.x; my[q] = v.y;
  }
  // residual of the 4x4 output pixels (same / nearest-up / 2x2-average addressed)
  constexpr int NRES = RES == BBDM_RES_NONE ? 1 : (RES == BBDM_RES_UP2 ? 4 : 16);
  float2 rs[NRES];
  if constexpr (RES == BBDM_RES_SAME) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        rs[i * 4 + j] = *reinterpret_cast<const float2*>(
            p.residual + (((int64_t)b * p.H + 4 * ty + i) * p.W + 4 * tx + j) * p.Cout + c);
  } else if constexpr (RES == BBDM_RES_UP2) {
    // output pixels (4ty+i, 4tx+j) read source pixel (2ty + i/2, 2tx + j/2): 2x2 distinct values per tile
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j)
        rs[i * 2 + j] = *reinterpret_cast<const float2*>(
            p.residual + (((int64_t)b * (p.H >> 1) + 2 * ty + i) * (p.W >> 1) + 2 * tx + j) * p.Cout + c);
  } else if constexpr (RES == BBDM_RES_DOWN2) {
    const int64_t W2 = (int64_t)p.W * 2;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float* rp = p.residual + (((int64_t)b * p.H * 2 + (4 * ty + i) * 2) * W2 + (4 * tx + j) * 2) * p.Cout + c;
        const float2 t0 = *reinterpret_cast<const float2*>(rp), t1 = *reinterpret_cast<const float2*>(rp + p.Cout);
        const float2 t2 = *reinterpret_cast<const float2*>(rp + W2 * p.Cout);
        const float2 t3 = *reinterpret_cast<const float2*>(rp + (W2 + 1) * p.Cout);
        rs[i * 4 + j] = make_float2(0.25f * (((t0.x + t1.x) + t2.x) + t3.x), 0.25f * (((t0.y + t1.y) + t2.y) + t3.y));
      }
  }
  // Y = A^T M A: columns (6 -> 4 rows), then rows (6 -> 4 columns)
  float tx4[24], ty4[24], yx[16], yy[16];
#pragma unroll
  for (int j = 0; j < 6; ++j) { wino_at6<6, 6>(mx + j, tx4 + j); wino_at6<6, 6>(my + j, ty4 + j); }
#pragma unroll
  for (int i = 0; i < 4; ++i) { wino_at6<1, 1>(tx4 + 6 * i, yx + 4 * i); wino_at6<1, 1>(ty4 + 6 * i, yy + 4 * i); }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int hh = 4 * ty + i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ww = 4 * tx + j;
      float r0 = fmaf(yx[i * 4 + j], inv, bv.x), r1 = fmaf(yy[i * 4 + j], inv, bv.y);
      if constexpr (RES == BBDM_RES_SAME || RES == BBDM_RES_DOWN2) {
        r0 += rs[i * 4 + j].x; r1 += rs[i * 4 + j].y;
      } else if constexpr (RES == BBDM_RES_UP2) {
        r0 += rs[(i >> 1) * 2 + (j >> 1)].x; r1 += rs[(i >> 1) * 2 + (j >> 1)].y;
      }
      *reinterpret_cast<float2*>(p.out + (((int64_t)b * p.H + hh) * p.W + ww) * p.Cout + c) = make_float2(r0, r1);
      sum0 += r0; sum1 += r1;
      sq0 = fmaf(r0, r0, sq0); sq1 = fmaf(r1, r1, sq1);
    }
  }
}

template <int RES>
__global__ void __launch_bounds__(256, 2)
wino_output_kernel(const WinoOutParams p) {
  __shared__ float red[8][64][2];
  const int cg = blockIdx.x, ty = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, tl = threadIdx.x >> 5;
  const int c = cg * 64 + lane * 2;
  float2 bv = make_float2(0.f, 0.f);
  if (p.bias) bv = *reinterpret_cast<const float2*>(p.bias + c);
  const float inv = p.inv_wscale ? __ldg(p.inv_wscale) : 1.0f / WINO_WSCALE_FIXED;
  float sum0 = 0.f, sum1 = 0.f, sq0 = 0.f, sq1 = 0.f;
  for (int tx = tl; tx < p.tw; tx += 8) wino_output_tile<RES>(p, b, ty, tx, c, bv, inv, sum0, sum1, sq0, sq1);
  if (p.stats) {
    // fixed-order combine of the 8 tile-column lanes => deterministic partial sums
    red[tl][lane * 2][0] = sum0; red[tl][lane * 2][1] = sq0;
    red[tl][lane * 2 + 1][0] = sum1; red[tl][lane * 2 + 1][1] = sq1;
    __syncthreads();
    if (threadIdx.x < 64) {
      float a = 0.f, q = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) { a += red[k][threadIdx.x][0]; q += red[k][threadIdx.x][1]; }
      const int64_t prow = (int64_t)b * p.th + ty;
      *reinterpret_cast<float2*>(p.stats + (prow * p.Cout + cg * 64 + threadIdx.x) * 2) = make_float2(a, q);
    }
  }
}

// F(6,3) output form of the phase-stacked nearest-2x conv (used as the RES template value, no residual): M holds 4*Cout
// channels c' = phase * Cout + co on the LOW-RES tile grid of an H x W map, and pixel (i, j) of tile (ty, tx) in phase
// (a, b) = (phase >> 1, phase & 1) is output pixel (2(6ty+i)+a, 2(6tx+j)+b), channel co, of the [B, 2H, 2W, Cout] result.
constexpr int WINO6_UP_PHASES = 4;

// F(6x6,3x3): one output tile (6x6 pixels) of ONE channel (64 M values instead of 2 x 36: one channel per thread keeps
// the F(4,3) kernel's register budget).  Tiles run over ceil(H/6) x ceil(W/6): pixels, residual reads and partial sums
// past H or W are masked.  c is the channel of M (WINO6_UP_PHASES: phase * Cout + co); bv the bias of its output
// channel.  __host__ __device__: tools/host_check_wino6_output.cu and tools/host_check_wino6_up2_output.cu run it on
// the CPU.
template <int RES>
__host__ __device__ __forceinline__ void wino6_output_tile(const WinoOutParams& p, int b, int ty, int tx, int c, float bv,
                                                           float inv, float& sum, float& sq) {
  constexpr bool UP = RES == WINO6_UP_PHASES;
  const int64_t m = ((int64_t)b * p.th + ty) * p.tw + tx;
  const int ldm = UP ? 4 * p.Cout : p.Cout;
  float mm[64];
#pragma unroll
  for (int q = 0; q < 64; ++q) mm[q] = p.m[((int64_t)q * p.Mtot + m) * ldm + c];
  // Y = A^T M A: columns (8 -> 6 rows), then rows (8 -> 6 columns)
  float t6[48], y[36];
#pragma unroll
  for (int j = 0; j < 8; ++j) wino_at8<8, 8>(mm + j, t6 + j);
#pragma unroll
  for (int i = 0; i < 6; ++i) wino_at8<1, 1>(t6 + 8 * i, y + 6 * i);
  const int h0 = 6 * ty, w0 = 6 * tx;
  float rup[RES == BBDM_RES_UP2 ? 9 : 1];
  if constexpr (RES == BBDM_RES_UP2) {
    // output pixels (6ty+i, 6tx+j) read source pixel (3ty + i/2, 3tx + j/2): 3x3 distinct values per tile
    const int H2 = p.H >> 1, W2 = p.W >> 1;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j)
        rup[i * 3 + j] = 3 * ty + i < H2 && 3 * tx + j < W2
                             ? p.residual[(((int64_t)b * H2 + 3 * ty + i) * W2 + 3 * tx + j) * p.Cout + c] : 0.f;
  }
  // three output rows at a time: their residual values (same / 2x2-average addressed) are fetched as one batch ahead
  // of their stores
  int co = c;
  int64_t pix0 = ((int64_t)b * p.H + h0) * p.W + w0;                // first pixel of the tile
  int64_t rstep = p.W, cstep = 1;                                   // output pixels per tile row / column
  if constexpr (UP) {
    const int ph = c / p.Cout;
    co = c - ph * p.Cout;
    pix0 = ((int64_t)b * 2 * p.H + 2 * h0 + (ph >> 1)) * (2 * p.W) + 2 * w0 + (ph & 1);
    rstep = 4 * (int64_t)p.W;
    cstep = 2;
  }
#pragma unroll
  for (int i0 = 0; i0 < 6; i0 += 3) {
    float rs[18];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        rs[i * 6 + j] = 0.f;
        if (h0 + i0 + i >= p.H || w0 + j >= p.W) continue;
        if constexpr (RES == BBDM_RES_SAME) {
          rs[i * 6 + j] = p.residual[(pix0 + (int64_t)(i0 + i) * p.W + j) * p.Cout + c];
        } else if constexpr (RES == BBDM_RES_DOWN2) {
          const int64_t W2 = (int64_t)p.W * 2;
          const float* rp = p.residual + (((int64_t)b * p.H * 2 + (h0 + i0 + i) * 2) * W2 + (w0 + j) * 2) * p.Cout + c;
          rs[i * 6 + j] = 0.25f * (((rp[0] + rp[p.Cout]) + rp[W2 * p.Cout]) + rp[(W2 + 1) * p.Cout]);
        }
      }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        if (h0 + i0 + i >= p.H || w0 + j >= p.W) continue;
        float r = fmaf(y[(i0 + i) * 6 + j], inv, bv);
        if constexpr (RES == BBDM_RES_SAME || RES == BBDM_RES_DOWN2) r += rs[i * 6 + j];
        else if constexpr (RES == BBDM_RES_UP2) r += rup[((i0 + i) >> 1) * 3 + (j >> 1)];
        p.out[(pix0 + (i0 + i) * rstep + j * cstep) * p.Cout + co] = r;
        sum += r;
        sq = fmaf(r, r, sq);
      }
  }
}

// One CTA per (64-channel group, tile row ty, sample b): 64 channels x 4 tile-column lanes (a warp reads 128
// contiguous bytes of M per position).  WINO6_UP_PHASES: 4*Cout/64 channel groups of M, each inside one phase, and one
// partial-sum row per (tile row, phase).
// The same-addressed and 2x2-averaged residual modes need more than 128 registers (ptxas: spills at 2 CTAs per SM).
template <int RES>
__global__ void __launch_bounds__(256, RES == BBDM_RES_SAME || RES == BBDM_RES_DOWN2 ? 1 : 2)
wino6_output_kernel(const WinoOutParams p) {
  __shared__ float red[4][64][2];
  const int cg = blockIdx.x, ty = blockIdx.y, b = blockIdx.z;
  const int cl = threadIdx.x & 63, tl = threadIdx.x >> 6;
  const int c = cg * 64 + cl;
  const int ph = RES == WINO6_UP_PHASES ? cg * 64 / p.Cout : 0;
  const int co0 = cg * 64 - ph * p.Cout;                            // first output channel of the group
  const float bv = p.bias ? p.bias[co0 + cl] : 0.f;
  const float inv = p.inv_wscale ? __ldg(p.inv_wscale) : 1.0f / WINO_WSCALE_FIXED;
  float sum = 0.f, sq = 0.f;
  for (int tx = tl; tx < p.tw; tx += 4) wino6_output_tile<RES>(p, b, ty, tx, c, bv, inv, sum, sq);
  if (p.stats) {
    // fixed-order combine of the 4 tile-column lanes => deterministic partial sums
    red[tl][cl][0] = sum; red[tl][cl][1] = sq;
    __syncthreads();
    if (threadIdx.x < 64) {
      float a = 0.f, q = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) { a += red[k][threadIdx.x][0]; q += red[k][threadIdx.x][1]; }
      const int64_t prow = RES == WINO6_UP_PHASES ? ((int64_t)b * p.th + ty) * 4 + ph : (int64_t)b * p.th + ty;
      *reinterpret_cast<float2*>(p.stats + (prow * p.Cout + co0 + threadIdx.x) * 2) = make_float2(a, q);
    }
  }
}

// ------------------------------------------------------------------------------------------
// max|w| over the whole tensor: atomicMax on the bit patterns of the non-negative floats |w| (their integer order is
// their value order), so the result does not depend on the order the blocks run in.  *wmax must be zeroed first.
__global__ void __launch_bounds__(256)
wino_wmax_kernel(const float* __restrict__ w, int64_t n, uint32_t* __restrict__ wmax) {
  uint32_t m = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    m = max(m, __float_as_uint(fabsf(w[i])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(wmax, m);
}

// *inv = 1/s, in place over the max|w| bits it is computed from (after the packing kernel has read them)
__global__ void wino_wscale_store_kernel(float* inv) {
  *inv = 1.0f / wino_wscale(__float_as_uint(*inv));
}

// G (N x 3) applied to g0..g2 in fp64 -> u[0..N-1].  F(4,3): absolute row sums <= 1; F(6,3): <= 56/45, so
// |s U| <= (56/45)^2 2^14 < 65504 with the same power-of-two scale.
template <int T>
__device__ __forceinline__ void wino_g(double g0, double g1, double g2, double* u) {
  if constexpr (T == 4) {
    u[0] = g0 / 4.0;
    u[1] = -(g0 + g1 + g2) / 6.0;
    u[2] = -(g0 - g1 + g2) / 6.0;
    u[3] = g0 / 24.0 + g1 / 12.0 + g2 / 6.0;
    u[4] = g0 / 24.0 - g1 / 12.0 + g2 / 6.0;
    u[5] = g2;
  } else {
    u[0] = g0;
    u[1] = -2.0 * (g0 + g1 + g2) / 9.0;
    u[2] = -2.0 * (g0 - g1 + g2) / 9.0;
    u[3] = g0 / 90.0 + g1 / 45.0 + 2.0 * g2 / 45.0;
    u[4] = g0 / 90.0 - g1 / 45.0 + 2.0 * g2 / 45.0;
    u[5] = 32.0 * g0 / 45.0 + 16.0 * g1 / 45.0 + 8.0 * g2 / 45.0;
    u[6] = 32.0 * g0 / 45.0 - 16.0 * g1 / 45.0 + 8.0 * g2 / 45.0;
    u[7] = g2;
  }
}

// U[q][co][ci] = s * (G g G^T)[q] in fp64, split into fp16 planes ((T+2)^2 positions q).  One thread per (co, ci).
// dgrad != 0: the data-gradient conv's weights instead -- kernel flipped, channels swapped: U[q][ci][co] from
// g'[ky][kx] = w[co][ci][2-ky][2-kx] (threads run over co fastest so the stores stay coalesced).
template <int T>
__global__ void __launch_bounds__(256)
wino_weight_kernel(const float* __restrict__ w, int Cout, int Cin, int dgrad, const uint32_t* __restrict__ wmax,
                   __half* __restrict__ u_hi, __half* __restrict__ u_lo) {
  constexpr int N = T + 2;
  const int64_t n = (int64_t)Cout * Cin;
  const double s = wmax ? (double)wino_wscale(*wmax) : (double)WINO_WSCALE_FIXED;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * blockDim.x) {
    double g[3][3], t[N][3];
    int64_t src = idx;
    if (dgrad) { const int64_t ci = idx / Cout, co = idx - ci * Cout; src = co * Cin + ci; }
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const int k = dgrad ? 8 - i : i;
      g[i / 3][i % 3] = (double)w[src * 9 + k];
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      double u[N];
      wino_g<T>(g[0][j], g[1][j], g[2][j], u);
#pragma unroll
      for (int i = 0; i < N; ++i) t[i][j] = u[i];
    }
#pragma unroll
    for (int i = 0; i < N; ++i) {
      double u[N];
      wino_g<T>(t[i][0], t[i][1], t[i][2], u);
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const float v = (float)(u[j] * s);
        const __half h = __float2half_rn(v);
        const __half l = __float2half_rn(v - __half2float(h));
        const int64_t off = (int64_t)(i * N + j) * n + idx;
        u_hi[off] = h;
        u_lo[off] = l;
      }
    }
  }
}

}  // namespace bbdm

using namespace bbdm;

namespace {

// Tile grid of a T x T output tiling.  F(4,3): H, W multiples of 4, tiles_total = B*th*tw.  F(6,3): ceil(H/6) x
// ceil(W/6) tiles (edge tiles past H or W read zero padding and store nothing there), tiles_total padded with zero V
// rows to the GEMM's multiple of 16 and to at least one 128-row M block, so that eligibility never depends on the
// batch size (a 64x64 image has 121 tiles).  The GEMM views the tile axis as rows of 16 with 128-tile M blocks inside
// one transform position.
template <int T>
int wino_geometry_t(int B, int H, int W, int* tiles_h, int* tiles_w, int64_t* tiles_total, int* eligible) {
  BBDM_REQUIRE(B > 0 && H > 0 && W > 0, "wino_geometry: bad shape");
  const int th = T == 4 ? H / 4 : (H + 5) / 6, tw = T == 4 ? W / 4 : (W + 5) / 6;
  int64_t mtot = (int64_t)B * th * tw;
  if (T == 6) mtot = mtot < 128 ? 128 : (mtot + 15) / 16 * 16;
  if (tiles_h) *tiles_h = th;
  if (tiles_w) *tiles_w = tw;
  if (tiles_total) *tiles_total = mtot;
  const bool aligned = T == 6 || (H % 4 == 0 && W % 4 == 0);
  if (eligible) *eligible = (aligned && mtot % 16 == 0 && mtot >= 128) ? 1 : 0;
  return BBDM_OK;
}

template <int T, bool POOL>
int launch_wino_input_smem(const WinoInParams& p, dim3 grid, void* stream) {
  static DeviceOnce configured;
  if (configured.need()) {
    BBDM_CUDA_CHECK(cudaFuncSetAttribute(wino_input_smem_kernel<T, POOL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)WinoIn<T>::SMEM));
    configured.mark();
  }
  wino_input_smem_kernel<T, POOL><<<grid, 256, WinoIn<T>::SMEM, (cudaStream_t)stream>>>(p);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

template <int T>
int wino_input_t(const BbdmWinoInputArgs* a, void* stream) {
  BBDM_REQUIRE(a && a->src1 && a->v_hi && a->v_lo, "wino_input: null args");
  WinoInParams p;
  p.src1 = a->src1; p.c1 = a->c1;
  p.src2 = a->src2; p.c2 = a->src2 ? a->c2 : 0;
  p.B = a->B; p.H = a->H; p.W = a->W;
  p.C = p.c1 + p.c2;
  p.groups = a->groups;
  if (T == 4)
    BBDM_REQUIRE(p.B > 0 && p.H > 0 && p.W > 0 && p.H % 4 == 0 && p.W % 4 == 0, "wino_input: H, W must be multiples of 4");
  else
    BBDM_REQUIRE(p.B > 0 && p.H > 0 && p.W > 0, "wino6_input: bad shape");
  BBDM_REQUIRE(p.c1 % 2 == 0 && p.c2 % 2 == 0 && p.C > 0, "wino_input: channel counts must be even");
  if (a->mean) {
    BBDM_REQUIRE(a->rstd && a->gamma && a->beta && p.groups > 0 && p.C % p.groups == 0, "wino_input: incomplete GroupNorm args");
  } else {
    BBDM_REQUIRE(!a->silu && !a->film_scale, "wino_input: identity mode (mean == NULL) takes no activation / FiLM");
    if (p.groups <= 0) p.groups = 1;
  }
  BBDM_REQUIRE((a->act_hi == nullptr) == (a->act_lo == nullptr), "wino_input: act hi/lo must come in pairs");
  BBDM_REQUIRE((a->film_scale == nullptr) == (a->film_shift == nullptr), "wino_input: film scale/shift mismatch");
  BBDM_REQUIRE((a->raw_hi == nullptr) == (a->raw_lo == nullptr), "wino_input: raw hi/lo must come in pairs");
  p.cpg = p.C / p.groups;
  p.sH = p.H; p.sW = p.W;
  if (a->down2) {
    BBDM_REQUIRE(T == 6 && !a->raw_hi && !a->act_hi && p.H >= 2 && p.W >= 2,
                 "wino_input: down2 is an F(6,3) form without raw / act planes (H, W >= 2)");
    p.H /= 2; p.W /= 2;
  }
  wino_geometry_t<T>(p.B, p.H, p.W, &p.th, &p.tw, &p.Mtot, nullptr);
  p.mean = a->mean; p.rstd = a->rstd; p.gamma = a->gamma; p.beta = a->beta;
  p.fscale = a->film_scale; p.fshift = a->film_shift; p.fstride = a->film_stride;
  p.silu = a->silu;
  p.v_hi = (__half*)a->v_hi; p.v_lo = (__half*)a->v_lo;
  p.raw_hi = (__nv_bfloat16*)a->raw_hi; p.raw_lo = (__nv_bfloat16*)a->raw_lo;
  p.act_hi = (__nv_bfloat16*)a->act_hi; p.act_lo = (__nv_bfloat16*)a->act_lo;
  p.fault = nullptr;
  if (T == 6) {
    p.fault = device_fault_ptr();
    BBDM_REQUIRE(p.fault != nullptr, "wino6_input: device fault word unavailable");
  }
  const bool smem_only = a->mean == nullptr || a->act_hi != nullptr;      // features only the staged kernel has
  const int64_t ctas = (int64_t)p.B * p.th;
  BBDM_REQUIRE(ctas < (1ll << 31), "wino_input: too many tile rows");
  constexpr int CC = WinoIn<T>::CC;
  // default: the shared-memory staged kernel (needs 64-channel chunks inside one source tensor);
  // BBDM_WINO_IN_VEC=1|2 selects the register-only F(4,3) variant with 1 or 2 channels per thread (fallback / A-B
  // switch).  F(6,3) has the staged kernel only.
  static int vec = -1;
  if (vec < 0) { const char* e = getenv("BBDM_WINO_IN_VEC"); vec = e ? (atoi(e) == 2 ? 2 : 1) : 0; }
  if ((T == 6 || vec == 0) && p.c1 % CC == 0 && p.c2 % CC == 0) {
    const dim3 grid((unsigned)ctas, p.C / CC);
    if constexpr (T == 6) {
      if (a->down2) return launch_wino_input_smem<T, true>(p, grid, stream);
    }
    return launch_wino_input_smem<T, false>(p, grid, stream);
  } else if (T == 6) {
    BBDM_REQUIRE(false, "wino6_input: channel counts must be multiples of 64");
  } else if (smem_only) {
    BBDM_REQUIRE(false, "wino_input: identity mode / act planes need channel counts that are multiples of 64");
  } else if (vec == 2 || (vec == 0 && p.c1 % 2 == 0 && p.c2 % 2 == 0)) {
    dim3 grid((unsigned)ctas, (p.C / 2 + 255) / 256);
    wino_input_kernel<2><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  } else {
    dim3 grid((unsigned)ctas, (p.C + 255) / 256);
    wino_input_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  }
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

template <int T>
int wino_output_t(const BbdmWinoOutputArgs* a, void* stream) {
  BBDM_REQUIRE(a && a->m && a->out, "wino_output: null args");
  WinoOutParams p;
  p.m = a->m; p.inv_wscale = a->inv_wscale;
  p.B = a->B; p.H = a->H; p.W = a->W; p.Cout = a->Cout;
  if (T == 4)
    BBDM_REQUIRE(p.B > 0 && p.B <= 65535 && p.H > 0 && p.W > 0 && p.H % 4 == 0 && p.W % 4 == 0,
                 "wino_output: H, W must be multiples of 4 (B <= 65535)");
  else
    BBDM_REQUIRE(p.B > 0 && p.B <= 65535 && p.H > 0 && p.W > 0, "wino6_output: bad shape (B <= 65535)");
  BBDM_REQUIRE(p.Cout > 0 && p.Cout % 64 == 0, "wino_output: Cout %% 64 != 0");
  BBDM_REQUIRE(a->res_mode >= 0 && a->res_mode <= 3 && (a->res_mode == 0 || a->residual), "wino_output: bad residual");
  if (a->res_mode == BBDM_RES_UP2) BBDM_REQUIRE(p.H % 2 == 0 && p.W % 2 == 0, "wino_output: RES_UP2 needs even H, W");
  BBDM_REQUIRE(!a->up2_phases || (T == 6 && a->res_mode == BBDM_RES_NONE),
               "wino_output: up2_phases is an F(6,3) form without a residual");
  wino_geometry_t<T>(p.B, p.H, p.W, &p.th, &p.tw, &p.Mtot, nullptr);
  BBDM_REQUIRE(p.th <= 65535, "wino_output: too many tile rows");
  p.bias = a->bias; p.residual = a->residual; p.res_mode = a->res_mode;
  p.out = a->out; p.stats = a->stats_partial;
  dim3 grid(p.Cout / 64 * (a->up2_phases ? 4 : 1), p.th, p.B);
  cudaStream_t st = (cudaStream_t)stream;
  if (a->up2_phases) {
    wino6_output_kernel<WINO6_UP_PHASES><<<grid, 256, 0, st>>>(p);
  } else if constexpr (T == 4) {
    switch (p.res_mode) {
      case BBDM_RES_SAME: wino_output_kernel<BBDM_RES_SAME><<<grid, 256, 0, st>>>(p); break;
      case BBDM_RES_UP2: wino_output_kernel<BBDM_RES_UP2><<<grid, 256, 0, st>>>(p); break;
      case BBDM_RES_DOWN2: wino_output_kernel<BBDM_RES_DOWN2><<<grid, 256, 0, st>>>(p); break;
      default: wino_output_kernel<BBDM_RES_NONE><<<grid, 256, 0, st>>>(p); break;
    }
  } else {
    switch (p.res_mode) {
      case BBDM_RES_SAME: wino6_output_kernel<BBDM_RES_SAME><<<grid, 256, 0, st>>>(p); break;
      case BBDM_RES_UP2: wino6_output_kernel<BBDM_RES_UP2><<<grid, 256, 0, st>>>(p); break;
      case BBDM_RES_DOWN2: wino6_output_kernel<BBDM_RES_DOWN2><<<grid, 256, 0, st>>>(p); break;
      default: wino6_output_kernel<BBDM_RES_NONE><<<grid, 256, 0, st>>>(p); break;
    }
  }
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

template <int T>
int wino_pack_weight_t(const float* w, int Cout, int Cin, int dgrad, void* u_hi, void* u_lo, float* inv_wscale,
                       void* stream) {
  BBDM_REQUIRE(w && u_hi && u_lo && Cout > 0 && Cin > 0, "wino_pack_weight: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = (int64_t)Cout * Cin;
  // inv_wscale holds max|w| (as bits) until the packing kernel has read it, then 1/s.  Without it: the fixed 2^8.
  uint32_t* wmax = reinterpret_cast<uint32_t*>(inv_wscale);
  if (wmax) {
    BBDM_CUDA_CHECK(cudaMemsetAsync(wmax, 0, sizeof(uint32_t), st));
    int64_t g = (n * 9 + 255) / 256;
    if (g > (int64_t)num_sms() * 8) g = (int64_t)num_sms() * 8;
    wino_wmax_kernel<<<(unsigned)g, 256, 0, st>>>(w, n * 9, wmax);
  }
  int64_t g = (n + 255) / 256;
  if (g > (int64_t)num_sms() * 16) g = (int64_t)num_sms() * 16;
  wino_weight_kernel<T><<<(unsigned)g, 256, 0, st>>>(w, Cout, Cin, dgrad, wmax, (__half*)u_hi, (__half*)u_lo);
  if (wmax) wino_wscale_store_kernel<<<1, 1, 0, st>>>(inv_wscale);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // namespace

extern "C" {

int bbdm_wino_geometry(int B, int H, int W, int* tiles_h, int* tiles_w, int64_t* tiles_total, int* eligible) {
  return wino_geometry_t<4>(B, H, W, tiles_h, tiles_w, tiles_total, eligible);
}
int bbdm_wino_input(const BbdmWinoInputArgs* a, void* stream) { return wino_input_t<4>(a, stream); }
int bbdm_wino_output(const BbdmWinoOutputArgs* a, void* stream) { return wino_output_t<4>(a, stream); }
int bbdm_wino_pack_weight(const float* w, int Cout, int Cin, int dgrad, void* u_hi, void* u_lo, float* inv_wscale,
                          void* stream) {
  return wino_pack_weight_t<4>(w, Cout, Cin, dgrad, u_hi, u_lo, inv_wscale, stream);
}

int bbdm_wino6_geometry(int B, int H, int W, int* tiles_h, int* tiles_w, int64_t* tiles_total, int* eligible) {
  return wino_geometry_t<6>(B, H, W, tiles_h, tiles_w, tiles_total, eligible);
}
int bbdm_wino6_input(const BbdmWinoInputArgs* a, void* stream) { return wino_input_t<6>(a, stream); }
int bbdm_wino6_output(const BbdmWinoOutputArgs* a, void* stream) { return wino_output_t<6>(a, stream); }
int bbdm_wino6_pack_weight(const float* w, int Cout, int Cin, int dgrad, void* u_hi, void* u_lo, float* inv_wscale,
                           void* stream) {
  return wino_pack_weight_t<6>(w, Cout, Cin, dgrad, u_hi, u_lo, inv_wscale, stream);
}

}  // extern "C"
