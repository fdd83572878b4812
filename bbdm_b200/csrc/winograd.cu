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
  int B, H, W, C, groups, cpg, th, tw;
  int64_t Mtot;
  const float* mean; const float* rstd; const float* gamma; const float* beta;
  const float* fscale; const float* fshift; int64_t fstride;
  int silu;
  __half* v_hi; __half* v_lo;
  __nv_bfloat16* raw_hi; __nv_bfloat16* raw_lo;
  __nv_bfloat16* act_hi; __nv_bfloat16* act_lo;   // optional split-bf16 planes of the ACTIVATED tensor (wgrad operand)
};

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
// tile row in segments of 8 tiles.  Per segment: (1) cp.async stages the 6 x 34 pixel x 64 channel input patch
// (double buffered: the next segment's loads fly while this one is transformed -- the register variant above is
// bound by exposed load latency, ncu: 65 % long-scoreboard stalls, 29 % issue utilisation); (2) every pixel is
// activated ONCE in place (GroupNorm affine x FiLM, SiLU; out-of-image pixels become exact zeros = the conv padding
// of the activated tensor); (3) thread (tile, channel pair) reads its 6x6 tile with conflict-free 8-byte LDS,
// transforms, splits to fp16 hi/lo and stores (128 contiguous bytes per warp, position and plane).
constexpr int WI_CC = 64;                 // channels per CTA
constexpr int WI_TX = 8;                  // tiles per segment
constexpr int WI_COLS = 4 * WI_TX + 2;    // patch columns
constexpr int WI_PATCH = 6 * WI_COLS * WI_CC;          // floats per buffer
constexpr size_t WI_SMEM = 2 * (size_t)WI_PATCH * sizeof(float);

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(g) : "memory");
}

__global__ void __launch_bounds__(256, 2)
wino_input_smem_kernel(const WinoInParams p) {
  extern __shared__ __align__(16) float patch[];          // [2][6][WI_COLS][WI_CC]
  const int b = blockIdx.x / p.th, ty = blockIdx.x % p.th;
  const int cbase = blockIdx.y * WI_CC;                    // first channel of this CTA (in the concatenation)
  const float* base;
  int cs, cc0;
  if (cbase < p.c1) { base = p.src1; cs = p.c1; cc0 = cbase; } else { base = p.src2; cs = p.c2; cc0 = cbase - p.c1; }
  const int y0 = 4 * ty - 1;
  const int tid = threadIdx.x;
  const int ch4 = tid & 15;                                // this thread's 4-channel group in phases 1/2
  const int pix0 = tid >> 4;                               // first patch pixel of this thread (stride 16 pixels)
  constexpr int NPIX = 6 * WI_COLS;                        // 204 pixels per patch

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
  const int nseg = (p.tw + WI_TX - 1) / WI_TX;
  const uint32_t patch_s = (uint32_t)__cvta_generic_to_shared(patch);

  auto stage = [&](int seg, int buf) {
    const int x0 = 4 * WI_TX * seg - 1;
    int i = 0, j = pix0;                                  // pix0 < 16 < WI_COLS: row 0
    for (int px = pix0; px < NPIX; px += 16, j += 16) {
      if (j >= WI_COLS) { j -= WI_COLS; ++i; }
      const int iy = y0 + i, ix = x0 + j;
      if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W)
        cp_async16(patch_s + (uint32_t)(((buf * NPIX + px) * WI_CC + ch4 * 4) * 4),
                   base + (((int64_t)b * p.H + iy) * p.W + ix) * cs + cc0 + ch4 * 4);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
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
    float* pb = patch + buf * WI_PATCH;
    const int x0 = 4 * WI_TX * seg - 1;
    // ---- phase 2: activate every staged pixel once, in place ------------------------------------------------
    int i = 0, j = pix0;
    for (int px = pix0; px < NPIX; px += 16, j += 16) {
      if (j >= WI_COLS) { j -= WI_COLS; ++i; }
      const int iy = y0 + i, ix = x0 + j;
      float4* q = reinterpret_cast<float4*>(pb + px * WI_CC + ch4 * 4);
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
        const float4 x = *q;
        if (p.raw_hi && i >= 1 && i <= 4 && j >= 1 && j <= 4 * WI_TX) {
          // pixels this segment owns: raw split-bf16 planes for the 1x1 skip conv
          uint2 h, l;
          split4(x, h, l);
          const int64_t off = (((int64_t)b * p.H + iy) * p.W + ix) * p.C + cbase + ch4 * 4;
          *reinterpret_cast<uint2*>(p.raw_hi + off) = h;
          *reinterpret_cast<uint2*>(p.raw_lo + off) = l;
        }
        a.x = fmaf(x.x, sc[0], sh[0]); a.y = fmaf(x.y, sc[1], sh[1]);
        a.z = fmaf(x.z, sc[2], sh[2]); a.w = fmaf(x.w, sc[3], sh[3]);
        if (p.silu) {
          a.x = __fdividef(a.x, 1.0f + __expf(-a.x)); a.y = __fdividef(a.y, 1.0f + __expf(-a.y));
          a.z = __fdividef(a.z, 1.0f + __expf(-a.z)); a.w = __fdividef(a.w, 1.0f + __expf(-a.w));
        }
        if (p.act_hi && i >= 1 && i <= 4 && j >= 1 && j <= 4 * WI_TX) {
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
    // ---- phase 3: one (tile, channel pair) per thread -------------------------------------------------------
    const int txl = tid >> 5, c0 = (tid & 31) * 2;
    const int tx = WI_TX * seg + txl;
    if (tx < p.tw) {
      float t0[36], t1[36];
#pragma unroll
      for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          const float2 v = *reinterpret_cast<const float2*>(pb + ((i * WI_COLS + 4 * txl + j) * WI_CC + c0));
          t0[i * 6 + j] = v.x;
          t1[i * 6 + j] = v.y;
        }
#pragma unroll
      for (int j = 0; j < 6; ++j) { wino_bt6<6>(t0 + j); wino_bt6<6>(t1 + j); }
#pragma unroll
      for (int i = 0; i < 6; ++i) { wino_bt6<1>(t0 + 6 * i); wino_bt6<1>(t1 + 6 * i); }
      const int64_t m = ((int64_t)b * p.th + ty) * p.tw + tx;
      const int64_t plane = p.Mtot * p.C;
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

// U[q][co][ci] = s * (G g G^T)[q] in fp64, split into fp16 planes.  One thread per (co, ci).
// dgrad != 0: the data-gradient conv's weights instead -- kernel flipped, channels swapped: U[q][ci][co] from
// g'[ky][kx] = w[co][ci][2-ky][2-kx] (threads run over co fastest so the stores stay coalesced).
__global__ void __launch_bounds__(256)
wino_weight_kernel(const float* __restrict__ w, int Cout, int Cin, int dgrad, const uint32_t* __restrict__ wmax,
                   __half* __restrict__ u_hi, __half* __restrict__ u_lo) {
  const int64_t n = (int64_t)Cout * Cin;
  const double s = wmax ? (double)wino_wscale(*wmax) : (double)WINO_WSCALE_FIXED;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * blockDim.x) {
    double g[3][3], t[6][3];
    int64_t src = idx;
    if (dgrad) { const int64_t ci = idx / Cout, co = idx - ci * Cout; src = co * Cin + ci; }
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const int k = dgrad ? 8 - i : i;
      g[i / 3][i % 3] = (double)w[src * 9 + k];
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double g0 = g[0][j], g1 = g[1][j], g2 = g[2][j];
      t[0][j] = g0 / 4.0;
      t[1][j] = -(g0 + g1 + g2) / 6.0;
      t[2][j] = -(g0 - g1 + g2) / 6.0;
      t[3][j] = g0 / 24.0 + g1 / 12.0 + g2 / 6.0;
      t[4][j] = g0 / 24.0 - g1 / 12.0 + g2 / 6.0;
      t[5][j] = g2;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      const double g0 = t[i][0], g1 = t[i][1], g2 = t[i][2];
      double u[6];
      u[0] = g0 / 4.0;
      u[1] = -(g0 + g1 + g2) / 6.0;
      u[2] = -(g0 - g1 + g2) / 6.0;
      u[3] = g0 / 24.0 + g1 / 12.0 + g2 / 6.0;
      u[4] = g0 / 24.0 - g1 / 12.0 + g2 / 6.0;
      u[5] = g2;
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        const float v = (float)(u[j] * s);
        const __half h = __float2half_rn(v);
        const __half l = __float2half_rn(v - __half2float(h));
        const int64_t off = (int64_t)(i * 6 + j) * n + idx;
        u_hi[off] = h;
        u_lo[off] = l;
      }
    }
  }
}

}  // namespace bbdm

using namespace bbdm;

extern "C" {

int bbdm_wino_geometry(int B, int H, int W, int* tiles_h, int* tiles_w, int64_t* tiles_total, int* eligible) {
  BBDM_REQUIRE(B > 0 && H > 0 && W > 0, "wino_geometry: bad shape");
  const int th = H / 4, tw = W / 4;
  const int64_t mtot = (int64_t)B * th * tw;
  if (tiles_h) *tiles_h = th;
  if (tiles_w) *tiles_w = tw;
  if (tiles_total) *tiles_total = mtot;
  // the GEMM views the tile axis as rows of 16 with 128-tile M blocks inside one transform position
  if (eligible) *eligible = (H % 4 == 0 && W % 4 == 0 && mtot % 16 == 0 && mtot >= 128) ? 1 : 0;
  return BBDM_OK;
}

int bbdm_wino_input(const BbdmWinoInputArgs* a, void* stream) {
  BBDM_REQUIRE(a && a->src1 && a->v_hi && a->v_lo, "wino_input: null args");
  WinoInParams p;
  p.src1 = a->src1; p.c1 = a->c1;
  p.src2 = a->src2; p.c2 = a->src2 ? a->c2 : 0;
  p.B = a->B; p.H = a->H; p.W = a->W;
  p.C = p.c1 + p.c2;
  p.groups = a->groups;
  BBDM_REQUIRE(p.B > 0 && p.H > 0 && p.W > 0 && p.H % 4 == 0 && p.W % 4 == 0, "wino_input: H, W must be multiples of 4");
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
  p.th = p.H / 4; p.tw = p.W / 4;
  p.Mtot = (int64_t)p.B * p.th * p.tw;
  p.mean = a->mean; p.rstd = a->rstd; p.gamma = a->gamma; p.beta = a->beta;
  p.fscale = a->film_scale; p.fshift = a->film_shift; p.fstride = a->film_stride;
  p.silu = a->silu;
  p.v_hi = (__half*)a->v_hi; p.v_lo = (__half*)a->v_lo;
  p.raw_hi = (__nv_bfloat16*)a->raw_hi; p.raw_lo = (__nv_bfloat16*)a->raw_lo;
  p.act_hi = (__nv_bfloat16*)a->act_hi; p.act_lo = (__nv_bfloat16*)a->act_lo;
  const bool smem_only = a->mean == nullptr || a->act_hi != nullptr;      // features only the staged kernel has
  const int64_t ctas = (int64_t)p.B * p.th;
  BBDM_REQUIRE(ctas < (1ll << 31), "wino_input: too many tile rows");
  // default: the shared-memory staged kernel (needs 64-channel chunks inside one source tensor);
  // BBDM_WINO_IN_VEC=1|2 selects the register-only variant with 1 or 2 channels per thread (fallback / A-B switch)
  static int vec = -1;
  if (vec < 0) { const char* e = getenv("BBDM_WINO_IN_VEC"); vec = e ? (atoi(e) == 2 ? 2 : 1) : 0; }
  if (vec == 0 && p.c1 % WI_CC == 0 && p.c2 % WI_CC == 0) {
    static DeviceOnce configured;
    if (configured.need()) {
      BBDM_CUDA_CHECK(cudaFuncSetAttribute(wino_input_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WI_SMEM));
      configured.mark();
    }
    dim3 grid((unsigned)ctas, p.C / WI_CC);
    wino_input_smem_kernel<<<grid, 256, WI_SMEM, (cudaStream_t)stream>>>(p);
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

int bbdm_wino_output(const BbdmWinoOutputArgs* a, void* stream) {
  BBDM_REQUIRE(a && a->m && a->out, "wino_output: null args");
  WinoOutParams p;
  p.m = a->m; p.inv_wscale = a->inv_wscale;
  p.B = a->B; p.H = a->H; p.W = a->W; p.Cout = a->Cout;
  BBDM_REQUIRE(p.B > 0 && p.B <= 65535 && p.H > 0 && p.W > 0 && p.H % 4 == 0 && p.W % 4 == 0,
               "wino_output: H, W must be multiples of 4 (B <= 65535)");
  BBDM_REQUIRE(p.Cout > 0 && p.Cout % 64 == 0, "wino_output: Cout %% 64 != 0");
  BBDM_REQUIRE(a->res_mode >= 0 && a->res_mode <= 3 && (a->res_mode == 0 || a->residual), "wino_output: bad residual");
  if (a->res_mode == BBDM_RES_UP2) BBDM_REQUIRE(p.H % 2 == 0 && p.W % 2 == 0, "wino_output: RES_UP2 needs even H, W");
  p.th = p.H / 4; p.tw = p.W / 4;
  BBDM_REQUIRE(p.th <= 65535, "wino_output: too many tile rows");
  p.Mtot = (int64_t)p.B * p.th * p.tw;
  p.bias = a->bias; p.residual = a->residual; p.res_mode = a->res_mode;
  p.out = a->out; p.stats = a->stats_partial;
  dim3 grid(p.Cout / 64, p.th, p.B);
  cudaStream_t st = (cudaStream_t)stream;
  switch (p.res_mode) {
    case BBDM_RES_SAME: wino_output_kernel<BBDM_RES_SAME><<<grid, 256, 0, st>>>(p); break;
    case BBDM_RES_UP2: wino_output_kernel<BBDM_RES_UP2><<<grid, 256, 0, st>>>(p); break;
    case BBDM_RES_DOWN2: wino_output_kernel<BBDM_RES_DOWN2><<<grid, 256, 0, st>>>(p); break;
    default: wino_output_kernel<BBDM_RES_NONE><<<grid, 256, 0, st>>>(p); break;
  }
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

int bbdm_wino_pack_weight(const float* w, int Cout, int Cin, int dgrad, void* u_hi, void* u_lo, float* inv_wscale,
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
  wino_weight_kernel<<<(unsigned)g, 256, 0, st>>>(w, Cout, Cin, dgrad, wmax, (__half*)u_hi, (__half*)u_lo);
  if (wmax) wino_wscale_store_kernel<<<1, 1, 0, st>>>(inv_wscale);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // extern "C"
