// The two VQGAN-specific steps either side of the latent bridge loop :
//   * row softmax of the single-head AttnBlock's T x Tp score matrix (Tp = T rounded up to 64, the padding columns
//     masked), written as split-bf16 planes (the A operand of the P.V tensor-core GEMM)   model/VQGAN/model.py:140-192,
//     and its backward (the dS planes of the GEMM-composed attention's training route for heads wider than 256)
//   * VectorQuantizer2 nearest-codebook lookup                          model/VQGAN/quantize.py:271-312
// Everything else of the autoencoder (ResnetBlocks, 1x1/3x3 convs, GroupNorm, resampling) runs on the
// same kernels as the UNet.
#include "common.cuh"

namespace bbdm {

__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, u) : v + u;
  }
  __syncthreads();                      // red may still be read from a previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < nw; ++i) r = is_max ? fmaxf(r, red[i]) : r + red[i];   // fixed order, every thread
  return r;
}

// exp(scale*s - m) with the product rounded first, as the reference scales the scores before its softmax
__device__ __forceinline__ float sexp(float s, float scale, float m) { return expf(__fsub_rn(__fmul_rn(s, scale), m)); }

// columns i+1..i+3 of a float4 at or past V take `fill` (column i < V is the caller's condition)
__device__ __forceinline__ void mask_tail(float4& v, int64_t i, int64_t V, float fill) {
  if (i + 1 >= V) v.y = fill;
  if (i + 2 >= V) v.z = fill;
  if (i + 3 >= V) v.w = fill;
}

// one CTA per row: p = softmax(scale * s) over the first V columns -> hi/lo planes, exact zeros in columns V..N-1
// (the padding of a key axis rounded up to the GEMM's 64-column tile).  N % 4 == 0, 0 < V <= N; MASKED == (V < N).
// Only the float4 that straddles V is masked, so the first V columns see the unmasked arithmetic and reduction order.
template <bool MASKED>
__global__ void __launch_bounds__(256)
softmax_rows_split_kernel(const float* __restrict__ src, int64_t N, int64_t V, float scale,
                          __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  __shared__ float red[8];
  const float* row = src + (int64_t)blockIdx.x * N;
  float mx = -INFINITY;
  for (int64_t i = threadIdx.x * 4; i < V; i += 1024) {
    float4 v = ld_f4(row + i);
    if (MASKED && i + 4 > V) mask_tail(v, i, V, -INFINITY);
    mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  // scale > 0: max(scale * s) = scale * max(s) exactly (monotone rounding)
  const float m = block_reduce(mx, red, true) * scale;
  float sum = 0.f;
  for (int64_t i = threadIdx.x * 4; i < V; i += 1024) {
    const float4 v = ld_f4(row + i);
    float4 e = make_float4(sexp(v.x, scale, m), sexp(v.y, scale, m), sexp(v.z, scale, m), sexp(v.w, scale, m));
    if (MASKED && i + 4 > V) mask_tail(e, i, V, 0.f);
    sum += e.x + e.y + e.z + e.w;
  }
  const float inv = 1.0f / block_reduce(sum, red, false);
  __nv_bfloat16* h = hi + (int64_t)blockIdx.x * N;
  __nv_bfloat16* l = lo + (int64_t)blockIdx.x * N;
  for (int64_t i = threadIdx.x * 4; i < N; i += 1024) {
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!MASKED || i < V) {
      const float4 v = ld_f4(row + i);
      p = make_float4(sexp(v.x, scale, m) * inv, sexp(v.y, scale, m) * inv, sexp(v.z, scale, m) * inv,
                      sexp(v.w, scale, m) * inv);
      if (MASKED && i + 4 > V) mask_tail(p, i, V, 0.f);
    }
    uint2 ph, pl;
    split4(p, ph, pl);
    *reinterpret_cast<uint2*>(h + i) = ph;
    *reinterpret_cast<uint2*>(l + i) = pl;
  }
}

// Backward of the row softmax above, one CTA per row: recomputes p = softmax(scale * s) over the first V columns with
// the forward's loops, reductions and expressions (the same p the forward split), then writes the score gradient
// ds = scale * p * (dp - sum_j p_j dp_j) as split-bf16 planes (the A operand of dQ = dS K and of the dK weight
// gradient), exact zeros in columns V..N-1.  The row (N <= a few thousand floats of s and of dp) is re-read from L1/L2
// by the later loops, not from HBM.
template <bool MASKED>
__global__ void __launch_bounds__(256)
softmax_rows_bwd_kernel(const float* __restrict__ s_in, const float* __restrict__ dp_in, int64_t N, int64_t V,
                        float scale, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  __shared__ float red[8];
  const float* row = s_in + (int64_t)blockIdx.x * N;
  const float* drow = dp_in + (int64_t)blockIdx.x * N;
  float mx = -INFINITY;
  for (int64_t i = threadIdx.x * 4; i < V; i += 1024) {
    float4 v = ld_f4(row + i);
    if (MASKED && i + 4 > V) mask_tail(v, i, V, -INFINITY);
    mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  const float m = block_reduce(mx, red, true) * scale;
  float sum = 0.f;
  for (int64_t i = threadIdx.x * 4; i < V; i += 1024) {
    const float4 v = ld_f4(row + i);
    float4 e = make_float4(sexp(v.x, scale, m), sexp(v.y, scale, m), sexp(v.z, scale, m), sexp(v.w, scale, m));
    if (MASKED && i + 4 > V) mask_tail(e, i, V, 0.f);
    sum += e.x + e.y + e.z + e.w;
  }
  const float inv = 1.0f / block_reduce(sum, red, false);
  // sum_j p_j dp_j over the valid columns, in the same per-thread order and fixed cross-warp order
  float dot = 0.f;
  for (int64_t i = threadIdx.x * 4; i < V; i += 1024) {
    const float4 v = ld_f4(row + i);
    float4 p = make_float4(sexp(v.x, scale, m) * inv, sexp(v.y, scale, m) * inv, sexp(v.z, scale, m) * inv,
                           sexp(v.w, scale, m) * inv);
    float4 g = ld_f4(drow + i);
    if (MASKED && i + 4 > V) { mask_tail(p, i, V, 0.f); mask_tail(g, i, V, 0.f); }
    dot += p.x * g.x + p.y * g.y + p.z * g.z + p.w * g.w;
  }
  dot = block_reduce(dot, red, false);
  __nv_bfloat16* h = hi + (int64_t)blockIdx.x * N;
  __nv_bfloat16* l = lo + (int64_t)blockIdx.x * N;
  for (int64_t i = threadIdx.x * 4; i < N; i += 1024) {
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!MASKED || i < V) {
      const float4 v = ld_f4(row + i);
      const float4 g = ld_f4(drow + i);
      const float4 p = make_float4(sexp(v.x, scale, m) * inv, sexp(v.y, scale, m) * inv, sexp(v.z, scale, m) * inv,
                                   sexp(v.w, scale, m) * inv);
      d = make_float4(scale * p.x * (g.x - dot), scale * p.y * (g.y - dot), scale * p.z * (g.z - dot),
                      scale * p.w * (g.w - dot));
      if (MASKED && i + 4 > V) mask_tail(d, i, V, 0.f);
    }
    uint2 dh, dl;
    split4(d, dh, dl);
    *reinterpret_cast<uint2*>(h + i) = dh;
    *reinterpret_cast<uint2*>(l + i) = dl;
  }
}

// nearest codebook entry per latent vector; d = (|z|^2 + |e|^2) - 2 z.e exactly as the reference writes it
// (fp32, first minimum wins); z_q = z + (e - z) (the straight-through expression's forward value).
constexpr int VQ_TILE = 512;
constexpr int VQ_MAXD = 16;

__global__ void __launch_bounds__(256)
vq_nearest_kernel(const float* __restrict__ z, const float* __restrict__ cb, int64_t N, int n_e, int D,
                  float* __restrict__ zq, long long* __restrict__ idx) {
  __shared__ float es[VQ_TILE * VQ_MAXD];
  __shared__ float e2[VQ_TILE];
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float zv[VQ_MAXD];
  float z2 = 0.f;
#pragma unroll
  for (int d = 0; d < VQ_MAXD; ++d) {
    zv[d] = (n < N && d < D) ? z[n * D + d] : 0.f;
    if (d < D) z2 = __fadd_rn(z2, __fmul_rn(zv[d], zv[d]));
  }
  float best = INFINITY;
  int best_i = 0;
  for (int t0 = 0; t0 < n_e; t0 += VQ_TILE) {
    const int cnt = min(VQ_TILE, n_e - t0);
    __syncthreads();
    for (int i = threadIdx.x; i < cnt * D; i += blockDim.x) es[i] = cb[(int64_t)t0 * D + i];
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      float s = 0.f;
      for (int d = 0; d < D; ++d) s = __fadd_rn(s, __fmul_rn(es[i * D + d], es[i * D + d]));
      e2[i] = s;
    }
    __syncthreads();
    for (int i = 0; i < cnt; ++i) {
      float dot = 0.f;
#pragma unroll
      for (int d = 0; d < VQ_MAXD; ++d)
        if (d < D) dot = fmaf(zv[d], es[i * D + d], dot);
      const float dist = __fsub_rn(__fadd_rn(z2, e2[i]), __fmul_rn(2.0f, dot));
      if (dist < best) { best = dist; best_i = t0 + i; }
    }
  }
  if (n < N) {
    idx[n] = best_i;
#pragma unroll
    for (int d = 0; d < VQ_MAXD; ++d)
      if (d < D) zq[n * D + d] = __fadd_rn(zv[d], __fsub_rn(cb[(int64_t)best_i * D + d], zv[d]));
  }
}

// space-to-depth by 2 + bf16 split: dst[b, i, j, (a*2+b2)*C + c] = src[b, 2i+a, 2j+b2, c]
__global__ void __launch_bounds__(256)
s2d_split_kernel(const float* __restrict__ src, int64_t n4, int H, int W, int C, __nv_bfloat16* __restrict__ hi,
                 __nv_bfloat16* __restrict__ lo) {
  const int C4 = C / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int c = (int)(r % C4) * 4; r /= C4;
    const int w = (int)(r % W); r /= W;
    const int h = (int)(r % H);
    const int64_t b = r / H;
    const float4 v = ld_f4(src + i * 4);
    uint2 ph, pl;
    split4(v, ph, pl);
    const int64_t o = (((b * (H / 2) + h / 2) * (W / 2) + w / 2) * 4 + (h & 1) * 2 + (w & 1)) * C + c;
    *reinterpret_cast<uint2*>(hi + o) = ph;
    *reinterpret_cast<uint2*>(lo + o) = pl;
  }
}

}  // namespace bbdm

using namespace bbdm;

// [B,H,W,C] fp32 -> split-bf16 planes [B,H/2,W/2,4C] (channel = (row parity*2 + col parity)*C + c): the A operand
// of a stride-2 3x3 convolution run as a 2x2-tap tensor-core conv (BbdmConvArgs.taps = 4).
extern "C" int bbdm_s2d_split(const float* src, int B, int H, int W, int C, void* out_hi, void* out_lo, void* stream) {
  BBDM_REQUIRE(src && out_hi && out_lo, "s2d_split: null pointer");
  BBDM_REQUIRE(B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C > 0 && C % 4 == 0, "s2d_split: bad shape");
  const int64_t n4 = (int64_t)B * H * W * (C / 4);
  int64_t blocks = (n4 + 255) / 256;
  if (blocks > num_sms() * 32) blocks = num_sms() * 32;
  s2d_split_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(src, n4, H, W, C, (__nv_bfloat16*)out_hi,
                                                                       (__nv_bfloat16*)out_lo);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

extern "C" int bbdm_softmax_rows_split(const float* src, int64_t rows, int64_t cols, int64_t valid_cols, float scale,
                                       void* out_hi, void* out_lo, void* stream) {
  BBDM_REQUIRE(src && out_hi && out_lo, "softmax_rows_split: null pointer");
  BBDM_REQUIRE(rows > 0 && rows < (1ll << 31) && cols > 0 && cols % 4 == 0 && scale > 0.f,
               "softmax_rows_split: bad shape (cols must be a multiple of 4, scale > 0)");
  BBDM_REQUIRE(valid_cols > 0 && valid_cols <= cols, "softmax_rows_split: valid_cols %lld not in 1..cols = %lld",
               (long long)valid_cols, (long long)cols);
  if (valid_cols == cols)
    softmax_rows_split_kernel<false><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(
        src, cols, cols, scale, (__nv_bfloat16*)out_hi, (__nv_bfloat16*)out_lo);
  else
    softmax_rows_split_kernel<true><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(
        src, cols, valid_cols, scale, (__nv_bfloat16*)out_hi, (__nv_bfloat16*)out_lo);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

extern "C" int bbdm_softmax_rows_bwd(const float* s, const float* dp, int64_t rows, int64_t cols, int64_t valid_cols,
                                     float scale, void* ds_hi, void* ds_lo, void* stream) {
  BBDM_REQUIRE(s && dp && ds_hi && ds_lo, "softmax_rows_bwd: null pointer");
  BBDM_REQUIRE(rows > 0 && rows < (1ll << 31) && cols > 0 && cols % 4 == 0 && scale > 0.f,
               "softmax_rows_bwd: bad shape (cols must be a multiple of 4, scale > 0)");
  BBDM_REQUIRE(valid_cols > 0 && valid_cols <= cols, "softmax_rows_bwd: valid_cols %lld not in 1..cols = %lld",
               (long long)valid_cols, (long long)cols);
  if (valid_cols == cols)
    softmax_rows_bwd_kernel<false><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(
        s, dp, cols, cols, scale, (__nv_bfloat16*)ds_hi, (__nv_bfloat16*)ds_lo);
  else
    softmax_rows_bwd_kernel<true><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(
        s, dp, cols, valid_cols, scale, (__nv_bfloat16*)ds_hi, (__nv_bfloat16*)ds_lo);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

extern "C" int bbdm_vq_nearest(const float* z, const float* codebook, int64_t n_vectors, int n_embed, int dim,
                               float* z_q, long long* indices, void* stream) {
  BBDM_REQUIRE(z && codebook && z_q && indices, "vq_nearest: null pointer");
  BBDM_REQUIRE(n_vectors > 0 && n_embed > 0 && dim > 0 && dim <= VQ_MAXD, "vq_nearest: bad shape (dim <= %d)", VQ_MAXD);
  const int64_t blocks = (n_vectors + 255) / 256;
  BBDM_REQUIRE(blocks < (1ll << 31), "vq_nearest: too many vectors");
  vq_nearest_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(z, codebook, n_vectors, n_embed, dim, z_q, indices);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}
