// Operand-producing passes of the SpatialTransformer (reference attention.py:36-50, 196-216): LayerNorm and GEGLU,
// each fused with the split into the bf16 (hi, lo) planes the following wgmma GEMM reads.  HBM-bound:
//   layernorm_split : 4 B read + 4 B written per element
//   geglu_split     : 8 B read + 4 B written per output element
// and the backward passes of both (training path):
//   layernorm_bwd   : 8 B read + 4 B written per element, plus fixed-order column partials of dgamma / dbeta
//   geglu_bwd       : 12 B read + 8 B written per output element
#include "common.cuh"

namespace bbdm {

// One warp per token row: the row is held in registers (C <= 32 * LN_MAX_PER_LANE), two-pass mean / variance in
// fp32 like torch's LayerNorm (biased variance, eps inside the sqrt), then y = (x - mean) * rstd * gamma + beta.
constexpr int LN_MAX_PER_LANE = 64;       // C <= 2048

__global__ void __launch_bounds__(256)
layernorm_split_kernel(const float* __restrict__ x, int64_t rows, int C, const float* __restrict__ gamma,
                       const float* __restrict__ beta, float eps, float* __restrict__ out_f32,
                       __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + row * C;
  const int n2 = C >> 1;                      // float2 elements per row
  float2 v[LN_MAX_PER_LANE / 2];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_PER_LANE / 2; ++i) {
    const int j = lane + 32 * i;
    v[i] = make_float2(0.f, 0.f);
    if (j < n2) { v[i] = *reinterpret_cast<const float2*>(xr + 2 * j); s += v[i].x + v[i].y; }
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_PER_LANE / 2; ++i) {
    const int j = lane + 32 * i;
    if (j < n2) { const float a = v[i].x - mean, b = v[i].y - mean; q = fmaf(a, a, fmaf(b, b, q)); }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < LN_MAX_PER_LANE / 2; ++i) {
    const int j = lane + 32 * i;
    if (j < n2) {
      const float2 g = *reinterpret_cast<const float2*>(gamma + 2 * j), b = *reinterpret_cast<const float2*>(beta + 2 * j);
      const float y0 = fmaf((v[i].x - mean) * rstd, g.x, b.x), y1 = fmaf((v[i].y - mean) * rstd, g.y, b.y);
      const int64_t off = row * C + 2 * j;
      if (out_f32) *reinterpret_cast<float2*>(out_f32 + off) = make_float2(y0, y1);
      if (out_hi) {
        uint32_t h, l;
        split2x(y0, y1, h, l);
        *reinterpret_cast<uint32_t*>(out_hi + off) = h;
        *reinterpret_cast<uint32_t*>(out_lo + off) = l;
      }
    }
  }
}

// out[r][n] = u[r][n] * gelu(u[r][N + n]), exact (erf) GELU like F.gelu's default; u = the GEGLU projection [rows][2N]
__global__ void __launch_bounds__(256)
geglu_split_kernel(const float* __restrict__ u, int64_t rows, int N, float* __restrict__ out_f32,
                   __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo) {
  const int64_t n4 = rows * (N / 4);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / (N / 4);
    const int c = (int)(i - r * (N / 4)) * 4;
    const float4 a = ld_f4(u + r * 2 * N + c), g = ld_f4(u + r * 2 * N + N + c);
    float4 o;
    o.x = a.x * (0.5f * g.x * (1.0f + erff(g.x * 0.70710678118654752440f)));
    o.y = a.y * (0.5f * g.y * (1.0f + erff(g.y * 0.70710678118654752440f)));
    o.z = a.z * (0.5f * g.z * (1.0f + erff(g.z * 0.70710678118654752440f)));
    o.w = a.w * (0.5f * g.w * (1.0f + erff(g.w * 0.70710678118654752440f)));
    const int64_t off = r * N + c;
    if (out_f32) st_f4(out_f32 + off, o);
    if (out_hi) {
      uint2 h, l;
      split4(o, h, l);
      *reinterpret_cast<uint2*>(out_hi + off) = h;
      *reinterpret_cast<uint2*>(out_lo + off) = l;
    }
  }
}

// LayerNorm backward, one warp per token row as in the forward (same two-pass mean / rstd, recomputed from x):
//   xh = (x - mean) * rstd,  gy = gamma * dy
//   dx = rstd * (gy - mean_c(gy) - xh * mean_c(gy * xh))
//   dgamma = sum_rows dy * xh,  dbeta = sum_rows dy
// Each CTA takes LNB_ROWS consecutive rows; every warp accumulates its rows' dgamma / dbeta terms in its own shared
// memory row, the 8 warp rows are added in a fixed order into the CTA's partial [2][C], and layernorm_bwd_reduce sums
// the CTA partials in a fixed order (deterministic, no atomics).
constexpr int LNB_ROWS = 64;

__global__ void __launch_bounds__(256)
layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, int64_t rows, int C,
                     const float* __restrict__ gamma, float eps, float* __restrict__ dx, float* __restrict__ part) {
  extern __shared__ __align__(16) float lnb_acc[];          // [8 warps][2][C]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* acc_g = lnb_acc + (int64_t)warp * 2 * C;
  float* acc_b = acc_g + C;
  const int n2 = C >> 1;
#pragma unroll
  for (int i = 0; i < LN_MAX_PER_LANE / 2; ++i) {
    const int j = lane + 32 * i;
    if (j < n2) {
      *reinterpret_cast<float2*>(acc_g + 2 * j) = make_float2(0.f, 0.f);
      *reinterpret_cast<float2*>(acc_b + 2 * j) = make_float2(0.f, 0.f);
    }
  }
  const int64_t r0 = (int64_t)blockIdx.x * LNB_ROWS;
  const int64_t r1 = r0 + LNB_ROWS < rows ? r0 + LNB_ROWS : rows;
  for (int64_t row = r0 + warp; row < r1; row += 8) {
    const float* xr = x + row * C;
    const float* dyr = dy + row * C;
    float2 v[LN_MAX_PER_LANE / 2];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 2; ++i) {
      const int j = lane + 32 * i;
      v[i] = make_float2(0.f, 0.f);
      if (j < n2) { v[i] = *reinterpret_cast<const float2*>(xr + 2 * j); s += v[i].x + v[i].y; }
    }
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 2; ++i) {
      const int j = lane + 32 * i;
      if (j < n2) { const float a = v[i].x - mean, b = v[i].y - mean; q = fmaf(a, a, fmaf(b, b, q)); }
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 2; ++i) {
      const int j = lane + 32 * i;
      if (j < n2) {
        v[i] = make_float2((v[i].x - mean) * rstd, (v[i].y - mean) * rstd);          // xh from here on
        const float2 g = *reinterpret_cast<const float2*>(gamma + 2 * j), d = *reinterpret_cast<const float2*>(dyr + 2 * j);
        const float gy0 = g.x * d.x, gy1 = g.y * d.y;
        s1 += gy0 + gy1;
        s2 = fmaf(gy0, v[i].x, fmaf(gy1, v[i].y, s2));
      }
    }
    const float m1 = warp_sum(s1) / (float)C, m2 = warp_sum(s2) / (float)C;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 2; ++i) {
      const int j = lane + 32 * i;
      if (j < n2) {
        const float2 g = *reinterpret_cast<const float2*>(gamma + 2 * j), d = *reinterpret_cast<const float2*>(dyr + 2 * j);
        *reinterpret_cast<float2*>(dx + row * C + 2 * j) =
            make_float2(rstd * (g.x * d.x - m1 - v[i].x * m2), rstd * (g.y * d.y - m1 - v[i].y * m2));
        float2 ag = *reinterpret_cast<float2*>(acc_g + 2 * j), ab = *reinterpret_cast<float2*>(acc_b + 2 * j);
        ag.x = fmaf(d.x, v[i].x, ag.x); ag.y = fmaf(d.y, v[i].y, ag.y);
        ab.x += d.x; ab.y += d.y;
        *reinterpret_cast<float2*>(acc_g + 2 * j) = ag;
        *reinterpret_cast<float2*>(acc_b + 2 * j) = ab;
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += 256) {
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) a += lnb_acc[(int64_t)w * 2 * C + c];
    part[(int64_t)blockIdx.x * 2 * C + c] = a;                 // [block][dgamma C | dbeta C]
  }
}

// one warp per column of the [nblk][2C] partials: lanes stride over the blocks, fixed-order fp64 shuffle tree
__global__ void __launch_bounds__(256)
layernorm_bwd_reduce_kernel(const float* __restrict__ part, int nblk, int C, float* __restrict__ dgamma,
                            float* __restrict__ dbeta) {
  const int64_t c = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (c >= 2 * C) return;
  double s = 0.0;
  for (int b = lane; b < nblk; b += 32) s += (double)part[(int64_t)b * 2 * C + c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    if (c < C) dgamma[c] = (float)s;
    else dbeta[c - C] = (float)s;
  }
}

// GEGLU backward: out = a * gelu(g), u = [a | g]  ->  du_a = dy * gelu(g),  du_g = dy * a * gelu'(g),
// gelu'(g) = Phi(g) + g * phi(g) (exact erf GELU, as geglu_split_kernel)
__global__ void __launch_bounds__(256)
geglu_bwd_kernel(const float* __restrict__ u, const float* __restrict__ dy, int64_t rows, int N, float* __restrict__ du) {
  const int64_t n4 = rows * (N / 4);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / (N / 4);
    const int c = (int)(i - r * (N / 4)) * 4;
    const float4 a4 = ld_f4(u + r * 2 * N + c), g4 = ld_f4(u + r * 2 * N + N + c), d4 = ld_f4(dy + r * N + c);
    const float av[4] = {a4.x, a4.y, a4.z, a4.w}, gv[4] = {g4.x, g4.y, g4.z, g4.w}, dv[4] = {d4.x, d4.y, d4.z, d4.w};
    float da[4], dg[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float cdf = 0.5f * (1.0f + erff(gv[k] * 0.70710678118654752440f));
      const float pdf = 0.39894228040143267794f * expf(-0.5f * gv[k] * gv[k]);
      da[k] = dv[k] * (gv[k] * cdf);
      dg[k] = dv[k] * av[k] * fmaf(gv[k], pdf, cdf);
    }
    st_f4(du + r * 2 * N + c, make_float4(da[0], da[1], da[2], da[3]));
    st_f4(du + r * 2 * N + N + c, make_float4(dg[0], dg[1], dg[2], dg[3]));
  }
}

}  // namespace bbdm

using namespace bbdm;

extern "C" {

int bbdm_layernorm_split(const float* x, int64_t rows, int C, const float* gamma, const float* beta, float eps,
                         float* out_f32, void* out_hi, void* out_lo, void* stream) {
  BBDM_REQUIRE(x && gamma && beta && rows > 0 && C > 0, "layernorm_split: bad args");
  BBDM_REQUIRE(C % 2 == 0 && C <= 32 * LN_MAX_PER_LANE, "layernorm_split: C must be even and <= %d (got %d)", 32 * LN_MAX_PER_LANE, C);
  BBDM_REQUIRE(out_f32 || (out_hi && out_lo), "layernorm_split: no output");
  BBDM_REQUIRE((out_hi == nullptr) == (out_lo == nullptr), "layernorm_split: hi/lo must come in pairs");
  const int64_t blocks = (rows + 7) / 8;
  BBDM_REQUIRE(blocks < (1ll << 31), "layernorm_split: too many rows");
  layernorm_split_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, rows, C, gamma, beta, eps, out_f32,
                                                                           (__nv_bfloat16*)out_hi, (__nv_bfloat16*)out_lo);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

int bbdm_geglu_split(const float* u, int64_t rows, int N, float* out_f32, void* out_hi, void* out_lo, void* stream) {
  BBDM_REQUIRE(u && rows > 0 && N > 0 && N % 4 == 0, "geglu_split: bad args (N %% 4 == 0 required)");
  BBDM_REQUIRE(out_f32 || (out_hi && out_lo), "geglu_split: no output");
  BBDM_REQUIRE((out_hi == nullptr) == (out_lo == nullptr), "geglu_split: hi/lo must come in pairs");
  const int64_t n4 = rows * (N / 4);
  int64_t g = (n4 + 255) / 256;
  if (g > (int64_t)num_sms() * 16) g = (int64_t)num_sms() * 16;
  geglu_split_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(u, rows, N, out_f32, (__nv_bfloat16*)out_hi,
                                                                   (__nv_bfloat16*)out_lo);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

int bbdm_layernorm_bwd(const float* x, const float* dy, int64_t rows, int C, const float* gamma, float eps, float* dx,
                       float* dgamma, float* dbeta, float* workspace, void* stream) {
  BBDM_REQUIRE(x && dy && gamma && dx && dgamma && dbeta && workspace && rows > 0, "layernorm_bwd: bad args");
  BBDM_REQUIRE(C > 0 && C % 2 == 0 && C <= 32 * LN_MAX_PER_LANE, "layernorm_bwd: C must be even and <= %d (got %d)",
               32 * LN_MAX_PER_LANE, C);
  const int64_t blocks = (rows + LNB_ROWS - 1) / LNB_ROWS;
  BBDM_REQUIRE(blocks < (1ll << 31), "layernorm_bwd: too many rows");
  const int smem = 8 * 2 * C * (int)sizeof(float);
  BBDM_CUDA_CHECK(cudaFuncSetAttribute(layernorm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  cudaStream_t s = (cudaStream_t)stream;
  layernorm_bwd_kernel<<<(unsigned)blocks, 256, smem, s>>>(x, dy, rows, C, gamma, eps, dx, workspace);
  BBDM_LAUNCH_CHECK();
  layernorm_bwd_reduce_kernel<<<(unsigned)((2 * C + 7) / 8), 256, 0, s>>>(workspace, (int)blocks, C, dgamma, dbeta);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

int bbdm_geglu_bwd(const float* u, const float* dy, int64_t rows, int N, float* du, void* stream) {
  BBDM_REQUIRE(u && dy && du && rows > 0 && N > 0 && N % 4 == 0, "geglu_bwd: bad args (N %% 4 == 0 required)");
  const int64_t n4 = rows * (N / 4);
  int64_t g = (n4 + 255) / 256;
  if (g > (int64_t)num_sms() * 16) g = (int64_t)num_sms() * 16;
  geglu_bwd_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(u, dy, rows, N, du);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // extern "C"
