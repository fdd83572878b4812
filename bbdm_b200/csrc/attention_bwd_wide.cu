// Flash-style attention backward (attention_bwd.cu) at head sizes wider than 128: every multiple of 8 up to 256.
// Same arithmetic as the narrow kernels: exact fp32 FMA on CUDA cores over 64 x 64 tiles with 4 x 4 register
// micro-tiles, the same lse / delta outputs, deterministic (no atomics), no T x T tensor.
//
// The narrow kernels keep every operand of a tile resident in both orientations: five (dQ kernel) and six (dK/dV
// kernel) fp32 DP x 64 tiles, 345 KB and 414 KB at DP = 256 against the 232,448 B a CTA may opt in to.  Here only the
// operands that stay for the CTA's whole loop are resident (Q and dO for the dQ kernel, K and V for the dK/dV kernel);
// the streamed operands share one DP x 64 buffer, refilled for each product in turn:
//   dQ kernel, per key tile:   K^T -> S = Q K^T ;  V^T -> dP = dO V^T, dS ;  K rows -> dQ += dS K
//   dK/dV kernel, per query tile: Q^T -> S ;  dO^T -> dP, P, dS ;  Q rows -> dK += dS^T Q ;  dO rows -> dV += P^T dO
// Shared memory at DP = 256: dQ kernel 3 x 65,536 + 17,408 + 256 = 214,272 B, dK/dV kernel 3 x 65,536 + 2 x 17,408
// + 512 = 231,936 B.  The streamed operands are read from L2 once more per tile (K twice per key tile, Q and dO twice
// per query tile).
// Instantiated per padded width DP in {160, 192, 224, 256} with the head_dim D a run-time argument, DP - 32 < D <= DP:
// the loaders zero-fill the columns [D, DP), which add exact zeros to S and dP, and only the columns < D are stored.
#include "attention_bwd.cuh"

namespace bbdm {

namespace {

// 64 rows x D columns of a [*, ld] fp32 matrix -> transposed tile dst_t[DP][64], zero past row T and past column D
template <int DP>
__device__ __forceinline__ void load_cols(const float* __restrict__ src, int64_t ld, int t0, int T, int D, float* dst_t) {
  for (int i = threadIdx.x; i < AB_T * (DP / 4); i += 256) {
    const int row = i % AB_T, ch = i / AB_T;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t0 + row < T && ch * 4 < D) v = ld_f4(src + (int64_t)(t0 + row) * ld + ch * 4);
    dst_t[(ch * 4 + 0) * AB_T + row] = v.x;
    dst_t[(ch * 4 + 1) * AB_T + row] = v.y;
    dst_t[(ch * 4 + 2) * AB_T + row] = v.z;
    dst_t[(ch * 4 + 3) * AB_T + row] = v.w;
  }
}

// ... -> row-major tile dst_r[64][DP]
template <int DP>
__device__ __forceinline__ void load_rows(const float* __restrict__ src, int64_t ld, int t0, int T, int D, float* dst_r) {
  for (int i = threadIdx.x; i < AB_T * (DP / 4); i += 256) {
    const int row = i / (DP / 4), ch = i % (DP / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t0 + row < T && ch * 4 < D) v = ld_f4(src + (int64_t)(t0 + row) * ld + ch * 4);
    *reinterpret_cast<float4*>(dst_r + row * DP + ch * 4) = v;
  }
}

// ---------------------------------------------------------------------------------------------
// kernel 1: per 64-query tile -- delta, log-sum-exp, dQ
// ---------------------------------------------------------------------------------------------
template <int DP>
__global__ void __launch_bounds__(256)
attn_bwd_dq_wide_kernel(const AttnBwdParams p, int D) {
  constexpr int DC = DP / 16;       // dQ columns per thread
  extern __shared__ __align__(16) float sm[];
  float* Qt = sm;                   // [DP][64]
  float* dOt = Qt + DP * AB_T;      // [DP][64]
  float* buf = dOt + DP * AB_T;     // K^T, V^T [DP][64] or K [64][DP]
  float* dSs = buf + DP * AB_T;     // [64][AB_LD]
  float* delta_s = dSs + AB_T * AB_LD;   // [64]

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int bh = blockIdx.y, b = bh / p.heads, head = bh % p.heads;
  const int q0 = blockIdx.x * AB_T;
  int qoff, koff, voff;
  head_offsets(p, head, qoff, koff, voff);
  const float* q_b = p.q + (int64_t)b * p.Tq * p.ldq;
  const float* kv_b = p.kv + (int64_t)b * p.Tkv * p.ldkv;
  const float* do_b = p.dout + (int64_t)b * p.Tq * p.C + head * D;
  const float* o_b = p.o + (int64_t)b * p.Tq * p.C + head * D;
  const int n_tiles = (p.Tkv + AB_T - 1) / AB_T;

  load_cols<DP>(q_b + qoff, p.ldq, q0, p.Tq, D, Qt);
  load_cols<DP>(do_b, p.C, q0, p.Tq, D, dOt);
  __syncthreads();
  {
    // delta_i = <dO_i, O_i>: 4 threads per row
    const int row = tid >> 2, part = tid & 3;
    float s = 0.f;
    if (q0 + row < p.Tq) {
      const float* orow = o_b + (int64_t)(q0 + row) * p.C;
      for (int d = part * (D / 4); d < (part + 1) * (D / 4); ++d) s = fmaf(dOt[d * AB_T + row], orow[d], s);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    if (part == 0) {
      delta_s[row] = s;
      if (q0 + row < p.Tq) p.delta[(int64_t)bh * p.Tq + q0 + row] = s;
    }
  }

  // ---- pass 1: row-wise log-sum-exp (base 2) of the scaled scores --------------------------------
  float m[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { m[i] = -INFINITY; l[i] = 0.f; }
  for (int j = 0; j < n_tiles; ++j) {
    const int k0 = j * AB_T;
    __syncthreads();
    load_cols<DP>(kv_b + koff, p.ldkv, k0, p.Tkv, D, buf);
    __syncthreads();
    float s[4][4];
    mm_tt<DP>(Qt, buf, ty, tx, s);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        s[i][c] = (k0 + tx * 4 + c < p.Tkv) ? s[i][c] * p.scale_log2 : -INFINITY;
        mx = fmaxf(mx, s[i][c]);
      }
      mx = group16_max(mx);
      const float mn = fmaxf(m[i], mx);           // finite: every tile holds at least one valid key
      float rs = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) rs += exp2f(s[i][c] - mn);
      rs = group16_sum(rs);
      l[i] = l[i] * exp2f(m[i] - mn) + rs;
      m[i] = mn;
    }
  }
  float lse[4], dl[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    lse[i] = m[i] + log2f(l[i]);
    dl[i] = delta_s[ty * 4 + i];
    if (tx == 0 && q0 + ty * 4 + i < p.Tq) p.lse[(int64_t)bh * p.Tq + q0 + ty * 4 + i] = lse[i];
  }

  // ---- pass 2: dQ = s^2 * sum_j dS_j K_j -------------------------------------------------------
  float dq[4][DC];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < DC; ++c) dq[i][c] = 0.f;
  for (int j = 0; j < n_tiles; ++j) {
    const int k0 = j * AB_T;
    float s[4][4], dp[4][4];
    __syncthreads();
    load_cols<DP>(kv_b + koff, p.ldkv, k0, p.Tkv, D, buf);
    __syncthreads();
    mm_tt<DP>(Qt, buf, ty, tx, s);
    __syncthreads();
    load_cols<DP>(kv_b + voff, p.ldkv, k0, p.Tkv, D, buf);
    __syncthreads();
    mm_tt<DP>(dOt, buf, ty, tx, dp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float ds[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float pr = (k0 + tx * 4 + c < p.Tkv) ? exp2f(fmaf(s[i][c], p.scale_log2, -lse[i])) : 0.f;
        ds[c] = pr * (dp[i][c] - dl[i]);
      }
      *reinterpret_cast<float4*>(dSs + (ty * 4 + i) * AB_LD + tx * 4) = make_float4(ds[0], ds[1], ds[2], ds[3]);
    }
    __syncthreads();
    load_rows<DP>(kv_b + koff, p.ldkv, k0, p.Tkv, D, buf);
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < AB_T; ++k) {
      float kv[DC];
#pragma unroll
      for (int c = 0; c < DC; ++c) kv[c] = buf[k * DP + tx * DC + c];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float a = dSs[(ty * 4 + i) * AB_LD + k];
#pragma unroll
        for (int c = 0; c < DC; ++c) dq[i][c] = fmaf(a, kv[c], dq[i][c]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = q0 + ty * 4 + i;
    if (q >= p.Tq) continue;
    float* dst = p.dq + ((int64_t)b * p.Tq + q) * p.ldq + qoff + tx * DC;
#pragma unroll
    for (int c = 0; c < DC; ++c)
      if (tx * DC + c < D) dst[c] = dq[i][c] * p.scale2;
  }
}

// ---------------------------------------------------------------------------------------------
// kernel 2: per 64-key tile -- dK, dV
// ---------------------------------------------------------------------------------------------
template <int DP>
__global__ void __launch_bounds__(256)
attn_bwd_dkv_wide_kernel(const AttnBwdParams p, int D) {
  constexpr int DC = DP / 16;
  extern __shared__ __align__(16) float sm[];
  float* Kt = sm;                   // [DP][64]
  float* Vt = Kt + DP * AB_T;       // [DP][64]
  float* buf = Vt + DP * AB_T;      // Q^T, dO^T [DP][64] or Q, dO [64][DP]
  float* Ps = buf + DP * AB_T;      // [64 q][AB_LD]
  float* dSs = Ps + AB_T * AB_LD;   // [64 q][AB_LD]
  float* lse_s = dSs + AB_T * AB_LD;
  float* delta_s = lse_s + AB_T;

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int bh = blockIdx.y, b = bh / p.heads, head = bh % p.heads;
  const int k0 = blockIdx.x * AB_T;
  int qoff, koff, voff;
  head_offsets(p, head, qoff, koff, voff);
  const float* q_b = p.q + (int64_t)b * p.Tq * p.ldq;
  const float* kv_b = p.kv + (int64_t)b * p.Tkv * p.ldkv;
  const float* do_b = p.dout + (int64_t)b * p.Tq * p.C + head * D;
  const int n_tiles = (p.Tq + AB_T - 1) / AB_T;

  load_cols<DP>(kv_b + koff, p.ldkv, k0, p.Tkv, D, Kt);
  load_cols<DP>(kv_b + voff, p.ldkv, k0, p.Tkv, D, Vt);

  float dk[4][DC], dv[4][DC];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < DC; ++c) { dk[i][c] = 0.f; dv[i][c] = 0.f; }

  for (int j = 0; j < n_tiles; ++j) {
    const int q0 = j * AB_T;
    float s[4][4], dp[4][4];
    __syncthreads();
    load_cols<DP>(q_b + qoff, p.ldq, q0, p.Tq, D, buf);
    if (tid < AB_T) {
      const bool ok = q0 + tid < p.Tq;
      lse_s[tid] = ok ? p.lse[(int64_t)bh * p.Tq + q0 + tid] : 0.f;
      delta_s[tid] = ok ? p.delta[(int64_t)bh * p.Tq + q0 + tid] : 0.f;
    }
    __syncthreads();
    mm_tt<DP>(buf, Kt, ty, tx, s);      // rows = queries (ty), cols = keys (tx)
    __syncthreads();
    load_cols<DP>(do_b, p.C, q0, p.Tq, D, buf);
    __syncthreads();
    mm_tt<DP>(buf, Vt, ty, tx, dp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = ty * 4 + i;
      const bool qok = q0 + r < p.Tq;
      float pr[4], ds[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        pr[c] = (qok && k0 + tx * 4 + c < p.Tkv) ? exp2f(fmaf(s[i][c], p.scale_log2, -lse_s[r])) : 0.f;
        ds[c] = pr[c] * (dp[i][c] - delta_s[r]);
      }
      *reinterpret_cast<float4*>(Ps + r * AB_LD + tx * 4) = make_float4(pr[0], pr[1], pr[2], pr[3]);
      *reinterpret_cast<float4*>(dSs + r * AB_LD + tx * 4) = make_float4(ds[0], ds[1], ds[2], ds[3]);
    }
    __syncthreads();
    // dK[k][d] += sum_q dS[q][k] Q[q][d]   (keys ty*4.., d tx*DC..)
    load_rows<DP>(q_b + qoff, p.ldq, q0, p.Tq, D, buf);
    __syncthreads();
#pragma unroll 4
    for (int q = 0; q < AB_T; ++q) {
      const float4 da = *reinterpret_cast<const float4*>(dSs + q * AB_LD + ty * 4);
      const float dsv[4] = {da.x, da.y, da.z, da.w};
      float qv[DC];
#pragma unroll
      for (int c = 0; c < DC; ++c) qv[c] = buf[q * DP + tx * DC + c];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < DC; ++c) dk[i][c] = fmaf(dsv[i], qv[c], dk[i][c]);
    }
    __syncthreads();
    // dV[k][d] += sum_q P[q][k] dO[q][d]
    load_rows<DP>(do_b, p.C, q0, p.Tq, D, buf);
    __syncthreads();
#pragma unroll 4
    for (int q = 0; q < AB_T; ++q) {
      const float4 pa = *reinterpret_cast<const float4*>(Ps + q * AB_LD + ty * 4);
      const float pv[4] = {pa.x, pa.y, pa.z, pa.w};
      float dov[DC];
#pragma unroll
      for (int c = 0; c < DC; ++c) dov[c] = buf[q * DP + tx * DC + c];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < DC; ++c) dv[i][c] = fmaf(pv[i], dov[c], dv[i][c]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = k0 + ty * 4 + i;
    if (k >= p.Tkv) continue;
    float* row = p.dkv + ((int64_t)b * p.Tkv + k) * p.ldkv;
#pragma unroll
    for (int c = 0; c < DC; ++c) {
      if (tx * DC + c >= D) continue;
      row[koff + tx * DC + c] = dk[i][c] * p.scale2;
      row[voff + tx * DC + c] = dv[i][c];
    }
  }
}

template <int DP>
int launch_bwd_wide_dp(const AttnBwdParams& p, int D, int B, cudaStream_t s) {
  constexpr size_t sm1 = (size_t)(3 * DP * AB_T + AB_T * AB_LD + AB_T) * sizeof(float);
  constexpr size_t sm2 = (size_t)(3 * DP * AB_T + 2 * AB_T * AB_LD + 2 * AB_T) * sizeof(float);
  static_assert(sm1 <= 232448 && sm2 <= 232448, "wide attention backward: shared memory over the per-CTA limit");
  BBDM_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dq_wide_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
  BBDM_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dkv_wide_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
  attn_bwd_dq_wide_kernel<DP><<<dim3((p.Tq + AB_T - 1) / AB_T, B * p.heads), 256, sm1, s>>>(p, D);
  BBDM_LAUNCH_CHECK();
  attn_bwd_dkv_wide_kernel<DP><<<dim3((p.Tkv + AB_T - 1) / AB_T, B * p.heads), 256, sm2, s>>>(p, D);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // namespace

int launch_attention_bwd_wide(const char* what, const AttnBwdParams& p, int D, int B, cudaStream_t s) {
  if (D % 8 == 0 && D > 128 && D <= 256) {
    switch ((D + 31) / 32 * 32) {
#define BBDM_ABW(DP) \
      case DP: return launch_bwd_wide_dp<DP>(p, D, B, s);
      BBDM_ATTN_WIDE_PADDED_DIMS(BBDM_ABW)
#undef BBDM_ABW
    }
  }
  BBDM_REQUIRE(false, "%s: head_dim %d not supported (a multiple of 8 up to 256)", what, D);
}

}  // namespace bbdm
