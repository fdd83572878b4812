// Backward of the multi-head softmax attention core (training path), FlashAttention-style: the
// T x T probability matrix is recomputed tile by tile, never materialised (the reference's autograd
// keeps [B*heads, T, T] fp32 -- 17 GB at T = 4096, B = 16 -- and recomputes it under checkpoint(),
// openaimodel.py:318, util.py:119-148).
//
//   forward (QKVAttentionLegacy / QKVAttention, openaimodel.py:350-413):
//     S = (q s)(k s)^T, s = D^-1/4 ;  P = softmax_row(S) ;  O = P V
//   given dO:
//     delta_i = sum_d dO_id O_id            L_i = log2 sum_j 2^(S_ij log2e)          (kernel 1)
//     P_ij = 2^(S_ij log2e - L_i) ;  dP = dO V^T ;  dS = P o (dP - delta)
//     dQ = s^2 dS K   (kernel 1, one CTA per 64-query tile, loops over the key tiles twice: L, then dQ)
//     dK = s^2 dS^T Q ;  dV = P^T dO   (kernel 2, one CTA per 64-key tile, loops over the query tiles)
//
// Exact fp32 FMA arithmetic on CUDA cores (64x64 tiles, 4x4 register micro-tiles, operands staged in
// shared memory in both orientations); deterministic (no atomics).  The attention core is <= 1.7 % of
// the UNet's FLOPs, so this kernel is about correctness and memory, not the tensor pipe.
// A head_dim D that is not a multiple of 16 is staged at DP = D rounded up to 16 columns, zero past D, so that the
// 16 column threads of dQ / dK / dV hold DP / 16 columns each; only the columns < D are stored.  With D == DP the
// padding tests are compile-time constants.
#include "attention_bwd.cuh"

namespace bbdm {

// ---------------------------------------------------------------------------------------------
// kernel 1: per 64-query tile -- delta, log-sum-exp, dQ
// ---------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(256)
attn_bwd_dq_kernel(const AttnBwdParams p) {
  constexpr int DP = ab_dp<D>();
  constexpr int DC = DP / 16;       // dQ columns per thread
  extern __shared__ __align__(16) float sm[];
  float* Qt = sm;                   // [DP][64]
  float* dOt = Qt + DP * AB_T;      // [DP][64]
  float* Kt = dOt + DP * AB_T;      // [DP][64]
  float* Vt = Kt + DP * AB_T;       // [DP][64]
  float* Ks = Vt + DP * AB_T;       // [64][DP]
  float* dSs = Ks + AB_T * DP;      // [64][AB_LD]
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

  load_tile<D>(q_b + qoff, p.ldq, q0, p.Tq, Qt, nullptr);
  load_tile<D>(do_b, p.C, q0, p.Tq, dOt, nullptr);
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
    load_tile<D>(kv_b + koff, p.ldkv, k0, p.Tkv, Kt, nullptr);
    __syncthreads();
    float s[4][4];
    mm_tt<D>(Qt, Kt, ty, tx, s);
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
    __syncthreads();
    load_tile<D>(kv_b + koff, p.ldkv, k0, p.Tkv, Kt, Ks);
    load_tile<D>(kv_b + voff, p.ldkv, k0, p.Tkv, Vt, nullptr);
    __syncthreads();
    float s[4][4], dp[4][4];
    mm_tt<D>(Qt, Kt, ty, tx, s);
    mm_tt<D>(dOt, Vt, ty, tx, dp);
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
#pragma unroll 4
    for (int k = 0; k < AB_T; ++k) {
      float kv[DC];
#pragma unroll
      for (int c = 0; c < DC; ++c) kv[c] = Ks[k * DP + tx * DC + c];
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
      if (D == DP || tx * DC + c < D) dst[c] = dq[i][c] * p.scale2;
  }
}

// ---------------------------------------------------------------------------------------------
// kernel 2: per 64-key tile -- dK, dV
// ---------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(256)
attn_bwd_dkv_kernel(const AttnBwdParams p) {
  constexpr int DP = ab_dp<D>();
  constexpr int DC = DP / 16;
  extern __shared__ __align__(16) float sm[];
  float* Kt = sm;                   // [DP][64]
  float* Vt = Kt + DP * AB_T;
  float* Qt = Vt + DP * AB_T;
  float* dOt = Qt + DP * AB_T;
  float* Qs = dOt + DP * AB_T;      // [64][DP]
  float* dOs = Qs + AB_T * DP;      // [64][DP]
  float* Ps = dOs + AB_T * DP;      // [64 q][AB_LD]
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

  load_tile<D>(kv_b + koff, p.ldkv, k0, p.Tkv, Kt, nullptr);
  load_tile<D>(kv_b + voff, p.ldkv, k0, p.Tkv, Vt, nullptr);

  float dk[4][DC], dv[4][DC];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < DC; ++c) { dk[i][c] = 0.f; dv[i][c] = 0.f; }

  for (int j = 0; j < n_tiles; ++j) {
    const int q0 = j * AB_T;
    __syncthreads();
    load_tile<D>(q_b + qoff, p.ldq, q0, p.Tq, Qt, Qs);
    load_tile<D>(do_b, p.C, q0, p.Tq, dOt, dOs);
    if (tid < AB_T) {
      const bool ok = q0 + tid < p.Tq;
      lse_s[tid] = ok ? p.lse[(int64_t)bh * p.Tq + q0 + tid] : 0.f;
      delta_s[tid] = ok ? p.delta[(int64_t)bh * p.Tq + q0 + tid] : 0.f;
    }
    __syncthreads();
    float s[4][4], dp[4][4];
    mm_tt<D>(Qt, Kt, ty, tx, s);        // rows = queries (ty), cols = keys (tx)
    mm_tt<D>(dOt, Vt, ty, tx, dp);
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
    // dV[k][d] += sum_q P[q][k] dO[q][d] ;  dK[k][d] += sum_q dS[q][k] Q[q][d]   (keys ty*4.., d tx*DC..)
#pragma unroll 4
    for (int q = 0; q < AB_T; ++q) {
      const float4 pa = *reinterpret_cast<const float4*>(Ps + q * AB_LD + ty * 4);
      const float4 da = *reinterpret_cast<const float4*>(dSs + q * AB_LD + ty * 4);
      const float pv[4] = {pa.x, pa.y, pa.z, pa.w}, dsv[4] = {da.x, da.y, da.z, da.w};
      float qv[DC], dov[DC];
#pragma unroll
      for (int c = 0; c < DC; ++c) { qv[c] = Qs[q * DP + tx * DC + c]; dov[c] = dOs[q * DP + tx * DC + c]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < DC; ++c) {
          dv[i][c] = fmaf(pv[i], dov[c], dv[i][c]);
          dk[i][c] = fmaf(dsv[i], qv[c], dk[i][c]);
        }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = k0 + ty * 4 + i;
    if (k >= p.Tkv) continue;
    float* row = p.dkv + ((int64_t)b * p.Tkv + k) * p.ldkv;
#pragma unroll
    for (int c = 0; c < DC; ++c) {
      if (D != DP && tx * DC + c >= D) continue;
      row[koff + tx * DC + c] = dk[i][c] * p.scale2;
      row[voff + tx * DC + c] = dv[i][c];
    }
  }
}

template <int D>
static int launch_bwd(const AttnBwdParams& p, int B, cudaStream_t s) {
  constexpr int DP = ab_dp<D>();
  const size_t sm1 = (size_t)(5 * DP * AB_T + AB_T * AB_LD + AB_T) * sizeof(float);
  const size_t sm2 = (size_t)(6 * DP * AB_T + 2 * AB_T * AB_LD + 2 * AB_T) * sizeof(float);
  BBDM_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dq_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
  BBDM_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dkv_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
  attn_bwd_dq_kernel<D><<<dim3((p.Tq + AB_T - 1) / AB_T, B * p.heads), 256, sm1, s>>>(p);
  BBDM_LAUNCH_CHECK();
  attn_bwd_dkv_kernel<D><<<dim3((p.Tkv + AB_T - 1) / AB_T, B * p.heads), 256, sm2, s>>>(p);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

// shape checks, the D^-1/4 scales and the head_dim dispatch shared by both entry points
static int attention_bwd_launch(const char* what, AttnBwdParams p, int B, void* stream) {
  BBDM_REQUIRE(p.q && p.kv && p.o && p.dout && p.dq && p.dkv && p.lse && p.delta, "%s: null pointer", what);
  BBDM_REQUIRE(B > 0 && p.Tq > 0 && p.Tkv > 0 && p.heads > 0 && p.C % p.heads == 0, "%s: bad shape", what);
  BBDM_REQUIRE((int64_t)B * p.heads <= 65535, "%s: B*heads = %lld exceeds the grid limit", what, (long long)B * p.heads);
  const int D = p.C / p.heads;
  const double scale = 1.0 / sqrt(sqrt((double)D));
  p.scale2 = (float)(scale * scale);
  p.scale_log2 = (float)(scale * scale * 1.4426950408889634);
  cudaStream_t s = (cudaStream_t)stream;
  // at D = 128 kernel 2 takes 231,936 B of the 232,448 B opt-in shared memory; DP <= 128 takes no more.  Wider heads
  // run on the kernels of attention_bwd_wide.cu.
#define BBDM_AB(DD) \
  case DD: return launch_bwd<DD>(p, B, s);
  switch (D) {
    BBDM_FOR_ATTN_HEAD_DIMS(BBDM_AB)
    default: return launch_attention_bwd_wide(what, p, D, B, s);
  }
#undef BBDM_AB
  return BBDM_OK;
}

}  // namespace bbdm

using namespace bbdm;

// dqkv [B,T,3C] = gradient of the attention core w.r.t. its qkv input, given out = attention(qkv)
// [B,T,C] (saved from the forward) and dout [B,T,C].  lse / delta: [B*heads*T] fp32 workspaces.
extern "C" int bbdm_attention_bwd(const float* qkv, const float* out, const float* dout, int B, int T, int C, int heads,
                                  int order, float* dqkv, float* lse, float* delta, void* stream) {
  BBDM_REQUIRE(order == 0 || order == 1, "attention_bwd: bad shape");
  BBDM_REQUIRE(heads > 0 && C % heads == 0, "attention_bwd: bad shape");
  const int D = C / heads;
  AttnBwdParams p{};
  p.q = p.kv = qkv; p.dq = p.dkv = dqkv;
  p.o = out; p.dout = dout; p.lse = lse; p.delta = delta;
  p.Tq = p.Tkv = T; p.C = C; p.heads = heads;
  p.ldq = p.ldkv = 3 * (int64_t)C;
  if (order == 0) { p.q_base = 0; p.k_base = D; p.v_base = 2 * D; p.q_hstride = p.kv_hstride = 3 * D; }
  else { p.q_base = 0; p.k_base = C; p.v_base = 2 * C; p.q_hstride = p.kv_hstride = D; }
  return attention_bwd_launch("attention_bwd", p, B, stream);
}

// Backward of bbdm_attention_cross: q [B,Tq,C], kv [B,Tkv,2C] (k = columns [0,C), v = [C,2C)) fp32, out [B,Tq,C] saved
// from the forward, dout [B,Tq,C] -> dq [B,Tq,C], dkv [B,Tkv,2C].  lse / delta: [B*heads*Tq] fp32 workspaces.
extern "C" int bbdm_attention_cross_bwd(const float* q, const float* kv, const float* out, const float* dout, int B,
                                        int Tq, int Tkv, int C, int heads, float* dq, float* dkv, float* lse,
                                        float* delta, void* stream) {
  BBDM_REQUIRE(heads > 0 && C % heads == 0, "attention_cross_bwd: bad shape");
  AttnBwdParams p{};
  p.q = q; p.kv = kv; p.o = out; p.dout = dout; p.dq = dq; p.dkv = dkv; p.lse = lse; p.delta = delta;
  p.Tq = Tq; p.Tkv = Tkv; p.C = C; p.heads = heads;
  p.ldq = C; p.ldkv = 2 * (int64_t)C;
  p.q_base = 0; p.k_base = 0; p.v_base = C; p.q_hstride = p.kv_hstride = C / heads;
  return attention_bwd_launch("attention_cross_bwd", p, B, stream);
}
