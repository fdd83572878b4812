// Shared pieces of the flash-style attention backward: its parameter block, the fp32 tile loader and the register
// micro-tile product (attention_bwd.cu: head_dim <= 128; attention_bwd_wide.cu: 136 to 256).
#pragma once
#include "common.cuh"

namespace bbdm {

constexpr int AB_T = 64;           // tile edge (queries and keys)
constexpr int AB_LD = AB_T + 4;    // row stride of the P / dS tiles (float4-aligned, conflict-free)
template <int D>
constexpr int ab_dp() { return (D + 15) / 16 * 16; }   // head_dim padded to the 16 column threads

// Queries come from q [B, Tq, ldq], keys and values from kv [B, Tkv, ldkv] (the same tensor for self-attention);
// head h reads columns q_base + h*q_hstride (q), k_base / v_base + h*kv_hstride (k, v) and its gradients go to the
// same columns of dq / dkv, whose row strides equal ldq / ldkv.
struct AttnBwdParams {
  const float* q; const float* kv; const float* o; const float* dout; float* dq; float* dkv;
  float* lse; float* delta;        // [B*heads, Tq]
  int Tq, Tkv, C, heads;
  int64_t ldq, ldkv;
  int q_base, k_base, v_base, q_hstride, kv_hstride;
  float scale2, scale_log2;
};

__device__ __forceinline__ void head_offsets(const AttnBwdParams& p, int head, int& qoff, int& koff, int& voff) {
  qoff = p.q_base + head * p.q_hstride;
  koff = p.k_base + head * p.kv_hstride;
  voff = p.v_base + head * p.kv_hstride;
}

// 64 rows x D columns of a [*, ld] fp32 matrix -> transposed tile dst_t[DP][64] (and row-major dst_r[64][DP]),
// zero past row T and past column D
template <int D>
__device__ __forceinline__ void load_tile(const float* __restrict__ src, int64_t ld, int t0, int T, float* dst_t, float* dst_r) {
  constexpr int DP = ab_dp<D>();
  for (int i = threadIdx.x; i < AB_T * (DP / 4); i += 256) {
    const int row = i % AB_T, ch = i / AB_T;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t0 + row < T && (D == DP || ch * 4 < D)) v = ld_f4(src + (int64_t)(t0 + row) * ld + ch * 4);
    dst_t[(ch * 4 + 0) * AB_T + row] = v.x;
    dst_t[(ch * 4 + 1) * AB_T + row] = v.y;
    dst_t[(ch * 4 + 2) * AB_T + row] = v.z;
    dst_t[(ch * 4 + 3) * AB_T + row] = v.w;
    if (dst_r) *reinterpret_cast<float4*>(dst_r + row * DP + ch * 4) = v;
  }
}

// acc[i][j] = sum_d At[d][ty*4+i] * Bt[d][tx*4+j]
template <int D>
__device__ __forceinline__ void mm_tt(const float* At, const float* Bt, int ty, int tx, float (&acc)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 8
  for (int d = 0; d < D; ++d) {
    const float4 a = *reinterpret_cast<const float4*>(At + d * AB_T + ty * 4);
    const float4 b = *reinterpret_cast<const float4*>(Bt + d * AB_T + tx * 4);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
  }
}

__device__ __forceinline__ float group16_max(float v) {
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float group16_sum(float v) {
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Head dims 136 to 256 (attention_bwd_wide.cu).  Any other head_dim fails here with BBDM_E_INVALID.
int launch_attention_bwd_wide(const char* what, const AttnBwdParams& p, int D, int B, cudaStream_t s);

}  // namespace bbdm
