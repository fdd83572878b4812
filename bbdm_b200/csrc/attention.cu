// Flash-style multi-head attention core for AttentionBlock (openaimodel.py:350-413).
//   out = softmax((q*s)(k*s)^T) v,  s = head_dim^-1/4, softmax in fp32, no T x T buffer.
// Tensor-core products use split-bf16 operands (hi.hi + lo.hi + hi.lo, fp32 accumulate) so the
// result is fp32-class accurate.  mma.sync.m16n8k16 variant reading fp32 qkv: serves UNets whose
// qkv conv runs on the fp32 direct kernel (unaligned channel counts).  The template UNets
// (head_dim 64) use the warp-specialised wgmma kernel in attention_tc.cu.
//
// CTA = 4 warps x 16 query rows = 64 queries of one (batch, head); KV tiles of 64 keys.  The K and V^T
// tiles live in static shared memory for head_dim <= 64; at 128 they take 71.7 KB, over the 48 KB static
// limit, so that instance stages them in dynamic shared memory with the same layout.  At 128 the Q fragments
// (64 registers) are also parked there, in fragment order (each thread reads back only its own 16-byte words),
// and the S product runs k-step outer, n-tile inner: the same products in the same order per S entry.
#include "common.cuh"

namespace bbdm {

__device__ __forceinline__ void mma_bf16_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void split2(float x, float y, uint32_t& hi, uint32_t& lo) { split2x(x, y, hi, lo); }

constexpr int ATT_KT = 64;          // keys per tile
constexpr int ATT_LDV = ATT_KT + 8;   // padded V^T row (bf16 elements)

template <int D>
__device__ __forceinline__ void attention_body(const float* __restrict__ qkv, int T, int C, int heads, int order, float scale,
                                               float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_hi,
                                               __nv_bfloat16* __restrict__ out_lo,
                                               __nv_bfloat16 (&Kh)[ATT_KT][D + 8], __nv_bfloat16 (&Kl)[ATT_KT][D + 8],
                                               __nv_bfloat16 (&Vh)[D][ATT_LDV], __nv_bfloat16 (&Vl)[D][ATT_LDV],
                                               uint4* __restrict__ qfrag) {     // D > 64: [KS][hi, lo][128 threads]
  constexpr int KT = ATT_KT;        // keys per tile
  constexpr int KS = D / 16;        // k-steps over head_dim

  const int bh = blockIdx.y;
  const int b = bh / heads, head = bh % heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int64_t row_stride = 3 * (int64_t)C;
  int qoff, koff, voff;
  if (order == 0) { qoff = head * 3 * D; koff = qoff + D; voff = qoff + 2 * D; }
  else { qoff = head * D; koff = C + head * D; voff = 2 * C + head * D; }
  const float* base = qkv + (int64_t)b * T * row_stride;

  // ---- Q fragments (scaled, split) for this warp's 16 rows --------------------------------
  const int q0 = blockIdx.x * 64 + warp * 16;
  uint32_t qh[KS][4], ql[KS][4];
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {        // h2: 0 -> d offset 0, 1 -> d offset 8
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) {      // r2: row g / g+8
        const int qr = q0 + g + r2 * 8;
        float2 v = make_float2(0.f, 0.f);
        if (qr < T) v = *reinterpret_cast<const float2*>(base + qr * row_stride + qoff + ks * 16 + h2 * 8 + 2 * t);
        split2(v.x * scale, v.y * scale, qh[ks][h2 * 2 + r2], ql[ks][h2 * 2 + r2]);
      }
    }
  }
  if constexpr (D > 64) {
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      qfrag[(2 * ks) * 128 + threadIdx.x] = make_uint4(qh[ks][0], qh[ks][1], qh[ks][2], qh[ks][3]);
      qfrag[(2 * ks + 1) * 128 + threadIdx.x] = make_uint4(ql[ks][0], ql[ks][1], ql[ks][2], ql[ks][3]);
    }
  }

  float o[D / 8][4];
#pragma unroll
  for (int j = 0; j < D / 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  for (int k0 = 0; k0 < T; k0 += KT) {
    // ---- stage K (scaled) and V^T tiles, split into hi/lo planes --------------------------
    for (int idx = threadIdx.x; idx < KT * (D / 4); idx += 128) {
      const int key = idx / (D / 4), c4 = (idx % (D / 4)) * 4;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (k0 + key < T) {
        const float* rp = base + (int64_t)(k0 + key) * row_stride;
        kv = ld_f4(rp + koff + c4);
        vv = ld_f4(rp + voff + c4);
      }
      kv.x *= scale; kv.y *= scale; kv.z *= scale; kv.w *= scale;
      uint2 h, l;
      split4(kv, h, l);
      *reinterpret_cast<uint2*>(&Kh[key][c4]) = h;
      *reinterpret_cast<uint2*>(&Kl[key][c4]) = l;
      __nv_bfloat16 vh, vl;
      split_bf16(vv.x, vh, vl); Vh[c4 + 0][key] = vh; Vl[c4 + 0][key] = vl;
      split_bf16(vv.y, vh, vl); Vh[c4 + 1][key] = vh; Vl[c4 + 1][key] = vl;
      split_bf16(vv.z, vh, vl); Vh[c4 + 2][key] = vh; Vl[c4 + 2][key] = vl;
      split_bf16(vv.w, vh, vl); Vh[c4 + 3][key] = vh; Vl[c4 + 3][key] = vl;
    }
    __syncthreads();

    // ---- S = Q K^T (16 x 64 per warp) -----------------------------------------------------
    float s[KT / 8][4];
    if constexpr (D > 64) {
#pragma unroll
      for (int j = 0; j < KT / 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        const uint4 h4 = qfrag[(2 * ks) * 128 + threadIdx.x], l4 = qfrag[(2 * ks + 1) * 128 + threadIdx.x];
        const uint32_t qh1[4] = {h4.x, h4.y, h4.z, h4.w}, ql1[4] = {l4.x, l4.y, l4.z, l4.w};
#pragma unroll
        for (int j = 0; j < KT / 8; ++j) {
          const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(&Kh[j * 8 + g][ks * 16 + 2 * t]);
          const uint32_t bh1 = *reinterpret_cast<const uint32_t*>(&Kh[j * 8 + g][ks * 16 + 8 + 2 * t]);
          const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(&Kl[j * 8 + g][ks * 16 + 2 * t]);
          const uint32_t bl1 = *reinterpret_cast<const uint32_t*>(&Kl[j * 8 + g][ks * 16 + 8 + 2 * t]);
          mma_bf16_16816(s[j], ql1, bh0, bh1);
          mma_bf16_16816(s[j], qh1, bl0, bl1);
          mma_bf16_16816(s[j], qh1, bh0, bh1);
        }
      }
    } else
#pragma unroll
    for (int j = 0; j < KT / 8; ++j) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(&Kh[j * 8 + g][ks * 16 + 2 * t]);
        const uint32_t bh1 = *reinterpret_cast<const uint32_t*>(&Kh[j * 8 + g][ks * 16 + 8 + 2 * t]);
        const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(&Kl[j * 8 + g][ks * 16 + 2 * t]);
        const uint32_t bl1 = *reinterpret_cast<const uint32_t*>(&Kl[j * 8 + g][ks * 16 + 8 + 2 * t]);
        // A fragment register order: a0=(g, k lo) a1=(g+8, k lo) a2=(g, k hi) a3=(g+8, k hi)
        mma_bf16_16816(s[j], ql[ks], bh0, bh1);
        mma_bf16_16816(s[j], qh[ks], bl0, bl1);
        mma_bf16_16816(s[j], qh[ks], bh0, bh1);
      }
    }
    // ---- mask keys beyond T, online softmax ------------------------------------------------
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < KT / 8; ++j) {
      const int key = k0 + j * 8 + 2 * t;
      if (key >= T) { s[j][0] = -INFINITY; s[j][2] = -INFINITY; }
      if (key + 1 >= T) { s[j][1] = -INFINITY; s[j][3] = -INFINITY; }
      mx[0] = fmaxf(mx[0], fmaxf(s[j][0], s[j][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[j][2], s[j][3]));
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      corr[r] = (m_run[r] == -INFINITY) ? 0.f : expf(m_run[r] - m_new);
      m_run[r] = m_new;
      l_run[r] *= corr[r];
    }
#pragma unroll
    for (int j = 0; j < D / 8; ++j) { o[j][0] *= corr[0]; o[j][1] *= corr[0]; o[j][2] *= corr[1]; o[j][3] *= corr[1]; }
#pragma unroll
    for (int j = 0; j < KT / 8; ++j) {
      s[j][0] = expf(s[j][0] - m_run[0]); s[j][1] = expf(s[j][1] - m_run[0]);
      s[j][2] = expf(s[j][2] - m_run[1]); s[j][3] = expf(s[j][3] - m_run[1]);
      l_run[0] += s[j][0] + s[j][1];
      l_run[1] += s[j][2] + s[j][3];
    }
    // ---- O += P V.  The tensor core's accumulator add truncates, so each KV tile's product is
    // formed from a zero accumulator (12 k-steps) and added to O with a round-to-nearest fp32 add.
#pragma unroll
    for (int jd = 0; jd < D / 8; ++jd) {
      float ot[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk) {
        uint32_t ph[4], pl[4];
        split2(s[2 * kk][0], s[2 * kk][1], ph[0], pl[0]);          // row g,   keys 2t,2t+1
        split2(s[2 * kk][2], s[2 * kk][3], ph[1], pl[1]);          // row g+8
        split2(s[2 * kk + 1][0], s[2 * kk + 1][1], ph[2], pl[2]);  // row g,   keys 8+2t,..
        split2(s[2 * kk + 1][2], s[2 * kk + 1][3], ph[3], pl[3]);  // row g+8
        const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(&Vh[jd * 8 + g][kk * 16 + 2 * t]);
        const uint32_t bh1 = *reinterpret_cast<const uint32_t*>(&Vh[jd * 8 + g][kk * 16 + 8 + 2 * t]);
        const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(&Vl[jd * 8 + g][kk * 16 + 2 * t]);
        const uint32_t bl1 = *reinterpret_cast<const uint32_t*>(&Vl[jd * 8 + g][kk * 16 + 8 + 2 * t]);
        mma_bf16_16816(ot, pl, bh0, bh1);
        mma_bf16_16816(ot, ph, bl0, bl1);
        mma_bf16_16816(ot, ph, bh0, bh1);
      }
      o[jd][0] += ot[0]; o[jd][1] += ot[1]; o[jd][2] += ot[2]; o[jd][3] += ot[3];
    }
    __syncthreads();
  }

  // ---- normalise and store ---------------------------------------------------------------
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    const int qr = q0 + g + r2 * 8;
    if (qr >= T) continue;
    const float inv = 1.0f / l_run[r2];
    const int64_t off = ((int64_t)b * T + qr) * C + head * D + 2 * t;
#pragma unroll
    for (int jd = 0; jd < D / 8; ++jd) {
      const float x = o[jd][2 * r2] * inv, y = o[jd][2 * r2 + 1] * inv;
      if (out_f32) *reinterpret_cast<float2*>(out_f32 + off + jd * 8) = make_float2(x, y);
      if (out_hi) {
        uint32_t h, l;
        split2(x, y, h, l);
        *reinterpret_cast<uint32_t*>(out_hi + off + jd * 8) = h;
        *reinterpret_cast<uint32_t*>(out_lo + off + jd * 8) = l;
      }
    }
  }
}

template <int D>
__global__ void __launch_bounds__(128)
attention_kernel(const float* __restrict__ qkv, int T, int C, int heads, int order, float scale,
                 float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_hi,
                 __nv_bfloat16* __restrict__ out_lo) {
  constexpr int LDK = D + 8;        // padded row (bf16 elements)
  __shared__ __align__(16) __nv_bfloat16 Kh[ATT_KT][LDK], Kl[ATT_KT][LDK];
  __shared__ __align__(16) __nv_bfloat16 Vh[D][ATT_LDV], Vl[D][ATT_LDV];
  attention_body<D>(qkv, T, C, heads, order, scale, out_f32, out_hi, out_lo, Kh, Kl, Vh, Vl, nullptr);
}

// Kh Kl Vh Vl, then the Q fragments: 2 planes x D/16 k-steps x 128 threads x 16 B
template <int D>
constexpr size_t attention_dyn_smem() { return (size_t)2 * (ATT_KT * (D + 8) + D * ATT_LDV) * 2 + (size_t)2 * (D / 16) * 128 * 16; }

template <int D>
__global__ void __launch_bounds__(128)
attention_kernel_dyn(const float* __restrict__ qkv, int T, int C, int heads, int order, float scale,
                     float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_hi,
                     __nv_bfloat16* __restrict__ out_lo) {
  typedef __nv_bfloat16 KTile[ATT_KT][D + 8];
  typedef __nv_bfloat16 VTile[D][ATT_LDV];
  extern __shared__ __align__(16) uint8_t att_smem[];     // Kh Kl Vh Vl Q-fragments, each 16-byte aligned
  KTile& Kh = *reinterpret_cast<KTile*>(att_smem);
  KTile& Kl = *reinterpret_cast<KTile*>(att_smem + sizeof(KTile));
  VTile& Vh = *reinterpret_cast<VTile*>(att_smem + 2 * sizeof(KTile));
  VTile& Vl = *reinterpret_cast<VTile*>(att_smem + 2 * sizeof(KTile) + sizeof(VTile));
  uint4* qfrag = reinterpret_cast<uint4*>(att_smem + 2 * sizeof(KTile) + 2 * sizeof(VTile));
  attention_body<D>(qkv, T, C, heads, order, scale, out_f32, out_hi, out_lo, Kh, Kl, Vh, Vl, qfrag);
}

}  // namespace bbdm

using namespace bbdm;

extern "C" int bbdm_attention(const float* qkv, int B, int T, int C, int heads, int order,
                              float* out_f32, void* out_hi, void* out_lo, void* stream) {
  BBDM_REQUIRE(qkv && (out_f32 || (out_hi && out_lo)), "attention: null pointer");
  BBDM_REQUIRE((out_hi == nullptr) == (out_lo == nullptr), "attention: hi/lo must come in pairs");
  BBDM_REQUIRE(B > 0 && T > 0 && heads > 0 && C % heads == 0, "attention: bad shape");
  BBDM_REQUIRE(order == 0 || order == 1, "attention: order must be 0 (legacy) or 1");
  const int D = C / heads;
  BBDM_REQUIRE((int64_t)B * heads <= 65535, "attention: B*heads too large");
  dim3 grid((T + 63) / 64, B * heads);
  cudaStream_t s = (cudaStream_t)stream;
  __nv_bfloat16* oh = (__nv_bfloat16*)out_hi;
  __nv_bfloat16* ol = (__nv_bfloat16*)out_lo;
  // the reference multiplies q and k by the python double 1/sqrt(sqrt(ch)) rounded to fp32
  const float scale = (float)(1.0 / sqrt(sqrt((double)D)));
  if (D == 64) attention_kernel<64><<<grid, 128, 0, s>>>(qkv, T, C, heads, order, scale, out_f32, oh, ol);
  else if (D == 32) attention_kernel<32><<<grid, 128, 0, s>>>(qkv, T, C, heads, order, scale, out_f32, oh, ol);
  else if (D == 16) attention_kernel<16><<<grid, 128, 0, s>>>(qkv, T, C, heads, order, scale, out_f32, oh, ol);
  else if (D == 128) {
    constexpr size_t smem = attention_dyn_smem<128>();
    static DeviceOnce cfgd;
    if (cfgd.need()) {
      BBDM_CUDA_CHECK(cudaFuncSetAttribute(attention_kernel_dyn<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      cfgd.mark();
    }
    attention_kernel_dyn<128><<<grid, 128, smem, s>>>(qkv, T, C, heads, order, scale, out_f32, oh, ol);
  } else {
    set_error("attention: head_dim %d not supported (16, 32, 64, 128)", D);
    return BBDM_E_UNSUPPORTED;
  }
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}
