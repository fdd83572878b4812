// The mma.sync attention core (attention_split.cuh) at head sizes wider than 128: every multiple of 8 up to 256, in all
// three operand forms (pre-split bf16 planes, fp32 qkv, cross-attention).  Same products and the same softmax as the
// narrow kernel: split-bf16 x3 on mma.sync.m16n8k16 with fp32 accumulate, each KV tile's P.V product added to O with a
// round-to-nearest fp32 add, ex2.approx in the log2 domain on the pre-split planes and expf on fp32 qkv, whose q and k
// are multiplied by D^-1/4 before they are split.
//
// The narrow layout does not stretch this far: at DP = 256 its 64-key stages alone would take 270 KB of shared memory
// and its 16 x DP output fragment 128 fp32 registers on top of a 256-thread CTA's budget.  Here:
//   - CTA = 4 warps x 16 query rows = 64 queries of one (batch, head), __launch_bounds__(128): each warp holds its
//     rows' O (DP / 2 registers per thread);
//   - KV tiles of 32 keys, double-buffered with cp.async (16-byte chunks, zero-fill past T and past D);
//   - Q staged in shared memory once (both planes) and read back with ldmatrix per pair of k-steps.
// Shared memory at DP = 256: 2 stages x [Kh, Kl, Vh, Vl] x 32 x 264 bf16 = 135,168 B, Q 2 x 64 x 264 bf16 = 67,584 B:
// 202,752 B of the 232,448 B a CTA may opt in to (F32IN: 200,704 B, see below).
// The kernels are instantiated per padded width DP in {160, 192, 224, 256} with the head_dim D a run-time argument,
// DP - 32 < D <= DP: the loaders zero-fill the columns [D, DP), so Q.K^T is exact, the P.V n-tiles past D are
// skipped, and only the columns < D are stored.
// F32IN copies each raw fp32 K / V row into a row of 2 DP + 8 bf16 and splits it in place, hi in the row's first DP
// elements and lo in the next DP: one warp owns a row, so the split needs no CTA barrier and no fp32 staging buffer.
// These instances live in a translation unit of their own so that the narrow kernels compile to the code they had.
#include "attention_split.cuh"

namespace bbdm {

namespace {

constexpr int kWideKT = 32;    // keys per tile
constexpr int kWideQT = 64;    // queries per CTA
constexpr int kWideThreads = 128;

template <int DP, bool F32IN>
struct WideLayout {
  static constexpr int LD = DP + 8;                                  // Q row (elements): 16 B skew, conflict-free
  static constexpr int KROW = F32IN ? 2 * DP + 8 : DP + 8;           // K / V row stride (elements)
  static constexpr int LOOFF = F32IN ? DP : kWideKT * (DP + 8);      // lo plane offset from the hi plane (elements)
  static constexpr int TSZ = F32IN ? kWideKT * KROW : 2 * kWideKT * KROW;   // one tensor's (K or V) hi + lo
  static constexpr int SSZ = 2 * TSZ;                                // one stage: K then V
  static constexpr size_t smem_bytes() { return ((size_t)2 * SSZ + (size_t)2 * kWideQT * LD) * 2; }
};

__device__ __forceinline__ __nv_bfloat16* attn_smem_wide() {
  extern __shared__ __align__(16) __nv_bfloat16 sm_wide[];
  return sm_wide;
}

// scale: F32IN, s = D^-1/4 applied to q and k; otherwise log2(e) D^-1/2 applied to S
template <int DP, bool F32IN>
__global__ void __launch_bounds__(kWideThreads)
attention_wide_kernel(const AttnOperands ops, int T, int C, int heads, int D, float scale,
                      float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_hi,
                      __nv_bfloat16* __restrict__ out_lo) {
  static_assert(DP % 32 == 0 && DP > 128 && DP <= 256, "padded head_dim: a multiple of 32 in (128, 256]");
  using L = WideLayout<DP, F32IN>;
  constexpr int KT = kWideKT, LD = L::LD, KROW = L::KROW;
  constexpr int KS = DP / 16;             // k-steps over the padded head_dim (even)
  constexpr int CPR = DP / 8;             // 16-byte bf16 chunks per row
  constexpr int FC = DP / 4;              // F32IN: 16-byte chunks per fp32 row
  // [2 stages][K, V][hi, lo][KT][...] + [Qh, Ql][64][LD]
  __nv_bfloat16* const sm = attn_smem_wide();
  __nv_bfloat16* const qs = sm + 2 * L::SSZ;

  const int bh = blockIdx.y;
  const int b = bh / heads, head = bh % heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int64_t rs = ops.rs_kv, rs_q = ops.rs_q;
  const int Tq = ops.Tq;
  const int D8 = D / 8;
  const int qoff = ops.qoff0 + head * ops.hstride, koff = ops.koff0 + head * ops.hstride,
            voff = ops.voff0 + head * ops.hstride;
  const __nv_bfloat16* base_hi = ops.kv_hi + (int64_t)b * T * rs;
  const __nv_bfloat16* base_lo = ops.kv_lo + (int64_t)b * T * rs;
  const __nv_bfloat16* qbase_hi = ops.q_hi + (int64_t)b * Tq * rs_q;
  const __nv_bfloat16* qbase_lo = ops.q_lo + (int64_t)b * Tq * rs_q;
  const float* base_f = ops.qkv + (int64_t)b * T * rs;
  const float* qbase_f = ops.qkv + (int64_t)b * Tq * rs_q;

  // ---- stage loader: K then V, KT rows each, zero past T and past D --------------------------------
  auto load_tile = [&](int stage, int k0) {
    __nv_bfloat16* sbase = sm + stage * L::SSZ;
    if constexpr (F32IN) {                // raw fp32 rows, split in place once the stage has landed
      for (int i = threadIdx.x; i < 2 * KT * FC; i += kWideThreads) {
        const int tensor = i / (KT * FC), rem = i % (KT * FC);
        const int key = rem / FC, c4 = rem % FC * 4;
        const int kk = k0 + key;
        const bool col_ok = c4 < D;
        const bool ok = kk < T && col_ok;
        const float* src = base_f + (int64_t)(ok ? kk : 0) * rs + (tensor ? voff : koff) + (col_ok ? c4 : 0);
        cp_async16(smem_u32(reinterpret_cast<float*>(sbase + tensor * L::TSZ + key * KROW) + c4), src, ok ? 16 : 0);
      }
    } else {
      for (int i = threadIdx.x; i < 4 * KT * CPR; i += kWideThreads) {
        const int plane = i / (KT * CPR), rem = i % (KT * CPR);
        const int key = rem / CPR, ch = rem % CPR;
        const int kk = k0 + key;
        const bool col_ok = ch < D8;
        const bool ok = kk < T && col_ok;
        const __nv_bfloat16* src = ((plane & 1) ? base_lo : base_hi) + (int64_t)(ok ? kk : 0) * rs +
                                   ((plane < 2) ? koff : voff) + (col_ok ? ch : 0) * 8;
        cp_async16(smem_u32(sbase + (plane >> 1) * L::TSZ + (plane & 1) * L::LOOFF + key * KROW + ch * 8), src,
                   ok ? 16 : 0);
      }
    }
  };

  // ---- Q: 64 rows x DP columns per plane, zero-filled past Tq and D ------------------------------------
  if constexpr (F32IN) {                  // scaled and split on the way
    for (int i = threadIdx.x; i < kWideQT * FC; i += kWideThreads) {
      const int row = i / FC, c4 = i % FC * 4;
      const int qr = blockIdx.x * kWideQT + row;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (qr < Tq && c4 < D) v = ld_f4(qbase_f + (int64_t)qr * rs_q + qoff + c4);
      v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
      uint2 h, l;
      split4(v, h, l);
      *reinterpret_cast<uint2*>(qs + row * LD + c4) = h;
      *reinterpret_cast<uint2*>(qs + kWideQT * LD + row * LD + c4) = l;
    }
  } else {
    for (int i = threadIdx.x; i < 2 * kWideQT * CPR; i += kWideThreads) {
      const int plane = i / (kWideQT * CPR), rem = i % (kWideQT * CPR);
      const int row = rem / CPR, ch = rem % CPR;
      const int qr = blockIdx.x * kWideQT + row;
      const bool col_ok = ch < D8;
      const bool ok = qr < Tq && col_ok;
      const __nv_bfloat16* src = (plane ? qbase_lo : qbase_hi) + (int64_t)(ok ? qr : 0) * rs_q + qoff +
                                 (col_ok ? ch : 0) * 8;
      cp_async16(smem_u32(qs + plane * kWideQT * LD + row * LD + ch * 8), src, ok ? 16 : 0);
    }
  }

  float o[DP / 8][4];
#pragma unroll
  for (int j = 0; j < DP / 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  auto softmax_exp = [](float x) {
    if constexpr (F32IN) return expf(x);
    else return ex2_approx(x);
  };

  const uint32_t qh_a = smem_u32(qs), ql_a = qh_a + kWideQT * LD * 2;
  const uint32_t qrow = (uint32_t)(((warp * 16 + (lane & 15)) * LD + (lane >> 4) * 8) * 2);
  const int n_tiles = (T + KT - 1) / KT;
  load_tile(0, 0);                        // (the Q copies join this first group)
  cp_commit();
  for (int it = 0; it < n_tiles; ++it) {
    const int stage = it & 1;
    if (it + 1 < n_tiles) load_tile(stage ^ 1, (it + 1) * KT);
    cp_commit();
    cp_wait<1>();
    __nv_bfloat16* const sbase = sm + stage * L::SSZ;
    if constexpr (F32IN) {
      // warp w splits rows w, w + 4, ... of K then V: every lane reads its chunks of the row, then writes their hi
      // and lo halves over the row (scaling K by s first)
      __syncthreads();
      constexpr int U = (FC + 31) / 32;
      for (int r = warp; r < 2 * KT; r += kWideThreads / 32) {
        const int tensor = r / KT;
        __nv_bfloat16* row = sbase + tensor * L::TSZ + (r % KT) * KROW;
        float4 raw[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (lane + 32 * u < FC) raw[u] = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(row) + 4 * (lane + 32 * u));
        __syncwarp();
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int c = lane + 32 * u;
          if (c >= FC) continue;
          float4 v = raw[u];
          if (tensor == 0) { v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale; }
          uint2 h, l;
          split4(v, h, l);
          *reinterpret_cast<uint2*>(row + 4 * c) = h;
          *reinterpret_cast<uint2*>(row + DP + 4 * c) = l;
        }
        __syncwarp();
      }
    }
    __syncthreads();
    const uint32_t kh_a = smem_u32(sbase), kl_a = kh_a + L::LOOFF * 2;
    const uint32_t vh_a = kh_a + L::TSZ * 2, vl_a = vh_a + L::LOOFF * 2;
    const int k0 = it * KT;

    // ---- S = Q K^T: per k-step pair, the Q fragments from shared memory, then every 8-key n-tile ---------------
    float s[KT / 8][4];
#pragma unroll
    for (int j = 0; j < KT / 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int k2 = 0; k2 < KS / 2; ++k2) {
      uint32_t ah0[4], al0[4], ah1[4], al1[4];
      ldsm_x4(qh_a + qrow + k2 * 64, ah0[0], ah0[1], ah0[2], ah0[3]);
      ldsm_x4(ql_a + qrow + k2 * 64, al0[0], al0[1], al0[2], al0[3]);
      ldsm_x4(qh_a + qrow + k2 * 64 + 32, ah1[0], ah1[1], ah1[2], ah1[3]);
      ldsm_x4(ql_a + qrow + k2 * 64 + 32, al1[0], al1[1], al1[2], al1[3]);
#pragma unroll
      for (int j = 0; j < KT / 8; ++j) {
        const uint32_t roff = (uint32_t)(((j * 8 + (lane & 7)) * KROW + (lane >> 3) * 8) * 2);
        uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
        ldsm_x4(kh_a + roff + k2 * 64, h0, h1, h2, h3);
        ldsm_x4(kl_a + roff + k2 * 64, l0, l1, l2, l3);
        mma16816(s[j], al0, h0, h1);
        mma16816(s[j], ah0, l0, l1);
        mma16816(s[j], ah0, h0, h1);
        mma16816(s[j], al1, h2, h3);
        mma16816(s[j], ah1, l2, l3);
        mma16816(s[j], ah1, h2, h3);
      }
    }
    // ---- scale (log2 domain; F32IN: already scaled), mask keys >= T, online softmax -----------------
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < KT / 8; ++j) {
      const int key = k0 + j * 8 + 2 * t;
      if constexpr (!F32IN) { s[j][0] *= scale; s[j][1] *= scale; s[j][2] *= scale; s[j][3] *= scale; }
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
      corr[r] = (m_run[r] == -INFINITY) ? 0.f : softmax_exp(m_run[r] - m_new);
      m_run[r] = m_new;
      l_run[r] *= corr[r];
    }
#pragma unroll
    for (int j = 0; j < DP / 8; ++j) { o[j][0] *= corr[0]; o[j][1] *= corr[0]; o[j][2] *= corr[1]; o[j][3] *= corr[1]; }
    uint32_t ph[KT / 16][4], pl[KT / 16][4];
#pragma unroll
    for (int j = 0; j < KT / 8; ++j) {
      s[j][0] = softmax_exp(s[j][0] - m_run[0]); s[j][1] = softmax_exp(s[j][1] - m_run[0]);
      s[j][2] = softmax_exp(s[j][2] - m_run[1]); s[j][3] = softmax_exp(s[j][3] - m_run[1]);
      l_run[0] += s[j][0] + s[j][1];
      l_run[1] += s[j][2] + s[j][3];
      // C-fragment of two adjacent n-tiles == A-fragment of one 16-key k-step
      split2x(s[j][0], s[j][1], ph[j >> 1][(j & 1) * 2 + 0], pl[j >> 1][(j & 1) * 2 + 0]);   // row g
      split2x(s[j][2], s[j][3], ph[j >> 1][(j & 1) * 2 + 1], pl[j >> 1][(j & 1) * 2 + 1]);   // row g+8
    }
    // ---- O += P V : V^T fragments by ldmatrix.trans; x4 = (keys 0-7 | 8-15) x (d-tile jd | jd+1) ------
#pragma unroll
    for (int jd2 = 0; jd2 < DP / 16; ++jd2) {
      if (2 * jd2 >= D8) continue;        // both n-tiles past D
      float ot0[4] = {0.f, 0.f, 0.f, 0.f}, ot1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk) {
        const uint32_t voff2 = (uint32_t)(((kk * 16 + (lane >> 3 & 1) * 8 + (lane & 7)) * KROW + jd2 * 16 + (lane >> 4) * 8) * 2);
        uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
        ldsm_x4_t(vh_a + voff2, h0, h1, h2, h3);
        ldsm_x4_t(vl_a + voff2, l0, l1, l2, l3);
        mma16816(ot0, pl[kk], h0, h1);
        mma16816(ot0, ph[kk], l0, l1);
        mma16816(ot0, ph[kk], h0, h1);
        if (2 * jd2 + 1 < D8) {           // the n-tile [D, DP) is zero
          mma16816(ot1, pl[kk], h2, h3);
          mma16816(ot1, ph[kk], l2, l3);
          mma16816(ot1, ph[kk], h2, h3);
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) { o[2 * jd2][c] += ot0[c]; o[2 * jd2 + 1][c] += ot1[c]; }
    }
    __syncthreads();     // all warps done with this stage before it is refilled
  }
  cp_wait<0>();

  // ---- normalise and store the columns < D ----------------------------------------------------------
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const int q0 = blockIdx.x * kWideQT + warp * 16;
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    const int qr = q0 + g + r2 * 8;
    if (qr >= Tq) continue;
    const float inv = 1.0f / l_run[r2];
    const int64_t off = ((int64_t)b * Tq + qr) * C + head * D + 2 * t;
#pragma unroll
    for (int jd = 0; jd < DP / 8; ++jd) {
      if (jd >= D8) continue;
      const float x = o[jd][2 * r2] * inv, y = o[jd][2 * r2 + 1] * inv;
      if (out_f32) *reinterpret_cast<float2*>(out_f32 + off + jd * 8) = make_float2(x, y);
      if (out_hi) {
        uint32_t h, l;
        split2x(x, y, h, l);
        *reinterpret_cast<uint32_t*>(out_hi + off + jd * 8) = h;
        *reinterpret_cast<uint32_t*>(out_lo + off + jd * 8) = l;
      }
    }
  }
}

template <int DP, bool F32IN>
int launch_wide_dp(const AttnOperands& ops, int BH, int T, int C, int heads, int D, float scale, float* out_f32,
                   __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, cudaStream_t s) {
  constexpr size_t smem = WideLayout<DP, F32IN>::smem_bytes();
  static_assert(smem <= 232448, "wide attention: shared memory over the per-CTA limit");
  static DeviceOnce cfgd;
  if (cfgd.need()) {
    BBDM_CUDA_CHECK(cudaFuncSetAttribute(attention_wide_kernel<DP, F32IN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
    cfgd.mark();
  }
  const dim3 grid((ops.Tq + kWideQT - 1) / kWideQT, BH);
  attention_wide_kernel<DP, F32IN><<<grid, kWideThreads, smem, s>>>(ops, T, C, heads, D, scale, out_f32, out_hi, out_lo);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // namespace

template <bool F32IN>
int launch_attention_wide(const char* who, int D, const AttnOperands& ops, dim3 grid, int T, int C, int heads,
                          float scale, float* out_f32, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, cudaStream_t s) {
  if (D % 8 == 0 && D > 128 && D <= 256) {
    switch ((D + 31) / 32 * 32) {
#define BBDM_AW(DP) \
      case DP: return launch_wide_dp<DP, F32IN>(ops, grid.y, T, C, heads, D, scale, out_f32, out_hi, out_lo, s);
      BBDM_ATTN_WIDE_PADDED_DIMS(BBDM_AW)
#undef BBDM_AW
    }
  }
  set_error("%s: head_dim %d not supported (a multiple of 8 up to 256)", who, D);
  return BBDM_E_UNSUPPORTED;
}

template int launch_attention_wide<false>(const char*, int, const AttnOperands&, dim3, int, int, int, float, float*,
                                          __nv_bfloat16*, __nv_bfloat16*, cudaStream_t);
template int launch_attention_wide<true>(const char*, int, const AttnOperands&, dim3, int, int, int, float, float*,
                                         __nv_bfloat16*, __nv_bfloat16*, cudaStream_t);

}  // namespace bbdm
