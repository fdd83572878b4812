// Flash-style attention core on mma.sync, for every head_dim (multiples of 8 up to 128) and operand form the
// tensor-core kernel in attention_tc.cu does not take:
//   - pre-split bf16 planes (bbdm_attention_split, bbdm_attention_cross): the qkv 1x1 conv's epilogue writes
//     qkv as hi/lo bf16 planes, so nothing is converted or re-split here;
//       S = (q . k) * D^-1/2        (= (q D^-1/4) . (k D^-1/4) of openaimodel.py:359-375)
//       O = softmax_fp32(S) v       with the exponential as ex2.approx in the log2 domain;
//   - fp32 qkv (F32IN, bbdm_attention): UNets whose qkv conv runs on the fp32 direct kernel (unaligned channel
//     counts), the VQGAN AttnBlocks and the training forward.  q and k are multiplied by s = D^-1/4 before they
//     are split, as the reference does, S is used as it comes out of the products and the softmax runs on expf.
//
// CTA = 8 warps x 16 query rows = 128 queries of one (batch, head); KV tiles of 64 keys,
// double-buffered with cp.async (16-byte chunks, zero-fill past T); fragments via ldmatrix
// (K plain, V transposed); split-bf16 x3 products on mma.sync.m16n8k16 with fp32 accumulate;
// every KV tile's P.V product starts from a zero accumulator and is added to O with a
// round-to-nearest fp32 add (the tensor core's own accumulate truncates).
// F32IN copies the raw fp32 K and V rows into the span of the stage's hi/lo planes (an fp32 row is the size of
// its two bf16 rows) and splits them in place once the stage has landed.
// Q fragments stay in registers for D <= 64.  At D = 128 they would take 64 registers on top of the 64-float
// output, so the CTA's 128 query rows are staged in shared memory once (both planes, same padded rows) and
// each pair of k-steps is read back with ldmatrix while the S product walks the key n-tiles.
// A head_dim that is not a multiple of the 16-wide k-step runs at DP = D rounded up to 16: the loaders zero-fill
// the columns [D, DP) of Q, K and V (16-byte chunks with src_bytes = 0, as for the keys past T), so Q.K^T is exact,
// the P.V products of the zero columns are skipped and only the columns < D are stored.  With D == DP every
// padding test is a compile-time constant and the code is that of the unpadded kernel.
#pragma once
#include "tc_common.cuh"

namespace bbdm {

__device__ __forceinline__ void mma16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Operand addressing: queries come from (q_hi, q_lo) [B][Tq][rs_q] at column qoff0 + head*hstride, keys / values from
// (kv_hi, kv_lo) [B][T][rs_kv] at koff0 / voff0 + head*hstride.  Self-attention passes the same planes for both
// (T == Tq); cross-attention (SpatialTransformer.attn2, reference attention.py:152-192) a separate K|V tensor with
// its own length T.  F32IN reads q, k and v from the fp32 rows at qkv instead, with the same strides and offsets.
struct AttnOperands {
  const __nv_bfloat16* q_hi; const __nv_bfloat16* q_lo; int64_t rs_q; int qoff0;
  const __nv_bfloat16* kv_hi; const __nv_bfloat16* kv_lo; int64_t rs_kv; int koff0, voff0;
  int hstride, Tq;
  const float* qkv;
};

// Dynamic shared memory of the kernel below.  The fp32-input instances reach it through a symbol of their own: they
// also store fp32 rows there, and one symbol shared with the split-plane instances changes the code the compiler
// generates for those (the head_dim 128 split-plane kernel ran 5-14% slower).
__device__ __forceinline__ __nv_bfloat16* attn_smem_split() {
  extern __shared__ __align__(16) __nv_bfloat16 sm[];
  return sm;
}
__device__ __forceinline__ __nv_bfloat16* attn_smem_f32() {
  extern __shared__ __align__(16) __nv_bfloat16 sm_f32[];
  return sm_f32;
}

// scale: F32IN, s = D^-1/4 applied to q and k; otherwise log2(e) D^-1/2 applied to S
template <int D, bool F32IN>
__global__ void __launch_bounds__(256)
attention_split_kernel(const AttnOperands ops, int T, int C, int heads, float scale,
                       float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_hi,
                       __nv_bfloat16* __restrict__ out_lo) {
  static_assert(D % 8 == 0 && D >= 8 && D <= 128, "head_dim: a multiple of 8 up to 128");
  constexpr int DP = (D + 15) / 16 * 16;  // head_dim padded to the k-step
  constexpr int KT = 64;                  // keys per tile
  constexpr int KS = DP / 16;             // k-steps over head_dim
  constexpr int LD = DP + 8;              // padded smem row (elements): 16 B skew, conflict-free ldmatrix
  constexpr int TILE = KT * LD;           // elements per plane tile
  constexpr bool QS = DP > 64;            // Q fragments from shared memory
  constexpr int FCPR = DP / 4;            // F32IN: 16-byte chunks per fp32 row
  constexpr int FCW = FCPR <= 4 ? 4 : FCPR <= 8 ? 8 : FCPR <= 16 ? 16 : 32;   // ... rounded up to divide 256
  constexpr int FN = 2 * KT * FCW / 256;  // F32IN: chunk slots of a K + V tile per thread
  // [2 stages][Kh, Kl, Vh, Vl][KT][LD] (QS: + [Qh, Ql][128][LD])
  __nv_bfloat16* const sm = F32IN ? attn_smem_f32() : attn_smem_split();

  const int bh = blockIdx.y;
  const int b = bh / heads, head = bh % heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int64_t rs = ops.rs_kv, rs_q = ops.rs_q;      // row strides (elements)
  const int Tq = ops.Tq;
  const int qoff = ops.qoff0 + head * ops.hstride, koff = ops.koff0 + head * ops.hstride,
            voff = ops.voff0 + head * ops.hstride;
  const __nv_bfloat16* base_hi = ops.kv_hi + (int64_t)b * T * rs;
  const __nv_bfloat16* base_lo = ops.kv_lo + (int64_t)b * T * rs;
  const __nv_bfloat16* qbase_hi = ops.q_hi + (int64_t)b * Tq * rs_q;
  const __nv_bfloat16* qbase_lo = ops.q_lo + (int64_t)b * Tq * rs_q;
  const float* base_f = ops.qkv + (int64_t)b * T * rs;
  const float* qbase_f = ops.qkv + (int64_t)b * Tq * rs_q;

  // ---- stage loader: 4 plane tiles x KT rows x (DP/8) 16-byte chunks ------------------------
  // F32IN: the K and V tiles as 2 KT fp32 rows (K's, then V's; row stride LD floats, so each tile lies over
  // its hi/lo plane pair) of DP/4 16-byte chunks, split in place after the copy.  Thread chunk slot u is column
  // chunk threadIdx.x % FCW of row threadIdx.x / FCW + u * 256 / FCW.  When FCW > FCPR the slots past DP are
  // idle; the chunks in [D, DP) are zero-filled like the keys past T.
  auto f32_chunk = [&](int u, int& tensor, int& key, int& c4) {
    const int row = threadIdx.x / FCW + u * (256 / FCW);
    tensor = u * (256 / FCW) >= KT;       // 0: K, 1: V
    key = row - tensor * KT;
    c4 = threadIdx.x % FCW * 4;
  };
  const bool f32_slot = FCW == FCPR || threadIdx.x % FCW < FCPR;   // F32IN: this thread's slots hold chunks
  auto load_tile = [&](int stage, int k0) {
    constexpr int CPR = DP / 8;           // chunks per row
    constexpr int N = 4 * KT * CPR;
    __nv_bfloat16* sbase = sm + stage * 4 * TILE;
    if constexpr (F32IN) {
      // padded grids issue their copies from a rolled loop: unrolled, every slot's clamped source address and
      // predicates would be hoisted and held across the key loop
#pragma unroll (D == DP ? FN : 1)
      for (int u = 0; u < FN; ++u) {
        int tensor, key, c4;
        f32_chunk(u, tensor, key, c4);
        if (!f32_slot) continue;
        const int kk = k0 + key;
        const bool col_ok = D == DP || c4 < D;
        const bool ok = kk < T && col_ok;
        const float* src = base_f + (int64_t)(ok ? kk : 0) * rs + (tensor ? voff : koff) + (col_ok ? c4 : 0);
        cp_async16(smem_u32(reinterpret_cast<float*>(sbase + tensor * 2 * TILE) + key * LD + c4), src, ok ? 16 : 0);
      }
    } else {
      for (int i = threadIdx.x; i < N; i += 256) {
        const int plane = i / (KT * CPR), rem = i % (KT * CPR);
        const int key = rem / CPR, ch = rem % CPR;
        const int kk = k0 + key;
        const bool col_ok = D == DP || ch < D / 8;
        const bool ok = kk < T && col_ok;
        const __nv_bfloat16* src = ((plane & 1) ? base_lo : base_hi) + (int64_t)(ok ? kk : 0) * rs +
                                   ((plane < 2) ? koff : voff) + (col_ok ? ch : 0) * 8;
        cp_async16(smem_u32(sbase + plane * TILE + key * LD + ch * 8), src, ok ? 16 : 0);
      }
    }
  };

  // ---- Q fragments for this warp's 16 rows (registers, both planes) ----------------------------
  const int q0 = blockIdx.x * 128 + warp * 16;
  uint32_t qh[QS ? 1 : KS][4], ql[QS ? 1 : KS][4];
  if constexpr (QS) {                     // 128 rows x DP/8 16-byte chunks per plane, zero-filled past Tq and D
    constexpr int CPR = DP / 8;
    __nv_bfloat16* qs = sm + 2 * 4 * TILE;
    if constexpr (F32IN) {                // scaled and split on the way: 128 rows x DP/4 float4
      for (int i = threadIdx.x; i < 128 * FCPR; i += 256) {
        const int row = i / FCPR, c4 = i % FCPR * 4;
        const int qr = blockIdx.x * 128 + row;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (qr < Tq && (D == DP || c4 < D)) v = ld_f4(qbase_f + (int64_t)qr * rs_q + qoff + c4);
        v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
        uint2 h, l;
        split4(v, h, l);
        *reinterpret_cast<uint2*>(qs + row * LD + c4) = h;
        *reinterpret_cast<uint2*>(qs + 128 * LD + row * LD + c4) = l;
      }
    } else {
      for (int i = threadIdx.x; i < 2 * 128 * CPR; i += 256) {
        const int plane = i / (128 * CPR), rem = i % (128 * CPR);
        const int row = rem / CPR, ch = rem % CPR;
        const int qr = blockIdx.x * 128 + row;
        const bool col_ok = D == DP || ch < D / 8;
        const bool ok = qr < Tq && col_ok;
        const __nv_bfloat16* src = (plane ? qbase_lo : qbase_hi) + (int64_t)(ok ? qr : 0) * rs_q + qoff +
                                   (col_ok ? ch : 0) * 8;
        cp_async16(smem_u32(qs + plane * 128 * LD + row * LD + ch * 8), src, ok ? 16 : 0);
      }
    }
  } else
#pragma unroll
  for (int ks = 0; ks < KS; ++ks)
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2)
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) {
        const int qr = q0 + g + r2 * 8;
        uint32_t vh = 0, vl = 0;
        if ((D == DP || ks * 16 + h2 * 8 < D) && qr < Tq) {
          const int64_t o = qr * rs_q + qoff + ks * 16 + h2 * 8 + 2 * t;
          if constexpr (F32IN) {
            const float2 v = *reinterpret_cast<const float2*>(qbase_f + o);
            split2x(v.x * scale, v.y * scale, vh, vl);
          } else {
            vh = *reinterpret_cast<const uint32_t*>(qbase_hi + o);
            vl = *reinterpret_cast<const uint32_t*>(qbase_lo + o);
          }
        }
        qh[ks][h2 * 2 + r2] = vh;
        ql[ks][h2 * 2 + r2] = vl;
      }

  float o[DP / 8][4];
#pragma unroll
  for (int j = 0; j < DP / 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  auto softmax_exp = [](float x) {
    if constexpr (F32IN) return expf(x);
    else return ex2_approx(x);
  };

  const int n_tiles = (T + KT - 1) / KT;
  load_tile(0, 0);
  cp_commit();
  for (int it = 0; it < n_tiles; ++it) {
    const int stage = it & 1;
    if (it + 1 < n_tiles) load_tile(stage ^ 1, (it + 1) * KT);
    cp_commit();
    cp_wait<1>();
    if constexpr (F32IN) {
      // each thread splits the chunks its own copies brought in (visible to it after the wait); the planes
      // overwrite the fp32 rows, so every thread has read its chunks before any plane is written.  The padded
      // chunk grids split K, then V (one more barrier): the padding's predicates and the idle slots keep more
      // registers live, and holding half the chunks keeps those instances from spilling.
      constexpr int NP = (D != DP || FCW != FCPR) ? 2 : 1;
      __nv_bfloat16* sbase = sm + stage * 4 * TILE;
#pragma unroll
      for (int pass = 0; pass < NP; ++pass) {
        float4 raw[FN / NP];
#pragma unroll
        for (int w = 0; w < FN / NP; ++w) {
          int tensor, key, c4;
          f32_chunk(pass * (FN / NP) + w, tensor, key, c4);
          if (f32_slot) raw[w] = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(sbase + tensor * 2 * TILE) + key * LD + c4);
        }
        __syncthreads();
#pragma unroll
        for (int w = 0; w < FN / NP; ++w) {
          int tensor, key, c4;
          f32_chunk(pass * (FN / NP) + w, tensor, key, c4);
          if (!f32_slot) continue;
          float4 v = raw[w];
          if (tensor == 0) { v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale; }
          uint2 h, l;
          split4(v, h, l);
          *reinterpret_cast<uint2*>(sbase + tensor * 2 * TILE + key * LD + c4) = h;
          *reinterpret_cast<uint2*>(sbase + (tensor * 2 + 1) * TILE + key * LD + c4) = l;
        }
      }
    }
    __syncthreads();
    const __nv_bfloat16* Kh = sm + stage * 4 * TILE;
    const uint32_t kh_a = smem_u32(Kh), kl_a = kh_a + TILE * 2, vh_a = kh_a + 2 * TILE * 2, vl_a = kh_a + 3 * TILE * 2;
    const int k0 = it * KT;

    // ---- S = Q K^T : per 8-key n-tile j, ldmatrix.x4 covers two k-steps (b0,b1 | b0,b1) -----------
    float s[KT / 8][4];
    if constexpr (QS) {
      // same products in the same order per s[j]; the k-step pair is the outer loop so that only its
      // Q fragments are live.  A fragment by ldmatrix.x4: matrix m = lane>>3 is (rows 8*(m&1).., k 8*(m>>1)..)
      const uint32_t qh_a = smem_u32(sm + 2 * 4 * TILE), ql_a = qh_a + 128 * LD * 2;
      const uint32_t qrow = (uint32_t)(((warp * 16 + (lane & 15)) * LD + (lane >> 4) * 8) * 2);
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
          const uint32_t roff = (uint32_t)(((j * 8 + (lane & 7)) * LD + (lane >> 3) * 8) * 2);
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
      if constexpr (KS % 2 == 1) {        // odd KS: the last k-step alone; K matrices 2, 3 re-read 0, 1
        constexpr int k2 = KS / 2;
        uint32_t ah0[4], al0[4];
        ldsm_x4(qh_a + qrow + k2 * 64, ah0[0], ah0[1], ah0[2], ah0[3]);
        ldsm_x4(ql_a + qrow + k2 * 64, al0[0], al0[1], al0[2], al0[3]);
#pragma unroll
        for (int j = 0; j < KT / 8; ++j) {
          const uint32_t r16 = (uint32_t)(((j * 8 + (lane & 7)) * LD + ((lane >> 3) & 1) * 8) * 2) + k2 * 64;
          uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
          ldsm_x4(kh_a + r16, h0, h1, h2, h3);
          ldsm_x4(kl_a + r16, l0, l1, l2, l3);
          mma16816(s[j], al0, h0, h1);
          mma16816(s[j], ah0, l0, l1);
          mma16816(s[j], ah0, h0, h1);
        }
      }
    } else
#pragma unroll
    for (int j = 0; j < KT / 8; ++j) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
      // lane -> row address: matrices (m = lane>>3): d offset m*8 within a 32-wide d span, row = key j*8 + (lane&7)
      const uint32_t roff = (uint32_t)(((j * 8 + (lane & 7)) * LD + (lane >> 3) * 8) * 2);
#pragma unroll
      for (int k2 = 0; k2 < (KS + 1) / 2; ++k2) {
        uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
        if (2 * k2 + 1 < KS) {
          ldsm_x4(kh_a + roff + k2 * 64, h0, h1, h2, h3);
          ldsm_x4(kl_a + roff + k2 * 64, l0, l1, l2, l3);
        } else {   // odd KS, last k-step: only matrices 0,1 are in range; re-read them for 2,3 (unused)
          const uint32_t r16 = (uint32_t)(((j * 8 + (lane & 7)) * LD + ((lane >> 3) & 1) * 8) * 2) + k2 * 64;
          ldsm_x4(kh_a + r16, h0, h1, h2, h3);
          ldsm_x4(kl_a + r16, l0, l1, l2, l3);
        }
        mma16816(s[j], ql[2 * k2], h0, h1);
        mma16816(s[j], qh[2 * k2], l0, l1);
        mma16816(s[j], qh[2 * k2], h0, h1);
        if (2 * k2 + 1 < KS) {
          mma16816(s[j], ql[2 * k2 + 1], h2, h3);
          mma16816(s[j], qh[2 * k2 + 1], l2, l3);
          mma16816(s[j], qh[2 * k2 + 1], h2, h3);
        }
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
      float ot0[4] = {0.f, 0.f, 0.f, 0.f}, ot1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk) {
        // matrix m = lane>>3: key block (m&1)*8, d block (m>>1)*8 ; row within = lane&7 (a key)
        const uint32_t voff2 = (uint32_t)(((kk * 16 + (lane >> 3 & 1) * 8 + (lane & 7)) * LD + jd2 * 16 + (lane >> 4) * 8) * 2);
        uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
        ldsm_x4_t(vh_a + voff2, h0, h1, h2, h3);
        ldsm_x4_t(vl_a + voff2, l0, l1, l2, l3);
        mma16816(ot0, pl[kk], h0, h1);
        mma16816(ot0, ph[kk], l0, l1);
        mma16816(ot0, ph[kk], h0, h1);
        if (2 * jd2 + 1 < D / 8) {        // the n-tile [D, DP) is zero
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

  // ---- normalise and store -------------------------------------------------------------------
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    const int qr = q0 + g + r2 * 8;
    if (qr >= Tq) continue;
    const float inv = 1.0f / l_run[r2];
    const int64_t off = ((int64_t)b * Tq + qr) * C + head * D + 2 * t;
#pragma unroll
    for (int jd = 0; jd < D / 8; ++jd) {
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

// one head_dim's launch: dynamic shared memory (set once per device), grid over (query tiles, batch x heads)
template <int D, bool F32IN>
int launch_attention_d(const AttnOperands& ops, dim3 grid, int T, int C, int heads, float scale, float* out_f32,
                       __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, cudaStream_t s) {
  constexpr int DP = (D + 15) / 16 * 16;
  const size_t smem = (size_t)2 * 4 * 64 * (DP + 8) * 2 + (DP > 64 ? (size_t)2 * 128 * (DP + 8) * 2 : 0);
  static DeviceOnce cfgd;
  if (cfgd.need()) {
    BBDM_CUDA_CHECK(cudaFuncSetAttribute(attention_split_kernel<D, F32IN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
    cfgd.mark();
  }
  attention_split_kernel<D, F32IN><<<grid, 256, smem, s>>>(ops, T, C, heads, scale, out_f32, out_hi, out_lo);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

// The head sizes that are not multiples of 16 (attention_split_padded.cu).  They are compiled in a translation unit
// of their own: instantiated next to them, the D = 128 kernels compiled to different code and ran 5% slower.
template <bool F32IN>
int launch_attention_padded(const char* who, int D, const AttnOperands& ops, dim3 grid, int T, int C, int heads,
                            float scale, float* out_f32, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, cudaStream_t s);

// Head sizes 136 to 256 (attention_split_wide.cu): 64-query CTAs over 32-key tiles, so that the stages and the output
// fragment fit.  Any other head_dim fails here with BBDM_E_UNSUPPORTED.
template <bool F32IN>
int launch_attention_wide(const char* who, int D, const AttnOperands& ops, dim3 grid, int T, int C, int heads,
                          float scale, float* out_f32, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, cudaStream_t s);

}  // namespace bbdm
