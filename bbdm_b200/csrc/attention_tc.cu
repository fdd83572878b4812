// FlashAttention-style, warp-specialised attention core on Hopper wgmma tensor cores (sm_90a).
// AttentionBlock of the reference: openaimodel.py:281-413 (softmax((q s)(k s)^T) v, s = D^-1/4).
//
//   * one CTA = 128 queries of one (batch, head); KV tiles of 64 keys; head_dim D = 64 or 128.
//   * operands are the split-bf16 planes the qkv 1x1 conv wrote (qkv_hi/qkv_lo [B,T,3C]);
//     TMA (3-D tiled maps, SWIZZLE_128B) stages Q once and K/V tiles through a ring (4 stages at D = 64,
//     2 at D = 128).  A SWIZZLE_128B box is 64 bf16 wide, so every Q/K/V tile is D/64 column panels
//     of 64, each loaded by its own TMA copy.
//   * warps 0-7 = two consumer warpgroups, 64 query rows each; warp 8 = TMA producer.  Both warpgroups
//     walk every KV tile, so the tensor core works for one while the other runs its softmax.
//   * S_j = Q K_j^T : m64n64k16 wgmma, A = Q (K-major, shared), B = K_j (K-major); the D/16 k-steps
//                     walk the panels in turn                                              -> registers
//     O_j = P_j V_j : m64n64k16 wgmma, A = P_j from registers (the S fragment re-packed to bf16),
//                     B = V_j as an MN-major operand, one m64n64 product per V panel       -> registers
//     every product is split-bf16 x3 (lo.hi + hi.lo + hi.hi, fp32 accumulate).
//   * each O_j panel starts from a zero accumulator and is folded into the fp32 running output with
//     round-to-nearest adds and the online-softmax rescale (the tensor core's own accumulate truncates).
//     At D = 128 the two panels share one 32-float scratch next to the 64-float running output.  That is
//     more than the 168 registers a thread gets when 9 warps share an SM (warps are allocated in groups
//     of 4), so the D = 128 CTA has a full producer warpgroup that gives up registers with setmaxnreg
//     (24 each) and the consumers take 240.
//   * all mbarrier waits are watchdogged (device fault word, no GPU hang); fault codes 0xB0/B1/B2 at
//     D = 64, 0xB4/B5/B6 at D = 128 (Q load / ring slot free / ring slot full, low bits = KV tile).
#include "tc_common.cuh"

namespace bbdm {

constexpr int AT_PANEL = 64;              // bf16 columns per SWIZZLE_128B box
constexpr int AT_BQ = 128;                // queries per CTA
constexpr int AT_BK = 64;                 // keys per tile
constexpr uint32_t AT_QP_BYTES = AT_BQ * AT_PANEL * 2;    // 16 KiB per Q panel
constexpr uint32_t AT_KVP_BYTES = AT_BK * AT_PANEL * 2;   // 8 KiB per K / V panel

template <int D>
struct AtCfg {
  static constexpr int PANELS = D / AT_PANEL;
  static constexpr int STAGES = D == 64 ? 4 : 2;
  static constexpr uint32_t Q_BYTES = AT_BQ * D * 2;        // per plane
  static constexpr uint32_t KV_BYTES = AT_BK * D * 2;       // per plane tile
  static constexpr uint32_t STAGE_BYTES = 4 * KV_BYTES;     // K_hi K_lo V_hi V_lo
  static constexpr uint32_t SMEM = 2 * Q_BYTES + STAGES * STAGE_BYTES + 1024;
  static constexpr unsigned long long FAULT = D == 64 ? 0xB0000000ull : 0xB4000000ull;
  // D = 64: warps 0-7 consume, warp 8 produces.  D = 128: warps 8-11 form a producer warpgroup that hands
  // registers to the consumers (setmaxnreg), since 288 threads cap every thread at 168 registers.
  static constexpr int THREADS = D == 64 ? 288 : 384;
};
// D = 128 register split (65,536 per SM): 128 x 24 for the producer warpgroup + 256 x 240 for the consumers
constexpr int AT_PRODUCER_REGS = 24, AT_CONSUMER_REGS = 240;
static_assert(128 * AT_PRODUCER_REGS + 256 * AT_CONSUMER_REGS <= 65536, "attention_tc<128>: register split");
static_assert(AtCfg<128>::SMEM <= 227 * 1024, "attention_tc<128>: shared memory");

struct AttnParams {
  int T, C, heads, order;
  float scale_log2;
  float* out_f32; __nv_bfloat16* out_hi; __nv_bfloat16* out_lo;
  unsigned long long* fault;
};

template <int D>
__global__ void __launch_bounds__(AtCfg<D>::THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap map_q_hi, const __grid_constant__ CUtensorMap map_q_lo,
                    const __grid_constant__ CUtensorMap map_kv_hi, const __grid_constant__ CUtensorMap map_kv_lo,
                    const AttnParams p) {
  using Cfg = AtCfg<D>;
  constexpr int STAGES = Cfg::STAGES, PANELS = Cfg::PANELS;
  constexpr uint32_t Q_BYTES = Cfg::Q_BYTES, KV_BYTES = Cfg::KV_BYTES, STAGE_BYTES = Cfg::STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bars[1 + 2 * STAGES];
  __shared__ int abort_s;

  // each plane tile is PANELS column panels of 64, stored one after the other (Q: 16 KiB, K/V: 8 KiB each)
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_hi_a = base, q_lo_a = base + Q_BYTES;
  const uint32_t kv_a = base + 2 * Q_BYTES;                          // [stage][Kh Kl Vh Vl]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar_q = smem_u32(&bars[0]);
  const uint32_t bar_kvf = smem_u32(&bars[1]);                        // [STAGES]
  const uint32_t bar_kve = smem_u32(&bars[1 + STAGES]);               // [STAGES]
  volatile int* abort_flag = &abort_s;

  if (threadIdx.x == 0) {
    abort_s = 0;
    mbar_init(bar_q, 1);
    for (int i = 0; i < STAGES; ++i) { mbar_init(bar_kvf + 8 * i, 1); mbar_init(bar_kve + 8 * i, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int bh = blockIdx.y, b = bh / p.heads, head = bh % p.heads;
  int qoff, koff, voff;
  if (p.order == 0) { qoff = head * 3 * D; koff = qoff + D; voff = qoff + 2 * D; }
  else { qoff = head * D; koff = p.C + head * D; voff = 2 * p.C + head * D; }
  const int q0 = blockIdx.x * AT_BQ;
  const int n_tiles = (p.T + AT_BK - 1) / AT_BK;

  if (D == 64 ? warp == 8 : warp >= 8) {
    // ================================ TMA producer ============================================
    if constexpr (D != 64) setmaxnreg_dec<AT_PRODUCER_REGS>();
    if (warp == 8 && lane == 0) {
      mbar_expect_tx(bar_q, 2 * Q_BYTES);
#pragma unroll
      for (int pn = 0; pn < PANELS; ++pn)
        tma_load_3d(q_hi_a + pn * AT_QP_BYTES, &map_q_hi, bar_q, qoff + pn * AT_PANEL, q0, b);
#pragma unroll
      for (int pn = 0; pn < PANELS; ++pn)
        tma_load_3d(q_lo_a + pn * AT_QP_BYTES, &map_q_lo, bar_q, qoff + pn * AT_PANEL, q0, b);
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j % STAGES, u = j / STAGES;
        mbar_wait(bar_kve + 8 * st, (u & 1) ^ 1, abort_flag, p.fault, (Cfg::FAULT + 0x1000000ull) | (unsigned)j);
        const uint32_t sb = kv_a + st * STAGE_BYTES, full = bar_kvf + 8 * st;
        mbar_expect_tx(full, STAGE_BYTES);
#pragma unroll
        for (int pn = 0; pn < PANELS; ++pn)
          tma_load_3d(sb + pn * AT_KVP_BYTES, &map_kv_hi, full, koff + pn * AT_PANEL, j * AT_BK, b);
#pragma unroll
        for (int pn = 0; pn < PANELS; ++pn)
          tma_load_3d(sb + KV_BYTES + pn * AT_KVP_BYTES, &map_kv_lo, full, koff + pn * AT_PANEL, j * AT_BK, b);
#pragma unroll
        for (int pn = 0; pn < PANELS; ++pn)
          tma_load_3d(sb + 2 * KV_BYTES + pn * AT_KVP_BYTES, &map_kv_hi, full, voff + pn * AT_PANEL, j * AT_BK, b);
#pragma unroll
        for (int pn = 0; pn < PANELS; ++pn)
          tma_load_3d(sb + 3 * KV_BYTES + pn * AT_KVP_BYTES, &map_kv_lo, full, voff + pn * AT_PANEL, j * AT_BK, b);
      }
    }
    return;
  }

  // ================================ consumer warpgroups: S, softmax, PV, epilogue ===============
  // thread holds rows r0 = 16 * (warp % 4) + lane / 4 and r0 + 8 of its warpgroup's 64 queries,
  // columns 8 * (i >> 2) + 2 * (lane % 4) + (i & 1) of every m64n64 fragment (tc_common.cuh);
  // o_reg[32 * pn + i] is that fragment entry of output panel pn
  if constexpr (D != 64) setmaxnreg_inc<AT_CONSUMER_REGS>();
  const int wg = warp >> 2;
  const uint32_t q_off = (uint32_t)wg * 64 * 128;
  const uint64_t dq_hi = make_sw128_desc(q_hi_a + q_off), dq_lo = make_sw128_desc(q_lo_a + q_off);
  float o_reg[32 * PANELS];
#pragma unroll
  for (int i = 0; i < 32 * PANELS; ++i) o_reg[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: this thread's share of the row sum

  mbar_wait(bar_q, 0, abort_flag, p.fault, Cfg::FAULT);
  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % STAGES, u = j / STAGES;
    const int k0 = j * AT_BK;
    mbar_wait(bar_kvf + 8 * st, u & 1, abort_flag, p.fault, (Cfg::FAULT + 0x2000000ull) | (unsigned)j);
    const uint32_t sb = kv_a + st * STAGE_BYTES;
    const uint64_t dk_hi = make_sw128_desc(sb), dk_lo = make_sw128_desc(sb + KV_BYTES);
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k) {
      // k-step k: panel k / 4 (Q panels 16 KiB apart, K panels 8 KiB), 32 B into the panel's swizzle atom
      const uint64_t qo = (uint64_t)(((k >> 2) * AT_QP_BYTES + (k & 3) * 32) >> 4);
      const uint64_t ko = (uint64_t)(((k >> 2) * AT_KVP_BYTES + (k & 3) * 32) >> 4);
      wgmma_n64_bf16<0>(s, dq_lo + qo, dk_hi + ko, 1u);
      wgmma_n64_bf16<0>(s, dq_hi + qo, dk_lo + ko, 1u);
      wgmma_n64_bf16<0>(s, dq_hi + qo, dk_hi + ko, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<32>(s);

    // online softmax over the two rows (a row is spread over the 4 lanes of a quad)
    float corr[2];
#pragma unroll
    for (int ri = 0; ri < 2; ++ri) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        if (((i >> 1) & 1) != ri) continue;
        const int key = k0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        if (key < p.T) mx = fmaxf(mx, s[i] * p.scale_log2);
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[ri], mx);
      corr[ri] = (m_run[ri] == -INFINITY) ? 0.f : ex2_approx(m_run[ri] - m_new);
      m_run[ri] = m_new;
      float rs = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        if (((i >> 1) & 1) != ri) continue;
        const int key = k0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        s[i] = (key < p.T) ? ex2_approx(fmaf(s[i], p.scale_log2, -m_new)) : 0.f;
        rs += s[i];
      }
      l_run[ri] = l_run[ri] * corr[ri] + rs;
    }

    // P_j as register A fragments: k16 slice kk = columns 16kk .. 16kk+15 = fragment entries 8kk .. 8kk+7
    uint32_t ph[16], pl[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) split2x(s[2 * i], s[2 * i + 1], ph[i], pl[i]);
    // one m64n64 product per V panel, each from a zero accumulator, folded before the next starts
#pragma unroll
    for (int pn = 0; pn < PANELS; ++pn) {
      float o_j[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) o_j[i] = 0.f;
      const uint32_t vb = sb + 2 * KV_BYTES + pn * AT_KVP_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < AT_BK / 16; ++k) {
        const uint64_t dv_hi = make_sw128_desc(vb + k * 16 * 128), dv_lo = make_sw128_desc(vb + KV_BYTES + k * 16 * 128);
        wgmma_rs_n64_bf16<1>(o_j, pl + 4 * k, dv_hi, 1u);
        wgmma_rs_n64_bf16<1>(o_j, ph + 4 * k, dv_lo, 1u);
        wgmma_rs_n64_bf16<1>(o_j, ph + 4 * k, dv_hi, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence<32>(o_j);
      if (pn == PANELS - 1) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_kve + 8 * st);      // K_j / V_j slot free
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) o_reg[32 * pn + i] = o_reg[32 * pn + i] * corr[(i >> 1) & 1] + o_j[i];
    }
  }

  // ---- epilogue: full row sums over the quad, normalise, store ---------------------------------
#pragma unroll
  for (int ri = 0; ri < 2; ++ri) {
    float l = l_run[ri];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int qr = q0 + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * ri;
    if (qr < p.T) {
      const int64_t off = ((int64_t)b * p.T + qr) * p.C + head * D + 2 * (lane & 3);
      // column 8 * jj + 2 * (lane % 4) = panel jj / 8, fragment entries 4 * (jj % 8) + 2 * ri (+1)
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj) {
        const float2 v = make_float2(o_reg[4 * jj + 2 * ri] * inv, o_reg[4 * jj + 2 * ri + 1] * inv);
        if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + off + 8 * jj) = v;
        if (p.out_hi) {
          uint32_t h, l2;
          split2x(v.x, v.y, h, l2);
          *reinterpret_cast<uint32_t*>(p.out_hi + off + 8 * jj) = h;
          *reinterpret_cast<uint32_t*>(p.out_lo + off + 8 * jj) = l2;
        }
      }
    }
  }
}

// qkv plane [B][T][3C] bf16 -> 3-D map (3C, T, B), box (64, rows, 1), SWIZZLE_128B
static int make_qkv_map(CUtensorMap* m, const void* ptr, int B, int T, int C3, int rows) {
  EncodeTiledFn enc = get_encode();
  BBDM_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[3] = {(cuuint64_t)C3, (cuuint64_t)T, (cuuint64_t)B};
  cuuint64_t strides[2] = {(cuuint64_t)C3 * 2, (cuuint64_t)T * C3 * 2};
  cuuint32_t box[3] = {(cuuint32_t)AT_PANEL, (cuuint32_t)rows, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  BBDM_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(qkv) failed: %d", (int)r);
  return BBDM_OK;
}

template <int D>
static int launch_attention_tc(const CUtensorMap* maps, const AttnParams& p, int B, int T, int heads, cudaStream_t s) {
  constexpr uint32_t smem = AtCfg<D>::SMEM;
  static DeviceOnce configured;
  if (configured.need()) {
    BBDM_CUDA_CHECK(cudaFuncSetAttribute(attention_tc_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured.mark();
  }
  dim3 grid((T + AT_BQ - 1) / AT_BQ, B * heads);
  attention_tc_kernel<D><<<grid, AtCfg<D>::THREADS, smem, s>>>(maps[0], maps[1], maps[2], maps[3], p);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // namespace bbdm

using namespace bbdm;

// head_dim 64 (the template UNets) or 128; other head dims are served by bbdm_attention_split.
extern "C" int bbdm_attention_tc(const void* qkv_hi, const void* qkv_lo, int B, int T, int C, int heads, int order,
                                 float* out_f32, void* out_hi, void* out_lo, void* stream) {
  BBDM_REQUIRE(qkv_hi && qkv_lo && (out_f32 || (out_hi && out_lo)), "attention_tc: null pointer");
  BBDM_REQUIRE((out_hi == nullptr) == (out_lo == nullptr), "attention_tc: hi/lo must come in pairs");
  BBDM_REQUIRE(B > 0 && T > 0 && heads > 0 && C % heads == 0 && (order == 0 || order == 1), "attention_tc: bad shape");
  const int D = C / heads;
  if (D != 64 && D != 128) {
    set_error("attention_tc: head_dim %d not supported (64, 128)", D);
    return BBDM_E_UNSUPPORTED;
  }
  BBDM_REQUIRE((int64_t)B * heads <= 65535, "attention_tc: B*heads too large");
  CUtensorMap maps[4];
  int rc;
  if ((rc = make_qkv_map(&maps[0], qkv_hi, B, T, 3 * C, AT_BQ))) return rc;
  if ((rc = make_qkv_map(&maps[1], qkv_lo, B, T, 3 * C, AT_BQ))) return rc;
  if ((rc = make_qkv_map(&maps[2], qkv_hi, B, T, 3 * C, AT_BK))) return rc;
  if ((rc = make_qkv_map(&maps[3], qkv_lo, B, T, 3 * C, AT_BK))) return rc;
  AttnParams p;
  p.T = T; p.C = C; p.heads = heads; p.order = order;
  p.scale_log2 = (float)(1.4426950408889634 / sqrt((double)D));
  p.out_f32 = out_f32; p.out_hi = (__nv_bfloat16*)out_hi; p.out_lo = (__nv_bfloat16*)out_lo;
  p.fault = device_fault_ptr();
  BBDM_REQUIRE(p.fault != nullptr, "attention_tc: device fault word unavailable");
  if (D == 64) return launch_attention_tc<64>(maps, p, B, T, heads, (cudaStream_t)stream);
  return launch_attention_tc<128>(maps, p, B, T, heads, (cudaStream_t)stream);
}
