// Entry points of the mma.sync attention core (attention_split.cuh): head sizes 16, 32, 64 and 128 are instantiated
// here, the other multiples of 8 up to 128 in attention_split_padded.cu and the multiples of 8 from 136 to 256 in
// attention_split_wide.cu.
#include "attention_split.cuh"

using namespace bbdm;

template <bool F32IN>
static int launch_attention(const char* who, const AttnOperands& ops, int B, int T, int C, int heads, float* out_f32,
                            void* out_hi, void* out_lo, void* stream) {
  const int D = C / heads;
  BBDM_REQUIRE((int64_t)B * heads <= 65535, "%s: B*heads too large", who);
  dim3 grid((ops.Tq + 127) / 128, B * heads);
  cudaStream_t s = (cudaStream_t)stream;
  // F32IN: the reference multiplies q and k by the python double 1/sqrt(sqrt(ch)) rounded to fp32.
  // Split planes: softmax((q s)(k s)) with s = D^-1/4  ==  2^(log2(e) * D^-1/2 * (q.k) - max)
  const float scale = F32IN ? (float)(1.0 / sqrt(sqrt((double)D))) : (float)(1.4426950408889634 / sqrt((double)D));
  __nv_bfloat16* oh = (__nv_bfloat16*)out_hi;
  __nv_bfloat16* ol = (__nv_bfloat16*)out_lo;
#define BBDM_AL(DD) \
  case DD: return launch_attention_d<DD, F32IN>(ops, grid, T, C, heads, scale, out_f32, oh, ol, s);
  switch (D) {
    BBDM_ATTN_POW2_HEAD_DIMS(BBDM_AL)
    default: return launch_attention_padded<F32IN>(who, D, ops, grid, T, C, heads, scale, out_f32, oh, ol, s);
  }
#undef BBDM_AL
}

// q, k and v of self-attention: [B][T][3C] rows in the channel order `order` (see include/bbdm_b200.h)
static AttnOperands self_attention_operands(int T, int C, int heads, int order) {
  const int D = C / heads;
  AttnOperands ops{};
  ops.rs_q = ops.rs_kv = 3 * (int64_t)C;
  ops.Tq = T;
  if (order == 0) { ops.hstride = 3 * D; ops.qoff0 = 0; ops.koff0 = D; ops.voff0 = 2 * D; }
  else { ops.hstride = D; ops.qoff0 = 0; ops.koff0 = C; ops.voff0 = 2 * C; }
  return ops;
}

extern "C" int bbdm_attention(const float* qkv, int B, int T, int C, int heads, int order,
                              float* out_f32, void* out_hi, void* out_lo, void* stream) {
  BBDM_REQUIRE(qkv && (out_f32 || (out_hi && out_lo)), "attention: null pointer");
  BBDM_REQUIRE((out_hi == nullptr) == (out_lo == nullptr), "attention: hi/lo must come in pairs");
  BBDM_REQUIRE(B > 0 && T > 0 && heads > 0 && C % heads == 0, "attention: bad shape");
  BBDM_REQUIRE(order == 0 || order == 1, "attention: order must be 0 (legacy) or 1");
  AttnOperands ops = self_attention_operands(T, C, heads, order);
  ops.qkv = qkv;
  return launch_attention<true>("attention", ops, B, T, C, heads, out_f32, out_hi, out_lo, stream);
}

extern "C" int bbdm_attention_split(const void* qkv_hi, const void* qkv_lo, int B, int T, int C, int heads,
                                    int order, float* out_f32, void* out_hi, void* out_lo, void* stream) {
  BBDM_REQUIRE(qkv_hi && qkv_lo && (out_f32 || (out_hi && out_lo)), "attention_split: null pointer");
  BBDM_REQUIRE((out_hi == nullptr) == (out_lo == nullptr), "attention_split: hi/lo must come in pairs");
  BBDM_REQUIRE(B > 0 && T > 0 && heads > 0 && C % heads == 0, "attention_split: bad shape");
  BBDM_REQUIRE(order == 0 || order == 1, "attention_split: order must be 0 (legacy) or 1");
  AttnOperands ops = self_attention_operands(T, C, heads, order);
  ops.q_hi = ops.kv_hi = (const __nv_bfloat16*)qkv_hi;
  ops.q_lo = ops.kv_lo = (const __nv_bfloat16*)qkv_lo;
  return launch_attention<false>("attention_split", ops, B, T, C, heads, out_f32, out_hi, out_lo, stream);
}

extern "C" int bbdm_attention_cross(const void* q_hi, const void* q_lo, const void* kv_hi, const void* kv_lo, int B,
                                    int Tq, int Tkv, int C, int heads, float* out_f32, void* out_hi, void* out_lo,
                                    void* stream) {
  BBDM_REQUIRE(q_hi && q_lo && kv_hi && kv_lo && (out_f32 || (out_hi && out_lo)), "attention_cross: null pointer");
  BBDM_REQUIRE((out_hi == nullptr) == (out_lo == nullptr), "attention_cross: hi/lo must come in pairs");
  BBDM_REQUIRE(B > 0 && Tq > 0 && Tkv > 0 && heads > 0 && C % heads == 0, "attention_cross: bad shape");
  AttnOperands ops{};
  ops.q_hi = (const __nv_bfloat16*)q_hi; ops.q_lo = (const __nv_bfloat16*)q_lo;
  ops.kv_hi = (const __nv_bfloat16*)kv_hi; ops.kv_lo = (const __nv_bfloat16*)kv_lo;
  ops.rs_q = C; ops.rs_kv = 2 * (int64_t)C;
  ops.Tq = Tq;
  ops.hstride = C / heads; ops.qoff0 = 0; ops.koff0 = 0; ops.voff0 = C;
  return launch_attention<false>("attention_split", ops, B, Tkv, C, heads, out_f32, out_hi, out_lo, stream);
}
