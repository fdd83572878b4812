// The mma.sync attention core (attention_split.cuh) at the head sizes that are not multiples of 16: run at the next
// multiple of 16 with the columns past D zero-filled.
#include "attention_split.cuh"

namespace bbdm {

template <bool F32IN>
int launch_attention_padded(const char* who, int D, const AttnOperands& ops, dim3 grid, int T, int C, int heads,
                            float scale, float* out_f32, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, cudaStream_t s) {
#define BBDM_AL(DD) \
  case DD: return launch_attention_d<DD, F32IN>(ops, grid, T, C, heads, scale, out_f32, out_hi, out_lo, s);
  switch (D) {
    BBDM_ATTN_PADDED_HEAD_DIMS(BBDM_AL)
    default: return launch_attention_wide<F32IN>(who, D, ops, grid, T, C, heads, scale, out_f32, out_hi, out_lo, s);
  }
#undef BBDM_AL
}

template int launch_attention_padded<false>(const char*, int, const AttnOperands&, dim3, int, int, int, float, float*,
                                            __nv_bfloat16*, __nv_bfloat16*, cudaStream_t);
template int launch_attention_padded<true>(const char*, int, const AttnOperands&, dim3, int, int, int, float, float*,
                                           __nv_bfloat16*, __nv_bfloat16*, cudaStream_t);

}  // namespace bbdm
