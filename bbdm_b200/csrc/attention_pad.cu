// Repack of attention heads whose width d is not a multiple of 8 (bbdm_attention_pad_heads / _unpad_heads).
//
// The attention kernels take head widths that are multiples of 8.  A head of width d runs on them at dp = d rounded up
// to 8: every group of d consecutive columns (one head's q, k or v) is laid out dp columns wide with zeros past d.
// The zero columns add exactly 0 to q.k and give zero output columns, so the kernels' results at dp are those at d up
// to the softmax scale, which they take from dp; the caller folds (dp/d)^(1/4) into q and k through the per-tensor
// scales here.  Memory-bound element-wise passes: no shared memory, no host synchronisation, no allocation.
#include <algorithm>

#include "common.cuh"

namespace bbdm {
namespace {

constexpr int kThreads = 256;

struct HeadGroups {
  int heads, tensors, d, dp, order;
  float scale[3];
};

// Scale of column group g: the groups of a row are tensors x heads; order 0 (the legacy qkv layout) interleaves the
// tensors per head, order 1 puts all heads of one tensor first
__device__ __forceinline__ float group_scale(const HeadGroups& s, int g) {
  const int t = s.order ? g / s.heads : g % s.tensors;
  return t == 0 ? s.scale[0] : t == 1 ? s.scale[1] : s.scale[2];     // selects: no local-memory copy of the array
}

// [rows, G*d] -> [rows, G*dp]; each thread writes 4 consecutive columns (dp % 8 == 0: never across two groups)
__global__ void __launch_bounds__(kThreads)
pad_heads_kernel(const float* __restrict__ src, int64_t rows, HeadGroups s, float* __restrict__ out_f32,
                 __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo) {
  const int G = s.heads * s.tensors;
  const int64_t quads = (int64_t)G * s.dp / 4;
  const int64_t n = rows * quads;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / quads;
    const int j = (int)(i - r * quads) * 4;
    const int g = j / s.dp, c = j - g * s.dp;
    const float sc = group_scale(s, g);
    const float* in = src + r * G * s.d + (int64_t)g * s.d;
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = c + k < s.d ? __fmul_rn(in[c + k], sc) : 0.f;   // no FMA into the split
    const int64_t o = r * G * s.dp + j;
    if (out_f32) st_f4(out_f32 + o, make_float4(v[0], v[1], v[2], v[3]));
    if (out_hi) {
      uint2 hi, lo;
      split4(make_float4(v[0], v[1], v[2], v[3]), hi, lo);
      *reinterpret_cast<uint2*>(out_hi + o) = hi;
      *reinterpret_cast<uint2*>(out_lo + o) = lo;
    }
  }
}

// [rows, G*dp] -> [rows, G*d]
__global__ void __launch_bounds__(kThreads)
unpad_heads_kernel(const float* __restrict__ src, int64_t rows, HeadGroups s, float* __restrict__ out_f32,
                   __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo) {
  const int G = s.heads * s.tensors;
  const int64_t cols = (int64_t)G * s.d;
  const int64_t n = rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cols;
    const int j = (int)(i - r * cols);
    const int g = j / s.d, c = j - g * s.d;
    const float v = __fmul_rn(src[r * G * s.dp + (int64_t)g * s.dp + c], group_scale(s, g));
    if (out_f32) out_f32[i] = v;
    if (out_hi) split_bf16(v, out_hi[i], out_lo[i]);
  }
}

int launch_repack(bool pad, const float* src, int64_t rows, int heads, int tensors, int d, int order, float scale0,
                  float scale1, float scale2, float* out_f32, void* out_hi, void* out_lo, void* stream) {
  const char* name = pad ? "bbdm_attention_pad_heads" : "bbdm_attention_unpad_heads";
  BBDM_REQUIRE(src && rows >= 0 && heads >= 1 && tensors >= 1 && tensors <= 3 && d >= 1 && (order == 0 || order == 1),
               "%s: src, rows >= 0, heads >= 1, tensors 1..3, d >= 1, order 0 or 1", name);
  BBDM_REQUIRE((out_f32 || out_hi) && !out_hi == !out_lo, "%s: out_f32 and/or both planes", name);
  BBDM_REQUIRE(!(pad && ((reinterpret_cast<uintptr_t>(out_f32) & 15) || (reinterpret_cast<uintptr_t>(out_hi) & 7) ||
                          (reinterpret_cast<uintptr_t>(out_lo) & 7))),
               "%s: outputs 16-byte (fp32) and 8-byte (planes) aligned", name);
  BBDM_REQUIRE((int64_t)heads * tensors * (d + 7) <= (1 << 30), "%s: row too wide", name);
  HeadGroups s{heads, tensors, d, (d + 7) / 8 * 8, order, {scale0, scale1, scale2}};
  const int64_t n = rows * heads * tensors * (pad ? s.dp / 4 : d);
  if (n == 0) return BBDM_OK;
  const int blocks = (int)std::min<int64_t>((n + kThreads - 1) / kThreads, (int64_t)num_sms() * 16);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto* hi = static_cast<__nv_bfloat16*>(out_hi);
  auto* lo = static_cast<__nv_bfloat16*>(out_lo);
  if (pad)
    pad_heads_kernel<<<blocks, kThreads, 0, st>>>(src, rows, s, out_f32, hi, lo);
  else
    unpad_heads_kernel<<<blocks, kThreads, 0, st>>>(src, rows, s, out_f32, hi, lo);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // namespace
}  // namespace bbdm

extern "C" int bbdm_attention_pad_heads(const float* src, int64_t rows, int heads, int tensors, int d, int order,
                                        float scale0, float scale1, float scale2, float* out_f32, void* out_hi,
                                        void* out_lo, void* stream) {
  return bbdm::launch_repack(true, src, rows, heads, tensors, d, order, scale0, scale1, scale2, out_f32, out_hi,
                             out_lo, stream);
}

extern "C" int bbdm_attention_unpad_heads(const float* src, int64_t rows, int heads, int tensors, int d, int order,
                                          float scale0, float scale1, float scale2, float* out_f32, void* out_hi,
                                          void* out_lo, void* stream) {
  return bbdm::launch_repack(false, src, rows, heads, tensors, d, order, scale0, scale1, scale2, out_f32, out_hi,
                             out_lo, stream);
}
